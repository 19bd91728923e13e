// dv_probe.cu -- libdivans_b200_probe.so: the product's arithmetic device functions as plain C entry points, for
// tests/test_gpu_arith.py.  TEST INFRASTRUCTURE: built by divans_b200/csrc/Makefile next to libdivans_b200.so, never
// linked into it.  It includes the product sources unchanged and calls their functions, not copies of them.
//
// Every entry point takes host arrays, allocates, copies, launches on device 0, copies back and frees, and returns a CUDA
// error code (0 = success).  Every buffer is sized by the caller or bounded here: a wrong result is a wrong number.
#include <stdio.h>
#include "dv_encode.cu"     // div_by_u15, launch_rcp15_init; through dv_core.cuh: cdf_div, cdf_div_pos, weights_update(32), speed_is_small
#include "dv2_core.cuh"     // recip32, divq
#include "numeric_ref.h"

namespace {

#define PK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { err = e_; goto done; } } while (0)

constexpr int MAX_EX = 64;
struct SweepOut { unsigned long long mismatches, cases, c_over_max; int n_ex; int ex[MAX_EX][4]; };

// mode 0: cdf_div(c, d) against numeric.rs, c and d over all of i16
// mode 1: cdf_div_pos(c, d) against (c << 15) / d, 0 <= c <= d
// mode 2: divq(c, recip32(d), d) against (c << 15) / d, 0 <= c <= d
// one block per divisor d in [d_lo, d_hi)
__global__ void sweep_kernel(int mode, int d_lo, SweepOut *o) {
    const int d = d_lo + (int)blockIdx.x;
    const int c_lo = mode == 0 ? -32768 : 0, c_hi = mode == 0 ? 32767 : d;
    unsigned long long bad = 0, n = 0, over = 0;
    const uint32_t inv = mode == 2 ? dv::recip32((uint32_t)d) : 0u;
    for (int c = c_lo + (int)threadIdx.x; c <= c_hi; c += (int)blockDim.x) {
        int got, want;
        if (mode == 0) {
            got = dv::cdf_div(c, d);
            want = dvp_cdf_quotient((int16_t)c, (int16_t)d);
            over += (c > d && d > 0) ? 1u : 0u;
        } else {
            want = (int)(((uint32_t)c << 15) / (uint32_t)d);
            got = mode == 1 ? dv::cdf_div_pos(c, d) : (int)dv::divq((uint32_t)c, inv, (uint32_t)d);
        }
        n++;
        if (got != want) {
            bad++;
            const int k = atomicAdd(&o->n_ex, 1);
            if (k < MAX_EX) { o->ex[k][0] = c; o->ex[k][1] = d; o->ex[k][2] = got; o->ex[k][3] = want; }
        }
    }
    atomicAdd(&o->mismatches, bad); atomicAdd(&o->cases, n); atomicAdd(&o->c_over_max, over);
}

__global__ void div_u15_kernel(const uint64_t *tab, const uint64_t *x, const uint32_t *f, size_t n, uint64_t *q, uint32_t *r) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t fi = f[i] & 0x7fffu;   // the reverse pass reads the 15-bit frequency field of a log entry
    uint32_t rem;
    q[i] = dv::div_by_u15(x[i], fi ? fi : 1u, tab[fi ? fi : 1u], rem);
    r[i] = rem;
}

__global__ void weights_kernel(int variant, size_t n, const int32_t *in, int32_t *out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int32_t *a = in + 5 * i;   // w0, w1, f_cm, f_nb, weighted
    dv::Weights w; w.w0 = a[0]; w.w1 = a[1]; w.norm = 0;
    if (variant == 0) dv::weights_update(w, a[2], a[3], a[4]); else dv::weights_update32(w, a[2], a[3], a[4]);
    out[3 * i] = w.w0; out[3 * i + 1] = w.w1; out[3 * i + 2] = w.norm;
}

// row inc (low half of the packed speed, as u16): how many of the 65536 lim halves the gate accepts, and the least and
// greatest accepted lim (as i16)
__global__ void gate_kernel(int32_t *out) {
    __shared__ int cnt, lo, hi;
    if (threadIdx.x == 0) { cnt = 0; lo = 1 << 20; hi = -(1 << 20); }
    __syncthreads();
    const uint32_t inc = blockIdx.x;
    int my = 0, mlo = 1 << 20, mhi = -(1 << 20);
    for (uint32_t l = threadIdx.x; l < 65536u; l += blockDim.x) {
        if (dv::speed_is_small((int)((l << 16) | inc))) { my++; mlo = min(mlo, (int)(int16_t)l); mhi = max(mhi, (int)(int16_t)l); }
    }
    atomicAdd(&cnt, my); atomicMin(&lo, mlo); atomicMax(&hi, mhi);
    __syncthreads();
    if (threadIdx.x == 0) { out[3 * inc] = cnt; out[3 * inc + 1] = lo; out[3 * inc + 2] = hi; }
}

// ---- one coding step at CDF level, one lane group per case ----
enum StepVariant { V2_16 = 0, V2_8 = 1, R1_ENC = 3, FAST_16 = 4, FAST_8 = 5, FAST_MIX_16 = 6 };   // (2 is unused: the values seed the tests' cases)
struct StepIo {
    const int16_t *cdf, *cdf2; const int32_t *wts, *speeds; const uint64_t *state; const int32_t *sym_in;
    int16_t *s_cdf, *s_cdf2; dv::Cold *cold; uint32_t *log; const uint32_t *zero_word;   // per padded case scratch
    int32_t *sym, *start, *freq, *status; uint64_t *state_out; int32_t *wts_out;
    size_t n; int mix; uint32_t gen;
};
template <int V>
__global__ void step_kernel(StepIo io) {
    constexpr int NL = (V == V2_8 || V == FAST_8) ? 8 : 16;
    const int lane = threadIdx.x & 31;
    const size_t pc = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / NL;   // padded case: its own scratch
    const size_t i = pc < io.n ? pc : io.n - 1;                               // input case
    const bool valid = pc < io.n;
    dv::G2 g;
    g.l16 = lane & (NL - 1); g.shift = lane & (32 - NL); g.gmask = (NL == 16 ? 0xffffu : 0xffu) << g.shift;
    g.store0 = g.l16 == 0; g.nl = NL; g.grp = 0; g.blend = false;
    int16_t *cdf = io.s_cdf + 16 * pc, *cdf2 = io.s_cdf2 + 16 * pc;
    for (int k = g.l16; k < 16; k += NL) { cdf[k] = io.cdf[16 * i + k]; cdf2[k] = io.cdf2[16 * i + k]; }
    dv::Cold *c = io.cold + pc;
    dv::Weights w0; w0.w0 = io.wts[3 * i]; w0.w1 = io.wts[3 * i + 1]; w0.norm = io.wts[3 * i + 2];
    if (g.store0) { c->w_hi = w0; c->ad_cm_hi = io.speeds[2 * i + 1]; }
    __syncwarp();
    const uint64_t st0 = io.state[i];
    int sym = 0, start = 0, freq = 0, status = 0;
    uint64_t st = 0;
    dv::Weights w = w0;
    if (V == V2_16 || V == V2_8 || V == R1_ENC) {
        dv::St s;
        memset(&s, 0, sizeof s);
        s.c = c; s.state = 1; s.status = dv::ST_OK; s.gen = io.gen; s.tagged = false;
        if (V == R1_ENC) dv::coder_init_enc(s.cur, io.log + pc);
        else { s.cur.a = st0; s.cur.b = 0; s.cur.need_a = 0; s.cur.need_b = 0; s.cur.sym_count = 0; s.cur.p = io.zero_word; s.cur.left = 0; }
        dv::Next nx;
        nx.cdf = cdf; nx.cdf2 = io.mix ? cdf2 : nullptr; nx.speed = io.speeds[2 * i]; nx.sym = io.sym_in[i]; nx.mix_hi = true; nx.tagged = false;
        if (V == V2_16) sym = dv::nibble_core_v2<16>(s, nx, g);
        else if (V == V2_8) sym = dv::nibble_core_v2<8>(s, nx, g);
        else sym = dv::nibble_core_enc(s, nx, g);
        __syncwarp();
        st = s.cur.b;
        status = s.status;
        if (V == R1_ENC) { const uint32_t e = io.log[pc]; start = (int16_t)(e & 0xffffu); freq = (int16_t)(e >> 16); }
        w = c->w_hi;
    } else {
        // the fast loops' pieces on a validated prior (tag bits stripped), storing with this stream's tag bits
        const int li = g.l16;
        dv::FastK f;
        f.wbase = io.zero_word; f.wi = 0; f.wmax = 0; f.wnext = 0;
        f.inc = (int)(short)(io.speeds[2 * i] & 0xffff); f.lim = io.speeds[2 * i] >> 16;
        f.incp = (uint32_t)f.inc * 0x10001u;
        f.kp = NL == 16 ? (uint32_t)(li + 1) : ((uint32_t)(2 * li + 1) | ((uint32_t)(2 * li + 2) << 16));
        f.mytag = dv::lane_tag<NL>(io.gen, li);
        const uint32_t bsel = NL == 16 ? (0xffffu << g.shift) : ((uint32_t)(g.shift >> 3) * 0x1111u + 0x4040u);
        const char *p = reinterpret_cast<const char *>(cdf);
        if (V == FAST_MIX_16) {
            dv::MixV v = dv::mixv_load(p, reinterpret_cast<const char *>(cdf2), li);
            v.c &= 0x7fffu; v.maxv &= 0x7fffu;
            const dv::MixS ms = dv::mixv_search(st0, v, w.norm, bsel);
            st = st0;
            dv::mixv_finish(st, v, ms, w, p, reinterpret_cast<const char *>(cdf2), g, f, (int)(short)(io.speeds[2 * i + 1] & 0xffff),
                            io.speeds[2 * i + 1] >> 16);
            sym = ms.sym;
        } else {
            const uint32_t ev = NL == 16 ? (uint32_t)(uint16_t)cdf[li] : ((uint32_t)(uint16_t)cdf[2 * li] | ((uint32_t)(uint16_t)cdf[2 * li + 1] << 16));
            const uint32_t mv = (uint32_t)(uint16_t)cdf[15];
            __syncwarp();
            sym = dv::search_v2<NL>(st0, ev, mv, bsel);
            st = dv::rans_advance_v2<NL>(st0, ev, mv, sym);
            dv::blend_store_v2<NL>(ev, mv, sym, p, g, f);
        }
        __syncwarp();
    }
    if (valid && g.store0) {
        io.sym[i] = sym; io.start[i] = start; io.freq[i] = freq; io.status[i] = status; io.state_out[i] = st;
        io.wts_out[3 * i] = w.w0; io.wts_out[3 * i + 1] = w.w1; io.wts_out[3 * i + 2] = w.norm;
    }
}

}  // namespace

extern "C" {

// One coding step per case (see StepVariant; mix: every case mixes cdf2 with weights (w0, w1, norm), high-nibble weight set).
// Inputs per case: cdf[16], cdf2[16], wts[3], speeds[2] (packed inc | lim << 16: stride, context map), state (decode), sym_in
// (encode).  Outputs: sym, start / freq (R1_ENC: as logged), status (R1_ENC: 3 = refused), state (decode: after the step,
// before renormalisation; FAST_MIX_16: renormalised with a zero word), the CDFs as stored (fast pieces: with tag bits), weights.
int dvp_step(int variant, size_t n, int mix, uint32_t gen, const int16_t *cdf, const int16_t *cdf2, const int32_t *wts,
             const int32_t *speeds, const uint64_t *state, const int32_t *sym_in, int32_t *sym, int32_t *start, int32_t *freq,
             int32_t *status, uint64_t *state_out, int16_t *cdf_out, int16_t *cdf2_out, int32_t *wts_out) {
    cudaError_t err = cudaSuccess;
    StepIo io;
    memset(&io, 0, sizeof io);
    const int nl = (variant == V2_8 || variant == FAST_8) ? 8 : 16;
    const size_t per_block = 256 / nl, np = (n + per_block - 1) / per_block * per_block;
    void *bufs[17] = {};
    if (n == 0) return 0;
    if (variant < 0 || variant > 6 || variant == 2) return (int)cudaErrorInvalidValue;
    PK(cudaSetDevice(0));
#define ALLOC(k, ptr, bytes) do { PK(cudaMalloc(&bufs[k], (bytes))); PK(cudaMemset(bufs[k], 0, (bytes))); ptr = decltype(ptr)(bufs[k]); } while (0)
    ALLOC(0, io.cdf, n * 32); ALLOC(1, io.cdf2, n * 32); ALLOC(2, io.wts, n * 12); ALLOC(3, io.speeds, n * 8);
    ALLOC(4, io.state, n * 8); ALLOC(5, io.sym_in, n * 4);
    ALLOC(6, io.s_cdf, np * 32); ALLOC(7, io.s_cdf2, np * 32); ALLOC(8, io.cold, np * sizeof(dv::Cold)); ALLOC(9, io.log, np * 4);
    ALLOC(10, io.zero_word, 16);
    ALLOC(11, io.sym, n * 4); ALLOC(12, io.start, n * 4); ALLOC(13, io.freq, n * 4); ALLOC(14, io.status, n * 4);
    ALLOC(15, io.state_out, n * 8); ALLOC(16, io.wts_out, n * 12);
#undef ALLOC
    PK(cudaMemcpy((void *)io.cdf, cdf, n * 32, cudaMemcpyHostToDevice));
    PK(cudaMemcpy((void *)io.cdf2, cdf2, n * 32, cudaMemcpyHostToDevice));
    PK(cudaMemcpy((void *)io.wts, wts, n * 12, cudaMemcpyHostToDevice));
    PK(cudaMemcpy((void *)io.speeds, speeds, n * 8, cudaMemcpyHostToDevice));
    PK(cudaMemcpy((void *)io.state, state, n * 8, cudaMemcpyHostToDevice));
    PK(cudaMemcpy((void *)io.sym_in, sym_in, n * 4, cudaMemcpyHostToDevice));
    io.n = n; io.mix = mix; io.gen = gen;
    {
        const unsigned blocks = (unsigned)(np / per_block);
        switch (variant) {
            case V2_16: step_kernel<V2_16><<<blocks, 256>>>(io); break;
            case V2_8: step_kernel<V2_8><<<blocks, 256>>>(io); break;
            case R1_ENC: step_kernel<R1_ENC><<<blocks, 256>>>(io); break;
            case FAST_16: step_kernel<FAST_16><<<blocks, 256>>>(io); break;
            case FAST_8: step_kernel<FAST_8><<<blocks, 256>>>(io); break;
            default: step_kernel<FAST_MIX_16><<<blocks, 256>>>(io); break;
        }
    }
    PK(cudaGetLastError());
    PK(cudaDeviceSynchronize());
    PK(cudaMemcpy(sym, io.sym, n * 4, cudaMemcpyDeviceToHost));
    PK(cudaMemcpy(start, io.start, n * 4, cudaMemcpyDeviceToHost));
    PK(cudaMemcpy(freq, io.freq, n * 4, cudaMemcpyDeviceToHost));
    PK(cudaMemcpy(status, io.status, n * 4, cudaMemcpyDeviceToHost));
    PK(cudaMemcpy(state_out, io.state_out, n * 8, cudaMemcpyDeviceToHost));
    PK(cudaMemcpy(cdf_out, io.s_cdf, n * 32, cudaMemcpyDeviceToHost));
    PK(cudaMemcpy(cdf2_out, io.s_cdf2, n * 32, cudaMemcpyDeviceToHost));
    PK(cudaMemcpy(wts_out, io.wts_out, n * 12, cudaMemcpyDeviceToHost));
done:
    for (void *b : bufs) cudaFree(b);
    return (int)err;
}


// divisions, exhaustive over divisors [d_lo, d_hi): counts[0..2] = mismatches, cases, cases with c > max (mode 0);
// ex[64][4] = up to 64 mismatches (c, d, got, want), n_ex = how many mismatches were offered (may exceed 64); ms = kernel time
int dvp_div_sweep(int mode, int d_lo, int d_hi, unsigned long long *counts, int32_t *ex, int *n_ex, float *ms) {
    cudaError_t err = cudaSuccess;
    SweepOut *d_o = nullptr, h_o;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (mode < 0 || mode > 2 || d_hi <= d_lo) return (int)cudaErrorInvalidValue;
    PK(cudaSetDevice(0));
    PK(cudaMalloc((void **)&d_o, sizeof(SweepOut)));
    PK(cudaMemset(d_o, 0, sizeof(SweepOut)));
    PK(cudaEventCreate(&e0)); PK(cudaEventCreate(&e1));
    PK(cudaEventRecord(e0));
    sweep_kernel<<<(unsigned)(d_hi - d_lo), 256>>>(mode, d_lo, d_o);
    PK(cudaGetLastError());
    PK(cudaEventRecord(e1));
    PK(cudaEventSynchronize(e1));
    PK(cudaEventElapsedTime(ms, e0, e1));
    PK(cudaMemcpy(&h_o, d_o, sizeof(SweepOut), cudaMemcpyDeviceToHost));
    counts[0] = h_o.mismatches; counts[1] = h_o.cases; counts[2] = h_o.c_over_max;
    *n_ex = h_o.n_ex;
    memcpy(ex, h_o.ex, sizeof h_o.ex);
done:
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    cudaFree(d_o);
    return (int)err;
}

// the encoder's reciprocal table as launch_rcp15_init builds it (32768 entries)
int dvp_rcp15_table(uint64_t *out) {
    cudaError_t err = cudaSuccess;
    uint64_t *tab = nullptr;
    PK(cudaSetDevice(0));
    PK(cudaMalloc((void **)&tab, 32768 * sizeof(uint64_t)));
    dv::launch_rcp15_init(tab, 0);
    PK(cudaGetLastError());
    PK(cudaMemcpy(out, tab, 32768 * sizeof(uint64_t), cudaMemcpyDeviceToHost));
done:
    cudaFree(tab);
    return (int)err;
}

// q[i], r[i] = div_by_u15(x[i], f[i]) with the table of launch_rcp15_init (f in 1..32767; x < 2^63)
int dvp_div_u15(const uint64_t *x, const uint32_t *f, size_t n, uint64_t *q, uint32_t *r) {
    cudaError_t err = cudaSuccess;
    uint64_t *tab = nullptr, *dx = nullptr, *dq = nullptr;
    uint32_t *df = nullptr, *dr = nullptr;
    if (n == 0) return 0;
    PK(cudaSetDevice(0));
    PK(cudaMalloc((void **)&tab, 32768 * sizeof(uint64_t)));
    PK(cudaMalloc((void **)&dx, n * 8)); PK(cudaMalloc((void **)&dq, n * 8));
    PK(cudaMalloc((void **)&df, n * 4)); PK(cudaMalloc((void **)&dr, n * 4));
    dv::launch_rcp15_init(tab, 0);
    PK(cudaMemcpy(dx, x, n * 8, cudaMemcpyHostToDevice));
    PK(cudaMemcpy(df, f, n * 4, cudaMemcpyHostToDevice));
    div_u15_kernel<<<(unsigned)((n + 255) / 256), 256>>>(tab, dx, df, n, dq, dr);
    PK(cudaGetLastError());
    PK(cudaMemcpy(q, dq, n * 8, cudaMemcpyDeviceToHost));
    PK(cudaMemcpy(r, dr, n * 4, cudaMemcpyDeviceToHost));
done:
    cudaFree(tab); cudaFree(dx); cudaFree(dq); cudaFree(df); cudaFree(dr);
    return (int)err;
}

// variant 0: weights_update, 1: weights_update32.  in: n x (w0, w1, f_cm, f_nb, weighted); out: n x (w0, w1, norm)
int dvp_weights(int variant, size_t n, const int32_t *in, int32_t *out) {
    cudaError_t err = cudaSuccess;
    int32_t *di = nullptr, *dout = nullptr;
    if (n == 0) return 0;
    PK(cudaSetDevice(0));
    PK(cudaMalloc((void **)&di, n * 5 * 4)); PK(cudaMalloc((void **)&dout, n * 3 * 4));
    PK(cudaMemcpy(di, in, n * 5 * 4, cudaMemcpyHostToDevice));
    weights_kernel<<<(unsigned)((n + 255) / 256), 256>>>(variant, n, di, dout);
    PK(cudaGetLastError());
    PK(cudaMemcpy(out, dout, n * 3 * 4, cudaMemcpyDeviceToHost));
done:
    cudaFree(di); cudaFree(dout);
    return (int)err;
}

// speed_is_small on every packed i16 (inc, lim): out[65536][3] = per inc row (as u16): accepted count, least and greatest lim
int dvp_speed_gate(int32_t *out) {
    cudaError_t err = cudaSuccess;
    int32_t *d = nullptr;
    PK(cudaSetDevice(0));
    PK(cudaMalloc((void **)&d, 65536 * 3 * 4));
    gate_kernel<<<65536, 256>>>(d);
    PK(cudaGetLastError());
    PK(cudaMemcpy(out, d, 65536 * 3 * 4, cudaMemcpyDeviceToHost));
done:
    cudaFree(d);
    return (int)err;
}

}  // extern "C"
