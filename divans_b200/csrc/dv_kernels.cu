// dv_kernels.cu -- sm_90a kernels of the divANS batch engine: the framing/CRC pre-pass every decode runs first, and the
// stream decoder of the reference's feature="blend" probability model (dv_blend.cuh).  Frequentist streams decode on the
// v2 engine (dv2_kernels.cu).
#include "dv_core.cuh"

namespace dv {

// ---------------------------------------------------------------------------------------------------------------
// framing pre-pass: frame kernel (header, record walk, trailer, CRC32C -- one warp per stream), payload scan, demux.
// ---------------------------------------------------------------------------------------------------------------
// frame kernel: one WARP per stream.  Lane 0 walks the 16-byte header and the mux record chain (mux.rs:384-444) to the
// EOF marker and checks the trailer magic; the warp checks the CRC32C of header..EOF marker (codec/decoder.rs:186-213).
__global__ void __launch_bounds__(128) frame_kernel(FrameParams p) {
    __shared__ uint32_t tab[4][256];   // slice-by-4 tables for the Castagnoli polynomial (reflected 0x82F63B78)
    __shared__ uint32_t x2n[32];       // x^(2^k) mod P
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) {
        uint32_t c = i;
        for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ CRC32C_POLY : (c >> 1);
        tab[0][i] = c;
    }
    if (threadIdx.x == 0) {
        uint32_t v = 0x40000000u;      // x^1
        x2n[0] = v;
        for (int k = 1; k < 32; k++) { v = gf_mul(v, v); x2n[k] = v; }
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) {
        uint32_t c = tab[0][i];
        for (int t = 1; t < 4; t++) { c = tab[0][c & 0xff] ^ (c >> 8); tab[t][i] = c; }
    }
    __syncthreads();
    const uint32_t sidx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (sidx >= p.n_streams) return;
    const uint8_t *in = p.in + p.in_off[sidx];
    const uint64_t n = p.in_len[sidx];
    int32_t st = ST_OK;
    uint32_t body_end = 0, pay0 = 0, pay1 = 0;
    if (lane == 0) {
        if (n < 16) st = ST_NEED_INPUT;
        else if (in[0] != 0xff || in[1] != 0xe5 || in[2] != 0x8c || in[3] != 0x9f) st = ST_FAIL;   // MAGIC_NUMBER, src/interface.rs:164
        else if (in[5] < 10 || in[5] >= 25) st = ST_FAIL;                                             // BadWindowSize, divans_decompressor.rs:47-50
        else {
            uint64_t pos = 16;
            for (;;) {
                if (pos >= n) { st = ST_NEED_INPUT; break; }
                uint32_t b = in[pos];
                if (b == 0xff) {
                    if (pos + 3 > n) { st = ST_NEED_INPUT; break; }
                    if (in[pos + 1] != 0xfe || in[pos + 2] != 0xff) { st = ST_FAIL; break; }
                    body_end = (uint32_t)pos;
                    break;
                }
                uint64_t len, hdr;
                if (b < 16) { if (pos + 3 > n) { st = ST_NEED_INPUT; break; } len = ((uint64_t)in[pos + 1] | ((uint64_t)in[pos + 2] << 8)) + 1; hdr = 3; }
                else { uint32_t k = b >> 4; if (k > 3) { st = ST_FAIL; break; } len = 1024ull << (k << 1); hdr = 1; }
                if (pos + hdr + len > n) { st = ST_NEED_INPUT; break; }
                if (b & 1) pay1 += (uint32_t)len; else pay0 += (uint32_t)len;
                pos += hdr + len;
            }
            if (st == ST_OK) {
                const uint64_t tr = (uint64_t)body_end + 3;
                if (tr + 8 > n) st = ST_NEED_INPUT;
                else if (in[tr + 4] != 'a' || in[tr + 5] != 'n' || in[tr + 6] != 's' || in[tr + 7] != '~') st = ST_FAIL;
            }
        }
    }
    st = __shfl_sync(FULL, st, 0);
    body_end = __shfl_sync(FULL, body_end, 0);
    if (st == ST_OK && !(p.flags & 3u)) {
        const uint32_t tr = body_end + 3;
        const uint32_t crc = warp_crc32c(tab, x2n, in, tr, lane);
        const uint32_t want = (uint32_t)in[tr] | ((uint32_t)in[tr + 1] << 8) | ((uint32_t)in[tr + 2] << 16) | ((uint32_t)in[tr + 3] << 24);
        if (crc != want) st = ST_FAIL;   // BadChecksum
    }
    if (lane == 0) {
        p.frame[4 * sidx + 0] = st == ST_OK ? body_end : 0;
        p.frame[4 * sidx + 1] = st == ST_OK ? pay0 : 0;
        p.frame[4 * sidx + 2] = st == ST_OK ? pay1 : 0;
        p.status[sidx] = st;
    }
}

// exclusive scan of the per-stream payload footprints -> frame[4i+3] = base of stream i's compacted payload (16-byte units)
// A stream whose compacted payload would not fit the payload buffer (`cap16` 16-byte units: aliased / overlapping input
// regions, or an underestimated in_total_bytes) is failed here instead of letting the demux kernel write past the end.
__global__ void __launch_bounds__(1024) payload_scan_kernel(uint32_t *frame, uint32_t n, int32_t *status, uint64_t cap16) {
    __shared__ uint32_t part[1024];
    const uint32_t t = threadIdx.x;
    const uint32_t per = (n + 1023) / 1024;
    const uint32_t lo = min(n, t * per), hi = min(n, lo + per);
    uint32_t sum = 0;
    for (uint32_t i = lo; i < hi; i++) sum += ((frame[4 * i + 1] + 15) >> 4) + ((frame[4 * i + 2] + 15) >> 4) + 1;
    part[t] = sum;
    __syncthreads();
    for (uint32_t o = 1; o < 1024; o <<= 1) {
        uint32_t v = t >= o ? part[t - o] : 0;
        __syncthreads();
        part[t] += v;
        __syncthreads();
    }
    uint32_t base = part[t] - sum;
    for (uint32_t i = lo; i < hi; i++) {
        const uint32_t need = ((frame[4 * i + 1] + 15) >> 4) + ((frame[4 * i + 2] + 15) >> 4) + 1;
        if ((uint64_t)base + need > cap16) {
            if (status[i] == ST_OK) status[i] = ST_FAIL;
            frame[4 * i + 1] = 0; frame[4 * i + 2] = 0; frame[4 * i + 3] = 0;
        } else frame[4 * i + 3] = base;
        base += need;
    }
}

// demux (mux.rs:384-444): one warp per stream copies the payload of every record to the stream's compact area:
// command-coder bytes at base, literal-coder bytes at base + align16(cmd bytes)
__global__ void __launch_bounds__(128) demux_kernel(FrameParams p, uint8_t *payload) {
    const uint32_t sidx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (sidx >= p.n_streams || p.status[sidx] != ST_OK) return;
    const uint8_t *in = p.in + p.in_off[sidx];
    const uint32_t body_end = p.frame[4 * sidx + 0];
    uint8_t *dst0 = payload + 16ull * p.frame[4 * sidx + 3];
    uint8_t *dst1 = dst0 + (((uint64_t)p.frame[4 * sidx + 1] + 15) & ~15ull);
    uint32_t pos = 16;
    while (pos < body_end) {
        uint32_t b = in[pos], len, hdr;
        if (b < 16) { len = ((uint32_t)in[pos + 1] | ((uint32_t)in[pos + 2] << 8)) + 1; hdr = 3; }
        else { len = 1024u << ((b >> 4) << 1); hdr = 1; }
        const uint8_t *src = in + pos + hdr;
        uint8_t *d = (b & 1) ? dst1 : dst0;
        // byte head to a 4-byte aligned destination, then words assembled from (possibly unaligned) source bytes
        uint32_t head = min(len, (uint32_t)((4 - ((uintptr_t)d & 3)) & 3));
        if (lane < head) d[lane] = src[lane];
        uint32_t nw = (len - head) >> 2;
        const uint8_t *s2 = src + head; uint32_t *d2 = reinterpret_cast<uint32_t *>(d + head);
        const uint32_t *sa = reinterpret_cast<const uint32_t *>((uintptr_t)s2 & ~(uintptr_t)3);
        const uint32_t sh = ((uint32_t)(uintptr_t)s2 & 3u) * 8u;
        for (uint32_t i = lane; i < nw; i += 32) d2[i] = __funnelshift_r(sa[i], sa[i + 1], sh);   // over-read <= 3 B stays inside the stream (EOF marker + trailer follow)
        uint32_t tail = (len - head) & 3;
        if (lane < tail) d[head + 4 * nw + lane] = src[head + 4 * nw + lane];
        if (b & 1) dst1 += len; else dst0 += len;
        pos += hdr + len;
    }
}

void launch_frame(const FrameParams &p, uint8_t *payload, uint64_t payload_cap_bytes, cudaStream_t st) {
    uint32_t blocks = (p.n_streams + 3) / 4;   // one warp per stream
    frame_kernel<<<blocks, 128, 0, st>>>(p);
    payload_scan_kernel<<<1, 1024, 0, st>>>(p.frame, p.n_streams, p.status, payload_cap_bytes / 16);
    demux_kernel<<<(p.n_streams + 3) / 4, 128, 0, st>>>(p, payload);
}

// ---------------------------------------------------------------------------------------------------------------
// blend stream decoder: persistent warps, two streams per warp in lock step (dv_engine.cuh), work pulled from a global
// counter.  Every nibble goes through the blend core (nibble_core_blend): the model has no literal fast loop.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(DECODE_BLOCK_THREADS, 8) decode_kernel_blend(DecodeParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x & 31;
    const int group_in_block = (threadIdx.x >> 5) * 2 + (lane >> 4);
    const uint32_t slot = blockIdx.x * (DECODE_BLOCK_THREADS / 16) + group_in_block;
    G2 g;
    g.l16 = lane & 15;
    g.shift = lane & 16;
    g.gmask = 0xffffu << (lane & 16);
    g.store0 = (lane & 15) == 0;
    g.nl = 16;
    g.grp = group_in_block;
    g.blend = true;

    St s;
    s.slot = p.arena + (uint64_t)slot * SLOT_STRIDE;
    s.c = reinterpret_cast<Cold *>(smem + group_in_block * SMEM_BYTES_PER_GROUP);
    s.tables = p.tables;
    s.state = S_IDLE;
    s.c->desired_context_mixing = 0; s.c->desired_prior_depth = 0; s.c->desired_force_stride = 9; s.c->desired_do_context_map = true;
    s.c->have_desired_adapt = false; s.c->desired_adapt0 = s.c->desired_adapt1 = s.c->desired_adapt2 = s.c->desired_adapt3 = 0;
    s.c->in.cmds = nullptr; s.c->in.n_cmds = 0; s.c->in.pos = 0; s.c->in.n_pms = 0; s.c->in.pms = nullptr; s.c->in.lits = nullptr;
    s.c->model_rev = p.model_rev;
    s.c->sidx = 0; s.out = nullptr; s.out_pos = 0; s.c->out_cap = 0; s.c->ring_len = 1024;
    st_reset(s);
    coder_init_dec(s.cur, nullptr, 0); s.cur.need_a = 0; coder_init_dec(s.c->oth, nullptr, 0);
    Next nx; nx.cdf = A_misc(s, MI_DUMMY); nx.cdf2 = nullptr; nx.speed = SPK_NONE; nx.tagged = false; nx.sym = 0; nx.mix_hi = false;
    store_default_cdfs(g, reinterpret_cast<int16_t *>(s.slot + OFF_MISC), (uint32_t)MISC_CDFS);   // incl. the dummy CDF
    bool exhausted = false;

    for (;;) {
        __syncwarp();
        // ---- fetch work for idle groups (converged; the broadcast shuffle is executed by every lane) ----
        const bool want = (s.state == S_IDLE) && !exhausted;
        if (__any_sync(FULL, want)) {
            uint32_t v = 0;
            if (want && g.store0) v = atomicAdd(p.work_counter, 1u);
            v = __shfl_sync(FULL, v, 0, 16);
            if (want) {
                if (v >= p.n_streams) exhausted = true;
                else if (p.status[v] != ST_OK) { if (g.store0) p.out_len[v] = 0; }   // framing / CRC failure: stay idle, fetch again
                else {
                    const uint8_t *in = p.in + p.in_off[v];
                    const uint32_t pay0 = p.frame[4 * v + 1], pay1 = p.frame[4 * v + 2];
                    const uint8_t *pl = p.payload + 16ull * p.frame[4 * v + 3];
                    s.c->sidx = v;
                    s.out = p.out + p.out_off[v];
                    uint64_t cap = p.out_cap[v];
                    s.c->out_cap = cap > 0xffffffffull ? 0xffffffffu : (uint32_t)cap; s.out_pos = 0;
                    s.c->ring_len = 1u << in[5];
                    reset_slot(g, s.slot);
                    st_reset(s);
                    coder_init_dec(s.cur, reinterpret_cast<const uint32_t *>(pl), pay0 >> 2);   // command stream (CMD_CODER, codec/interface.rs:49)
                    coder_init_dec(s.c->oth, reinterpret_cast<const uint32_t *>(pl + (((uint64_t)pay0 + 15) & ~15ull)), pay1 >> 2);   // literal stream (LIT_CODER, :50)
                    enter_cmd_type<false>(s, nx);
                }
            }
            if (__all_sync(FULL, exhausted && s.state == S_IDLE)) break;
            __syncwarp();
        }
        // ---- one nibble per group ----
        const bool busy = s.state != S_IDLE;
        int sym = nibble_core_blend<false>(s, nx, g);
        // ---- per-group scalar state machines (divergent) ----
        if (busy) {
            if (s.cur.underflow) s.status = ST_NEED_INPUT;
            else transition<false>(s, nx, g, sym);
            if (s.status != ST_OK || s.state == S_IDLE) {
                if (s.status == ST_OK && s.c->oth.underflow) s.status = ST_NEED_INPUT;
                if (g.store0) { p.out_len[s.c->sidx] = s.out_pos; p.status[s.c->sidx] = s.status; }
                s.state = S_IDLE; s.status = ST_OK;
                nx.cdf = A_misc(s, MI_DUMMY); nx.cdf2 = nullptr; nx.speed = SPK_NONE; nx.tagged = false;
                coder_init_dec(s.cur, nullptr, 0); s.cur.need_a = 0;
            }
        }
    }
}

void launch_decode16_blend(const DecodeParams &p, uint32_t n_blocks, cudaStream_t st) {
    size_t smem = (size_t)(DECODE_BLOCK_THREADS / 16) * SMEM_BYTES_PER_GROUP;
    decode_kernel_blend<<<n_blocks, DECODE_BLOCK_THREADS, smem, st>>>(p);
}
int decode_max_blocks_per_sm16_blend() {
    return stream_kernel_blocks_per_sm(decode_kernel_blend, DECODE_BLOCK_THREADS, (size_t)(DECODE_BLOCK_THREADS / 16) * SMEM_BYTES_PER_GROUP);
}

}  // namespace dv
