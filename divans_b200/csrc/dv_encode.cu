// dv_encode.cu -- sm_90a kernels of the divANS batch ENCODER (SURVEY 8a "next": GPU encoder, BASELINE config 4).
//
// The reference's encoder (codec/mod.rs:280-560 + ans.rs:289-378) interleaves three things per stream: the adaptive
// model walk, a reverse rANS pass every 65536 symbols, and the mux.  They are separate passes here:
//   1. encode_model_kernel  the lock-step engine (dv_engine.cuh) run with ENC=true: walks the command list, adapts
//                           the priors exactly as the decoder will, and logs one (start | freq << 16) word per nibble
//                           into the stream's command / literal log.
//   2. encode_flush_kernel  one thread per (65536-symbol chunk, rANS state) runs the recurrence last symbol -> first
//                           symbol (ans.rs:302-378); encode_pack_kernel then stacks the renormalisation words in
//                           symbol order IN PLACE at the top of the chunk's own log region (<= one word per symbol).
//   3. encode_mux_kernel    one warp per stream: header, the record chain of Mux::serialize_close with everything
//                           still buffered (mux.rs:478-561), EOF marker, CRC32C and trailer (codec/mod.rs:493-560).
#include "dv_core.cuh"

namespace dv {

template <bool BLEND>
__global__ void __launch_bounds__(DECODE_BLOCK_THREADS, 8) encode_model_kernel(EncodeParams p) {
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
    g.blend = BLEND;

    St s;
    s.slot = p.arena + (uint64_t)slot * SLOT_STRIDE;
    s.c = reinterpret_cast<Cold *>(smem + group_in_block * SMEM_BYTES_PER_GROUP);
    s.tables = p.tables;
    s.state = S_IDLE;
    s.c->in.cmds = nullptr; s.c->in.n_cmds = 0; s.c->in.pos = 0; s.c->in.n_pms = 0; s.c->in.pms = nullptr; s.c->in.lits = nullptr;
    s.c->model_rev = (uint32_t)p.model_rev;
    s.c->sidx = 0; s.c->raw_len = 0; s.c->lit_log_cap = p.lit_cap;
    s.out = p.replay + (uint64_t)slot * p.replay_stride; s.out_pos = 0;
    s.c->out_cap = p.replay_stride > 0xffffffffull ? 0xffffffffu : (uint32_t)p.replay_stride;
    s.c->ring_len = 1u << p.window_size;
    st_reset(s);
    uint32_t *const dummy_log = p.sf_dummy + slot;
    coder_init_enc(s.cur, dummy_log); coder_init_enc(s.c->oth, dummy_log);
    Next nx; nx.cdf = A_misc(s, MI_DUMMY); nx.cdf2 = nullptr; nx.speed = SPK_NONE; nx.tagged = false; nx.sym = 0; nx.mix_hi = false;
    store_default_cdfs(g, reinterpret_cast<int16_t *>(s.slot + OFF_MISC), (uint32_t)MISC_CDFS);
    bool exhausted = false;
    const uint32_t per_stream = p.cmd_cap + p.lit_cap;

    for (;;) {
        __syncwarp();
        const bool want = (s.state == S_IDLE) && !exhausted;
        if (__any_sync(FULL, want)) {
            uint32_t v = 0;
            if (want && g.store0) v = atomicAdd(p.work_counter, 1u);
            v = __shfl_sync(FULL, v, 0, 16);
            if (want) {
                if (v >= p.n_streams) exhausted = true;
                else {
                    const uint8_t *blob = p.in + p.in_off[v];
                    const uint64_t blen = p.in_len[v];
                    bool ok = true;
                    s.c->sidx = v;
                    s.out_pos = 0;
                    reset_slot(g, s.slot);
                    st_reset(s);
                    // CrossCommandBookKeeping::new, codec/interface.rs:360-366
                    uint32_t dcm = (uint32_t)p.dynamic_context_mixing;
                    if (p.force_stride != 0 && dcm == 0 && p.use_context_map) dcm = 1;
                    s.c->desired_context_mixing = dcm; s.c->desired_prior_depth = (uint32_t)p.prior_depth;
                    s.c->desired_force_stride = (uint32_t)p.force_stride; s.c->desired_do_context_map = p.use_context_map != 0;
                    s.c->have_desired_adapt = p.have_literal_adaptation != 0;
                    s.c->desired_adapt0 = p.literal_adaptation[0]; s.c->desired_adapt1 = p.literal_adaptation[1];
                    s.c->desired_adapt2 = p.literal_adaptation[2]; s.c->desired_adapt3 = p.literal_adaptation[3];
                    s.c->in.pos = 0;
                    if (p.raw_mode) {
                        if (blen > 0xffffffffull - 16) ok = false;
                        s.c->in.cmds = nullptr; s.c->in.pms = p.pm_internal; s.c->in.n_pms = 1; s.c->in.lits = blob;
                        s.c->raw_len = (uint32_t)blen;
                        s.c->in.n_cmds = 1u + (uint32_t)((blen + s.c->ring_len - 1) >> p.window_size);
                    } else {
                        const uint32_t *h = reinterpret_cast<const uint32_t *>(blob);
                        if (blen < 32 || h[0] != 0x4c435644u || h[1] != 1u) ok = false;
                        else {
                            const uint64_t need = 32ull + 20ull * h[2] + (uint64_t)PM_RECORD_BYTES * h[3] + h[4];
                            if (need > blen) ok = false;
                            s.c->in.cmds = h + 8; s.c->in.n_cmds = h[2]; s.c->in.n_pms = h[3];
                            s.c->in.pms = blob + 32 + 20ull * h[2];
                            s.c->in.lits = s.c->in.pms + (uint64_t)PM_RECORD_BYTES * h[3];
                            s.c->raw_len = h[4];
                        }
                    }
                    if (!ok) { if (g.store0) { p.status[v] = ST_FAIL; p.sf_counts[2 * v] = 0; p.sf_counts[2 * v + 1] = 0; } }
                    else {
                        coder_init_enc(s.cur, p.sf + (uint64_t)v * per_stream);                   // CMD_CODER
                        coder_init_enc(s.c->oth, p.sf + (uint64_t)v * per_stream + p.cmd_cap);   // LIT_CODER
                        enter_cmd_type<true>(s, nx);
                    }
                }
            }
            if (__all_sync(FULL, exhausted && s.state == S_IDLE)) break;
            __syncwarp();
        }
        // end of a stream: report it, park the group on the dummy prior
        auto finish = [&]() {
            const uint32_t v = s.c->sidx;
            if (g.store0) {
                p.status[v] = s.status;
                const uint32_t nc = s.c->cur_is_lit ? s.c->oth.left : s.cur.left, nl = s.c->cur_is_lit ? s.cur.left : s.c->oth.left;
                p.sf_counts[2 * v] = s.status == ST_OK ? nc : 0; p.sf_counts[2 * v + 1] = s.status == ST_OK ? nl : 0;
            }
            s.state = S_IDLE; s.status = ST_OK;
            nx.cdf = A_misc(s, MI_DUMMY); nx.cdf2 = nullptr; nx.speed = SPK_NONE; nx.tagged = false; nx.sym = 0;
            coder_init_enc(s.cur, dummy_log);
        };
        if (!BLEND && __all_sync(FULL, s.state == S_LIT_HI)) {
            literal_fast_enc(s, nx, g);
            if (s.lit_left == 0 && s.status == ST_OK) { swap_coders(s, g); s.c->in.pos++; enter_cmd_type<true>(s, nx); }
            if (s.status != ST_OK) finish();   // a symbol the loop could not code (enc_log): the stream ends here
            continue;
        }
        const bool busy = s.state != S_IDLE;
        int sym = core_dispatch<BLEND>(s, nx, g);
        if (!busy) s.cur.left = 0;
        else {
            if (s.status == ST_OK) {   // (else the core could not code the symbol: enc_log)
                // log overflow cannot happen for command lists whose sizes match the header; guard hostile blobs anyway
                if (s.cur.left + 1 >= (s.c->cur_is_lit ? p.lit_cap : p.cmd_cap)) s.status = ST_FAIL;
                else transition<true>(s, nx, g, sym);
            }
            if (s.status != ST_OK || s.state == S_IDLE) finish();
        }
    }
}

#ifndef DV_BLEND   // (the rANS / mux passes do not depend on the probability model: they live in the default translation unit)
// ---------------------------------------------------------------------------------------------------------------
// reverse rANS pass.  thread <-> (stream, chunk record)
// ---------------------------------------------------------------------------------------------------------------
// st / f through a table of 64-bit reciprocals M[f] = floor((2^64 - 1) / f): q = mulhi64(st, M[f]) is the true
// quotient or one less (st < 2^63), fixed by one remainder test.  The table load depends only on the log entry, so it
// is off the state-to-state dependency chain.
__device__ __forceinline__ uint64_t div_by_u15(uint64_t x, uint32_t f, uint64_t M, uint32_t &rem) {
    uint64_t q = __umul64hi(x, M);
    uint64_t r = x - q * (uint64_t)f;
    if (r >= (uint64_t)f) { q++; r -= (uint64_t)f; }
    rem = (uint32_t)r;
    return q;
}

// thread <-> (stream, chunk record, rANS state).  The two interleaved states of a chunk are independent recurrences
// (symbol j counted from the end belongs to state j & 1, ans.rs:350-352); only the ORDER of their renormalisation words
// in the byte stack couples them.  So each state runs in its own thread, leaves a word in place of the log entry that
// produced it plus one bit in its emission bitmap, and encode_pack_kernel stacks the words in symbol order afterwards.
__global__ void __launch_bounds__(128) encode_flush_kernel(EncodeParams p) {
    const uint64_t tt = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t t = tt >> 1;
    const uint32_t parity = (uint32_t)tt & 1u;
    const uint32_t v = (uint32_t)(t / p.max_chunks), j = (uint32_t)(t % p.max_chunks);
    if (v >= p.n_streams) return;
    const bool lit = j >= p.cmd_chunks;
    const uint32_t cj = lit ? j - p.cmd_chunks : j;
    const uint32_t count = p.sf_counts[2 * v + (lit ? 1 : 0)];
    const uint32_t first = cj * NUM_SYMBOLS_BEFORE_FLUSH;
    if (first >= count) { if (!parity) p.chunk_w[t] = 0xffffffffu; return; }
    const uint32_t last = min(count, first + NUM_SYMBOLS_BEFORE_FLUSH);
    const uint32_t cnt = last - first;
    uint32_t *sf = p.sf + (uint64_t)v * (p.cmd_cap + p.lit_cap) + (lit ? p.cmd_cap : 0);
    uint32_t *bits = p.emit_bits + tt * (NUM_SYMBOLS_BEFORE_FLUSH / 64);
    const uint32_t mine = (cnt + 1 - parity) >> 1;          // symbols of this state
    uint64_t st = 1ull << 31;
    uint32_t acc = 0;
    // one step of ans.rs:330-352; a symbol emits at most one 32-bit word
#define DV_RANS_PUT(e, Mv, idx, slot)                                                                          \
    {                                                                                                          \
        const uint32_t f_ = ((e) >> 16) & 0x7fffu;     /* freq is 1..32767 for every prior the model can reach */ \
        const uint64_t start_ = (uint64_t)(int64_t)(short)((e) & 0xffffu);                                     \
        if ((uint32_t)(st >> 32) >= (f_ << 16)) { sf[slot] = (uint32_t)st; st >>= 32; acc |= 1u << ((idx) & 31); }  \
        uint32_t rem_;                                                                                         \
        const uint64_t q_ = div_by_u15(st, f_ ? f_ : 1u, (Mv), rem_);                                          \
        st = (q_ << 15) + rem_ + start_;                                                                       \
        if (((idx) & 31) == 31) { bits[(idx) >> 5] = acc; acc = 0; }                                           \
    }
    // log entries and reciprocals are fetched one block of 8 symbols ahead of the arithmetic
    constexpr int BLK = 8;
    const uint32_t n_blk = mine / BLK;
    uint32_t e[BLK]; uint64_t M[BLK];
    uint32_t k = last - 1 - parity;      // entry of this state's next symbol (valid while i < mine)
    if (n_blk) {
#pragma unroll
        for (int i = 0; i < BLK; i++) e[i] = sf[k - 2 * i];
#pragma unroll
        for (int i = 0; i < BLK; i++) { const uint32_t f_ = (e[i] >> 16) & 0x7fffu; M[i] = __ldg(p.rcp15 + (f_ ? f_ : 1u)); }
    }
    uint32_t idx = 0;
    for (uint32_t blk = 0; blk < n_blk; blk++) {
        uint32_t en[BLK]; uint64_t Mn[BLK];
        const bool more = blk + 1 < n_blk;
        if (more) {
#pragma unroll
            for (int i = 0; i < BLK; i++) en[i] = sf[k - 2 * BLK - 2 * i];
#pragma unroll
            for (int i = 0; i < BLK; i++) { const uint32_t f_ = (en[i] >> 16) & 0x7fffu; Mn[i] = __ldg(p.rcp15 + (f_ ? f_ : 1u)); }
        }
#pragma unroll
        for (int i = 0; i < BLK; i++) DV_RANS_PUT(e[i], M[i], idx + i, k - 2 * i)
        k -= 2 * BLK; idx += BLK;
        if (more) {
#pragma unroll
            for (int i = 0; i < BLK; i++) { e[i] = en[i]; M[i] = Mn[i]; }
        }
    }
    for (; idx < mine; idx++, k -= 2) {
        const uint32_t e1 = sf[k];
        const uint32_t f1 = (e1 >> 16) & 0x7fffu;
        const uint64_t M1 = __ldg(p.rcp15 + (f1 ? f1 : 1u));
        DV_RANS_PUT(e1, M1, idx, k)
    }
#undef DV_RANS_PUT
    if (mine & 31) bits[mine >> 5] = acc;
    // final states: after cnt rotations (and the closing swap of ans.rs:354-360) state 0 lands in slot (cnt even ? 1 : 0)
    uint64_t *cs = reinterpret_cast<uint64_t *>(p.chunk_state + 16 * t);
    cs[((cnt & 1u) ? parity : (parity ^ 1u))] = st;
}

// one warp per chunk record: stack the renormalisation words in symbol order (last symbol first) at the top of the
// chunk's own log region.  Pair i = symbols 2i (state 0) and 2i+1 (state 1) counted from the end; the two emission
// bitmaps are the ballots, so destinations are prefix popcounts.
__global__ void __launch_bounds__(128) encode_pack_kernel(EncodeParams p) {
    const uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t v = (uint32_t)(t / p.max_chunks), j = (uint32_t)(t % p.max_chunks);
    if (v >= p.n_streams) return;
    const bool lit = j >= p.cmd_chunks;
    const uint32_t cj = lit ? j - p.cmd_chunks : j;
    const uint32_t count = p.sf_counts[2 * v + (lit ? 1 : 0)];
    const uint32_t first = cj * NUM_SYMBOLS_BEFORE_FLUSH;
    if (first >= count) return;
    const uint32_t last = min(count, first + NUM_SYMBOLS_BEFORE_FLUSH);
    const uint32_t cnt = last - first;
    uint32_t *sf = p.sf + (uint64_t)v * (p.cmd_cap + p.lit_cap) + (lit ? p.cmd_cap : 0);
    const uint32_t *bits0 = p.emit_bits + (2 * t) * (NUM_SYMBOLS_BEFORE_FLUSH / 64), *bits1 = bits0 + NUM_SYMBOLS_BEFORE_FLUSH / 64;
    const uint32_t n0 = (cnt + 1) >> 1, n1 = cnt >> 1;
    uint32_t w = last;
    const uint32_t below = (1u << lane) - 1u;
    for (uint32_t base = 0; base < n0; base += 32) {
        uint32_t m0 = bits0[base >> 5], m1 = base < n1 ? bits1[base >> 5] : 0u;
        if (n0 - base < 32) m0 &= (1u << (n0 - base)) - 1u;
        if (base < n1 && n1 - base < 32) m1 &= (1u << (n1 - base)) - 1u;
        const uint32_t i = base + lane;
        const bool e0 = (m0 >> lane) & 1u, e1 = (m1 >> lane) & 1u;
        const uint32_t w0 = e0 ? sf[last - 1 - 2 * i] : 0u, w1 = e1 ? sf[last - 2 - 2 * i] : 0u;
        __syncwarp();
        const uint32_t before = __popc(m0 & below) + __popc(m1 & below);
        if (e0) sf[w - 1 - before] = w0;
        if (e1) sf[w - 1 - before - (e0 ? 1u : 0u)] = w1;
        w -= __popc(m0) + __popc(m1);
        __syncwarp();
    }
    if (lane == 0) p.chunk_w[t] = w;
}

// ---------------------------------------------------------------------------------------------------------------
// mux + CRC pass: one warp per stream
// ---------------------------------------------------------------------------------------------------------------
struct VStream {            // one coder's byte stream = its chunks back to back: [16 B states][words w..last)
    const uint32_t *sf;     // log base of this coder
    const uint32_t *chunk_w;
    const uint8_t *chunk_state;
    uint32_t n_chunks, count;
};
__device__ __forceinline__ uint32_t vs_chunk_bytes(const VStream &s, uint32_t j) {
    const uint32_t last = min(s.count, (j + 1) * NUM_SYMBOLS_BEFORE_FLUSH);
    return 16u + 4u * (last - s.chunk_w[j]);
}
// copy bytes [pos, pos+len) of the virtual stream to dst (all lanes of the warp cooperate)
__device__ void vs_copy(const VStream &s, uint32_t pos, uint32_t len, uint8_t *dst, const int lane) {
    uint32_t base = 0;
    for (uint32_t j = 0; j < s.n_chunks && len; j++) {
        const uint32_t cb = vs_chunk_bytes(s, j);
        if (pos < base + cb) {
            const uint32_t o = pos - base, take = min(len, cb - o);
            const uint8_t *st = s.chunk_state + 16 * j;
            const uint8_t *wd = reinterpret_cast<const uint8_t *>(s.sf + s.chunk_w[j]);
            for (uint32_t i = lane; i < take; i += 32) { const uint32_t q = o + i; dst[i] = q < 16 ? st[q] : wd[q - 16]; }
            dst += take; pos += take; len -= take;
        }
        base += cb;
    }
}

__global__ void __launch_bounds__(128) encode_mux_kernel(EncodeParams p) {
    __shared__ uint32_t tab[4][256];
    __shared__ uint32_t x2n[32];
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
    const uint32_t v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (v >= p.n_streams) return;
    if (p.status[v] != ST_OK) { if (lane == 0) p.out_len[v] = 0; return; }
    VStream vs[2];
    const uint32_t lit_chunks = p.max_chunks - p.cmd_chunks;
    for (int c = 0; c < 2; c++) {
        vs[c].sf = p.sf + (uint64_t)v * (p.cmd_cap + p.lit_cap) + (c ? p.cmd_cap : 0);
        const uint64_t t0 = (uint64_t)v * p.max_chunks + (c ? p.cmd_chunks : 0);
        vs[c].chunk_w = p.chunk_w + t0; vs[c].chunk_state = p.chunk_state + 16 * t0;
        vs[c].count = p.sf_counts[2 * v + c];
        vs[c].n_chunks = min(c ? lit_chunks : p.cmd_chunks, (vs[c].count + NUM_SYMBOLS_BEFORE_FLUSH - 1) / NUM_SYMBOLS_BEFORE_FLUSH);
    }
    uint32_t rem[2];
    for (int c = 0; c < 2; c++) { uint32_t n = 0; for (uint32_t j = 0; j < vs[c].n_chunks; j++) n += vs_chunk_bytes(vs[c], j); rem[c] = n; }
    // size of the framed stream: the same walk as below, without the copies
    uint8_t *out = p.out + p.out_off[v];
    const uint64_t cap = p.out_cap[v];
    uint64_t total;
    for (int pass = 0; pass < 2; pass++) {
        uint32_t r[2] = {rem[0], rem[1]}, d[2] = {0, 0};
        uint64_t last_flush[2] = {0, 0}, bytes_flushed = 0, o = 16;
        if (pass == 1 && lane < 16) out[lane] = lane == 0 ? 0xff : lane == 1 ? 0xe5 : lane == 2 ? 0x8c : lane == 3 ? 0x9f : lane == 5 ? (uint8_t)p.window_size : 0;   // make_header, divans_compressor.rs:126-131
        for (;;) {   // flush_internal, mux.rs:500-548: alternate the streams, 65536-byte fixed records while they last
            bool any = false, have = false; uint64_t lf = 0;
            for (int i = 0; i < 2; i++) if (r[i]) { if (!have || last_flush[i] < lf) { lf = last_flush[i]; have = true; } }
            for (int i = 0; i < 2; i++) {
                if ((!have || last_flush[i] <= lf + 131073) && r[i]) {   // (the lag test never fails when all is flushed at close: DESIGN §2)
                    const uint32_t n = r[i];
                    uint32_t take, hdr;
                    if (n == 4096 || n == 16384 || n >= 65536) {   // get_code(.., is_lagging = true), mux.rs:55-78
                        take = n < 16384 ? 4096u : (n < 65536 ? 16384u : 65536u); hdr = 1;
                        if (pass == 1 && lane == 0) out[o] = (uint8_t)(i | ((n < 16384 ? 1 : (n < 65536 ? 2 : 3)) << 4));
                    } else {
                        take = n; hdr = 3;
                        if (pass == 1 && lane == 0) { out[o] = (uint8_t)i; out[o + 1] = (uint8_t)((n - 1) & 0xff); out[o + 2] = (uint8_t)(((n - 1) >> 8) & 0xff); }
                    }
                    if (pass == 1) vs_copy(vs[i], d[i], take, out + o + hdr, lane);
                    o += hdr + take; d[i] += take; r[i] -= take; bytes_flushed += take; last_flush[i] = bytes_flushed; any = true;
                }
            }
            if (!any) break;
        }
        if (pass == 0) {
            total = o + 3 + 8;
            if (total > cap) { if (lane == 0) { p.out_len[v] = total; p.status[v] = ST_NEED_OUTPUT; } return; }
        } else {
            if (lane == 0) { out[o] = 0xff; out[o + 1] = 0xfe; out[o + 2] = 0xff; }   // EOF marker, mux.rs:29
            __syncwarp();
            __threadfence_block();
            const uint64_t tr = o + 3;
            const uint32_t crc = warp_crc32c(tab, x2n, out, (uint32_t)tr, lane);   // codec/mod.rs:541-556
            if (lane == 0) {
                out[tr] = (uint8_t)crc; out[tr + 1] = (uint8_t)(crc >> 8); out[tr + 2] = (uint8_t)(crc >> 16); out[tr + 3] = (uint8_t)(crc >> 24);
                out[tr + 4] = 'a'; out[tr + 5] = 'n'; out[tr + 6] = 's'; out[tr + 7] = '~';   // codec/mod.rs:541-556
                p.out_len[v] = total;
            }
        }
    }
}

#endif  // !DV_BLEND

#ifdef DV_BLEND
void launch_encode_model_blend(const EncodeParams &p, uint32_t n_blocks, cudaStream_t st) {
    size_t smem = (size_t)(DECODE_BLOCK_THREADS / 16) * SMEM_BYTES_PER_GROUP;
    encode_model_kernel<true><<<n_blocks, DECODE_BLOCK_THREADS, smem, st>>>(p);
}
#else
void launch_encode_model(const EncodeParams &p, uint32_t n_blocks, cudaStream_t st) {
    size_t smem = (size_t)(DECODE_BLOCK_THREADS / 16) * SMEM_BYTES_PER_GROUP;
    encode_model_kernel<false><<<n_blocks, DECODE_BLOCK_THREADS, smem, st>>>(p);
}
// M[f] = floor((2^64 - 1) / f), f = 1..32767 (entry 0 unused)
__global__ void rcp15_init_kernel(uint64_t *tab) {
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < 32768) tab[f] = f ? 0xffffffffffffffffull / (uint64_t)f : 0ull;
}
void launch_rcp15_init(uint64_t *tab, cudaStream_t st) { rcp15_init_kernel<<<32768 / 256, 256, 0, st>>>(tab); }
void launch_encode_flush_mux(const EncodeParams &p, cudaStream_t st) {
    const uint64_t items = (uint64_t)p.n_streams * p.max_chunks;
    encode_flush_kernel<<<(unsigned)((2 * items + 127) / 128), 128, 0, st>>>(p);
    encode_pack_kernel<<<(unsigned)((items * 32 + 127) / 128), 128, 0, st>>>(p);
    encode_mux_kernel<<<(p.n_streams + 3) / 4, 128, 0, st>>>(p);
}
int encode_max_blocks_per_sm() {
    const int nb = stream_kernel_blocks_per_sm(encode_model_kernel<false>, DECODE_BLOCK_THREADS, (size_t)(DECODE_BLOCK_THREADS / 16) * SMEM_BYTES_PER_GROUP);
    return nb;
}

#endif  // DV_BLEND

}  // namespace dv
