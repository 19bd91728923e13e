// dv_core.cuh -- the encoder's converged per-nibble core and literal fast path (dv_encode.cu), and the warp CRC32C of the
// framing and mux passes (dv_kernels.cu, dv_encode.cu).
#pragma once
#include "dv_engine_kernel.cuh"
#include "dv_blend.cuh"
#include "dv_kernels.h"

namespace dv {

__device__ __forceinline__ uint32_t crc_step(const uint32_t *tab, uint32_t crc, uint32_t byte) {
    return tab[(crc ^ byte) & 0xff] ^ (crc >> 8);
}

// Encoder: log one coded nibble.  A frequency <= 0 (a stream-supplied speed wrapped an i16 counter) cannot be coded: the
// reference encoder panics on it and the oracle refuses the stream (ans_enc_put), so the stream fails, as in the blend core.
// An idle group codes the dummy prior and is never failed.
// TALLY (the cost-only pass, encode_model_kernel<BLEND, true>): nothing is logged.  The coder's `p` is the cost table and its
// `a` (unused by the encoder otherwise) the running cost; every lane of the group adds the same value.
template <bool TALLY = false>
__device__ __forceinline__ void enc_log(St &s, const G2 g, int start, int freq) {
    if (freq <= 0 && s.state != S_IDLE) s.status = ST_FAIL;
    if constexpr (TALLY) s.cur.a += __ldg(s.cur.p + ((uint32_t)freq & 0x7fffu));
    else if (g.store0) const_cast<uint32_t *>(s.cur.p)[s.cur.left] = ((uint32_t)start & 0xffffu) | ((uint32_t)freq << 16);
    s.cur.left++;
}

// The encoder's converged nibble core.  Every lane of the warp executes it every iteration, unpredicated: a group without
// work codes against its slot's dummy CDF with a parked coder (no memory side effects that matter).
template <bool TALLY = false>
__device__ __forceinline__ int nibble_core_enc(St &s, const Next &nx, const G2 g) {
    const Grp gg = {FULL, g.l16};
    const int c = nx.cdf[g.l16], maxv = nx.cdf[15];
    const int inc = (int)(short)(nx.speed & 0xffff), lim = nx.speed >> 16;
    const int sym = nx.sym;
    int start, freq;
    if (!__any_sync(FULL, nx.cdf2 != nullptr)) {
        int cum = cdf_div(c, maxv);
        int hi = __shfl_sync(FULL, cum, sym, 16);
        int lo = __shfl_sync(FULL, cum, (sym - 1) & 15, 16);
        if (sym == 0) lo = 0;
        start = (int)(short)(lo + 1); freq = (int)(short)(hi - lo - 1);   // "major hax", probability/interface.rs:103-104
        enc_log<TALLY>(s, g, start, freq);
        int c2 = cdf_blend(gg, c, maxv, sym, inc, lim);
        nx.cdf[g.l16] = (int16_t)c2;
        return sym;
    }
    // ---- at least one group mixes two priors (dynamic context mixing >= 2, codec/literal.rs:219-243) ----
    const bool mixg = nx.cdf2 != nullptr;
    int cc = c, mc = maxv;
    if (mixg) { cc = nx.cdf2[g.l16]; mc = nx.cdf2[15]; }
    Weights w = nx.mix_hi ? s.c->w_hi : s.c->w_lo;
    int prod = mc * maxv;
    int lz = prod == 0 ? 32 : __clz(prod); if (lz > 17) lz = 17;
    int shift = 17 - lz;
    int mixr = w.norm, inv = (1 << 15) - mixr;
    int rs = (cc * maxv) >> shift, ro = (c * mc) >> shift;
    int ca = (int)(short)((int)((unsigned)rs * (unsigned)mixr + (unsigned)ro * (unsigned)inv + 1u) >> 15);   // frequentist_cdf.rs:58-72
    int ma = __shfl_sync(FULL, ca, 15, 16);
    int cu = mixg ? ca : c, mu = mixg ? ma : maxv;
    int cum = cdf_div(cu, mu);
    int hi = __shfl_sync(FULL, cum, sym, 16);
    int lo = __shfl_sync(FULL, cum, (sym - 1) & 15, 16);
    if (sym == 0) lo = 0;
    start = (int)(short)(lo + 1); freq = (int)(short)(hi - lo - 1);
    int f_cm = cdf_freq(gg, cc, mc, sym);
    int f_nb = cdf_freq(gg, c, maxv, sym);
    enc_log<TALLY>(s, g, start, freq);
    if (mixg) {
        weights_update(w, f_cm, f_nb, freq);
        if (nx.mix_hi) s.c->w_hi = w; else s.c->w_lo = w;
        const int sp = nx.mix_hi ? s.c->ad_cm_hi : s.c->ad_cm_lo;
        int c2 = cdf_blend(gg, cc, mc, sym, (int)(short)(sp & 0xffff), sp >> 16);
        nx.cdf2[g.l16] = (int16_t)c2;
    }
    int s2 = cdf_blend(gg, c, maxv, sym, inc, lim);
    nx.cdf[g.l16] = (int16_t)s2;
    return sym;
}

// ---- CRC32C of one buffer by a whole warp: 32 contiguous segments, then a shuffle tree of CRC combinations ----
// (crc(A || B) = crc(A) * x^(8 |B|) mod P  xor  crc(B), polynomials in the reflected representation)
constexpr uint32_t CRC32C_POLY = 0x82F63B78u;
__device__ __forceinline__ uint32_t gf_mul(uint32_t a, uint32_t b) {   // a * b mod P
    uint32_t p = 0;
#pragma unroll 4
    for (int i = 0; i < 32; i++) {
        p ^= (a & 0x80000000u) ? b : 0u;
        a <<= 1;
        b = (b & 1u) ? (b >> 1) ^ CRC32C_POLY : (b >> 1);
    }
    return p;
}
// x^(8 n) mod P by square-and-multiply over x2n[k] = x^(2^k) mod P
__device__ __forceinline__ uint32_t gf_x8n(const uint32_t *x2n, uint32_t n) {
    uint32_t p = 0x80000000u;   // x^0
    for (uint32_t k = 3; n; n >>= 1, k++)
        if (n & 1u) p = gf_mul(x2n[k & 31], p);
    return p;
}
__device__ __forceinline__ uint32_t crc32c_bytes(const uint32_t (*tab)[256], const uint8_t *q, uint32_t n) {
    uint32_t crc = 0xffffffffu, i = 0;
    for (; i < n && (((uintptr_t)(q + i)) & 3); i++) crc = crc_step(tab[0], crc, q[i]);
    for (; i + 4 <= n; i += 4) {
        const uint32_t w = *reinterpret_cast<const uint32_t *>(q + i) ^ crc;
        crc = tab[3][w & 0xff] ^ tab[2][(w >> 8) & 0xff] ^ tab[1][(w >> 16) & 0xff] ^ tab[0][w >> 24];
    }
    for (; i < n; i++) crc = crc_step(tab[0], crc, q[i]);
    return ~crc;
}
static __device__ uint32_t warp_crc32c(const uint32_t (*tab)[256], const uint32_t *x2n, const uint8_t *buf, uint32_t len, const int lane) {
    const uint32_t seg = (len / 32u) & ~3u;
    const uint32_t my_off = seg * (uint32_t)lane;
    uint32_t my_len = lane == 31 ? len - 31u * seg : seg;
    uint32_t crc = crc32c_bytes(tab, buf + my_off, my_len);
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
        const uint32_t crc2 = __shfl_down_sync(FULL, crc, s), len2 = __shfl_down_sync(FULL, my_len, s);
        if ((lane & (2 * s - 1)) == 0) {
            crc = len2 ? (gf_mul(gf_x8n(x2n, len2), crc) ^ crc2) : crc;
            my_len += len2;
        }
    }
    return __shfl_sync(FULL, crc, 0);
}

// sign-extending 16-bit load (LDG.E.S16: no separate PRMT); ordered against the surrounding stores by the memory clobber
__device__ __forceinline__ int ld_s16(const char *p) { int v; asm volatile("ld.global.s16 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
// One literal nibble coded against the mix of two priors (dynamic context mixing >= 2, codec/literal.rs:219-259):
// `nb` = the stride prior, `cm` = the context-map prior, weights `w` (model_weights[high nibble ? 1 : 0]).
// Three phases so that the loop can issue the loads of the next nibble before the long finish of the current one.
struct MixVals { int c, maxv, cc, mc; };
__device__ __forceinline__ MixVals mix_load(const G2 g, const char *nb, const char *cm) {
    MixVals v; v.c = ld_s16(nb + 2 * g.l16); v.maxv = ld_s16(nb + 30); v.cc = ld_s16(cm + 2 * g.l16); v.mc = ld_s16(cm + 30); return v;
}
struct MixSym { int sym, ca, ma; };
__device__ __forceinline__ MixSym mix_search(const MixVals v, const Weights &w, const int sym) {
    const int prod = v.mc * v.maxv;
    int lz = prod == 0 ? 32 : __clz(prod); if (lz > 17) lz = 17;
    const int shift = 17 - lz;
    const int mixr = w.norm, inv = (1 << 15) - mixr;
    const int rs = (v.cc * v.maxv) >> shift, ro = (v.c * v.mc) >> shift;
    MixSym r;
    r.ca = (int)(short)((int)((unsigned)rs * (unsigned)mixr + (unsigned)ro * (unsigned)inv + 1u) >> 15);   // frequentist_cdf.rs:58-72
    r.ma = __shfl_sync(FULL, r.ca, 15, 16);
    r.sym = sym;
    return r;
}
template <bool TALLY>
__device__ __forceinline__ void mix_finish(Coder &k, const G2 g, char *nb, char *cm, const MixVals v, const MixSym ms, Weights &w,
                                           const int nb_inc, const int nb_lim, const int cm_inc, const int cm_lim, bool &refused) {
    const int sym = ms.sym;
    // cumulative values of the three CDFs at sym and sym-1: two registers, four shuffles
    const int cum_a = cdf_div(ms.ca, ms.ma);
    const int cum_pn = cdf_div(v.cc, v.mc) | (cdf_div(v.c, v.maxv) << 16);
    const int prev = (sym - 1) & 15;
    const int hi_a = __shfl_sync(FULL, cum_a, sym, 16), hi_pn = __shfl_sync(FULL, cum_pn, sym, 16);
    int lo_a = __shfl_sync(FULL, cum_a, prev, 16), lo_pn = __shfl_sync(FULL, cum_pn, prev, 16);
    if (sym == 0) { lo_a = 0; lo_pn = 0; }
    const int start = (int)(short)(lo_a + 1), freq = (int)(short)(hi_a - lo_a - 1);
    const int f_cm = (int)(short)((hi_pn & 0xffff) - (lo_pn & 0xffff) - 1);
    const int f_nb = (int)(short)(((unsigned)hi_pn >> 16) - ((unsigned)lo_pn >> 16) - 1);
    // small speeds keep both priors' steps >= 3, but their average can still round to a step of 1: freq 0 (see enc_log)
    refused |= freq <= 0;
    if constexpr (TALLY) k.a += __ldg(k.p + ((uint32_t)freq & 0x7fffu));
    else if (g.store0) const_cast<uint32_t *>(k.p)[k.left] = ((uint32_t)start & 0xffffu) | ((uint32_t)freq << 16);
    k.left++;
    weights_update32(w, f_cm, f_nb, freq);
    const Grp gg = {FULL, g.l16};
    const int c2 = cdf_blend(gg, v.cc, v.mc, sym, cm_inc, cm_lim);
    const int s2 = cdf_blend(gg, v.c, v.maxv, sym, nb_inc, nb_lim);
    *reinterpret_cast<int16_t *>(cm + 2 * g.l16) = (int16_t)c2; *reinterpret_cast<int16_t *>(nb + 2 * g.l16) = (int16_t)s2;
}

// The cost of a stream's literal nibbles (encode_speeds_kernel's cost pass): hi = the high nibbles, lit = all of them.
struct LitHalves { uint64_t hi, lit; };

// The encoder's converged literal fast path: when both groups of the warp sit at the start of a literal byte, code whole
// bytes (high nibble, low nibble, context of the next byte) back to back without going through the state-machine dispatch.
// This is code_nibble_array (codec/literal.rs:261-394) for two streams at once.  The common case -- no dynamic context
// mixing and one mixing-mask value for the whole map -- gets a loop with every selector hoisted out.
// HALVES (TALLY as well): the cost of the high nibbles is added to hv->hi; the caller sums the whole delta of the coder's cost.
// The plain loop's sums are read by no call today (the speeds calls read halves only at dynamic mixing 2, which takes the mixing
// loop); they are kept so that the cost pass reports the same halves whichever loop codes a literal.
template <bool TALLY, bool HALVES = false>
__device__ __forceinline__ void literal_fast_enc(St &s, Next &nx, const G2 g, LitHalves *hv = nullptr) {
    const uint32_t n = min(s.lit_left, __shfl_xor_sync(FULL, s.lit_left, 16));
    const bool simple = __all_sync(FULL, !s.mixing_trait && s.lit_cfg >= 0 && s.speeds_small);
    if (simple) {
        const int cfg = s.lit_cfg;
        const uint32_t mm = (cfg & 0x100) ? 0xffu : 0u, o1 = (cfg & 0x200) ? 0xfu : 0u, fc = (cfg & 0x400) ? 0xffu : 0u;
        const uint32_t sh = (uint32_t)(cfg >> 2) & 63u, which = (uint32_t)cfg & 3u;
        const bool ro = (cfg & 0x800) != 0;   // mixing value 2: the flat prior, never adapted (one CDF, index scale 0)
        const int inc = ro ? 0 : (int)(short)(s.ad_stride & 0xffff), lim = ro ? 0x7fff : (s.ad_stride >> 16);
        const uint32_t scale = ro ? 0u : 32u;
        char *const hi_tab = ro ? reinterpret_cast<char *>(A_misc(s, MI_FLAT)) : reinterpret_cast<char *>(A_lit(s, true) + (size_t)which * 256 * 256 * 16);
        char *const lo_tab = ro ? reinterpret_cast<char *>(A_misc(s, MI_FLAT)) : reinterpret_cast<char *>(A_lit(s, false) + (size_t)which * 256 * 256 * 16);
        const uint8_t *const lcm = A_lcm(s) + (s.btype_last << 6);
        const uint8_t *const lut = s.tables + TB_CTX + 512 * s.pred_mode;
        const uint32_t pm = s.pred_mode;
        const uint8_t *src = s.c->in.lits + s.c->e0 + (s.c->e1 - s.lit_left);
        unsigned long long l8 = s.l8;
        uint32_t ctx = s.lit_ctx;
        uint8_t *dst = s.out + s.out_pos;
        Coder k = s.cur;
        const uint32_t src_last = s.lit_left - 1;                   // (lit_left >= 1 here)
        const uint32_t pm_shift = pm == 1 ? 2u : 0u;
        uint64_t hh = 0;
        uint32_t done = 0;
        while (done < n) {
            uint32_t m = n - done;
            // Software pipeline (the loads of the NEXT prior are issued before the bookkeeping of the CURRENT nibble):
            //   search(hi) -> load(lo) -> finish(hi) -> search(lo) -> context -> load(next hi) -> finish(lo)
            // The high and low tables never alias, so the early loads cannot overtake a store to the same CDF; the
            // __syncwarp()s order each store against the next load of the same table across lanes.
            // The loop uses plain 32-bit arithmetic where the reference wraps i16: only entered when speeds_small says no
            // adaptive value can leave [0, 0x7fff] (dv_engine.cuh: speed_is_small).
            char *ph = hi_tab + (ctx * 256u + ((uint32_t)(l8 >> sh) & mm & (~o1 & 0xffu))) * scale;
            __syncwarp();
            int ch = ld_s16(ph + 2 * g.l16), mh = ld_s16(ph + 30);
            uint32_t nxt_in = src[done];                              // the input byte is fetched one iteration ahead
            for (uint32_t i = 0; i < m; i++) {
                const uint32_t ssb = (uint32_t)(l8 >> sh) & 0xffu;
                const uint32_t byte_in = nxt_in;
                nxt_in = src[min(done + i + 1, src_last)];
                // -- high nibble
                const int h = (int)(byte_in >> 4);
                const uint32_t ib = (mm & ssb) | ((~mm & 0xffu) & ctx), ic = ((uint32_t)h & fc) | ((ctx & o1) << 4);
                char *const pl = lo_tab + (ic * 256u + ib) * scale;
                __syncwarp();
                const int cl = ld_s16(pl + 2 * g.l16), ml = ld_s16(pl + 30);
                // -- high nibble: finish
                {
                    const int cum = cdf_div_pos(ch, mh);
                    const int hi = __shfl_sync(FULL, cum, h, 16);
                    int lo = __shfl_sync(FULL, cum, (h - 1) & 15, 16);
                    if (h == 0) lo = 0;
                    const uint32_t start = (uint32_t)(lo + 1), freq = (uint32_t)(hi - lo - 1);   // "major hax", probability/interface.rs:103-104
                    if constexpr (TALLY) { const uint32_t cst = __ldg(k.p + (freq & 0x7fffu)); k.a += cst; if constexpr (HALVES) hh += cst; }
                    else if (g.store0) const_cast<uint32_t *>(k.p)[k.left] = (start & 0xffffu) | (freq << 16);
                    k.left++;
                    int c2 = ch + ((g.l16 >= h) ? inc : 0);
                    if (mh + inc >= lim) { const int t = c2 + g.l16 + 1; c2 = t - (t >> 2); }
                    *reinterpret_cast<int16_t *>(ph + 2 * g.l16) = (int16_t)c2;
                }
                // -- low nibble
                const int l = (int)(byte_in & 0xf);
                const uint32_t cur = ((uint32_t)l | ((uint32_t)h << 4)) & 0xff;
                l8 = (l8 >> 8) | ((unsigned long long)cur << 56);   // push_literal_byte, codec/interface.rs:280-284
                if (g.store0) dst[done + i] = (uint8_t)cur;
                uint32_t sel = (cur >> pm_shift) & 0x3fu;             // get_prev_word_context, codec/literal.rs:87-117: LSB6 / MSB6
                if (pm >= 2) sel = __ldg(lut + cur) | __ldg(lut + 256 + ((uint32_t)(l8 >> 48) & 0xff));   // UTF8 / SIGN
                ctx = lcm[sel];
                ph = hi_tab + (ctx * 256u + ((uint32_t)(l8 >> sh) & mm & (~o1 & 0xffu))) * scale;
                __syncwarp();
                ch = ld_s16(ph + 2 * g.l16); mh = ld_s16(ph + 30);   // speculative on the last byte: a valid, initialised slab
                // -- low nibble: finish
                {
                    const int cum = cdf_div_pos(cl, ml);
                    const int hi = __shfl_sync(FULL, cum, l, 16);
                    int lo = __shfl_sync(FULL, cum, (l - 1) & 15, 16);
                    if (l == 0) lo = 0;
                    const uint32_t start = (uint32_t)(lo + 1), freq = (uint32_t)(hi - lo - 1);
                    if constexpr (TALLY) k.a += __ldg(k.p + (freq & 0x7fffu));
                    else if (g.store0) const_cast<uint32_t *>(k.p)[k.left] = (start & 0xffffu) | (freq << 16);
                    k.left++;
                    int c2 = cl + ((g.l16 >= l) ? inc : 0);
                    if (ml + inc >= lim) { const int t = c2 + g.l16 + 1; c2 = t - (t >> 2); }
                    *reinterpret_cast<int16_t *>(pl + 2 * g.l16) = (int16_t)c2;
                }
            }
            done += m;
        }
        s.cur = k; s.l8 = l8; s.lit_ctx = ctx; s.out_pos += done; s.lit_left -= done;
        if constexpr (HALVES) hv->hi += hh;
        enter_lit_nibble<true, true>(s, nx);
        return;
    }
    if (__all_sync(FULL, s.mixing_trait && s.lit_cfg >= 0 && s.speeds_small)) {
        // every group mixes the stride prior with the context-map prior, one mixing-mask value for the whole map
        const int cfg = s.lit_cfg;
        const uint32_t mm = (cfg & 0x100) ? 0xffu : 0u, o1 = (cfg & 0x200) ? 0xfu : 0u, fc = (cfg & 0x400) ? 0xffu : 0u;
        const uint32_t sh = (uint32_t)(cfg >> 2) & 63u, which = (uint32_t)cfg & 3u;
        const bool ro = (cfg & 0x800) != 0;
        const int inc = ro ? 0 : (int)(short)(s.ad_stride & 0xffff), lim = ro ? 0x7fff : (s.ad_stride >> 16);
        const int ch_inc = (int)(short)(s.c->ad_cm_hi & 0xffff), ch_lim = s.c->ad_cm_hi >> 16;
        const int cl_inc = (int)(short)(s.c->ad_cm_lo & 0xffff), cl_lim = s.c->ad_cm_lo >> 16;
        int16_t *const hi_base = A_lit(s, true) + (size_t)which * 256 * 256 * 16;
        int16_t *const lo_base = A_lit(s, false) + (size_t)which * 256 * 256 * 16;
        char *const cmb = reinterpret_cast<char *>(A_litcm(s));
        char *const hi_tab = reinterpret_cast<char *>(hi_base), *const lo_tab = reinterpret_cast<char *>(lo_base);
        const uint8_t *const lcm = A_lcm(s) + (s.btype_last << 6);
        const uint8_t *const lut = s.tables + TB_CTX + 512 * s.pred_mode;
        const uint32_t pm = s.pred_mode;
        const uint8_t *src = s.c->in.lits + s.c->e0 + (s.c->e1 - s.lit_left);
        unsigned long long l8 = s.l8;
        uint32_t ctx = s.lit_ctx;
        uint8_t *dst = s.out + s.out_pos;
        Coder k = s.cur;
        Weights wh = s.c->w_hi, wl = s.c->w_lo;
        bool refused = false;
        uint64_t hh = 0;
        uint32_t done = 0;
        while (done < n) {
            uint32_t m = n - done;
            // search(hi) -> load(lo) -> finish(hi) -> search(lo) -> context -> load(next hi) -> finish(lo); the stride tables
            // of the two nibbles are distinct and so are their context-map regions (FirstNibble / SecondNibble), so an
            // early load never overtakes a store to the same CDF
            char *nbh = hi_tab + (ctx * 256u + ((uint32_t)(l8 >> sh) & mm & (~o1 & 0xffu))) * 32u, *cmh = cmb + ctx * 32u;
            __syncwarp();
            MixVals vh = mix_load(g, nbh, cmh);
            for (uint32_t i = 0; i < m; i++) {
                const uint32_t ssb = (uint32_t)(l8 >> sh) & 0xffu;
                const uint32_t byte_in = src[done + i];
                const MixSym sh_ = mix_search(vh, wh, (int)(byte_in >> 4));
                const uint32_t h = (uint32_t)sh_.sym;
                const uint32_t ib = (mm & ssb) | ((~mm & 0xffu) & ctx), ic = (h & fc) | ((ctx & o1) << 4);
                char *const nbl = lo_tab + (ic * 256u + ib) * 32u, *const cml = cmb + (256u + h + 16u * ctx) * 32u;
                __syncwarp();
                const MixVals vl = mix_load(g, nbl, cml);
                const uint64_t a_h = k.a;
                mix_finish<TALLY>(k, g, nbh, cmh, vh, sh_, wh, inc, lim, ch_inc, ch_lim, refused);
                if constexpr (HALVES) hh += k.a - a_h;
                const MixSym sl_ = mix_search(vl, wl, (int)(byte_in & 0xf));
                const uint32_t cur = ((uint32_t)sl_.sym | (h << 4)) & 0xff;
                l8 = (l8 >> 8) | ((unsigned long long)cur << 56);
                if (g.store0) dst[done + i] = (uint8_t)cur;
                uint32_t sel = (cur >> (pm == 1 ? 2u : 0u)) & 0x3fu;
                if (pm >= 2) sel = __ldg(lut + cur) | __ldg(lut + 256 + ((uint32_t)(l8 >> 48) & 0xff));
                ctx = lcm[sel];
                nbh = hi_tab + (ctx * 256u + ((uint32_t)(l8 >> sh) & mm & (~o1 & 0xffu))) * 32u; cmh = cmb + ctx * 32u;
                __syncwarp();
                vh = mix_load(g, nbh, cmh);   // speculative on the last byte: initialised slabs
                mix_finish<TALLY>(k, g, nbl, cml, vl, sl_, wl, inc, lim, cl_inc, cl_lim, refused);
            }
            done += m;
        }
        s.cur = k; s.l8 = l8; s.lit_ctx = ctx; s.out_pos += done; s.lit_left -= done;
        s.c->w_hi = wh; s.c->w_lo = wl;
        if constexpr (HALVES) hv->hi += hh;
        if (refused) s.status = ST_FAIL;
        enter_lit_nibble<true, true>(s, nx);
        return;
    }
    for (uint32_t i = 0; i < n; i++) {
        __syncwarp();
        const uint64_t a_h = s.cur.a;
        int h = nibble_core_enc<TALLY>(s, nx, g);
        if constexpr (HALVES) hv->hi += s.cur.a - a_h;
        s.lit_h = (uint32_t)h;
        enter_lit_nibble<true, false>(s, nx);
        __syncwarp();
        int l = nibble_core_enc<TALLY>(s, nx, g);
        uint32_t cur = ((uint32_t)l | ((uint32_t)h << 4)) & 0xff;
        s.l8 = (s.l8 >> 8) | ((unsigned long long)cur << 56);   // push_literal_byte, codec/interface.rs:280-284
        if (g.store0) s.out[s.out_pos] = (uint8_t)cur;
        s.out_pos++;
        s.lit_left--;
        lit_context(s);
        enter_lit_nibble<true, true>(s, nx);
    }
}

// the encoder's nibble core of the kernel's probability model
template <bool BLEND, bool TALLY>
__device__ __forceinline__ int core_dispatch(St &s, const Next &nx, const G2 g) {
    if constexpr (BLEND) return nibble_core_blend<true, TALLY>(s, nx, g);
    else return nibble_core_enc<TALLY>(s, nx, g);
}

}  // namespace dv
