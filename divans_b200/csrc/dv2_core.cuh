// dv2_core.cuh -- the decode engine of round 2 ("v2"), templated on the lanes that share one stream:
//   LPG = 16: two streams per warp, lane j of a group holds CDF element j;
//   LPG = 8:  four streams per warp, lane j holds elements 2j and 2j+1 packed in one register (c[2j] | c[2j+1] << 16).
//
// What bounds the decoder: with 4096 streams a GPU of ~130-150 SMs has fewer than 8 streams per warp scheduler, each one a
// serial dependency chain -- a warp issues one instruction every 5-6 cycles, so the time of a batch is
//     bytes per stream x (warp instructions per byte) x ~5.5 cycles     (until the issue slots run out, at larger batches)
// and the levers are the instructions in the per-byte loop and the streams that share each of them.  v2 versus the
// round-1 loop (dv_core.cuh, still used by the encoder's model pass):
//   * generation tags instead of initialisation: a literal prior carries a 16-bit tag in the free sign bits of its elements; a
//     prior whose tag differs from the stream's generation reads as the default CDF and takes the tag with its first write
//     (dv_common.cuh): no per-stream initialisation of literal priors at all (round 1 wrote 640 KB of defaults per 64 KiB
//     stream -- 11x the algorithmic DRAM traffic), no extra memory access (the fast loop searches speculatively with the
//     loaded values and repeats the search in the rare iteration where some group's tag ballot fails);
//   * literal context in ONE lookup: T2[byte][class of the byte before] (OFF_T2), rebuilt per PredictionMode / block switch,
//     replaces lut0 / lut1 / context-map (three dependent loads, codec/literal.rs:87-117);
//   * slots are 16 MiB aligned: every address inside a slot is (slot_hi : slot_lo + offset) -- one 32-bit add, no 64-bit
//     address arithmetic in the loop;
//   * exact start/freq (probability/interface.rs:97-108) from an under-estimated reciprocal 2^32/max, one multiply-high and
//     ONE fix-up per quotient;
//   * the next payload word of the eager-refill coder is always in a register; decoded literals leave as aligned 8-byte
//     stores of last_8_literals;
//   * LPG = 8: blend and rescale (frequentist_cdf.rs:74-85) are one packed add / one packed subtract for two elements;
//   * literal priors in a dense order (lit_index_hi / lit_index_lo, dv_common.cuh): the priors a stream uses share cache lines,
//     so that the hot priors of the resident streams stay in L1.
// Decode only.
#pragma once
#include "dv_engine_kernel.cuh"
#include "dv_kernels.h"

namespace dv {

__device__ __forceinline__ const char *mk_ptr(const uint32_t lo, const uint32_t hi) {
    unsigned long long p; asm("mov.b64 %0, {%1, %2};" : "=l"(p) : "r"(lo), "r"(hi)); return reinterpret_cast<const char *>(p);
}
__device__ __forceinline__ uint32_t ld_u32(const void *p) { uint32_t v; asm volatile("ld.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ uint32_t ld_u16g(const void *p) { uint32_t v; asm volatile("ld.global.u16 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ int ld_s16g(const void *p) { int v; asm volatile("ld.global.s16 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ uint32_t ld_u8g(const void *p) { uint32_t v; asm volatile("ld.global.u8 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void st_u32(const void *p, uint32_t v) { asm volatile("st.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void st_u16(const void *p, uint32_t v) { asm volatile("st.global.u16 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
// streaming accesses (touched once: payload words, decoded output): evict-first, so that they do not push the priors out of L2
__device__ __forceinline__ uint32_t ld_stream_u32(const void *p) { uint32_t v; asm volatile("ld.global.cs.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void st_stream_u64(const void *p, unsigned long long v) { asm volatile("st.global.cs.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
__device__ __forceinline__ void st_u8(const void *p, uint32_t v) { asm volatile("st.global.u8 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t ld_shared_u8(const uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ void st_shared_u8(const uint32_t a, const uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }

// tag bits of this lane's element(s): element i carries bit i of the 16-bit generation in its bit 15
template <int LPG> __device__ __forceinline__ uint32_t lane_tag(const uint32_t gen, const int li) {
    return LPG == 16 ? ((gen >> li) & 1u) << 15 : ((((gen >> (2 * li)) & 1u) << 15) | (((gen >> (2 * li + 1)) & 1u) << 31));
}
constexpr uint32_t TAG_BITS16 = 0x8000u, TAG_BITS8 = 0x80008000u;

// the prior of one nibble as a lane holds it: LPG 16 -> element `li` in the low half; LPG 8 -> elements 2li | (2li+1) << 16
template <int LPG> __device__ __forceinline__ uint32_t default_elems(const int li) {   // [4,8,...,64], frequentist_cdf.rs:17-23
    return LPG == 16 ? (uint32_t)(4 * li + 4) : ((uint32_t)(8 * li + 4) | ((uint32_t)(8 * li + 8) << 16));
}
template <int LPG> __device__ __forceinline__ uint32_t load_elems(const char *cdf, const int li) {
    return LPG == 16 ? ld_u16g(cdf + 2 * li) : ld_u32(cdf + 4 * li);
}
template <int LPG> __device__ __forceinline__ void store_elems(const char *cdf, const int li, const uint32_t v) {
    if (LPG == 16) st_u16(cdf + 2 * li, v); else st_u32(cdf + 4 * li, v);
}

// ---------------------------------------------------------------------------------------------------------------
// generic nibble core (command nibbles, literals outside the fast loop, dynamic context mixing): the reference's i16
// semantics, wrap included, on one (LPG 16) or two (LPG 8) elements per lane.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int blend_elem(int c, int elem, int maxv, int sym, int inc, int lim) {   // frequentist_cdf.rs:74-85, i16 wrapping
    int c2 = (int)(short)(c + ((elem >= sym) ? inc : 0));
    const int nm = (int)(short)(maxv + inc);
    if (nm >= lim) { const int t = (int)(short)(c2 + elem + 1); c2 = (int)(short)(t - (t >> 2)); }
    return c2;
}
// cumulative values (c << 15) / max of elements `sym` and `sym - 1`, fetched from the lanes that own them
template <int LPG> __device__ __forceinline__ void cum_pair(const int cum0, const int cum1, const int sym, int &hi, int &lo) {
    const int prev = (sym - 1) & 15;
    if (LPG == 16) { hi = __shfl_sync(FULL, cum0, sym, 16); lo = __shfl_sync(FULL, cum0, prev, 16); }
    else { hi = __shfl_sync(FULL, (sym & 1) ? cum1 : cum0, sym >> 1, 8); lo = __shfl_sync(FULL, (prev & 1) ? cum1 : cum0, prev >> 1, 8); }
    if (sym == 0) lo = 0;
}
// index of the first element i with r < c[i], else 15 (probability/interface.rs:152-185)
template <int LPG> __device__ __forceinline__ int first_true(const bool p0, const bool p1, const G2 g) {
    if (LPG == 16) {
        const unsigned b = __ballot_sync(FULL, p0 || g.l16 == 15);
        return __ffs((b >> g.shift) & 0xffffu) - 1;
    }
    const unsigned b0 = __ballot_sync(FULL, p0), b1 = __ballot_sync(FULL, p1 || g.l16 == 7);
    const int f0 = __ffs((b0 >> g.shift) & 0xffu), f1 = __ffs((b1 >> g.shift) & 0xffu);   // element 2j: bit j of b0; 2j+1: bit j of b1
    return min(f0 ? 2 * f0 - 2 : 99, 2 * f1 - 1);
}

template <int LPG>
__device__ __forceinline__ int nibble_core_v2(St &s, const Next &nx, const G2 g) {
    const int li = g.l16;
    const char *const cdf = reinterpret_cast<const char *>(nx.cdf);
    uint32_t raw = load_elems<LPG>(cdf, li);
    int maxv = ld_s16g(cdf + 30);
    // tagged literal prior: every lane of the group must see its bit(s) of the stream's generation, else the prior belongs to an
    // older stream and reads as the default CDF
    const uint32_t tbits = LPG == 16 ? TAG_BITS16 : TAG_BITS8, mytag = lane_tag<LPG>(s.gen, li);
    const unsigned okb = __ballot_sync(FULL, !nx.tagged || (raw & tbits) == mytag);
    if (nx.tagged) {
        const unsigned gm = (LPG == 16 ? 0xffffu : 0xffu) << g.shift;
        if ((okb & gm) == gm) { raw &= ~tbits; maxv &= 0x7fff; } else { raw = default_elems<LPG>(li); maxv = 64; }
    }
    __syncwarp();
    const int e0 = LPG == 16 ? li : 2 * li, e1 = 2 * li + 1;
    const int c0 = (int)(short)(raw & 0xffffu), c1 = (int)(short)(raw >> 16);   // (c1: LPG 8 only)
    const int inc = (int)(short)(nx.speed & 0xffff), lim = nx.speed >> 16;
    int sym, start, freq, hi, lo;
    if (!__any_sync(FULL, nx.cdf2 != nullptr)) {
        coder_fill(s.cur);
        const int off = (int)(s.cur.a & 0x7fff);
        const int r = (int)(short)((off * maxv) >> 15);                     // probability/interface.rs:140
        sym = first_true<LPG>(r < c0, r < c1, g);
        cum_pair<LPG>(cdf_div(c0, maxv), LPG == 16 ? 0 : cdf_div(c1, maxv), sym, hi, lo);
        start = (int)(short)(lo + 1); freq = (int)(short)(hi - lo - 1);   // "major hax", probability/interface.rs:103-104
        coder_advance(s.cur, start, freq);
        const int n0 = blend_elem(c0, e0, maxv, sym, inc, lim);
        const int n1 = LPG == 16 ? 0 : blend_elem(c1, e1, maxv, sym, inc, lim);
        store_elems<LPG>(cdf, li, (((uint32_t)n0 & 0xffffu) | ((uint32_t)n1 << 16)) | (nx.tagged ? mytag : 0u));
        return sym;
    }
    // ---- at least one group mixes two priors (dynamic context mixing >= 2, codec/literal.rs:219-243) ----
    const bool mixg = nx.cdf2 != nullptr;
    const char *const cdf2 = reinterpret_cast<const char *>(nx.cdf2);
    int cc0 = c0, cc1 = c1, mc = maxv;
    if (mixg) {
        const uint32_t q = load_elems<LPG>(cdf2, li);
        cc0 = (int)(short)(q & 0xffffu); cc1 = (int)(short)(q >> 16); mc = ld_s16g(cdf2 + 30);
    }
    Weights w = nx.mix_hi ? s.c->w_hi : s.c->w_lo;
    const int prod = mc * maxv;
    int lz = prod == 0 ? 32 : __clz(prod); if (lz > 17) lz = 17;
    const int shift = 17 - lz;
    const int mixr = w.norm, inv = (1 << 15) - mixr;
    // frequentist_cdf.rs:58-72
    const int ca0 = (int)(short)((int)((unsigned)((cc0 * maxv) >> shift) * (unsigned)mixr + (unsigned)((c0 * mc) >> shift) * (unsigned)inv + 1u) >> 15);
    const int ca1 = (int)(short)((int)((unsigned)((cc1 * maxv) >> shift) * (unsigned)mixr + (unsigned)((c1 * mc) >> shift) * (unsigned)inv + 1u) >> 15);
    const int ma = LPG == 16 ? __shfl_sync(FULL, ca0, 15, 16) : __shfl_sync(FULL, ca1, 7, 8);
    const int cu0 = mixg ? ca0 : c0, cu1 = mixg ? ca1 : c1, mu = mixg ? ma : maxv;
    coder_fill(s.cur);
    const int off = (int)(s.cur.a & 0x7fff);
    const int r = (int)(short)((off * mu) >> 15);
    sym = first_true<LPG>(r < cu0, r < cu1, g);
    cum_pair<LPG>(cdf_div(cu0, mu), LPG == 16 ? 0 : cdf_div(cu1, mu), sym, hi, lo);
    start = (int)(short)(lo + 1); freq = (int)(short)(hi - lo - 1);
    int h2, l2;
    cum_pair<LPG>(cdf_div(cc0, mc), LPG == 16 ? 0 : cdf_div(cc1, mc), sym, h2, l2);
    const int f_cm = (int)(short)(h2 - l2 - 1);
    cum_pair<LPG>(cdf_div(c0, maxv), LPG == 16 ? 0 : cdf_div(c1, maxv), sym, h2, l2);
    const int f_nb = (int)(short)(h2 - l2 - 1);
    coder_advance(s.cur, start, freq);
    if (mixg) {
        weights_update(w, f_cm, f_nb, freq);
        if (nx.mix_hi) s.c->w_hi = w; else s.c->w_lo = w;
        const int sp = nx.mix_hi ? s.c->ad_cm_hi : s.c->ad_cm_lo;
        const int ci = (int)(short)(sp & 0xffff), cl = sp >> 16;
        const int m0 = blend_elem(cc0, e0, mc, sym, ci, cl);
        const int m1 = LPG == 16 ? 0 : blend_elem(cc1, e1, mc, sym, ci, cl);
        store_elems<LPG>(cdf2, li, ((uint32_t)m0 & 0xffffu) | ((uint32_t)m1 << 16));
    }
    const int n0 = blend_elem(c0, e0, maxv, sym, inc, lim);
    const int n1 = LPG == 16 ? 0 : blend_elem(c1, e1, maxv, sym, inc, lim);
    store_elems<LPG>(cdf, li, (((uint32_t)n0 & 0xffffu) | ((uint32_t)n1 << 16)) | (nx.tagged ? mytag : 0u));
    return sym;
}

// ---------------------------------------------------------------------------------------------------------------
// literal context table: T2[byte * 8 + class] = literal_context_map[(btype << 6) + (lut0[byte] | class)] | lut1[byte] << 8, where
// class = lut1[byte before] in 0..7 (codec/literal.rs:87-117, codec/interface.rs:199-238): the context of the next byte AND the
// class that the byte after it will need, in one 16-bit load.  Rebuilt by the group when the prediction mode, the context
// map or the literal block type changed.
// LSB6 and MSB6 have no classes (lut1 is all zeros, codec/interface.rs:210-217): for them the 16-lane plain loop reads the
// context from T2S[byte] = T2[byte * 8] & 0xff, 256 bytes per stream in SHARED memory (`t2s`: its shared address, 0 = none).
// ---------------------------------------------------------------------------------------------------------------
constexpr int T2S_BYTES = 256;
__device__ __forceinline__ bool t2s_mode(const uint32_t pred_mode) { return pred_mode < 2; }   // LSB6, MSB6
static __device__ __noinline__ void build_t2(const G2 g, uint8_t *slot, const uint8_t *tables, uint32_t pred_mode, uint32_t btype_last,
                                             const uint32_t t2s) {
    const uint8_t *lut0 = tables + TB_CTX + 512 * pred_mode, *lut1 = lut0 + 256;
    const uint8_t *lcm = slot + OFF_LCM + (btype_last << 6);
    uint32_t *t2 = reinterpret_cast<uint32_t *>(slot + OFF_T2);
    for (uint32_t w = (uint32_t)g.l16; w < 1024; w += (uint32_t)g.nl) {     // word w holds classes 2*(w&3), +1 of byte w >> 2
        const uint32_t byte = w >> 2, a = lut0[byte], k = (w & 3) * 2, cls = (uint32_t)(lut1[byte] & 7u) << 8;
        t2[w] = ((uint32_t)lcm[a | k] | cls) | (((uint32_t)lcm[a | (k + 1)] | cls) << 16);
    }
    if (t2s && t2s_mode(pred_mode))
        for (uint32_t b = (uint32_t)g.l16; b < (uint32_t)T2S_BYTES; b += (uint32_t)g.nl) st_shared_u8(t2s + b, lcm[lut0[b]]);
    __syncwarp(g.gmask);
}

// under-estimate of 2^32 / d for 16 <= d < 2^15 (relative error in (0, 2^-17]): a quotient by multiply-high needs ONE fix-up
__device__ __forceinline__ uint32_t recip32(const uint32_t d) {
    float rc;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(__uint2float_rz(d)));
    return __float2uint_rz(rc * 4294965248.0f);   // 2^32 * (1 - 2^-21): rcp.approx is within 2^-22 relative
}
// floor((c << 15) / d) for 0 <= c <= d
__device__ __forceinline__ uint32_t divq(const uint32_t c, const uint32_t inv, const uint32_t d) {
    const uint32_t n = c << 15;
    uint32_t q = __umulhi(n, inv);
    if (n - q * d >= d) q++;
    return q;
}

// what the fast loop keeps per stream besides the two rANS states
struct FastK {
    const uint32_t *wbase; uint32_t wi, wmax, wnext;   // eager-refill payload cursor; wnext = wbase[wi], already loaded
    uint32_t incp; int inc, lim; uint32_t kp;          // speed (packed twice for LPG 8) and the lane's rescale constant
    uint32_t mytag;                                    // this lane's bit(s) of the stream's generation (lane_tag)
};

// The eager-refill coder of the fast loops.  The reference refills a state right before it is used (ans.rs:428-442); the word
// order in the stream is the order in which states were produced, so refilling a state as soon as it drops below 2^31 consumes
// the same words.  Payload words are addressed by a saturating index: the demux kernel leaves >= 16 readable bytes after every
// coder's payload, so index n_words may be read once; an index that ends above n_words means underflow.
// coder_to_eager: the lazy Coder the state machine keeps -> eager form (pending refill or 16-byte (re)initialisation of `a`
// done, `b` refilled now).  A group that is not `active` rides along as a dummy: states that never refill, payload words read
// from its own slot.
__device__ __forceinline__ void coder_to_eager(Coder &k, FastK &f, const uint8_t *slot, const bool active) {
    if (!active) { k.p = reinterpret_cast<const uint32_t *>(slot + OFF_T2); k.left = 0; k.need_a = 0; k.need_b = 0; k.sym_count = 0; k.a = k.b = 1ull << 40; }
    f.wbase = k.p; f.wmax = k.left + 1; f.wi = 0;
    coder_fill(k);
    f.wi = (uint32_t)(k.p - f.wbase);
    if (k.need_b) { k.b = (k.b << 32) | (uint64_t)f.wbase[f.wi]; f.wi = min(f.wi + 1, f.wmax); k.need_b = 0; }
    f.wnext = f.wbase[f.wi];
}
// ... and back: `a` is the state the next nibble uses, every produced state is refilled already
__device__ __forceinline__ void coder_from_eager(Coder &k, FastK &f) {
    if (f.wi >= f.wmax) { k.underflow = 1; f.wi = f.wmax - 1; }
    k.p = f.wbase + f.wi; k.left = f.wmax - 1 - f.wi;
    k.need_a = (k.sym_count >= NUM_SYMBOLS_BEFORE_FLUSH) ? 8u : 0u; k.need_b = 0;
}
__device__ __forceinline__ void eager_refill(uint64_t &x, FastK &f) {
    x = (x << 32) | (uint64_t)f.wnext; f.wi = min(f.wi + 1, f.wmax); f.wnext = ld_stream_u32(f.wbase + f.wi);
}

// One literal nibble after its symbol is known, in two parts.  (1) blend + store (+ tag) happens at once: the same prior may
// be the next one to be loaded.  (2) exact start/freq and the rANS step with eager refill only have to be done before the state
// is used again, one byte later: the loop runs the two steps of a byte back to back so that their (long, serial) dependency
// chains overlap.  `ev` / `mv`: the validated prior (elements of this lane, max).
template <int LPG>
__device__ __forceinline__ uint32_t blend_v2(const uint32_t ev, const uint32_t mv, const int sym, const G2 g, const FastK &f) {
    uint32_t c2;
    if (LPG == 16) {
        c2 = ev + ((g.l16 >= sym) ? (uint32_t)f.inc : 0u);
        if ((int)mv + f.inc >= f.lim) { const uint32_t u = c2 + f.kp; c2 = u - (u >> 2); }   // frequentist_cdf.rs:79-84
    } else {
        const int d = sym - 2 * g.l16;                                       // elements >= sym take the increment
        const uint32_t m = d <= 0 ? 0xffffffffu : (d == 1 ? 0xffff0000u : 0u);
        c2 = ev + (f.incp & m);
        if ((int)mv + f.inc >= f.lim) { const uint32_t u = c2 + f.kp; c2 = u - ((u >> 2) & 0x3fff3fffu); }
    }
    return c2;
}
template <int LPG>
__device__ __forceinline__ void blend_store_v2(const uint32_t ev, const uint32_t mv, const int sym, const char *const p, const G2 g, const FastK &f) {
    store_elems<LPG>(p, g.l16, blend_v2<LPG>(ev, mv, sym, g, f) | f.mytag);
}
// state after coding `sym` of the validated prior (ev, mv), before renormalisation (ans.rs:230-244)
template <int LPG>
__device__ __forceinline__ uint64_t rans_advance_v2(const uint64_t st, const uint32_t ev, const uint32_t mv, const int sym) {
    const uint32_t inv = recip32(mv);
    uint32_t hi, lo;
    // lo: the cumulative value of element sym - 1, 0 for sym = 0, taken as element (sym - 1) mod 16 masked to 15 bits.  For
    // sym >= 1 on a monotone CDF the search found c[sym - 1] <= r < max, so divq gives less than 0x8000 and the mask keeps
    // it.  For sym = 0 the source is element 15, the max itself, whose cumulative value is exactly 0x8000: it masks to 0.
    // (At 16 lanes the shuffle takes its source lane mod 16.)
    const int prev = sym - 1;
    if (LPG == 16) {
        const uint32_t cum = divq(ev, inv, mv);
        hi = __shfl_sync(FULL, cum, sym, 16); lo = __shfl_sync(FULL, cum, prev, 16);
    } else {
        const uint32_t cum = divq(ev & 0xffffu, inv, mv) | (divq(ev >> 16, inv, mv) << 16);   // element 15: 0x8000
        const uint32_t whi = __shfl_sync(FULL, cum, sym >> 1, 8), wlo = __shfl_sync(FULL, cum, (prev & 15) >> 1, 8);
        hi = (sym & 1) ? (whi >> 16) : (whi & 0xffffu);
        lo = (prev & 1) ? (wlo >> 16) : wlo;
    }
    lo &= 0x7fffu;
    const uint32_t freq = hi - lo - 1;                                       // "major hax": start = lo + 1 (probability/interface.rs:103-104)
    // 0 <= t < freq in every stream an encoder wrote.  A corrupted payload can put the offset below the bin: offset 0 decodes
    // symbol 0, whose bin starts at 1 ("major hax"), so t = -1.  The reference computes the state in 64-bit wrapping arithmetic
    // (ans.rs:230-244, coder_advance): t is sign-extended, not taken modulo 2^32.
    const uint32_t t = ((uint32_t)st & 0x7fffu) - lo - 1;
    return (uint64_t)freq * (st >> 15) + (uint64_t)(int64_t)(int32_t)t;
}
// The two rANS steps of a byte (state a: high nibble, b: low nibble), then the eager refills in payload order (a before b).  A
// state needs a word once per ~16 nibbles of text: with 16 lanes per stream the refill code sits behind ONE warp-uniform branch
// instead of being sixteen predicated-off instructions in every byte.
template <int LPG>
__device__ __forceinline__ void rans_pair_v2(uint64_t &a, uint64_t &b, const uint32_t eh, const uint32_t mh, const int h,
                                             const uint32_t el, const uint32_t ml, const int l, FastK &f) {
    uint64_t xa = rans_advance_v2<LPG>(a, eh, mh, h), xb = rans_advance_v2<LPG>(b, el, ml, l);
    const bool na = xa < (1ull << 31), nb = xb < (1ull << 31);
    // two streams per warp: no state refills in 78 % of the bytes, the branch pays; four streams per warp: 61 %, the
    // predicated form is the faster one
    if (LPG == 8 || __any_sync(FULL, na || nb)) {
        if (na) eager_refill(xa, f);
        if (nb) eager_refill(xb, f);
    }
    a = xa; b = xb;
}

// bin search: for a monotone CDF whose last element is max (> r) the number of elements with c[i] <= r is sym (the vote
// counts it directly: no 16 - popc of the complement)
template <int LPG>
__device__ __forceinline__ int search_v2(const uint64_t st, const uint32_t ev, const uint32_t mv, const uint32_t bsel) {
    const uint32_t rr = (((uint32_t)st & 0x7fffu) * mv) >> 15;              // probability/interface.rs:140
    if (LPG == 16) return __popc(__ballot_sync(FULL, rr >= ev) & bsel);     // bsel: the group's 16 ballot bits
    const unsigned b0 = __ballot_sync(FULL, rr >= (ev & 0xffffu)), b1 = __ballot_sync(FULL, rr >= (ev >> 16));
    return __popc(__byte_perm(b0, b1, bsel)) >> 1;                          // bsel: PRMT selector [g, 4+g, g, 4+g]
}

// ---- dynamic context mixing >= 2 (codec/literal.rs:219-259), 16 lanes per stream: the stride prior `nb` (tagged literal table) is
// mixed with the context-map prior `cm` (LIT_CM, untagged, defaulted eagerly), weights model_weights[high nibble ? 1 : 0] ----
struct MixV { uint32_t c, maxv, cc, mc; };
__device__ __forceinline__ MixV mixv_load(const char *nb, const char *cm, const int li) {
    MixV v; v.c = ld_u16g(nb + 2 * li); v.maxv = ld_u16g(nb + 30); v.cc = ld_u16g(cm + 2 * li); v.mc = ld_u16g(cm + 30); return v;
}
struct MixS { int sym; uint32_t ca, ma; };
__device__ __forceinline__ MixS mixv_search(const uint64_t st, const MixV v, const int norm, const uint32_t bsel) {
    const uint32_t prod = v.mc * v.maxv;
    int lz = prod == 0 ? 32 : __clz((int)prod); if (lz > 17) lz = 17;
    const int shift = 17 - lz;
    const uint32_t mixr = (uint32_t)norm, inv = (1u << 15) - mixr;
    const uint32_t rs = (v.cc * v.maxv) >> shift, ro = (v.c * v.mc) >> shift;
    MixS r;
    r.ca = (uint32_t)(int)(short)((int)(rs * mixr + ro * inv + 1u) >> 15);   // frequentist_cdf.rs:58-72
    r.ma = __shfl_sync(FULL, r.ca, 15, 16);
    const uint32_t q = (((uint32_t)st & 0x7fffu) * r.ma) >> 15;
    r.sym = 16 - __popc(__ballot_sync(FULL, q < r.ca) & bsel);
    return r;
}
__device__ __forceinline__ void mixv_finish(uint64_t &st, const MixV v, const MixS ms, Weights &w, const char *nb, const char *cm, const G2 g, FastK &f,
                                            const int cm_inc, const int cm_lim) {
    const int sym = ms.sym, prev = (sym - 1) & 15;
    const uint32_t cum_a = divq(ms.ca, recip32(ms.ma), ms.ma);
    const uint32_t cum_pn = divq(v.cc, recip32(v.mc), v.mc) | (divq(v.c, recip32(v.maxv), v.maxv) << 16);
    const uint32_t hi_a = __shfl_sync(FULL, cum_a, sym, 16), hi_pn = __shfl_sync(FULL, cum_pn, sym, 16);
    uint32_t lo_a = __shfl_sync(FULL, cum_a, prev, 16), lo_pn = __shfl_sync(FULL, cum_pn, prev, 16);
    if (sym == 0) { lo_a = 0; lo_pn = 0; }
    const uint32_t freq = hi_a - lo_a - 1;
    const int f_cm = (int)(short)((hi_pn & 0xffffu) - (lo_pn & 0xffffu) - 1);
    const int f_nb = (int)(short)((hi_pn >> 16) - (lo_pn >> 16) - 1);
    const uint32_t t = ((uint32_t)st & 0x7fffu) - lo_a - 1;
    uint64_t x = (uint64_t)(int64_t)(int16_t)freq * (st >> 15) + (uint64_t)(int64_t)(int32_t)t;   // ans.rs:230-244 (t < 0: see rans_advance_v2)
    const bool refill = x < (1ull << 31);
    if (__any_sync(FULL, refill)) {   // (one warp-uniform branch instead of predicated-off refill code in every nibble, see rans_pair_v2)
        if (refill) eager_refill(x, f);
    }
    st = x;
    weights_update32(w, f_cm, f_nb, (int)(short)freq);
    uint32_t c2 = v.cc + ((g.l16 >= sym) ? (uint32_t)cm_inc : 0u);
    if ((int)v.mc + cm_inc >= cm_lim) { const uint32_t u = c2 + f.kp; c2 = u - (u >> 2); }
    st_u16(cm + 2 * g.l16, c2);
    uint32_t s2 = v.c + ((g.l16 >= sym) ? (uint32_t)f.inc : 0u);
    if ((int)v.maxv + f.inc >= f.lim) { const uint32_t u = s2 + f.kp; s2 = u - (u >> 2); }
    st_u16(nb + 2 * g.l16, s2 | f.mytag);
}
// the mixing loop proper; same skeleton as the plain loop of literal_fast_v2 (which calls it)
__device__ __forceinline__ void literal_mix_loop16(St &s, const G2 g, const bool active, uint32_t n) {
    const int li = g.l16;
    const int cfg = active ? s.lit_cfg : mm_cfg(4);
    const uint32_t mm = (cfg & 0x100) ? 0xffu : 0u, o1 = (cfg & 0x200) ? 0xfu : 0u, fc = (cfg & 0x400) ? 0xfu : 0u;
    const uint32_t sh = (uint32_t)(cfg >> 2) & 63u, which = (uint32_t)cfg & 3u, mhi = mm & (~o1 & 0xffu);
    const bool ro = (cfg & 0x800) != 0;                                      // mixing value 2: the stride prior is read, never adapted
    FastK f;
    f.inc = !active ? 0x10 : ro ? 0 : (int)(short)(s.ad_stride & 0xffff); f.lim = !active ? 0x2000 : ro ? 0x7fff : (s.ad_stride >> 16);
    f.incp = 0; f.kp = (uint32_t)(li + 1);
    f.mytag = lane_tag<16>(s.gen, li);
    const int ch_inc = active ? (int)(short)(s.c->ad_cm_hi & 0xffff) : 0x10, ch_lim = active ? (s.c->ad_cm_hi >> 16) : 0x2000;
    const int cl_inc = active ? (int)(short)(s.c->ad_cm_lo & 0xffff) : 0x10, cl_lim = active ? (s.c->ad_cm_lo >> 16) : 0x2000;
    const uint32_t defe = default_elems<16>(li), bsel = 0xffffu << g.shift;
    const unsigned gm = g.gmask;
    const uint32_t slot_lo = (uint32_t)(uintptr_t)s.slot, slot_hi = (uint32_t)((uintptr_t)s.slot >> 32);
    const uint32_t hi_tab = slot_lo + (uint32_t)OFF_LIT_HI + which * (65536u * 32u), lo_tab = slot_lo + (uint32_t)OFF_LIT_LO + which * (65536u * 32u);
    const uint32_t cmb = slot_lo + (uint32_t)OFF_LIT_CM, t2 = slot_lo + (uint32_t)OFF_T2;
    unsigned long long l8 = active ? s.l8 : 0ull;
    uint32_t ctx = active ? s.lit_ctx : 0u;
    uint32_t pcp = ld_u16g(mk_ptr(t2 + (uint32_t)(l8 >> 56) * 16u, slot_hi)) >> 8;
    uint8_t *const dbase = s.out + s.out_pos;
    uint32_t ap = (uint32_t)(uintptr_t)dbase & 7u;
    const bool st_lane = g.store0 && active;
    Coder k = s.cur;
    Weights wh = s.c->w_hi, wl = s.c->w_lo;
    coder_to_eager(k, f, s.slot, active);
    uint32_t done = 0;
    while (done < n) {
        uint32_t m = n - done;
        if (k.sym_count >= NUM_SYMBOLS_BEFORE_FLUSH) {   // chunk restart, ans.rs:173-189
            if (f.wi + 5 <= f.wmax) { k.a = (uint64_t)f.wbase[f.wi] | ((uint64_t)f.wbase[f.wi + 1] << 32); k.b = (uint64_t)f.wbase[f.wi + 2] | ((uint64_t)f.wbase[f.wi + 3] << 32); f.wi += 4; }
            else { k.a = k.b = 0; f.wi = f.wmax; }
            f.wnext = f.wbase[f.wi];
            k.sym_count = 0;
        }
        m = min(m, (NUM_SYMBOLS_BEFORE_FLUSH - k.sym_count) >> 1);
        m = min(m, __shfl_xor_sync(FULL, m, 16));
        if (m == 0) break;
        uint32_t ssb = (uint32_t)(l8 >> sh) & 0xffu;
        const char *nbh = mk_ptr(hi_tab + lit_index_hi(which, ctx, ssb & mhi) * 32u, slot_hi), *cmh = mk_ptr(cmb + ctx * 32u, slot_hi);
        __syncwarp();
        MixV vh = mixv_load(nbh, cmh, li);
        for (uint32_t i = 0; i < m; i++) {
            // -- high nibble
            const unsigned okh = __ballot_sync(FULL, !active || (vh.c & TAG_BITS16) == f.mytag);
            if ((okh & gm) == gm) { vh.c &= 0x7fffu; vh.maxv &= 0x7fffu; } else { vh.c = defe; vh.maxv = 64u; }
            const MixS sh_ = mixv_search(k.a, vh, wh.norm, bsel);
            const uint32_t h = (uint32_t)sh_.sym;
            const uint32_t ib = (mm & ssb) | ((~mm & 0xffu) & ctx), ic = (h & fc) + ((ctx & o1) << 4);
            const char *const nbl = mk_ptr(lo_tab + lit_index_lo(which, ic, ib) * 32u, slot_hi), *const cml = mk_ptr(cmb + (256u + h + 16u * ctx) * 32u, slot_hi);
            __syncwarp();
            MixV vl = mixv_load(nbl, cml, li);
            mixv_finish(k.a, vh, sh_, wh, nbh, cmh, g, f, ch_inc, ch_lim);
            // -- low nibble
            const unsigned okl = __ballot_sync(FULL, !active || (vl.c & TAG_BITS16) == f.mytag);
            if ((okl & gm) == gm) { vl.c &= 0x7fffu; vl.maxv &= 0x7fffu; } else { vl.c = defe; vl.maxv = 64u; }
            const MixS sl_ = mixv_search(k.b, vl, wl.norm, bsel);
            const uint32_t cur = ((uint32_t)sl_.sym | (h << 4)) & 0xffu;
            l8 = (l8 >> 8) | ((unsigned long long)cur << 56);
            if (st_lane && (ap & 7u) == 7u) st_stream_u64(dbase + (done + i) - 7, l8);
            ap++;
            const uint32_t cv = ld_u16g(mk_ptr(t2 + (cur * 8u + pcp) * 2u, slot_hi));
            ctx = cv & 0xffu; pcp = cv >> 8;
            ssb = (uint32_t)(l8 >> sh) & 0xffu;
            nbh = mk_ptr(hi_tab + lit_index_hi(which, ctx, ssb & mhi) * 32u, slot_hi); cmh = mk_ptr(cmb + ctx * 32u, slot_hi);
            __syncwarp();
            vh = mixv_load(nbh, cmh, li);   // speculative on the last byte: inside the slot
            mixv_finish(k.b, vl, sl_, wl, nbl, cml, g, f, cl_inc, cl_lim);
        }
        done += m;
        if (active) k.sym_count += 2 * m;
    }
    if (!active) return;
    if (g.store0) {
        const uint32_t tail = min(ap & 7u, done);
        for (uint32_t t = 0; t < tail; t++) dbase[done - tail + t] = (uint8_t)(l8 >> (8 * (8 - tail + t)));
    }
    coder_from_eager(k, f);
    s.cur = k; s.l8 = l8; s.lit_ctx = ctx; s.out_pos += done; s.lit_left -= done;
    s.c->w_hi = wh; s.c->w_lo = wl;
}

// The plain loop of literal_fast_v2 (below).  SMALL: every group reads its context from T2S (16 lanes, LSB6 / MSB6); the loop is
// compiled once for each case so that the one taken does not issue the other's predicated-off context load.
template <int LPG, bool SMALL>
__device__ __forceinline__ bool literal_plain_loop_v2(St &s, Next &nx, const G2 g, const bool active, const uint32_t t2s, const uint32_t n) {
    constexpr bool small = SMALL;
    const int li = g.l16;
    const int cfg = active ? s.lit_cfg : mm_cfg(4);
    const uint32_t mm = (cfg & 0x100) ? 0xffu : 0u, o1 = (cfg & 0x200) ? 0xfu : 0u, fc = (cfg & 0x400) ? 0xfu : 0u;
    const uint32_t sh = (uint32_t)(cfg >> 2) & 63u, which = (uint32_t)cfg & 3u, mhi = mm & (~o1 & 0xffu);
    FastK f;
    f.inc = active ? (int)(short)(s.ad_stride & 0xffff) : 0x10; f.lim = active ? (s.ad_stride >> 16) : 0x2000;
    f.incp = (uint32_t)f.inc * 0x10001u;
    f.kp = LPG == 16 ? (uint32_t)(li + 1) : ((uint32_t)(2 * li + 1) | ((uint32_t)(2 * li + 2) << 16));
    f.mytag = lane_tag<LPG>(s.gen, li);
    const uint32_t tbits = LPG == 16 ? TAG_BITS16 : TAG_BITS8;
    // the tag check is ((element ^ mytag) & tchk) == 0: a dummy group's priors always pass, so its own test stays out of the vote
    const uint32_t tchk = active ? tbits : 0u;
    const uint32_t defe = default_elems<LPG>(li);
    const uint32_t bsel = LPG == 16 ? (0xffffu << g.shift) : ((uint32_t)(g.shift >> 3) * 0x1111u + 0x4040u);
    const unsigned gm = g.gmask;
    // every address inside the slot is (slot_hi : slot_lo + offset): slots are 16 MiB aligned
    const uint32_t slot_lo = (uint32_t)(uintptr_t)s.slot, slot_hi = (uint32_t)((uintptr_t)s.slot >> 32);
    const uint32_t hi_tab = slot_lo + (uint32_t)OFF_LIT_HI + which * (65536u * 32u), lo_tab = slot_lo + (uint32_t)OFF_LIT_LO + which * (65536u * 32u);
    const uint32_t t2 = slot_lo + (uint32_t)OFF_T2;
    unsigned long long l8 = active ? s.l8 : 0ull;
    uint32_t ctx = active ? s.lit_ctx : 0u;
    uint32_t pcp = ld_u16g(mk_ptr(t2 + (uint32_t)(l8 >> 56) * 16u, slot_hi)) >> 8;   // class of the byte before the next one to decode
    // output: an aligned 8-byte store of l8 whenever the cursor completes an 8-byte word (l8 mirrors the 8 bytes in front of
    // the cursor here: the caller keeps the first 7 bytes of a literal that began within 8 bytes of the ring start away)
    uint8_t *const dbase = s.out + s.out_pos;
    uint32_t ap = (uint32_t)(uintptr_t)dbase & 7u;                        // alignment of the ADDRESS of the byte being decoded
    const bool st_lane = g.store0 && active;
    // eager-refill coder for the duration of the loop (coder_to_eager).  The literal coder codes nibbles in pairs: state `a`
    // serves every high nibble, `b` every low nibble (two rotations of ans.rs:240-243 are the identity), so the loop never
    // swaps them.
    Coder k = s.cur;
    coder_to_eager(k, f, s.slot, active);
    uint32_t done = 0;
    while (done < n) {
        uint32_t m = n - done;
        if (k.sym_count >= NUM_SYMBOLS_BEFORE_FLUSH) {   // chunk restart, ans.rs:173-189
            if (f.wi + 5 <= f.wmax) { k.a = (uint64_t)f.wbase[f.wi] | ((uint64_t)f.wbase[f.wi + 1] << 32); k.b = (uint64_t)f.wbase[f.wi + 2] | ((uint64_t)f.wbase[f.wi + 3] << 32); f.wi += 4; }
            else { k.a = k.b = 0; f.wi = f.wmax; }
            f.wnext = f.wbase[f.wi];
            k.sym_count = 0;
        }
        m = min(m, (NUM_SYMBOLS_BEFORE_FLUSH - k.sym_count) >> 1);
        if (LPG == 8) m = min(m, __shfl_xor_sync(FULL, m, 8));
        m = min(m, __shfl_xor_sync(FULL, m, 16));
        if (m == 0) break;   // unreachable: the literal coder codes nibbles in pairs, sym_count stays even
        // ---- priors of the first byte ----
        // (low nibble: index_c = (high nibble & fc) + ((ctx & o1) << 4), index_b = ib -- all but the high nibble known a byte ahead)
        uint32_t ssb = (uint32_t)(l8 >> sh) & 0xffu;
        uint32_t cl = (ctx & o1) << 4, ib = (mm & ssb) | ((~mm & 0xffu) & ctx);
        const char *ph = mk_ptr(hi_tab + lit_index_hi(which, ctx, ssb & mhi) * 32u, slot_hi);
        __syncwarp();
        uint32_t eh = load_elems<LPG>(ph, li), mh = ld_u16g(ph + 30);
// (16 lanes per stream: not unrolled -- the literal loop itself times the same with 1, 2 or 4 bytes per trip, but the
        // command path, which is instruction-fetch bound, is faster with the smaller kernel.  8 lanes per stream: two bytes
        // per trip)
#pragma unroll (LPG == 16 ? 1 : 2)
        for (uint32_t i = 0; i < m; i++) {
            // -- high nibble: search (speculative: the prior is almost always one this stream has written)
            uint32_t eh_v = eh & ~tbits, mh_v = mh & 0x7fffu;
            int h = search_v2<LPG>(k.a, eh_v, mh_v, bsel);
            if (__builtin_expect(!__all_sync(FULL, ((eh ^ f.mytag) & tchk) == 0), 0)) {   // some group met a prior of an older
                const unsigned okh = __ballot_sync(FULL, ((eh ^ f.mytag) & tchk) == 0);      // stream: default CDF
                if ((okh & gm) != gm) { eh_v = defe; mh_v = 64u; }
                h = search_v2<LPG>(k.a, eh_v, mh_v, bsel);
            }
            // -- low nibble: prior
            const char *const pl = mk_ptr(lo_tab + lit_index_lo(which, ((uint32_t)h & fc) + cl, ib) * 32u, slot_hi);
            __syncwarp();
            const uint32_t el = load_elems<LPG>(pl, li), ml = ld_u16g(pl + 30);
            // -- high nibble: blend (this prior may be the next one to be loaded)
            blend_store_v2<LPG>(eh_v, mh_v, h, ph, g, f);
            // -- low nibble: search
            uint32_t el_v = el & ~tbits, ml_v = ml & 0x7fffu;
            int l = search_v2<LPG>(k.b, el_v, ml_v, bsel);
            if (__builtin_expect(!__all_sync(FULL, ((el ^ f.mytag) & tchk) == 0), 0)) {
                const unsigned okl = __ballot_sync(FULL, ((el ^ f.mytag) & tchk) == 0);
                if ((okl & gm) != gm) { el_v = defe; ml_v = 64u; }
                l = search_v2<LPG>(k.b, el_v, ml_v, bsel);
            }
            const uint32_t cur = ((uint32_t)l | ((uint32_t)h << 4)) & 0xffu;
            l8 = (l8 >> 8) | ((unsigned long long)cur << 56);              // push_literal_byte, codec/interface.rs:280-284
            if (st_lane && (ap & 7u) == 7u) st_stream_u64(dbase + (done + i) - 7, l8);
            ap++;
            // -- context and priors of the next byte (get_prev_word_context, codec/literal.rs:87-117, through T2)
            const uint32_t cv = small ? ld_shared_u8(t2s + cur) : ld_u16g(mk_ptr(t2 + (cur * 8u + pcp) * 2u, slot_hi));
            ctx = cv & 0xffu; pcp = cv >> 8;
            ssb = (uint32_t)(l8 >> sh) & 0xffu;
            ph = mk_ptr(hi_tab + lit_index_hi(which, ctx, ssb & mhi) * 32u, slot_hi);
            __syncwarp();
            eh = load_elems<LPG>(ph, li); mh = ld_u16g(ph + 30);   // speculative on the last byte: inside the slot
            cl = (ctx & o1) << 4; ib = (mm & ssb) | ((~mm & 0xffu) & ctx);
            // -- low nibble: blend; then the rANS steps of both nibbles (state a before b: the order of the payload words)
            blend_store_v2<LPG>(el_v, ml_v, l, pl, g, f);
            rans_pair_v2<LPG>(k.a, k.b, eh_v, mh_v, h, el_v, ml_v, l, f);
        }
        done += m;
        if (active) k.sym_count += 2 * m;
    }
    if (!active) return true;
    // the bytes after the last aligned 8-byte store are still only in l8
    if (g.store0) {
        const uint32_t tail = min(ap & 7u, done);
        for (uint32_t t = 0; t < tail; t++) dbase[done - tail + t] = (uint8_t)(l8 >> (8 * (8 - tail + t)));
    }
    coder_from_eager(k, f);                                               // back to the lazy representation the state machine uses
    s.cur = k; s.l8 = l8; s.lit_ctx = ctx; s.out_pos += done; s.lit_left -= done;
    enter_lit_nibble<false, true, true>(s, nx);
    return true;
}

// Converged literal fast path: code_nibble_array (codec/literal.rs:261-394) for whole bytes of every stream of the warp.
// `active`: this group really is at the start of a literal byte.  A group that has run out of streams rides along as a dummy
// (it codes garbage against its own slot and stores no output) so that its warp-mates keep the fast loop.
// Returns false (nothing done) when some group cannot take the fast loop: dynamic context mixing, per-context mixing values, the
// flat prior, wide speeds, untagged priors, or the first 7 bytes of a literal that began within 8 bytes of the ring start -- the
// caller then codes one nibble per group through the generic core and the state machine.
// `t2s`: shared address of this group's T2S (16 lanes per stream), else 0.
template <int LPG>
__device__ __forceinline__ bool literal_fast_v2(St &s, Next &nx, const G2 g, const bool active, const uint32_t t2s) {
    uint32_t n = active ? s.lit_left : 0xffffffffu;
    if (LPG == 8) n = min(n, __shfl_xor_sync(FULL, n, 8));
    n = min(n, __shfl_xor_sync(FULL, n, 16));
    if (n < 12) return false;   // entering and leaving the loop costs about as much as a dozen nibbles of the generic path
    // dynamic context mixing >= 2 with one mixing value for the whole map (16 lanes per stream): its own loop
    if (LPG == 16 && __all_sync(FULL, !active || (s.mixing_trait && s.lit_cfg >= 0 && s.speeds_small && s.tagged &&
                                                  !(s.c->lit_quirk && s.c->lit_total - s.lit_left < 7u)))) {
        if (active && s.c->t2_dirty) { build_t2(g, s.slot, s.tables, s.pred_mode, s.btype_last, t2s); s.c->t2_dirty = false; }
        __syncwarp();
        literal_mix_loop16(s, g, active, n);
        if (active) enter_lit_nibble<false, true, true>(s, nx);
        return true;
    }
    // plain literals, one mixing value for the whole map (not the never-adapted flat prior), speeds that cannot wrap i16, tagged
    // priors; and not the first 7 bytes of a literal that began within 8 bytes of the ring start (also: of the stream): until then
    // last_8_literals is not a mirror of the output (cmd_to_raw/mod.rs:69-86) and cannot feed the 8-byte stores
    if (!__all_sync(FULL, !active || (!s.mixing_trait && s.lit_cfg >= 0 && !(s.lit_cfg & 0x800) && s.speeds_small && s.tagged &&
                                      !(s.c->lit_quirk && s.c->lit_total - s.lit_left < 7u)))) return false;
    {
        if (active && s.c->t2_dirty) { build_t2(g, s.slot, s.tables, s.pred_mode, s.btype_last, t2s); s.c->t2_dirty = false; }
        __syncwarp();
        // every group in LSB6 / MSB6 (16 lanes): the context comes from T2S in shared memory (a dummy group reads garbage
        // contexts, which still address inside its own slot)
        const bool small = LPG == 16 && __all_sync(FULL, !active || t2s_mode(s.pred_mode));
        if (small) return literal_plain_loop_v2<LPG, LPG == 16>(s, nx, g, active, t2s, n);
        return literal_plain_loop_v2<LPG, false>(s, nx, g, active, t2s, n);
    }
}

// Converged fast path for the 8192 mixing values of a PredictionMode command (context_map.rs:385-425), every group of the warp
// in S_PM_MIXVAL (`active`) or out of work (a dummy, as in literal_fast_v2).  Each value is one nibble of the command coder
// against an untagged MISC prior adapted at SPK_PLANE, a speed that keeps every adaptive value inside i16 (speed_is_small): the
// 32-bit arithmetic of the literal loops is exact.  The prior of value f1 depends on the value coded 256 nibbles earlier, not
// on the nibble just coded, and consecutive nibbles alternate between the two rANS states (ans.rs:240-243), so a nibble's
// dependency chain is search -> blend of the same prior -> the next search; the rANS step stays off it.
// The run stops short of two positions, where the generic path, which keeps the reference's lazy refills, codes the nibbles:
//   * value 8190: the last value ends the command (mixing_param, pred_mode, the speeds, t2_dirty, the f0 > 3 failure), and an
//     underflow of the last eager refill must not be reported before the failure of the nibble after it;
//   * symbol 65534 of the coder's chunk: the 16-byte re-initialisation after symbol 65535 drops the refill of the state of
//     symbol 65534 and moves that of symbol 65535 behind its own words (ans.rs:230-244).
// The run proper, out of line: the command path that shares the kernel is instruction-fetch bound (DESIGN section 4), and the
// loop inlined into the main loop made LZ77 command streams slower.  Everything crosses the call by value, so that the caller's
// St stays in registers.  Returns the coder (lazy form) and the next mixing value.
struct MixvalRun { Coder k; uint32_t f1; };
template <int LPG>
static __device__ __noinline__ MixvalRun mixval_run_v2(Coder k, const uint32_t f1, const uint32_t n, uint8_t *const slot, const bool rev,
                                                       const G2 g, const bool active) {
    const int li = g.l16;
    FastK f;
    f.inc = (int)(short)(SPK_PLANE & 0xffff); f.lim = SPK_PLANE >> 16;
    f.incp = (uint32_t)f.inc * 0x10001u;
    f.kp = LPG == 16 ? (uint32_t)(li + 1) : ((uint32_t)(2 * li + 1) | ((uint32_t)(2 * li + 2) << 16));
    f.mytag = 0;
    const uint32_t bsel = LPG == 16 ? (0xffffu << g.shift) : ((uint32_t)(g.shift >> 3) * 0x1111u + 0x4040u);
    const uint32_t slot_lo = (uint32_t)(uintptr_t)slot, slot_hi = (uint32_t)((uintptr_t)slot >> 32);
    // (32-bit addresses inside the slot, as in the literal loops; `pe` below: this lane's element(s) of the prior's CDF)
    const uint32_t pbase = slot_lo + (uint32_t)OFF_MISC + (uint32_t)(MI_PRED + PM_MIXING_VALUE) * CDF_BYTES, mixb = slot_lo + (uint32_t)OFF_MIX;
    const auto mix = [slot_hi, mixb](uint32_t i) { return ld_u8g(mk_ptr(mixb + i, slot_hi)); };
    const bool st_lane = g.store0 && active;
    coder_to_eager(k, f, slot, active);
    if (st_lane && f1 == 0) reinterpret_cast<uint32_t *>(slot + OFF_HDR)[3] = 1u;   // the mask is about to hold this stream's values
    // Runs of values whose prior stays the same for every group: the prior is loaded once and then kept in registers (each blend
    // is stored as well).  With one mixing value for the whole map, the usual case, the prior changes once, at value 256.
    // Consecutive values alternate between the states (ans.rs:240-243): the loop codes them in pairs, value 2j on `a` and 2j + 1
    // on `b`, and swaps the two only when a run ends after an odd number of values.
    constexpr uint32_t EB = CDF_BYTES / LPG;                              // bytes of a lane's element(s)
    uint32_t pi = mixval_prior(f1, rev, mix), i = 0;
    while (i < n) {
        const uint32_t pa = pbase + pi * CDF_BYTES;
        __syncwarp();                                                    // (the other lanes' stores: mixing values, the max)
        const char *const pe = mk_ptr(pa + EB * li, slot_hi);
        uint32_t ev = load_elems<LPG>(pe, 0), mv = ld_u16g(mk_ptr(pa + 30u, slot_hi));
        uint32_t pn;
        // value f1 + i on state `st`; true when the run ends after it
        const auto value = [&](uint64_t &st) {
            pn = mixval_prior(f1 + i + 1, rev, mix);                     // its mixing value was coded 255 nibbles ago
            const int sym = search_v2<LPG>(st, ev, mv, bsel);
            if (st_lane) st_u8(mk_ptr(mixb + f1 + i, slot_hi), (uint32_t)sym);
            const uint32_t ne = blend_v2<LPG>(ev, mv, sym, g, f);
            store_elems<LPG>(pe, 0, ne);
            uint32_t nm = mv + (uint32_t)f.inc;                          // element 15 of `ne`: the new max
            if ((int)nm >= f.lim) { const uint32_t u = nm + 16u; nm = u - (u >> 2); }
            uint64_t x = rans_advance_v2<LPG>(st, ev, mv, sym);
            const bool rf = x < (1ull << 31);
            if (LPG == 8 || __any_sync(FULL, rf)) { if (rf) eager_refill(x, f); }   // (as in rans_pair_v2)
            st = x; ev = ne; mv = nm;
            __syncwarp();
            const bool change = __any_sync(FULL, pn != pi);              // (not behind `||`: a branch costs more than the vote)
            return (++i == n) | change;
        };
        for (;;) {
            if (value(k.a)) { const uint64_t t = k.a; k.a = k.b; k.b = t; break; }
            if (value(k.b)) break;
        }
        pi = pn;
    }
    k.sym_count += n;
    coder_from_eager(k, f);
    return MixvalRun{k, f1 + n};
}
// Returns false (nothing done) when some group has fewer than 8 values to go before one of them.
template <int LPG>
__device__ __forceinline__ bool mixval_fast_v2(St &s, Next &nx, const G2 g, const bool active) {
    const uint32_t sc = s.cur.need_a > 1 ? 0u : s.cur.sym_count;       // (a pending 16-byte initialisation starts a new chunk)
    uint32_t n = active ? min(8190u - min(s.f1, 8190u), 65534u - min(sc, 65534u)) : 0xffffffffu;
    if (LPG == 8) n = min(n, __shfl_xor_sync(FULL, n, 8));
    n = min(n, __shfl_xor_sync(FULL, n, 16));
    if (n < 8) return false;
    // a dummy codes against slot 16 of its own slot
    const MixvalRun r = mixval_run_v2<LPG>(s.cur, active ? s.f1 : 0u, n, s.slot, !active || s.c->model_rev, g, active);
    if (!active) return true;
    s.cur = r.k; s.f1 = r.f1;
    enter_pm_mixval<false>(s, nx);
    return true;
}

}  // namespace dv
