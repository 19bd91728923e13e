// dv_model.cuh -- the divANS model + rANS coder as warp-level device code (sm_90a).
//
// One 16-lane group owns one stream: lane i (0..15) of the group holds element i of whichever 16-entry adaptive
// CDF is being coded, so the reference's per-symbol work becomes
//   bin search  (probability/interface.rs:136-198)  -> per-lane compare + __ballot_sync + __ffs
//   start/freq  (probability/interface.rs:97-108)   -> per-lane exact (c<<15)/max, two __shfl_sync
//   blend       (probability/frequentist_cdf.rs:74-85) -> per-lane predicated add + uniform rescale branch
//   average     (probability/frequentist_cdf.rs:58-72) -> per-lane integer mad
// Everything that is scalar in the reference (rANS states, book-keeping) is replicated across the lanes of the
// group (uniform registers).  With LANES_PER_STREAM==32 the upper half-warp mirrors the lower one (same stream);
// with 16 the two half-warps run two different streams.
//
// The same code runs as decoder (ENC=false: symbols come out of the rANS state) and as encoder (ENC=true: symbols
// are given, (start,freq) pairs are recorded for the reverse rANS pass) -- exactly how the reference shares
// DivansCodec between ANSDecoder and ANSEncoder (codec/mod.rs:160-186).
#pragma once
#include "dv_common.cuh"

namespace dv {


struct Speed2 { int inc, lim; };

// ---------------------------------------------------------------------------------------------------------------
// rANS coder state (src/ans.rs:142-148 decoder; :254-301 encoder records (start,freq)).
// The decoder reads its byte stream as aligned 32-bit words from a CONTIGUOUS payload: the mux records of the two
// interleaved streams (mux.rs:384-444) are compacted by dv::demux_kernel before the stream kernel runs.
// ---------------------------------------------------------------------------------------------------------------
struct Coder {
    uint64_t a, b;
    const uint32_t *p;     // DEC: next payload word.  ENC: base of this coder's (start | freq<<16) log
    uint32_t left;         // DEC: payload words left. ENC: symbols logged so far
    uint32_t sym_count, need_a, need_b, underflow;
};

__device__ __forceinline__ void coder_init_dec(Coder &k, const uint32_t *payload, uint32_t n_words) {
    k.a = k.b = 0; k.sym_count = 0; k.need_a = 8; k.need_b = 0; k.underflow = 0;   // ans.rs:150-162
    k.p = payload; k.left = n_words;
}
__device__ __forceinline__ void coder_init_enc(Coder &k, uint32_t *log) {
    k.a = k.b = 0; k.sym_count = 0; k.need_a = 0; k.need_b = 0; k.underflow = 0;
    k.p = log; k.left = 0;
}
__device__ __forceinline__ void coder_fill(Coder &k) {
    // ans.rs:428-442 (push_data) and :173-189 (16-byte (re)initialisation at stream start / every 65536 symbols)
    if (k.need_a == 0) return;
    if (k.need_a == 1) {
        if (k.left >= 1) { uint32_t w = __ldg(k.p); k.p += 1; k.left -= 1; k.a = (k.a << 32) | (uint64_t)w; }
        else { k.underflow = 1; k.a <<= 32; }
    } else {
        if (k.left >= 4) {
            uint4 w = make_uint4(__ldg(k.p), __ldg(k.p + 1), __ldg(k.p + 2), __ldg(k.p + 3));
            k.p += 4; k.left -= 4;
            k.a = (uint64_t)w.x | ((uint64_t)w.y << 32);
            k.b = (uint64_t)w.z | ((uint64_t)w.w << 32);
        } else { k.underflow = 1; k.a = k.b = 0; k.left = 0; }
        k.sym_count = 0;
    }
    k.need_a = 0;
}
__device__ __forceinline__ void coder_advance(Coder &k, int start, int freq) {
    // ans.rs:230-244
    k.need_a = k.need_b | ((k.sym_count == NUM_SYMBOLS_BEFORE_FLUSH - 1) ? 8u : 0u);
    uint64_t x = (uint64_t)(int64_t)freq * (k.a >> 15) + (k.a & 0x7fff) - (uint64_t)(int64_t)start;
    k.sym_count = k.sym_count + 1;   // reset by the 16-byte re-initialisation that always follows symbol 65535
    k.need_b = (x < (1ull << 31)) ? 1u : 0u;
    k.a = k.b; k.b = x;
}

// exact floor((c<<15)/max): the reference divides through a reciprocal LUT that is asserted equal to integer
// division (probability/numeric.rs:26-31, make_div_lut.rs:37-39).  fp32 estimate + integer fix-up: c<<15 has <=16
// significant bits, so the estimate is within 1 of the true quotient (<= 2^16).
// The reference's divide, literally (probability/numeric.rs:14-31 with RECIPROCAL[d as u16] = compute_divisor(d),
// make_div_lut.rs:29-41).  Only reached with operands outside the adaptive range 0 <= c <= max <= 0x7fff, i.e. after a
// stream-supplied speed made an i16 counter wrap (frequentist_cdf.rs:74-85): there the LUT divide is NOT integer division
// and the decoder has to reproduce its exact value to stay in step with the reference.
static __device__ __noinline__ int cdf_div_ref(int c, int maxv) {
    const uint32_t d = (uint32_t)maxv & 0xffffu;
    const int32_t num = (int32_t)((uint32_t)c << 15);
    long long inv = 0; int shift = 0;
    if (d != 0) {
        const int bit_len = 32 - __clz((int)d);   // 16 - leading_zeros(u16)
        inv = ((((long long)1 << bit_len) - (long long)d) << 31) / (long long)d + 1;
        shift = bit_len - 1;
    }
    const long long m = inv * (long long)num;
    const int32_t t = (int32_t)(m >> 31);
    return (t + (((int32_t)((long long)num - (m >> 31))) >> 1)) >> shift;
}
__device__ __forceinline__ int cdf_div(int c, int maxv) {
    if (((unsigned)c | (unsigned)(maxv - 1)) > 0x7fffu) return cdf_div_ref(c, maxv);   // wrapped counters (never with the named speeds)
    uint32_t d = (uint32_t)maxv & 0xffffu;
    uint32_t n = (uint32_t)(c << 15);
    float rc;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(__uint2float_rz(d)));   // 1 ulp, fixed up below
    float q = __uint2float_rz(n) * rc;
    uint32_t qi = __float2uint_rz(q);
    int32_t r = (int32_t)(n - qi * d);
    if (r < 0) { qi--; r += (int32_t)d; }
    if (r >= (int32_t)d) qi++;
    return (int)qi;
}

// cdf_div for the literal fast loops: operands are known to be valid adaptive values (0 <= c <= max < 2^15), which lets
// both conversions use the 32-bit ALU path (I2FP) instead of the 16-bit XU conversion.
__device__ __forceinline__ int cdf_div_pos(int c, int maxv) {
    const uint32_t d = (uint32_t)maxv;
    const uint32_t n = (uint32_t)c << 15;
    float rc;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(__uint2float_rz(d)));
    uint32_t qi = __float2uint_rz(__uint2float_rz(n) * rc);
    int32_t r = (int32_t)(n - qi * d);
    if (r < 0) { qi--; r += (int32_t)d; }
    if (r >= (int32_t)d) qi++;
    return (int)qi;
}

// group-wide context handed around (all uniform except l16)
struct Grp {
    unsigned mask;     // participating lanes of this group
    int shift;         // 0 or 16: position of the group's 16 ballot bits
    int l16;           // lane & 15
    bool writer;       // lane that performs CDF stores for element l16 (false on the mirrored upper half)
    bool lane0;        // l16 == 0 (scalar work; true on lane 16 too when the upper half mirrors)
    bool store0;       // the single lane that performs scalar stores for the group
};

// freq only (for the mixing weights: codec/literal.rs:236-239)
__device__ __forceinline__ int cdf_freq(const Grp g, int c, int maxv, int sym) {
    int cum = cdf_div(c, maxv);
    int hi = __shfl_sync(g.mask, cum, sym, 16);
    int lo = __shfl_sync(g.mask, cum, (sym - 1) & 15, 16);
    if (sym == 0) lo = 0;
    return (int)(short)(hi - lo - 1);
}

__device__ __forceinline__ int cdf_blend(const Grp g, int c, int maxv, int sym, int inc, int lim) {
    // probability/frequentist_cdf.rs:74-85, i16 wrapping
    int c2 = (int)(short)(c + ((g.l16 >= sym) ? inc : 0));
    int nm = (int)(short)(maxv + inc);
    if (nm >= lim) {
        int t = (int)(short)(c2 + g.l16 + 1);
        c2 = (int)(short)(t - (t >> 2));
    }
    return c2;
}

// ---------------------------------------------------------------------------------------------------------------
// mixing weights (codec/weights.rs) -- uniform scalar math
// ---------------------------------------------------------------------------------------------------------------
struct Weights { int w0, w1; int norm; };   // norm kept as the u16 view used by literal.rs:230
__device__ __forceinline__ int weights_new(int prob, int weighted, int wi) {
    long long p1 = weighted, total = 1 << 15, p0 = total - p1;
    long long efficacy = total * (long long)prob - p1 * total;
    unsigned long long geo = (unsigned long long)(p1 * p0);
    int lg = geo ? 64 - __clzll((long long)geo) : 0;
    long long prod = (total - p1) * efficacy;
    long long adj = prod >> lg;
    int nw = (int)(unsigned int)(unsigned long long)((long long)wi + adj);
    return nw > 1 ? nw : 1;
}
__device__ __forceinline__ void weights_update(Weights &w, int f_cm, int f_nb, int weighted) {
    if (((w.w0 | w.w1) & 0x7f000000) != 0) {   // fix_weights, codec/weights.rs:64-79
        int ilog = 32 - min(__clz(w.w0), __clz(w.w1));
        if (ilog >= 24) { w.w0 >>= ilog - 24; w.w1 >>= ilog - 24; }
    }
    int n0 = weights_new(f_cm, weighted, w.w0);
    int n1 = weights_new(f_nb, weighted, w.w1);
    w.w0 = n0; w.w1 = n1;
    long long total = (long long)n0 + (long long)n1;        // compute_normalized_weight, :54-62
    int lz = __clzll(total);
    int shift = max(56 - lz, 0);
    unsigned d = (unsigned)(total >> shift) & 0xffu;
    int recip = d ? 1 + (1 << 24) / (int)d : 0;             // RECIPROCAL8 (div_lut.rs)
    unsigned num = ((unsigned)(n0 >> shift) << 8) & 0xffffu;
    int q = (int)(short)(((long long)recip * (long long)num) >> 24);
    w.norm = (int)(unsigned short)(q << 7);
}

// RECIPROCAL8[d] = 1 + 2^24 / d (d = 1..255; the reference's div_lut.rs table for compute_normalized_weight), [0] = 0
__constant__ uint32_t c_recip8[256] = {
    0u, 16777217u, 8388609u, 5592406u, 4194305u, 3355444u, 2796203u, 2396746u,
    2097153u, 1864136u, 1677722u, 1525202u, 1398102u, 1290556u, 1198373u, 1118482u,
    1048577u, 986896u, 932068u, 883012u, 838861u, 798916u, 762601u, 729445u,
    699051u, 671089u, 645278u, 621379u, 599187u, 578525u, 559241u, 541201u,
    524289u, 508401u, 493448u, 479350u, 466034u, 453439u, 441506u, 430186u,
    419431u, 409201u, 399458u, 390168u, 381301u, 372828u, 364723u, 356963u,
    349526u, 342393u, 335545u, 328966u, 322639u, 316552u, 310690u, 305041u,
    299594u, 294338u, 289263u, 284360u, 279621u, 275037u, 270601u, 266306u,
    262145u, 258112u, 254201u, 250407u, 246724u, 243149u, 239675u, 236299u,
    233017u, 229825u, 226720u, 223697u, 220753u, 217886u, 215093u, 212370u,
    209716u, 207127u, 204601u, 202136u, 199729u, 197380u, 195084u, 192842u,
    190651u, 188509u, 186414u, 184366u, 182362u, 180401u, 178482u, 176603u,
    174763u, 172961u, 171197u, 169467u, 167773u, 166112u, 164483u, 162886u,
    161320u, 159784u, 158276u, 156797u, 155345u, 153920u, 152521u, 151147u,
    149797u, 148471u, 147169u, 145889u, 144632u, 143396u, 142180u, 140986u,
    139811u, 138655u, 137519u, 136401u, 135301u, 134218u, 133153u, 132105u,
    131073u, 130056u, 129056u, 128071u, 127101u, 126145u, 125204u, 124276u,
    123362u, 122462u, 121575u, 120700u, 119838u, 118988u, 118150u, 117324u,
    116509u, 115705u, 114913u, 114131u, 113360u, 112599u, 111849u, 111108u,
    110377u, 109656u, 108943u, 108241u, 107547u, 106862u, 106185u, 105518u,
    104858u, 104207u, 103564u, 102928u, 102301u, 101681u, 101068u, 100463u,
    99865u, 99274u, 98690u, 98113u, 97542u, 96979u, 96421u, 95870u,
    95326u, 94787u, 94255u, 93728u, 93207u, 92692u, 92183u, 91679u,
    91181u, 90688u, 90201u, 89718u, 89241u, 88769u, 88302u, 87839u,
    87382u, 86929u, 86481u, 86038u, 85599u, 85164u, 84734u, 84308u,
    83887u, 83469u, 83056u, 82647u, 82242u, 81841u, 81443u, 81050u,
    80660u, 80274u, 79892u, 79513u, 79138u, 78767u, 78399u, 78034u,
    77673u, 77315u, 76960u, 76609u, 76261u, 75916u, 75574u, 75235u,
    74899u, 74566u, 74236u, 73909u, 73585u, 73263u, 72945u, 72629u,
    72316u, 72006u, 71698u, 71393u, 71090u, 70790u, 70493u, 70198u,
    69906u, 69616u, 69328u, 69043u, 68760u, 68479u, 68201u, 67924u,
    67651u, 67379u, 67109u, 66842u, 66577u, 66314u, 66053u, 65794u,
};

// 32-bit restatement of weights_update for the literal fast path.  Identical results whenever the coded frequencies
// are in 1..32767 (always true for streams an encoder can produce): efficacy = 2^15 * (prob - p1) and
// prod = p0 * efficacy, so prod >> lg is (p0 * (prob - p1)) shifted by (15 - lg) -- no 64-bit arithmetic needed.
__device__ __forceinline__ int weights_new32(int prob, int p1, int p0, int lg, int wi) {
    const int t = p0 * (prob - p1);
    const int adj = lg <= 15 ? (int)((unsigned)t << (15 - lg)) : (t >> (lg - 15));
    const int nw = (int)((unsigned)wi + (unsigned)adj);
    return nw > 1 ? nw : 1;
}
__device__ __forceinline__ void weights_update32(Weights &w, int f_cm, int f_nb, int weighted) {
    if (((w.w0 | w.w1) & 0x7f000000) != 0) {   // fix_weights, codec/weights.rs:64-79
        int ilog = 32 - min(__clz(w.w0), __clz(w.w1));
        if (ilog >= 24) { w.w0 >>= ilog - 24; w.w1 >>= ilog - 24; }
    }
    const int p0 = (1 << 15) - weighted;
    const unsigned geo = (unsigned)(weighted * p0);
    const int lg = geo ? 32 - __clz((int)geo) : 0;
    const int n0 = weights_new32(f_cm, weighted, p0, lg, w.w0);
    const int n1 = weights_new32(f_nb, weighted, p0, lg, w.w1);
    w.w0 = n0; w.w1 = n1;
    const unsigned total = (unsigned)n0 + (unsigned)n1;       // compute_normalized_weight, :54-62 (total < 2^32)
    const int shift = max(24 - __clz((int)total), 0);
    const unsigned d = (total >> shift) & 0xffu;
    const int recip = (int)c_recip8[d];
    const unsigned num = ((unsigned)(n0 >> shift) << 8) & 0xffffu;
    const int q = (int)(short)(((unsigned long long)(unsigned)recip * num) >> 24);
    w.norm = (int)(unsigned short)(q << 7);
}

}  // namespace dv
