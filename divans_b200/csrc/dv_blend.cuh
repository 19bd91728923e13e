// dv_blend.cuh -- the reference's feature="blend" probability model (BlendCDF16, probability/blend_cdf.rs:109-208) for the
// generic nibble core: SURVEY 8 row f-4.  A compile-time switch of the whole crate there (src/interface.rs:146-147), a kernel
// template parameter here; streams coded with it are not marked, caller and producer have to agree
// (DIVANS_B200_FLAG_CDF_BLEND / divans_b200_encode_options::cdf_model).
//
// State of a BlendCDF16: 16 cumulative counts in [0, CDF_MAX - 16] (i16), `count` (only count & 15 is ever used) and
// `mix_rate` (1536, multiplied by 127/128 after every blend until it stays at 127: a function of the number of blends).
// In HBM a blend prior is the same 32 bytes as a frequentist one: the counts are non-negative, so the sign bits of elements
// 0..8 hold the number of blends k (k -> k + 1, 511 -> 496: congruent to count modulo 16 and past step 386, where the rate
// reaches 127).  A zeroed prior is BlendCDF16::default().  The model needs no division: max() is the constant CDF_MAX and
// div_by_max is a shift (:148-159).
#pragma once
#include "dv_engine_kernel.cuh"

namespace dv {

constexpr int BLEND_CDF_MAX = 32767;             // probability/interface.rs:429
constexpr int BLEND_DEL = BLEND_CDF_MAX - 16;    // blend_cdf.rs:80,90
// mix_rate before blend number k (k = 0, 1, ...): m(0) = (1 << 10) + (1 << 9), m(k + 1) = m(k) - (m(k) >> 7)   (:131-134,203)
static __constant__ uint16_t c_blend_mix[512] = {
    1536, 1524, 1513, 1502, 1491, 1480, 1469, 1458, 1447, 1436, 1425, 1414, 1403, 1393, 1383, 1373,
    1363, 1353, 1343, 1333, 1323, 1313, 1303, 1293, 1283, 1273, 1264, 1255, 1246, 1237, 1228, 1219,
    1210, 1201, 1192, 1183, 1174, 1165, 1156, 1147, 1139, 1131, 1123, 1115, 1107, 1099, 1091, 1083,
    1075, 1067, 1059, 1051, 1043, 1035, 1027, 1019, 1012, 1005,  998,  991,  984,  977,  970,  963,
     956,  949,  942,  935,  928,  921,  914,  907,  900,  893,  887,  881,  875,  869,  863,  857,
     851,  845,  839,  833,  827,  821,  815,  809,  803,  797,  791,  785,  779,  773,  767,  762,
     757,  752,  747,  742,  737,  732,  727,  722,  717,  712,  707,  702,  697,  692,  687,  682,
     677,  672,  667,  662,  657,  652,  647,  642,  637,  633,  629,  625,  621,  617,  613,  609,
     605,  601,  597,  593,  589,  585,  581,  577,  573,  569,  565,  561,  557,  553,  549,  545,
     541,  537,  533,  529,  525,  521,  517,  513,  509,  506,  503,  500,  497,  494,  491,  488,
     485,  482,  479,  476,  473,  470,  467,  464,  461,  458,  455,  452,  449,  446,  443,  440,
     437,  434,  431,  428,  425,  422,  419,  416,  413,  410,  407,  404,  401,  398,  395,  392,
     389,  386,  383,  381,  379,  377,  375,  373,  371,  369,  367,  365,  363,  361,  359,  357,
     355,  353,  351,  349,  347,  345,  343,  341,  339,  337,  335,  333,  331,  329,  327,  325,
     323,  321,  319,  317,  315,  313,  311,  309,  307,  305,  303,  301,  299,  297,  295,  293,
     291,  289,  287,  285,  283,  281,  279,  277,  275,  273,  271,  269,  267,  265,  263,  261,
     259,  257,  255,  254,  253,  252,  251,  250,  249,  248,  247,  246,  245,  244,  243,  242,
     241,  240,  239,  238,  237,  236,  235,  234,  233,  232,  231,  230,  229,  228,  227,  226,
     225,  224,  223,  222,  221,  220,  219,  218,  217,  216,  215,  214,  213,  212,  211,  210,
     209,  208,  207,  206,  205,  204,  203,  202,  201,  200,  199,  198,  197,  196,  195,  194,
     193,  192,  191,  190,  189,  188,  187,  186,  185,  184,  183,  182,  181,  180,  179,  178,
     177,  176,  175,  174,  173,  172,  171,  170,  169,  168,  167,  166,  165,  164,  163,  162,
     161,  160,  159,  158,  157,  156,  155,  154,  153,  152,  151,  150,  149,  148,  147,  146,
     145,  144,  143,  142,  141,  140,  139,  138,  137,  136,  135,  134,  133,  132,  131,  130,
     129,  128,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,
     127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,
     127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,
     127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,
     127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,
     127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,
     127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,
     127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127,  127};

// BaseCDF::cdf() of every lane's symbol (:160-171): the difference between cdf[15] and CDF_MAX is a latent uniform distribution
__device__ __forceinline__ int blend_value(const int c, const int l16) {
    const int c15 = __shfl_sync(FULL, c, 15, 16);
    return l16 == 15 ? BLEND_CDF_MAX : (int)(short)(c + (((BLEND_CDF_MAX - c15) * (l16 + 1)) >> 4));
}
// blend_internal (:111-126): mul_blend of the lane's element (:15-55), then the early-growth step
__device__ __forceinline__ int blend_internal(const int base, const int to_blend, const int mix_rate, const int count) {
    const int bias = (count & 0xf) << (15 - 4);
    int e = (int)((unsigned)to_blend * (unsigned)mix_rate + (unsigned)base * (unsigned)((1 << 15) - mix_rate) + (unsigned)bias) >> 15;
    e = (int)(short)e;
    const int e15 = __shfl_sync(FULL, e, 15, 16);
    if (e15 < (int)(short)(BLEND_DEL - (e15 >> 1))) e = (int)(short)(e + (e >> 1));
    return e;
}
// CDF16::blend (:186-208; the Speed argument is computed into `_mix_rate` and not used) on the lane's element; returns the
// element to store, sign bit = this lane's bit of the new number of blends
__device__ __forceinline__ int blend_update(const int c, const int k, const int sym, const int l16) {
    const int e = blend_internal(c, l16 >= sym ? BLEND_DEL : 0, (int)c_blend_mix[k], k + 1);   // count is incremented first
    const int k2 = k == 511 ? 496 : k + 1;
    return (e & 0x7fff) | ((l16 < 9 && ((k2 >> l16) & 1)) ? 0x8000 : 0);
}

// one nibble of a 16-lane group, decoded (ENC = false) or encoded (ENC = true)
template <bool ENC>
__device__ __forceinline__ int nibble_core_blend(St &s, const Next &nx, const G2 g) {
    const int raw = nx.cdf[g.l16];
    const int c = raw & 0x7fff;
    const int k = (int)((__ballot_sync(FULL, raw < 0) >> g.shift) & 0x1ffu);
    const bool mixg = nx.cdf2 != nullptr;
    const bool anymix = __any_sync(FULL, mixg);
    const int v_nb = blend_value(c, g.l16);
    int cc = 0, k_cm = 0, v_cm = 0, cu = v_nb;
    Weights w = {1, 1, 1 << 14};
    if (anymix) {   // dynamic context mixing >= 2 (codec/literal.rs:219-243): cm_prob.average(nibble_prob, norm_weight)
        const int raw2 = mixg ? (int)nx.cdf2[g.l16] : 0;
        cc = raw2 & 0x7fff;
        k_cm = (int)((__ballot_sync(FULL, raw2 < 0) >> g.shift) & 0x1ffu);
        w = nx.mix_hi ? s.c->w_hi : s.c->w_lo;
        v_cm = blend_value(cc, g.l16);
        const int avg = blend_internal(cc, c, w.norm, k_cm);   // average(): self = the context-map prior, its count, no increment (:181-185)
        const int v_avg = blend_value(avg, g.l16);
        if (mixg) cu = v_avg;
    }
    int sym;
    if (!ENC) {
        coder_fill(s.cur);
        const int off = (int)(s.cur.a & 0x7fff);
        const int r = (int)(short)((off * BLEND_CDF_MAX) >> 15);              // probability/interface.rs:140, max() = CDF_MAX
        const unsigned bal = __ballot_sync(FULL, (g.l16 == 15) || (r < cu));
        sym = __ffs((bal >> g.shift) & 0xffffu) - 1;
    } else sym = nx.sym;
    // sym_to_start_and_freq (probability/interface.rs:97-108) with div_by_max = >> 15: the values themselves
    const int prev = (sym - 1) & 15;
    const int hi = __shfl_sync(FULL, cu, sym, 16);
    int lo = __shfl_sync(FULL, cu, prev, 16);
    if (sym == 0) lo = 0;
    const int start = (int)(short)(lo + 1), freq = (int)(short)(hi - lo - 1);
    if (!ENC) coder_advance(s.cur, start, freq);
    else {
        if (freq <= 0 && s.state != S_IDLE) s.status = ST_FAIL;   // a symbol whose probability has decayed to the bias floor cannot be coded
        if (g.store0) const_cast<uint32_t *>(s.cur.p)[s.cur.left] = ((uint32_t)start & 0xffffu) | ((uint32_t)freq << 16);
        s.cur.left++;
    }
    if (anymix) {
        const int h_cm = __shfl_sync(FULL, v_cm, sym, 16), h_nb = __shfl_sync(FULL, v_nb, sym, 16);
        int l_cm = __shfl_sync(FULL, v_cm, prev, 16), l_nb = __shfl_sync(FULL, v_nb, prev, 16);
        if (sym == 0) { l_cm = 0; l_nb = 0; }
        const int cm_new = blend_update(cc, k_cm, sym, g.l16);
        if (mixg) {
            weights_update(w, (int)(short)(h_cm - l_cm - 1), (int)(short)(h_nb - l_nb - 1), freq);
            if (nx.mix_hi) s.c->w_hi = w; else s.c->w_lo = w;
            nx.cdf2[g.l16] = (int16_t)cm_new;
        }
    }
    const int nb_new = blend_update(c, k, sym, g.l16);
    if (nx.speed != SPK_NONE) nx.cdf[g.l16] = (int16_t)nb_new;   // SPK_NONE: the never-adapted default prior / a read-only stride prior
    return sym;
}

}  // namespace dv
