// numeric_ref.h -- the reference's CDF division (probability/numeric.rs:14-31, the divisor rule of make_div_lut.rs:29-41)
// restated in 64-bit integers, independently of the product's cdf_div_ref.  Host and device: dv_probe.cu compares the
// product's cdf_div with it on the GPU, and tests/test_arith_domains.py compiles it with g++ and compares it with the
// oracle's dvo_fast_divide on every (c, max) of the i16 domain.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define DVP_HD __host__ __device__
#else
#define DVP_HD
#endif

// compute_divisor(d as u16): (inv, shift) with bit_len = the number of significant bits of d; d = 0 gives (0, 0)
DVP_HD inline void dvp_divisor(uint16_t d, int64_t &inv, int &shift) {
    inv = 0; shift = 0;
    if (d == 0) return;
    int bit_len = 0;
    while (bit_len < 16 && (d >> bit_len) != 0) bit_len++;
    inv = ((((int64_t)1 << bit_len) - (int64_t)d) << 31) / (int64_t)d + 1;
    shift = bit_len - 1;
}
// fast_divide_30bit_by_16bit(num, divisor): i64 product, i32 truncations and arithmetic shifts as numeric.rs:26-31 writes them
DVP_HD inline int32_t dvp_fast_divide(int32_t num, int64_t inv, int shift) {
    const int64_t m = inv * (int64_t)num;
    const int32_t t = (int32_t)(m >> 31);
    const int32_t half = (int32_t)((int64_t)num - (m >> 31)) >> 1;
    return (int32_t)((uint32_t)t + (uint32_t)half) >> shift;   // the i32 sum wraps
}
// the quotient the reference's CDF uses for element c of a CDF whose last element is maxv (probability/interface.rs:97-108):
// (c << 15) in i32 (wrapping), divided by maxv as u16
DVP_HD inline int32_t dvp_cdf_quotient(int16_t c, int16_t maxv) {
    int64_t inv; int shift;
    dvp_divisor((uint16_t)maxv, inv, shift);
    return dvp_fast_divide((int32_t)((uint32_t)(int32_t)c << 15), inv, shift);
}
