// dv_split_probe.cu -- libdivans_b200_split_probe.so: the split rANS step of the 16-lane plain literal loop (rans_split16,
// dv2_core.cuh) as a plain C entry point, for tests/test_gpu_split_pair.py.  TEST INFRASTRUCTURE: built by
// divans_b200/csrc/Makefile next to libdivans_b200.so, never linked into it.  It includes the product sources unchanged and
// calls their functions, not copies of them.  The entry point takes host arrays, allocates, copies, launches on device 0,
// copies back and frees, and returns a CUDA error code (0 = success).
#include <stdio.h>
#include <string.h>
#include "dv2_core.cuh"

namespace {

#define PK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { err = e_; goto done; } } while (0)

// ---- one literal byte of the 16-lane plain loop with its rANS pair split across the group (rans_split16), one group per case:
// both searches, then the split step and its refill from the case's 8 payload words ----
struct SplitIo {
    const int16_t *cdf_h, *cdf_l; const uint64_t *a, *b; const uint32_t *words, *wi, *wmax;
    int32_t *h, *l; uint64_t *a_out, *b_out; uint32_t *wi_out, *under;
    size_t n;
};
__global__ void split_byte_kernel(SplitIo io) {
    const int lane = threadIdx.x & 31;
    const size_t pc = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) / 16, i = pc < io.n ? pc : io.n - 1;
    dv::G2 g;
    g.l16 = lane & 15; g.shift = lane & 16; g.gmask = 0xffffu << g.shift; g.store0 = g.l16 == 0; g.nl = 16; g.grp = 0; g.blend = false;
    const uint32_t eh = (uint16_t)io.cdf_h[16 * i + g.l16], mh = (uint16_t)io.cdf_h[16 * i + 15];
    const uint32_t el = (uint16_t)io.cdf_l[16 * i + g.l16], ml = (uint16_t)io.cdf_l[16 * i + 15];
    dv::FastK f;
    f.wbase = io.words + 8 * i; f.wi = io.wi[i]; f.wmax = io.wmax[i]; f.wnext = f.wbase[f.wi];
    const uint32_t bsel = 0xffffu << g.shift;
    const int h = dv::search_v2<16>(io.a[i], eh, mh, bsel), l = dv::search_v2<16>(io.b[i], el, ml, bsel);
    const bool bl = g.l16 >= 8;
    uint64_t x = bl ? io.b[i] : io.a[i];
    dv::rans_split16(x, eh, mh, h, el, ml, l, bl, bl ? 0x4432u : 0x4410u, g, f);
    const uint64_t a = __shfl_sync(dv::FULL, x, 0, 16), b = __shfl_sync(dv::FULL, x, 8, 16);
    if (pc < io.n && g.store0) {
        io.h[i] = h; io.l[i] = l; io.a_out[i] = a; io.b_out[i] = b; io.wi_out[i] = f.wi; io.under[i] = f.wi >= f.wmax;
    }
}

}  // namespace

extern "C" {

// One byte per case through rans_split16.  Inputs per case: the two validated priors (cdf_h[16], cdf_l[16], no tag bits), the
// states a and b, 8 payload words, the cursor wi and its bound wmax (wmax <= 7).  Outputs: both symbols, both states after
// the step and refill, the cursor, and whether it ended at or past wmax (the underflow coder_from_eager reports).
int dvp_split_byte(size_t n, const int16_t *cdf_h, const int16_t *cdf_l, const uint64_t *a, const uint64_t *b, const uint32_t *words,
                   const uint32_t *wi, const uint32_t *wmax, int32_t *h, int32_t *l, uint64_t *a_out, uint64_t *b_out,
                   uint32_t *wi_out, uint32_t *under) {
    cudaError_t err = cudaSuccess;
    SplitIo io;
    memset(&io, 0, sizeof io);
    void *bufs[14] = {};
    if (n == 0) return 0;
    for (size_t k = 0; k < n; k++) if (wmax[k] > 7 || wi[k] > wmax[k]) return (int)cudaErrorInvalidValue;
    PK(cudaSetDevice(0));
#define ALLOC(k, ptr, bytes) do { PK(cudaMalloc(&bufs[k], (bytes))); ptr = decltype(ptr)(bufs[k]); } while (0)
#define IN(k, ptr, src, bytes) do { ALLOC(k, ptr, bytes); PK(cudaMemcpy((void *)ptr, src, bytes, cudaMemcpyHostToDevice)); } while (0)
    IN(0, io.cdf_h, cdf_h, n * 32); IN(1, io.cdf_l, cdf_l, n * 32); IN(2, io.a, a, n * 8); IN(3, io.b, b, n * 8);
    IN(4, io.words, words, n * 32); IN(5, io.wi, wi, n * 4); IN(6, io.wmax, wmax, n * 4);
    ALLOC(7, io.h, n * 4); ALLOC(8, io.l, n * 4); ALLOC(9, io.a_out, n * 8); ALLOC(10, io.b_out, n * 8);
    ALLOC(11, io.wi_out, n * 4); ALLOC(12, io.under, n * 4);
#undef IN
#undef ALLOC
    io.n = n;
    split_byte_kernel<<<(unsigned)((n * 16 + 255) / 256), 256>>>(io);
    PK(cudaGetLastError());
    PK(cudaDeviceSynchronize());
    PK(cudaMemcpy(h, io.h, n * 4, cudaMemcpyDeviceToHost)); PK(cudaMemcpy(l, io.l, n * 4, cudaMemcpyDeviceToHost));
    PK(cudaMemcpy(a_out, io.a_out, n * 8, cudaMemcpyDeviceToHost)); PK(cudaMemcpy(b_out, io.b_out, n * 8, cudaMemcpyDeviceToHost));
    PK(cudaMemcpy(wi_out, io.wi_out, n * 4, cudaMemcpyDeviceToHost)); PK(cudaMemcpy(under, io.under, n * 4, cudaMemcpyDeviceToHost));
done:
    for (void *p : bufs) cudaFree(p);
    return (int)err;
}

}  // extern "C"
