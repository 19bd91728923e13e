// Micro-benchmark (dev tool): does prefetch.global.L1 shorten a later dependent load on sm_90a, and what do the load
// latencies look like?  One warp, one lane measuring with clock64.  Build: nvcc -gencode arch=compute_90a,code=sm_90a
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__global__ void k(const uint32_t *buf, size_t n_words, long long *out, int mode) {
    // buf is 1 GiB of words; walk random-ish addresses far apart so every first touch misses L1 and L2
    const int lane = threadIdx.x;
    unsigned long long acc = 0;
    long long tsum = 0;
    size_t idx = 12345 + 977 * blockIdx.x;
    for (int it = 0; it < 256; it++) {
        idx = (idx * 2862933555777941757ull + 3037000493ull) % (n_words / 64);
        const uint32_t *p = buf + idx * 64 + lane % 8;    // 8 lanes share a 32 B sector
        if (mode == 1) asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
        if (mode == 2) asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
        if (mode == 3) { uint32_t t; asm volatile("ld.global.ca.u32 %0, [%1];" : "=r"(t) : "l"(p)); acc += t; }
        // wait ~3000 cycles doing ALU work that does not depend on memory
        long long t0 = clock64();
        while (clock64() - t0 < 3000) { }
        long long a = clock64();
        uint32_t v;
        asm volatile("ld.global.ca.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
        acc += v;
        asm volatile("" ::"l"(acc));
        long long b = clock64();
        // second touch: L1 hit latency
        uint32_t v2;
        asm volatile("ld.global.ca.u32 %0, [%1];" : "=r"(v2) : "l"(p + 0) : "memory");
        acc += v2;
        asm volatile("" ::"l"(acc));
        long long c = clock64();
        if (lane == 0) { tsum += b - a; out[2 + it % 2] = c - b; }
    }
    if (lane == 0) { out[0] = tsum / 256; out[1] = (long long)acc; }
}
int main() {
    size_t n = (size_t)1 << 28;   // 1 GiB
    uint32_t *buf; cudaMalloc(&buf, n * 4); cudaMemset(buf, 1, n * 4);
    long long *out; cudaMallocManaged(&out, 64);
    const char *names[] = {"no prefetch (first touch)", "prefetch.global.L1 3000 cyc earlier", "prefetch.global.L2 3000 cyc earlier", "ld.ca dummy 3000 cyc earlier"};
    for (int mode = 0; mode < 4; mode++) {
        k<<<1, 32>>>(buf, n, out, mode);
        cudaDeviceSynchronize();
        printf("%-40s first load %lld cycles, repeat (L1 hit) %lld cycles\n", names[mode], out[0], out[2]);
    }
    printf("err=%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
