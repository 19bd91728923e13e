// arith_host.cpp -- host-side halves of tests/test_arith_domains.py, compiled with g++.
//   arith_host divide <liboracle.so>: numeric_ref.h's dvp_cdf_quotient against the oracle's dvo_fast_divide on every (c, max)
//                                     of i16 x i16.  Prints "cases mismatches".
//   arith_host gate:                  for every i16 (inc, lim) that the fast-loop speed gate accepts (its four comparisons
//                                     restated here, dv_engine.cuh speed_is_small), the max recurrence of the blend
//                                     (frequentist_cdf.rs:74-85, the max is always incremented) from the default max 64
//                                     until it cycles.  Prints "accepted lowest highest" over every value an element takes
//                                     (before a rescale, the rescale's intermediate t, after it).
#include <dlfcn.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <thread>
#include <vector>

#include "numeric_ref.h"

static void parallel(int n_items, void (*fn)(int, void *), void *arg) {
    const int nt = std::max(1u, std::thread::hardware_concurrency());
    std::atomic<int> next(0);
    std::vector<std::thread> ts;
    for (int t = 0; t < nt; t++)
        ts.emplace_back([&] { for (int i; (i = next.fetch_add(1)) < n_items;) fn(i, arg); });
    for (auto &t : ts) t.join();
}

typedef int32_t (*fast_divide_fn)(int32_t, int16_t);
struct DivideJob { fast_divide_fn oracle; std::atomic<unsigned long long> cases, bad; };
static void divide_row(int row, void *arg) {
    DivideJob *j = (DivideJob *)arg;
    const int16_t d = (int16_t)(row - 32768);
    unsigned long long bad = 0;
    for (int c = -32768; c <= 32767; c++) {
        if (dvp_cdf_quotient((int16_t)c, d) != j->oracle((int32_t)((uint32_t)(int32_t)c << 15), d)) {
            if (bad < 4) printf("# mismatch c=%d max=%d\n", c, d);
            bad++;
        }
    }
    j->cases += 65536; j->bad += bad;
}

struct GateJob { std::atomic<unsigned long long> accepted; std::atomic<int> lowest, highest; };
// The authoritative gate is the product's speed_is_small (dv_engine.cuh).  tests/test_gpu_arith.py ties its restatement in
// tests/regimes.py to it on every i16 pair; this copy must equal that restatement, and the gate test checks its accepted count.
static bool gate(int inc, int lim) { return inc >= 0 && lim >= 0 && lim + inc + 16 <= 0x7fff && 4 * (inc + 16) <= 0x7fff; }
struct Wave { int inc, lim, lo, hi; };
// from max m (a value after a rescale, or the default): the plain steps, then the one that rescales; returns the max after
// that rescale (m itself when no step ever rescales).  Records every value on the way in lo / hi.
static int wave(Wave &w, int m) {
    if (m + w.inc < w.lim) {
        if (w.inc == 0) return m;                                  // never rescales: a fixed point
        const int p = (w.lim - m - w.inc + w.inc - 1) / w.inc;     // plain steps: m + j * inc < lim for j = 1..p
        m += p * w.inc;
        w.hi = std::max(w.hi, m);
    }
    const int nm = m + w.inc, t = nm + 16;                         // nm >= lim: rescale, t = c + 15 + 1 for the max
    w.hi = std::max(w.hi, t);
    const int r = t - (t >> 2);
    w.lo = std::min(w.lo, r);
    return r;
}
static void gate_row(int row, void *arg) {
    GateJob *j = (GateJob *)arg;
    const int inc = row - 32768;
    unsigned long long acc = 0;
    int lo = 64, hi = 64;
    for (int lim = -32768; lim <= 32767; lim++) {
        if (!gate(inc, lim)) continue;
        acc++;
        Wave w{inc, lim, 64, 64};
        // Brent's cycle detection on the wave map: the hare visits every wave up to and through the first full cycle
        int power = 1, lam = 1, tortoise = 64, hare = wave(w, 64);
        while (tortoise != hare) {
            if (power == lam) { tortoise = hare; power *= 2; lam = 0; }
            hare = wave(w, hare);
            lam++;
        }
        lo = std::min(lo, w.lo); hi = std::max(hi, w.hi);
    }
    j->accepted += acc;
    int v = j->lowest.load();
    while (lo < v && !j->lowest.compare_exchange_weak(v, lo)) {}
    v = j->highest.load();
    while (hi > v && !j->highest.compare_exchange_weak(v, hi)) {}
}

int main(int argc, char **argv) {
    if (argc >= 3 && !strcmp(argv[1], "divide")) {
        void *h = dlopen(argv[2], RTLD_NOW);
        if (!h) { fprintf(stderr, "%s\n", dlerror()); return 2; }
        DivideJob j;
        j.oracle = (fast_divide_fn)dlsym(h, "dvo_fast_divide");
        j.cases = 0; j.bad = 0;
        if (!j.oracle) return 2;
        parallel(65536, divide_row, &j);
        printf("%llu %llu\n", j.cases.load(), j.bad.load());
        return 0;
    }
    if (argc >= 2 && !strcmp(argv[1], "gate")) {
        GateJob j;
        j.accepted = 0; j.lowest = 64; j.highest = 64;
        parallel(65536, gate_row, &j);
        printf("%llu %d %d\n", j.accepted.load(), j.lowest.load(), j.highest.load());
        return 0;
    }
    fprintf(stderr, "usage: arith_host divide <liboracle.so> | gate\n");
    return 2;
}
