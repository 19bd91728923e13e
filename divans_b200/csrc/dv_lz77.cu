// dv_lz77.cu -- sm_90a kernel of divans_b200_lz77_cmds_batch_device: the library's greedy hash-chain LZ77 (dv_ir.cpp,
// lz77_blob) run next to raw buffers in HBM.  Every blob is byte for byte the one the host generator writes for the same input
// and arguments.  The host's rules:
//   h4(i) = (le32(in + i) * 2654435761) >> 17, for positions with i + 4 <= n only; every such position is inserted, in order,
//   copies included.  The candidates of position i are the (at most 16) most recent earlier positions of the same hash, walked
//   newest first and up to the first farther than 2^window - 16.  The longest match of at most min(n - i, 65535) bytes wins, a
//   tie going to the newer candidate; a match of 4 or more bytes is a copy, anything shorter leaves the byte a literal.
//
// One warp per stream; persistent warps pull stream indices from the work counter, so any n runs in one launch.  Each warp owns
// a head table (2^15 entries) and prev[max_in_len] in global memory.  Per stream:
//  1. Chain pass.  prev[i] = the most recent j < i of the same hash (or -1): the candidates of i are prev[i], prev[prev[i]], ...
//     whatever the parse does, so the whole array is built first, 32 positions at a time.  Lanes of equal hash are grouped by
//     __match_any_sync; a lane's prev is the nearest lower lane of its group, or head[h]; the highest lane of a group writes
//     head[h].  The head table is reset for every stream: a stale entry would be a candidate from another stream.
//  2. Parse, 32 positions per window.  Lane t walks the chain of position p + t and compares every candidate up to LZ_CAP
//     bytes, word by word.  The warp then replays the greedy parse over the window from the ballot of lanes with a match of
//     4 or more: literal bytes up to the next such lane, its copy, and on from the copy's end while it stays in the window.  A
//     copy whose capped length reached LZ_CAP (and could be longer) is measured exactly, by the whole warp, for each candidate
//     that reached the cap, in chain order: only those can be the longest.  So per window a lane spends at most 16 capped
//     compares, and exact lengths are measured only where the parse lands.
//  3. Emit.  Records go out as they are found, at blob + 32 + 20k, while they fit the region; then the header, the
//     PredictionMode record (built once per call on the host) and the literal pool, which is the raw stream.  A blob that
//     does not fit is still parsed to the end, so its exact size is reported.
#include "dv_common.cuh"
#include "dv_lz77.h"

namespace dv {

constexpr int LZ_BLOCK_THREADS = 64;
constexpr int LZ_WARPS = LZ_BLOCK_THREADS / 32;
constexpr unsigned LZ_FULL = 0xffffffffu;
constexpr int LZ_CHAIN = 16;           // candidates per position
constexpr int32_t LZ_CAP = 64;         // bytes of the capped compare
constexpr int32_t LZ_MAX_COPY = 65535;
constexpr uint32_t LZ_MIN_COPY = 4;

// The four bytes at p (p < end) as a little-endian word, from the aligned words that hold them.  The second word is read only
// when it starts below `end`: no word without a byte of the stream is read.
__device__ __forceinline__ uint32_t lz_word(const uint8_t *p, const uint8_t *end) {
    const uintptr_t a = (uintptr_t)p;
    const uint32_t *w = reinterpret_cast<const uint32_t *>(a & ~(uintptr_t)3);
    const uint32_t lo = __ldg(w);
    const uint32_t hi = reinterpret_cast<const uint8_t *>(w + 1) < end ? __ldg(w + 1) : 0u;
    return __funnelshift_r(lo, hi, (uint32_t)(a & 3u) * 8u);
}

// Candidates of position q, newest first: c = prev[q], prev[c], ... while c >= 0, at most LZ_CHAIN of them, stopping at the
// first farther than maxdist.  Lane-private.  Returns the longest match capped at cl = min(lim, LZ_CAP) (the first of equal
// length) and sets bit j of `hits` for every candidate j that reached the cap.
__device__ __forceinline__ int32_t lz_capped(const uint8_t *in, const uint8_t *end, const int32_t *prev, int32_t q, int32_t lim,
                                             int32_t maxdist, int32_t &dist, uint32_t &hits) {
    const int32_t cl = min(lim, LZ_CAP);
    int32_t best = 0, c = prev[q];
    for (int j = 0; c >= 0 && q - c <= maxdist; j++) {
        int32_t l = 0;
        for (; l < cl; l += 4) {
            const uint32_t x = lz_word(in + c + l, end) ^ lz_word(in + q + l, end);
            if (x) { l += (__ffs(x) - 1) >> 3; break; }
        }
        l = min(l, cl);
        if (l == cl) hits |= 1u << j;
        if (l > best) { best = l; dist = q - c; }
        if (j + 1 == LZ_CHAIN) break;
        c = prev[c];
    }
    return best;
}

// The exact length of the copy at q (warp-uniform arguments): the candidates in `hits` (chain indices that reached LZ_CAP) are
// measured in chain order from LZ_CAP on, 128 bytes per step across the warp; the longest wins, ties to the newer one.
// Returns (length, distance).  (Out of line: the common short copy keeps the kernel's registers.)
__device__ __noinline__ int2 lz_extend(const uint8_t *in, const uint8_t *end, const int32_t *prev, int32_t q, int32_t lim, uint32_t hits) {
    const int lane = threadIdx.x & 31;
    int32_t best = 0, dist = 0, c = prev[q];
    for (int j = 0; hits >> j; j++) {
        if ((hits >> j) & 1u) {
            int32_t l = LZ_CAP;
            for (;;) {
                const int32_t o = l + 4 * lane;
                int32_t stop = -1;   // where this lane's four bytes end the match, if they do
                if (o >= lim) stop = lim;
                else {
                    const uint32_t x = lz_word(in + c + o, end) ^ lz_word(in + q + o, end);
                    if (x) stop = min(o + (int32_t)((__ffs(x) - 1) >> 3), lim);
                }
                const uint32_t b = __ballot_sync(LZ_FULL, stop >= 0);
                if (b) { l = __shfl_sync(LZ_FULL, stop, __ffs(b) - 1); break; }
                l += 128;
            }
            if (l > best) { best = l; dist = q - c; }
        }
        c = prev[c];
    }
    return make_int2(best, dist);
}

// (launch bounds: 16 blocks, 32 warps per SM, the most a context's max_resident asks for; without the minimum ptxas spilled)
__global__ void __launch_bounds__(LZ_BLOCK_THREADS, 16) lz77_cmds_kernel(Lz77Params p) {
    const int lane = threadIdx.x & 31;
    const uint32_t warp = blockIdx.x * LZ_WARPS + (threadIdx.x >> 5);
    if (warp >= p.n_warps) return;
    int32_t *const head = p.scratch + (size_t)warp * p.stride;
    int32_t *const prev = head + LZ_HEAD_ENTRIES;
    const int32_t maxdist = (int32_t)((1u << p.window) - 16u);
    for (;;) {
        uint32_t v = 0;
        if (lane == 0) v = atomicAdd(p.work_counter, 1u);
        v = __shfl_sync(LZ_FULL, v, 0);
        if (v >= p.n_streams) break;
        const uint64_t n64 = p.in_len[v], boff = p.blob_off[v], cap = p.blob_cap[v];
        // refused, with nothing read: records are written as u32, and positions are int32 as in the host generator.  Below,
        // int32 positions stay below n, and what can pass n (the chain pass's window base) is 64-bit, so no stream of up to
        // 2^31 - 1 bytes wraps.
        if ((boff & 3u) != 0 || n64 > p.max_in_len || n64 >= (1ull << 31)) {
            if (lane == 0) { p.blob_len[v] = 0; p.status[v] = ST_FAIL; }
            continue;
        }
        const int32_t n = (int32_t)n64, nh = n - 3;   // positions i < nh have i + 4 <= n
        const uint8_t *const in = p.in + p.in_off[v], *const end = in + n;
        uint8_t *const blob = p.blobs + boff;

        // 1. chain pass
        int4 *const h4 = reinterpret_cast<int4 *>(head);
        for (uint32_t k = lane; k < LZ_HEAD_ENTRIES / 4; k += 32) h4[k] = make_int4(-1, -1, -1, -1);
        __syncwarp();
        for (int64_t base = 0; base < nh; base += 32) {
            const bool ok = base + lane < nh;
            const int32_t i = ok ? (int32_t)(base + lane) : 0;
            const uint32_t h = ok ? (lz_word(in + i, end) * 2654435761u) >> 17 : 0x80000000u | lane;   // (unique: no group)
            const uint32_t grp = __match_any_sync(LZ_FULL, h);
            const uint32_t lower = grp & ((1u << lane) - 1u);
            int32_t pv = 0;
            if (ok) pv = lower ? (int32_t)base + 31 - __clz(lower) : head[h];
            __syncwarp();   // every lane has read head before a group's highest lane replaces the entry
            if (ok) {
                prev[i] = pv;
                if ((grp >> lane) == 1u) head[h] = i;
            }
            __syncwarp();
        }

        // 2. parse, 3. records
        uint32_t n_cmds = 0;
        auto emit = [&](uint32_t type, uint32_t a, uint32_t b) {
            if (32ull + 20ull * (n_cmds + 1) <= cap && lane < 5)
                reinterpret_cast<uint32_t *>(blob + 32 + 20ull * n_cmds)[lane] = lane == 0 ? type : lane == 1 ? a : lane == 2 ? b : 0u;
            n_cmds++;
        };
        emit(7, 0, 0);   // the PredictionMode command: record 0
        int32_t pos = 0, lit_start = 0;
        while (pos < n) {
            const int32_t span = min(32, n - pos);   // the window: positions pos .. pos + span - 1, all below n
            const int32_t q = lane < span ? pos + lane : n;
            int32_t best = 0, dist = 0, lim = 0;
            uint32_t hits = 0;
            if (q < nh) {
                lim = min(n - q, LZ_MAX_COPY);
                best = lz_capped(in, end, prev, q, lim, maxdist, dist, hits);
            }
            const uint32_t copies = __ballot_sync(LZ_FULL, best >= (int32_t)LZ_MIN_COPY);
            const int32_t wend = pos + span;
            int32_t at = pos;   // the parse position in this window
            while (at < wend) {
                const uint32_t s = (uint32_t)(at - pos);
                const uint32_t m = copies >> s << s;
                if (!m) { at = wend; break; }   // literals to the end of the window
                const int t = __ffs(m) - 1;
                const int32_t cq = pos + t;
                int32_t len = __shfl_sync(LZ_FULL, best, t), d = __shfl_sync(LZ_FULL, dist, t);
                const int32_t lt = __shfl_sync(LZ_FULL, lim, t);
                const uint32_t ht = __shfl_sync(LZ_FULL, hits, t);
                if (len == LZ_CAP && lt > LZ_CAP) {
                    const int2 e = lz_extend(in, end, prev, cq, lt, ht);
                    len = e.x; d = e.y;
                }
                if (cq > lit_start) emit(3, (uint32_t)lit_start, (uint32_t)(cq - lit_start));
                emit(1, (uint32_t)d, (uint32_t)len);
                at = cq + len;
                lit_start = at;
            }
            pos = at;
        }
        if (n > lit_start) emit(3, (uint32_t)lit_start, (uint32_t)(n - lit_start));

        // header, PredictionMode record, literal pool
        const uint64_t rec_end = 32ull + 20ull * n_cmds, total = rec_end + PM_RECORD_BYTES + (uint64_t)n;
        if (total <= cap) {
            uint32_t *const w = reinterpret_cast<uint32_t *>(blob);
            if (lane < 8)   // magic, version, n_cmds, n_predmodes, n_literal_bytes, window, 0, 0
                w[lane] = lane == 0 ? 0x4c435644u : lane == 2 ? n_cmds : lane == 4 ? (uint32_t)n : lane == 5 ? (uint32_t)p.window
                        : (lane == 1 || lane == 3) ? 1u : 0u;
            uint32_t *const pm = reinterpret_cast<uint32_t *>(blob + rec_end);
            const uint32_t *const src = reinterpret_cast<const uint32_t *>(p.pm);
            for (uint32_t k = lane; k < PM_RECORD_BYTES / 4; k += 32) pm[k] = __ldg(src + k);
            uint8_t *const pool = blob + rec_end + PM_RECORD_BYTES;   // 4-byte aligned
            for (int32_t k = lane; k < (n >> 2); k += 32) reinterpret_cast<uint32_t *>(pool)[k] = lz_word(in + 4 * (size_t)k, end);
            if (lane < (n & 3)) pool[(n & ~3) + lane] = in[(n & ~3) + lane];   // the last 1..3 bytes
        }
        if (lane == 0) { p.blob_len[v] = total; p.status[v] = total <= cap ? ST_OK : ST_NEED_OUTPUT; }
        __syncwarp();   // this stream's reads of the scratch are done before the next stream resets it
    }
}

void launch_lz77_cmds(const Lz77Params &p, cudaStream_t st) {
    const unsigned blocks = (p.n_warps + LZ_WARPS - 1) / LZ_WARPS;
    lz77_cmds_kernel<<<blocks, LZ_BLOCK_THREADS, 0, st>>>(p);
}

}  // namespace dv
