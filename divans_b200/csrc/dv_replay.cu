// dv_replay.cu -- sm_90a kernel that realises DVCL command lists as raw bytes (the reference's `recode`, src/bin/divans.rs:1108,
// and DivansRecodeState, cmd_to_raw/mod.rs): divans_b200_replay_cmds_batch_host / _device.
//
// One warp per list; persistent warps pull list indices from the work counter, so any n runs in one launch.  The warp checks
// the header, then fetches the command records 32 at a time (lane k loads record pos + k) and applies them in order, the
// fields broadcast by shuffles:
//   literal     all lanes copy pool bytes to the output;
//   copy        replay_copy (dv_engine.cuh) with the warp as one 32-lane group: lane j writes the bytes i = j (mod 32), each
//               from out[pos - dist + (i mod dist)], a byte that existed before the copy started;
//   dictionary  dict_word (dv_engine.cuh) builds the transformed word in the warp's Cold::scratch on lane 0, the warp stores it.
// Commands are separated by a __syncwarp: a later copy may read what an earlier command wrote.  Once the output region is
// full the warp keeps walking the list without moving bytes, so out_len is exact and every refusal rule still applies.
#include "dv_engine.cuh"
#include "dv_kernels.h"

namespace dv {

constexpr int REPLAY_BLOCK_THREADS = 256;
constexpr int REPLAY_WARPS = REPLAY_BLOCK_THREADS / 32;   // (launch bounds: 4 blocks per SM, 64 registers, no spills)
constexpr size_t REPLAY_SMEM = (size_t)REPLAY_WARPS * SMEM_BYTES_PER_GROUP;   // one Cold per warp (cold_of_group)
constexpr uint64_t REPLAY_COPY_CHUNK = 1ull << 31;   // the longest copy one replay_copy call takes

__device__ __forceinline__ uint64_t replay_room(uint64_t pos, uint64_t cap, uint64_t len) { return pos >= cap ? 0 : min(len, cap - pos); }

// A copy of more than REPLAY_COPY_CHUNK bytes.  replay_copy's lanes step a 32-bit index by 32, which wraps for lengths near
// 2^32: it gets chunks of at most 2^31 bytes, each rebased at its own source once the output holds a period.  (Out of line:
// the common short copy keeps the kernel's registers.)
static __device__ __noinline__ void replay_long_copy(const G2 g, uint8_t *out, uint64_t at, uint32_t dist, uint64_t left) {
    while (left) {
        const uint32_t chunk = (uint32_t)min(left, REPLAY_COPY_CHUNK);
        if (at >= dist) replay_copy(g, out + (at - dist), dist, dist, chunk);
        else replay_copy(g, out, (uint32_t)at, dist, chunk);
        at += chunk; left -= chunk;
        __syncwarp();   // the next chunk reads the last period of this one
    }
}

__global__ void __launch_bounds__(REPLAY_BLOCK_THREADS, 4) replay_cmds_kernel(ReplayParams p) {
    const int lane = threadIdx.x & 31;
    G2 g;
    g.l16 = lane; g.shift = 0; g.gmask = FULL; g.store0 = lane == 0; g.nl = 32; g.grp = threadIdx.x >> 5; g.blend = false;
    const uint8_t *const scratch = cold_of_group(g)->scratch;
    for (;;) {
        uint32_t v = 0;
        if (lane == 0) v = atomicAdd(p.work_counter, 1u);
        v = __shfl_sync(FULL, v, 0);
        if (v >= p.n_lists) break;
        const uint8_t *const blob = p.blobs + p.blob_off[v];
        const uint64_t blen = p.blob_len[v], cap = p.out_cap[v];
        uint8_t *const out = p.out + p.out_off[v];
        uint64_t pos = 0;
        int st = ST_OK;
        // header: read only when the blob holds one, at a 4-byte aligned address (the records are read as u32)
        uint32_t hw = 0;
        const bool hdr_ok = ((uintptr_t)blob & 3u) == 0 && blen >= 32;
        if (hdr_ok && lane < 8) hw = reinterpret_cast<const uint32_t *>(blob)[lane];
        const uint32_t magic = __shfl_sync(FULL, hw, 0), version = __shfl_sync(FULL, hw, 1), n_cmds = __shfl_sync(FULL, hw, 2);
        const uint32_t n_pms = __shfl_sync(FULL, hw, 3), n_lits = __shfl_sync(FULL, hw, 4), hwin = __shfl_sync(FULL, hw, 5);
        const uint64_t lit_base = 32ull + 20ull * n_cmds + (uint64_t)PM_RECORD_BYTES * n_pms;
        if (!hdr_ok || magic != 0x4c435644u || version != 1u || lit_base + n_lits > blen) st = ST_FAIL;
        const uint32_t win = p.window != 0 ? (uint32_t)p.window : min(max(hwin, 10u), 24u);
        const uint32_t ring = 1u << win;
        const uint32_t *const recs = reinterpret_cast<const uint32_t *>(blob + 32);
        const uint8_t *const lits = blob + lit_base;
        for (uint32_t base = 0; st == ST_OK && base < n_cmds; base += 32) {
            uint32_t r0 = 0, r1 = 0, r2 = 0, r3 = 0, r4 = 0;
            if (base + lane < n_cmds) {
                const uint32_t *r = recs + 5ull * (base + lane);
                r0 = r[0]; r1 = r[1]; r2 = r[2]; r3 = r[3]; r4 = r[4];
            }
            const uint32_t cnt = min(32u, n_cmds - base);
            for (uint32_t k = 0; k < cnt; k++) {
                const uint32_t type = __shfl_sync(FULL, r0, k), a = __shfl_sync(FULL, r1, k), b = __shfl_sync(FULL, r2, k);
                const uint32_t c = __shfl_sync(FULL, r3, k), d = __shfl_sync(FULL, r4, k);
                if (type == 3) {   // literal: pool bytes [a, a + b)
                    if ((uint64_t)a + b > n_lits) { st = ST_FAIL; break; }
                    const uint64_t take = replay_room(pos, cap, b);
                    for (uint64_t i = (uint64_t)lane; i < take; i += 32) out[pos + i] = lits[(uint64_t)a + i];
                    pos += b;
                } else if (type == 1) {   // copy: b bytes at distance a
                    if (a == 0 || a >= ring) { st = ST_FAIL; break; }
                    const uint64_t take = replay_room(pos, cap, b);
                    // replay_copy takes 32-bit positions: past the first period, rebase the output at the copy's source
                    if (take > REPLAY_COPY_CHUNK) replay_long_copy(g, out, pos, a, take);
                    else if (take) {
                        if (pos >= a) replay_copy(g, out + (pos - a), a, a, (uint32_t)take);
                        else replay_copy(g, out, (uint32_t)pos, a, (uint32_t)take);
                    }
                    pos += b;
                } else if (type == 2) {   // dictionary word a of size b under transform c; d != 0: the length it must have
                    int n = 0;
                    if (lane == 0) n = dict_word(g, p.tables, b, a, c);
                    n = __shfl_sync(FULL, n, 0);
                    __syncwarp();   // lane 0's scratch stores are visible to the warp
                    if (n < 0 || (d != 0 && (uint32_t)n != d)) { st = ST_FAIL; break; }
                    const uint64_t take = replay_room(pos, cap, (uint64_t)n);
                    for (uint32_t i = (uint32_t)lane; i < take; i += 32) out[pos + i] = scratch[i];
                    pos += (uint64_t)n;
                } else if (type < 1 || type > 7) { st = ST_FAIL; break; }
                // (4..7: block switches and PredictionMode commands append nothing)
                __syncwarp();   // what this command wrote is visible to the next one's reads (and scratch is free again)
            }
        }
        if (st == ST_OK && pos > cap) st = ST_NEED_OUTPUT;
        if (lane == 0) { p.out_len[v] = pos; p.status[v] = st; }
    }
}

void launch_replay_cmds(const ReplayParams &p, int sm_count, cudaStream_t st) {
    static const int per_sm = [] {
        int nb = stream_kernel_blocks_per_sm(replay_cmds_kernel, REPLAY_BLOCK_THREADS, REPLAY_SMEM);
        return nb < 1 ? 1 : nb;
    }();
    const uint64_t want = ((uint64_t)p.n_lists + REPLAY_WARPS - 1) / REPLAY_WARPS, most = (uint64_t)sm_count * (uint64_t)per_sm;
    replay_cmds_kernel<<<(unsigned)(want < most ? want : most), REPLAY_BLOCK_THREADS, REPLAY_SMEM, st>>>(p);
}

}  // namespace dv
