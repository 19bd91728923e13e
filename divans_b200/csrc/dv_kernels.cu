// dv_kernels.cu -- sm_90a kernels of the divANS batch engine around the stream decoder (dv2_kernels.cu): the framing/CRC
// pre-pass every decode runs first (frame, payload scan, demux), and the pack kernel of the recording decoders.
#include "dv_core.cuh"

namespace dv {

// ---------------------------------------------------------------------------------------------------------------
// framing pre-pass: frame kernel (header, record walk, trailer, CRC32C -- one warp per stream), payload scan, demux.
// ---------------------------------------------------------------------------------------------------------------
// frame kernel: one WARP per stream.  Lane 0 walks the 16-byte header and the mux record chain (mux.rs:384-444) to the
// EOF marker and checks the trailer magic; the warp checks the CRC32C of header..EOF marker (codec/decoder.rs:186-213).
__global__ void __launch_bounds__(128) frame_kernel(FrameParams p) {
    __shared__ uint32_t tab[4][256];   // slice-by-4 tables for the Castagnoli polynomial (reflected 0x82F63B78)
    __shared__ uint32_t x2n[32];       // x^(2^k) mod P
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) {
        uint32_t c = i;
        for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ CRC32C_POLY : (c >> 1);
        tab[0][i] = c;
    }
    if (threadIdx.x == 0) {
        uint32_t v = 0x40000000u;      // x^1
        x2n[0] = v;
        for (int k = 1; k < 32; k++) { v = gf_mul(v, v); x2n[k] = v; }
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) {
        uint32_t c = tab[0][i];
        for (int t = 1; t < 4; t++) { c = tab[0][c & 0xff] ^ (c >> 8); tab[t][i] = c; }
    }
    __syncthreads();
    const uint32_t sidx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (sidx >= p.n_streams) return;
    const uint8_t *in = p.in + p.in_off[sidx];
    const uint64_t n = p.in_len[sidx];
    int32_t st = ST_OK;
    uint32_t body_end = 0, pay0 = 0, pay1 = 0;
    if (lane == 0) {
        if (n < 16) st = ST_NEED_INPUT;
        else if (in[0] != 0xff || in[1] != 0xe5 || in[2] != 0x8c || in[3] != 0x9f) st = ST_FAIL;   // MAGIC_NUMBER, src/interface.rs:164
        else if (in[5] < 10 || in[5] >= 25) st = ST_FAIL;                                             // BadWindowSize, divans_decompressor.rs:47-50
        else {
            uint64_t pos = 16;
            for (;;) {
                if (pos >= n) { st = ST_NEED_INPUT; break; }
                uint32_t b = in[pos];
                if (b == 0xff) {
                    if (pos + 3 > n) { st = ST_NEED_INPUT; break; }
                    if (in[pos + 1] != 0xfe || in[pos + 2] != 0xff) { st = ST_FAIL; break; }
                    body_end = (uint32_t)pos;
                    break;
                }
                uint64_t len, hdr;
                if (b < 16) { if (pos + 3 > n) { st = ST_NEED_INPUT; break; } len = ((uint64_t)in[pos + 1] | ((uint64_t)in[pos + 2] << 8)) + 1; hdr = 3; }
                else { uint32_t k = b >> 4; if (k > 3) { st = ST_FAIL; break; } len = 1024ull << (k << 1); hdr = 1; }
                if (pos + hdr + len > n) { st = ST_NEED_INPUT; break; }
                if (b & 1) pay1 += (uint32_t)len; else pay0 += (uint32_t)len;
                pos += hdr + len;
            }
            if (st == ST_OK) {
                const uint64_t tr = (uint64_t)body_end + 3;
                if (tr + 8 > n) st = ST_NEED_INPUT;
                else if (in[tr + 4] != 'a' || in[tr + 5] != 'n' || in[tr + 6] != 's' || in[tr + 7] != '~') st = ST_FAIL;
            }
        }
    }
    st = __shfl_sync(FULL, st, 0);
    body_end = __shfl_sync(FULL, body_end, 0);
    if (st == ST_OK && !(p.flags & 3u)) {
        const uint32_t tr = body_end + 3;
        const uint32_t crc = warp_crc32c(tab, x2n, in, tr, lane);
        const uint32_t want = (uint32_t)in[tr] | ((uint32_t)in[tr + 1] << 8) | ((uint32_t)in[tr + 2] << 16) | ((uint32_t)in[tr + 3] << 24);
        if (crc != want) st = ST_FAIL;   // BadChecksum
    }
    if (lane == 0) {
        p.frame[4 * sidx + 0] = st == ST_OK ? body_end : 0;
        p.frame[4 * sidx + 1] = st == ST_OK ? pay0 : 0;
        p.frame[4 * sidx + 2] = st == ST_OK ? pay1 : 0;
        p.status[sidx] = st;
    }
}

// exclusive scan of the per-stream payload footprints -> frame[4i+3] = base of stream i's compacted payload (16-byte units)
// A stream whose compacted payload would not fit the payload buffer (`cap16` 16-byte units: aliased / overlapping input
// regions, or an underestimated in_total_bytes) is failed here instead of letting the demux kernel write past the end.
__global__ void __launch_bounds__(1024) payload_scan_kernel(uint32_t *frame, uint32_t n, int32_t *status, uint64_t cap16) {
    __shared__ uint32_t part[1024];
    const uint32_t t = threadIdx.x;
    const uint32_t per = (n + 1023) / 1024;
    const uint32_t lo = min(n, t * per), hi = min(n, lo + per);
    uint32_t sum = 0;
    for (uint32_t i = lo; i < hi; i++) sum += ((frame[4 * i + 1] + 15) >> 4) + ((frame[4 * i + 2] + 15) >> 4) + 1;
    part[t] = sum;
    __syncthreads();
    for (uint32_t o = 1; o < 1024; o <<= 1) {
        uint32_t v = t >= o ? part[t - o] : 0;
        __syncthreads();
        part[t] += v;
        __syncthreads();
    }
    uint32_t base = part[t] - sum;
    for (uint32_t i = lo; i < hi; i++) {
        const uint32_t need = ((frame[4 * i + 1] + 15) >> 4) + ((frame[4 * i + 2] + 15) >> 4) + 1;
        if ((uint64_t)base + need > cap16) {
            if (status[i] == ST_OK) status[i] = ST_FAIL;
            frame[4 * i + 1] = 0; frame[4 * i + 2] = 0; frame[4 * i + 3] = 0;
        } else frame[4 * i + 3] = base;
        base += need;
    }
}

// demux (mux.rs:384-444): one warp per stream copies the payload of every record to the stream's compact area:
// command-coder bytes at base, literal-coder bytes at base + align16(cmd bytes)
__global__ void __launch_bounds__(128) demux_kernel(FrameParams p, uint8_t *payload) {
    const uint32_t sidx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (sidx >= p.n_streams || p.status[sidx] != ST_OK) return;
    const uint8_t *in = p.in + p.in_off[sidx];
    const uint32_t body_end = p.frame[4 * sidx + 0];
    uint8_t *dst0 = payload + 16ull * p.frame[4 * sidx + 3];
    uint8_t *dst1 = dst0 + (((uint64_t)p.frame[4 * sidx + 1] + 15) & ~15ull);
    uint32_t pos = 16;
    while (pos < body_end) {
        uint32_t b = in[pos], len, hdr;
        if (b < 16) { len = ((uint32_t)in[pos + 1] | ((uint32_t)in[pos + 2] << 8)) + 1; hdr = 3; }
        else { len = 1024u << ((b >> 4) << 1); hdr = 1; }
        const uint8_t *src = in + pos + hdr;
        uint8_t *d = (b & 1) ? dst1 : dst0;
        // byte head to a 4-byte aligned destination, then words assembled from (possibly unaligned) source bytes
        uint32_t head = min(len, (uint32_t)((4 - ((uintptr_t)d & 3)) & 3));
        if (lane < head) d[lane] = src[lane];
        uint32_t nw = (len - head) >> 2;
        const uint8_t *s2 = src + head; uint32_t *d2 = reinterpret_cast<uint32_t *>(d + head);
        const uint32_t *sa = reinterpret_cast<const uint32_t *>((uintptr_t)s2 & ~(uintptr_t)3);
        const uint32_t sh = ((uint32_t)(uintptr_t)s2 & 3u) * 8u;
        for (uint32_t i = lane; i < nw; i += 32) d2[i] = __funnelshift_r(sa[i], sa[i + 1], sh);   // over-read <= 3 B stays inside the stream (EOF marker + trailer follow)
        uint32_t tail = (len - head) & 3;
        if (lane < tail) d[head + 4 * nw + lane] = src[head + 4 * nw + lane];
        if (b & 1) dst1 += len; else dst0 += len;
        pos += hdr + len;
    }
}

// pack kernel of the recording decoders (decode to command lists): one warp per stream turns what the decoder recorded into the
// stream's DVCL blob (include/divans_b200.h).  The decoder left the command records at byte 32 (a literal's `a` = the output
// position of its bytes) and prediction-mode record j at the region's end minus j + 1 records; counts[] says how many of each
// and how many literal bytes.  The warp puts the prediction-mode records in order behind the commands, gathers the literal
// bytes from the decoded output into the pool, rewrites each literal's `a` to its pool offset and writes the header.
__device__ __forceinline__ uint32_t ld_le32(const uint8_t *p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
__global__ void __launch_bounds__(128) pack_cmds_kernel(DecodeParams p, RecParams r) {
    const uint32_t sidx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (sidx >= p.n_streams) return;
    uint8_t *blob = r.blobs + r.blob_off[sidx];
    const uint64_t cap = r.blob_cap[sidx];
    const uint32_t *cnt = r.counts + 3 * (size_t)sidx;   // (zeros for a stream the decoder never started)
    const uint32_t nc = cnt[0], np = cnt[1], nl = cnt[2];
    const uint64_t cmd_end = 32ull + 20ull * nc, pm_bytes = (uint64_t)PM_RECORD_BYTES * np;
    const uint64_t need = cmd_end + pm_bytes + nl;
    const bool ok = p.status[sidx] == ST_OK;
    if (!ok || need > cap) {
        // a failed stream (blob_len 0) or a region too small for the blob (status 2, blob_len = the size it needs): the region
        // keeps no partial records
        const uint64_t lo_end = min(cap, cmd_end), hi_beg = cap - min(cap, pm_bytes);
        for (uint64_t i = 32 + lane; i < lo_end; i += 32) blob[i] = 0;
        for (uint64_t i = hi_beg + lane; i < cap; i += 32) blob[i] = 0;
        if (lane == 0) { r.blob_len[sidx] = ok ? need : 0; if (ok) p.status[sidx] = ST_NEED_OUTPUT; }
        return;
    }
    // prediction-mode records: reverse their order in place, then move them down behind the commands (by at least the literal
    // pool's size: every chunk is read before it is written)
    for (uint32_t j = 0; j < np / 2; j++) {
        uint8_t *x = blob + cap - (uint64_t)PM_RECORD_BYTES * (j + 1), *y = blob + cap - (uint64_t)PM_RECORD_BYTES * (np - j);
        for (uint32_t i = lane; i < PM_RECORD_BYTES; i += 32) { const uint8_t t = x[i]; x[i] = y[i]; y[i] = t; }
    }
    __syncwarp();
    const uint64_t src = cap - pm_bytes;
    if (src != cmd_end) {
        for (uint64_t i = 0; i < pm_bytes; i += 128) {
            uint8_t v[4];
#pragma unroll
            for (int k = 0; k < 4; k++) { const uint64_t x = i + lane + 32 * k; v[k] = x < pm_bytes ? blob[src + x] : (uint8_t)0; }
            __syncwarp();
#pragma unroll
            for (int k = 0; k < 4; k++) { const uint64_t x = i + lane + 32 * k; if (x < pm_bytes) blob[cmd_end + x] = v[k]; }
            __syncwarp();
        }
        for (uint64_t i = max(src, need) + lane; i < cap; i += 32) blob[i] = 0;   // where they were, past the blob
    }
    // literal pool: 32 command records at a time, pool offsets by a warp scan of the literal lengths
    uint8_t *pool = blob + cmd_end + pm_bytes;
    const uint8_t *out = p.out + p.out_off[sidx];
    uint32_t base = 0;
    for (uint32_t c0 = 0; c0 < nc; c0 += 32) {
        const uint32_t c = c0 + lane;
        uint8_t *rec = blob + 32 + 20ull * c;
        const bool lit = c < nc && ld_le32(rec) == 3u;
        const uint32_t pos = lit ? ld_le32(rec + 4) : 0u, len = lit ? ld_le32(rec + 8) : 0u;
        uint32_t incl = len;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(FULL, incl, o); if ((int)lane >= o) incl += t; }
        const uint32_t off = base + incl - len;
        if (lit) st_le32(rec + 4, off);
        for (uint32_t m = __ballot_sync(FULL, len != 0); m; m &= m - 1) {
            const int l = __ffs((int)m) - 1;
            const uint32_t lp = __shfl_sync(FULL, pos, l), ll = __shfl_sync(FULL, len, l), lo = __shfl_sync(FULL, off, l);
            for (uint32_t i = lane; i < ll; i += 32) pool[lo + i] = out[lp + i];
        }
        base += __shfl_sync(FULL, incl, 31);
    }
    if (lane < 8) {
        const uint32_t window = p.in[p.in_off[sidx] + 5];
        const uint32_t w = lane == 0 ? 0x4c435644u : lane == 1 ? 1u : lane == 2 ? nc : lane == 3 ? np : lane == 4 ? nl : lane == 5 ? window : 0u;
        st_le32(blob + 4 * lane, w);
    }
    if (lane == 0) r.blob_len[sidx] = need;
}
void launch_pack_cmds(const DecodeParams &p, const RecParams &r, cudaStream_t st) {
    pack_cmds_kernel<<<(p.n_streams + 3) / 4, 128, 0, st>>>(p, r);   // one warp per stream
}

void launch_frame(const FrameParams &p, uint8_t *payload, uint64_t payload_cap_bytes, cudaStream_t st) {
    uint32_t blocks = (p.n_streams + 3) / 4;   // one warp per stream
    frame_kernel<<<blocks, 128, 0, st>>>(p);
    payload_scan_kernel<<<1, 1024, 0, st>>>(p.frame, p.n_streams, p.status, payload_cap_bytes / 16);
    demux_kernel<<<(p.n_streams + 3) / 4, 128, 0, st>>>(p, payload);
}

}  // namespace dv
