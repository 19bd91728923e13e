// dv_capi.cu -- the C ABI of libdivans_b200.so: batch engine context + the reference's FFI surface as a drop-in.
//
// Host side only marshals: offsets/lengths tables, H2D/D2H copies, kernel launches.  All model/entropy work runs in
// the sm_90a kernels (dv2_kernels.cu, dv_kernels.cu, dv_encode.cu); there is no CPU decode path in this library.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <new>

#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/divans_b200.h"
#include "dv_kernels.h"
#include "dv_lz77.h"

#ifndef DV_TABLES_PATH
#error "DV_TABLES_PATH must point at brotli_tables.bin"
#endif
__asm__(".section .rodata\n"
        ".global dv_tables_blob\n"
        ".balign 16\n"
        "dv_tables_blob:\n"
        ".incbin \"" DV_TABLES_PATH "\"\n"
        ".previous\n");
extern "C" const uint8_t dv_tables_blob[];

using namespace dv;

// HBM copies of a host batch (grow-only): the input blob, the output regions, and the descriptor arrays
// in_off,in_len,out_off,out_cap,out_len (+status; decode_cmds: + blob_off,blob_cap,blob_len; encode_auto: + chosen,cost)
struct HostBufs {
    uint8_t *d_in = nullptr; size_t d_in_cap = 0;
    uint8_t *d_out = nullptr; size_t d_out_cap = 0;
    uint64_t *d_meta = nullptr; size_t d_meta_cap = 0;
};
static void free_host_bufs(HostBufs &b) { cudaFree(b.d_in); cudaFree(b.d_out); cudaFree(b.d_meta); }

struct divans_b200_ctx {
    int device = 0;
    int lanes_per_stream = 8;
    int sm_count = 0;
    uint32_t max_resident = 0;       // slots in the arena
    cudaStream_t stream = nullptr;
    uint8_t *d_arena = nullptr; size_t arena_slots = 0;   // 16 MiB aligned view of d_arena_raw
    uint8_t *d_arena_raw = nullptr;
    bool auto_lanes = false;         // lanes_per_stream 0: 16 lanes, or 8 where their residency holds the batch in fewer passes
    int last_lanes = 0;              // layout the most recent decode call used
    uint32_t cap16 = 0, cap8 = 0;    // resident streams of the two v2 layouts
    uint8_t *d_tables = nullptr;
    uint32_t *d_counter = nullptr;
    uint64_t *d_nibbles = nullptr;
    // grow-only scratch
    uint32_t *d_frame = nullptr; size_t frame_cap = 0;
    uint8_t *d_payload = nullptr; size_t payload_cap = 0;
    HostBufs host;                                         // the blocking host calls (decode and encode)
    uint8_t *d_blobs = nullptr; size_t d_blobs_cap = 0;   // decode_cmds_batch_host: the DVCL blob regions
    uint32_t *d_rec_counts = nullptr; size_t rec_counts_cap = 0;   // decode_cmds: per stream [3] what the recording decoder counted
    // pipelined host API (decode_batch_host_async): two batches in flight, copies on their own streams
    struct Lane {
        HostBufs bufs;
        cudaEvent_t e_in = nullptr, e_k = nullptr, e_out = nullptr;
        uint8_t *h_res = nullptr; size_t h_res_cap = 0;      // pinned staging of out_len[] + status[] (the caller's arrays may be pageable)
        uint64_t *u_out_len = nullptr; int32_t *u_status = nullptr; size_t n = 0;
        bool pending = false;
    } lane[2];
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
    uint64_t async_seq = 0;
    uint32_t *d_sf = nullptr; size_t sf_cap = 0;               // encoder: symbol logs
    uint8_t *d_replay = nullptr; size_t replay_cap = 0;
    uint32_t *d_enc_scratch = nullptr; size_t enc_scratch_cap = 0;
    uint8_t *d_pm_internal = nullptr; std::vector<uint8_t> h_pm;
    uint64_t *d_rcp15 = nullptr;
    // literal model selection (encode_auto_*): the candidates' PredictionMode records, the cost table, per (stream, candidate)
    // scratch: offsets, lengths, record index, status and cost
    uint8_t *d_pm_records = nullptr; uint32_t *d_cost_tab = nullptr;
    uint64_t *d_auto = nullptr; size_t auto_cap = 0;
    // per-context mixing values (encode_mixmap_*): per-stream scratch (per-entry winners, mixed pass, record index), the k uniform
    // and n mixed records, the binned cost pass's per-slot bins, and the host calls' staging of the mixing / bins outputs
    uint64_t *d_mix = nullptr; size_t mix_cap = 0;
    uint8_t *d_mix_records = nullptr; size_t mix_records_cap = 0;
    uint64_t *d_slot_bins = nullptr; size_t slot_bins_cap = 0;
    uint64_t *d_mix_out = nullptr; size_t mix_out_cap = 0;
    // LZ77 command generator (lz77_cmds_batch_device): per-warp head table + prev array, and the PredictionMode record it copies
    // (lz_scratch_asked: the request the allocation was made for, which free memory may have cut down to lz_scratch_words)
    int32_t *d_lz_scratch = nullptr; size_t lz_scratch_words = 0, lz_scratch_asked = 0;
    uint8_t *d_lz_pm = nullptr;
    bool main_end_is_evm1 = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, evm = nullptr, evm1 = nullptr;   // ev0 | frame kernel | evm | decode kernel | ev1
    cudaEvent_t ev_busy = nullptr; bool busy_recorded = false;                 // end of the most recent launch set on any stream
    float last_kernel_ms = 0.f;
    uint64_t launches = 0;
    std::string err;
    std::mutex mu;
};

static bool ck(divans_b200_ctx *c, cudaError_t e, const char *what) {
    if (e == cudaSuccess) return true;
    // a failed allocation is reported here; clear it, or the launch check of the next call on this context reports it again
    if (e == cudaErrorMemoryAllocation) cudaGetLastError();
    char buf[512];
    snprintf(buf, sizeof buf, "divans_b200: %s failed: %s", what, cudaGetErrorString(e));
    if (c) c->err = buf;
    fprintf(stderr, "%s\n", buf);
    return false;
}
#define CK(call) do { if (!ck(ctx, (call), #call)) return DIVANS_FAILURE; } while (0)

template <typename T>
static bool grow(divans_b200_ctx *ctx, T **p, size_t *cap, size_t need) {
    if (need <= *cap) return true;
    if (*p) cudaFree(*p);
    *p = nullptr; *cap = 0;
    size_t want = need + need / 4 + 256;
    if (!ck(ctx, cudaMalloc((void **)p, want * sizeof(T)), "cudaMalloc(scratch)")) return false;
    *cap = want;
    return true;
}

extern "C" divans_b200_ctx *divans_b200_create(int device, uint32_t max_resident, uint32_t lanes_per_stream) {
    divans_b200_ctx *ctx = new (std::nothrow) divans_b200_ctx();
    if (!ctx) return nullptr;
    ctx->device = device;
    // 8: v2 engine, four streams per warp; anything else: v2 engine, two streams per warp (0: chosen per batch, see decode)
    ctx->auto_lanes = lanes_per_stream == 0;
    ctx->lanes_per_stream = lanes_per_stream == 8 ? 8 : 16;
    cudaDeviceProp prop;
    if (!ck(ctx, cudaSetDevice(device), "cudaSetDevice") || !ck(ctx, cudaGetDeviceProperties(&prop, device), "cudaGetDeviceProperties")) {
        fprintf(stderr, "divans_b200: no usable CUDA device %d -- this library has no CPU path\n", device);
        delete ctx; return nullptr;
    }
    if (prop.major != 9 || prop.minor != 0) {   // sm_90a code runs on compute capability 9.0 only
        fprintf(stderr, "divans_b200: device %d is sm_%d%d; the kernels are built for sm_90a only\n", device, prop.major, prop.minor);
        delete ctx; return nullptr;
    }
    ctx->sm_count = prop.multiProcessorCount;
    bool ok = ck(ctx, cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking), "cudaStreamCreate") &&
              ck(ctx, cudaEventCreate(&ctx->ev0), "cudaEventCreate") && ck(ctx, cudaEventCreate(&ctx->ev1), "cudaEventCreate") &&
              ck(ctx, cudaEventCreate(&ctx->evm), "cudaEventCreate") && ck(ctx, cudaEventCreate(&ctx->evm1), "cudaEventCreate") &&
              ck(ctx, cudaEventCreateWithFlags(&ctx->ev_busy, cudaEventDisableTiming), "cudaEventCreate") &&
              ck(ctx, cudaMalloc((void **)&ctx->d_tables, TB_TOTAL), "cudaMalloc(tables)") &&
              ck(ctx, cudaMemcpy(ctx->d_tables, dv_tables_blob, TB_TOTAL, cudaMemcpyHostToDevice), "cudaMemcpy(tables)") &&
              ck(ctx, cudaMalloc((void **)&ctx->d_counter, 64), "cudaMalloc(counter)") &&
              ck(ctx, cudaMalloc((void **)&ctx->d_nibbles, 64), "cudaMalloc(nibbles)") &&
              ck(ctx, cudaMemset(ctx->d_nibbles, 0, 64), "cudaMemset");
    if (!ok) { delete ctx; return nullptr; }
    int per_sm = decode_max_blocks_per_sm_v2(ctx->lanes_per_stream);
    if (per_sm < 1) per_sm = 1;
    const uint32_t groups_per_block = (uint32_t)decode_groups_per_block_v2(ctx->lanes_per_stream);
    uint32_t auto_res = (uint32_t)ctx->sm_count * (uint32_t)per_sm * groups_per_block;
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    // Leave room for batch buffers.  85 %: on an 80 GB H100 the full 16-lane residency (132 SMs x 32 streams, 66 GiB of slots)
    // must fit, or a 4096-stream batch would leave a second wave behind.
    uint32_t mem_cap = (uint32_t)((free_b * 17 / 20) / SLOT_STRIDE);
    if (auto_res > mem_cap) auto_res = mem_cap;
    ctx->max_resident = max_resident ? (max_resident < auto_res ? max_resident : auto_res) : auto_res;
    if (ctx->max_resident < groups_per_block) ctx->max_resident = groups_per_block;
    auto cap = [&](int lanes) {
        uint32_t c = (uint32_t)ctx->sm_count * (uint32_t)std::max(1, decode_max_blocks_per_sm_v2(lanes)) * (uint32_t)decode_groups_per_block_v2(lanes);
        if (c > mem_cap) c = mem_cap;
        if (max_resident && c > max_resident) c = max_resident;
        return std::max(c, (uint32_t)decode_groups_per_block_v2(lanes));
    };
    ctx->cap16 = cap(16); ctx->cap8 = cap(8);
    return ctx;
}

extern "C" void divans_b200_destroy(divans_b200_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    for (int t = 0; t < 2; t++) divans_b200_decode_batch_host_wait(ctx, t);   // in-flight pipelined batches still write caller memory
    cudaStreamSynchronize(ctx->stream);
    if (ctx->s_h2d) cudaStreamSynchronize(ctx->s_h2d);
    if (ctx->s_d2h) cudaStreamSynchronize(ctx->s_d2h);
    cudaFree(ctx->d_arena_raw); cudaFree(ctx->d_tables); cudaFree(ctx->d_counter); cudaFree(ctx->d_nibbles);
    cudaFree(ctx->d_frame); cudaFree(ctx->d_payload); free_host_bufs(ctx->host);
    cudaFree(ctx->d_blobs); cudaFree(ctx->d_rec_counts);
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    if (ctx->evm) cudaEventDestroy(ctx->evm);
    if (ctx->evm1) cudaEventDestroy(ctx->evm1);
    if (ctx->ev_busy) cudaEventDestroy(ctx->ev_busy);
    cudaFree(ctx->d_sf); cudaFree(ctx->d_replay); cudaFree(ctx->d_enc_scratch); cudaFree(ctx->d_pm_internal); cudaFree(ctx->d_rcp15);
    cudaFree(ctx->d_pm_records); cudaFree(ctx->d_cost_tab); cudaFree(ctx->d_auto);
    cudaFree(ctx->d_mix); cudaFree(ctx->d_mix_records); cudaFree(ctx->d_slot_bins); cudaFree(ctx->d_mix_out);
    cudaFree(ctx->d_lz_scratch); cudaFree(ctx->d_lz_pm);
    for (auto &ln : ctx->lane) {
        free_host_bufs(ln.bufs);
        if (ln.h_res) cudaFreeHost(ln.h_res);
        if (ln.e_in) cudaEventDestroy(ln.e_in);
        if (ln.e_k) cudaEventDestroy(ln.e_k);
        if (ln.e_out) cudaEventDestroy(ln.e_out);
    }
    if (ctx->s_h2d) cudaStreamDestroy(ctx->s_h2d);
    if (ctx->s_d2h) cudaStreamDestroy(ctx->s_d2h);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}
// bumped whenever a decode kernel changes: bench.py quotes a stored DRAM-traffic capture (profiles/traffic.json) only for the version it measured
#define DV_KERNEL_VERSION "r2.20-lean-literal-loop"
extern "C" const char *divans_b200_kernel_version(void) { return DV_KERNEL_VERSION; }
extern "C" const char *divans_b200_last_error(divans_b200_ctx *ctx) { return ctx ? ctx->err.c_str() : "null context"; }
extern "C" int divans_b200_last_lanes(divans_b200_ctx *ctx) { return ctx ? ctx->last_lanes : 0; }
extern "C" uint64_t divans_b200_launch_count(divans_b200_ctx *ctx) { return ctx ? ctx->launches : 0; }
extern "C" float divans_b200_last_kernel_ms(divans_b200_ctx *ctx) {
    if (!ctx) return 0.f;
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1) == cudaSuccess) ctx->last_kernel_ms = ms;
    return ctx->last_kernel_ms;
}
extern "C" float divans_b200_last_main_kernel_ms(divans_b200_ctx *ctx) {
    if (!ctx) return 0.f;
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ctx->evm, ctx->main_end_is_evm1 ? ctx->evm1 : ctx->ev1) != cudaSuccess) return -1.f;
    return ms;
}
extern "C" DivansResult divans_b200_synchronize(divans_b200_ctx *ctx) {
    if (!ctx) return DIVANS_FAILURE;
    CK(cudaStreamSynchronize(ctx->stream));
    return DIVANS_SUCCESS;
}
extern "C" DivansResult divans_b200_debug_slot_header(divans_b200_ctx *ctx, uint32_t slot, uint32_t out[4]) {
    if (!ctx || !out) return DIVANS_FAILURE;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (slot >= ctx->arena_slots) { ctx->err = "slot index beyond the arena"; return DIVANS_FAILURE; }
    CK(cudaSetDevice(ctx->device));
    if (ctx->busy_recorded) CK(cudaEventSynchronize(ctx->ev_busy));   // the last launch set of this context, on whatever stream
    CK(cudaMemcpy(out, ctx->d_arena + (size_t)slot * SLOT_STRIDE + OFF_HDR, 16, cudaMemcpyDeviceToHost));
    return DIVANS_SUCCESS;
}

static DivansResult ensure_arena(divans_b200_ctx *ctx, size_t slots) {
    if (slots <= ctx->arena_slots) return DIVANS_SUCCESS;
    if (ctx->d_arena_raw) { cudaFree(ctx->d_arena_raw); ctx->d_arena_raw = ctx->d_arena = nullptr; ctx->arena_slots = 0; }
    CK(cudaMalloc((void **)&ctx->d_arena_raw, (slots + 1) * SLOT_STRIDE));
    ctx->d_arena = reinterpret_cast<uint8_t *>(((uintptr_t)ctx->d_arena_raw + SLOT_STRIDE - 1) & ~(uintptr_t)(SLOT_STRIDE - 1));   // slots are 16 MiB aligned (dv_common.cuh)
    // the v2 engine reads literal priors it has never written (tag 0 = never valid) and keeps a header per slot: zero it all once
    CK(cudaMemset(ctx->d_arena, 0, slots * SLOT_STRIDE));
    CK(cudaDeviceSynchronize());   // the memset runs on the legacy stream, the kernels on non-blocking ones: finish it before any launch
    ctx->arena_slots = slots;
    return DIVANS_SUCCESS;
}

// One context = one set of scratch buffers (work counter, frame table, compacted payload, arena slots, timing events):
// launches of different calls must not overlap on the GPU.  Calls are serialised on the host by ctx->mu and on the device
// by `ev_busy`: a launch set on any stream first waits for the previous call's last kernel.
// `rec` (decode to command lists): the recording decoder on 16 lanes per stream, then the pack kernel that finishes the blobs.
static DivansResult decode_device_nolock(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                         const uint64_t *d_in_len, uint8_t *d_out, const uint64_t *d_out_off,
                                         const uint64_t *d_out_cap, uint64_t *d_out_len, int32_t *d_status,
                                         uint64_t in_total_bytes, uint32_t flags, void *cuda_stream, const RecParams *rec = nullptr) {
    if (n > 0xffffffffull) { ctx->err = "too many streams"; return DIVANS_FAILURE; }
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
    if (ctx->busy_recorded) CK(cudaStreamWaitEvent(st, ctx->ev_busy, 0));
    int lanes = ctx->lanes_per_stream;
    const bool blend = (flags & DIVANS_B200_FLAG_CDF_BLEND) != 0;   // BlendCDF16 streams: the decoder's blend model
    // 16 lanes per stream unless 8 hold the batch in fewer passes.  At equal residency 8 lanes is the slower layout (half the
    // warps per scheduler); it only pays where registers, not slot memory, cap residency: there it keeps twice the streams in
    // flight.  On an 80 GB H100 both layouts are capped by slot memory (cap8 ~ cap16), so 16 lanes run every batch size.
    if (ctx->auto_lanes) {
        const uint64_t passes16 = (n + ctx->cap16 - 1) / ctx->cap16, passes8 = (n + ctx->cap8 - 1) / ctx->cap8;
        lanes = passes8 < passes16 ? 8 : 16;
    }
    if (rec || blend) lanes = 16;   // the recording decoder and the blend model have the 16-lane layout only
    uint32_t gpb = (uint32_t)decode_groups_per_block_v2(lanes), cap = lanes == 16 ? ctx->cap16 : ctx->cap8;
    if (blend) { gpb = DECODE_BLOCK_THREADS / 16; cap = std::max(cap / gpb * gpb, gpb); }   // whole blocks of the blend kernels
    ctx->last_lanes = lanes;
    uint32_t resident = (uint32_t)(n < cap ? n : cap);
    uint32_t blocks = (resident + gpb - 1) / gpb;
    if (ensure_arena(ctx, (size_t)blocks * gpb) != DIVANS_SUCCESS) return DIVANS_FAILURE;
    if (!grow(ctx, &ctx->d_frame, &ctx->frame_cap, 4 * n)) return DIVANS_FAILURE;
    if (!grow(ctx, &ctx->d_payload, &ctx->payload_cap, (size_t)in_total_bytes + 48 * n + 64)) return DIVANS_FAILURE;
    CK(cudaMemsetAsync(ctx->d_counter, 0, 4, st));
    RecParams rp;
    if (rec) {
        if (!grow(ctx, &ctx->d_rec_counts, &ctx->rec_counts_cap, 3 * n)) return DIVANS_FAILURE;
        rp = *rec; rp.counts = ctx->d_rec_counts;
        CK(cudaMemsetAsync(rp.counts, 0, 12 * n, st));   // (the pack kernel reads zeros for streams the decoder never started)
    }
    FrameParams fp;
    fp.in = d_in; fp.in_off = d_in_off; fp.in_len = d_in_len; fp.frame = ctx->d_frame; fp.status = d_status;
    fp.n_streams = (uint32_t)n; fp.flags = flags;
    DecodeParams dp;
    dp.in = d_in; dp.in_off = d_in_off; dp.in_len = d_in_len; dp.out = d_out; dp.out_off = d_out_off; dp.out_cap = d_out_cap;
    dp.out_len = d_out_len; dp.status = d_status; dp.frame = ctx->d_frame; dp.payload = ctx->d_payload; dp.n_streams = (uint32_t)n;
    dp.work_counter = ctx->d_counter; dp.arena = ctx->d_arena; dp.tables = ctx->d_tables; dp.nibble_counts = ctx->d_nibbles;
    dp.model_rev = (flags & DIVANS_B200_FLAG_MODEL_WASM_2018) ? 1u : 0u;
    static const bool dbg = getenv("DIVANS_B200_DEBUG") != nullptr;
    static const bool skip_decode = getenv("DIVANS_B200_SKIP_DECODE") != nullptr;
    CK(cudaEventRecord(ctx->ev0, st));
    launch_frame(fp, ctx->d_payload, (uint64_t)ctx->payload_cap, st);
    if (dbg) { CK(cudaStreamSynchronize(st)); fprintf(stderr, "divans_b200[debug]: frame kernel ok (n=%zu)\n", n); }
    CK(cudaEventRecord(ctx->evm, st));
    if (rec) {
        launch_decode_v2_rec(blend, dp, rp, blocks, st);
        CK(cudaEventRecord(ctx->evm1, st));
        launch_pack_cmds(dp, rp, st);
    } else if (!skip_decode) launch_decode_v2(lanes, blend, dp, blocks, st);
    if (dbg) { CK(cudaStreamSynchronize(st)); fprintf(stderr, "divans_b200[debug]: decode kernel ok (blocks=%u, lps=%d)\n", blocks, ctx->lanes_per_stream); }
    CK(cudaEventRecord(ctx->ev1, st));
    CK(cudaEventRecord(ctx->ev_busy, st)); ctx->busy_recorded = true;
    ctx->main_end_is_evm1 = rec != nullptr;
    ctx->launches += rec ? 5 : skip_decode ? 3 : 4;
    CK(cudaGetLastError());
    return DIVANS_SUCCESS;
}
extern "C" DivansResult divans_b200_decode_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                        const uint64_t *d_in_len, uint8_t *d_out, const uint64_t *d_out_off,
                                                        const uint64_t *d_out_cap, uint64_t *d_out_len, int32_t *d_status,
                                                        uint64_t in_total_bytes, uint32_t flags, void *cuda_stream) {
    if (!ctx) return DIVANS_FAILURE;
    if (n == 0) return DIVANS_SUCCESS;
    std::lock_guard<std::mutex> lk(ctx->mu);
    return decode_device_nolock(ctx, n, d_in, d_in_off, d_in_len, d_out, d_out_off, d_out_cap, d_out_len, d_status, in_total_bytes, flags, cuda_stream);
}

// ---- host-buffer decode ----
// the blob regions of divans_b200_decode_cmds_batch_host
struct HostBlobs {
    uint8_t *blobs; const uint64_t *off, *cap; uint64_t *len;
};

// [lo, hi): the span of the regions off[i] .. +cap[i] (n > 0)
static void regions_span(size_t n, const uint64_t *off, const uint64_t *cap, uint64_t &lo, uint64_t &hi) {
    lo = ~0ull; hi = 0;
    for (size_t i = 0; i < n; i++) { lo = std::min(lo, off[i]); hi = std::max(hi, off[i] + cap[i]); }
}

// Stage a host batch into `b`: the input and the descriptor arrays in_off | in_len | out_off | out_cap (| blob_off | blob_cap
// at 6n, 7n) are copied on `h2d`; then, on `st` (ordered after them by `e_in` when the two streams differ), the output (and
// blob) regions are zeroed.  The regions are copied back whole, so what they hold past the lengths is zeros, not an earlier
// batch.  Input regions may alias (the same stream decoded n times): `in_total` bounds the decoder's payload by the larger
// of their sum and their extent.
static DivansResult stage_decode(divans_b200_ctx *ctx, HostBufs &b, size_t n, const uint8_t *in, const uint64_t *in_off,
                                 const uint64_t *in_len, const uint64_t *out_off, const uint64_t *out_cap, const HostBlobs *bl,
                                 cudaStream_t h2d, cudaEvent_t e_in, cudaStream_t st, uint64_t &in_total) {
    uint64_t in_end = 0, in_sum = 0, out_lo, out_hi, blob_lo = 0, blob_hi = 0;
    for (size_t i = 0; i < n; i++) { in_end = std::max(in_end, in_off[i] + in_len[i]); in_sum += in_len[i]; }
    regions_span(n, out_off, out_cap, out_lo, out_hi);
    if (bl) regions_span(n, bl->off, bl->cap, blob_lo, blob_hi);
    // (re)allocation synchronises the device: with the pipelined call, only while it warms up
    if (!grow(ctx, &b.d_in, &b.d_in_cap, (size_t)in_end + 64)) return DIVANS_FAILURE;
    if (!grow(ctx, &b.d_out, &b.d_out_cap, (size_t)out_hi + 64)) return DIVANS_FAILURE;
    if (!grow(ctx, &b.d_meta, &b.d_meta_cap, n * (bl ? 9 : 6))) return DIVANS_FAILURE;
    if (bl && !grow(ctx, &ctx->d_blobs, &ctx->d_blobs_cap, (size_t)blob_hi + 64)) return DIVANS_FAILURE;
    uint64_t *m = b.d_meta;
    CK(cudaMemcpyAsync(b.d_in, in, in_end, cudaMemcpyHostToDevice, h2d));
    CK(cudaMemcpyAsync(m, in_off, n * 8, cudaMemcpyHostToDevice, h2d));
    CK(cudaMemcpyAsync(m + n, in_len, n * 8, cudaMemcpyHostToDevice, h2d));
    CK(cudaMemcpyAsync(m + 2 * n, out_off, n * 8, cudaMemcpyHostToDevice, h2d));
    CK(cudaMemcpyAsync(m + 3 * n, out_cap, n * 8, cudaMemcpyHostToDevice, h2d));
    if (bl) {
        CK(cudaMemcpyAsync(m + 6 * n, bl->off, n * 8, cudaMemcpyHostToDevice, h2d));
        CK(cudaMemcpyAsync(m + 7 * n, bl->cap, n * 8, cudaMemcpyHostToDevice, h2d));
    }
    if (h2d != st) {
        CK(cudaEventRecord(e_in, h2d));
        CK(cudaStreamWaitEvent(st, e_in, 0));
    }
    if (out_hi > out_lo) CK(cudaMemsetAsync(b.d_out + out_lo, 0, out_hi - out_lo, st));
    if (blob_hi > blob_lo) CK(cudaMemsetAsync(ctx->d_blobs + blob_lo, 0, blob_hi - blob_lo, st));
    in_total = std::max(in_sum, in_end);
    return DIVANS_SUCCESS;
}

// D2H of whole regions src[off[i] .. +cap[i]) to dst, one transfer per run of exactly adjacent regions: nothing outside them is written
static DivansResult copy_regions_back(divans_b200_ctx *ctx, size_t n, uint8_t *dst, const uint8_t *src, const uint64_t *off,
                                      const uint64_t *cap, cudaStream_t st) {
    for (size_t i = 0; i < n;) {
        const uint64_t lo = off[i]; uint64_t hi = lo + cap[i];
        size_t j = i + 1;
        while (j < n && off[j] == hi) { hi += cap[j]; j++; }
        if (hi > lo) CK(cudaMemcpyAsync(dst + lo, src + lo, hi - lo, cudaMemcpyDeviceToHost, st));
        i = j;
    }
    return DIVANS_SUCCESS;
}

// divans_b200_decode_batch_host, and with `bl` divans_b200_decode_cmds_batch_host: one synchronisation, at the end
static DivansResult decode_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off, const uint64_t *in_len,
                                uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap, uint64_t *out_len, int32_t *status,
                                uint32_t flags, const HostBlobs *bl) {
    if (!ctx) return DIVANS_FAILURE;
    if (n == 0) return DIVANS_SUCCESS;
    std::lock_guard<std::mutex> lk(ctx->mu);
    CK(cudaSetDevice(ctx->device));
    HostBufs &b = ctx->host;
    cudaStream_t st = ctx->stream;
    uint64_t in_total;
    if (stage_decode(ctx, b, n, in, in_off, in_len, out_off, out_cap, bl, st, nullptr, st, in_total) != DIVANS_SUCCESS) return DIVANS_FAILURE;
    uint64_t *m = b.d_meta;
    int32_t *d_status = reinterpret_cast<int32_t *>(m + 5 * n);
    RecParams rp;
    if (bl) { rp.blobs = ctx->d_blobs; rp.blob_off = m + 6 * n; rp.blob_cap = m + 7 * n; rp.blob_len = m + 8 * n; rp.counts = nullptr; }
    DivansResult r = decode_device_nolock(ctx, n, b.d_in, m, m + n, b.d_out, m + 2 * n, m + 3 * n, m + 4 * n, d_status, in_total, flags,
                                          st, bl ? &rp : nullptr);
    if (r != DIVANS_SUCCESS) return r;
    CK(cudaMemcpyAsync(out_len, m + 4 * n, n * 8, cudaMemcpyDeviceToHost, st));
    if (bl) CK(cudaMemcpyAsync(bl->len, m + 8 * n, n * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(status, d_status, n * 4, cudaMemcpyDeviceToHost, st));
    if (copy_regions_back(ctx, n, out, b.d_out, out_off, out_cap, st) != DIVANS_SUCCESS) return DIVANS_FAILURE;
    if (bl && copy_regions_back(ctx, n, bl->blobs, ctx->d_blobs, bl->off, bl->cap, st) != DIVANS_SUCCESS) return DIVANS_FAILURE;
    CK(cudaStreamSynchronize(st));
    return DIVANS_SUCCESS;
}
extern "C" DivansResult divans_b200_decode_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                                      const uint64_t *in_len, uint8_t *out, const uint64_t *out_off,
                                                      const uint64_t *out_cap, uint64_t *out_len, int32_t *status, uint32_t flags) {
    return decode_host(ctx, n, in, in_off, in_len, out, out_off, out_cap, out_len, status, flags, nullptr);
}

// ---- decode to command lists ----
extern "C" DivansResult divans_b200_decode_cmds_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                             const uint64_t *d_in_len, uint8_t *d_out, const uint64_t *d_out_off,
                                                             const uint64_t *d_out_cap, uint64_t *d_out_len, uint8_t *d_blobs,
                                                             const uint64_t *d_blob_off, const uint64_t *d_blob_cap, uint64_t *d_blob_len,
                                                             int32_t *d_status, uint64_t in_total_bytes, uint32_t flags, void *cuda_stream) {
    if (!ctx) return DIVANS_FAILURE;
    if (n == 0) return DIVANS_SUCCESS;
    std::lock_guard<std::mutex> lk(ctx->mu);
    RecParams rp;
    rp.blobs = d_blobs; rp.blob_off = d_blob_off; rp.blob_cap = d_blob_cap; rp.blob_len = d_blob_len; rp.counts = nullptr;
    return decode_device_nolock(ctx, n, d_in, d_in_off, d_in_len, d_out, d_out_off, d_out_cap, d_out_len, d_status, in_total_bytes, flags,
                                cuda_stream, &rp);
}
extern "C" DivansResult divans_b200_decode_cmds_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                                           const uint64_t *in_len, uint8_t *out, const uint64_t *out_off,
                                                           const uint64_t *out_cap, uint64_t *out_len, uint8_t *blobs,
                                                           const uint64_t *blob_off, const uint64_t *blob_cap, uint64_t *blob_len,
                                                           int32_t *status, uint32_t flags) {
    const HostBlobs bl = {blobs, blob_off, blob_cap, blob_len};
    return decode_host(ctx, n, in, in_off, in_len, out, out_off, out_cap, out_len, status, flags, &bl);
}

extern "C" void divans_b200_encode_options_default(divans_b200_encode_options *o) {
    memset(o, 0, sizeof *o);
    o->window_size = 22; o->dynamic_context_mixing = 0; o->prior_depth = 0; o->use_context_map = 1; o->force_stride = 9;
    o->literal_pred_mode = 0; o->literal_mixing_value = 4;
}
// ---- pipelined host-buffer decode: H2D of batch k+1 and D2H of batch k-1 overlap the kernels of batch k ----
static DivansResult lane_wait_nolock(divans_b200_ctx *ctx, int t) {
    divans_b200_ctx::Lane &ln = ctx->lane[t];
    if (!ln.pending) return DIVANS_SUCCESS;
    CK(cudaSetDevice(ctx->device));
    CK(cudaEventSynchronize(ln.e_out));
    memcpy(ln.u_out_len, ln.h_res, ln.n * 8);
    memcpy(ln.u_status, ln.h_res + ln.n * 8, ln.n * 4);
    ln.pending = false; ln.u_out_len = nullptr; ln.u_status = nullptr;
    return DIVANS_SUCCESS;
}
extern "C" DivansResult divans_b200_decode_batch_host_wait(divans_b200_ctx *ctx, int32_t ticket) {
    if (!ctx) return DIVANS_FAILURE;
    if (ticket == DIVANS_B200_TICKET_EMPTY) return DIVANS_SUCCESS;   // an empty batch holds no lane
    if (ticket < 0 || ticket > 1) return DIVANS_FAILURE;
    std::lock_guard<std::mutex> lk(ctx->mu);
    return lane_wait_nolock(ctx, ticket);
}
extern "C" DivansResult divans_b200_decode_batch_host_async(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                                            const uint64_t *in_len, uint8_t *out, const uint64_t *out_off,
                                                            const uint64_t *out_cap, uint64_t *out_len, int32_t *status, uint32_t flags,
                                                            int32_t *ticket) {
    if (!ctx || !ticket) return DIVANS_FAILURE;
    if (n == 0) { *ticket = DIVANS_B200_TICKET_EMPTY; return DIVANS_SUCCESS; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    const int t = (int)(ctx->async_seq++ & 1);
    if (lane_wait_nolock(ctx, t) != DIVANS_SUCCESS) return DIVANS_FAILURE;   // a third batch first retires the oldest one
    CK(cudaSetDevice(ctx->device));
    divans_b200_ctx::Lane &ln = ctx->lane[t];
    if (!ctx->s_h2d) { CK(cudaStreamCreateWithFlags(&ctx->s_h2d, cudaStreamNonBlocking)); CK(cudaStreamCreateWithFlags(&ctx->s_d2h, cudaStreamNonBlocking)); }
    if (!ln.e_in) {
        CK(cudaEventCreateWithFlags(&ln.e_in, cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&ln.e_k, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&ln.e_out, cudaEventDisableTiming));
    }
    if (ln.h_res_cap < n * 12) {
        if (ln.h_res) cudaFreeHost(ln.h_res);
        ln.h_res = nullptr; ln.h_res_cap = 0;
        CK(cudaMallocHost((void **)&ln.h_res, n * 12 + 64));
        ln.h_res_cap = n * 12 + 64;
    }
    uint64_t in_total;
    if (stage_decode(ctx, ln.bufs, n, in, in_off, in_len, out_off, out_cap, nullptr, ctx->s_h2d, ln.e_in, ctx->stream, in_total) !=
        DIVANS_SUCCESS)
        return DIVANS_FAILURE;
    ln.u_out_len = out_len; ln.u_status = status; ln.n = n;
    uint64_t *m = ln.bufs.d_meta;
    int32_t *d_status = reinterpret_cast<int32_t *>(m + 5 * n);
    DivansResult r = decode_device_nolock(ctx, n, ln.bufs.d_in, m, m + n, ln.bufs.d_out, m + 2 * n, m + 3 * n, m + 4 * n, d_status,
                                          in_total, flags, ctx->stream);
    if (r != DIVANS_SUCCESS) return r;
    CK(cudaEventRecord(ln.e_k, ctx->stream));
    CK(cudaStreamWaitEvent(ctx->s_d2h, ln.e_k, 0));
    CK(cudaMemcpyAsync(ln.h_res, m + 4 * n, n * 8, cudaMemcpyDeviceToHost, ctx->s_d2h));
    CK(cudaMemcpyAsync(ln.h_res + n * 8, d_status, n * 4, cudaMemcpyDeviceToHost, ctx->s_d2h));
    if (copy_regions_back(ctx, n, out, ln.bufs.d_out, out_off, out_cap, ctx->s_d2h) != DIVANS_SUCCESS) return DIVANS_FAILURE;
    CK(cudaEventRecord(ln.e_out, ctx->s_d2h));
    ln.pending = true;
    *ticket = t;
    return DIVANS_SUCCESS;
}

// ---- encoder ----
static inline int pack_speed(const int16_t sp[2]) { return (int)((uint32_t)(uint16_t)sp[0] | ((uint32_t)(uint16_t)sp[1] << 16)); }

// Arena slots the encoder's model pass uses for n streams: whole blocks of 16-lane groups, capped by its residency.
constexpr uint32_t ENCODE_GROUPS_PER_BLOCK = DECODE_BLOCK_THREADS / 16;
static size_t encode_slots(const divans_b200_ctx *ctx, size_t n) {
    int per_sm = encode_max_blocks_per_sm(); if (per_sm < 1) per_sm = 1;
    uint32_t max_res = (uint32_t)ctx->sm_count * (uint32_t)per_sm * ENCODE_GROUPS_PER_BLOCK;
    if (ctx->max_resident < max_res) max_res = ctx->max_resident;
    const uint32_t resident = (uint32_t)(n < max_res ? n : max_res);
    return (size_t)((resident + ENCODE_GROUPS_PER_BLOCK - 1) / ENCODE_GROUPS_PER_BLOCK) * ENCODE_GROUPS_PER_BLOCK;
}

static int clamp_window(int w) { return w < 10 ? 10 : (w > 24 ? 24 : w); }

// The PredictionMode record every raw stream starts with (zeroed by the caller), raw_to_cmd/mod.rs:116-143: 64-entry identity
// literal map, 4 distance entries, one mixing value for all 8192 entries, speeds unset.
static void raw_record(uint8_t *pm, int pred_mode, int mixing_value) {
    pm[0] = (uint8_t)pred_mode; pm[2] = 1;
    pm[28] = 64; pm[30] = 4;
    for (int i = 0; i < 64; i++) pm[32 + i] = (uint8_t)i;
    for (int i = 0; i < 4; i++) pm[32 + 16384 + i] = (uint8_t)i;
    memset(pm + 32 + 16384 + 1024, mixing_value, 8192);
}

// ---- encoder log sizing ----
// Every stream of a launch owns `cmd` + `lit` u32 symbol-log entries, and every resident slot `replay` bytes of replay window.
struct LogCaps {
    uint64_t cmd, lit, replay;
};

// the replay window of a stream whose commands replay at most `len` bytes
static uint64_t replay_bytes(uint64_t len) { return (len + 31) & ~15ull; }

static uint32_t raw_cmd_cap(uint64_t max_len, int window) { return (uint32_t)(32 * (2 + (max_len >> window)) + 62000 + 64); }
// raw buffers of at most max_len bytes, coded with `window` (10..24)
static LogCaps raw_log_caps(uint64_t max_len, int window) { return {raw_cmd_cap(max_len, window), 2 * max_len + 16, replay_bytes(max_len)}; }

// Log entries of the command lists of one device call: at most L bytes each, replaying at most max_raw_len bytes each.
//  * Command entries.  The host call sizes a list with header (n_cmds c, n_predmodes p) at 32c + 62000p + 64, and a list the
//    model pass accepts has 20c + 25632p <= R = L - 32.  For a fixed p the most commands are c = floor((R - 25632p) / 20).  One
//    more record (p + 1) costs 25632 bytes, at most ceil(25632 / 20) = 1282 commands, and gains 62000 - 32 * 1282 = 20976 > 0
//    entries: the maximum is at the most records, p = floor(R / 25632), with the rest of the bytes in commands.
//  * Literal entries.  The host call sizes a list at 2s + 16, s = the sum of its literal records' lengths; records may re-read
//    pool bytes, so s is not bounded by L.  But every literal byte coded is also replayed, and the model pass refuses a literal
//    that would not fit the replay window (status 2) before it checks the log: s <= replay, and 2 * replay + 16 always suffices.
static LogCaps cmds_log_caps(uint64_t L, uint64_t max_raw_len) {
    const uint64_t R = L > 32 ? L - 32 : 0, p = R / PM_RECORD_BYTES, replay = replay_bytes(max_raw_len);
    return {32 * ((R - (uint64_t)PM_RECORD_BYTES * p) / 20) + 62000 * p + 64, 2 * replay + 16, replay};
}
//  * A candidate literal model (encode_cmds_auto) replaces records, not commands, so (c, p) and the bound stay those of the blob.
//    But the bound holds per record, not per PredictionMode command: any number of commands may re-read one record, and each
//    codes the whole record.  A raw record codes 64 literal-map and 4 distance-map entries more than a minimal one (empty maps),
//    so a list whose commands re-read minimal records can fit the logs as given and outgrow them under every replacing record.
//    The cost pass therefore counts each pair's entries against these same capacities: a pair that would outgrow them fails
//    there (cost UINT64_MAX), and KEEP or another candidate that fits is chosen (test_many_commands_re_reading_small_records).

// The host call sizes each command list exactly, from its header and commands: 32c + 62000p + 64 command entries, 2s + 16
// literal entries (s: the bytes its literal records code), and the window of the bytes its commands replay.  A list that does
// not parse gets the capacities of its header, and the model pass refuses it.  False: a list too large to encode.
static bool list_log_caps(const uint8_t *b, uint64_t len, LogCaps &caps) {
    uint32_t h[8] = {0};
    if (len >= 32) memcpy(h, b, 32);
    const uint64_t need = 32ull + 20ull * h[2] + (uint64_t)PM_RECORD_BYTES * h[3] + h[4];
    uint64_t lit = 0, rep = 0;
    if (len >= 32 && h[0] == 0x4c435644u && h[1] == 1 && need <= len) {
        for (uint32_t c = 0; c < h[2]; c++) {
            uint32_t r[5]; memcpy(r, b + 32 + 20ull * c, 20);
            if (r[0] == 1) rep += r[2];
            else if (r[0] == 2) rep += 64;            // dictionary word + transform prefix/suffix
            else if (r[0] == 3) { lit += r[2]; rep += r[2]; }
        }
    }
    if (lit > 0x7fff0000ull || rep > 0xfffffff0ull) return false;
    caps = {32ull * h[2] + 62000ull * h[3] + 64, 2 * lit + 16, replay_bytes(rep)};
    return true;
}

// Command-list records are read as u32, so the host calls (encode_host_common, divans_b200_replay_cmds_batch_host) re-base
// blobs that a caller may place at any offset: src[0 .. len) is appended to `staged` at its next 4-byte aligned offset, which is
// returned.
static uint64_t stage_aligned(std::vector<uint8_t> &staged, const uint8_t *src, uint64_t len) {
    const uint64_t o = (staged.size() + 3) & ~(uint64_t)3;
    staged.resize(o + len);
    if (len) memcpy(staged.data() + o, src, len);
    return o;
}

// The EncodeParams fields the model pass and the cost pass share: the n streams at d_in[d_in_off[v] .. +d_in_len[v]), the
// context's arena, tables and replay windows, the log capacities `caps` (sized for streams of up to max_in_len bytes), the
// window (10..24, or 0 for each command list's own) and the options.  Every other field is zero.
static EncodeParams encode_params(const divans_b200_ctx *ctx, size_t n, int raw_mode, const uint8_t *d_in, const uint64_t *d_in_off,
                                  const uint64_t *d_in_len, uint64_t max_in_len, const LogCaps &caps, const divans_b200_encode_options *o,
                                  int window) {
    EncodeParams ep;
    memset(&ep, 0, sizeof ep);
    ep.in = d_in; ep.in_off = d_in_off; ep.in_len = d_in_len; ep.raw_mode = raw_mode; ep.n_streams = (uint32_t)n;
    ep.work_counter = ctx->d_counter; ep.arena = ctx->d_arena; ep.tables = ctx->d_tables;
    ep.replay = ctx->d_replay; ep.replay_stride = caps.replay;
    ep.cmd_cap = (uint32_t)caps.cmd; ep.lit_cap = (uint32_t)caps.lit;
    ep.window_size = window; ep.max_in_len = max_in_len; ep.dynamic_context_mixing = o->dynamic_context_mixing & 0xff; ep.prior_depth = o->prior_depth & 0xff;
    ep.use_context_map = o->use_context_map; ep.force_stride = o->force_stride; ep.have_literal_adaptation = o->have_literal_adaptation;
    for (int k = 0; k < 4; k++) ep.literal_adaptation[k] = pack_speed(o->literal_adaptation[k]);
    ep.model_rev = o->model_rev == DIVANS_B200_MODEL_WASM_2018 ? 1 : 0;
    return ep;
}

// One launch set over n streams whose inputs/outputs already sit in HBM, with the log capacities `caps`.  Like every launch
// sequence of a context, it waits for the previous call's last kernel (`ev_busy`, on whatever stream) before its first write to
// the context's scratch.  `d_pm_records`: the caller's records (encode_auto_device_nolock), else raw streams start with the
// record of the options.
static DivansResult encode_device_internal(divans_b200_ctx *ctx, size_t n, int raw_mode, const uint8_t *d_in, const uint64_t *d_in_off,
                                           const uint64_t *d_in_len, uint64_t max_in_len, const LogCaps &caps, uint8_t *d_out,
                                           const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len, int32_t *d_status,
                                           const divans_b200_encode_options *o, int window, cudaStream_t st,
                                           const uint8_t *d_pm_records = nullptr, const uint32_t *d_pm_index = nullptr, uint32_t pm_keep = 0) {
    const size_t slots = encode_slots(ctx, n);
    const uint32_t blocks = (uint32_t)(slots / ENCODE_GROUPS_PER_BLOCK);
    if (ensure_arena(ctx, slots) != DIVANS_SUCCESS) return DIVANS_FAILURE;
    const uint32_t cmd_cap = (uint32_t)caps.cmd, lit_cap = (uint32_t)caps.lit;
    const uint32_t cmd_chunks = (cmd_cap + NUM_SYMBOLS_BEFORE_FLUSH - 1) / NUM_SYMBOLS_BEFORE_FLUSH;
    const uint32_t lit_chunks = (lit_cap + NUM_SYMBOLS_BEFORE_FLUSH - 1) / NUM_SYMBOLS_BEFORE_FLUSH;
    const uint32_t max_chunks = cmd_chunks + lit_chunks;
    if (!grow(ctx, &ctx->d_sf, &ctx->sf_cap, n * ((size_t)cmd_cap + lit_cap))) return DIVANS_FAILURE;
    if (!grow(ctx, &ctx->d_replay, &ctx->replay_cap, slots * (size_t)caps.replay)) return DIVANS_FAILURE;
    // small per-stream scratch: counts [2n] | window [n] | dummy [slots] | chunk_w [n*max_chunks] | chunk_state [16*n*max_chunks]
    size_t words = 3 * n + slots + n * (size_t)max_chunks + 4 * n * (size_t)max_chunks + 16 + 2 * n * (size_t)max_chunks * (NUM_SYMBOLS_BEFORE_FLUSH / 64);
    if (!grow(ctx, &ctx->d_enc_scratch, &ctx->enc_scratch_cap, words)) return DIVANS_FAILURE;
    if (!ctx->d_pm_internal) CK(cudaMalloc((void **)&ctx->d_pm_internal, PM_RECORD_BYTES));
    if (ctx->busy_recorded) CK(cudaStreamWaitEvent(st, ctx->ev_busy, 0));
    if (!ctx->d_rcp15) { CK(cudaMalloc((void **)&ctx->d_rcp15, 32768 * sizeof(uint64_t))); launch_rcp15_init(ctx->d_rcp15, st); ctx->launches += 1; }
    if (raw_mode && !d_pm_records) {
        std::vector<uint8_t> &pm = ctx->h_pm;
        pm.assign(PM_RECORD_BYTES, 0);
        raw_record(pm.data(), o->literal_pred_mode, o->literal_mixing_value);
        CK(cudaMemcpyAsync(ctx->d_pm_internal, pm.data(), PM_RECORD_BYTES, cudaMemcpyHostToDevice, st));
    }
    EncodeParams ep = encode_params(ctx, n, raw_mode, d_in, d_in_off, d_in_len, max_in_len, caps, o, window);
    ep.pm_internal = d_pm_records ? d_pm_records : ctx->d_pm_internal; ep.pm_index = d_pm_index; ep.pm_keep = pm_keep;
    ep.sf = ctx->d_sf;
    uint32_t *w = ctx->d_enc_scratch;
    ep.sf_counts = w; w += 2 * n;
    ep.stream_window = w; w += n;
    ep.sf_dummy = w; w += slots;
    ep.chunk_w = w; w += n * (size_t)max_chunks;
    w = reinterpret_cast<uint32_t *>(((uintptr_t)w + 15) & ~(uintptr_t)15);
    ep.chunk_state = reinterpret_cast<uint8_t *>(w);
    ep.emit_bits = w + 4 * n * (size_t)max_chunks;
    ep.rcp15 = ctx->d_rcp15;
    ep.max_chunks = max_chunks; ep.cmd_chunks = cmd_chunks;
    ep.out = d_out; ep.out_off = d_out_off; ep.out_cap = d_out_cap; ep.out_len = d_out_len; ep.status = d_status;
    CK(cudaMemsetAsync(ctx->d_counter, 0, 4, st));
    CK(cudaEventRecord(ctx->ev0, st));
    CK(cudaEventRecord(ctx->evm, st));
    if (o->cdf_model == DIVANS_B200_CDF_BLEND) launch_encode_model_blend(ep, blocks, st); else launch_encode_model(ep, blocks, st);
    CK(cudaEventRecord(ctx->evm1, st));
    launch_encode_flush_mux(ep, st);
    CK(cudaEventRecord(ctx->ev1, st));
    CK(cudaEventRecord(ctx->ev_busy, st)); ctx->busy_recorded = true;
    ctx->main_end_is_evm1 = true;
    ctx->launches += 4;
    CK(cudaGetLastError());
    return DIVANS_SUCCESS;
}

// literal model selection of a batch (encode_host_common, encode_device_common): the candidates, and where chosen / cost go.
// mixmap (divans_b200_encode_mixmap_*): the candidates are (opts->literal_pred_mode, v[c]); chosen may be NULL, cost has k + 1
// columns, and mixing / bins are the optional per-context outputs.
struct AutoSel {
    const divans_b200_literal_model *cands; uint32_t n_cands;
    uint32_t *chosen; uint64_t *cost;
    bool mixmap = false; uint8_t *mixing = nullptr; uint64_t *bins = nullptr;
};

// ---- literal model selection ----
// Cost of coding a nibble of frequency f (1..32767 of 32768) in 1/65536 bit: 65536 * (15 - log2 f), the 16 fraction bits of
// log2 f by repeated squaring of the mantissa (each round: square, and one more bit when the square reaches 2).  Integer-only,
// so the CPU oracle's tally (oracle_tally/tally_api.c, dvo_cost_table) computes the same table.  T[0] (freq 0: the stream fails) = T[1].
static uint32_t freq_cost(uint32_t f) {
    if (f == 0) f = 1;
    uint32_t e = 0;
    while ((f >> (e + 1)) != 0) e++;
    uint64_t x = (uint64_t)f << (31 - e);   // f / 2^e in [1, 2), Q31
    uint32_t frac = 0;
    for (int i = 0; i < 16; i++) {
        x = (x * x) >> 31;
        frac <<= 1;
        if (x >= (1ull << 32)) { x >>= 1; frac |= 1; }
    }
    return (15u << 16) - ((e << 16) | frac);
}

// DIVANS_B200_LITERAL_MODEL_KEEP: a command list's own PredictionMode records (command-list calls only)
static bool is_keep(const divans_b200_literal_model &c) { return c.literal_pred_mode == -1 && c.literal_mixing_value == -1; }

// `cmds`: the candidates of a command-list call, which may also be KEEP
static bool check_cands(divans_b200_ctx *ctx, const divans_b200_literal_model *cands, uint32_t n_cands, bool cmds) {
    const char *who = cmds ? "encode_cmds_auto" : "encode_auto";
    char buf[200];
    if (!cands || n_cands < 1 || n_cands > 16) {
        snprintf(buf, sizeof buf, "%s: 1..16 candidate literal models are required", who);
        ctx->err = buf;
        return false;
    }
    for (uint32_t c = 0; c < n_cands; c++)
        if ((cands[c].literal_pred_mode < 0 || cands[c].literal_pred_mode > 3 || cands[c].literal_mixing_value < 0 ||
             cands[c].literal_mixing_value > 15) && !(cmds && is_keep(cands[c]))) {
            snprintf(buf, sizeof buf, "%s: candidate %u (pred_mode %d, mixing value %d) is outside pred_mode 0..3, mixing value 0..15%s",
                     who, c, (int)cands[c].literal_pred_mode, (int)cands[c].literal_mixing_value, cmds ? ", and is not KEEP (-1, -1)" : "");
            ctx->err = buf;
            return false;
        }
    return true;
}

// the cost table of the cost passes, on the context (uploaded on `st` by the first call that needs it)
static bool ensure_cost_tab(divans_b200_ctx *ctx, cudaStream_t st) {
    if (ctx->d_cost_tab) return true;
    static uint32_t tab[32768];
    static std::once_flag once;
    std::call_once(once, [] { for (uint32_t f = 0; f < 32768; f++) tab[f] = freq_cost(f); });
    if (!ck(ctx, cudaMalloc((void **)&ctx->d_cost_tab, sizeof tab), "cudaMalloc(cost table)")) return false;
    return ck(ctx, cudaMemcpyAsync(ctx->d_cost_tab, tab, sizeof tab, cudaMemcpyHostToDevice, st), "cudaMemcpyAsync(cost table)");
}

// One launch sequence over n streams in HBM (raw buffers, or command lists with raw_mode 0): fan out to n * C virtual streams
// (dv_encode.cu: candidate-major), the cost-only model pass over all of them, the per-stream argmin into d_chosen, then the
// encoder pipeline with stream i coded under candidate d_chosen[i] (raw: its starting record; command lists: the record that
// replaces each of the list's own, unless the candidate is KEEP).  The cost pass pulls virtual streams from the work counter
// like the model pass, so however many there are, the context's encoder slots code them as many at a time as they hold.
// caps / window: those of the plain call over the same n streams.
static DivansResult encode_auto_device_nolock(divans_b200_ctx *ctx, size_t n, int raw_mode, const uint8_t *d_in, const uint64_t *d_in_off,
                                              const uint64_t *d_in_len, uint64_t max_in_len, const LogCaps &caps, uint8_t *d_out,
                                              const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len, int32_t *d_status,
                                              const divans_b200_encode_options *o, int window, const divans_b200_literal_model *cands,
                                              uint32_t n_cands, uint32_t *d_chosen, uint64_t *d_cost, cudaStream_t st) {
    const uint64_t nv = (uint64_t)n * n_cands;
    const size_t vslots = encode_slots(ctx, nv);
    if (ensure_arena(ctx, vslots) != DIVANS_SUCCESS) return DIVANS_FAILURE;
    if (!grow(ctx, &ctx->d_replay, &ctx->replay_cap, vslots * (size_t)caps.replay)) return DIVANS_FAILURE;
    // v_off [nv] | v_len [nv] | tally [nv] | v_pm u32 [nv] | v_status i32 [nv]
    if (!grow(ctx, &ctx->d_auto, &ctx->auto_cap, 4 * nv + 2)) return DIVANS_FAILURE;
    uint64_t *v_off = ctx->d_auto, *v_len = v_off + nv, *tally = v_len + nv;
    uint32_t *v_pm = reinterpret_cast<uint32_t *>(tally + nv);
    int32_t *v_status = reinterpret_cast<int32_t *>(v_pm + nv);
    if (!ctx->d_pm_records) CK(cudaMalloc((void **)&ctx->d_pm_records, 16 * (size_t)PM_RECORD_BYTES));
    if (ctx->busy_recorded) CK(cudaStreamWaitEvent(st, ctx->ev_busy, 0));
    if (!ensure_cost_tab(ctx, st)) return DIVANS_FAILURE;
    std::vector<uint8_t> &pm = ctx->h_pm;
    pm.assign((size_t)n_cands * PM_RECORD_BYTES, 0);
    uint32_t keep = 0;   // bit c: candidate c is KEEP (its record stays zero and is never read)
    for (uint32_t c = 0; c < n_cands; c++) {
        if (is_keep(cands[c])) keep |= 1u << c;
        else raw_record(pm.data() + (size_t)c * PM_RECORD_BYTES, cands[c].literal_pred_mode, cands[c].literal_mixing_value);
    }
    CK(cudaMemcpyAsync(ctx->d_pm_records, pm.data(), pm.size(), cudaMemcpyHostToDevice, st));
    launch_auto_fanout(d_in_off, d_in_len, n, n_cands, v_off, v_len, v_pm, st);

    // no logs: cmd_cap / lit_cap are the final encode's capacities, which a pair must fit to be chosen
    EncodeParams tp = encode_params(ctx, nv, raw_mode, d_in, v_off, v_len, max_in_len, caps, o, window);
    tp.pm_internal = ctx->d_pm_records; tp.pm_index = v_pm; tp.pm_keep = keep;
    tp.status = v_status; tp.cost_tab = ctx->d_cost_tab; tp.tally = tally;
    CK(cudaMemsetAsync(ctx->d_counter, 0, 4, st));
    const uint32_t blocks = (uint32_t)(vslots / ENCODE_GROUPS_PER_BLOCK);
    if (o->cdf_model == DIVANS_B200_CDF_BLEND) launch_encode_tally_blend(tp, blocks, st); else launch_encode_tally(tp, blocks, st);
    launch_auto_select(tally, v_status, n, n_cands, d_chosen, d_cost, st);
    ctx->launches += 3;
    CK(cudaGetLastError());
    return encode_device_internal(ctx, n, raw_mode, d_in, d_in_off, d_in_len, max_in_len, caps, d_out, d_out_off, d_out_cap, d_out_len,
                                  d_status, o, window, st, ctx->d_pm_records, d_chosen, keep);
}

// Per-context mixing values: one launch sequence over n streams in HBM.  Records [0, k) are R(p, v[c]), records [k, k + n) the
// streams' mixed records M_i.
//  1. the binned cost pass over the n * k pairs (fan-out as encode_auto): totals u[i][c], per-entry winners best[i][e]
//  2. mixmap_map_kernel builds M_i;  3. the cost pass of every stream under M_i: x[i]
//  4. mixmap_select_kernel: record c* or k + i per stream;  5. the plain pipeline from that record.
// Command lists: every record of a list is replaced (pm_keep 0).  The record index of a mixed stream, k + i, can exceed 31; the
// model pass tests it against pm_keep with a 32-bit shift (shr.u32 yields 0 for counts of 32 or more), so it still reads as "replace".
static DivansResult encode_mixmap_device_nolock(divans_b200_ctx *ctx, size_t n, int raw_mode, const uint8_t *d_in, const uint64_t *d_in_off,
                                                const uint64_t *d_in_len, uint64_t max_in_len, const LogCaps &caps, uint8_t *d_out,
                                                const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len, int32_t *d_status,
                                                const divans_b200_encode_options *o, int window, const divans_b200_literal_model *cands,
                                                uint32_t k, uint32_t *d_chosen, uint64_t *d_cost, uint8_t *d_mixing, uint64_t *d_bins,
                                                cudaStream_t st) {
    const uint64_t nv = (uint64_t)n * k;
    const size_t vslots = encode_slots(ctx, nv);
    if (ensure_arena(ctx, vslots) != DIVANS_SUCCESS) return DIVANS_FAILURE;
    if (!grow(ctx, &ctx->d_replay, &ctx->replay_cap, vslots * (size_t)caps.replay)) return DIVANS_FAILURE;
    // v_off [nv] | v_len [nv] | tally [nv] | v_pm u32 [nv] | v_status i32 [nv]
    if (!grow(ctx, &ctx->d_auto, &ctx->auto_cap, 4 * nv + 2)) return DIVANS_FAILURE;
    uint64_t *v_off = ctx->d_auto, *v_len = v_off + nv, *tally = v_len + nv;
    uint32_t *v_pm = reinterpret_cast<uint32_t *>(tally + nv);
    int32_t *v_status = reinterpret_cast<int32_t *>(v_pm + nv);
    // best [n * 8192] | x_tally [n] | x_status i32 [n] | mix_idx u32 [n] | rec_idx u32 [n]
    if (!grow(ctx, &ctx->d_mix, &ctx->mix_cap, (size_t)n * MIX_ENTRIES + 3 * n)) return DIVANS_FAILURE;
    uint64_t *best = ctx->d_mix, *x_tally = best + (size_t)n * MIX_ENTRIES;
    int32_t *x_status = reinterpret_cast<int32_t *>(x_tally + n);
    uint32_t *mix_idx = reinterpret_cast<uint32_t *>(x_status + n), *rec_idx = mix_idx + n;
    if (!grow(ctx, &ctx->d_mix_records, &ctx->mix_records_cap, (k + n) * (size_t)PM_RECORD_BYTES)) return DIVANS_FAILURE;
    if (!grow(ctx, &ctx->d_slot_bins, &ctx->slot_bins_cap, vslots * (size_t)MIX_ENTRIES)) return DIVANS_FAILURE;
    if (ctx->busy_recorded) CK(cudaStreamWaitEvent(st, ctx->ev_busy, 0));
    if (!ensure_cost_tab(ctx, st)) return DIVANS_FAILURE;
    std::vector<uint8_t> &pm = ctx->h_pm;
    pm.assign((size_t)k * PM_RECORD_BYTES, 0);
    MixValues vals; memset(&vals, 0, sizeof vals); vals.k = k;
    for (uint32_t c = 0; c < k; c++) {
        raw_record(pm.data() + (size_t)c * PM_RECORD_BYTES, cands[c].literal_pred_mode, cands[c].literal_mixing_value);
        vals.v[c] = (uint8_t)cands[c].literal_mixing_value;
    }
    CK(cudaMemcpyAsync(ctx->d_mix_records, pm.data(), pm.size(), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(best, 0xff, (size_t)n * MIX_ENTRIES * 8, st));
    launch_auto_fanout(d_in_off, d_in_len, n, k, v_off, v_len, v_pm, st);

    // 1. uniform passes, binned
    EncodeParams tp = encode_params(ctx, nv, raw_mode, d_in, v_off, v_len, max_in_len, caps, o, window);
    tp.pm_internal = ctx->d_mix_records; tp.pm_index = v_pm; tp.pm_keep = 0;
    tp.status = v_status; tp.cost_tab = ctx->d_cost_tab; tp.tally = tally;
    BinParams bp;
    bp.slot_bins = ctx->d_slot_bins; bp.best = best; bp.bins_out = d_bins; bp.n = (uint32_t)n; bp.k = k;
    CK(cudaMemsetAsync(ctx->d_counter, 0, 4, st));
    if (o->cdf_model == DIVANS_B200_CDF_BLEND) launch_encode_bins_blend(tp, bp, (uint32_t)(vslots / ENCODE_GROUPS_PER_BLOCK), st);
    else launch_encode_bins(tp, bp, (uint32_t)(vslots / ENCODE_GROUPS_PER_BLOCK), st);
    // 2. mixed records;  3. the mixed pass, the plain cost pass (a mixed record is not uniform, so its literals take the per-nibble loop)
    launch_mixmap_map(best, n, vals, ctx->d_mix_records, mix_idx, st);
    EncodeParams xp = encode_params(ctx, n, raw_mode, d_in, d_in_off, d_in_len, max_in_len, caps, o, window);
    xp.pm_internal = ctx->d_mix_records; xp.pm_index = mix_idx; xp.pm_keep = 0;
    xp.status = x_status; xp.cost_tab = ctx->d_cost_tab; xp.tally = x_tally;
    CK(cudaMemsetAsync(ctx->d_counter, 0, 4, st));
    const uint32_t xblocks = (uint32_t)(encode_slots(ctx, n) / ENCODE_GROUPS_PER_BLOCK);
    if (o->cdf_model == DIVANS_B200_CDF_BLEND) launch_encode_tally_blend(xp, xblocks, st); else launch_encode_tally(xp, xblocks, st);
    // 4. choice
    launch_mixmap_select(tally, v_status, x_tally, x_status, n, vals, ctx->d_mix_records, rec_idx, d_chosen, d_cost, d_mixing, st);
    ctx->launches += 5;
    CK(cudaGetLastError());
    return encode_device_internal(ctx, n, raw_mode, d_in, d_in_off, d_in_len, max_in_len, caps, d_out, d_out_off, d_out_cap, d_out_len,
                                  d_status, o, window, st, ctx->d_mix_records, rec_idx, 0);
}

// `values` (1..16 mixing values 0..15) and the mode of opts as candidate literal models; false (and the error) for anything else
static bool mixmap_cands(divans_b200_ctx *ctx, const int32_t *values, uint32_t k, const divans_b200_encode_options *o,
                         divans_b200_literal_model *cands) {
    char buf[200];
    if (!values || k < 1 || k > 16) { ctx->err = "encode_mixmap: 1..16 mixing values are required"; return false; }
    if (o->literal_pred_mode < 0 || o->literal_pred_mode > 3) {
        snprintf(buf, sizeof buf, "encode_mixmap: opts->literal_pred_mode %d is outside 0..3", (int)o->literal_pred_mode);
        ctx->err = buf;
        return false;
    }
    for (uint32_t c = 0; c < k; c++) {
        if (values[c] < 0 || values[c] > 15) {
            snprintf(buf, sizeof buf, "encode_mixmap: mixing value %u (%d) is outside 0..15", c, (int)values[c]);
            ctx->err = buf;
            return false;
        }
        cands[c].literal_pred_mode = o->literal_pred_mode; cands[c].literal_mixing_value = values[c];
    }
    return true;
}

// The four device encode calls: raw buffers (max_raw_len = max_in_len) or command lists (raw_mode 0), each plain or, with
// `sel` (device chosen / cost), coded under the cheapest candidate literal model.  Host marshalling (the candidates' records,
// the error strings) may throw, and no C++ exception may cross the C boundary.
static DivansResult encode_device_common(divans_b200_ctx *ctx, size_t n, int raw_mode, const uint8_t *d_in, const uint64_t *d_in_off,
                                         const uint64_t *d_in_len, uint64_t max_in_len, uint64_t max_raw_len, uint8_t *d_out,
                                         const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len, int32_t *d_status,
                                         const divans_b200_encode_options *opts, void *cuda_stream, const AutoSel *sel) try {
    if (!ctx || !opts) return DIVANS_FAILURE;
    if (sel && !check_cands(ctx, sel->cands, sel->n_cands, !raw_mode)) return DIVANS_FAILURE;
    if (n == 0) return DIVANS_SUCCESS;
    if (sel && !sel->mixmap && !sel->chosen) { ctx->err = raw_mode ? "encode_auto: d_chosen is required" : "encode_cmds_auto: d_chosen is required"; return DIVANS_FAILURE; }
    if (sel && sel->mixmap && n > 0x7fffffffull) { ctx->err = "batch too large"; return DIVANS_FAILURE; }   // (one block per stream)
    const uint64_t nv = (uint64_t)n * (sel ? sel->n_cands : 1);
    if (nv > 0xffffffffull || max_in_len > 0x7fff0000ull || max_raw_len > 0x7fff0000ull) { ctx->err = "batch too large"; return DIVANS_FAILURE; }
    const int window = !raw_mode && opts->window_size == 0 ? 0 : clamp_window(opts->window_size);
    const LogCaps caps = raw_mode ? raw_log_caps(max_in_len, window) : cmds_log_caps(max_in_len, max_raw_len);
    // the kernels address a stream's logs at v * (cmd_cap + lit_cap) with a 32-bit stride
    if (caps.cmd + caps.lit > 0xffffffffull) { ctx->err = "batch too large"; return DIVANS_FAILURE; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
    if (!raw_mode) {
        // the slots first, as in the host call: the logs are sized from what is left, and a failure names them.  (The cost pass of
        // the n * C pairs has no logs; it runs in as many slots as the pairs fill.)
        if (ensure_arena(ctx, encode_slots(ctx, nv)) != DIVANS_SUCCESS) return DIVANS_FAILURE;
        // No sub-batching: the logs of all n streams are one allocation, of exactly their size (they are most of what the call
        // needs next to the arena).  When it fails, the call fails and says how much it asked for.
        const size_t words = n * (size_t)(caps.cmd + caps.lit);
        if (words > ctx->sf_cap) {
            cudaFree(ctx->d_sf); ctx->d_sf = nullptr; ctx->sf_cap = 0;
            if (cudaMalloc((void **)&ctx->d_sf, words * 4) != cudaSuccess) {
                cudaGetLastError();
                char buf[200];
                snprintf(buf, sizeof buf, "divans_b200: cannot allocate the symbol logs of %zu command lists of up to %llu bytes: %llu bytes", n,
                         (unsigned long long)max_in_len, (unsigned long long)words * 4);
                ctx->err = buf;
                return DIVANS_FAILURE;
            }
            ctx->sf_cap = words;
        }
    }
    if (sel && sel->mixmap)
        return encode_mixmap_device_nolock(ctx, n, raw_mode, d_in, d_in_off, d_in_len, max_in_len, caps, d_out, d_out_off, d_out_cap, d_out_len,
                                           d_status, opts, window, sel->cands, sel->n_cands, sel->chosen, sel->cost, sel->mixing, sel->bins, st);
    if (sel)
        return encode_auto_device_nolock(ctx, n, raw_mode, d_in, d_in_off, d_in_len, max_in_len, caps, d_out, d_out_off, d_out_cap, d_out_len,
                                         d_status, opts, window, sel->cands, sel->n_cands, sel->chosen, sel->cost, st);
    return encode_device_internal(ctx, n, raw_mode, d_in, d_in_off, d_in_len, max_in_len, caps, d_out, d_out_off, d_out_cap, d_out_len,
                                  d_status, opts, window, st);
} catch (...) {
    if (ctx) ctx->err = "divans_b200: out of host memory";
    return DIVANS_FAILURE;
}

extern "C" DivansResult divans_b200_encode_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                        const uint64_t *d_in_len, uint64_t max_in_len, uint8_t *d_out,
                                                        const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len,
                                                        int32_t *d_status, const divans_b200_encode_options *opts, void *cuda_stream) {
    return encode_device_common(ctx, n, 1, d_in, d_in_off, d_in_len, max_in_len, max_in_len, d_out, d_out_off, d_out_cap, d_out_len,
                                d_status, opts, cuda_stream, nullptr);
}
extern "C" DivansResult divans_b200_encode_auto_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                             const uint64_t *d_in_len, uint64_t max_in_len, uint8_t *d_out,
                                                             const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len,
                                                             int32_t *d_status, const divans_b200_encode_options *opts,
                                                             const divans_b200_literal_model *cands, uint32_t n_cands, uint32_t *d_chosen,
                                                             uint64_t *d_cost, void *cuda_stream) {
    const AutoSel sel = {cands, n_cands, d_chosen, d_cost};
    return encode_device_common(ctx, n, 1, d_in, d_in_off, d_in_len, max_in_len, max_in_len, d_out, d_out_off, d_out_cap, d_out_len,
                                d_status, opts, cuda_stream, &sel);
}
extern "C" DivansResult divans_b200_encode_cmds_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_blobs, const uint64_t *d_blob_off,
                                                             const uint64_t *d_blob_len, uint64_t max_blob_len, uint64_t max_raw_len,
                                                             uint8_t *d_out, const uint64_t *d_out_off, const uint64_t *d_out_cap,
                                                             uint64_t *d_out_len, int32_t *d_status, const divans_b200_encode_options *opts,
                                                             void *cuda_stream) {
    return encode_device_common(ctx, n, 0, d_blobs, d_blob_off, d_blob_len, max_blob_len, max_raw_len, d_out, d_out_off, d_out_cap,
                                d_out_len, d_status, opts, cuda_stream, nullptr);
}
extern "C" DivansResult divans_b200_encode_cmds_auto_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_blobs,
                                                                  const uint64_t *d_blob_off, const uint64_t *d_blob_len,
                                                                  uint64_t max_blob_len, uint64_t max_raw_len, uint8_t *d_out,
                                                                  const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len,
                                                                  int32_t *d_status, const divans_b200_encode_options *opts,
                                                                  const divans_b200_literal_model *cands, uint32_t n_cands,
                                                                  uint32_t *d_chosen, uint64_t *d_cost, void *cuda_stream) {
    const AutoSel sel = {cands, n_cands, d_chosen, d_cost};
    return encode_device_common(ctx, n, 0, d_blobs, d_blob_off, d_blob_len, max_blob_len, max_raw_len, d_out, d_out_off, d_out_cap,
                                d_out_len, d_status, opts, cuda_stream, &sel);
}

// The four host encode calls: marshal, split into sub-batches whose symbol logs fit in HBM, run, copy back.  Host marshalling
// uses std::vector sized by the caller's arguments, and no C++ exception may cross the C boundary.
static DivansResult encode_host_common(divans_b200_ctx *ctx, size_t n, int raw_mode, const uint8_t *in, const uint64_t *in_off,
                                       const uint64_t *in_len, uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap,
                                       uint64_t *out_len, int32_t *status, const divans_b200_encode_options *opts,
                                       const AutoSel *sel) try {
    if (!ctx || !opts) return DIVANS_FAILURE;
    if (sel && !check_cands(ctx, sel->cands, sel->n_cands, !raw_mode)) return DIVANS_FAILURE;
    if (n == 0) return DIVANS_SUCCESS;
    if (sel && !sel->mixmap && !sel->chosen) { ctx->err = raw_mode ? "encode_auto: chosen is required" : "encode_cmds_auto: chosen is required"; return DIVANS_FAILURE; }
    if (sel && (uint64_t)n * sel->n_cands > 0xffffffffull) { ctx->err = "batch too large"; return DIVANS_FAILURE; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    CK(cudaSetDevice(ctx->device));
    const int window = clamp_window(opts->window_size);
    // per-stream requirements
    std::vector<uint64_t> s_off(n);
    std::vector<LogCaps> need(n);
    std::vector<uint8_t> staged;   // command lists are re-based to 4-byte aligned offsets
    uint64_t in_end = 0;
    for (size_t i = 0; i < n; i++) {
        status[i] = DIVANS_FAILURE; out_len[i] = 0;
        if (raw_mode) {
            if (in_len[i] > 0x7fff0000ull) { ctx->err = "stream too large"; return DIVANS_FAILURE; }
            s_off[i] = in_off[i];
            need[i] = raw_log_caps(in_len[i], window);
            if (in_off[i] + in_len[i] > in_end) in_end = in_off[i] + in_len[i];
        } else {
            if (!list_log_caps(in + in_off[i], in_len[i], need[i])) { ctx->err = "stream too large"; return DIVANS_FAILURE; }
            s_off[i] = stage_aligned(staged, in + in_off[i], in_len[i]);
            in_end = staged.size();
        }
    }
    const uint8_t *src = raw_mode ? in : staged.data();
    // the slots first: the symbol logs are sized from what is left (on an 80 GB GPU the slots take most of the memory)
    if (ensure_arena(ctx, encode_slots(ctx, n)) != DIVANS_SUCCESS) return DIVANS_FAILURE;
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    const uint64_t budget = (uint64_t)(free_b + ctx->sf_cap * 4) * 6 / 10;
    HostBufs &b = ctx->host;
    if (!grow(ctx, &b.d_in, &b.d_in_cap, (size_t)in_end + 64)) return DIVANS_FAILURE;
    cudaStream_t st = ctx->stream;
    CK(cudaMemcpyAsync(b.d_in, src, in_end, cudaMemcpyHostToDevice, st));
    size_t i0 = 0;
    while (i0 < n) {
        // grow the sub-batch while its uniform-capacity logs fit
        LogCaps mc = {0, 0, 0};
        uint64_t mx = 0; size_t i1 = i0;
        while (i1 < n) {
            const LogCaps c = {std::max(need[i1].cmd, mc.cmd), std::max(need[i1].lit, mc.lit), std::max(need[i1].replay, mc.replay)};
            // encode_auto: the cost pass also holds a replay window per slot for up to m * C pairs.  encode_mixmap: and 64 KiB of
            // bins per slot, and per stream its winners, mixed record, mixing output and (when asked for) C x 64 KiB of bins
            const uint64_t vs = sel ? (uint64_t)encode_slots(ctx, (i1 - i0 + 1) * (size_t)sel->n_cands) : 0;
            uint64_t rep = vs * c.replay;
            if (sel && sel->mixmap)
                rep += vs * MIX_ENTRIES * 8 + (uint64_t)(i1 - i0 + 1) * (MIX_ENTRIES * 9 + PM_RECORD_BYTES + (sel->bins ? sel->n_cands * MIX_ENTRIES * 8ull : 0));
            if (i1 > i0 && (c.cmd + c.lit) * 4 * (uint64_t)(i1 - i0 + 1) + rep > budget) break;
            mc = c;
            if (in_len[i1] > mx) mx = in_len[i1];
            i1++;
        }
        if (mc.cmd + mc.lit > 0xffffffffull) { ctx->err = "stream too large"; return DIVANS_FAILURE; }   // (the kernels' 32-bit log stride)
        const size_t m = i1 - i0;
        uint64_t out_lo, out_hi;
        regions_span(m, out_off + i0, out_cap + i0, out_lo, out_hi);
        if (!grow(ctx, &b.d_out, &b.d_out_cap, (size_t)(out_hi - out_lo) + 64)) return DIVANS_FAILURE;
        // in_off | in_len | out_off | out_cap | out_len | status (+ encode_auto: chosen | cost [m * C]; encode_mixmap: cost [m * (C + 1)])
        const size_t cost_cols = sel ? sel->n_cands + (sel->mixmap ? 1 : 0) : 0;
        if (!grow(ctx, &b.d_meta, &b.d_meta_cap, m * 6 + (sel ? m + m * cost_cols : 0))) return DIVANS_FAILURE;
        // encode_mixmap: mixing [m * 8192 bytes] | bins [m * C * 8192]
        uint8_t *d_mixing = nullptr; uint64_t *d_bins = nullptr;
        if (sel && sel->mixmap) {
            const size_t bw = sel->bins ? m * (size_t)sel->n_cands * MIX_ENTRIES : 0;
            if (!grow(ctx, &ctx->d_mix_out, &ctx->mix_out_cap, m * (size_t)MIX_ENTRIES / 8 + bw)) return DIVANS_FAILURE;
            if (sel->mixing) d_mixing = reinterpret_cast<uint8_t *>(ctx->d_mix_out);
            if (sel->bins) d_bins = ctx->d_mix_out + m * (size_t)MIX_ENTRIES / 8;
        }
        std::vector<uint64_t> rel(m);
        for (size_t i = 0; i < m; i++) rel[i] = out_off[i0 + i] - out_lo;
        uint64_t *mm = b.d_meta;
        CK(cudaMemcpyAsync(mm, s_off.data() + i0, m * 8, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(mm + m, in_len + i0, m * 8, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(mm + 2 * m, rel.data(), m * 8, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(mm + 3 * m, out_cap + i0, m * 8, cudaMemcpyHostToDevice, st));
        int32_t *d_status = reinterpret_cast<int32_t *>(mm + 5 * m);
        uint32_t *d_chosen = reinterpret_cast<uint32_t *>(mm + 6 * m);
        uint64_t *d_cost = mm + 7 * m;
        DivansResult r = sel && sel->mixmap
                             ? encode_mixmap_device_nolock(ctx, m, raw_mode, b.d_in, mm, mm + m, mx, mc, b.d_out, mm + 2 * m, mm + 3 * m, mm + 4 * m,
                                                           d_status, opts, window, sel->cands, sel->n_cands, d_chosen, d_cost, d_mixing, d_bins, st)
                         : sel ? encode_auto_device_nolock(ctx, m, raw_mode, b.d_in, mm, mm + m, mx, mc, b.d_out, mm + 2 * m, mm + 3 * m,
                                                           mm + 4 * m, d_status, opts, window, sel->cands, sel->n_cands, d_chosen, d_cost, st)
                               : encode_device_internal(ctx, m, raw_mode, b.d_in, mm, mm + m, mx, mc, b.d_out, mm + 2 * m, mm + 3 * m,
                                                        mm + 4 * m, d_status, opts, window, st);
        if (r != DIVANS_SUCCESS) return r;
        if (sel) {
            if (sel->chosen) CK(cudaMemcpyAsync(sel->chosen + i0, d_chosen, m * 4, cudaMemcpyDeviceToHost, st));
            if (sel->cost) CK(cudaMemcpyAsync(sel->cost + i0 * cost_cols, d_cost, m * cost_cols * 8, cudaMemcpyDeviceToHost, st));
            if (d_mixing) CK(cudaMemcpyAsync(sel->mixing + i0 * (size_t)MIX_ENTRIES, d_mixing, m * (size_t)MIX_ENTRIES, cudaMemcpyDeviceToHost, st));
            if (d_bins) CK(cudaMemcpyAsync(sel->bins + i0 * (size_t)sel->n_cands * MIX_ENTRIES, d_bins, m * (size_t)sel->n_cands * MIX_ENTRIES * 8,
                                           cudaMemcpyDeviceToHost, st));
        }
        CK(cudaMemcpyAsync(out_len + i0, mm + 4 * m, m * 8, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(status + i0, d_status, m * 4, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        for (size_t i = i0; i < i1; i++) {
            if (status[i] == DIVANS_SUCCESS && out_len[i]) CK(cudaMemcpyAsync(out + out_off[i], b.d_out + (out_off[i] - out_lo), out_len[i], cudaMemcpyDeviceToHost, st));
        }
        CK(cudaStreamSynchronize(st));
        i0 = i1;
    }
    return DIVANS_SUCCESS;
} catch (...) {
    if (ctx) ctx->err = "divans_b200: out of host memory while marshalling the batch";
    return DIVANS_FAILURE;
}
extern "C" DivansResult divans_b200_encode_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                                      const uint64_t *in_len, uint8_t *out, const uint64_t *out_off,
                                                      const uint64_t *out_cap, uint64_t *out_len, int32_t *status,
                                                      const divans_b200_encode_options *opts) {
    return encode_host_common(ctx, n, 1, in, in_off, in_len, out, out_off, out_cap, out_len, status, opts, nullptr);
}
extern "C" DivansResult divans_b200_encode_auto_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                                           const uint64_t *in_len, uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap,
                                                           uint64_t *out_len, int32_t *status, const divans_b200_encode_options *opts,
                                                           const divans_b200_literal_model *cands, uint32_t n_cands, uint32_t *chosen,
                                                           uint64_t *cost) {
    const AutoSel sel = {cands, n_cands, chosen, cost};
    return encode_host_common(ctx, n, 1, in, in_off, in_len, out, out_off, out_cap, out_len, status, opts, &sel);
}
extern "C" DivansResult divans_b200_encode_cmds_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *blobs, const uint64_t *blob_off,
                                                           const uint64_t *blob_len, uint8_t *out, const uint64_t *out_off,
                                                           const uint64_t *out_cap, uint64_t *out_len, int32_t *status,
                                                           const divans_b200_encode_options *opts) {
    return encode_host_common(ctx, n, 0, blobs, blob_off, blob_len, out, out_off, out_cap, out_len, status, opts, nullptr);
}
extern "C" DivansResult divans_b200_encode_cmds_auto_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *blobs, const uint64_t *blob_off,
                                                                const uint64_t *blob_len, uint8_t *out, const uint64_t *out_off,
                                                                const uint64_t *out_cap, uint64_t *out_len, int32_t *status,
                                                                const divans_b200_encode_options *opts, const divans_b200_literal_model *cands,
                                                                uint32_t n_cands, uint32_t *chosen, uint64_t *cost) {
    const AutoSel sel = {cands, n_cands, chosen, cost};
    return encode_host_common(ctx, n, 0, blobs, blob_off, blob_len, out, out_off, out_cap, out_len, status, opts, &sel);
}

// ---- per-context mixing values ----
extern "C" DivansResult divans_b200_encode_mixmap_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                                             const uint64_t *in_len, uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap,
                                                             uint64_t *out_len, int32_t *status, const divans_b200_encode_options *opts,
                                                             const int32_t *values, uint32_t n_values, uint32_t *chosen, uint8_t *mixing,
                                                             uint64_t *cost, uint64_t *bins) {
    divans_b200_literal_model cands[16];
    if (!ctx || !opts || !mixmap_cands(ctx, values, n_values, opts, cands)) return DIVANS_FAILURE;
    const AutoSel sel = {cands, n_values, chosen, cost, true, mixing, bins};
    return encode_host_common(ctx, n, 1, in, in_off, in_len, out, out_off, out_cap, out_len, status, opts, &sel);
}
extern "C" DivansResult divans_b200_encode_mixmap_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                               const uint64_t *d_in_len, uint64_t max_in_len, uint8_t *d_out,
                                                               const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len,
                                                               int32_t *d_status, const divans_b200_encode_options *opts, const int32_t *values,
                                                               uint32_t n_values, uint32_t *d_chosen, uint8_t *d_mixing, uint64_t *d_cost,
                                                               uint64_t *d_bins, void *cuda_stream) {
    divans_b200_literal_model cands[16];
    if (!ctx || !opts || !mixmap_cands(ctx, values, n_values, opts, cands)) return DIVANS_FAILURE;
    const AutoSel sel = {cands, n_values, d_chosen, d_cost, true, d_mixing, d_bins};
    return encode_device_common(ctx, n, 1, d_in, d_in_off, d_in_len, max_in_len, max_in_len, d_out, d_out_off, d_out_cap, d_out_len,
                                d_status, opts, cuda_stream, &sel);
}
extern "C" DivansResult divans_b200_encode_cmds_mixmap_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *blobs, const uint64_t *blob_off,
                                                                  const uint64_t *blob_len, uint8_t *out, const uint64_t *out_off,
                                                                  const uint64_t *out_cap, uint64_t *out_len, int32_t *status,
                                                                  const divans_b200_encode_options *opts, const int32_t *values, uint32_t n_values,
                                                                  uint32_t *chosen, uint8_t *mixing, uint64_t *cost, uint64_t *bins) {
    divans_b200_literal_model cands[16];
    if (!ctx || !opts || !mixmap_cands(ctx, values, n_values, opts, cands)) return DIVANS_FAILURE;
    const AutoSel sel = {cands, n_values, chosen, cost, true, mixing, bins};
    return encode_host_common(ctx, n, 0, blobs, blob_off, blob_len, out, out_off, out_cap, out_len, status, opts, &sel);
}
extern "C" DivansResult divans_b200_encode_cmds_mixmap_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_blobs,
                                                                    const uint64_t *d_blob_off, const uint64_t *d_blob_len,
                                                                    uint64_t max_blob_len, uint64_t max_raw_len, uint8_t *d_out,
                                                                    const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len,
                                                                    int32_t *d_status, const divans_b200_encode_options *opts,
                                                                    const int32_t *values, uint32_t n_values, uint32_t *d_chosen,
                                                                    uint8_t *d_mixing, uint64_t *d_cost, uint64_t *d_bins, void *cuda_stream) {
    divans_b200_literal_model cands[16];
    if (!ctx || !opts || !mixmap_cands(ctx, values, n_values, opts, cands)) return DIVANS_FAILURE;
    const AutoSel sel = {cands, n_values, d_chosen, d_cost, true, d_mixing, d_bins};
    return encode_device_common(ctx, n, 0, d_blobs, d_blob_off, d_blob_len, max_blob_len, max_raw_len, d_out, d_out_off, d_out_cap,
                                d_out_len, d_status, opts, cuda_stream, &sel);
}

// ---- replaying command lists to raw bytes ----
// One launch (dv_replay.cu) over n lists in HBM.  It uses the context's work counter, tables and timing events only: no slot,
// arena or encoder log, so it runs on a context that has never decoded or encoded.
static DivansResult replay_device_nolock(divans_b200_ctx *ctx, size_t n, const uint8_t *d_blobs, const uint64_t *d_blob_off,
                                         const uint64_t *d_blob_len, uint8_t *d_out, const uint64_t *d_out_off, const uint64_t *d_out_cap,
                                         uint64_t *d_out_len, int32_t *d_status, int32_t window_size, cudaStream_t st) {
    if (n > 0xffffffffull) { ctx->err = "too many command lists"; return DIVANS_FAILURE; }
    if (ctx->busy_recorded) CK(cudaStreamWaitEvent(st, ctx->ev_busy, 0));
    ReplayParams rp;
    rp.blobs = d_blobs; rp.blob_off = d_blob_off; rp.blob_len = d_blob_len;
    rp.out = d_out; rp.out_off = d_out_off; rp.out_cap = d_out_cap; rp.out_len = d_out_len; rp.status = d_status;
    rp.n_lists = (uint32_t)n; rp.window = window_size == 0 ? 0 : clamp_window(window_size);   // the encoder's window rule
    rp.work_counter = ctx->d_counter; rp.tables = ctx->d_tables;
    CK(cudaMemsetAsync(ctx->d_counter, 0, 4, st));
    CK(cudaEventRecord(ctx->ev0, st));
    CK(cudaEventRecord(ctx->evm, st));
    launch_replay_cmds(rp, ctx->sm_count, st);
    CK(cudaEventRecord(ctx->ev1, st));
    CK(cudaEventRecord(ctx->ev_busy, st)); ctx->busy_recorded = true;
    ctx->main_end_is_evm1 = false;
    ctx->launches += 1;
    CK(cudaGetLastError());
    return DIVANS_SUCCESS;
}
extern "C" DivansResult divans_b200_replay_cmds_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_blobs, const uint64_t *d_blob_off,
                                                             const uint64_t *d_blob_len, uint8_t *d_out, const uint64_t *d_out_off,
                                                             const uint64_t *d_out_cap, uint64_t *d_out_len, int32_t *d_status,
                                                             int32_t window_size, void *cuda_stream) {
    if (!ctx) return DIVANS_FAILURE;
    if (n == 0) return DIVANS_SUCCESS;
    std::lock_guard<std::mutex> lk(ctx->mu);
    CK(cudaSetDevice(ctx->device));
    return replay_device_nolock(ctx, n, d_blobs, d_blob_off, d_blob_len, d_out, d_out_off, d_out_cap, d_out_len, d_status, window_size,
                                cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream);
}
// Staged like a host decode (stage_decode, copy_regions_back); the records are read as u32, so blobs at offsets that are not
// 4-byte aligned are first re-based on the host, as divans_b200_encode_cmds_batch_host does.
extern "C" DivansResult divans_b200_replay_cmds_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *blobs, const uint64_t *blob_off,
                                                           const uint64_t *blob_len, uint8_t *out, const uint64_t *out_off,
                                                           const uint64_t *out_cap, uint64_t *out_len, int32_t *status,
                                                           int32_t window_size) try {
    if (!ctx) return DIVANS_FAILURE;
    if (n == 0) return DIVANS_SUCCESS;
    const uint8_t *src = blobs;
    const uint64_t *src_off = blob_off;
    std::vector<uint64_t> s_off;
    std::vector<uint8_t> staged;
    if (std::any_of(blob_off, blob_off + n, [](uint64_t o) { return (o & 3u) != 0; })) {
        s_off.resize(n);
        for (size_t i = 0; i < n; i++) s_off[i] = stage_aligned(staged, blobs + blob_off[i], blob_len[i]);
        src = staged.data(); src_off = s_off.data();
    }
    std::lock_guard<std::mutex> lk(ctx->mu);
    CK(cudaSetDevice(ctx->device));
    HostBufs &b = ctx->host;
    cudaStream_t st = ctx->stream;
    uint64_t in_total;
    if (stage_decode(ctx, b, n, src, src_off, blob_len, out_off, out_cap, nullptr, st, nullptr, st, in_total) != DIVANS_SUCCESS)
        return DIVANS_FAILURE;
    uint64_t *m = b.d_meta;
    int32_t *d_status = reinterpret_cast<int32_t *>(m + 5 * n);
    DivansResult r = replay_device_nolock(ctx, n, b.d_in, m, m + n, b.d_out, m + 2 * n, m + 3 * n, m + 4 * n, d_status, window_size, st);
    if (r != DIVANS_SUCCESS) return r;
    CK(cudaMemcpyAsync(out_len, m + 4 * n, n * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(status, d_status, n * 4, cudaMemcpyDeviceToHost, st));
    if (copy_regions_back(ctx, n, out, b.d_out, out_off, out_cap, st) != DIVANS_SUCCESS) return DIVANS_FAILURE;
    CK(cudaStreamSynchronize(st));
    return DIVANS_SUCCESS;
} catch (...) {
    if (ctx) ctx->err = "divans_b200: out of host memory while staging the command lists";
    return DIVANS_FAILURE;
}

// ---- generating LZ77 command lists on the GPU ----
// One launch (dv_lz77.cu) over n raw buffers in HBM: the blobs of divans_b200_lz77_cmds_batch.  Like the replay call it uses the
// context's work counter and timing events only, and its own scratch: 2^15 + max_in_len int32 per warp, kept and grown on demand.
// The warps are the fewest of n, the context's max_resident and what the scratch allocation holds.
extern "C" DivansResult divans_b200_lz77_cmds_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                           const uint64_t *d_in_len, uint64_t max_in_len, int32_t window, int32_t pred_mode,
                                                           int32_t mixing_value, uint8_t *d_blobs, const uint64_t *d_blob_off,
                                                           const uint64_t *d_blob_cap, uint64_t *d_blob_len, int32_t *d_status,
                                                           void *cuda_stream) try {
    if (!ctx) return DIVANS_FAILURE;
    if (window < 10 || window > 24) { ctx->err = "lz77_cmds_batch_device: window must be 10..24"; return DIVANS_FAILURE; }
    if (n > 0xffffffffull) { ctx->err = "lz77_cmds_batch_device: too many streams"; return DIVANS_FAILURE; }
    if (n == 0) return DIVANS_SUCCESS;
    std::lock_guard<std::mutex> lk(ctx->mu);
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
    // streams of 2^31 bytes or more are refused by the kernel, so prev never needs more entries than that
    const uint64_t stride = lz77_scratch_words(std::min<uint64_t>(max_in_len, 0x7fffffffull));
    uint64_t warps = std::min<uint64_t>(n, std::max<uint32_t>(ctx->max_resident, 1u));
    // Grown when it holds fewer warps than asked for, unless free memory already cut an equal or larger request down: that
    // allocation is as large as it gets, and asking again would only free it and wait for the device.
    const uint64_t want = warps * stride;
    if (ctx->lz_scratch_words < stride || (ctx->lz_scratch_words < want && want > ctx->lz_scratch_asked)) {
        // the old scratch may still be in use by the previous launch: cudaFree waits for the device
        cudaFree(ctx->d_lz_scratch); ctx->d_lz_scratch = nullptr; ctx->lz_scratch_words = ctx->lz_scratch_asked = 0;
        size_t free_b = 0, total_b = 0;
        cudaMemGetInfo(&free_b, &total_b);
        warps = std::min<uint64_t>(warps, (uint64_t)free_b * 9 / 10 / (stride * 4));
        while (warps > 0 && cudaMalloc((void **)&ctx->d_lz_scratch, warps * stride * 4) != cudaSuccess) {
            cudaGetLastError();
            ctx->d_lz_scratch = nullptr;
            warps /= 2;
        }
        if (warps == 0) {
            char buf[200];
            snprintf(buf, sizeof buf, "divans_b200: cannot allocate the LZ77 scratch of one warp for streams of up to %llu bytes: %llu bytes",
                     (unsigned long long)max_in_len, (unsigned long long)stride * 4);
            ctx->err = buf;
            return DIVANS_FAILURE;
        }
        ctx->lz_scratch_words = warps * stride;
        ctx->lz_scratch_asked = want;
    }
    warps = std::min<uint64_t>(warps, ctx->lz_scratch_words / stride);
    if (!ctx->d_lz_pm) CK(cudaMalloc((void **)&ctx->d_lz_pm, PM_RECORD_BYTES));
    if (ctx->busy_recorded) CK(cudaStreamWaitEvent(st, ctx->ev_busy, 0));
    // the record of lz77_blob: pred_mode and mixing_value stored as bytes
    std::vector<uint8_t> &pm = ctx->h_pm;
    pm.assign(PM_RECORD_BYTES, 0);
    raw_record(pm.data(), pred_mode, mixing_value);
    CK(cudaMemcpyAsync(ctx->d_lz_pm, pm.data(), PM_RECORD_BYTES, cudaMemcpyHostToDevice, st));
    Lz77Params lp;
    lp.in = d_in; lp.in_off = d_in_off; lp.in_len = d_in_len; lp.max_in_len = max_in_len;
    lp.blobs = d_blobs; lp.blob_off = d_blob_off; lp.blob_cap = d_blob_cap; lp.blob_len = d_blob_len; lp.status = d_status;
    lp.pm = ctx->d_lz_pm; lp.n_streams = (uint32_t)n; lp.window = window;
    lp.work_counter = ctx->d_counter; lp.scratch = ctx->d_lz_scratch; lp.stride = stride; lp.n_warps = (uint32_t)warps;
    CK(cudaMemsetAsync(ctx->d_counter, 0, 4, st));
    CK(cudaEventRecord(ctx->ev0, st));
    CK(cudaEventRecord(ctx->evm, st));
    launch_lz77_cmds(lp, st);
    CK(cudaEventRecord(ctx->ev1, st));
    CK(cudaEventRecord(ctx->ev_busy, st)); ctx->busy_recorded = true;
    ctx->main_end_is_evm1 = false;
    ctx->launches += 1;
    CK(cudaGetLastError());
    return DIVANS_SUCCESS;
} catch (...) {
    if (ctx) ctx->err = "divans_b200: out of host memory";
    return DIVANS_FAILURE;
}

// =================================================================================================================
// reference FFI surface (src/ffi/mod.rs).  Streaming contract on top of batch-of-one GPU calls.
// =================================================================================================================
static divans_b200_ctx *g_shared_ctx = nullptr;
static std::mutex g_shared_mu;
static divans_b200_ctx *shared_ctx() {
    std::lock_guard<std::mutex> lk(g_shared_mu);
    if (!g_shared_ctx) {
        int dev = 0;
        const char *e = getenv("DIVANS_B200_DEVICE");
        if (e) dev = atoi(e);
        g_shared_ctx = divans_b200_create(dev, 0, 0);
    }
    return g_shared_ctx;
}

struct HostAlloc {   // CAllocator or malloc (ffi/alloc_util.rs:70-99: memory is zero-initialised)
    CAllocator a{nullptr, nullptr, nullptr};
    void *alloc(size_t n) {
        void *p = a.alloc_func ? a.alloc_func(a.opaque, n) : malloc(n);
        if (p) memset(p, 0, n);
        return p;
    }
    void free(void *p) { if (!p) return; if (a.free_func) a.free_func(a.opaque, p); else ::free(p); }
};

// Growable byte buffer whose storage comes from the state's allocator (the reference routes every allocation through the
// CAllocator, ffi/alloc_util.rs:70-99: a NO_MALLOC client -- c/custom_alloc.h -- must never see a malloc from us).
// Growth is geometric and frees the old block after the copy; a bump arena that only reclaims LIFO still bounds the total at
// about 3x the final size.
struct ByteBuf {
    HostAlloc *al = nullptr; uint8_t *p = nullptr; size_t n = 0, cap = 0;
    bool reserve(size_t want) {
        if (want <= cap) return true;
        size_t nc = cap ? cap : 4096;
        while (nc < want) { if (nc > ((size_t)1 << 62)) return false; nc *= 2; }
        uint8_t *q = (uint8_t *)al->alloc(nc);
        if (!q) return false;
        if (n) memcpy(q, p, n);
        al->free(p); p = q; cap = nc;
        return true;
    }
    bool append(const uint8_t *src, size_t m) { if (!reserve(n + m)) return false; if (m) memcpy(p + n, src, m); n += m; return true; }
    bool resize(size_t m) { if (!reserve(m)) return false; n = m; return true; }
    void release() { al->free(p); p = nullptr; n = cap = 0; }
    size_t size() const { return n; }
    uint8_t *data() { return p; }
    uint8_t operator[](size_t i) const { return p[i]; }
};

// A reference built with `--features blend` uses BlendCDF16 everywhere (src/interface.rs:146-147); a deployment that replaces such
// a build says so once, through the environment of the process that loads this library: DIVANS_B200_FFI_CDF=blend.
static bool ffi_cdf_blend() {
    static const bool b = [] { const char *e = getenv("DIVANS_B200_FFI_CDF"); return e && strcmp(e, "blend") == 0; }();
    return b;
}
struct DivansDecompressorState {
    HostAlloc al;
    bool self_in_custom = false;
    uint8_t skip_crc = 0;
    ByteBuf inbuf;                            // buffered compressed stream
    ByteBuf outbuf;                           // decoded stream waiting to be handed out
    size_t out_cursor = 0;
    // incremental framing scan (host): how far the record chain has been walked
    size_t scan_pos = 16; bool saw_eof = false; size_t total_len = 0; bool decoded = false; bool failed = false;
};

static DivansDecompressorState *new_decomp(CAllocator a, uint8_t skip_crc) {
    DivansDecompressorState *s;
    if (a.alloc_func) {
        void *mem = a.alloc_func(a.opaque, sizeof(DivansDecompressorState));
        if (!mem) return nullptr;
        s = new (mem) DivansDecompressorState();
        s->self_in_custom = true;
    } else s = new (std::nothrow) DivansDecompressorState();
    if (!s) return nullptr;
    s->al.a = a; s->skip_crc = skip_crc;
    s->inbuf.al = &s->al; s->outbuf.al = &s->al;
    if (!shared_ctx()) { s->failed = true; }
    return s;
}
extern "C" DivansDecompressorState *divans_new_decompressor(void) { return new_decomp(CAllocator{nullptr, nullptr, nullptr}, 0); }
extern "C" DivansDecompressorState *divans_new_serial_decompressor(void) { return new_decomp(CAllocator{nullptr, nullptr, nullptr}, 0); }
extern "C" DivansDecompressorState *divans_new_decompressor_with_custom_alloc(CAllocator alloc, uint8_t skip_crc, uint8_t /*multithread*/) {
    return new_decomp(alloc, skip_crc);
}
extern "C" void divans_free_decompressor(DivansDecompressorState *s) {
    if (!s) return;
    s->outbuf.release(); s->inbuf.release();
    if (s->self_in_custom) { HostAlloc al = s->al; s->~DivansDecompressorState(); al.free(s); }
    else delete s;
}
extern "C" uint8_t *divans_decompressor_malloc_u8(DivansDecompressorState *s, size_t n) { return (uint8_t *)s->al.alloc(n); }
extern "C" void divans_decompressor_free_u8(DivansDecompressorState *s, uint8_t *p, size_t) { s->al.free(p); }
extern "C" size_t *divans_decompressor_malloc_usize(DivansDecompressorState *s, size_t n) { return (size_t *)s->al.alloc(n * sizeof(size_t)); }
extern "C" void divans_decompressor_free_usize(DivansDecompressorState *s, size_t *p, size_t) { s->al.free(p); }

// walk record headers over what has been buffered so far; sets saw_eof/total_len once the EOF marker is visible
static int scan_frames(DivansDecompressorState *s) {
    const ByteBuf &b = s->inbuf;
    if (b.size() < 16) return 0;
    if (b[0] != 0xff || b[1] != 0xe5 || b[2] != 0x8c || b[3] != 0x9f) return -1;
    if (b[5] < 10 || b[5] >= 25) return -1;
    while (!s->saw_eof) {
        size_t pos = s->scan_pos;
        if (pos >= b.size()) return 0;
        uint8_t h = b[pos];
        if (h == 0xff) {
            if (pos + 3 > b.size()) return 0;
            if (b[pos + 1] != 0xfe || b[pos + 2] != 0xff) return -1;
            s->saw_eof = true; s->total_len = pos + 3 + 8;
            break;
        }
        size_t len, hdr;
        if (h < 16) { if (pos + 3 > b.size()) return 0; len = ((size_t)b[pos + 1] | ((size_t)b[pos + 2] << 8)) + 1; hdr = 3; }
        else { unsigned k = h >> 4; if (k > 3) return -1; len = (size_t)1024 << (k << 1); hdr = 1; }
        s->scan_pos = pos + hdr + len;   // may point beyond what is buffered; resolved when more input arrives
    }
    return 1;
}

extern "C" DivansResult divans_decode(DivansDecompressorState *s, const uint8_t *input_buf_ptr, size_t input_size, size_t *input_offset,
                                      uint8_t *output_buf_ptr, size_t output_size, size_t *output_offset) {
    if (!s || !input_offset || !output_offset) return DIVANS_FAILURE;   // ffi/mod.rs:241-262
    if (s->failed) return DIVANS_FAILURE;
    if (!s->decoded) {
        // take input until the whole stream (through the 8-byte trailer) is buffered
        while (*input_offset < input_size) {
            size_t want;
            if (s->saw_eof) want = s->total_len - s->inbuf.size();
            else {
                size_t have = s->inbuf.size();
                size_t target = have < 16 ? 16 : (s->scan_pos + 3 > have ? s->scan_pos + 3 : have + 1);
                want = target - have;
            }
            if (want == 0) break;
            size_t avail = input_size - *input_offset;
            size_t take = want < avail ? want : avail;
            if (!s->inbuf.append(input_buf_ptr + *input_offset, take)) { s->failed = true; return DIVANS_FAILURE; }
            *input_offset += take;
            int sc = scan_frames(s);
            if (sc < 0) { s->failed = true; return DIVANS_FAILURE; }
            if (s->saw_eof && s->inbuf.size() >= s->total_len) break;
        }
        if (!(s->saw_eof && s->inbuf.size() >= s->total_len)) return DIVANS_NEEDS_MORE_INPUT;
        divans_b200_ctx *ctx = shared_ctx();
        if (!ctx) { s->failed = true; return DIVANS_FAILURE; }
        // The output size is not in the header: start from a guess and grow on NEEDS_MORE_OUTPUT.  Growth is bounded by the
        // largest output a divANS stream of this size can describe per coded nibble (a copy command of 2^24 - 1 bytes
        // costs >= 3 nibbles of the command coder), by DIVANS_B200_MAX_OUTPUT (default 2^32) and by what the allocator
        // hands out: a decompression bomb ends in DIVANS_FAILURE, not in an exception crossing the C boundary.
        static const size_t max_out = []() { const char *e = getenv("DIVANS_B200_MAX_OUTPUT"); return e ? (size_t)strtoull(e, nullptr, 0) : ((size_t)1 << 32); }();
        size_t cap = s->inbuf.size() * 8 + (1 << 16);
        for (;;) {
            if (cap > max_out) cap = max_out;
            if (!s->outbuf.resize(cap)) { s->failed = true; return DIVANS_FAILURE; }
            uint64_t in_off = 0, in_len = s->inbuf.size(), out_off = 0, out_cap = cap, out_len = 0; int32_t status = DIVANS_FAILURE;
            DivansResult r = divans_b200_decode_batch_host(ctx, 1, s->inbuf.data(), &in_off, &in_len, s->outbuf.data(), &out_off, &out_cap,
                                                           &out_len, &status, (s->skip_crc ? DIVANS_B200_FLAG_SKIP_CRC : 0u) | (ffi_cdf_blend() ? DIVANS_B200_FLAG_CDF_BLEND : 0u));
            if (r != DIVANS_SUCCESS) { s->failed = true; return DIVANS_FAILURE; }
            if (status == DIVANS_NEEDS_MORE_OUTPUT && cap < max_out) { s->outbuf.release(); cap *= 4; continue; }
            if (status != DIVANS_SUCCESS) { s->failed = true; return DIVANS_FAILURE; }
            s->outbuf.n = out_len;
            break;
        }
        s->decoded = true;
        // (the input buffer is kept until free: a LIFO arena could not reclaim it from under the output buffer anyway)
    }
    size_t remaining = s->outbuf.size() - s->out_cursor;
    size_t room = output_size - *output_offset;
    size_t give = remaining < room ? remaining : room;
    if (give) memcpy(output_buf_ptr + *output_offset, s->outbuf.data() + s->out_cursor, give);
    s->out_cursor += give; *output_offset += give;
    return s->out_cursor == s->outbuf.size() ? DIVANS_SUCCESS : DIVANS_NEEDS_MORE_OUTPUT;
}

// ---- compressor side ----
struct DivansCompressorState {
    HostAlloc al;
    bool self_in_custom = false;
    divans_b200_encode_options opts;
    int use_brotli = 1;
    bool started = false, flushed = false, failed = false;
    ByteBuf inbuf, outbuf;
    size_t out_cursor = 0;
};
extern "C" DivansCompressorState *divans_new_compressor_with_custom_alloc(CAllocator a) {
    DivansCompressorState *s;
    if (a.alloc_func) {
        void *mem = a.alloc_func(a.opaque, sizeof(DivansCompressorState));
        if (!mem) return nullptr;
        s = new (mem) DivansCompressorState(); s->self_in_custom = true;
    } else s = new (std::nothrow) DivansCompressorState();
    if (!s) return nullptr;
    s->al.a = a;
    divans_b200_encode_options_default(&s->opts);
    s->opts.dynamic_context_mixing = 1;   // DivansCompressorOptions::default(), src/interface.rs:462-484
    s->opts.cdf_model = ffi_cdf_blend() ? DIVANS_B200_CDF_BLEND : DIVANS_B200_CDF_FREQUENTIST;
    s->inbuf.al = &s->al; s->outbuf.al = &s->al;
    return s;
}
extern "C" DivansCompressorState *divans_new_compressor(void) { return divans_new_compressor_with_custom_alloc(CAllocator{nullptr, nullptr, nullptr}); }
extern "C" void divans_free_compressor(DivansCompressorState *s) {
    if (!s) return;
    s->outbuf.release(); s->inbuf.release();
    if (s->self_in_custom) { HostAlloc al = s->al; s->~DivansCompressorState(); al.free(s); }
    else delete s;
}
extern "C" uint8_t *divans_compressor_malloc_u8(DivansCompressorState *s, size_t n) { return (uint8_t *)s->al.alloc(n); }
extern "C" void divans_compressor_free_u8(DivansCompressorState *s, uint8_t *p, size_t) { s->al.free(p); }
extern "C" size_t *divans_compressor_malloc_usize(DivansCompressorState *s, size_t n) { return (size_t *)s->al.alloc(n * sizeof(size_t)); }
extern "C" void divans_compressor_free_usize(DivansCompressorState *s, size_t *p, size_t) { s->al.free(p); }

static const int16_t kPalette[15][2] = {   // Speed::ENCODER_DEFAULT_PALETTE, probability/interface.rs:303-320
    {0, 1024}, {2, 1024}, {1, 128}, {1, 16384}, {2, 2048}, {4, 1024}, {8, 8192}, {16, 48}, {16, 8192}, {32, 4096},
    {64, 16384}, {128, 256}, {128, 16384}, {512, 16384}, {1664, 16384}};
extern "C" DivansResult divans_set_option(DivansCompressorState *s, DivansOptionSelect selector, uint32_t value) {
    if (!s || s->started) return DIVANS_FAILURE;   // options only in the OptionStage, ffi/compressor.rs:63-166
    divans_b200_encode_options &o = s->opts;
    auto set_adapt = [&](int idx) -> DivansResult {
        if (value >= 15) return DIVANS_FAILURE;
        if (!o.have_literal_adaptation) { o.have_literal_adaptation = 1; for (int k = 0; k < 4; k++) { o.literal_adaptation[k][0] = kPalette[value][0]; o.literal_adaptation[k][1] = kPalette[value][1]; } }
        else { o.literal_adaptation[idx][0] = kPalette[value][0]; o.literal_adaptation[idx][1] = kPalette[value][1]; }
        return DIVANS_SUCCESS;
    };
    switch (selector) {
    case DIVANS_OPTION_QUALITY: case DIVANS_OPTION_LGBLOCK: case DIVANS_OPTION_STRIDE_DETECTION_QUALITY:
    case DIVANS_OPTION_PRIOR_BITMASK_DETECTION: case DIVANS_OPTION_SPEED_DETECTION_QUALITY: case DIVANS_OPTION_BROTLI_LITERAL_BYTE_SCORE:
    case DIVANS_OPTION_Q9_5: case DIVANS_OPTION_IR_OPTIMIZER:
        return DIVANS_SUCCESS;   // command-selection knobs of the brotli crate: accepted, no effect on the entropy half
    case DIVANS_OPTION_WINDOW_SIZE: o.window_size = (int32_t)value; return DIVANS_SUCCESS;
    case DIVANS_OPTION_DYNAMIC_CONTEXT_MIXING: o.dynamic_context_mixing = (int32_t)(value & 0xff); return DIVANS_SUCCESS;
    case DIVANS_OPTION_USE_BROTLI_COMMAND_SELECTION: if (value > 2) return DIVANS_FAILURE; s->use_brotli = (int)value; return DIVANS_SUCCESS;
    case DIVANS_OPTION_USE_BROTLI_BITSTREAM: if (value != 1) return DIVANS_FAILURE; s->use_brotli = 2; return DIVANS_SUCCESS;
    case DIVANS_OPTION_USE_CONTEXT_MAP: if (value > 1) return DIVANS_FAILURE; o.use_context_map = (int32_t)value; return DIVANS_SUCCESS;
    case DIVANS_OPTION_FORCE_STRIDE_VALUE: if (value > 8) return DIVANS_FAILURE; o.force_stride = (int32_t)value; return DIVANS_SUCCESS;
    case DIVANS_OPTION_LITERAL_ADAPTATION_STRIDE_HIGH: return set_adapt(1);
    case DIVANS_OPTION_LITERAL_ADAPTATION_CM_HIGH: return set_adapt(3);
    case DIVANS_OPTION_LITERAL_ADAPTATION_STRIDE_LOW: return set_adapt(0);
    case DIVANS_OPTION_LITERAL_ADAPTATION_CM_LOW: return set_adapt(2);
    case DIVANS_OPTION_PRIOR_DEPTH: o.prior_depth = (int32_t)(value & 0xff); return DIVANS_SUCCESS;
    case DIVANS_OPTION_FORCE_LITERAL_CONTEXT_MODE: o.literal_pred_mode = (int32_t)(value & 0xff); return DIVANS_SUCCESS;
    default: return DIVANS_FAILURE;
    }
}
extern "C" DivansResult divans_encode(DivansCompressorState *s, const uint8_t *input_buf_ptr, size_t input_size, size_t *input_offset,
                                      uint8_t *, size_t, size_t *output_offset) {
    if (!s || !input_offset || !output_offset) return DIVANS_FAILURE;
    if (s->failed || s->flushed) return DIVANS_FAILURE;
    s->started = true;
    if (!s->inbuf.append(input_buf_ptr + *input_offset, input_size - *input_offset)) { s->failed = true; return DIVANS_FAILURE; }
    *input_offset = input_size;
    return DIVANS_NEEDS_MORE_INPUT;   // like the reference: all input consumed, nothing is "done" before flush
}
extern "C" DivansResult divans_encode_flush(DivansCompressorState *s, uint8_t *output_buf_ptr, size_t output_size, size_t *output_offset) {
    if (!s || !output_offset) return DIVANS_FAILURE;
    if (s->failed) return DIVANS_FAILURE;
    s->started = true;
    if (!s->flushed) {
        divans_b200_ctx *ctx = shared_ctx();
        if (!ctx) { s->failed = true; return DIVANS_FAILURE; }
        size_t cap = s->inbuf.size() + s->inbuf.size() / 2 + 70000;
        if (!s->outbuf.resize(cap)) { s->failed = true; return DIVANS_FAILURE; }
        uint64_t in_off = 0, in_len = s->inbuf.size(), out_off = 0, out_cap = cap, out_len = 0; int32_t status = DIVANS_FAILURE;
        static const uint8_t none = 0;
        DivansResult r = divans_b200_encode_batch_host(ctx, 1, in_len ? s->inbuf.data() : &none, &in_off, &in_len, s->outbuf.data(), &out_off, &out_cap, &out_len,
                                                       &status, &s->opts);
        if (r != DIVANS_SUCCESS || status != DIVANS_SUCCESS) { s->failed = true; return DIVANS_FAILURE; }
        s->outbuf.n = out_len;
        s->flushed = true;
    }
    size_t remaining = s->outbuf.size() - s->out_cursor, room = output_size - *output_offset;
    size_t give = remaining < room ? remaining : room;
    if (give) memcpy(output_buf_ptr + *output_offset, s->outbuf.data() + s->out_cursor, give);
    s->out_cursor += give; *output_offset += give;
    return s->out_cursor == s->outbuf.size() ? DIVANS_SUCCESS : DIVANS_NEEDS_MORE_OUTPUT;
}
