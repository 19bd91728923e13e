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
    uint8_t *d_in = nullptr; size_t d_in_cap = 0;
    uint8_t *d_out = nullptr; size_t d_out_cap = 0;
    uint64_t *d_meta = nullptr; size_t d_meta_cap = 0;   // in_off,in_len,out_off,out_cap,out_len (+status)
    // pipelined host API (decode_batch_host_async): two batches in flight, copies on their own streams
    struct Lane {
        uint8_t *d_in = nullptr; size_t d_in_cap = 0;
        uint8_t *d_out = nullptr; size_t d_out_cap = 0;
        uint64_t *d_meta = nullptr; size_t d_meta_cap = 0;
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
    cudaFree(ctx->d_frame); cudaFree(ctx->d_payload); cudaFree(ctx->d_in); cudaFree(ctx->d_out); cudaFree(ctx->d_meta);
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    if (ctx->evm) cudaEventDestroy(ctx->evm);
    if (ctx->evm1) cudaEventDestroy(ctx->evm1);
    if (ctx->ev_busy) cudaEventDestroy(ctx->ev_busy);
    cudaFree(ctx->d_sf); cudaFree(ctx->d_replay); cudaFree(ctx->d_enc_scratch); cudaFree(ctx->d_pm_internal); cudaFree(ctx->d_rcp15);
    for (auto &ln : ctx->lane) {
        cudaFree(ln.d_in); cudaFree(ln.d_out); cudaFree(ln.d_meta);
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
#define DV_KERNEL_VERSION "r2.17-v2-t2s-loop"
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
static DivansResult decode_device_nolock(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                         const uint64_t *d_in_len, uint8_t *d_out, const uint64_t *d_out_off,
                                         const uint64_t *d_out_cap, uint64_t *d_out_len, int32_t *d_status,
                                         uint64_t in_total_bytes, uint32_t flags, void *cuda_stream) {
    if (n > 0xffffffffull) { ctx->err = "too many streams"; return DIVANS_FAILURE; }
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
    if (ctx->busy_recorded) CK(cudaStreamWaitEvent(st, ctx->ev_busy, 0));
    int lanes = ctx->lanes_per_stream;
    uint32_t gpb, cap;
    const bool blend = (flags & DIVANS_B200_FLAG_CDF_BLEND) != 0;   // BlendCDF16 streams: the blend decoder (dv_kernels.cu), 16 lanes
    if (blend) {
        lanes = 16; gpb = (uint32_t)(DECODE_BLOCK_THREADS / 16);
        cap = (uint32_t)ctx->sm_count * (uint32_t)std::max(1, decode_max_blocks_per_sm16_blend()) * gpb;
        if (cap > ctx->max_resident) cap = std::max(ctx->max_resident / gpb * gpb, gpb);   // (memory / caller limits of the context)
    } else {
        // 16 lanes per stream unless 8 hold the batch in fewer passes.  At equal residency 8 lanes is the slower layout (half the
        // warps per scheduler); it only pays where registers, not slot memory, cap residency: there it keeps twice the streams in
        // flight.  On an 80 GB H100 both layouts are capped by slot memory (cap8 ~ cap16), so 16 lanes run every batch size.
        if (ctx->auto_lanes) {
            const uint64_t passes16 = (n + ctx->cap16 - 1) / ctx->cap16, passes8 = (n + ctx->cap8 - 1) / ctx->cap8;
            lanes = passes8 < passes16 ? 8 : 16;
        }
        gpb = (uint32_t)decode_groups_per_block_v2(lanes); cap = lanes == 16 ? ctx->cap16 : ctx->cap8;
    }
    ctx->last_lanes = lanes;
    uint32_t resident = (uint32_t)(n < cap ? n : cap);
    uint32_t blocks = (resident + gpb - 1) / gpb;
    if (ensure_arena(ctx, (size_t)blocks * gpb) != DIVANS_SUCCESS) return DIVANS_FAILURE;
    if (!grow(ctx, &ctx->d_frame, &ctx->frame_cap, 4 * n)) return DIVANS_FAILURE;
    if (!grow(ctx, &ctx->d_payload, &ctx->payload_cap, (size_t)in_total_bytes + 48 * n + 64)) return DIVANS_FAILURE;
    CK(cudaMemsetAsync(ctx->d_counter, 0, 4, st));
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
    if (!skip_decode) { if (blend) launch_decode16_blend(dp, blocks, st); else launch_decode_v2(lanes, dp, blocks, st); }
    if (dbg) { CK(cudaStreamSynchronize(st)); fprintf(stderr, "divans_b200[debug]: decode kernel ok (blocks=%u, lps=%d)\n", blocks, ctx->lanes_per_stream); }
    CK(cudaEventRecord(ctx->ev1, st));
    CK(cudaEventRecord(ctx->ev_busy, st)); ctx->busy_recorded = true;
    ctx->main_end_is_evm1 = false;
    ctx->launches += skip_decode ? 3 : 4;
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

extern "C" DivansResult divans_b200_decode_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                                      const uint64_t *in_len, uint8_t *out, const uint64_t *out_off,
                                                      const uint64_t *out_cap, uint64_t *out_len, int32_t *status, uint32_t flags) {
    if (!ctx) return DIVANS_FAILURE;
    if (n == 0) return DIVANS_SUCCESS;
    std::lock_guard<std::mutex> lk(ctx->mu);
    CK(cudaSetDevice(ctx->device));
    // extent of the input / output blobs
    uint64_t in_end = 0, out_end = 0, in_sum = 0;
    for (size_t i = 0; i < n; i++) {
        if (in_off[i] + in_len[i] > in_end) in_end = in_off[i] + in_len[i];
        if (out_off[i] + out_cap[i] > out_end) out_end = out_off[i] + out_cap[i];
        in_sum += in_len[i];                       // input regions may alias (the same stream decoded n times)
    }
    if (!grow(ctx, &ctx->d_in, &ctx->d_in_cap, (size_t)in_end + 64)) return DIVANS_FAILURE;
    if (!grow(ctx, &ctx->d_out, &ctx->d_out_cap, (size_t)out_end + 64)) return DIVANS_FAILURE;
    if (!grow(ctx, &ctx->d_meta, &ctx->d_meta_cap, n * 6)) return DIVANS_FAILURE;
    uint64_t *m = ctx->d_meta;
    cudaStream_t st = ctx->stream;
    CK(cudaMemcpyAsync(ctx->d_in, in, in_end, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(m, in_off, n * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(m + n, in_len, n * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(m + 2 * n, out_off, n * 8, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(m + 3 * n, out_cap, n * 8, cudaMemcpyHostToDevice, st));
    int32_t *d_status = reinterpret_cast<int32_t *>(m + 5 * n);
    CK(cudaMemsetAsync(ctx->d_out, 0, out_end, st));   // what the regions hold past out_len[i] is zeros, not an earlier batch
    DivansResult r = decode_device_nolock(ctx, n, ctx->d_in, m, m + n, ctx->d_out, m + 2 * n, m + 3 * n, m + 4 * n, d_status,
                                          in_sum > in_end ? in_sum : in_end, flags, st);
    if (r != DIVANS_SUCCESS) return r;
    CK(cudaMemcpyAsync(out_len, m + 4 * n, n * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(status, d_status, n * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    // Copy back whole regions (zeros past out_len[i]: d_out was cleared before the kernels) and never a byte outside a declared
    // region out[out_off[i] .. +out_cap[i]): consecutive streams whose regions are exactly adjacent share one transfer.
    for (size_t i = 0; i < n;) {
        const uint64_t lo = out_off[i]; uint64_t hi = lo + out_cap[i];
        size_t j = i + 1;
        while (j < n && out_off[j] == hi) { hi += out_cap[j]; j++; }
        if (hi > lo) CK(cudaMemcpyAsync(out + lo, ctx->d_out + lo, hi - lo, cudaMemcpyDeviceToHost, st));
        i = j;
    }
    CK(cudaStreamSynchronize(st));
    return DIVANS_SUCCESS;
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
    uint64_t in_end = 0, in_sum = 0, out_lo = ~0ull, out_hi = 0;
    for (size_t i = 0; i < n; i++) {
        if (in_off[i] + in_len[i] > in_end) in_end = in_off[i] + in_len[i];
        if (out_off[i] < out_lo) out_lo = out_off[i];
        if (out_off[i] + out_cap[i] > out_hi) out_hi = out_off[i] + out_cap[i];
        in_sum += in_len[i];
    }
    // (re)allocation of a lane's buffers synchronises the device: only while the pipeline warms up
    if (!grow(ctx, &ln.d_in, &ln.d_in_cap, (size_t)in_end + 64)) return DIVANS_FAILURE;
    if (!grow(ctx, &ln.d_out, &ln.d_out_cap, (size_t)out_hi + 64)) return DIVANS_FAILURE;
    if (!grow(ctx, &ln.d_meta, &ln.d_meta_cap, n * 6)) return DIVANS_FAILURE;
    if (ln.h_res_cap < n * 12) {
        if (ln.h_res) cudaFreeHost(ln.h_res);
        ln.h_res = nullptr; ln.h_res_cap = 0;
        CK(cudaMallocHost((void **)&ln.h_res, n * 12 + 64));
        ln.h_res_cap = n * 12 + 64;
    }
    ln.u_out_len = out_len; ln.u_status = status; ln.n = n;
    uint64_t *m = ln.d_meta;
    CK(cudaMemcpyAsync(ln.d_in, in, in_end, cudaMemcpyHostToDevice, ctx->s_h2d));
    CK(cudaMemcpyAsync(m, in_off, n * 8, cudaMemcpyHostToDevice, ctx->s_h2d));
    CK(cudaMemcpyAsync(m + n, in_len, n * 8, cudaMemcpyHostToDevice, ctx->s_h2d));
    CK(cudaMemcpyAsync(m + 2 * n, out_off, n * 8, cudaMemcpyHostToDevice, ctx->s_h2d));
    CK(cudaMemcpyAsync(m + 3 * n, out_cap, n * 8, cudaMemcpyHostToDevice, ctx->s_h2d));
    CK(cudaEventRecord(ln.e_in, ctx->s_h2d));
    CK(cudaStreamWaitEvent(ctx->stream, ln.e_in, 0));
    int32_t *d_status = reinterpret_cast<int32_t *>(m + 5 * n);
    // the regions are copied back whole (out_len is not known yet): zero them first so that the bytes past out_len are
    // zeros, not plaintext of an earlier batch
    if (out_hi > out_lo) CK(cudaMemsetAsync(ln.d_out + out_lo, 0, out_hi - out_lo, ctx->stream));
    DivansResult r = decode_device_nolock(ctx, n, ln.d_in, m, m + n, ln.d_out, m + 2 * n, m + 3 * n, m + 4 * n, d_status,
                                          in_sum > in_end ? in_sum : in_end, flags, ctx->stream);
    if (r != DIVANS_SUCCESS) return r;
    CK(cudaEventRecord(ln.e_k, ctx->stream));
    CK(cudaStreamWaitEvent(ctx->s_d2h, ln.e_k, 0));
    CK(cudaMemcpyAsync(ln.h_res, m + 4 * n, n * 8, cudaMemcpyDeviceToHost, ctx->s_d2h));
    CK(cudaMemcpyAsync(ln.h_res + n * 8, d_status, n * 4, cudaMemcpyDeviceToHost, ctx->s_d2h));
    // one transfer per run of exactly adjacent regions: nothing outside out[out_off[i] .. +out_cap[i]) is written
    for (size_t i = 0; i < n;) {
        const uint64_t lo = out_off[i]; uint64_t hi = lo + out_cap[i];
        size_t j = i + 1;
        while (j < n && out_off[j] == hi) { hi += out_cap[j]; j++; }
        if (hi > lo) CK(cudaMemcpyAsync(out + lo, ln.d_out + lo, hi - lo, cudaMemcpyDeviceToHost, ctx->s_d2h));
        i = j;
    }
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

// One launch set over n streams whose inputs/outputs already sit in HBM.  `cmd_cap`/`lit_cap`: log entries per stream,
// `replay_stride`: bytes of replay window per resident slot.
static DivansResult encode_device_internal(divans_b200_ctx *ctx, size_t n, int raw_mode, const uint8_t *d_in, const uint64_t *d_in_off,
                                           const uint64_t *d_in_len, uint32_t cmd_cap, uint32_t lit_cap, uint64_t replay_stride,
                                           uint8_t *d_out, const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len,
                                           int32_t *d_status, const divans_b200_encode_options *o, cudaStream_t st) {
    const size_t slots = encode_slots(ctx, n);
    const uint32_t blocks = (uint32_t)(slots / ENCODE_GROUPS_PER_BLOCK);
    if (ensure_arena(ctx, slots) != DIVANS_SUCCESS) return DIVANS_FAILURE;
    const uint32_t cmd_chunks = (cmd_cap + NUM_SYMBOLS_BEFORE_FLUSH - 1) / NUM_SYMBOLS_BEFORE_FLUSH;
    const uint32_t lit_chunks = (lit_cap + NUM_SYMBOLS_BEFORE_FLUSH - 1) / NUM_SYMBOLS_BEFORE_FLUSH;
    const uint32_t max_chunks = cmd_chunks + lit_chunks;
    if (!grow(ctx, &ctx->d_sf, &ctx->sf_cap, n * ((size_t)cmd_cap + lit_cap))) return DIVANS_FAILURE;
    if (!grow(ctx, &ctx->d_replay, &ctx->replay_cap, slots * (size_t)replay_stride)) return DIVANS_FAILURE;
    // small per-stream scratch: counts [2n] | dummy [slots] | chunk_w [n*max_chunks] | chunk_state [16*n*max_chunks]
    size_t words = 2 * n + slots + n * (size_t)max_chunks + 4 * n * (size_t)max_chunks + 16 + 2 * n * (size_t)max_chunks * (NUM_SYMBOLS_BEFORE_FLUSH / 64);
    if (!grow(ctx, &ctx->d_enc_scratch, &ctx->enc_scratch_cap, words)) return DIVANS_FAILURE;
    if (!ctx->d_pm_internal) CK(cudaMalloc((void **)&ctx->d_pm_internal, PM_RECORD_BYTES));
    if (!ctx->d_rcp15) { CK(cudaMalloc((void **)&ctx->d_rcp15, 32768 * sizeof(uint64_t))); launch_rcp15_init(ctx->d_rcp15, st); ctx->launches += 1; }
    if (raw_mode) {
        // raw_to_cmd/mod.rs:116-143: 64-entry identity literal map, 4 distance entries, one mixing value, speeds unset
        std::vector<uint8_t> &pm = ctx->h_pm;
        pm.assign(PM_RECORD_BYTES, 0);
        pm[0] = (uint8_t)o->literal_pred_mode; pm[2] = 1;
        pm[28] = 64; pm[30] = 4;
        for (int i = 0; i < 64; i++) pm[32 + i] = (uint8_t)i;
        for (int i = 0; i < 4; i++) pm[32 + 16384 + i] = (uint8_t)i;
        memset(pm.data() + 32 + 16384 + 1024, o->literal_mixing_value, 8192);
        CK(cudaMemcpyAsync(ctx->d_pm_internal, pm.data(), PM_RECORD_BYTES, cudaMemcpyHostToDevice, st));
    }
    EncodeParams ep;
    ep.in = d_in; ep.in_off = d_in_off; ep.in_len = d_in_len; ep.raw_mode = raw_mode; ep.n_streams = (uint32_t)n;
    ep.work_counter = ctx->d_counter; ep.arena = ctx->d_arena; ep.tables = ctx->d_tables; ep.pm_internal = ctx->d_pm_internal;
    ep.sf = ctx->d_sf; ep.cmd_cap = cmd_cap; ep.lit_cap = lit_cap;
    uint32_t *w = ctx->d_enc_scratch;
    ep.sf_counts = w; w += 2 * n;
    ep.sf_dummy = w; w += slots;
    ep.chunk_w = w; w += n * (size_t)max_chunks;
    w = reinterpret_cast<uint32_t *>(((uintptr_t)w + 15) & ~(uintptr_t)15);
    ep.chunk_state = reinterpret_cast<uint8_t *>(w);
    ep.emit_bits = w + 4 * n * (size_t)max_chunks;
    ep.rcp15 = ctx->d_rcp15;
    ep.replay = ctx->d_replay; ep.replay_stride = replay_stride;
    ep.max_chunks = max_chunks; ep.cmd_chunks = cmd_chunks;
    ep.out = d_out; ep.out_off = d_out_off; ep.out_cap = d_out_cap; ep.out_len = d_out_len; ep.status = d_status;
    int window = o->window_size < 10 ? 10 : (o->window_size > 24 ? 24 : o->window_size);
    ep.window_size = window; ep.dynamic_context_mixing = o->dynamic_context_mixing & 0xff; ep.prior_depth = o->prior_depth & 0xff;
    ep.use_context_map = o->use_context_map; ep.force_stride = o->force_stride; ep.have_literal_adaptation = o->have_literal_adaptation;
    for (int k = 0; k < 4; k++) ep.literal_adaptation[k] = pack_speed(o->literal_adaptation[k]);
    ep.model_rev = o->model_rev == DIVANS_B200_MODEL_WASM_2018 ? 1 : 0;
    if (ctx->busy_recorded) CK(cudaStreamWaitEvent(st, ctx->ev_busy, 0));
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

static uint32_t raw_cmd_cap(uint64_t max_len, int window) { return (uint32_t)(32 * (2 + (max_len >> window)) + 62000 + 64); }

extern "C" DivansResult divans_b200_encode_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                        const uint64_t *d_in_len, uint64_t max_in_len, uint8_t *d_out,
                                                        const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len,
                                                        int32_t *d_status, const divans_b200_encode_options *opts, void *cuda_stream) {
    if (!ctx || !opts) return DIVANS_FAILURE;
    if (n == 0) return DIVANS_SUCCESS;
    if (n > 0xffffffffull || max_in_len > 0x7fff0000ull) { ctx->err = "batch too large"; return DIVANS_FAILURE; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    CK(cudaSetDevice(ctx->device));
    int window = opts->window_size < 10 ? 10 : (opts->window_size > 24 ? 24 : opts->window_size);
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
    return encode_device_internal(ctx, n, 1, d_in, d_in_off, d_in_len, raw_cmd_cap(max_in_len, window), (uint32_t)(2 * max_in_len + 16),
                                  (max_in_len + 31) & ~15ull, d_out, d_out_off, d_out_cap, d_out_len, d_status, opts, st);
}

// host batch: marshal, split into sub-batches whose symbol logs fit in HBM, run, copy back
static DivansResult encode_host_common(divans_b200_ctx *ctx, size_t n, int raw_mode, const uint8_t *in, const uint64_t *in_off,
                                       const uint64_t *in_len, uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap,
                                       uint64_t *out_len, int32_t *status, const divans_b200_encode_options *opts) {
    if (!ctx || !opts) return DIVANS_FAILURE;
    if (n == 0) return DIVANS_SUCCESS;
    std::lock_guard<std::mutex> lk(ctx->mu);
    CK(cudaSetDevice(ctx->device));
    const int window = opts->window_size < 10 ? 10 : (opts->window_size > 24 ? 24 : opts->window_size);
    // per-stream requirements
    std::vector<uint64_t> s_off(n), need_cmd(n), need_lit(n), need_replay(n);
    std::vector<uint8_t> staged;   // command lists are re-based to 4-byte aligned offsets
    uint64_t in_end = 0;
    for (size_t i = 0; i < n; i++) {
        status[i] = DIVANS_FAILURE; out_len[i] = 0;
        if (raw_mode) {
            if (in_len[i] > 0x7fff0000ull) { ctx->err = "stream too large"; return DIVANS_FAILURE; }
            s_off[i] = in_off[i];
            need_cmd[i] = raw_cmd_cap(in_len[i], window); need_lit[i] = 2 * in_len[i] + 16; need_replay[i] = (in_len[i] + 31) & ~15ull;
            if (in_off[i] + in_len[i] > in_end) in_end = in_off[i] + in_len[i];
        } else {
            const uint8_t *b = in + in_off[i];
            uint32_t h[8] = {0};
            if (in_len[i] >= 32) memcpy(h, b, 32);
            uint64_t need = 32ull + 20ull * h[2] + (uint64_t)PM_RECORD_BYTES * h[3] + h[4];
            uint64_t lit = 0, rep = 0;
            if (in_len[i] >= 32 && h[0] == 0x4c435644u && h[1] == 1 && need <= in_len[i]) {
                for (uint32_t c = 0; c < h[2]; c++) {
                    uint32_t r[5]; memcpy(r, b + 32 + 20ull * c, 20);
                    if (r[0] == 1) rep += r[2];
                    else if (r[0] == 2) rep += 64;            // dictionary word + transform prefix/suffix
                    else if (r[0] == 3) { lit += r[2]; rep += r[2]; }
                }
            }
            if (lit > 0x7fff0000ull || rep > 0xfffffff0ull) { ctx->err = "stream too large"; return DIVANS_FAILURE; }
            need_cmd[i] = 32ull * h[2] + 62000ull * h[3] + 64; need_lit[i] = 2 * lit + 16; need_replay[i] = (rep + 31) & ~15ull;
            s_off[i] = (staged.size() + 3) & ~(size_t)3;
            staged.resize(s_off[i] + in_len[i]);
            if (in_len[i]) memcpy(staged.data() + s_off[i], b, in_len[i]);
            in_end = staged.size();
        }
    }
    const uint8_t *src = raw_mode ? in : staged.data();
    // the slots first: the symbol logs are sized from what is left (on an 80 GB GPU the slots take most of the memory)
    if (ensure_arena(ctx, encode_slots(ctx, n)) != DIVANS_SUCCESS) return DIVANS_FAILURE;
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    const uint64_t budget = (uint64_t)(free_b + ctx->sf_cap * 4) * 6 / 10;
    if (!grow(ctx, &ctx->d_in, &ctx->d_in_cap, (size_t)in_end + 64)) return DIVANS_FAILURE;
    cudaStream_t st = ctx->stream;
    CK(cudaMemcpyAsync(ctx->d_in, src, in_end, cudaMemcpyHostToDevice, st));
    size_t i0 = 0;
    while (i0 < n) {
        // grow the sub-batch while its uniform-capacity logs fit
        uint64_t mc = 0, ml = 0, mr = 0; size_t i1 = i0;
        while (i1 < n) {
            uint64_t c = need_cmd[i1] > mc ? need_cmd[i1] : mc, l = need_lit[i1] > ml ? need_lit[i1] : ml;
            if (i1 > i0 && (c + l) * 4 * (uint64_t)(i1 - i0 + 1) > budget) break;
            mc = c; ml = l; if (need_replay[i1] > mr) mr = need_replay[i1];
            i1++;
        }
        if (mc > 0xffffffffull || ml > 0xffffffffull) { ctx->err = "stream too large"; return DIVANS_FAILURE; }
        const size_t m = i1 - i0;
        uint64_t out_lo = ~0ull, out_hi = 0;
        for (size_t i = i0; i < i1; i++) { if (out_off[i] < out_lo) out_lo = out_off[i]; if (out_off[i] + out_cap[i] > out_hi) out_hi = out_off[i] + out_cap[i]; }
        if (!grow(ctx, &ctx->d_out, &ctx->d_out_cap, (size_t)(out_hi - out_lo) + 64)) return DIVANS_FAILURE;
        if (!grow(ctx, &ctx->d_meta, &ctx->d_meta_cap, m * 6)) return DIVANS_FAILURE;
        std::vector<uint64_t> rel(m);
        for (size_t i = 0; i < m; i++) rel[i] = out_off[i0 + i] - out_lo;
        uint64_t *mm = ctx->d_meta;
        CK(cudaMemcpyAsync(mm, s_off.data() + i0, m * 8, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(mm + m, in_len + i0, m * 8, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(mm + 2 * m, rel.data(), m * 8, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(mm + 3 * m, out_cap + i0, m * 8, cudaMemcpyHostToDevice, st));
        int32_t *d_status = reinterpret_cast<int32_t *>(mm + 5 * m);
        DivansResult r = encode_device_internal(ctx, m, raw_mode, ctx->d_in, mm, mm + m, (uint32_t)mc, (uint32_t)ml, mr, ctx->d_out, mm + 2 * m,
                                                mm + 3 * m, mm + 4 * m, d_status, opts, st);
        if (r != DIVANS_SUCCESS) return r;
        CK(cudaMemcpyAsync(out_len + i0, mm + 4 * m, m * 8, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(status + i0, d_status, m * 4, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        for (size_t i = i0; i < i1; i++) {
            if (status[i] == DIVANS_SUCCESS && out_len[i]) CK(cudaMemcpyAsync(out + out_off[i], ctx->d_out + (out_off[i] - out_lo), out_len[i], cudaMemcpyDeviceToHost, st));
        }
        CK(cudaStreamSynchronize(st));
        i0 = i1;
    }
    return DIVANS_SUCCESS;
}
extern "C" DivansResult divans_b200_encode_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                                      const uint64_t *in_len, uint8_t *out, const uint64_t *out_off,
                                                      const uint64_t *out_cap, uint64_t *out_len, int32_t *status,
                                                      const divans_b200_encode_options *opts) {
    // (host marshalling uses std::vector sized by the caller's arguments: no C++ exception may cross the C boundary)
    try { return encode_host_common(ctx, n, 1, in, in_off, in_len, out, out_off, out_cap, out_len, status, opts); }
    catch (...) { if (ctx) ctx->err = "divans_b200: out of host memory while marshalling the batch"; return DIVANS_FAILURE; }
}
extern "C" DivansResult divans_b200_encode_cmds_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *blobs, const uint64_t *blob_off,
                                                           const uint64_t *blob_len, uint8_t *out, const uint64_t *out_off,
                                                           const uint64_t *out_cap, uint64_t *out_len, int32_t *status,
                                                           const divans_b200_encode_options *opts) {
    try { return encode_host_common(ctx, n, 0, blobs, blob_off, blob_len, out, out_off, out_cap, out_len, status, opts); }
    catch (...) { if (ctx) ctx->err = "divans_b200: out of host memory while marshalling the batch"; return DIVANS_FAILURE; }
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
