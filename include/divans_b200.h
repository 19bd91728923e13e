/*
 * divans_b200.h -- C ABI of the H100-native divANS entropy engine (libdivans_b200.so).
 *
 * Two surfaces:
 *  (1) the reference's own C FFI, symbol for symbol (reference: src/ffi/mod.rs, c/divans/ffi.h), so a
 *      program written against libdivans links unchanged (c/example.c is the test client);
 *  (2) a batch extension (ours, additive) -- the shape the GPU wants: N independent streams per call,
 *      either from host buffers (end-to-end path, copies included) or device-resident.
 *
 * Every stream is decoded/encoded by hand-written sm_90a CUDA kernels; there is no CPU fallback:
 * if no CUDA device / context can be had, constructors return NULL and batch calls return
 * DIVANS_FAILURE after printing the CUDA error to stderr.
 */
#ifndef DIVANS_B200_H_
#define DIVANS_B200_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * (1) reference FFI surface
 * ------------------------------------------------------------------------------------------------ */
typedef uint8_t DivansResult;                     /* reference: src/ffi/interface.rs:8-12 */
#define DIVANS_SUCCESS ((uint8_t)0)
#define DIVANS_NEEDS_MORE_INPUT ((uint8_t)1)
#define DIVANS_NEEDS_MORE_OUTPUT ((uint8_t)2)
#define DIVANS_FAILURE ((uint8_t)3)

typedef uint8_t DivansOptionSelect;               /* reference: src/ffi/interface.rs:18-37 */
#define DIVANS_OPTION_QUALITY 1
#define DIVANS_OPTION_WINDOW_SIZE 2
#define DIVANS_OPTION_LGBLOCK 3
#define DIVANS_OPTION_DYNAMIC_CONTEXT_MIXING 4
#define DIVANS_OPTION_USE_BROTLI_COMMAND_SELECTION 5
#define DIVANS_OPTION_USE_BROTLI_BITSTREAM 6
#define DIVANS_OPTION_USE_CONTEXT_MAP 7
#define DIVANS_OPTION_LITERAL_ADAPTATION_CM_HIGH 8
#define DIVANS_OPTION_FORCE_STRIDE_VALUE 9
#define DIVANS_OPTION_STRIDE_DETECTION_QUALITY 10
#define DIVANS_OPTION_PRIOR_DEPTH 11
#define DIVANS_OPTION_LITERAL_ADAPTATION_STRIDE_HIGH 12
#define DIVANS_OPTION_LITERAL_ADAPTATION_CM_LOW 13
#define DIVANS_OPTION_LITERAL_ADAPTATION_STRIDE_LOW 14
#define DIVANS_OPTION_BROTLI_LITERAL_BYTE_SCORE 15
#define DIVANS_OPTION_SPEED_DETECTION_QUALITY 16
#define DIVANS_OPTION_PRIOR_BITMASK_DETECTION 17
#define DIVANS_OPTION_Q9_5 18
#define DIVANS_OPTION_FORCE_LITERAL_CONTEXT_MODE 19
#define DIVANS_OPTION_IR_OPTIMIZER 20

struct CAllocator {                               /* reference: src/ffi/interface.rs:40-47 */
    void *(*alloc_func)(void *opaque, size_t length);
    void (*free_func)(void *opaque, void *mfd);
    void *opaque;
};
struct DivansDecompressorState;
struct DivansCompressorState;

/* reference: src/ffi/mod.rs:178-187 (multithread=1, skip_crc=0) */
struct DivansDecompressorState *divans_new_decompressor(void);
/* reference: src/ffi/mod.rs:190-199 */
struct DivansDecompressorState *divans_new_serial_decompressor(void);
/* reference: src/ffi/mod.rs:213-232.  c/divans/ffi.h:61 declares only 2 arguments and c/example.c:62 calls it
 * that way, so `multithread` may be garbage: it is ignored (output is identical either way). */
struct DivansDecompressorState *divans_new_decompressor_with_custom_alloc(struct CAllocator alloc, uint8_t skip_crc,
                                                                          uint8_t multithread);
/* reference: src/ffi/mod.rs:236-262.  Streaming contract: offsets are cursors that are advanced; any call may
 * return NEEDS_MORE_INPUT / NEEDS_MORE_OUTPUT and be resumed at byte granularity.  Implementation: input is
 * buffered until the stream's 8-byte trailer has been seen, then the stream is decoded as a batch of one on
 * the GPU and the output is streamed back out. */
DivansResult divans_decode(struct DivansDecompressorState *state, const uint8_t *input_buf_ptr, size_t input_size,
                           size_t *input_offset, uint8_t *output_buf_ptr, size_t output_size, size_t *output_offset);
void divans_free_decompressor(struct DivansDecompressorState *mfd);          /* src/ffi/mod.rs:312-323 */
uint8_t *divans_decompressor_malloc_u8(struct DivansDecompressorState *s, size_t n);          /* :276-283 */
void divans_decompressor_free_u8(struct DivansDecompressorState *s, uint8_t *p, size_t n);     /* :285-292 */
size_t *divans_decompressor_malloc_usize(struct DivansDecompressorState *s, size_t n);        /* :294-301 */
void divans_decompressor_free_usize(struct DivansDecompressorState *s, size_t *p, size_t n);   /* :303-309 */

struct DivansCompressorState *divans_new_compressor(void);                                     /* :18-27 */
struct DivansCompressorState *divans_new_compressor_with_custom_alloc(struct CAllocator alloc); /* :38-52 */
DivansResult divans_set_option(struct DivansCompressorState *state, DivansOptionSelect selector, uint32_t value); /* :58-67 */
/* :70-91.  Input is buffered; the stream is produced by the GPU encoder at flush. */
DivansResult divans_encode(struct DivansCompressorState *state, const uint8_t *input_buf_ptr, size_t input_size,
                           size_t *input_offset, uint8_t *output_buf_ptr, size_t output_size, size_t *output_offset);
DivansResult divans_encode_flush(struct DivansCompressorState *state, uint8_t *output_buf_ptr, size_t output_size,
                                 size_t *output_offset);                                       /* :94-108 */
void divans_free_compressor(struct DivansCompressorState *mfd);                                /* :111-122 */
uint8_t *divans_compressor_malloc_u8(struct DivansCompressorState *s, size_t n);               /* :125-132 */
void divans_compressor_free_u8(struct DivansCompressorState *s, uint8_t *p, size_t n);         /* :134-141 */
size_t *divans_compressor_malloc_usize(struct DivansCompressorState *s, size_t n);             /* :143-150 */
void divans_compressor_free_usize(struct DivansCompressorState *s, size_t *p, size_t n);       /* :152-169 */

/* ------------------------------------------------------------------------------------------------
 * (2) batch extension
 * ------------------------------------------------------------------------------------------------ */
typedef struct divans_b200_ctx divans_b200_ctx;

#define DIVANS_B200_FLAG_SKIP_CRC 1u      /* same meaning as the reference's skip_crc (ffi/mod.rs:213) */
#define DIVANS_B200_FLAG_NO_CRC_KERNEL 2u /* do not even run the CRC kernel (trailer magic still checked) */
/* Model revision.  Default (0) = the reference tree as mounted.  DIVANS_B200_MODEL_WASM_2018 = the build that produced the
 * one compressed stream the reference tree holds (wasm/wasm.html:98-107): inside the PredictionMode command it codes the
 * context-map mnemonic nibbles (codec/context_map.rs:273) with the prior that DynamicContextMixingSpeed / PriorDepth /
 * ContextMapSpeedPalette[0] share (today: PredictionModePriorType::Mnemonic's own slots, codec/priors.rs:130) and every
 * mixing value (:395-405) with prior slot 16 (today: value[i - 256] & 15 for i >= 256); its encoder also never used
 * the `distance_lru[1] - 3` distance shortcut (codec/copy.rs:199-201).  Everything else is identical.  With the flag the
 * GPU decodes that stream bit-exactly and the GPU encoder reproduces its 113 bytes (tests/test_gpu_parity.py). */
#define DIVANS_B200_MODEL_CURRENT 0
#define DIVANS_B200_MODEL_WASM_2018 1
#define DIVANS_B200_FLAG_MODEL_WASM_2018 4u
/* Probability model.  Default = FrequentistCDF16, what every build of the reference uses unless it is compiled with
 * feature="blend", which swaps in BlendCDF16 for the whole crate (src/interface.rs:146-147, probability/blend_cdf.rs:109-208:
 * a division-free model that averages towards the coded symbol with a decaying rate and ignores the speeds).  Nothing in a
 * stream says which model coded it: the two sides have to agree, as with the reference's compile-time switch.  Blend streams
 * run on the generic per-nibble path (16 lanes per stream), not on the literal fast loops.  The reference's own entry points
 * (section 1) have no argument for it: a process that stands in for a `--features blend` build sets DIVANS_B200_FFI_CDF=blend
 * in its environment before the first divans_* call. */
#define DIVANS_B200_CDF_FREQUENTIST 0
#define DIVANS_B200_CDF_BLEND 1
#define DIVANS_B200_FLAG_CDF_BLEND 8u

/* per-stream status values are DivansResult codes (0 ok, 1 truncated input, 2 output capacity too small, 3 corrupt) */

/* device = CUDA ordinal; max_resident = cap on concurrently resident streams (0 = auto: sized to the GPU);
 * lanes_per_stream: 0 = by batch size (16 lanes per stream, 8 when their residency holds the batch in fewer passes); 16 = two
 * streams per warp, one CDF element per lane; 8 = four streams per warp, two elements per lane (up to twice the resident
 * streams where registers, not slot memory, limit residency).  Any other value means 16 (divans_b200_last_lanes reports
 * the layout a decode ran on). */
divans_b200_ctx *divans_b200_create(int device, uint32_t max_resident, uint32_t lanes_per_stream);
void divans_b200_destroy(divans_b200_ctx *ctx);
const char *divans_b200_last_error(divans_b200_ctx *ctx);
/* version string of the decode kernels in this build (quoted next to profile-derived numbers) */
const char *divans_b200_kernel_version(void);
/* lanes per stream the most recent decode call of this context ran with */
int divans_b200_last_lanes(divans_b200_ctx *ctx);
/* number of kernel launches issued by this context so far (bench.py's gpu_launches claim) */
uint64_t divans_b200_launch_count(divans_b200_ctx *ctx);
/* device time of the most recent decode/encode kernel(s) in milliseconds (CUDA events on the context stream) */
float divans_b200_last_kernel_ms(divans_b200_ctx *ctx);
/* device time of the dominant kernel alone (stream decoder / encoder model pass) of the most recent call */
float divans_b200_last_main_kernel_ms(divans_b200_ctx *ctx);

/* Decode n independent, complete .divans streams held in HOST memory.
 * stream i = in[in_off[i] .. in_off[i]+in_len[i]); its output goes to out[out_off[i] .. +out_cap[i]); the region is written
 * whole (zeros past out_len[i]), nothing outside the regions is touched.  Input regions may alias.
 * Includes H2D of the inputs and D2H of outputs inside the call.  Returns DIVANS_SUCCESS if the batch ran
 * (inspect status[] per stream), DIVANS_FAILURE on CUDA/context errors. */
DivansResult divans_b200_decode_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                           const uint64_t *in_len, uint8_t *out, const uint64_t *out_off,
                                           const uint64_t *out_cap, uint64_t *out_len, int32_t *status, uint32_t flags);
/* Pipelined variant of divans_b200_decode_batch_host for back-to-back batches: the call enqueues the H2D copies, the
 * kernels and the D2H copies on the context's copy / compute streams and returns a ticket (0 or 1; at most two batches
 * in flight, a third call first waits for the oldest).  The copies of one batch overlap the kernels of its neighbours.
 * `in` / `out` must stay valid (and should be pinned, else the copies degrade to synchronous ones) until
 * divans_b200_decode_batch_host_wait(ctx, ticket) returns -- out_len[] / status[] too: they are filled by the wait call (or by
 * the third async call, which retires the oldest batch, or by divans_b200_destroy).  Every region out[out_off[i] .. +out_cap[i])
 * is written whole (zeros past out_len[i]); nothing outside the regions is touched.  An empty batch (n == 0) returns
 * DIVANS_B200_TICKET_EMPTY, which wait() accepts as a no-op. */
#define DIVANS_B200_TICKET_EMPTY (-1)
DivansResult divans_b200_decode_batch_host_async(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                                 const uint64_t *in_len, uint8_t *out, const uint64_t *out_off,
                                                 const uint64_t *out_cap, uint64_t *out_len, int32_t *status, uint32_t flags,
                                                 int32_t *ticket);
DivansResult divans_b200_decode_batch_host_wait(divans_b200_ctx *ctx, int32_t ticket);
/* Same, all pointers are DEVICE pointers (inputs already resident in HBM, outputs left in HBM).
 * `in_total_bytes` >= sum(in_len) sizes the compacted-payload scratch (streams that would not fit it are failed with
 * status 3, never written out of bounds); `cuda_stream` is a cudaStream_t (NULL = the context's own stream).
 * Asynchronous: returns after enqueueing.  A context owns ONE set of scratch buffers: calls on the same context are
 * serialised (host mutex + an event that makes each launch set wait for the previous one, whatever stream it is on);
 * for concurrent batches create one context per batch in flight. */
DivansResult divans_b200_decode_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                             const uint64_t *d_in_len, uint8_t *d_out, const uint64_t *d_out_off,
                                             const uint64_t *d_out_cap, uint64_t *d_out_len, int32_t *d_status,
                                             uint64_t in_total_bytes, uint32_t flags, void *cuda_stream);
DivansResult divans_b200_synchronize(divans_b200_ctx *ctx);
/* For tests and diagnostics only: waits for the context's last call to finish, then copies the 16-byte header of arena
 * slot `slot` to out[4] -- the state a v2 decoder slot carries from stream to stream and from launch to launch:
 *   [0] generation counter (its low 16 bits tag the literal priors; 0 is skipped, the tables are wiped at the wrap),
 *   [1] nonzero: the literal tables may hold untagged 16-bit values (the next v2 stream wipes them),
 *   [2] literal-context-map bytes written since the map was last zeroed (high-water mark),
 *   [3] nonzero: the mixing mask holds an earlier stream's values.
 * Slot i of a decode launch is the i-th lane group (stream) of the grid.  Returns DIVANS_FAILURE when slot is not below the
 * number of slots the context has allocated (none before its first decode or encode call).  The layout is not a stable
 * interface. */
DivansResult divans_b200_debug_slot_header(divans_b200_ctx *ctx, uint32_t slot, uint32_t out[4]);

/* Encoder options (subset of the reference's DivansCompressorOptions, src/interface.rs:444-484, that affects the
 * entropy-coding half; command selection by the brotli crate is out of scope). */
typedef struct {
    int32_t window_size;            /* 10..24 */
    int32_t dynamic_context_mixing; /* 0,1,2 */
    int32_t prior_depth;
    int32_t use_context_map;
    int32_t force_stride;           /* 0..8, 9 = take the stride from the command */
    int32_t have_literal_adaptation;
    int16_t literal_adaptation[4][2];
    int32_t literal_pred_mode;      /* internal literal-only compressor: LSB6=0 MSB6=1 UTF8=2 SIGN=3 */
    int32_t literal_mixing_value;   /* internal literal-only compressor: value of all 8192 mixing entries (reference: 4) */
    int32_t model_rev;              /* DIVANS_B200_MODEL_CURRENT (default) or DIVANS_B200_MODEL_WASM_2018 */
    int32_t cdf_model;              /* DIVANS_B200_CDF_FREQUENTIST (default) or DIVANS_B200_CDF_BLEND */
} divans_b200_encode_options;
void divans_b200_encode_options_default(divans_b200_encode_options *o);

/* Encode n raw HOST buffers with the reference's internal literal-only command generator
 * (src/raw_to_cmd/mod.rs:105-181): one PredictionMode command + Literal commands. */
DivansResult divans_b200_encode_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                           const uint64_t *in_len, uint8_t *out, const uint64_t *out_off,
                                           const uint64_t *out_cap, uint64_t *out_len, int32_t *status,
                                           const divans_b200_encode_options *opts);
/* Same as divans_b200_encode_batch_host with every pointer a DEVICE pointer (raw inputs resident in HBM, framed streams
 * left in HBM); `max_in_len` >= every in_len[i] sizes the per-stream symbol logs.  Asynchronous on `cuda_stream`
 * (NULL = the context's own stream); status/out_len are valid after divans_b200_synchronize / a stream sync. */
DivansResult divans_b200_encode_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                             const uint64_t *d_in_len, uint64_t max_in_len, uint8_t *d_out,
                                             const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len,
                                             int32_t *d_status, const divans_b200_encode_options *opts, void *cuda_stream);
/* Encode n command lists ("DVCL" blobs, below) held in HOST memory: the entropy-coding half for arbitrary IR. */
DivansResult divans_b200_encode_cmds_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *blobs, const uint64_t *blob_off,
                                                const uint64_t *blob_len, uint8_t *out, const uint64_t *out_off,
                                                const uint64_t *out_cap, uint64_t *out_len, int32_t *status,
                                                const divans_b200_encode_options *opts);
/* IR text front-end (reference: src/bin/divans.rs:191-483, the textual IR that `divans -i` consumes): parse `ir_text` into a
 * DVCL blob.  *blob_len receives the size of the blob; with out == NULL or out_cap too small the call returns
 * DIVANS_NEEDS_MORE_OUTPUT.  *window_size (optional) receives the `window` line's value (0 if absent).  Host only. */
DivansResult divans_b200_ir_to_cmds(const char *ir_text, size_t ir_len, uint8_t *out, size_t out_cap, size_t *blob_len,
                                    int32_t *window_size);
/* Command generator for benchmarks / tools (ours, not a reference component): deterministic greedy hash-chain LZ77 (min
 * match 4, no dictionary words) -> one DVCL blob per raw buffer: a PredictionMode command (64-entry identity context map,
 * `mixing_value` everywhere, like src/raw_to_cmd/mod.rs:116-143) followed by Literal / Copy commands.  Blobs are written
 * at blob_off[i] (16-byte aligned) of `out`; with out == NULL or out_cap too small the call returns
 * DIVANS_NEEDS_MORE_OUTPUT and *total receives the size needed.  Host only, n_threads worker threads. */
DivansResult divans_b200_lz77_cmds_batch(size_t n, const uint8_t *in, const uint64_t *in_off, const uint64_t *in_len, int32_t window,
                                         int32_t pred_mode, int32_t mixing_value, uint8_t *out, size_t out_cap, uint64_t *blob_off,
                                         uint64_t *blob_len, size_t *total, int32_t n_threads);
/*
 * command list blob ("DVCL", little endian) -- the binary form of the reference's IR (src/bin/divans.rs:191-483):
 *   u32 magic 0x4c435644, u32 version 1, u32 n_cmds, u32 n_predmodes, u32 n_literal_bytes, u32 window, u32[2] 0
 *   n_cmds      x { u32 type, a, b, c, d }   type: 1 copy(a=distance,b=len) 2 dict(a=word_id,b=word_size,c=transform,d=final)
 *                                                  3 literal(a=offset into literal pool,b=len,c=high_entropy)
 *                                                  4/5/6 literal/command/distance block switch(a=type,b=stride) 7 prediction mode(a=index)
 *   n_predmodes x { u8 pred_mode, u8 is_adv, u8 has_speeds, u8 0, u16 cm_speed[2][2], u16 stride_speed[2][2],
 *                   u16 combined_speed[2][2], u16 lit_map_len, u16 dist_map_len, u8 lit_map[16384], u8 dist_map[1024],
 *                   u8 mixing[8192] }
 *   u8 literal pool[n_literal_bytes]
 */

#ifdef __cplusplus
}
#endif
#endif
