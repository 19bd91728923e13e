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
/* Decode n .divans streams held in HOST memory to their command lists: each stream is decoded as divans_b200_decode_batch_host
 * decodes it, and every command it carries is recorded as one DVCL record (the "command list blob" below), so a stored stream
 * can be re-encoded with divans_b200_encode_cmds_batch_host under other options.  The blob of stream i goes to
 * blobs[blob_off[i] .. +blob_cap[i]); its header's window is the stream's own.  Per stream:
 *   status 0: out_len[i] bytes were decoded and blob_len[i] bytes of DVCL were written;
 *   status 2 with blob_len[i] > blob_cap[i]: the blob region was too small.  The stream was still decoded to its end, out_len[i]
 *     is its full length, blob_len[i] the exact size its blob needs (retry with that);
 *   otherwise (output region too small, truncated or corrupt input): the status and out_len[i] of divans_b200_decode_batch_host,
 *     blob_len[i] = 0.
 * Both regions of every stream are written whole (zeros past the lengths; a failed stream's blob region is all zeros), nothing
 * outside them is touched.  Input regions may alias.  Frequentist streams run on the 16-lane layout whatever the context's
 * lanes_per_stream (divans_b200_last_lanes reports 16); flags as for decode (SKIP_CRC, NO_CRC_KERNEL, MODEL_WASM_2018, CDF_BLEND). */
DivansResult divans_b200_decode_cmds_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                                const uint64_t *in_len, uint8_t *out, const uint64_t *out_off,
                                                const uint64_t *out_cap, uint64_t *out_len, uint8_t *blobs, const uint64_t *blob_off,
                                                const uint64_t *blob_cap, uint64_t *blob_len, int32_t *status, uint32_t flags);
/* Same, all pointers are DEVICE pointers.  `in_total_bytes` and `cuda_stream` as for divans_b200_decode_batch_device; asynchronous
 * and serialised on the context exactly as that call.  Regions are not cleared first: past the lengths they hold what they held,
 * except that the records of a failed stream or of a region too small for its blob are zeroed. */
DivansResult divans_b200_decode_cmds_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                  const uint64_t *d_in_len, uint8_t *d_out, const uint64_t *d_out_off,
                                                  const uint64_t *d_out_cap, uint64_t *d_out_len, uint8_t *d_blobs,
                                                  const uint64_t *d_blob_off, const uint64_t *d_blob_cap, uint64_t *d_blob_len,
                                                  int32_t *d_status, uint64_t in_total_bytes, uint32_t flags, void *cuda_stream);
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
/* Same as divans_b200_encode_cmds_batch_host with every pointer a DEVICE pointer: command lists resident in HBM (for example
 * the blobs divans_b200_decode_cmds_batch_device wrote), framed streams left in HBM.
 *  - Every blob the host call accepts gives the same bytes, out_len and status as the host call with the same options: status 3
 *    for refused and hostile lists, status 2 with out_len the size the stream needs when out_cap is too small.  The logs here are
 *    at least as large as the host call's for the same batch, so the one refusal that can differ is the host call's own log
 *    overflow: a list whose PredictionMode commands share records can code more command symbols than its header's sizes
 *    provide for, and the host call refuses it when its sub-batch's logs are too small.
 *  - Asynchronous on `cuda_stream` (NULL = the context's own stream) and serialised on the context like the other device calls;
 *    divans_b200_last_kernel_ms / _last_main_kernel_ms are valid for it.
 *  - `max_blob_len` >= every blob_len[i] sizes the command logs, `max_raw_len` the literal logs, one capacity for the whole
 *    launch: a blob of up to max_blob_len bytes whose replay fits max_raw_len never fails for lack of log space.  A longer blob
 *    fails with status 3 and none of its bytes is read.
 *  - `max_raw_len` sizes the replay window of each slot: the decoded length of every list (one copy record can write megabytes).
 *    A list whose replay outgrows it fails with status 2 and out_len 0 (an output region too small gives out_len > out_cap).
 *  - blob_off[i] must be 4-byte aligned (records are read as u32): a blob at a misaligned address fails with status 3 unread.
 *  - opts->window_size == 0: each stream takes the window of its blob header (word 5), clamped to 10..24.  Any other value is
 *    clamped to 10..24 and applies to every stream, as in the host call.
 *  - The symbol logs of all n streams are one allocation, per stream about 10 bytes per byte of max_blob_len plus 8 per byte of
 *    max_raw_len; when it cannot be made the call returns DIVANS_FAILURE and divans_b200_last_error names the size.  There is no splitting into sub-batches.
 *  - Only d_out[out_off[i] .. +out_cap[i]) is written for stream i.  n == 0 returns DIVANS_SUCCESS. */
DivansResult divans_b200_encode_cmds_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_blobs, const uint64_t *d_blob_off,
                                                  const uint64_t *d_blob_len, uint64_t max_blob_len, uint64_t max_raw_len,
                                                  uint8_t *d_out, const uint64_t *d_out_off, const uint64_t *d_out_cap,
                                                  uint64_t *d_out_len, int32_t *d_status, const divans_b200_encode_options *opts,
                                                  void *cuda_stream);

/* ---- literal model selection ----
 * A candidate literal model of the raw-buffer encoder: the PredictionMode record divans_b200_encode_batch_host builds from
 * opts->literal_pred_mode / literal_mixing_value (LSB6=0 MSB6=1 UTF8=2 SIGN=3; mixing value 0..15). */
typedef struct {
    int32_t literal_pred_mode;
    int32_t literal_mixing_value;
} divans_b200_literal_model;
/* Encode n raw HOST buffers, each with the cheapest of n_cands candidate literal models.
 *  - A cost-only pass runs the encoder's model walk for every (stream, candidate) pair and sums, over every coded nibble of
 *    both coders, T[freq] = 65536 * -log2(freq / 32768) (1/65536 bit; the exact integer rule is freq_cost in dv_capi.cu).
 *    chosen[i] = the candidate with the lowest sum, ties to the lowest index.  Then stream i is encoded once with candidate
 *    chosen[i]: its bytes, out_len and status equal divans_b200_encode_batch_host's with opts->literal_pred_mode /
 *    literal_mixing_value set to that candidate (status 2: out_len is the size the chosen stream needs).
 *  - opts supplies every other option; its literal_pred_mode / literal_mixing_value are ignored.
 *  - cands: 1..16 entries, pred_mode 0..3, mixing value 0..15; anything else returns DIVANS_FAILURE (divans_b200_last_error
 *    says why) before any work.  Mixing value 2 (the flat prior that never adapts) is accepted but decodes on the generic path.
 *  - cost (may be NULL): n * n_cands sums, row per stream (cost[i * n_cands + c]).  A candidate whose pass failed (status 3, e.g.
 *    a literal_adaptation speed that wraps) costs UINT64_MAX; when every candidate failed, chosen[i] = 0 and the stream fails.
 *  - A stream's two coder payloads hold between cost / 8 bytes and 16 bytes per 65536-symbol rANS chunk more (DESIGN.md
 *    section 4, "Literal model selection").
 *  - The cost pass runs the model walk C times, so the call takes about C plain encodes.
 *  - n == 0 returns DIVANS_SUCCESS. */
DivansResult divans_b200_encode_auto_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                                const uint64_t *in_len, uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap,
                                                uint64_t *out_len, int32_t *status, const divans_b200_encode_options *opts,
                                                const divans_b200_literal_model *cands, uint32_t n_cands, uint32_t *chosen,
                                                uint64_t *cost);
/* Same as divans_b200_encode_auto_batch_host with the buffers, d_chosen and d_cost DEVICE pointers (cands is a host array,
 * copied before the call returns).  Conventions of divans_b200_encode_batch_device: `max_in_len` >= every in_len[i];
 * asynchronous on `cuda_stream` (NULL = the context's own stream), serialised on the context.  One launch sequence, no host
 * synchronisation: the cost pass runs the n * n_cands (stream, candidate) pairs through the context's encoder slots, as many at
 * a time as the slots hold. */
DivansResult divans_b200_encode_auto_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                  const uint64_t *d_in_len, uint64_t max_in_len, uint8_t *d_out,
                                                  const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len,
                                                  int32_t *d_status, const divans_b200_encode_options *opts,
                                                  const divans_b200_literal_model *cands, uint32_t n_cands, uint32_t *d_chosen,
                                                  uint64_t *d_cost, void *cuda_stream);
/* The candidate of the command-list calls below that keeps a list's own PredictionMode records (pred_mode -1, mixing value
 * -1; an initialiser of divans_b200_literal_model).  The raw calls above refuse it. */
#define DIVANS_B200_LITERAL_MODEL_KEEP { -1, -1 }
/* Encode n command lists (DVCL blobs) held in HOST memory, each coded under the cheapest of n_cands candidate literal models.
 *  - Coding a list under candidate c replaces EVERY PredictionMode record of the list by c's record: the one
 *    divans_b200_encode_batch_host builds from (pred_mode, mixing value), whole (mode, speeds, both context maps and the 8192
 *    mixing values; a context map only means something for the mode it was built for).  Commands, literal pool and window are
 *    unchanged.  KEEP ({-1, -1}) codes the list as given.
 *  - Contract: stream i's bytes, out_len and status equal divans_b200_encode_cmds_batch_host's for the same blob with every
 *    PredictionMode record replaced by candidate chosen[i]'s record (when chosen[i] is KEEP: the blob as given).
 *  - chosen[i] and cost as in divans_b200_encode_auto_batch_host: the sum of T[freq] over every coded nibble of both coders,
 *    ties to the lowest index, a failed pass costs UINT64_MAX.  A pass also fails when the list under that candidate would
 *    outgrow the symbol logs the final encode has for it: the log capacity holds per PredictionMode record, and commands that
 *    re-read small records code more entries under a replacing record than under their own.  So no chosen candidate is
 *    refused for lack of log space, and with KEEP among the candidates a list that the plain call encodes is encoded, at no
 *    higher cost than as given.
 *  - cands: 1..16 entries, each KEEP or pred_mode 0..3 with mixing value 0..15; anything else returns DIVANS_FAILURE before any
 *    work.  Sub-batched like divans_b200_encode_cmds_batch_host; n == 0 returns DIVANS_SUCCESS. */
DivansResult divans_b200_encode_cmds_auto_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *blobs, const uint64_t *blob_off,
                                                     const uint64_t *blob_len, uint8_t *out, const uint64_t *out_off,
                                                     const uint64_t *out_cap, uint64_t *out_len, int32_t *status,
                                                     const divans_b200_encode_options *opts, const divans_b200_literal_model *cands,
                                                     uint32_t n_cands, uint32_t *chosen, uint64_t *cost);
/* Same as divans_b200_encode_cmds_auto_batch_host with the buffers, d_chosen and d_cost DEVICE pointers (cands is a host array,
 * copied before the call returns).  Every convention of divans_b200_encode_cmds_batch_device holds: max_blob_len / max_raw_len,
 * window_size 0 = each blob's header window, status 2 and 3, guard rules, no sub-batching.  Its contract is with that call:
 * stream i equals divans_b200_encode_cmds_batch_device on the blob with its records replaced by chosen[i]'s.  One launch
 * sequence, no host synchronisation; the n * n_cands (stream, candidate) pairs run through the context's encoder slots in waves.
 * The cost pass holds a replay window of max_raw_len bytes per slot for up to n * n_cands pairs (the plain call: up to n). */
DivansResult divans_b200_encode_cmds_auto_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_blobs, const uint64_t *d_blob_off,
                                                       const uint64_t *d_blob_len, uint64_t max_blob_len, uint64_t max_raw_len,
                                                       uint8_t *d_out, const uint64_t *d_out_off, const uint64_t *d_out_cap,
                                                       uint64_t *d_out_len, int32_t *d_status, const divans_b200_encode_options *opts,
                                                       const divans_b200_literal_model *cands, uint32_t n_cands, uint32_t *d_chosen,
                                                       uint64_t *d_cost, void *cuda_stream);

/* ---- per-context mixing values ----
 * A PredictionMode record holds 8192 mixing values; each literal nibble reads the one at its mixing-mask index (the literal's
 * context byte, the nibble half, and the high nibble of the current or previous byte; codec/literal.rs:176-183).  These calls
 * choose each stream's values per entry, by coding cost, from k candidate values v[0..k) under the mode p =
 * opts->literal_pred_mode.  R(p, x) is the raw-buffer record of (p, x) (divans_b200_literal_model).  For stream i:
 *  1. Uniform passes: the cost walk under R(p, v[c]) gives the total u[i][c] (as encode_auto) and per-entry sums b[i][c][e]:
 *     the cost of the literal nibbles, of both coders, whose mixing-mask index is e.  Other nibbles count toward the total only.
 *  2. m[i][e] = argmin over c of b[i][c][e], ties to the lowest c (an entry no literal visits takes v[0]); a failed pass takes no
 *     part (when all failed, every entry takes v[0]).
 *  3. Mixed pass: M_i = R(p, v[0]) with mixing[e] = v[m[i][e]]; its cost walk gives x[i].
 *  4. c* = argmin of u[i][.], ties to the lowest c.  If x[i] < u[i][c*] stream i is encoded under M_i and chosen[i] = k, else
 *     under R(p, v[c*]) and chosen[i] = c*.  A tie keeps the uniform record, which decodes on the fast literal loop; a mixed
 *     record decodes on the generic per-nibble path.
 *  5. A uniform choice gives exactly the bytes, out_len and status of divans_b200_encode_batch_host with literal_mixing_value =
 *     v[c*]; a mixed one those of divans_b200_encode_cmds_batch_host on the stream's literal-only list with its record replaced
 *     by M_i.  So no stream costs more than under its best uniform candidate.
 *  6. A failed pass costs UINT64_MAX, as in encode_auto; status 2 as in encode_auto.
 * values: 1..16 entries, each 0..15, and opts->literal_pred_mode 0..3; anything else returns DIVANS_FAILURE before any work
 * (divans_b200_last_error says why).  Outputs, each may be NULL: chosen [n]; mixing [n * 8192], the values of the chosen record;
 * cost [n * (k + 1)], row i = u[i][0..k) then x[i]; bins [n * k * 8192], b[i][c][e] at (i * k + c) * 8192 + e (UINT64_MAX for a
 * failed pass).  Costs are in 1/65536 bit (T[freq], as encode_auto).  The encoder codes a record's mixing values only with
 * opts->use_context_map set and a nonzero dynamic_context_mixing or force_stride (the defaults); otherwise it codes one value
 * for every entry whatever the record holds, and every candidate costs the same.
 * The uniform passes run on the generic per-nibble path (their bins need each literal nibble's index), so the call takes
 * about k + 1 plain encodes and more.  Host calls are sub-batched like divans_b200_encode_auto_batch_host; n == 0 returns
 * DIVANS_SUCCESS. */
DivansResult divans_b200_encode_mixmap_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                                  const uint64_t *in_len, uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap,
                                                  uint64_t *out_len, int32_t *status, const divans_b200_encode_options *opts,
                                                  const int32_t *values, uint32_t n_values, uint32_t *chosen, uint8_t *mixing,
                                                  uint64_t *cost, uint64_t *bins);
/* Same with the buffers and outputs DEVICE pointers (values is a host array, copied before the call returns); conventions of
 * divans_b200_encode_auto_batch_device.  It also holds, per slot of the n * k pairs, 64 KiB of bins, and per stream 64 KiB of
 * per-entry winners and a record. */
DivansResult divans_b200_encode_mixmap_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                    const uint64_t *d_in_len, uint64_t max_in_len, uint8_t *d_out,
                                                    const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len,
                                                    int32_t *d_status, const divans_b200_encode_options *opts, const int32_t *values,
                                                    uint32_t n_values, uint32_t *d_chosen, uint8_t *d_mixing, uint64_t *d_cost,
                                                    uint64_t *d_bins, void *cuda_stream);
/* The same choice for command lists (DVCL blobs): every PredictionMode record of a list is replaced, by R(p, v[c]) in the
 * uniform passes and by M_i in the mixed pass, as encode_cmds_auto replaces them; commands, literal pool and window are kept.
 * Step 5's literal-only list is the list itself with its records replaced.  The log guard of encode_cmds_auto (a pass fails when
 * the replaced list would outgrow the final encode's logs) applies to all three kinds of pass.  Conventions of
 * divans_b200_encode_cmds_auto_batch_host / _device. */
DivansResult divans_b200_encode_cmds_mixmap_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *blobs, const uint64_t *blob_off,
                                                       const uint64_t *blob_len, uint8_t *out, const uint64_t *out_off,
                                                       const uint64_t *out_cap, uint64_t *out_len, int32_t *status,
                                                       const divans_b200_encode_options *opts, const int32_t *values, uint32_t n_values,
                                                       uint32_t *chosen, uint8_t *mixing, uint64_t *cost, uint64_t *bins);
DivansResult divans_b200_encode_cmds_mixmap_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_blobs, const uint64_t *d_blob_off,
                                                         const uint64_t *d_blob_len, uint64_t max_blob_len, uint64_t max_raw_len,
                                                         uint8_t *d_out, const uint64_t *d_out_off, const uint64_t *d_out_cap,
                                                         uint64_t *d_out_len, int32_t *d_status, const divans_b200_encode_options *opts,
                                                         const int32_t *values, uint32_t n_values, uint32_t *d_chosen, uint8_t *d_mixing,
                                                         uint64_t *d_cost, uint64_t *d_bins, void *cuda_stream);

/* ---- replaying command lists to raw bytes ----
 * Realise n command lists (DVCL blobs, below) as the bytes they describe: the reference's `recode` (src/bin/divans.rs:1108,
 * cmd_to_raw/mod.rs) on the GPU.  List i is blobs[blob_off[i] .. +blob_len[i]); its bytes go to out[out_off[i] .. +out_cap[i]).
 *  - Window: the ring is 1 << w.  window_size == 0: w is the blob header's window (word 5) clamped to 10..24; any other value is
 *    clamped to 10..24 and applies to every list.  This is the opts->window_size rule of divans_b200_encode_cmds_batch_device,
 *    so a list the encoder codes with window w replays with the same w.
 *  - Commands: literal (type 3) appends pool bytes [a, a + b); copy (1) appends b bytes at distance a, bytes before output
 *    position 0 reading as 0 (a fresh ring); dictionary (2) appends word a of size b under transform c, whose length must equal
 *    d when d != 0; block switches and PredictionMode commands (4..7) append nothing.
 *  - status 0: out_len[i] bytes were written at out + out_off[i].
 *  - status 2: the output needs more than out_cap[i] bytes.  out_len[i] is its exact length and the region holds its first
 *    out_cap[i] bytes: the walk goes on to the end of the list without moving bytes, applying every check below.  out_cap = 0
 *    measures lengths only (a length pass).
 *  - status 3 (refused): the blob is not 4-byte aligned (device call) or shorter than 32 bytes; the header's magic or version is
 *    wrong, or 32 + 20 * n_cmds + PM_RECORD_BYTES * n_predmodes + n_literal_bytes > blob_len (64-bit); a record's type is outside
 *    1..7; a literal has a + b > n_literal_bytes (64-bit); a copy has a == 0 or a >= 1 << w; a dictionary word or transform
 *    does not exist, or d != 0 differs from the transformed length.  Status 3 takes precedence over status 2.  out_len[i] counts
 *    the bytes of the commands before the refused one (0 for a refusal at blob or header level), and nothing past them is
 *    written.
 *  - No list reads outside its blob or writes outside its region.  Output positions and lengths are 64-bit.
 *  - One kernel launch per call; no arena slot or encoder log is used, so it works on a fresh context.
 * Host call: every region is written whole, with zeros past out_len[i]; nothing outside the regions is touched; input regions
 * may alias; blob offsets need no alignment (as for divans_b200_encode_cmds_batch_host).  n == 0 returns DIVANS_SUCCESS. */
DivansResult divans_b200_replay_cmds_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *blobs, const uint64_t *blob_off,
                                                const uint64_t *blob_len, uint8_t *out, const uint64_t *out_off,
                                                const uint64_t *out_cap, uint64_t *out_len, int32_t *status, int32_t window_size);
/* Same, all pointers DEVICE pointers.  Asynchronous on `cuda_stream` (NULL = the context's own stream) and serialised on the
 * context like every device call; divans_b200_last_kernel_ms is valid after it.  Regions are not cleared first.  With out_cap = 0
 * it sizes `max_raw_len` of divans_b200_encode_cmds_batch_device / _cmds_auto_batch_device for lists held in HBM: the largest
 * out_len of a length pass is the decoded length of every list. */
DivansResult divans_b200_replay_cmds_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_blobs, const uint64_t *d_blob_off,
                                                  const uint64_t *d_blob_len, uint8_t *d_out, const uint64_t *d_out_off,
                                                  const uint64_t *d_out_cap, uint64_t *d_out_len, int32_t *d_status,
                                                  int32_t window_size, void *cuda_stream);
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
/* The same generator on the GPU, next to raw buffers already in HBM; all pointers are DEVICE pointers.  Stream i is
 * in[in_off[i] .. +in_len[i]); its blob goes to blobs[blob_off[i] .. +blob_cap[i]).  Per stream:
 *  - status 0: blob_len[i] bytes were written at blobs + blob_off[i], byte for byte the blob divans_b200_lz77_cmds_batch writes
 *    for the same input, window, pred_mode and mixing_value (the last two stored as bytes, as there).
 *  - status 2: the region is too small; blob_len[i] is the exact size the blob needs.  The region's contents are unspecified.
 *  - status 3 (refused, the input is not read, blob_len[i] = 0): blob_off[i] is not 4-byte aligned (the encoders read records
 *    as u32), in_len[i] > max_in_len, or in_len[i] >= 2^31.
 *  - A region of 32 + 20 * (3 + 2 * floor(in_len / 5)) + PM_RECORD_BYTES + in_len bytes always holds the blob (Python:
 *    divans_b200.lz77_blob_cap): one PredictionMode command, and at most 2 + 2 * floor(in_len / 5) Literal and Copy commands.
 *    Proof: say a Copies have a Literal just before them and b do not.  Literal runs are maximal (never two in a row), so there
 *    are at most a + 1 of them.  A Copy covers at least 4 bytes and a Literal at least 1, so 5a + 4b <= in_len, and the Literal
 *    and Copy commands number at most 2a + b + 1 <= floor(2 in_len / 5) + 1 <= 2 floor(in_len / 5) + 2.
 *  - Nothing outside the regions is written, and regions are not cleared.
 * Call level: DIVANS_FAILURE for a window outside 10..24, n > 2^32 - 1, or when not even one warp's scratch (128 KiB +
 * 4 * max_in_len bytes, kept on the context and grown on demand) can be allocated; divans_b200_last_error names the size.  One
 * launch on min(n, max_resident, what the scratch holds) warps, asynchronous on `cuda_stream` (NULL = the context's stream) and
 * serialised on the context like every device call; divans_b200_last_kernel_ms is valid after it.  No arena slot or encoder
 * log is used, so it works on a fresh context.  Feed the blobs to divans_b200_encode_cmds_batch_device with max_blob_len from
 * the blob_len of this call and max_raw_len = max_in_len. */
DivansResult divans_b200_lz77_cmds_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                const uint64_t *d_in_len, uint64_t max_in_len, int32_t window, int32_t pred_mode,
                                                int32_t mixing_value, uint8_t *d_blobs, const uint64_t *d_blob_off,
                                                const uint64_t *d_blob_cap, uint64_t *d_blob_len, int32_t *d_status, void *cuda_stream);
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
 * A record is coded as command-coder nibbles, so the encoders (encode_cmds_*, and encode_cmds_auto_* / transcode with the
 * LITERAL_MODEL_KEEP candidate) refuse with status 3 a record they code whose is_adv is above 1, or whose mixing values, when
 * coded (dynamic context mixing or is_adv set, and the context map in use), include one above 15; a cost pass over such a
 * record costs UINT64_MAX.  pred_mode above 3 and map lengths above 16384 / 1024 are refused the same way.
 */

#ifdef __cplusplus
}
#endif
#endif
