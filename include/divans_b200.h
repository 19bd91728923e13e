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
 * the GPU and the output is streamed back out.
 *  - A bad magic number or a window byte outside 10..24 fails the call that completes the 16-byte header; a record header
 *    whose size code is above 3, or an end-of-stream marker other than ff fe ff, fails the call that delivers it (the whole
 *    marker).  The reference's demuxer checks neither (src/mux.rs: it reads a broken marker's next byte as a record header and
 *    sizes any code as 1024 << 2k); these refusals are the oracle's.  After a DIVANS_FAILURE every later call returns
 *    DIVANS_FAILURE.
 *  - Input is taken up to the end of the trailer and no further: *input_offset stops there when more bytes follow, as in the
 *    reference.  Once all output has been handed out every call returns DIVANS_SUCCESS and writes nothing.
 *  - The stream does not state its decoded size.  The first attempt decodes into 8 x the stream's size + 64 KiB and each
 *    NEEDS_MORE_OUTPUT retries at 4 x that, up to DIVANS_B200_MAX_OUTPUT bytes (environment, read once per process; default
 *    2^32).  A stream that decodes to more fails with DIVANS_FAILURE (so does one the allocator cannot hold). */
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
/* Options map to divans_b200_encode_options as in the reference (src/ffi/compressor.rs:63-166), starting from its defaults
 * (src/interface.rs:462-484: window 22, dynamic context mixing 1, context map on, stride from the command):
 *  - WINDOW_SIZE: any value, taken as an i32 and clamped to 10..24 (so 2^31 and above give 10).
 *  - the four LITERAL_ADAPTATION_*: a palette index 0..14 (Speed::ENCODER_DEFAULT_PALETTE).  The first of them sets all four
 *    speeds, later ones only their own: STRIDE_LOW [0], STRIDE_HIGH [1], CM_LOW [2], CM_HIGH [3].
 *  - FORCE_STRIDE_VALUE 0..8; USE_CONTEXT_MAP 0 or 1.
 *  - DYNAMIC_CONTEXT_MIXING and PRIOR_DEPTH keep the low byte of the value, FORCE_LITERAL_CONTEXT_MODE (LSB6=0 MSB6=1 UTF8=2
 *    SIGN=3, the mode of the literal-only record) too.
 *  - USE_BROTLI_COMMAND_SELECTION 0..2 and USE_BROTLI_BITSTREAM 1 are accepted, as are any value of QUALITY, LGBLOCK,
 *    STRIDE_DETECTION_QUALITY, PRIOR_BITMASK_DETECTION, SPEED_DETECTION_QUALITY, BROTLI_LITERAL_BYTE_SCORE, Q9_5 and
 *    IR_OPTIMIZER.  None of them changes the output: the encoder always codes the literal-only command list (see
 *    divans_b200_encode_batch_host), where the reference would select commands with the brotli crate.
 *  - Other values and selectors, and any call after the first divans_encode or divans_encode_flush, return DIVANS_FAILURE.
 * Departures: this library refuses at divans_set_option three kinds of value the reference accepts there but cannot code:
 *  - DYNAMIC_CONTEXT_MIXING with a low byte of 8 or more: the reference panics when encoding starts (the value must fit the
 *    low 3 bits of its PredictionMode nibble, codec/interface.rs:360, codec/context_map.rs:192);
 *  - PRIOR_DEPTH with a low byte above 15: the reference codes it as a nibble it does not fit, and fails (with the default
 *    probability model its stream does not decode back; a blend build indexes past the CDF);
 *  - FORCE_LITERAL_CONTEXT_MODE with a low byte above 3: only the reference's brotli command selection reads it, as SIGN; the
 *    mode here is the PredictionMode record's, which the decoder refuses above 3. */
/* :70-91.  Input is buffered; the stream is produced by the GPU encoder at flush.  After the flush, divans_encode returns
 * DIVANS_FAILURE, and a flush call once all output has been handed out returns DIVANS_SUCCESS and writes nothing. */
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
 * for concurrent batches create one context per batch in flight.  Regions are not cleared first: of region i only
 * out[out_off[i] .. +out_len[i]) is written (with status 2, the bytes of the commands that fit), the rest holds what it held. */
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
 * except that the records of a failed stream or of a region too small for its blob are zeroed, and that in a blob region the
 * bytes where the decoder staged the prediction-mode records (the region's last n_predmodes * PM_RECORD_BYTES) are zeroed past
 * blob_len[i]. */
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
    int32_t literal_pred_mode;      /* internal literal-only compressor: LSB6=0 MSB6=1 UTF8=2 SIGN=3; the raw calls that build
                                       their record from it (plain and speeds) return DIVANS_FAILURE for anything else */
    int32_t literal_mixing_value;   /* internal literal-only compressor: value of all 8192 mixing entries (reference: 4) */
    int32_t model_rev;              /* DIVANS_B200_MODEL_CURRENT (default) or DIVANS_B200_MODEL_WASM_2018 */
    int32_t cdf_model;              /* DIVANS_B200_CDF_FREQUENTIST (default) or DIVANS_B200_CDF_BLEND */
} divans_b200_encode_options;
void divans_b200_encode_options_default(divans_b200_encode_options *o);

/* Encode n raw HOST buffers with the reference's internal literal-only command generator
 * (src/raw_to_cmd/mod.rs:105-181): one PredictionMode command + Literal commands.  Of region i only out[out_off[i] ..
 * +out_len[i]) is written, and only with status 0: the rest of the region holds what it held, and a stream that fails or does
 * not fit (status 2, out_len the size it needs) writes nothing.  Every encode call below, host or device, writes its regions
 * the same way. */
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

/* ---- literal speeds ----
 * literal_adaptation[4] is ordered stride-low, stride-high, cm-low, cm-high.  [0] adapts both nibbles' stride priors; [1] is
 * coded in the stream and read by no literal; [2] and [3] adapt the context-map priors of the low and high nibble, which are read
 * only with dynamic_context_mixing 2.  These calls choose each stream's speeds, by coding cost, from k candidate speeds v[0..k)
 * under everything else the options say (mode, mixing value, maps).  For stream i:
 *  1. Uniform passes: the cost walk under (v[c], v[c], v[c], v[c]) gives u[i][c] (T[freq], as encode_auto).  c* = argmin,
 *     ties to the lowest c.
 *  2. Only with opts->dynamic_context_mixing >= 2 and k > 1 (and u[i][c*] < UINT64_MAX): halves passes under
 *     (v[c*], v[c*], v[d], v[d]) give lo[i][d] and hi[i][d], the cost of the literal low and high nibbles, both coders.  l* =
 *     argmin lo, h* = argmin hi, ties to the lowest d; a failed pass takes no part (all failed: l* = h* = c*).  With dynamic
 *     mixing 2 and S0 fixed, the low nibbles' cost depends on S2 alone and the high nibbles' on S3 alone, so each half is
 *     chosen on its own; the command coder also codes the four speeds, so the total is checked:
 *  3. Verify pass under (v[c*], v[c*], v[l*], v[h*]): x[i].  It is taken only if x[i] < u[i][c*].  When step 2 is skipped,
 *     x[i] = u[i][c*].  chosen[i] = (a, b, c): (c*, l*, h*) when taken, else (c*, c*, c*).
 *  4. Stream i's bytes, out_len and status equal divans_b200_encode_batch_host's with have_literal_adaptation = 1 and
 *     literal_adaptation = {v[a], v[a], v[b], v[c]}; for command lists, divans_b200_encode_cmds_batch_host's (the speeds override
 *     every record's, as opts->literal_adaptation does).  So no stream costs more than under its best uniform candidate.
 *  5. A failed pass costs UINT64_MAX.  If every uniform pass fails, chosen = (0, 0, 0) and the stream fails; status 2 as in
 *     encode_auto.
 * opts->have_literal_adaptation and opts->literal_adaptation are ignored.  values: 1..16 int16_t[2] (inc, lim), each unchanged by
 * the f8 round trip the stream codes speeds with and small enough that no literal prior can wrap its i16 counters (so the
 * streams stay on the decoder's literal fast loops); anything else returns DIVANS_FAILURE before any work, and
 * divans_b200_last_error names the entry.  Outputs, each may be NULL: chosen [n * 3]; cost [n * (k + 1)], row i = u[i][0..k)
 * then x[i]; halves [n * k * 2], (lo, hi) of stream i under d at (i * k + d) * 2 (UINT64_MAX for a failed or skipped pass).
 * Costs are in 1/65536 bit.  The call takes k cost walks (2k + 1 with the halves and verify passes) and the encode; the cost walks run
 * on the fast literal loops.  Host calls are sub-batched like divans_b200_encode_auto_batch_host; n == 0 returns
 * DIVANS_SUCCESS. */
DivansResult divans_b200_encode_speeds_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                                  const uint64_t *in_len, uint8_t *out, const uint64_t *out_off, const uint64_t *out_cap,
                                                  uint64_t *out_len, int32_t *status, const divans_b200_encode_options *opts,
                                                  const int16_t *values, uint32_t n_values, uint32_t *chosen, uint64_t *cost,
                                                  uint64_t *halves);
/* Same with the buffers and outputs DEVICE pointers (values is a host array, read before the call returns); one launch sequence,
 * no host sync; conventions of divans_b200_encode_auto_batch_device. */
DivansResult divans_b200_encode_speeds_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                    const uint64_t *d_in_len, uint64_t max_in_len, uint8_t *d_out,
                                                    const uint64_t *d_out_off, const uint64_t *d_out_cap, uint64_t *d_out_len,
                                                    int32_t *d_status, const divans_b200_encode_options *opts, const int16_t *values,
                                                    uint32_t n_values, uint32_t *d_chosen, uint64_t *d_cost, uint64_t *d_halves,
                                                    void *cuda_stream);
/* The same choice for command lists (DVCL blobs): the lists keep their records, commands, literal pool and window; the speeds
 * override the records'.  Conventions of divans_b200_encode_cmds_auto_batch_host / _device. */
DivansResult divans_b200_encode_cmds_speeds_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *blobs, const uint64_t *blob_off,
                                                       const uint64_t *blob_len, uint8_t *out, const uint64_t *out_off,
                                                       const uint64_t *out_cap, uint64_t *out_len, int32_t *status,
                                                       const divans_b200_encode_options *opts, const int16_t *values, uint32_t n_values,
                                                       uint32_t *chosen, uint64_t *cost, uint64_t *halves);
DivansResult divans_b200_encode_cmds_speeds_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_blobs, const uint64_t *d_blob_off,
                                                         const uint64_t *d_blob_len, uint64_t max_blob_len, uint64_t max_raw_len,
                                                         uint8_t *d_out, const uint64_t *d_out_off, const uint64_t *d_out_cap,
                                                         uint64_t *d_out_len, int32_t *d_status, const divans_b200_encode_options *opts,
                                                         const int16_t *values, uint32_t n_values, uint32_t *d_chosen, uint64_t *d_cost,
                                                         uint64_t *d_halves, void *cuda_stream);

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
/* ---- the LZ77 parse ----
 * How the generator above walks the positions of a stream of n bytes.  best(i) = (len(i), dist(i)) is the longest match at
 * position i exactly as above: the (at most 16) most recent earlier positions of the same hash, up to the first farther than
 * 2^window - 16, each compared up to min(n - i, 65535) bytes, ties to the most recent candidate, and len(i) = 0 where i + 4 > n
 * or i >= n.  Every position is inserted into the chain in order, copies included, so best(i) is a function of i alone, not of
 * the parse.  The parse starts at i = 0 with an empty literal run, and while i < n, with L = len(i):
 *  - it defers when lazy >= 1 and L < 32 and either len(i + 1) > L, or lazy == 2 and len(i + 2) > L + 1;
 *  - if L >= min_match and it does not defer, it emits the pending literal run (if any), then Copy(dist(i), L), and i += L;
 *  - otherwise byte i joins the literal run and i += 1.
 * The last literal run is emitted at the end.  Domain: min_match 4..32 and lazy 0..2; a parse outside it fails the call
 * (DIVANS_FAILURE) with nothing written.  {4, 0} is the parse of the two calls above, byte for byte.  Every copy is at least
 * 4 bytes long, so the region bound of divans_b200_lz77_cmds_batch_device (divans_b200.lz77_blob_cap) holds for every parse.
 * (The L < 32 guard keeps each comparison of lengths below the GPU generator's 64-byte capped compare, which is exact there.) */
typedef struct {
    int32_t min_match;   /* 4..32: the shortest match emitted as a copy */
    int32_t lazy;        /* 0..2: positions looked ahead before a match shorter than 32 bytes is taken */
} divans_b200_lz77_parse;
#define DIVANS_B200_LZ77_PARSE_DEFAULT { 4, 0 }
/* divans_b200_lz77_cmds_batch under `parse` (NULL or out of the domain: DIVANS_FAILURE, nothing written). */
DivansResult divans_b200_lz77_cmds_batch_parse(size_t n, const uint8_t *in, const uint64_t *in_off, const uint64_t *in_len, int32_t window,
                                               int32_t pred_mode, int32_t mixing_value, uint8_t *out, size_t out_cap, uint64_t *blob_off,
                                               uint64_t *blob_len, size_t *total, int32_t n_threads, const divans_b200_lz77_parse *parse);
/* divans_b200_lz77_cmds_batch_device under `parse`: every blob byte for byte divans_b200_lz77_cmds_batch_parse's, with every
 * other rule of that call (statuses, regions, refusals, scratch).  A parse that is NULL or outside the domain fails the call
 * (DIVANS_FAILURE, divans_b200_last_error says why) before any work.  The GPU walks 32 positions per step; a deferral whose
 * lookahead (i + 1 or i + 2) falls past those 32 is not decided there: the step ends before position i, and the next starts
 * at it.  So a lazy parse may take a few more steps than the greedy one. */
DivansResult divans_b200_lz77_cmds_batch_device_parse(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                      const uint64_t *d_in_len, uint64_t max_in_len, int32_t window, int32_t pred_mode,
                                                      int32_t mixing_value, uint8_t *d_blobs, const uint64_t *d_blob_off,
                                                      const uint64_t *d_blob_cap, uint64_t *d_blob_len, int32_t *d_status,
                                                      const divans_b200_lz77_parse *parse, void *cuda_stream);
/* ---- dictionary words in the LZ77 parse ----
 * The parse above with one more step: RFC 7932 static-dictionary words, emitted as Dictionary commands (DVCL type 2).
 *  - The transform set: the transforms whose prefix is empty and whose type is identity (0), so their output is word + suffix.
 *    It is derived from the RFC 7932 tables at load time; it has 44 members, 0 (""), 1 (" "), 5 (" the "), 8 (" of "), ...
 *  - dict(i) = (Ld, word id, word size, transform).  Among every word of size 4..24 with id below 2^size_bits_by_length[size],
 *    under every transform of the set, with transformed bytes w, i + |w| <= n and in[i .. i + |w|) == w: the longest |w|, ties
 *    to the lowest transform id, then the shortest word size, then the lowest word id.  Ld = 0 where none matches.  Like best(i),
 *    dict(i) is a function of i alone.  |w| is at most 24 + 7 = 31 bytes.
 *  - With dict_min = 0 the parse is exactly the one above.  With dict_min 4..32, at a position the parse reaches and does not
 *    defer, let Lc = len(i) if it is at least min_match (else 0) and Ld = dict(i)'s length if it is at least dict_min (else 0).
 *    If Ld > Lc the parse emits the pending literal run (if any), then Dictionary(a = word id, b = word size, c = transform,
 *    d = Ld), and i += Ld.  Otherwise it goes on exactly as above.
 *  - Deferral keeps its rule on copy lengths alone: a position deferred because len(i + 1) or len(i + 2) is longer becomes a
 *    literal even when a dictionary word starts there.  A deferral needs L = len(i) >= min_match, so a position with no copy
 *    is never deferred and may always take a word.
 *  - Every position is still inserted into the hash chain in order, so best(i) does not move.
 *  - Region bound: a Dictionary command covers |w| >= 4 bytes, as a Copy covers at least 4, and literal runs stay maximal.  So
 *    the proof of divans_b200_lz77_cmds_batch_device holds with "Copy" read as "Copy or Dictionary", and lz77_blob_cap holds
 *    every list of every parse.
 * Domain: min_match 4..32, lazy 0..2, dict_min 0 or 4..32, reserved 0. */
typedef struct {
    int32_t min_match;   /* 4..32: the shortest match emitted as a copy */
    int32_t lazy;        /* 0..2: positions looked ahead before a match shorter than 32 bytes is taken */
    int32_t dict_min;    /* 0 (no dictionary words) or 4..32: the shortest transformed word emitted as a Dictionary command */
    int32_t reserved;    /* 0 */
} divans_b200_lz77_dict_parse;
/* divans_b200_lz77_cmds_batch_parse under a parse with dictionary words (NULL or out of the domain: DIVANS_FAILURE, nothing
 * written).  dict_min = 0 writes divans_b200_lz77_cmds_batch_parse's blobs for {min_match, lazy}, byte for byte. */
DivansResult divans_b200_lz77_cmds_batch_dict(size_t n, const uint8_t *in, const uint64_t *in_off, const uint64_t *in_len, int32_t window,
                                              int32_t pred_mode, int32_t mixing_value, uint8_t *out, size_t out_cap, uint64_t *blob_off,
                                              uint64_t *blob_len, size_t *total, int32_t n_threads, const divans_b200_lz77_dict_parse *parse);
/* divans_b200_lz77_cmds_batch_device_parse under a parse with dictionary words: every blob byte for byte
 * divans_b200_lz77_cmds_batch_dict's, with every other rule of that call (statuses, regions, refusals, scratch, the step end
 * before a deferral whose lookahead falls past the 32 positions).  A parse that is NULL or outside the domain fails the call
 * (DIVANS_FAILURE, divans_b200_last_error says why) before any work.  With dict_min != 0 the first call on a context uploads a
 * dictionary index of 174,344 bytes next to the RFC 7932 tables (122,784 dictionary bytes) the decoder already holds; it stays
 * until the context is destroyed. */
DivansResult divans_b200_lz77_cmds_batch_device_dict(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                     const uint64_t *d_in_len, uint64_t max_in_len, int32_t window, int32_t pred_mode,
                                                     int32_t mixing_value, uint8_t *d_blobs, const uint64_t *d_blob_off,
                                                     const uint64_t *d_blob_cap, uint64_t *d_blob_len, int32_t *d_status,
                                                     const divans_b200_lz77_dict_parse *parse, void *cuda_stream);
/* ---- dictionary words under every transform in the LZ77 parse ----
 * The parse with dictionary words above, with a larger candidate set when transforms = 1.  Everything else is that parse's:
 * deferral on copy lengths only, Ld > Lc, every position inserted into the hash chain, the window rule.
 *  - transforms = 0: the 44-member set above; the lists are divans_b200_lz77_cmds_batch_dict's, byte for byte.
 *  - transforms = 1: every word of size 4..24 (id below 2^size_bits_by_length[size]) under every transform t of 0..120.  w is
 *    exactly what the decoder's dictionary step writes for (id, size, t): the prefix, then the core (the word after the
 *    transform's omission, with its case transform applied, by the decoder's UTF-8 uppercase rule), then the suffix.  Types:
 *    0 identity, 1..9 omit the last 1..9 bytes, 10 uppercase the first character, 11 uppercase all, 12..20 omit the first 1..9.
 *  - A candidate counts only when its core has at least 4 bytes.  Then each candidate is found by one 4-byte key at the core's
 *    start: the first 4 bytes of the core after the case transform, which depend on the core's first 4 bytes alone.
 *  - dict(i) is the longest w with i + |w| <= n and in[i .. i + |w|) == w; ties to the lowest transform, then the shortest word
 *    size, then the lowest word id (the order of the 44-member set).  There are 9 distinct prefixes and a prefix and suffix
 *    together have at most 13 bytes, so |w| <= 24 + 13 = 37: the GPU generator's capped copy compare of 64 bytes still orders a
 *    word against a copy exactly.  dict_min >= 4 keeps Ld >= 4, so lz77_blob_cap still holds every list.
 * Domain: min_match 4..32, lazy 0..2, dict_min 0 or 4..32, transforms 0 or 1. */
typedef struct {
    int32_t min_match;   /* 4..32: the shortest match emitted as a copy */
    int32_t lazy;        /* 0..2: positions looked ahead before a match shorter than 32 bytes is taken */
    int32_t dict_min;    /* 0 (no dictionary words) or 4..32: the shortest transformed word emitted as a Dictionary command */
    int32_t transforms;  /* 0: the 44 transforms with an empty prefix and the identity type; 1: all 121 */
} divans_b200_lz77_words_parse;
/* divans_b200_lz77_cmds_batch_dict under a words parse (NULL or out of the domain: DIVANS_FAILURE, nothing written).
 * transforms = 0 writes divans_b200_lz77_cmds_batch_dict's blobs for {min_match, lazy, dict_min, 0}, byte for byte. */
DivansResult divans_b200_lz77_cmds_batch_words(size_t n, const uint8_t *in, const uint64_t *in_off, const uint64_t *in_len, int32_t window,
                                               int32_t pred_mode, int32_t mixing_value, uint8_t *out, size_t out_cap, uint64_t *blob_off,
                                               uint64_t *blob_len, size_t *total, int32_t n_threads, const divans_b200_lz77_words_parse *parse);
/* divans_b200_lz77_cmds_batch_device_dict under a words parse: every blob byte for byte divans_b200_lz77_cmds_batch_words's, with
 * every other rule of that call (statuses, regions, refusals, scratch, the step end before a deferral whose lookahead falls past
 * the 32 positions).  A parse that is NULL or outside the domain fails the call (DIVANS_FAILURE, divans_b200_last_error says
 * why) before any work.  With dict_min != 0 and transforms = 1 the first call on a context uploads the index of every transform
 * (1,427,612 bytes, the dictionary bytes and their two uppercase forms included); it stays until the context is destroyed. */
DivansResult divans_b200_lz77_cmds_batch_device_words(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                                      const uint64_t *d_in_len, uint64_t max_in_len, int32_t window, int32_t pred_mode,
                                                      int32_t mixing_value, uint8_t *d_blobs, const uint64_t *d_blob_off,
                                                      const uint64_t *d_blob_cap, uint64_t *d_blob_len, int32_t *d_status,
                                                      const divans_b200_lz77_words_parse *parse, void *cuda_stream);
/* ---- choosing one of k command lists per stream by coding cost ----
 * n streams, each with k (1..16) candidate DVCL command lists already in HBM, candidate-major: list c of stream i is
 * d_blobs[d_blob_off[c * n + i] .. +d_blob_len[c * n + i]) (4-byte aligned).  The lists of a stream should replay to the same
 * bytes (several parses of one input, say), but any lists are accepted: host-generated, from the GPU generator, from IR.
 *  1. The cost pass of divans_b200_encode_cmds_auto_batch_device runs over the n * k (stream, list) pairs, each list under its
 *     own PredictionMode records: the sum of T[freq] over every coded nibble of both coders, in 1/65536 bit.  A pair whose pass
 *     fails (status 2 or 3, or a list that would outgrow the logs) costs UINT64_MAX.
 *  2. d_chosen[i] = the list of the lowest cost, ties to the lowest index; d_cost (may be NULL) = the n * k costs, row per stream
 *     (d_cost[i * k + c]).  When every list of a stream fails, d_chosen[i] = 0.
 *  3. Stream i is encoded from list d_chosen[i]: its bytes, out_len and status are exactly divans_b200_encode_cmds_batch_device's
 *     for that list (so a stream whose lists all fail fails as the plain call does on list 0).  With d_out == NULL the call
 *     stops after step 2, and d_out_off, d_out_cap, d_out_len and d_status are not read.
 * Every convention of divans_b200_encode_cmds_batch_device holds, with max_blob_len >= every list's length and max_raw_len >=
 * every list's decoded length: window_size 0 = each list's header window, status 2 and 3, no sub-batching.  One launch
 * sequence, no host synchronisation; the pairs run through the context's encoder slots in waves, each slot holding a replay
 * window of max_raw_len bytes.  k outside 1..16 or a NULL d_chosen returns DIVANS_FAILURE before any work; n == 0 returns
 * DIVANS_SUCCESS. */
DivansResult divans_b200_encode_cmds_choose_batch_device(divans_b200_ctx *ctx, size_t n, uint32_t k, const uint8_t *d_blobs,
                                                         const uint64_t *d_blob_off, const uint64_t *d_blob_len, uint64_t max_blob_len,
                                                         uint64_t max_raw_len, uint8_t *d_out, const uint64_t *d_out_off,
                                                         const uint64_t *d_out_cap, uint64_t *d_out_len, int32_t *d_status,
                                                         const divans_b200_encode_options *opts, uint32_t *d_chosen, uint64_t *d_cost,
                                                         void *cuda_stream);
/* ---- billing each stream's coding cost by coder state ----
 * The cost pass (encode_auto's cost, encode_cmds_choose's d_cost) gives one number per stream.  The bill splits that number by
 * the state of the encoder's command state machine that coded each nibble, as the reference's billing build does
 * (BillingDesignation, src/interface.rs:328-346; there the mantissa nibble states are folded together, here they are rows).
 *  - A stream's bill has DIVANS_B200_BILL_STATES rows, one per nibble-coding state, in the order of the table below (row index,
 *    name, the reference substate).  The order is part of the interface.
 *  - Each row holds two uint64_t: cost, the sum of T[freq] (1/65536 bit, as encode_auto) over every nibble coded in that state
 *    by either coder; nibbles, how many nibbles were coded in it.
 *  - A nibble's state is the state the encoder was in when it coded that nibble.  A literal byte is one LIT_HI and one LIT_LO
 *    nibble; the end-of-stream nibble is a CMD_TYPE nibble.
 *  - The sum of a stream's cost column equals, to the unit, the cost the cost pass gives the same stream under the same options
 *    and list: encode_auto's cost for that candidate, encode_cmds_choose's d_cost for that list.
 *  - A stream whose pass fails has status 3 (or 2, a command list that replays past max_raw_len) and an all-zero bill: the
 *    failures for which the cost pass gives UINT64_MAX (a refused record, a speed that wraps, a list that outgrows the logs).
 *  - Nothing is encoded and no output stream is written.
 * Rows (index  name              reference substate):
 *    0 CMD_TYPE          CrossCommandBilling::FullSelection: command type, end-of-stream nibble         codec/mod.rs:662-688
 *    1 LIT_HI            LiteralSubstate::LiteralNibbleIndex                                            codec/literal.rs:261-394
 *    2 LIT_LO            LiteralSubstate::LiteralNibbleLowerHalf
 *    3 LL_COUNT_SMALL    LiteralSubstate::LiteralCountSmall                                             codec/literal.rs:565-661
 *    4 LL_SIZE_BEG       LiteralSubstate::LiteralCountFirst
 *    5 LL_SIZE_LAST      LiteralSubstate::LiteralCountLengthGreater14Less25
 *    6 LL_MANT           LiteralSubstate::LiteralCountMantissaNibbles
 *    7 CP_COUNT_SMALL    CopySubstate::CountSmall                                                       codec/copy.rs:87-162
 *    8 CP_COUNT_BEG      CopySubstate::CountLengthFirst
 *    9 CP_COUNT_LAST     CopySubstate::CountLengthGreater18Less25
 *   10 CP_COUNT_MANT     CopySubstate::CountMantissaNibbles
 *   11 CP_MNEMONIC       CopySubstate::DistanceLengthMnemonic                                           codec/copy.rs:166-280
 *   12 CP_DIST_BEG       CopySubstate::DistanceLengthFirst
 *   13 CP_DIST_LAST      CopySubstate::DistanceLengthGreater14Less25
 *   14 CP_DIST_MANT      CopySubstate::DistanceMantissaNibbles
 *   15 DC_SIZE_BEG       DictSubstate::WordSizeFirst                                                    codec/dict.rs:81-170
 *   16 DC_SIZE_LAST      DictSubstate::WordSizeGreater18Less25
 *   17 DC_INDEX          DictSubstate::WordIndexMantissa
 *   18 DC_TR_HI          DictSubstate::TransformHigh
 *   19 DC_TR_LO          DictSubstate::TransformLow
 *   20 BT_MNEMONIC       BlockTypeState::Begin                                                          codec/block_type.rs:61-110
 *   21 BT_FIRST          BlockTypeState::TwoNibbleType
 *   22 BT_SECOND         BlockTypeState::FinalNibble
 *   23 BT_STRIDE         LiteralBlockSwitch's stride nibble                                             codec/block_type.rs:170-190
 *   24 PM_MODE           PredictionModeSubstate::Begin                                                  context_map.rs:172-425
 *   25 PM_MIX            PredictionModeSubstate::DynamicContextMixing
 *   26 PM_DEPTH          PredictionModeSubstate::PriorDepth
 *   27 PM_SPEED          PredictionModeSubstate::AdaptationSpeed
 *   28 PM_MAP_MNEMONIC   PredictionModeSubstate::ContextMapMnemonic
 *   29 PM_MAP_FIRST      PredictionModeSubstate::ContextMapFirstNibble
 *   30 PM_MAP_SECOND     PredictionModeSubstate::ContextMapSecondNibble
 *   31 PM_MIXVAL         PredictionModeSubstate::MixingValues
 * (32 rows in all; see DIVANS_B200_BILL_STATES.) */
#define DIVANS_B200_BILL_STATES 32
/* Raw buffers, coded as divans_b200_encode_batch_host codes them: the literal-only list with the record of
 * opts->literal_pred_mode and literal_mixing_value.  bill [n * DIVANS_B200_BILL_STATES * 2]: (cost, nibbles) of stream i, row r
 * at (i * DIVANS_B200_BILL_STATES + r) * 2; status [n].  Sub-batched like divans_b200_encode_auto_batch_host.  Options apply as
 * in the encoders, both probability models and DIVANS_B200_MODEL_WASM_2018 included.  n == 0 returns DIVANS_SUCCESS. */
DivansResult divans_b200_bill_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *in, const uint64_t *in_off,
                                         const uint64_t *in_len, const divans_b200_encode_options *opts, uint64_t *bill,
                                         int32_t *status);
/* Same with the buffers, d_bill and d_status DEVICE pointers: one launch sequence, no host synchronisation, asynchronous on
 * cuda_stream and serialised on the context; divans_b200_last_kernel_ms times the billing pass afterwards. */
DivansResult divans_b200_bill_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_in, const uint64_t *d_in_off,
                                           const uint64_t *d_in_len, uint64_t max_in_len, const divans_b200_encode_options *opts,
                                           uint64_t *d_bill, int32_t *d_status, void *cuda_stream);
/* DVCL command lists under their own records, with every convention of divans_b200_encode_cmds_batch_host / _device:
 * window_size 0 = each list's header window; device blobs 4-byte aligned, at most max_blob_len bytes, replaying at most
 * max_raw_len bytes (else status 3, or 2 past max_raw_len).  Outputs and synchronisation as the raw calls. */
DivansResult divans_b200_bill_cmds_batch_host(divans_b200_ctx *ctx, size_t n, const uint8_t *blobs, const uint64_t *blob_off,
                                              const uint64_t *blob_len, const divans_b200_encode_options *opts, uint64_t *bill,
                                              int32_t *status);
DivansResult divans_b200_bill_cmds_batch_device(divans_b200_ctx *ctx, size_t n, const uint8_t *d_blobs, const uint64_t *d_blob_off,
                                                const uint64_t *d_blob_len, uint64_t max_blob_len, uint64_t max_raw_len,
                                                const divans_b200_encode_options *opts, uint64_t *d_bill, int32_t *d_status,
                                                void *cuda_stream);
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
 * record costs UINT64_MAX.  pred_mode above 3 and map lengths above 16384 / 1024 are refused the same way.  So is every other
 * record whose fields no sequence of nibbles carries (status 3, a cost pass UINT64_MAX, where the first nibble that cannot
 * carry the value would be built; the stream's bytes are never written): a type outside 1..7 (15 would end
 * the stream early), a copy distance of 0 or of 2^30 and more, a literal length of 0 or above 2^30 + 14, a dictionary word
 * size outside 4..24, a word id of 2^round_up_mod_4(bits of the size) or more, or a transform above 255, a block type above
 * 255, and a literal block switch's stride above 15 when the stride is taken from the record (force_stride 9).  Other values
 * the stream carries but the decoder rejects (a distance past the window, a transform 121..255, a word id past the
 * dictionary) fail the encode with status 3 where the decoder would fail.  The fields no nibble codes (a dictionary record's
 * d, a copy's c and d, a block switch's c and d) are not read.
 */

#ifdef __cplusplus
}
#endif
#endif
