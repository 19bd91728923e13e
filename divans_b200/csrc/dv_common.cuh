// dv_common.cuh -- shared definitions for the sm_90a divANS kernels.
//
// Data layout in HBM (per resident "slot" = the private model state of one stream while a lane-group
// decodes/encodes it; slots are recycled from stream to stream):
//
//   [LIT_HI  3*256*256 CDFs][LIT_LO 3*256*256 CDFs][LIT_CM 4352 CDFs][CTYPE 256 slabs x 32 CDFs]
//   [DPRIOR 256 slabs x 32 CDFs][MISC 128 CDFs][literal ctx map 16384 B][mixing mask 8192 B][distance ctx map 1024 B]
//
// A CDF is 16 x int16 = 32 B = one DRAM sector; lane i of a 16-lane group owns element i.
// The in-memory order of priors is NOT on the wire (reference: src/priors.rs:211-237 only fixes the index rule),
// so the encoder and the blend decoder lay the literal tables out [which][index_c][index_b]: one (which, index_c) "slab" is 256
// consecutive CDFs (8 KiB) and is default-initialised lazily by the kernel the first time the stream's context map /
// mixing mask makes it reachable -- no 12.6 MB memset per stream (the reference default-initialises all of it,
// codec/interface.rs:728-729).  The v2 engine orders each which-block by lit_index_hi / lit_index_lo (below).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dv {

constexpr uint32_t CDF_BYTES = 32;
constexpr uint64_t LIT_TABLE_CDFS = 3ull * 256 * 256;
constexpr uint64_t OFF_LIT_HI = 0;
constexpr uint64_t OFF_LIT_LO = OFF_LIT_HI + LIT_TABLE_CDFS * CDF_BYTES;
constexpr uint64_t OFF_LIT_CM = OFF_LIT_LO + LIT_TABLE_CDFS * CDF_BYTES;
constexpr uint64_t LIT_CM_CDFS = 256 + 16 * 256;   // FirstNibble[ctx], SecondNibble[H + 16*ctx]  (codec/priors.rs:45-47)
constexpr uint64_t OFF_CTYPE = OFF_LIT_CM + LIT_CM_CDFS * CDF_BYTES;
constexpr uint64_t SLAB32_BYTES = 32 * CDF_BYTES;   // per-command-block-type / per-distance-prior slab
constexpr uint64_t OFF_DPRIOR = OFF_CTYPE + 256 * SLAB32_BYTES;
constexpr uint64_t OFF_MISC = OFF_DPRIOR + 256 * SLAB32_BYTES;
constexpr uint64_t MISC_CDFS = 128;
constexpr uint64_t OFF_LCM = OFF_MISC + MISC_CDFS * CDF_BYTES;   // literal context map (== the recycled PredictionMode buffer)
constexpr uint64_t OFF_MIX = OFF_LCM + 16384;                     // mixing mask
constexpr uint64_t OFF_DCM = OFF_MIX + 8192;                      // distance context map
// v2 engine (dv2_*.cu*).  Literal priors carry a 16-bit GENERATION TAG in the free sign bits of their 16 elements (element i
// holds bit i of the tag in its bit 15; adaptive values stay below 2^15 for every speed the fast paths accept): a prior whose
// tag differs from the generation of the stream that owns the slot reads as the default CDF [4,8,...,64] and takes the
// stream's tag with its first write -- no per-stream initialisation of the 12.6 MB of literal priors, not even of the
// reachable slabs (round 1 wrote 640 KB of defaults per 64 KiB stream).  Streams whose speeds could wrap an i16 counter
// (they need all 16 bits) switch the slot to untagged priors (dv_engine.cuh: v2_make_untagged).
// OFF_T2: the per-stream context table T2[byte][class of the byte before] = literal_context_map[block type][lut0[byte] | class]
// (8 classes = the values of lut1, codec/literal.rs:87-117 in one lookup; each entry also carries the class of `byte` itself); OFF_HDR: what survives from launch to launch (generation counter, dirty flag).
constexpr uint64_t OFF_T2 = OFF_DCM + 1024;           // 2048 x u16: context | (class of the byte itself) << 8
constexpr uint64_t OFF_HDR = OFF_T2 + 4096;           // u32 generation counter, u32 "literal tables may hold untagged 16-bit values"
constexpr uint64_t OFF_SLOT_END = OFF_HDR + 64;
// Slots are 16 MiB apart and the arena is 16 MiB aligned: any address inside a slot is (high word of the slot : low word of
// the slot + offset), i.e. ONE 32-bit add in the decode loop instead of 64-bit pointer arithmetic (dv2_core.cuh).
constexpr uint64_t SLOT_STRIDE = 16ull << 20;
static_assert(OFF_SLOT_END <= SLOT_STRIDE, "slot layout exceeds the slot stride");
// Literal prior order of the v2 engine: the CDF index of prior (index_c, index_b) inside the 65536-CDF block of `which` (the
// block itself starts at which << 16; all three blocks use the same order).  Every v2 access to LIT_HI / LIT_LO -- the generic
// path and both fast loops -- goes through these two functions, so they cannot disagree.  The order is chosen so that the priors
// one stream actually uses share cache lines (a 128-byte line holds 4 CDFs):
//   high nibble: row (index_c - (index_b & 63)) & 255, column index_b.  For fixed index_b the row is a bijection of index_c.
//     Under LSB6 with the identity context map and a stride byte that is the previous byte (mixing values 4-15 with stride 1),
//     index_c = prev & 63 = index_b & 63: all 256 high priors of a stream are row 0, one contiguous 8 KiB run;
//   low nibble: row index_c (the high nibble, plus the context's low bits for mixing value 1), column index_b: for text the
//     hot rows (high nibble 2, 6, 7) hold runs of adjacent previous bytes.
// The encoder and the blend decoder keep [which][index_c][index_b] (dv_engine_kernel.cuh, enter_lit_nibble<..., false>).
__host__ __device__ __forceinline__ uint32_t lit_index_hi(uint32_t which, uint32_t index_c, uint32_t index_b) {
    (void)which;
    return (((index_c - (index_b & 63u)) & 255u) << 8) + index_b;
}
__host__ __device__ __forceinline__ uint32_t lit_index_lo(uint32_t which, uint32_t index_c, uint32_t index_b) {
    (void)which;
    return (index_c << 8) + index_b;
}

// CTYPE slab entries (indexed by the current command block type)
constexpr int CT_LL_COUNT_SMALL = 0, CT_LL_SIZE_BEG = 1, CT_LL_SIZE_LAST = 2, CT_LL_MANTISSA = 3;
constexpr int CT_CP_COUNT_SMALL = 4;   // +index 0..15
constexpr int CT_CP_COUNT_BEG = 20, CT_CP_COUNT_LAST = 21, CT_CP_COUNT_MANT = 22;   // +index 0..4
constexpr int CT_DC_SIZE_BEG = 27, CT_DC_SIZE_LAST = 28;
// DPRIOR slab entries (indexed by the distance context map value)
constexpr int DP_DIST_BEG = 0;        // +index 0..8
constexpr int DP_MNEMONIC = 16;       // +0..1
constexpr int DP_DIST_LAST = 18, DP_DIST_MANT = 19;   // +0..4
constexpr int DP_DICT_INDEX = 24;     // +0..4
// MISC entries
constexpr int MI_CC = 0;              // +last_4_states>>4
constexpr int MI_TRANSFORM = 16;      // + i0 + 2*i1
constexpr int MI_PRED = 48;           // + reference flat index 0..30 (codec/priors.rs:125-133)
constexpr int MI_BTYPE = 80;          // + reference flat index 0..9 (codec/priors.rs:106-110)
// PredictionModePriors flat offsets; DynamicContextMixingSpeed/PriorDepth are not listed in the reference's
// define_prior_struct! and therefore alias ContextMapSpeedPalette[0] (src/priors.rs:226-236)
constexpr int PM_ONLY = 0, PM_FIRST_NIBBLE = 2, PM_SECOND_NIBBLE = 4, PM_MNEMONIC = 6, PM_MIXING_VALUE = 10,
              PM_SPEED_PALETTE = 27;
constexpr int BT_MNEMONIC = 0, BT_FIRST = 3, BT_SECOND = 6, BT_STRIDE = 9;

// named speeds (probability/interface.rs:321-328)
#define DV_SPEED_MUD 0x10, 0x2000
#define DV_SPEED_SLOW 0x20, 0x1000
#define DV_SPEED_MED 0x30, 0x4000
#define DV_SPEED_FAST 0x60, 0x4000
#define DV_SPEED_PLANE 0x80, 0x4000
#define DV_SPEED_ROCKET 0x180, 0x4000

constexpr uint32_t NUM_SYMBOLS_BEFORE_FLUSH = 65536;   // ans.rs:57,138

// brotli tables blob offsets (tools/gen_brotli_tables.py)
constexpr uint32_t TB_SIZE_BITS = 24, TB_OFFSETS = 56, TB_CTX = 184, TB_TRANSFORMS = 2232, TB_PSMAP = 2616, TB_PS = 2744,
                   TB_DICT = 3000, TB_DICT_SIZE = 122784, TB_TOTAL = 125784;

enum : int32_t { ST_OK = 0, ST_NEED_INPUT = 1, ST_NEED_OUTPUT = 2, ST_FAIL = 3 };

struct DecodeParams {
    const uint8_t *in;
    const uint64_t *in_off, *in_len;
    uint8_t *out;
    const uint64_t *out_off, *out_cap;
    uint64_t *out_len;
    int32_t *status;
    const uint32_t *frame;      // per stream [4]: body_end, cmd payload bytes, lit payload bytes, payload base offset (frame kernel)
    const uint8_t *payload;     // compacted per-coder byte streams (demux kernel)
    uint32_t n_streams;
    uint32_t *work_counter;
    uint8_t *arena;             // n_slots * SLOT_STRIDE
    const uint8_t *tables;      // brotli tables blob
    uint64_t *nibble_counts;    // optional [2] totals (cmd, lit) for profiling
    uint32_t model_rev;         // 0 = the reference tree as mounted; 1 = DIVANS_B200_MODEL_WASM_2018 (include/divans_b200.h)
};

// Decoding to command lists: the recording decoder writes each stream's records into its blob region and counts them, the pack
// kernel turns that into the stream's DVCL blob (include/divans_b200.h).
struct RecParams {
    uint8_t *blobs;
    const uint64_t *blob_off, *blob_cap;
    uint64_t *blob_len;
    uint32_t *counts;           // per stream [3]: commands, prediction-mode records, literal bytes
};

struct FrameParams {
    const uint8_t *in;
    const uint64_t *in_off, *in_len;
    uint32_t *frame;            // per stream [4]: body_end, cmd payload bytes, lit payload bytes, reserved
    int32_t *status;
    uint32_t n_streams;
    uint32_t flags;
};

// Encoder (model pass -> reverse rANS pass -> mux/CRC pass).  Every stream owns `cmd_cap + lit_cap` u32 log entries
// (start | freq << 16, ans.rs:289-301): the command coder's log first, then the literal coder's.
struct EncodeParams {
    const uint8_t *in;            // raw bytes, or DVCL command-list blobs (include/divans_b200.h)
    const uint64_t *in_off, *in_len;
    int raw_mode;                 // 1: raw bytes + the internal literal-only command generator (raw_to_cmd/mod.rs:105-181)
    uint32_t n_streams;
    uint32_t *work_counter;
    uint8_t *arena;
    const uint8_t *tables;
    const uint8_t *pm_internal;   // raw mode: the one PredictionMode record every stream starts with
    uint32_t *sf; uint32_t cmd_cap, lit_cap;
    uint32_t *sf_counts;          // per stream: [n_cmd_syms, n_lit_syms]
    uint32_t *sf_dummy;           // per slot: where an idle group's core writes
    uint8_t *replay; uint64_t replay_stride;   // per slot: the encoder replays its commands to mirror last_8_literals
    uint32_t max_chunks;          // per stream: chunk records (cmd chunks first, then literal chunks)
    uint32_t cmd_chunks;          //   = ceil(cmd_cap / 65536)
    uint32_t *chunk_w;            // per chunk: first u32 entry of the chunk's renormalisation words (in place in the log)
    uint8_t *chunk_state;         // per chunk: the 16 bytes of final states that precede them
    const uint64_t *rcp15;        // floor((2^64 - 1) / f) for f < 32768 (reverse rANS pass)
    uint32_t *emit_bits;          // per (chunk, state): 1024 words, bit i = the state's i-th symbol from the end emitted a word
    uint8_t *out; const uint64_t *out_off, *out_cap; uint64_t *out_len;
    int32_t *status;
    // options (reference: DivansCompressorOptions, src/interface.rs:444-484)
    int window_size, dynamic_context_mixing, prior_depth, use_context_map, force_stride, have_literal_adaptation;
    int literal_adaptation[4];    // packed inc | lim << 16
    int model_rev;                // see DecodeParams::model_rev
    // command lists: window_size 0 = each stream takes the window of its blob header (clamped to 10..24); a blob longer than
    // max_in_len (the bound cmd_cap / lit_cap were derived from) is refused unread
    uint64_t max_in_len;
    uint32_t *stream_window;      // per stream: the window the model pass coded it with (the mux writes it into the header)
    // raw mode: stream v starts with record pm_internal + pm_index[v] * PM_RECORD_BYTES (nullptr: record 0 for every stream).
    // command lists: stream v codes every PredictionMode command with that one record instead of the list's own, unless bit
    // pm_index[v] of pm_keep is set (nullptr: every stream keeps its records)
    const uint32_t *pm_index;
    uint32_t pm_keep;
    // cost-only model pass (encode_model_kernel<BLEND, true>): no logs; per stream the sum of cost_tab[freq] over every coded
    // nibble of both coders, in 1/65536 bit (cost_tab[f] = -log2(f / 32768), include/divans_b200.h)
    const uint32_t *cost_tab;
    uint64_t *tally;
};
constexpr uint32_t PM_RECORD_BYTES = 32 + 16384 + 1024 + 8192;

// Binned cost pass (encode_bins_kernel, divans_b200_encode_mixmap_*): the cost-only pass of n x k (stream, candidate) pairs,
// candidate-major (pair v = c * n + i), that also sums each literal nibble's cost into the bin of its mixing-mask index.
constexpr uint32_t MIX_ENTRIES = 8192;
struct BinParams {
    uint64_t *slot_bins;   // per slot: MIX_ENTRIES u64, cleared when the slot takes a pair
    uint64_t *best;        // per stream: MIX_ENTRIES packed (cost << 4) | c, atomicMin of every pair that did not fail
    uint64_t *bins_out;    // optional, per pair (stream i, candidate c) at (i * k + c) * MIX_ENTRIES: the bins; UINT64_MAX for a failed pair
    uint32_t n, k;
};
struct MixValues { uint8_t v[16]; uint32_t k; };   // the k (1..16) candidate mixing values of a mixmap call

}  // namespace dv
