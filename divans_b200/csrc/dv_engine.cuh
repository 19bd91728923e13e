// dv_engine.cuh -- lock-step warp engine for the divANS command codec (sm_90a).
//
// A warp runs two streams (one per 16-lane group) in LOCK STEP: every loop iteration the whole warp, converged under
// the compile-time mask 0xffffffff, codes exactly one nibble per group ("nibble core": CDF load, bin search by ballot,
// exact start/freq by two shuffles, rANS step, adaptive blend, store).  Between two cores each group runs its own
// scalar state machine ("transition": what does the decoded nibble mean, which prior comes next), which is ordinary
// divergent SIMT code without warp collectives.  This is the reference's own structure -- every command codec is a
// resumable sub-state machine (LiteralSubstate codec/literal.rs:29-40, CopySubstate copy.rs:19-31, DictSubstate
// dict.rs:22-31, BlockTypeState block_type.rs:19-24, PredictionModeSubstate context_map.rs:30-41, EncodeOrDecodeState
// codec/mod.rs:114-130) -- mapped onto SIMT: the part that needs the 16 lanes is converged, the part that is scalar
// control flow is allowed to diverge.
//
// The same state machine is the encoder (ENC=true): the symbol comes from the command list instead of the rANS state
// and (start,freq) pairs are logged for the reverse rANS pass (ans.rs:279-301,331-378).
#pragma once
#include "dv_model.cuh"

namespace dv {

constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ uint32_t bitlen32(uint32_t v) { return v ? 32u - (uint32_t)__clz((int)v) : 0u; }
__device__ __forceinline__ uint32_t round_up_mod_4(uint32_t v) { return ((((v - 1u) & 0xffu) | 3u) + 1u) & 0xffu; }   // codec/interface.rs:180-182 (u8)

// ---------------------------------------------------------------------------------------------------------------
// states (one nibble is coded in each; the comment names the reference substate)
// ---------------------------------------------------------------------------------------------------------------
enum : int {
    S_IDLE = 0,          // no stream / finished
    S_CMD_TYPE,          // EncodeOrDecodeState::Begin                                  codec/mod.rs:662-688
    S_LIT_HI, S_LIT_LO,  // LiteralNibbleIndex (code_nibble_array)                      codec/literal.rs:261-394
    S_LL_COUNT_SMALL, S_LL_SIZE_BEG, S_LL_SIZE_LAST, S_LL_MANT,                       // codec/literal.rs:565-661
    S_CP_COUNT_SMALL, S_CP_COUNT_BEG, S_CP_COUNT_LAST, S_CP_COUNT_MANT,               // codec/copy.rs:87-162
    S_CP_MNEMONIC, S_CP_DIST_BEG, S_CP_DIST_LAST, S_CP_DIST_MANT,                     // codec/copy.rs:166-280
    S_DC_SIZE_BEG, S_DC_SIZE_LAST, S_DC_INDEX, S_DC_TR_HI, S_DC_TR_LO,                // codec/dict.rs:81-170
    S_BT_MNEMONIC, S_BT_FIRST, S_BT_SECOND, S_BT_STRIDE,                              // codec/block_type.rs:61-110,170-190
    S_PM_MODE, S_PM_MIX, S_PM_DEPTH, S_PM_SPEED, S_PM_MAP_MNEMONIC, S_PM_MAP_FIRST, S_PM_MAP_SECOND, S_PM_MIXVAL,   // context_map.rs:172-425
    S_DICT_EMIT,         // no nibble: second half of the dictionary replay
};

struct Speed1 { int v; };   // inc | lim<<16
__device__ __forceinline__ int sp_pack(int inc, int lim) { return (inc & 0xffff) | (lim << 16); }
#define SPK_MUD sp_pack(0x10, 0x2000)
#define SPK_SLOW sp_pack(0x20, 0x1000)
#define SPK_MED sp_pack(0x30, 0x4000)
#define SPK_FAST sp_pack(0x60, 0x4000)
#define SPK_PLANE sp_pack(0x80, 0x4000)
#define SPK_ROCKET sp_pack(0x180, 0x4000)

// What the core has to code next for this group
struct Next {
    int16_t *cdf;      // prior in HBM (never null: "no prior" cases point at the slot's flat / dummy CDFs with SPK_NONE)
    int16_t *cdf2;     // context-map prior when dynamic context mixing >= 2 (literal.rs:219-243); else nullptr
    int speed;         // inc | lim<<16 for `cdf`; SPK_NONE = read-only (mm_opts == 2: literal.rs:213-216,252-256)
    int sym;           // ENC: symbol to code
    bool mix_hi;       // mixing: which of the two weight sets / cm speeds (true = high nibble)
    bool tagged;       // v2 engine: `cdf` is a literal prior that carries a generation tag in its sign bits (dv_common.cuh)
};
// A blend with inc 0 and an unreachable limit leaves the CDF bit-identical: "do not adapt" without a branch.
#define SPK_NONE sp_pack(0, 0x7fff)
constexpr int MI_FLAT = 126;    // MISC slot that always holds the default CDF (coded with SPK_NONE)
constexpr int MI_DUMMY = 127;   // MISC slot idle groups "code" against while their warp-mate still works

// encoder input (DVCL blob, include/divans_b200.h)
struct CmdIn {
    const uint32_t *cmds;    // 5 x u32 per command
    uint32_t n_cmds, pos, n_pms;
    uint32_t pm_mask;        // ~0: PredictionMode command k reads record k of `pms`; 0: every one reads record 0 (raw mode, or a
                             // list whose records a candidate literal model replaces; k is still checked against n_pms)
    const uint8_t *pms;      // prediction mode records (32 + 16384 + 1024 + 8192 each)
    const uint8_t *lits;     // literal pool
};
// recording decoder output: the DVCL blob region of the stream being decoded.  Command records grow forward from byte 32,
// prediction-mode records backward from the region's end; a record is written only while both ends stay apart, but every
// record is counted, so the pack kernel (dv_kernels.cu) knows the exact size the blob needs either way.
struct RecOut {
    uint8_t *blob;
    uint32_t cap;                            // region bytes (capped at 4 GiB - 1)
    uint32_t n_cmds, n_pms, n_lits;          // records so far; literal bytes so far
    uint32_t lit_map_len, dist_map_len;      // the index at which each map's mnemonic 14 arrived (PredictionMode in flight)
};
static_assert(sizeof(RecOut) <= sizeof(CmdIn) && alignof(RecOut) <= alignof(CmdIn), "RecOut shares CmdIn's storage");

// Per-stream state, split by temperature.
//  * Cold: everything only the command interpreter touches -- lives in SHARED memory (one struct per lane-group; every
//    lane of the group reads/writes the same word with the same value, so no synchronisation is needed).
//  * St:   what the per-nibble loop needs -- stays in registers (no address of it ever escapes).
// Keeping the cold two thirds out of the register file is what keeps the big transition switch from drowning in
// register-to-register moves at every control-flow merge.
struct Cold {
    Coder oth;                               // the parked coder (cmd coder while a literal is in flight, else the literal coder)
    bool cur_is_lit;
    // CrossCommandBookKeeping (codec/interface.rs:142-168)
    uint32_t lru0, lru1, lru2, lru3;        // distance_lru
    unsigned long long btype_lru;            // byte [2*k] = lru[k][0], byte [2*k+1] = lru[k][1], k=0 lit,1 cmd,2 dist
    uint32_t btype_max;                      // byte k = max_seen[k]
    uint32_t last_dlen, last_clen, last_llen, last_4_states;
    unsigned long long cmap_lo, cmap_hi;     // context-map LRU-13 as bytes: entries 0..7 in lo, 8..12 in hi
    // LiteralBookKeeping leftovers (codec/interface.rs:125-140)
    int ad_cm_lo, ad_cm_hi;                  // literal_adaptation[2], [3] packed
    Weights w_lo, w_hi;                      // model_weights[0], [1]
    uint32_t mixing_param;
    bool lit_slabs_ready;
    uint32_t out_cap, ring_len, raw_len;
    uint32_t lit_log_cap;                    // encoder: capacity (entries) of the literal coder's log
    uint32_t sidx;                           // stream index being processed
    uint32_t model_rev;                      // DecodeParams::model_rev
    uint32_t gen_ctr;                        // v2 engine: streams this slot has hosted (generation of the literal-prior tags)
    uint32_t lit_total;                      // v2 engine: length of the literal in flight
    bool lit_quirk;                          // v2 engine: the literal began within 8 bytes of the ring start (last_8_literals is not a plain mirror of the output)
    bool pm_seen;                            // a PredictionMode command of THIS stream has written the mixing mask
    bool t2_dirty;                           // v2 engine: the slot's context table (OFF_T2) does not match lcm / mode / block type
    // encoder input, or the recording decoder's output (a decoder never reads `in`)
    union { CmdIn in; RecOut rec; };
    uint32_t e0, e1, e2, e3;                 // current input command fields
    uint32_t desired_context_mixing, desired_prior_depth, desired_force_stride;
    bool desired_do_context_map, have_desired_adapt;
    int desired_adapt0, desired_adapt1, desired_adapt2, desired_adapt3;
    // lazily-initialised prior slabs: [0..47] literal, [48..55] ctype, [56..63] dprior, [64] flags; then dictionary scratch
    uint32_t bitmaps[66];
    uint8_t scratch[64];
};

struct St {
    Cold *c;
    int state;
    Coder cur;                               // the coder the current state codes with
    uint8_t *slot;                           // base of this group's arena slot
    const uint8_t *tables;
    unsigned long long l8;                   // last_8_literals
    uint32_t btype_last, pred_mode;
    int ad_stride;                           // literal_adaptation[0] packed
    bool mixing_trait;
    bool speeds_small;                       // every literal speed keeps adaptive values inside i16 (see speed_is_small)
    int lit_cfg;                             // >= 0: every mixing-mask entry is equal and this is its mm_cfg() (skip the table read)
    uint8_t *out;                            // output window
    uint32_t out_pos;
    int status;
    uint32_t f0, f1, f2, f3;                 // scratch of the command being coded (meaning depends on the state)
    uint32_t lit_left, lit_ctx, lit_h;       // literal in flight
    uint32_t gen;                            // v2 engine: 16-bit tag of the literal priors that belong to the current stream (never 0)
    bool tagged;                             // v2 engine: literal priors carry tags (false after v2_make_untagged)
};

// arena accessors
__device__ __forceinline__ int16_t *A_lit(const St &s, bool high) { return reinterpret_cast<int16_t *>(s.slot + (high ? OFF_LIT_HI : OFF_LIT_LO)); }
__device__ __forceinline__ int16_t *A_litcm(const St &s) { return reinterpret_cast<int16_t *>(s.slot + OFF_LIT_CM); }
__device__ __forceinline__ int16_t *A_misc(const St &s, int idx) { return reinterpret_cast<int16_t *>(s.slot + OFF_MISC) + idx * 16; }
__device__ __forceinline__ uint8_t *A_lcm(const St &s) { return s.slot + OFF_LCM; }
__device__ __forceinline__ uint8_t *A_mix(const St &s) { return s.slot + OFF_MIX; }
__device__ __forceinline__ uint8_t *A_dcm(const St &s) { return s.slot + OFF_DCM; }
__device__ __forceinline__ uint32_t BL(const St &s, int k, int j) { return (uint32_t)(s.c->btype_lru >> (8 * (2 * k + j))) & 0xffu; }
__device__ __forceinline__ uint32_t BMAX(const St &s, int k) { return (s.c->btype_max >> (8 * k)) & 0xffu; }

struct G2 {            // lane geometry of one lane-group (16 lanes: one CDF element per lane; 8 lanes: two per lane)
    int l16;           // lane index inside the group: lane & 15 (16 lanes per stream) or lane & 7 (8 lanes per stream)
    int shift;         // position of the group's ballot bits: 0 / 16, or 0 / 8 / 16 / 24
    unsigned gmask;    // this group's lanes
    bool store0;       // lane that performs the group's scalar stores
    int nl;            // lanes that share the group's loops: 16 or 8
    int grp;           // index of the group inside its block (= of its cold state in dynamic shared memory)
    bool blend;        // probability model: false = FrequentistCDF16, true = BlendCDF16 (dv_blend.cuh); a kernel template constant
};

// Dynamic shared memory of every kernel that runs groups (decoders, encoder, replay) starts with one Cold per group, at this
// stride.
constexpr int SMEM_BYTES_PER_GROUP = (int)((sizeof(Cold) + 15) / 16 * 16);
// The group's cold state, found from scratch.  The out-of-line helpers below use this instead of taking pointers into it: a
// generic pointer to shared memory costs two special-register reads to build, and the compiler builds the arguments of those
// (rare) calls at the head of every iteration of the main loop (~25 instructions per iteration).
__device__ __forceinline__ Cold *cold_of_group(const G2 g) {
    extern __shared__ __align__(16) uint8_t dv_dynamic_smem[];
    return reinterpret_cast<Cold *>(dv_dynamic_smem + (unsigned)g.grp * (size_t)SMEM_BYTES_PER_GROUP);
}

// ---------------------------------------------------------------------------------------------------------------
// out-of-line helpers (take plain values, never a reference to St)
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void store_default_cdfs(const G2 g, int16_t *base, uint32_t n_cdfs) {
    const uint4 lo = make_uint4(0x00080004u, 0x0010000cu, 0x00180014u, 0x0020001cu);   // [4,8,...,64], frequentist_cdf.rs:17-23
    const uint4 hi = make_uint4(0x00280024u, 0x0030002cu, 0x00380034u, 0x0040003cu);
    const uint4 z = make_uint4(0, 0, 0, 0);                                              // BlendCDF16::default(), blend_cdf.rs:128-136
    uint4 *p = reinterpret_cast<uint4 *>(base);
    uint32_t n16 = n_cdfs * 2;
    for (uint32_t i = g.l16; i < n16; i += g.nl) p[i] = g.blend ? z : ((i & 1) ? hi : lo);
}
static __device__ __noinline__ void init_slab32(const G2 g, int16_t *p, uint32_t first_word, uint32_t idx) {
    uint32_t *bm = cold_of_group(g)->bitmaps + first_word;
    store_default_cdfs(g, p, 32);
    __syncwarp(g.gmask);
    if (g.store0) bm[idx >> 5] |= 1u << (idx & 31);
    __syncwarp(g.gmask);
}
__device__ __forceinline__ int16_t *ctype_slab(const St &s, const G2 g, uint32_t ctype) {
    int16_t *p = reinterpret_cast<int16_t *>(s.slot + OFF_CTYPE) + (size_t)ctype * 32 * 16;
    if (!((s.c->bitmaps[48 + (ctype >> 5)] >> (ctype & 31)) & 1u)) init_slab32(g, p, 48, ctype);
    return p;
}
__device__ __forceinline__ int16_t *dprior_slab(const St &s, const G2 g, uint32_t prior) {
    int16_t *p = reinterpret_cast<int16_t *>(s.slot + OFF_DPRIOR) + (size_t)prior * 32 * 16;
    if (!((s.c->bitmaps[56 + (prior >> 5)] >> (prior & 31)) & 1u)) init_slab32(g, p, 56, prior);
    return p;
}
__device__ __forceinline__ uint32_t get_distance_prior(const St &s, uint32_t copy_len) {   // codec/interface.rs:426-430
    uint32_t m = copy_len < 2 ? 2 : copy_len;
    m -= 2; if (m > 3) m = 3;
    return A_dcm(s)[BL(s, 2, 0) * 4 + m];
}

// Default-initialise every literal-prior slab the current context map / mixing mask can reach; returns the uniform
// mixing value (or -1).  Every lane scans the maps itself (no collectives: this runs in divergent transition code).
static __device__ __noinline__ int ensure_literal_slabs(const G2 g, uint8_t *slot, bool mixing_trait) {
    uint32_t *bitmaps = cold_of_group(g)->bitmaps;
    uint32_t mx4 = 0;
    const uint4 *m4 = reinterpret_cast<const uint4 *>(slot + OFF_LCM);
    for (uint32_t i = 0; i < 1024; i++) {
        uint4 v = m4[i];
        mx4 = __vmaxu4(mx4, __vmaxu4(__vmaxu4(v.x, v.y), __vmaxu4(v.z, v.w)));
    }
    uint32_t mx = max(max(mx4 & 0xff, (mx4 >> 8) & 0xff), max((mx4 >> 16) & 0xff, mx4 >> 24));
    uint32_t present = 0;
    const uint4 *x4 = reinterpret_cast<const uint4 *>(slot + OFF_MIX);
    for (uint32_t i = 0; i < 512; i++) {
        uint4 v = x4[i];
        uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; j++) {
            present |= 1u << (w[j] & 15); present |= 1u << ((w[j] >> 8) & 15);
            present |= 1u << ((w[j] >> 16) & 15); present |= 1u << ((w[j] >> 24) & 15);
        }
    }
    // which: mm 0,3 -> 0 ; mm 1 -> 2 ; everything else -> 1   (codec/literal.rs:184-208)
    bool w0 = present & 0x9u, w2 = present & 0x2u, w1 = present & ~0xBu;
    int16_t *lit_hi = reinterpret_cast<int16_t *>(slot + OFF_LIT_HI), *lit_lo = reinterpret_cast<int16_t *>(slot + OFF_LIT_LO);
    for (uint32_t which = 0; which < 3; which++) {
        if (!(which == 0 ? w0 : (which == 1 ? w1 : w2))) continue;
        uint32_t lo_max = which == 2 ? (min(mx, 15u) << 4 | 15u) : 15u;
        for (uint32_t c = 0; c <= mx; c++) {
            uint32_t id = which * 256 + c;
            if (!((bitmaps[id >> 5] >> (id & 31)) & 1u)) {
                store_default_cdfs(g, lit_hi + (size_t)id * 256 * 16, 256);
                __syncwarp(g.gmask);
                if (g.store0) bitmaps[id >> 5] |= 1u << (id & 31);
                __syncwarp(g.gmask);
            }
        }
        for (uint32_t c = 0; c <= lo_max; c++) {
            uint32_t id = 768 + which * 256 + c;
            if (!((bitmaps[id >> 5] >> (id & 31)) & 1u)) {
                store_default_cdfs(g, lit_lo + (size_t)(which * 256 + c) * 256 * 16, 256);
                __syncwarp(g.gmask);
                if (g.store0) bitmaps[id >> 5] |= 1u << (id & 31);
                __syncwarp(g.gmask);
            }
        }
    }
    if (mixing_trait && !(bitmaps[64] & 1u)) {   // lit_cm_priors are allocated on the first mixing>=2 (codec/interface.rs:322-329)
        store_default_cdfs(g, reinterpret_cast<int16_t *>(slot + OFF_LIT_CM), (uint32_t)LIT_CM_CDFS);
        __syncwarp(g.gmask);
        if (g.store0) bitmaps[64] |= 1u;
    }
    __syncwarp(g.gmask);
    return (present & (present - 1)) == 0 ? (__ffs(present) - 1) : -1;
}

// v2 engine: what ensure_literal_slabs finds out without initialising anything (the literal priors are tagged):
// the uniform mixing value (or -1); the context-map priors of dynamic context mixing >= 2 are still defaulted eagerly, once.
static __device__ __noinline__ int scan_literal_config(const G2 g, uint8_t *slot, bool mixing_trait) {
    uint32_t *bitmaps = cold_of_group(g)->bitmaps;
    uint32_t present = 0;
    const uint4 *x4 = reinterpret_cast<const uint4 *>(slot + OFF_MIX);
    for (uint32_t i = 0; i < 512; i++) {
        uint4 v = x4[i];
        uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; j++) {
            present |= 1u << (w[j] & 15); present |= 1u << ((w[j] >> 8) & 15);
            present |= 1u << ((w[j] >> 16) & 15); present |= 1u << ((w[j] >> 24) & 15);
        }
    }
    if (mixing_trait && !(bitmaps[64] & 1u)) {   // lit_cm_priors are allocated on the first mixing>=2 (codec/interface.rs:322-329)
        store_default_cdfs(g, reinterpret_cast<int16_t *>(slot + OFF_LIT_CM), (uint32_t)LIT_CM_CDFS);
        __syncwarp(g.gmask);
        if (g.store0) bitmaps[64] |= 1u;
    }
    __syncwarp(g.gmask);
    return (present & (present - 1)) == 0 ? (__ffs(present) - 1) : -1;
}

// v2 engine: every literal prior of the slot becomes "never written" (tag 0 never matches a generation)
static __device__ __noinline__ void v2_clear_literal_tables(const G2 g, uint8_t *slot) {
    uint4 *p = reinterpret_cast<uint4 *>(slot + OFF_LIT_HI);
    const uint4 z = make_uint4(0, 0, 0, 0);
    for (uint32_t i = (uint32_t)g.l16; i < (uint32_t)(2 * LIT_TABLE_CDFS * CDF_BYTES / 16); i += (uint32_t)g.nl) p[i] = z;
    __syncwarp(g.gmask);
}
// v2 engine: a stream whose speeds can wrap i16 counters needs all 16 bits of every element.  Priors of the current generation
// lose their tag bits, every other prior becomes the default CDF, and every slab is marked initialised (the bitmaps the
// [which][index_c][index_b] layout keeps, dv_common.cuh).  From here on the stream's literal priors are plain i16 arrays.
static __device__ __noinline__ void v2_make_untagged(const G2 g, uint8_t *slot, uint32_t gen) {
    uint32_t *bitmaps = cold_of_group(g)->bitmaps;
    uint32_t *p = reinterpret_cast<uint32_t *>(slot + OFF_LIT_HI);
    const uint32_t n_cdf = (uint32_t)(2 * LIT_TABLE_CDFS);
    for (uint32_t c = (uint32_t)g.l16; c < n_cdf; c += (uint32_t)g.nl) {     // one CDF (8 words) per lane and step
        uint32_t w[8], tag = 0;
        for (int k = 0; k < 8; k++) { w[k] = p[(size_t)c * 8 + k]; tag |= ((w[k] >> 15) & 1u) << (2 * k) | ((w[k] >> 31) & 1u) << (2 * k + 1); }
        const bool mine = tag == gen;
        for (int k = 0; k < 8; k++) p[(size_t)c * 8 + k] = mine ? (w[k] & 0x7fff7fffu) : ((uint32_t)(8 * k + 4) | ((uint32_t)(8 * k + 8) << 16));
    }
    __syncwarp(g.gmask);
    for (uint32_t i = (uint32_t)g.l16; i < 48; i += (uint32_t)g.nl) bitmaps[i] = 0xffffffffu;
    if (g.store0) reinterpret_cast<uint32_t *>(slot + OFF_HDR)[1] = 1u;       // the next stream must not trust sign bits in this slot
    __syncwarp(g.gmask);
}

// fresh arena state for a new stream: zero the maps (ffi/alloc_util.rs:70-99), clear slab bitmaps, default the dense priors
// Slot header words (OFF_HDR, persistent): [0] generation counter, [1] literal tables may hold untagged 16-bit values,
// [2] literal-context-map bytes written since the map was last zeroed, [3] the mixing mask holds values of an earlier stream.
static __device__ __noinline__ void reset_slot(const G2 g, uint8_t *slot) {
    uint32_t *bitmaps = cold_of_group(g)->bitmaps;
    uint4 z = make_uint4(0, 0, 0, 0);
    uint4 *p = reinterpret_cast<uint4 *>(slot + OFF_LCM);
    for (uint32_t i = g.l16; i < (16384 + 8192 + 1024) / 16; i += g.nl) p[i] = z;   // lcm, mix, dcm are contiguous
    for (uint32_t i = g.l16; i < 65; i += g.nl) bitmaps[i] = 0;
    store_default_cdfs(g, reinterpret_cast<int16_t *>(slot + OFF_MISC), (uint32_t)MISC_CDFS);
    if (g.store0) {
        uint32_t *hdr = reinterpret_cast<uint32_t *>(slot + OFF_HDR); hdr[2] = 0; hdr[3] = 0;
        if (g.blend) hdr[1] = 1u;   // blend priors keep their step count in sign bits: the v2 engine must wipe before trusting tags
    }
    __syncwarp(g.gmask);
}
// v2 engine: the same fresh state without streaming 25 KB of zeros through L2 per stream.  Only the part of the literal context
// map that earlier streams wrote is zeroed (header word 2: 64 bytes for the usual one-block-type map); the mixing mask is
// left alone until it is needed -- a PredictionMode command rewrites all 8192 values, a literal that arrives before any
// such command zeroes it first (v2_mix_before_use).
static __device__ __noinline__ void reset_slot_v2(const G2 g, uint8_t *slot) {
    uint32_t *bitmaps = cold_of_group(g)->bitmaps;
    uint32_t *hdr = reinterpret_cast<uint32_t *>(slot + OFF_HDR);
    const uint4 z = make_uint4(0, 0, 0, 0);
    const uint32_t lcm16 = (min(hdr[2], 16384u) + 15u) / 16u;
    uint4 *p = reinterpret_cast<uint4 *>(slot + OFF_LCM);
    for (uint32_t i = g.l16; i < lcm16; i += g.nl) p[i] = z;
    uint4 *d = reinterpret_cast<uint4 *>(slot + OFF_DCM);
    for (uint32_t i = g.l16; i < 1024 / 16; i += g.nl) d[i] = z;
    for (uint32_t i = g.l16; i < 65; i += g.nl) bitmaps[i] = 0;
    store_default_cdfs(g, reinterpret_cast<int16_t *>(slot + OFF_MISC), (uint32_t)MISC_CDFS);
    __syncwarp(g.gmask);
    if (g.store0) hdr[2] = 0;
    __syncwarp(g.gmask);
}
static __device__ __noinline__ void v2_mix_before_use(const G2 g, uint8_t *slot) {
    uint32_t *hdr = reinterpret_cast<uint32_t *>(slot + OFF_HDR);
    if (hdr[3] != 0) {
        const uint4 z = make_uint4(0, 0, 0, 0);
        uint4 *p = reinterpret_cast<uint4 *>(slot + OFF_MIX);
        for (uint32_t i = g.l16; i < 8192 / 16; i += g.nl) p[i] = z;
        __syncwarp(g.gmask);
        if (g.store0) hdr[3] = 0;
    }
    __syncwarp(g.gmask);
}

// copy replay (cmd_to_raw/mod.rs:245-283): out[pos+i] = out[pos-dist+(i mod dist)] -- the copied region is periodic with
// period `dist` and its first period already exists, so the lanes copy independently (overlap included).
static __device__ __noinline__ void replay_copy(const G2 g, uint8_t *out, uint32_t pos, uint32_t dist, uint32_t len) {
    long long base = (long long)pos - (long long)dist;
    uint8_t *dst = out + pos;
    uint32_t off = (uint32_t)g.l16 % dist;
    uint32_t step = (uint32_t)g.nl % dist;
    for (uint32_t i = (uint32_t)g.l16; i < len; i += g.nl) {
        long long sp = base + (long long)off;
        dst[i] = sp >= 0 ? out[sp] : (uint8_t)0;   // a fresh ring is zero-initialised (ffi/alloc_util.rs:70-99)
        off += step; if (off >= dist) off -= dist;
    }
}

// dictionary word + RFC 7932 transform into `scratch` by the group's first lane (cmd_to_raw/mod.rs:284-309; the
// transform itself is the brotli crate's TransformDictionaryWord, NOT-IN-TREE); returns the length or -1
static __device__ __noinline__ int dict_word(const G2 g, const uint8_t *tb, uint32_t word_size, uint32_t word_id, uint32_t transform) {
    uint8_t *o = cold_of_group(g)->scratch;
    if (word_size < 4 || word_size > 24 || transform >= 121) return -1;
    uint64_t widx = (uint64_t)word_id * word_size + reinterpret_cast<const uint32_t *>(tb + TB_OFFSETS)[word_size];
    if (widx + word_size > TB_DICT_SIZE) return -1;
    const uint8_t *word = tb + TB_DICT + widx;
    const uint8_t *tr = tb + TB_TRANSFORMS + 3 * transform;
    const uint16_t *psmap = reinterpret_cast<const uint16_t *>(tb + TB_PSMAP);
    const uint8_t *prefix = tb + TB_PS + psmap[tr[0]], *suffix = tb + TB_PS + psmap[tr[2]];
    int n = 0, t = tr[1], len = (int)word_size;
    for (int i = 0; i < 64; i++) o[i] = 0;
    { int pl = *prefix++; while (pl--) o[n++] = *prefix++; }
    int skip = t < 12 ? 0 : t - 11; if (skip > len) skip = len;
    word += skip; len -= skip; if (t <= 9) len -= t;
    for (int i = 0; i < len; i++) o[n++] = word[i];
    if (len > 0 && (t == 10 || t == 11)) {
        uint8_t *up = o + n - len; int rem = t == 10 ? 1 : len;
        while (rem > 0) {
            int step;
            if (up[0] < 0xc0) { if (up[0] >= 'a' && up[0] <= 'z') up[0] ^= 32; step = 1; }
            else if (up[0] < 0xe0) { up[1] ^= 32; step = 2; }
            else { up[2] ^= 5; step = 3; }
            up += step; rem -= step;
            if (t == 10) break;
        }
    }
    { int sl = *suffix++; while (sl--) o[n++] = *suffix++; }
    return n;
}

// f8 speed codec (probability/interface.rs:566-585 and the brotli crate's u16 twins used by the PredictionMode setters)
__device__ __forceinline__ int u8_to_speed(uint32_t data) {
    if (data < 8) return 0;
    uint32_t log_val = (data >> 3) - 1;
    int rem = (int)(short)((data & 7) << log_val);
    return (int)(short)((short)(1 << log_val) | (rem >> 3));
}
__device__ __forceinline__ uint32_t speed_to_u8_u16(uint32_t data) {
    data &= 0xffff;
    if (data == 0) return 0;
    uint32_t length = 32 - __clz((int)data);
    uint32_t rem = (data - (1u << (length - 1))) & 0xffff;
    uint32_t mant = (((rem << 3) & 0xffff) >> (length - 1)) & 0xff;
    return ((length << 3) | mant) & 0xff;
}
__device__ __forceinline__ uint32_t speed_to_u8_i16(int data) {
    uint32_t u = (uint32_t)data & 0xffff;
    uint32_t length = u ? 32 - __clz((int)u) : 0;
    uint32_t mant = 0;
    if (data != 0) {
        int rem = (int)(short)(data - (short)(1 << (length - 1)));
        mant = (uint32_t)(((int)(short)(rem << 3)) >> (length - 1)) & 0xff;
    }
    return ((length << 3) | mant) & 0xff;
}
__device__ __forceinline__ uint32_t u8_to_speed_u16(uint32_t data) {
    if (data < 8) return 0;
    uint32_t log_val = (data >> 3) - 1;
    uint32_t rem = ((data & 7) << log_val) & 0xffff;
    return ((1u << log_val) | (rem >> 3)) & 0xffff;
}
__device__ __forceinline__ int f8_pair_to_speed(uint32_t a, uint32_t b) {   // nibbles -> stored f8 -> Speed::from_f8_tuple
    uint32_t ra = speed_to_u8_u16(u8_to_speed_u16(a)), rb = speed_to_u8_u16(u8_to_speed_u16(b));
    return sp_pack(u8_to_speed(ra), u8_to_speed(rb));
}

// The literal fast loops adapt in plain 32-bit arithmetic; the reference wraps i16 (frequentist_cdf.rs:74-85).  The two agree
// as long as no adaptive value can leave [0, 0x7fff]: a value is at most lim - 1 + inc before a rescale and
// 3/4 * (value + 16) after one.  Speeds are carried by the stream (f8: up to 30720), so streams whose speeds could wrap
// take the generic core, which keeps the i16 wrap.
__device__ __forceinline__ bool speed_is_small(int packed) {
    const int inc = (int)(short)(packed & 0xffff), lim = packed >> 16;
    return inc >= 0 && lim >= 0 && lim + inc + 16 <= 0x7fff && 4 * (inc + 16) <= 0x7fff;
}

// context-map LRU-13 held as 13 bytes in two registers (codec/interface.rs:439-453)
__device__ __forceinline__ uint32_t cmap_get(const St &s, int i) { return i < 8 ? (uint32_t)(s.c->cmap_lo >> (8 * i)) & 0xff : (uint32_t)(s.c->cmap_hi >> (8 * (i - 8))) & 0xff; }
__device__ __forceinline__ void cmap_reset(St &s) { s.c->cmap_lo = 0x0706050403020100ull; s.c->cmap_hi = 0x0000000c0b0a0908ull; }
__device__ __forceinline__ int cmap_find_first(const St &s, uint32_t val) { for (int i = 0; i < 13; i++) if (cmap_get(s, i) == val) return i; return -1; }
__device__ __forceinline__ int cmap_find_last(const St &s, uint32_t val) { int r = -1; for (int i = 0; i < 13; i++) if (cmap_get(s, i) == val) r = i; return r; }
__device__ __forceinline__ uint32_t cmap_max(const St &s) { uint32_t m = 0; for (int i = 0; i < 13; i++) m = max(m, cmap_get(s, i)); return m; }
__device__ __forceinline__ void cmap_touch(St &s, uint32_t val) {
    int f = cmap_find_first(s, val);
    if (f < 0) f = 12;
    // entries 1..f take entries 0..f-1; entry 0 = val
    unsigned long long lo = s.c->cmap_lo, hi = s.c->cmap_hi;
    unsigned long long nlo, nhi;
    if (f < 8) {
        unsigned long long keep = f == 7 ? 0ull : (lo >> (8 * (f + 1))) << (8 * (f + 1));
        unsigned long long moved = (lo << 8) & (f == 7 ? ~0ull : ((1ull << (8 * (f + 1))) - 1));
        nlo = keep | moved | val; nhi = hi;
        nlo = (nlo & ~0xffull) | val;
    } else {
        nlo = (lo << 8) | val;
        int fh = f - 8;   // 0..4
        unsigned long long carry = lo >> 56;
        unsigned long long keep = (hi >> (8 * (fh + 1))) << (8 * (fh + 1));
        unsigned long long moved = ((hi << 8) | carry) & ((1ull << (8 * (fh + 1))) - 1);
        nhi = keep | moved;
    }
    s.c->cmap_lo = nlo; s.c->cmap_hi = nhi & 0x000000ffffffffffull;
}

}  // namespace dv
