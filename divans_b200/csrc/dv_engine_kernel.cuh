// dv_engine_kernel.cuh -- the lock-step stream kernel (decoder and encoder model pass), see dv_engine.cuh.
#pragma once
#include "dv_engine.cuh"

namespace dv {


// ---------------------------------------------------------------------------------------------------------------
// transition helpers (all force-inlined into the kernel; St lives in registers)
// ---------------------------------------------------------------------------------------------------------------
// Fetch the next input command (encoder).  Either a record of the DVCL blob, or -- raw mode -- the commands of the
// reference's internal literal-only generator (raw_to_cmd/mod.rs:105-181): one PredictionMode, then one Literal per
// ring-buffer fill.
template <bool ENC>
__device__ __forceinline__ int load_cmd(St &s) {
    if (!ENC) return 0;
    const uint32_t pos = s.c->in.pos;
    if (s.c->in.cmds) {
        const uint32_t *c = s.c->in.cmds + 5 * (size_t)pos;
        s.c->e0 = c[1]; s.c->e1 = c[2]; s.c->e2 = c[3]; s.c->e3 = c[4];
        if (c[0] == 7u && c[1] >= s.c->in.n_pms) return 0;   // prediction-mode record out of range: not a command -> failure
        return (int)c[0];
    }
    if (pos == 0) { s.c->e0 = 0; s.c->e1 = 0; s.c->e2 = 0; s.c->e3 = 0; return 7; }
    const uint32_t off = (pos - 1) * s.c->ring_len;
    s.c->e0 = off; s.c->e1 = min(s.c->ring_len, s.c->raw_len - off); s.c->e2 = 0; s.c->e3 = 0;
    return 3;
}
template <bool ENC>
__device__ __forceinline__ void enter_cmd_type(St &s, Next &nx) {
    s.state = S_CMD_TYPE;
    nx.cdf = A_misc(s, MI_CC + (int)(s.c->last_4_states >> 4)); nx.cdf2 = nullptr; nx.speed = SPK_ROCKET; nx.tagged = false;
    if (ENC) {
        if (s.c->in.pos < s.c->in.n_cmds) nx.sym = load_cmd<ENC>(s);
        else nx.sym = 0xf;   // end of stream nibble (codec/mod.rs:143-148, flush :424-455)
    }
}

// mixing-mask value -> packed selector fields (codec/literal.rs:184-208):
//   bits 0-1 which, bits 2-7 shift of the stride byte inside last_8_literals, bit 8 mm, bit 9 opt_1_f, bit 10 fast_cm
__device__ __forceinline__ int mm_cfg(uint32_t mm_opts) {
    uint32_t mm = (mm_opts != 0 && mm_opts != 3) ? 1u : 0u;
    uint32_t o1 = (mm_opts == 1) ? 1u : 0u;
    uint32_t fc = (mm_opts != 3) ? 1u : 0u;
    uint32_t stride_offset = mm_opts < 4 ? 0u : (min(7u, mm_opts ^ 4u) << 3);
    uint32_t which = mm ^ (o1 ? 3u : 0u);
    uint32_t ro = (mm_opts == 2) ? 1u : 0u;   // bit 11: coder uses the flat CDF / stride prior is not adapted
    return (int)(which | ((0x38u - stride_offset) << 2) | (mm << 8) | (o1 << 9) | (fc << 10) | (ro << 11));
}
// literal nibble prior selection (codec/literal.rs:154-259)
template <bool ENC, bool HIGH, bool V2 = false>
__device__ __forceinline__ void enter_lit_nibble(St &s, Next &nx) {
    const uint32_t ctx = s.lit_ctx;
    int cfg = s.lit_cfg;
    if (cfg < 0) {
        uint32_t prev_byte = (uint32_t)(s.l8 >> 56);
        cfg = mm_cfg(A_mix(s)[ctx | (HIGH ? ((prev_byte >> 4) << 8) : (((s.lit_h & 0xf) << 8) | 4096u))]);
    }
    const uint32_t mm = (cfg & 0x100) ? 0xffu : 0u, o1 = (cfg & 0x200) ? 0xfu : 0u, fc = (cfg & 0x400) ? 0xffu : 0u;
    const uint32_t ssb = (uint32_t)(s.l8 >> ((cfg >> 2) & 63)) & 0xffu;
    uint32_t index_b, index_c;
    if (HIGH) { index_b = ssb & mm & (~o1 & 0xffu); index_c = ctx; }
    else { index_b = (mm & ssb) | ((~mm & 0xffu) & ctx); index_c = (s.lit_h & fc) | ((ctx & o1) << 4); }
    const uint32_t which = (uint32_t)cfg & 3u;
    // v2 engine: the order of lit_index_hi / lit_index_lo (dv_common.cuh), shared with the fast loops
    const uint32_t flat = V2 ? (which << 16) + (HIGH ? lit_index_hi(which, index_c, index_b) : lit_index_lo(which, index_c, index_b))
                             : (which * 256 + index_c) * 256 + index_b;
    int16_t *np = A_lit(s, HIGH) + (size_t)flat * 16;
    const bool ro = (cfg & 0x800) != 0;
    nx.mix_hi = HIGH;
    // (the never-adapted flat prior of mixing value 2 is MI_FLAT, untagged; with dynamic context mixing the stride prior is still READ)
    nx.tagged = V2 && s.tagged && (s.mixing_trait || !ro);
    if (s.mixing_trait) {
        nx.cdf = np; nx.speed = ro ? SPK_NONE : s.ad_stride;
        nx.cdf2 = HIGH ? A_litcm(s) + (size_t)ctx * 16 : A_litcm(s) + (size_t)(256 + s.lit_h + 16 * ctx) * 16;
    } else {
        nx.cdf = ro ? A_misc(s, MI_FLAT) : np; nx.speed = ro ? SPK_NONE : s.ad_stride;
        nx.cdf2 = nullptr;
    }
    if (ENC) {
        uint32_t byte = s.lit_left ? s.c->in.lits[s.c->e0 + (s.c->e1 - s.lit_left)] : 0u;   // (called once more after the last byte)
        nx.sym = HIGH ? (int)(byte >> 4) : (int)(byte & 0xf);
    }
    s.state = HIGH ? S_LIT_HI : S_LIT_LO;
}
__device__ __forceinline__ void lit_context(St &s) {   // get_prev_word_context, codec/literal.rs:87-117
    uint32_t prev = (uint32_t)(s.l8 >> 56), pp = (uint32_t)(s.l8 >> 48) & 0xff;
    uint32_t sel;
    if (s.pred_mode == 0) sel = prev & 0x3f;                 // LSB6  (codec/interface.rs:214-217)
    else if (s.pred_mode == 1) sel = prev >> 2;              // MSB6  (:210-213)
    else { const uint8_t *lut = s.tables + TB_CTX + 512 * s.pred_mode; sel = __ldg(lut + prev) | __ldg(lut + 256 + pp); }   // UTF8 / SIGN
    s.lit_ctx = A_lcm(s)[sel + (s.btype_last << 6)];
}
__device__ __forceinline__ unsigned long long reseed_last8(const St &s) {
    // codec/decoder.rs:361-375 + cmd_to_raw/mod.rs:69-86 (byte order flips when ring_buffer_decode_index < 8)
    uint32_t idx = s.out_pos & (s.c->ring_len - 1);
    unsigned long long v = 0;
    if (idx < 8) {
        for (uint32_t i = 0; i < 8; i++) {
            long long p = (long long)s.out_pos - 1 - (long long)i;
            unsigned long long b = p >= 0 ? s.out[p] : 0;
            v |= b << (8 * i);
        }
    } else {
        for (uint32_t i = 0; i < 8; i++) v |= (unsigned long long)s.out[s.out_pos - 8 + i] << (8 * i);
    }
    return v;
}
// The parked coder lives in the group's shared-memory state.  Every lane reads it, ONE lane writes the coder being parked (all
// lanes hold identical copies), with the group synchronised on both sides: single writer, no read of a half-written struct.
__device__ __forceinline__ void swap_coders(St &s, const G2 g) {
    const Coder parked = s.c->oth;
    const bool was_lit = s.c->cur_is_lit;
    __syncwarp(g.gmask);
    if (g.store0) { s.c->oth = s.cur; s.c->cur_is_lit = !was_lit; }
    __syncwarp(g.gmask);
    s.cur = parked;
}

// ---- recording decoder (REC): one DVCL record per command (include/divans_b200.h), the values the encoder reads back from
// it (load_cmd, pm_rec), written where the decoder resolves them.  A literal's `a` holds the output position of its bytes
// until the pack kernel (dv_kernels.cu) gathers them into the literal pool.
__device__ __forceinline__ void st_le32(uint8_t *p, uint32_t v) {   // blob regions may start at any byte
    p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24);
}
template <bool REC>
__device__ __forceinline__ void rec_cmd(St &s, const G2 g, uint32_t type, uint32_t a, uint32_t b, uint32_t c = 0, uint32_t d = 0) {
    if (!REC) return;
    RecOut &r = s.c->rec;
    const uint32_t k = r.n_cmds;
    if (g.store0 && 32ull + 20ull * (k + 1ull) + (uint64_t)PM_RECORD_BYTES * r.n_pms <= r.cap) {
        uint8_t *p = r.blob + 32 + 20ull * k;
        st_le32(p, type); st_le32(p + 4, a); st_le32(p + 8, b); st_le32(p + 12, c); st_le32(p + 16, d);
    }
    r.n_cmds = k + 1;
}
// The PredictionMode record of a decoded command: mode, has_speeds, the three speed pairs from the coded f8 bytes (`f8`
// byte 2k + j = pair k, element j; the stride and combined speeds are the same pairs), both maps with zeros past their
// lengths, the 8192 mixing values.  The group's lanes copy it out of the slot.
static __device__ __noinline__ void rec_predmode(const G2 g, const uint8_t *slot, uint8_t *dst, uint32_t pred_mode, unsigned long long f8,
                                                 uint32_t lit_len, uint32_t dist_len) {
    __syncwarp(g.gmask);   // the last mixing value, written by the group's store lane
    for (uint32_t i = (uint32_t)g.l16; i < 32; i += (uint32_t)g.nl) {
        uint32_t v;
        if (i < 4) v = i == 0 ? pred_mode : i == 2 ? 1u : 0u;
        else if (i < 28) {
            const uint32_t w = (i - 4) >> 1, pair = w < 4 ? w + 4 : (w - 4) & 3;   // cm_speed[2][2], stride_speed, combined_speed
            v = u8_to_speed_u16((uint32_t)(f8 >> (8 * pair)) & 0xffu) >> (8 * (i & 1));
        } else v = (i < 30 ? lit_len : dist_len) >> (8 * (i & 1));
        dst[i] = (uint8_t)v;
    }
    for (uint32_t i = (uint32_t)g.l16; i < 16384; i += (uint32_t)g.nl) dst[32 + i] = i < lit_len ? slot[OFF_LCM + i] : (uint8_t)0;
    for (uint32_t i = (uint32_t)g.l16; i < 1024; i += (uint32_t)g.nl) dst[32 + 16384 + i] = i < dist_len ? slot[OFF_DCM + i] : (uint8_t)0;
    for (uint32_t i = (uint32_t)g.l16; i < 8192; i += (uint32_t)g.nl) dst[32 + 16384 + 1024 + i] = slot[OFF_MIX + i];
    __syncwarp(g.gmask);
}
template <bool REC>
__device__ __forceinline__ void rec_pm(St &s, const G2 g) {
    if (!REC) return;
    RecOut &r = s.c->rec;
    const uint32_t j = r.n_pms;
    rec_cmd<REC>(s, g, 7, j, 0);
    if (32ull + 20ull * r.n_cmds + (uint64_t)PM_RECORD_BYTES * (j + 1ull) <= r.cap)
        rec_predmode(g, s.slot, r.blob + r.cap - (size_t)PM_RECORD_BYTES * (j + 1), s.f0, s.l8, r.lit_map_len, r.dist_map_len);
    r.n_pms = j + 1;
}

template <bool ENC, bool V2 = false, bool REC = false>
__device__ __forceinline__ void start_literal(St &s, Next &nx, const G2 g, uint32_t len) {
    if ((uint64_t)len > (uint64_t)(s.c->out_cap - s.out_pos)) { s.status = ST_NEED_OUTPUT; return; }
    if (REC) { rec_cmd<REC>(s, g, 3, s.out_pos, len, s.f3); s.c->rec.n_lits += len; }
    if (!s.c->lit_slabs_ready) {
        if (V2 && !s.c->pm_seen) v2_mix_before_use(g, s.slot);   // no PredictionMode command yet: the mask must read as zeros
        // v2 engine: literal priors carry generation tags and read as the default CDF until first written: nothing to initialise
        int u = (V2 && s.tagged) ? scan_literal_config(g, s.slot, s.mixing_trait) : ensure_literal_slabs(g, s.slot, s.mixing_trait);
        s.lit_cfg = u >= 0 ? mm_cfg((uint32_t)u) : -1; s.c->lit_slabs_ready = true;
    }
    s.l8 = reseed_last8(s);
    s.c->lit_quirk = (s.out_pos & (s.c->ring_len - 1)) < 8u; s.c->lit_total = len;
    swap_coders(s, g);
    s.lit_left = len;
    if (ENC) {
        s.c->e1 = len;
        // hostile command lists: the literal must lie inside the pool and its nibbles inside the log
        if ((uint64_t)s.c->e0 + len > s.c->raw_len || (uint64_t)s.cur.left + 2ull * len > s.c->lit_log_cap) { s.status = ST_FAIL; return; }
    }
    lit_context(s);
    enter_lit_nibble<ENC, true, V2>(s, nx);
}

__device__ __forceinline__ void obs_distance(St &s, uint32_t d) {   // codec/interface.rs:509-527
    if (d == s.c->lru1) { s.c->lru1 = s.c->lru0; s.c->lru0 = d; }
    else if (d == s.c->lru2) { s.c->lru2 = s.c->lru1; s.c->lru1 = s.c->lru0; s.c->lru0 = d; }
    else if (d != s.c->lru0) { s.c->lru3 = s.c->lru2; s.c->lru2 = s.c->lru1; s.c->lru1 = s.c->lru0; s.c->lru0 = d; }
}
__device__ __forceinline__ void distance_from_mnemonic(const St &s, uint32_t code, uint32_t &dist, bool &ok) {   // :979-1009
    if (code < 4) { dist = code == 0 ? s.c->lru0 : code == 1 ? s.c->lru1 : code == 2 ? s.c->lru2 : s.c->lru3; ok = true; return; }
    int us = (int)(code >> 2);
    int ss = us - (((-(int)(code & 1)) & us) << 1);
    int ret = (int)((code & 2) ? s.c->lru1 : s.c->lru0) + ss;
    dist = (uint32_t)ret; ok = ret > 0;
}
__device__ __forceinline__ void obs_btype(St &s, int k, uint32_t bt) {   // codec/interface.rs:528-532
    s.c->last_4_states >>= 2;
    unsigned long long old0 = BL(s, k, 0);
    uint32_t sh = 16 * k;
    s.c->btype_lru = (s.c->btype_lru & ~(0xffffull << sh)) | (((unsigned long long)bt | (old0 << 8)) << sh);
    if (bt > BMAX(s, k)) s.c->btype_max = (s.c->btype_max & ~(0xffu << (8 * k))) | (bt << (8 * k));
}

template <bool ENC> __device__ __forceinline__ void set_next(Next &nx, int16_t *cdf, int speed, int sym) {
    nx.cdf = cdf; nx.cdf2 = nullptr; nx.speed = speed; nx.tagged = false;
    if (ENC) nx.sym = sym;
}

// ---- "enter" functions: choose the prior of the next nibble (and, when encoding, the nibble itself) ----
template <bool ENC> __device__ __forceinline__ void enter_ll_count_small(St &s, Next &nx, const G2 g) {
    s.state = S_LL_COUNT_SMALL;
    uint32_t lm1 = s.c->e1 - 1u;
    int sym = (int)(lm1 < 14 ? lm1 : 14);
    if (ENC && s.c->e2 && !s.f3) sym = 15;   // high_entropy flag nibble (literal.rs:569-571)
    set_next<ENC>(nx, ctype_slab(s, g, BL(s, 1, 0)) + CT_LL_COUNT_SMALL * 16, SPK_MED, sym);
}
template <bool ENC> __device__ __forceinline__ void enter_ll_mant(St &s, Next &nx, const G2 g) {
    s.state = S_LL_MANT;
    int sym = (int)((((s.c->e1 - 15u) ^ s.f1) >> (s.f0 - 4)) & 0xf);
    set_next<ENC>(nx, ctype_slab(s, g, BL(s, 1, 0)) + CT_LL_MANTISSA * 16, SPK_MUD, sym);
}
template <bool ENC> __device__ __forceinline__ void enter_cp_count_small(St &s, Next &nx, const G2 g) {
    s.state = S_CP_COUNT_SMALL;
    uint32_t ll = s.c->last_llen - 1u; if (ll > 3) ll = 3;
    uint32_t index = ((s.c->last_4_states >> 4) & 3u) + 4u * ll;
    set_next<ENC>(nx, ctype_slab(s, g, BL(s, 1, 0)) + (CT_CP_COUNT_SMALL + index) * 16, SPK_MUD, (int)(s.c->e1 < 15 ? s.c->e1 : 15));
}
template <bool ENC> __device__ __forceinline__ void enter_cp_count_mant(St &s, Next &nx, const G2 g) {
    s.state = S_CP_COUNT_MANT;
    uint32_t index2 = s.f2 == 0 ? ((s.c->last_clen % 4) + 1) : 0u;
    int sym = (int)(((s.c->e1 ^ s.f0) >> (s.f1 - 4)) & 0xf);
    set_next<ENC>(nx, ctype_slab(s, g, BL(s, 1, 0)) + (CT_CP_COUNT_MANT + index2) * 16, SPK_SLOW, sym);
}
template <bool ENC> __device__ __forceinline__ void enter_cp_mnemonic(St &s, Next &nx, const G2 g) {
    s.state = S_CP_MNEMONIC;
    int sym = 15;
    if (ENC) {   // distance_mnemonic_code, codec/interface.rs:469-477
        for (uint32_t i = 0; i < 15; i++) { uint32_t d; bool ok; distance_from_mnemonic(s, i, d, ok); if (d == s.c->e0 && ok) { sym = (int)i; break; } }
    }
    s.f3 = get_distance_prior(s, s.f0);
    set_next<ENC>(nx, dprior_slab(s, g, s.f3) + (DP_MNEMONIC + (s.c->last_llen < 8 ? 1 : 0)) * 16, SPK_SLOW, sym);
}
template <bool ENC> __device__ __forceinline__ void enter_cp_dist_mant(St &s, Next &nx, const G2 g) {
    s.state = S_CP_DIST_MANT;
    uint32_t index2 = s.lit_h == 0 ? ((s.c->last_dlen & 3) + 1) : 0u;
    int inc = 0x4 << ((index2 & 6) << ((index2 & 2) >> 1));
    int sym = (int)(((s.c->e0 ^ s.f2) >> (s.f1 - 4)) & 0xf);
    set_next<ENC>(nx, dprior_slab(s, g, s.f3) + (DP_DIST_MANT + index2) * 16, sp_pack(inc, 0x4000), sym);
}
template <bool ENC> __device__ __forceinline__ void enter_dc_index(St &s, Next &nx, const G2 g) {
    s.state = S_DC_INDEX;
    uint32_t bits = s.tables[TB_SIZE_BITS + s.f0];
    uint32_t index = s.lit_h == 0 ? ((bits % 4) + 1) : 0u;
    uint32_t ap = get_distance_prior(s, s.f0);
    int sym = (int)(((s.c->e0 ^ s.f2) >> (s.f1 - 4)) & 0xf);
    set_next<ENC>(nx, dprior_slab(s, g, ap) + (DP_DICT_INDEX + index) * 16, SPK_MUD, sym);
}
template <bool ENC> __device__ __forceinline__ void enter_bt_mnemonic(St &s, Next &nx, int which) {
    s.state = S_BT_MNEMONIC; s.f0 = (uint32_t)which;
    int varint = 0;
    if (ENC) {
        uint32_t bt = s.c->e0 & 0xff;
        if (bt == BL(s, which, 1)) varint = 0;
        else if (bt == ((BMAX(s, which) + 1) & 0xff)) varint = 1;
        else if (bt <= 12) varint = (int)bt + 2;
        else varint = 15;
    }
    set_next<ENC>(nx, A_misc(s, MI_BTYPE + BT_MNEMONIC + which), SPK_SLOW, varint);
}
// returns true when the block switch is complete (the caller's common tail fetches the next command)
template <bool ENC, bool REC = false> __device__ __forceinline__ bool bt_done(St &s, Next &nx, const G2 g, uint32_t bt) {
    if (s.f0 == 0) {
        s.f1 = bt; s.state = S_BT_STRIDE;
        set_next<ENC>(nx, A_misc(s, MI_BTYPE + BT_STRIDE), SPK_SLOW, (int)(s.c->desired_force_stride == 9 ? (s.c->e1 & 0xf) : s.c->desired_force_stride));
        return false;
    }
    obs_btype(s, (int)s.f0, bt);
    rec_cmd<REC>(s, g, 4 + s.f0, bt, 0);
    return true;
}
template <bool ENC> __device__ __forceinline__ const uint8_t *pm_rec(const St &s) { return s.c->in.pms + (size_t)(s.c->e0 & s.c->in.pm_mask) * (32 + 16384 + 1024 + 8192); }
template <bool ENC> __device__ __forceinline__ void enter_pm_speed(St &s, Next &nx) {
    s.state = S_PM_SPEED;
    uint32_t si = s.f1 >> 2, pt = s.f1 & 3;
    int sym = 0;
    if (ENC) {
        int d = si == 0 ? s.c->desired_adapt0 : si == 1 ? s.c->desired_adapt1 : si == 2 ? s.c->desired_adapt2 : s.c->desired_adapt3;
        uint32_t c0 = speed_to_u8_i16((int)(short)(d & 0xffff)), c1 = speed_to_u8_i16(d >> 16);
        sym = (int)(pt == 0 ? ((c0 & 0x7f) >> 3) : pt == 1 ? (c0 & 7) : pt == 2 ? ((c1 & 0x7f) >> 3) : (c1 & 7));
    }
    set_next<ENC>(nx, A_misc(s, MI_PRED + PM_SPEED_PALETTE + (int)pt), SPK_FAST, sym);
}
template <bool ENC> __device__ __forceinline__ void enter_pm_map_mnemonic(St &s, Next &nx) {
    s.state = S_PM_MAP_MNEMONIC;
    int sym = 14;
    if (ENC) {
        const uint8_t *r = pm_rec<ENC>(s);
        uint32_t in_len = s.c->desired_do_context_map ? (s.f2 ? *reinterpret_cast<const uint16_t *>(r + 30) : *reinterpret_cast<const uint16_t *>(r + 28)) : 0u;
        if (s.f1 < in_len) {
            uint32_t target = s.f2 ? r[32 + 16384 + s.f1] : r[32 + s.f1];
            int hit = cmap_find_last(s, target);   // "last match wins" (context_map.rs:281-285)
            sym = hit >= 0 ? hit : 15;
            if (target == ((cmap_max(s) + 1) & 0xff)) sym = 13;
        }
    }
    // context_map.rs:273 + codec/priors.rs:130: Mnemonic has its own slots.  The build that produced the reference-held
    // stream wasm/wasm.html:98-107 coded both mnemonics with the slot DynamicContextMixingSpeed / PriorDepth /
    // ContextMapSpeedPalette[0] share (model_rev 1, include/divans_b200.h).
    set_next<ENC>(nx, A_misc(s, MI_PRED + (s.c->model_rev ? PM_SPEED_PALETTE : PM_MNEMONIC + (int)s.f2)), SPK_MED, sym);
}
// the MISC slot (after MI_PRED + PM_MIXING_VALUE) of mixing value f1: context_map.rs:395-399; model_rev 1: always slot 16.
// `mix(i)` reads mixing value i (the v2 fast loop addresses it in 32 bits)
template <class Mix> __device__ __forceinline__ uint32_t mixval_prior(const uint32_t f1, const bool model_rev, const Mix mix) {
    return (f1 >= 256 && !model_rev) ? (mix(f1 - 256) & 0xfu) : 16u;
}
template <bool ENC> __device__ __forceinline__ void enter_pm_mixval(St &s, Next &nx) {
    s.state = S_PM_MIXVAL;
    const uint8_t *const m = A_mix(s);
    const uint32_t prior = mixval_prior(s.f1, s.c->model_rev, [m](uint32_t i) { return (uint32_t)m[i]; });
    int sym = 0;
    if (ENC) {
        sym = !s.c->desired_do_context_map ? 4 : (!(s.f3 & 1) ? 0 : (int)pm_rec<ENC>(s)[32 + 16384 + 1024 + s.f1]);
        // a record byte above 15 is no nibble: the core would code the frequency of sym & 15 while this stream's own mask keeps
        // sym, so the stream would decode to other literals.  Refused (status 3; a cost pass: UINT64_MAX)
        if (sym > 15) { s.status = ST_FAIL; return; }
    }
    set_next<ENC>(nx, A_misc(s, MI_PRED + PM_MIXING_VALUE + (int)prior), SPK_PLANE, sym);
}
template <bool ENC> __device__ __forceinline__ void pm_map_store(St &s, Next &nx, const G2 g, uint32_t val) {
    uint32_t cap = s.f2 ? 1024u : 16384u;
    if (s.f1 >= cap) { s.status = ST_FAIL; return; }   // IndexBeyondContextMapSize
    cmap_touch(s, val);
    if (g.store0) {
        (s.f2 ? A_dcm(s) : A_lcm(s))[s.f1] = (uint8_t)val;
        if (!s.f2) { uint32_t *hdr = reinterpret_cast<uint32_t *>(s.slot + OFF_HDR); if (s.f1 >= hdr[2]) hdr[2] = s.f1 + 1; }   // high-water mark (reset_slot_v2)
    }
    s.f1++;
    enter_pm_map_mnemonic<ENC>(s, nx);
}

// The transition: consume the nibble just coded in state s.state, perform its side effects, choose the next prior.
template <bool ENC, bool V2 = false, bool REC = false>
__device__ __forceinline__ void transition(St &s, Next &nx, const G2 g, int nib) {
    // Two tails are shared by all states (one copy of their code keeps the kernel inside the instruction cache when the
    // streams of a batch are in different states): 1 = the command is complete, fetch the next one; 2 = a literal of tail_len bytes begins.
    int tail = 0; uint32_t tail_len = 0;
    // ---- hot: literal nibbles ----
    if (s.state == S_LIT_HI) { s.lit_h = (uint32_t)nib; enter_lit_nibble<ENC, false, V2>(s, nx); return; }
    if (s.state == S_LIT_LO) {
        uint32_t cur = ((uint32_t)nib | (s.lit_h << 4)) & 0xff;
        s.l8 = (s.l8 >> 8) | ((unsigned long long)cur << 56);   // push_literal_byte, codec/interface.rs:280-284
        if (g.store0) s.out[s.out_pos] = (uint8_t)cur;
        s.out_pos++;
        if (--s.lit_left != 0) { lit_context(s); enter_lit_nibble<ENC, true, V2>(s, nx); return; }
        swap_coders(s, g);
        tail = 1;
    } else if (s.state >= S_CP_MNEMONIC && s.state <= S_CP_DIST_MANT) {
        // ---- copy distance (codec/copy.rs:166-280): half of the command nibbles of a copy-dominated stream, tested before the switch
        uint32_t dist = 0; bool done = false;
        if (s.state == S_CP_DIST_MANT) {
            uint32_t next_rem = s.f1 - 4;
            s.f2 |= (uint32_t)nib << next_rem;
            s.lit_h += 4;
            if (next_rem == 0) { dist = s.f2; done = true; }
            else { s.f1 = next_rem; enter_cp_dist_mant<ENC>(s, nx, g); }
        } else if (s.state == S_CP_MNEMONIC) {
            if (nib != 15) {
                bool ok; distance_from_mnemonic(s, (uint32_t)nib, dist, ok);
                s.c->last_dlen = bitlen32(dist);
                if (!ok) { s.status = ST_FAIL; return; }   // CopyDistanceMnemonicCodeBad
                done = true;
            } else {
                s.state = S_CP_DIST_BEG;
                uint32_t dlen = bitlen32(s.c->e0);
                int sym = (int)min(14u, (dlen - 1u) & 0xffu);
                if (ENC && (s.c->lru1 - 3u) == s.c->e0 && !s.c->model_rev) sym = 15;   // copy.rs:199-201 (the model_rev 1 encoder did not take the shortcut)
                set_next<ENC>(nx, dprior_slab(s, g, s.f3) + (DP_DIST_BEG + (bitlen32(s.f0) >> 2)) * 16, SPK_SLOW, sym);
            }
        } else if (s.state == S_CP_DIST_BEG) {
            if (nib == 15) { dist = s.c->lru1 - 3u; s.c->last_dlen = bitlen32(dist); done = true; }
            else if (nib == 0) { s.c->last_dlen = 1; dist = 1; done = true; }
            else if (nib == 14) { s.state = S_CP_DIST_LAST; set_next<ENC>(nx, dprior_slab(s, g, s.f3) + DP_DIST_LAST * 16, SPK_ROCKET, (int)((bitlen32(s.c->e0) - 15u) & 0xf)); }
            else { s.c->last_dlen = (uint32_t)nib + 1; s.f1 = round_up_mod_4((uint32_t)nib); s.f2 = 1u << nib; s.lit_h = 0; enter_cp_dist_mant<ENC>(s, nx, g); }
        } else {   // S_CP_DIST_LAST
            s.c->last_dlen = (uint32_t)nib + 15; s.f1 = round_up_mod_4((uint32_t)nib + 14); s.f2 = (nib + 14) < 32 ? (1u << (nib + 14)) : 0u; s.lit_h = 0;
            enter_cp_dist_mant<ENC>(s, nx, g);
        }
        if (done) {
            obs_distance(s, dist);
            uint32_t len = s.f0;
            if (dist == 0 || dist >= s.c->ring_len) { s.status = ST_FAIL; return; }   // DistanceGreaterRingBuffer & friends
            if ((uint64_t)len > (uint64_t)(s.c->out_cap - s.out_pos)) { s.status = ST_NEED_OUTPUT; return; }
            rec_cmd<REC>(s, g, 1, dist, len);
            replay_copy(g, s.out, s.out_pos, dist, len);
            s.out_pos += len;
            tail = 1;
        }
    } else
    switch (s.state) {
    case S_CMD_TYPE: {
        if (nib == 0xf) { s.state = S_IDLE; return; }   // end of stream (trailer/CRC: frame kernel); the main loop parks the group
        if (nib == 1) { s.c->last_4_states = (s.c->last_4_states >> 2) | 64; if (ENC && s.c->e0 == 0) { s.status = ST_FAIL; return; } enter_cp_count_small<ENC>(s, nx, g); }
        else if (nib == 2) {
            s.c->last_4_states = (s.c->last_4_states >> 2) | 192; s.state = S_DC_SIZE_BEG;
            set_next<ENC>(nx, ctype_slab(s, g, BL(s, 1, 0)) + CT_DC_SIZE_BEG * 16, SPK_MUD, (int)min(15u, (s.c->e1 - 4u) & 0xffu));
        } else if (nib == 3) { s.c->last_4_states = (s.c->last_4_states >> 2) | 128; s.f3 = 0; if (!ENC) s.c->e1 = 0; enter_ll_count_small<ENC>(s, nx, g); }
        else if (nib == 4) enter_bt_mnemonic<ENC>(s, nx, 0);
        else if (nib == 5) enter_bt_mnemonic<ENC>(s, nx, 1);
        else if (nib == 6) enter_bt_mnemonic<ENC>(s, nx, 2);
        else if (nib == 7) {
            cmap_reset(s);                                                        // reset_context_map_lru
            for (uint32_t i = g.l16; i < 1024; i += g.nl) A_dcm(s)[i] = (uint8_t)(i & 3);   // reset_distance_context_map
            if (ENC) {   // encoder speed wishes, context_map.rs:123-146
                int d[4] = {SPK_MUD, SPK_MUD, SPK_MUD, SPK_MUD};
                const uint8_t *r = pm_rec<ENC>(s);
                if (r[2]) {
                    const uint16_t *sp = reinterpret_cast<const uint16_t *>(r + 4);
                    const uint16_t *cm = sp, *st = sp + (s.c->desired_context_mixing != 0 ? 8 : 4);
                    for (int k = 0; k < 2; k++) {
                        uint32_t a = speed_to_u8_u16(cm[k * 2]), b = speed_to_u8_u16(cm[k * 2 + 1]);
                        if (a != 0 || b != 0) d[2 + k] = sp_pack(u8_to_speed(a), u8_to_speed(b));
                        a = speed_to_u8_u16(st[k * 2]); b = speed_to_u8_u16(st[k * 2 + 1]);
                        if (a != 0 || b != 0) d[k] = sp_pack(u8_to_speed(a), u8_to_speed(b));
                    }
                }
                if (!s.c->have_desired_adapt) { s.c->desired_adapt0 = d[0]; s.c->desired_adapt1 = d[1]; s.c->desired_adapt2 = d[2]; s.c->desired_adapt3 = d[3]; }
            }
            s.state = S_PM_MODE;
            set_next<ENC>(nx, A_misc(s, MI_PRED + PM_ONLY), SPK_MED, ENC ? (int)pm_rec<ENC>(s)[0] : 0);
        } else s.status = ST_FAIL;   // CommandCodeOutOfBounds
    } break;
    // ---- literal length ----
    case S_LL_COUNT_SMALL: {
        if (nib == 14) {
            s.state = S_LL_SIZE_BEG;
            uint32_t lllen = bitlen32(s.c->e1 - 15u);
            set_next<ENC>(nx, ctype_slab(s, g, BL(s, 1, 0)) + CT_LL_SIZE_BEG * 16, SPK_MUD, (int)(lllen < 15 ? lllen : 15));
        } else if (nib == 15) { s.f3 = 1; enter_ll_count_small<ENC>(s, nx, g); }
        else { tail_len = (uint32_t)nib + 1; s.c->last_llen = tail_len; tail = 2; }
    } break;
    case S_LL_SIZE_BEG: {
        if (nib == 15) {
            s.state = S_LL_SIZE_LAST;
            set_next<ENC>(nx, ctype_slab(s, g, BL(s, 1, 0)) + CT_LL_SIZE_LAST * 16, SPK_MUD, (int)((bitlen32(s.c->e1 - 15u) - 15u) & 0xf));
        } else if (nib <= 1) { tail_len = 15u + (uint32_t)nib; tail = 2; }   // last_llen NOT updated (literal.rs:608-616)
        else { s.f0 = round_up_mod_4((uint32_t)nib - 1); s.f1 = 1u << (nib - 1); enter_ll_mant<ENC>(s, nx, g); }
    } break;
    case S_LL_SIZE_LAST: { s.f0 = round_up_mod_4((uint32_t)nib + 14); s.f1 = 1u << (nib + 14); enter_ll_mant<ENC>(s, nx, g); } break;
    case S_LL_MANT: {
        uint32_t next_rem = s.f0 - 4;
        s.f1 |= (uint32_t)nib << next_rem;
        if (next_rem == 0) { tail_len = s.f1 + 15u; s.c->last_llen = tail_len; tail = 2; }
        else { s.f0 = next_rem; enter_ll_mant<ENC>(s, nx, g); }
    } break;
    // ---- copy ----
    case S_CP_COUNT_SMALL: {
        if (nib != 15) { s.f0 = (uint32_t)nib; s.c->last_clen = bitlen32(s.f0); enter_cp_mnemonic<ENC>(s, nx, g); }
        else { s.state = S_CP_COUNT_BEG; set_next<ENC>(nx, ctype_slab(s, g, BL(s, 1, 0)) + CT_CP_COUNT_BEG * 16, SPK_FAST, (int)min(15u, (bitlen32(s.c->e1) - 4u) & 0xffu)); }
    } break;
    case S_CP_COUNT_BEG: {
        if (nib == 15) { s.state = S_CP_COUNT_LAST; set_next<ENC>(nx, ctype_slab(s, g, BL(s, 1, 0)) + CT_CP_COUNT_LAST * 16, SPK_FAST, (int)((bitlen32(s.c->e1) - 19u) & 0xf)); }
        else { s.c->last_clen = (uint32_t)nib + 4; s.f1 = round_up_mod_4((uint32_t)nib + 3); s.f0 = 1u << (nib + 3); s.f2 = 0; enter_cp_count_mant<ENC>(s, nx, g); }
    } break;
    case S_CP_COUNT_LAST: {
        s.c->last_clen = (uint32_t)nib + 19; s.f1 = round_up_mod_4((uint32_t)nib + 18); s.f0 = (nib + 18) < 32 ? (1u << (nib + 18)) : 0u; s.f2 = 0;
        enter_cp_count_mant<ENC>(s, nx, g);
    } break;
    case S_CP_COUNT_MANT: {
        uint32_t next_rem = s.f1 - 4;
        s.f0 |= (uint32_t)nib << next_rem;
        if (next_rem == 0) enter_cp_mnemonic<ENC>(s, nx, g);
        else { s.f1 = next_rem; s.f2 += 4; enter_cp_count_mant<ENC>(s, nx, g); }
    } break;
    // ---- dict ----
    case S_DC_SIZE_BEG: case S_DC_SIZE_LAST: {
        uint32_t ws;
        if (s.state == S_DC_SIZE_BEG) {
            if (nib == 15) { s.state = S_DC_SIZE_LAST; set_next<ENC>(nx, ctype_slab(s, g, BL(s, 1, 0)) + CT_DC_SIZE_LAST * 16, SPK_MUD, (int)((s.c->e1 - 19u) & 0xf)); return; }
            ws = (uint32_t)nib + 4;
        } else { ws = (uint32_t)nib + 19; if (ws > 24) { s.status = ST_FAIL; return; } }   // DictWordSizeTooLarge
        s.f0 = ws; s.f1 = round_up_mod_4(s.tables[TB_SIZE_BITS + ws]); s.f2 = 0; s.lit_h = 0;
        enter_dc_index<ENC>(s, nx, g);
    } break;
    case S_DC_INDEX: {
        uint32_t next_rem = s.f1 - 4;
        s.f2 |= (uint32_t)nib << next_rem;
        if (next_rem == 0) { s.state = S_DC_TR_HI; set_next<ENC>(nx, A_misc(s, MI_TRANSFORM + 0 + 2 * (int)(s.f0 >> 1)), SPK_FAST, (int)((s.c->e2 >> 4) & 0xf)); }
        else { s.f1 = next_rem; s.lit_h += 4; enter_dc_index<ENC>(s, nx, g); }
    } break;
    case S_DC_TR_HI: { s.f3 = (uint32_t)nib; s.state = S_DC_TR_LO; set_next<ENC>(nx, A_misc(s, MI_TRANSFORM + 1 + 2 * nib), SPK_FAST, (int)(s.c->e2 & 0xf)); } break;
    case S_DC_TR_LO: {
        uint32_t tr = (s.f3 << 4) | (uint32_t)nib;
        if (tr >= 121) { s.status = ST_FAIL; return; }   // DictTransformIndexUndefined
        int n = dict_word(g, s.tables, s.f0, s.f2, tr);   // every lane computes the same bytes (benign duplicate writes)
        if (n < 0) { s.status = ST_FAIL; return; }
        __syncwarp(g.gmask);
        if ((uint64_t)n > (uint64_t)(s.c->out_cap - s.out_pos)) { s.status = ST_NEED_OUTPUT; return; }
        rec_cmd<REC>(s, g, 2, s.f2, s.f0, tr, (uint32_t)n);
        for (int i = g.l16; i < n; i += g.nl) s.out[s.out_pos + i] = s.c->scratch[i];
        __syncwarp(g.gmask);
        s.out_pos += (uint32_t)n;
        tail = 1;
    } break;
    // ---- block switches ----
    case S_BT_MNEMONIC: {
        int which = (int)s.f0;
        if (nib == 0) tail = bt_done<ENC, REC>(s, nx, g, BL(s, which, 1)) ? 1 : 0;
        else if (nib == 1) tail = bt_done<ENC, REC>(s, nx, g, (BMAX(s, which) + 1) & 0xff) ? 1 : 0;
        else if (nib != 15) tail = bt_done<ENC, REC>(s, nx, g, (uint32_t)nib - 2) ? 1 : 0;
        else { s.state = S_BT_FIRST; set_next<ENC>(nx, A_misc(s, MI_BTYPE + BT_FIRST + which), SPK_SLOW, (int)(s.c->e0 & 0xf)); }
    } break;
    case S_BT_FIRST: { s.f1 = (uint32_t)nib; s.state = S_BT_SECOND; set_next<ENC>(nx, A_misc(s, MI_BTYPE + BT_SECOND + (int)s.f0), SPK_SLOW, (int)((s.c->e0 >> 4) & 0xf)); } break;
    case S_BT_SECOND: tail = bt_done<ENC, REC>(s, nx, g, ((uint32_t)nib << 4) | s.f1) ? 1 : 0; break;
    case S_BT_STRIDE: { obs_btype(s, 0, s.f1); s.btype_last = s.f1; s.c->t2_dirty = true; rec_cmd<REC>(s, g, 4, s.f1, (uint32_t)nib); tail = 1; } break;
    // ---- prediction mode ----
    case S_PM_MODE: {
        s.f0 = (uint32_t)nib; s.state = S_PM_MIX;
        if (ENC && pm_rec<ENC>(s)[1] > 1) { s.status = ST_FAIL; return; }   // is_adv: bit 3 of the nibble below, so 0 or 1
        set_next<ENC>(nx, A_misc(s, MI_PRED + PM_SPEED_PALETTE), SPK_MED, ENC ? (int)(s.c->desired_context_mixing | ((uint32_t)pm_rec<ENC>(s)[1] << 3)) : 0);   // aliases SpeedPalette[0]
    } break;
    case S_PM_MIX: {
        s.f3 = ((uint32_t)nib & 3) << 1 | (nib != 0 ? 1u : 0u);   // mixing math, combine_literal_predictions
        s.state = S_PM_DEPTH;
        set_next<ENC>(nx, A_misc(s, MI_PRED + PM_SPEED_PALETTE), SPK_FAST, (int)s.c->desired_prior_depth);   // aliases SpeedPalette[0]
    } break;
    case S_PM_DEPTH: { s.f1 = 0; s.l8 = 0; enter_pm_speed<ENC>(s, nx); } break;   // l8 doubles as the f8 accumulator (re-seeded at every literal)
    case S_PM_SPEED: {
        uint32_t si = s.f1 >> 2, pt = s.f1 & 3;
        uint32_t byte_idx = si * 2 + (pt >> 1);
        unsigned long long add = (pt & 1) ? (unsigned long long)nib : (((unsigned long long)nib << 3) & 0xff);
        s.l8 |= add << (8 * byte_idx);
        if (++s.f1 == 16) { s.f1 = 0; s.f2 = 0; enter_pm_map_mnemonic<ENC>(s, nx); }
        else enter_pm_speed<ENC>(s, nx);
    } break;
    case S_PM_MAP_MNEMONIC: {
        if (nib == 14) {
            if (s.f2 == 0) { if (REC) s.c->rec.lit_map_len = s.f1; cmap_reset(s); s.f2 = 1; s.f1 = 0; enter_pm_map_mnemonic<ENC>(s, nx); }
            else { if (REC) s.c->rec.dist_map_len = s.f1; s.f1 = 0; enter_pm_mixval<ENC>(s, nx); }
        } else if (nib == 15) {
            s.state = S_PM_MAP_FIRST;
            int sym = 0;
            if (ENC) { const uint8_t *r = pm_rec<ENC>(s); sym = (s.f2 ? r[32 + 16384 + s.f1] : r[32 + s.f1]) >> 4; }
            set_next<ENC>(nx, A_misc(s, MI_PRED + PM_FIRST_NIBBLE + (int)s.f2), SPK_MED, sym);
        } else pm_map_store<ENC>(s, nx, g, nib == 13 ? ((cmap_max(s) + 1) & 0xff) : cmap_get(s, nib));
    } break;
    case S_PM_MAP_FIRST: {
        s.lit_h = (uint32_t)nib; s.state = S_PM_MAP_SECOND;
        int sym = 0;
        if (ENC) { const uint8_t *r = pm_rec<ENC>(s); sym = (s.f2 ? r[32 + 16384 + s.f1] : r[32 + s.f1]) & 0xf; }
        set_next<ENC>(nx, A_misc(s, MI_PRED + PM_SECOND_NIBBLE + (int)s.f2), SPK_MED, sym);
    } break;
    case S_PM_MAP_SECOND: pm_map_store<ENC>(s, nx, g, (s.lit_h << 4) | (uint32_t)nib); break;
    case S_PM_MIXVAL: {
        if (g.store0) { A_mix(s)[s.f1] = (uint8_t)nib; if (s.f1 == 0) reinterpret_cast<uint32_t *>(s.slot + OFF_HDR)[3] = 1u; }
        if (++s.f1 == 8192) {   // obs_prediction_mode_context_map, codec/interface.rs:293-321
            uint32_t mixing_math = (s.f3 >> 1) & 3;
            s.c->mixing_param = mixing_math; s.mixing_trait = mixing_math > 1;
            if (s.f0 > 3) { s.status = ST_FAIL; return; }   // PredictionModeOutOfBounds
            s.pred_mode = s.f0;
            unsigned long long a = s.l8;
            s.ad_stride = f8_pair_to_speed((uint32_t)a & 0xff, (uint32_t)(a >> 8) & 0xff);
            s.c->ad_cm_lo = f8_pair_to_speed((uint32_t)(a >> 32) & 0xff, (uint32_t)(a >> 40) & 0xff);
            s.c->ad_cm_hi = f8_pair_to_speed((uint32_t)(a >> 48) & 0xff, (uint32_t)(a >> 56) & 0xff);
            s.speeds_small = speed_is_small(s.ad_stride) && speed_is_small(s.c->ad_cm_lo) && speed_is_small(s.c->ad_cm_hi);
            if (V2 && !s.speeds_small && s.tagged) { v2_make_untagged(g, s.slot, s.gen); s.tagged = false; }
            if (!V2 && !s.speeds_small && g.store0) reinterpret_cast<uint32_t *>(s.slot + OFF_HDR)[1] = 1u;   // elements may use their sign bits: the v2 engine must wipe before trusting tags
            s.c->lit_slabs_ready = false; s.c->t2_dirty = true; s.c->pm_seen = true;
            rec_pm<REC>(s, g);
            tail = 1;
        } else enter_pm_mixval<ENC>(s, nx);
    } break;
    default: s.status = ST_FAIL; break;
    }
    if (tail == 1) { if (ENC) s.c->in.pos++; enter_cmd_type<ENC>(s, nx); }
    else if (tail == 2) start_literal<ENC, V2, REC>(s, nx, g, tail_len);
}

// fresh book-keeping for a new stream (CrossCommandBookKeeping::new codec/interface.rs:348-402, LiteralBookKeeping::new :246-264)
__device__ __forceinline__ void st_reset(St &s) {
    s.c->lru0 = 4; s.c->lru1 = 11; s.c->lru2 = 15; s.c->lru3 = 16;
    s.c->btype_lru = 0x010001000100ull;                        // btype_lru: [[0,1];3]
    s.c->btype_max = 0;
    s.c->last_dlen = 1; s.c->last_clen = 1; s.c->last_llen = 1; s.c->last_4_states = 3 << 4;
    s.c->cmap_lo = 0; s.c->cmap_hi = 0;
    s.l8 = 0; s.btype_last = 0;
    s.pred_mode = 0;   // LiteralPredictionModeNibble::default() is in the brotli crate (NOT-IN-TREE): LSB6 assumed -- unpinned,
                       // unobservable when a PredictionMode command precedes the first literal
    s.ad_stride = s.c->ad_cm_lo = s.c->ad_cm_hi = SPK_MUD;
    s.c->w_lo.w0 = s.c->w_lo.w1 = 1; s.c->w_lo.norm = 1 << 14; s.c->w_hi = s.c->w_lo;
    s.speeds_small = true;   // MUD
    s.tagged = true;
    s.c->mixing_param = 1; s.mixing_trait = false; s.c->lit_slabs_ready = false; s.lit_cfg = -1;
    s.status = ST_OK; s.c->cur_is_lit = false; s.c->t2_dirty = true; s.c->pm_seen = false;
    s.f0 = s.f1 = s.f2 = s.f3 = 0; s.lit_left = s.lit_ctx = s.lit_h = 0;
    s.c->e0 = s.c->e1 = s.c->e2 = s.c->e3 = 0;
}

}  // namespace dv
