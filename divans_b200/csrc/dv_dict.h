// dv_dict.h -- the dictionary step of the LZ77 command generator (include/divans_b200.h, "dictionary words in the LZ77 parse"):
// the index of the RFC 7932 dictionary both generators search, and dict(i) itself.  The index is built once on the host from
// brotli_tables.bin (tools/gen_brotli_tables.py) and is one flat block without pointers, so the GPU generator uses the uploaded
// copy as it is.  dict_match is compiled for the host (dv_ir.cpp, lz77_blob) and for sm_90a (dv_lz77.cu, lz77_dict_kernel).
//
// Layout: the words of size 4..24 (id below 2^size_bits_by_length[size]) are hashed by their first four bytes, read as a
// little-endian u32 `key`, h = (key * 2654435761) >> (32 - DICT_HASH_BITS).  Bucket h is entry[bucket[h] .. bucket[h + 1]),
// each entry {key, size << 16 | id}, in order of size, then id.  The transform set is set_t[0 .. n_set) in ascending id, with
// each member's suffix.
#pragma once
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define DV_DICT_FN __host__ __device__ __forceinline__
#else
#define DV_DICT_FN inline
#endif

namespace dv {

constexpr int DICT_HASH_BITS = 14;
constexpr uint32_t DICT_BUCKETS = 1u << DICT_HASH_BITS;
constexpr uint32_t DICT_WORDS = 13504;     // sum over sizes 4..24 of 2^size_bits_by_length[size] (checked by the builder)
constexpr uint32_t DICT_SET_MAX = 64;      // room for the transform set (44 members)
constexpr uint32_t DICT_SFX_MAX = 8;       // room for a member's suffix (at most 7 bytes)
constexpr uint32_t DICT_MAX_MATCH = 31;    // the longest transformed word: 24 + 7
// offsets in brotli_tables.bin (tools/gen_brotli_tables.py)
constexpr uint32_t DICT_TB_SIZE_BITS = 24, DICT_TB_OFFSETS = 56, DICT_TB_TRANSFORMS = 2232, DICT_TB_PSMAP = 2616, DICT_TB_PS = 2744,
                   DICT_TB_DICT = 3000;

struct DictIndex {
    uint32_t bucket[DICT_BUCKETS + 1];
    uint32_t entry[DICT_WORDS][2];
    uint32_t word_off[32];                 // offsets_by_length: word (size, id) is dictionary[word_off[size] + id * size ..)
    uint32_t n_set;
    uint8_t set_t[DICT_SET_MAX], set_len[DICT_SET_MAX], set_sfx[DICT_SET_MAX][DICT_SFX_MAX];
};

// dict(i) packed so that a larger value is a better match under the rule's order: |w| << 23 | (127 - transform) << 16 |
// (31 - size) << 11 | (2047 - id); 0 where no word matches.  `p` is the stream at i, `avail` = n - i bytes, `dict` the
// dictionary bytes.
DV_DICT_FN constexpr uint32_t dict_len(uint32_t k) { return k >> 23; }
DV_DICT_FN constexpr uint32_t dict_transform(uint32_t k) { return 127u - ((k >> 16) & 127u); }
DV_DICT_FN constexpr uint32_t dict_size(uint32_t k) { return 31u - ((k >> 11) & 31u); }
DV_DICT_FN constexpr uint32_t dict_id(uint32_t k) { return 2047u - (k & 2047u); }

DV_DICT_FN uint32_t dict_match(const DictIndex &x, const uint8_t *dict, const uint8_t *p, uint32_t avail) {
    if (avail < 4) return 0;
    const uint32_t key = (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24;
    const uint32_t h = (key * 2654435761u) >> (32 - DICT_HASH_BITS);
    uint32_t best = 0;
    for (uint32_t e = x.bucket[h], e_end = x.bucket[h + 1]; e < e_end; e++) {
        if (x.entry[e][0] != key) continue;
        const uint32_t s = x.entry[e][1] >> 16, id = x.entry[e][1] & 0xffffu;
        if (s > avail) continue;
        const uint8_t *w = dict + x.word_off[s] + id * s;
        uint32_t k = 4;
        while (k < s && w[k] == p[k]) k++;
        if (k < s) continue;
        for (uint32_t j = 0; j < x.n_set; j++) {
            const uint32_t sl = x.set_len[j], L = s + sl;
            const uint32_t packed = L << 23 | (127u - x.set_t[j]) << 16 | (31u - s) << 11 | (2047u - id);
            if (L > avail || packed <= best) continue;
            uint32_t m = 0;
            while (m < sl && x.set_sfx[j][m] == p[s + m]) m++;
            if (m == sl) best = packed;
        }
    }
    return best;
}

// The index of brotli_tables.bin, built on first use and kept for the process (dv_ir.cpp); NULL if the tables do not have the
// shape the index assumes.
const DictIndex *host_dict_index();

// Fill `x` from the tables blob.  Returns false if the tables do not have the shape the index assumes.
inline bool dict_index_build(const uint8_t *tables, DictIndex &x) {
    const uint8_t *size_bits = tables + DICT_TB_SIZE_BITS, *tr = tables + DICT_TB_TRANSFORMS, *ps = tables + DICT_TB_PS;
    const uint8_t *dict = tables + DICT_TB_DICT;
    const uint8_t *psmap_b = tables + DICT_TB_PSMAP;
    auto psmap = [&](uint32_t i) { return (uint32_t)psmap_b[2 * i] | (uint32_t)psmap_b[2 * i + 1] << 8; };
    for (int s = 0; s < 32; s++) {
        const uint8_t *o = tables + DICT_TB_OFFSETS + 4 * s;
        x.word_off[s] = (uint32_t)o[0] | (uint32_t)o[1] << 8 | (uint32_t)o[2] << 16 | (uint32_t)o[3] << 24;
    }
    x.n_set = 0;
    for (uint32_t t = 0; t < 121; t++) {
        const uint8_t *prefix = ps + psmap(tr[3 * t]), *suffix = ps + psmap(tr[3 * t + 2]);
        if (prefix[0] != 0 || tr[3 * t + 1] != 0) continue;
        if (x.n_set == DICT_SET_MAX || suffix[0] >= DICT_SFX_MAX) return false;
        x.set_t[x.n_set] = (uint8_t)t;
        x.set_len[x.n_set] = suffix[0];
        for (uint32_t m = 0; m < DICT_SFX_MAX; m++) x.set_sfx[x.n_set][m] = m < suffix[0] ? suffix[1 + m] : 0;
        x.n_set++;
    }
    // counting sort of the words into buckets, in order of size then id
    for (uint32_t h = 0; h <= DICT_BUCKETS; h++) x.bucket[h] = 0;
    uint32_t n = 0;
    auto key_of = [&](uint32_t s, uint32_t id) {
        const uint8_t *w = dict + x.word_off[s] + id * s;
        return (uint32_t)w[0] | (uint32_t)w[1] << 8 | (uint32_t)w[2] << 16 | (uint32_t)w[3] << 24;
    };
    for (uint32_t s = 4; s <= 24; s++) {
        if (size_bits[s] == 0 || size_bits[s] > 11) return false;
        for (uint32_t id = 0; id < (1u << size_bits[s]); id++, n++) x.bucket[((key_of(s, id) * 2654435761u) >> (32 - DICT_HASH_BITS)) + 1]++;
    }
    if (n != DICT_WORDS) return false;
    for (uint32_t h = 0; h < DICT_BUCKETS; h++) x.bucket[h + 1] += x.bucket[h];
    uint32_t fill[DICT_BUCKETS];
    for (uint32_t h = 0; h < DICT_BUCKETS; h++) fill[h] = x.bucket[h];
    for (uint32_t s = 4; s <= 24; s++)
        for (uint32_t id = 0; id < (1u << size_bits[s]); id++) {
            const uint32_t key = key_of(s, id), e = fill[(key * 2654435761u) >> (32 - DICT_HASH_BITS)]++;
            x.entry[e][0] = key;
            x.entry[e][1] = s << 16 | id;
        }
    return true;
}

// ---- every transform (include/divans_b200.h, "dictionary words under every transform in the LZ77 parse") ----
// A candidate (word, transform) is found at the start of its core, the word after the transform's omission and case change.
// The index holds one entry per (word, variant) that some transform uses and whose core has at least 4 bytes; variant 0 is
// the word itself (identity and omit-last-k, whose cores are its prefixes), 1 its uppercase-first form, 2 its uppercase-all
// form, 2 + k the word without its first k bytes.  Entries are hashed by the first four bytes of the core (little-endian u32
// `key`, h = (key * 2654435761) >> (32 - WORDS_HASH_BITS)); bucket h is entry[bucket[h] .. bucket[h + 1]), each entry {key,
// variant << 24 | size << 16 | id}.  The cores are read from bytes[]: the dictionary, then its words uppercased first and
// uppercased all by the decoder's rule.  The transforms are grouped by prefix (9 distinct ones, in order of first use) and by
// the variant they read: the rules of prefix j and variant v are rule[rule_start[j * WORDS_VARIANTS + v] .. next), in
// ascending transform id.
constexpr int WORDS_HASH_BITS = 16;
constexpr uint32_t WORDS_BUCKETS = 1u << WORDS_HASH_BITS;
constexpr uint32_t WORDS_ENTRIES = 99392;   // (word, variant) pairs with a core of 4 or more bytes (checked by the builder)
constexpr uint32_t WORDS_DICT_BYTES = 122784;
constexpr uint32_t WORDS_PREFIXES = 9, WORDS_PREFIX_MAX = 8, WORDS_VARIANTS = 12, WORDS_SFX_MAX = 8;
constexpr uint32_t WORDS_MAX_MATCH = 37;    // 24 + the longest prefix and suffix together (13; checked by the builder)

struct WordIndex {
    uint32_t bucket[WORDS_BUCKETS + 1];
    uint32_t entry[WORDS_ENTRIES][2];
    uint32_t word_off[32];
    uint32_t rule_start[WORDS_PREFIXES * WORDS_VARIANTS + 1];
    uint8_t pre_len[WORDS_PREFIXES], pre[WORDS_PREFIXES][WORDS_PREFIX_MAX];
    uint8_t rule_t[121], rule_type[121], rule_slen[121], rule_sfx[121][WORDS_SFX_MAX];
    uint8_t bytes[3][WORDS_DICT_BYTES];
};

// dict(i) under every transform, packed as dict_match packs it; `p` is the stream at i, `avail` = n - i bytes.  For each prefix
// that matches at p, one bucket is probed at the core's start; an entry's core is compared as far as it matches (k bytes),
// and each rule of its variant whose core fits in those k bytes has its suffix compared.  Entries that share the key are all
// walked: on English text that is about 20 per position (428 cores begin "tion", 362 " the"), which is what makes this
// lookup several times dict_match's (DESIGN.md section 4, "Dictionary words under every transform").
DV_DICT_FN uint32_t words_match(const WordIndex &x, const uint8_t *p, uint32_t avail) {
    uint32_t best = 0;
    for (uint32_t j = 0; j < WORDS_PREFIXES; j++) {
        const uint32_t pl = x.pre_len[j];
        if (pl + 4 > avail) continue;
        uint32_t m = 0;
        while (m < pl && x.pre[j][m] == p[m]) m++;
        if (m < pl) continue;
        const uint8_t *const q = p + pl;
        const uint32_t qa = avail - pl;
        const uint32_t key = (uint32_t)q[0] | (uint32_t)q[1] << 8 | (uint32_t)q[2] << 16 | (uint32_t)q[3] << 24;
        const uint32_t h = (key * 2654435761u) >> (32 - WORDS_HASH_BITS);
        for (uint32_t e = x.bucket[h], e_end = x.bucket[h + 1]; e < e_end; e++) {
            if (x.entry[e][0] != key) continue;
            const uint32_t info = x.entry[e][1], v = info >> 24, s = (info >> 16) & 31u, id = info & 0xffffu;
            const uint32_t skip = v >= 3 ? v - 2 : 0, cl = s - skip;
            const uint8_t *const core = x.bytes[v == 1 ? 1 : v == 2 ? 2 : 0] + x.word_off[s] + id * s + skip;
            const uint32_t lim = cl < qa ? cl : qa;
            uint32_t k = 4;
            while (k < lim && core[k] == q[k]) k++;
            for (uint32_t r = x.rule_start[j * WORDS_VARIANTS + v], r_end = x.rule_start[j * WORDS_VARIANTS + v + 1]; r < r_end; r++) {
                const uint32_t type = x.rule_type[r];
                const uint32_t need = type >= 1 && type <= 9 ? cl - type : cl;   // (variant 0 only: omit-last-k)
                if ((int32_t)need < 4 || k < need) continue;
                const uint32_t sl = x.rule_slen[r], L = pl + need + sl;
                const uint32_t packed = L << 23 | (127u - x.rule_t[r]) << 16 | (31u - s) << 11 | (2047u - id);
                if (L > avail || packed <= best) continue;
                uint32_t b = 0;
                while (b < sl && x.rule_sfx[r][b] == q[need + b]) b++;
                if (b == sl) best = packed;
            }
        }
    }
    return best;
}

// The index of every transform, built on first use and kept for the process (dv_ir.cpp); NULL if the tables do not have the
// shape the index assumes.
const WordIndex *host_words_index();

// The decoder's uppercase rule on a core of `len` bytes: uppercase the first character (all = false) or every character.  A
// step whose change falls past the core changes nothing the decoder keeps: the suffix, or nothing, is written there.
inline void words_uppercase(uint8_t *w, uint32_t len, bool all) {
    for (uint32_t at = 0; at < len;) {
        uint32_t step;
        if (w[at] < 0xc0) { if (w[at] >= 'a' && w[at] <= 'z') w[at] ^= 32; step = 1; }
        else if (w[at] < 0xe0) { if (at + 1 < len) w[at + 1] ^= 32; step = 2; }
        else { if (at + 2 < len) w[at + 2] ^= 5; step = 3; }
        at += step;
        if (!all) break;
    }
}

// Fill `x` from the tables blob.  Returns false if the tables do not have the shape the index assumes.
inline bool words_index_build(const uint8_t *tables, WordIndex &x) {
    const uint8_t *size_bits = tables + DICT_TB_SIZE_BITS, *tr = tables + DICT_TB_TRANSFORMS, *ps = tables + DICT_TB_PS;
    const uint8_t *psmap_b = tables + DICT_TB_PSMAP;
    auto psmap = [&](uint32_t i) { return (uint32_t)psmap_b[2 * i] | (uint32_t)psmap_b[2 * i + 1] << 8; };
    for (int s = 0; s < 32; s++) {
        const uint8_t *o = tables + DICT_TB_OFFSETS + 4 * s;
        x.word_off[s] = (uint32_t)o[0] | (uint32_t)o[1] << 8 | (uint32_t)o[2] << 16 | (uint32_t)o[3] << 24;
    }
    for (uint32_t s = 4; s <= 24; s++)
        if (size_bits[s] == 0 || size_bits[s] > 11 || x.word_off[s] + (s << size_bits[s]) > WORDS_DICT_BYTES) return false;
    // prefixes in order of first use, and each transform's (prefix, variant)
    uint32_t n_pre = 0, t_pre[121], t_var[121];
    bool var_used[WORDS_VARIANTS] = {};
    for (uint32_t t = 0; t < 121; t++) {
        const uint8_t *prefix = ps + psmap(tr[3 * t]), *suffix = ps + psmap(tr[3 * t + 2]);
        const uint32_t type = tr[3 * t + 1];
        if (prefix[0] > WORDS_PREFIX_MAX || suffix[0] > WORDS_SFX_MAX || 24u + prefix[0] + suffix[0] > WORDS_MAX_MATCH || type > 20)
            return false;
        uint32_t j = 0;
        while (j < n_pre && !(x.pre_len[j] == prefix[0] && memcmp(x.pre[j], prefix + 1, prefix[0]) == 0)) j++;
        if (j == n_pre) {
            if (n_pre == WORDS_PREFIXES) return false;
            x.pre_len[j] = prefix[0];
            for (uint32_t m = 0; m < WORDS_PREFIX_MAX; m++) x.pre[j][m] = m < prefix[0] ? prefix[1 + m] : 0;
            n_pre++;
        }
        t_pre[t] = j;
        t_var[t] = type <= 9 ? 0 : type - 9;
        var_used[t_var[t]] = true;
    }
    if (n_pre != WORDS_PREFIXES) return false;
    uint32_t r = 0;
    for (uint32_t g = 0; g < WORDS_PREFIXES * WORDS_VARIANTS; g++) {
        x.rule_start[g] = r;
        for (uint32_t t = 0; t < 121; t++) {
            if (t_pre[t] * WORDS_VARIANTS + t_var[t] != g) continue;
            const uint8_t *suffix = ps + psmap(tr[3 * t + 2]);
            x.rule_t[r] = (uint8_t)t;
            x.rule_type[r] = tr[3 * t + 1];
            x.rule_slen[r] = suffix[0];
            for (uint32_t m = 0; m < WORDS_SFX_MAX; m++) x.rule_sfx[r][m] = m < suffix[0] ? suffix[1 + m] : 0;
            r++;
        }
    }
    x.rule_start[WORDS_PREFIXES * WORDS_VARIANTS] = r;
    // the cores' bytes
    memcpy(x.bytes[0], tables + DICT_TB_DICT, WORDS_DICT_BYTES);
    memcpy(x.bytes[1], tables + DICT_TB_DICT, WORDS_DICT_BYTES);
    memcpy(x.bytes[2], tables + DICT_TB_DICT, WORDS_DICT_BYTES);
    for (uint32_t s = 4; s <= 24; s++)
        for (uint32_t id = 0; id < (1u << size_bits[s]); id++) {
            words_uppercase(x.bytes[1] + x.word_off[s] + id * s, s, false);
            words_uppercase(x.bytes[2] + x.word_off[s] + id * s, s, true);
        }
    // the entries: counting sort by bucket (bucket[h] counts, then ends, then, filled from the end down, starts)
    auto for_each_entry = [&](auto f) {
        for (uint32_t s = 4; s <= 24; s++)
            for (uint32_t id = 0; id < (1u << size_bits[s]); id++)
                for (uint32_t v = 0; v < WORDS_VARIANTS; v++) {
                    const uint32_t skip = v >= 3 ? v - 2 : 0;
                    if (!var_used[v] || s < skip + 4) continue;
                    const uint8_t *c = x.bytes[v == 1 ? 1 : v == 2 ? 2 : 0] + x.word_off[s] + id * s + skip;
                    const uint32_t key = (uint32_t)c[0] | (uint32_t)c[1] << 8 | (uint32_t)c[2] << 16 | (uint32_t)c[3] << 24;
                    f(key, v << 24 | s << 16 | id);
                }
    };
    for (uint32_t h = 0; h <= WORDS_BUCKETS; h++) x.bucket[h] = 0;
    uint32_t n = 0;
    for_each_entry([&](uint32_t key, uint32_t) { x.bucket[(key * 2654435761u) >> (32 - WORDS_HASH_BITS)]++; n++; });
    if (n != WORDS_ENTRIES) return false;
    for (uint32_t h = 1; h <= WORDS_BUCKETS; h++) x.bucket[h] += x.bucket[h - 1];
    for_each_entry([&](uint32_t key, uint32_t info) {
        const uint32_t e = --x.bucket[(key * 2654435761u) >> (32 - WORDS_HASH_BITS)];
        x.entry[e][0] = key;
        x.entry[e][1] = info;
    });
    return true;
}

}  // namespace dv
