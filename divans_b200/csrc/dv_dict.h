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

}  // namespace dv
