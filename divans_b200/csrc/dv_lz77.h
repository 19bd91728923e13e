// dv_lz77.h -- host-visible launch wrapper of the LZ77 command generator (dv_lz77.cu): divans_b200_lz77_cmds_batch_device.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dv_dict.h"

namespace dv {

constexpr uint32_t LZ_HEAD_ENTRIES = 1u << 15;   // the hash table of the host generator (dv_ir.cpp, lz77_blob): 15-bit hashes

// Scratch of one warp, in int32 words: the head table, then prev[max_in_len], rounded up to 256 bytes.
static inline uint64_t lz77_scratch_words(uint64_t max_in_len) { return (LZ_HEAD_ENTRIES + max_in_len + 63) & ~63ull; }

// Stream i is in[in_off[i] .. +in_len[i]); its DVCL blob goes to blobs[blob_off[i] .. +blob_cap[i]).  `pm` is the one
// PredictionMode record (PM_RECORD_BYTES, 16-byte aligned) every blob carries.  Warp w of n_warps owns scratch[w * stride ..).
struct Lz77Params {
    const uint8_t *in; const uint64_t *in_off, *in_len; uint64_t max_in_len;
    uint8_t *blobs; const uint64_t *blob_off, *blob_cap; uint64_t *blob_len; int32_t *status;
    const uint8_t *pm; uint32_t n_streams; int32_t window;
    int32_t min_match, lazy;   // the parse (include/divans_b200.h): min_match 4..32, lazy 0..2
    uint32_t *work_counter; int32_t *scratch; uint64_t stride; uint32_t n_warps;
};
// The dictionary step (include/divans_b200.h, "dictionary words in the LZ77 parse"): dict_min 0 (off) or 4..32, the index and
// the dictionary bytes.  A parameter of its own: the kernels without the step keep Lz77Params, and with it their code.
struct Lz77Dict {
    const DictIndex *index; const uint8_t *words; int32_t dict_min;
};
// The dictionary step under every transform (include/divans_b200.h, "dictionary words under every transform in the LZ77
// parse"): dict_min 4..32 and the index, which holds the dictionary bytes it reads.
struct Lz77Words {
    const WordIndex *index; int32_t dict_min;
};
// one launch, n_warps persistent warps (a kernel per lazy 0..2, with the dictionary step when d.dict_min != 0)
void launch_lz77_cmds(const Lz77Params &p, const Lz77Dict &d, cudaStream_t st);
// the same with the dictionary step under every transform (w.dict_min 4..32)
void launch_lz77_words(const Lz77Params &p, const Lz77Words &w, cudaStream_t st);

}  // namespace dv
