// dv_kernels.h -- host-visible launch wrappers of the divANS kernels.
#pragma once
#include "dv_common.cuh"

namespace dv {
constexpr int DECODE_BLOCK_THREADS = 64;   // the encoder's model pass and the blend decoder: two warps of two 16-lane groups per block

// Resident blocks per SM of a stream kernel (register-limited; the kernels use ~2.3 KB of shared memory per block, so no
// shared-memory carve-out preference is set).
template <typename K> static inline int stream_kernel_blocks_per_sm(K kernel, int threads, size_t dyn_smem) {
    int nb = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, threads, dyn_smem);
    return nb;
}

void launch_frame(const FrameParams &p, uint8_t *payload, uint64_t payload_cap_bytes, cudaStream_t st);   // frame + payload scan + demux (3 launches)
// the stream decoder (dv2_kernels.cu), lanes_per_stream = 16 (two streams per warp) or 8 (four).  blend = the reference's
// feature="blend" probability model (dv_blend.cuh): 16 lanes per stream whatever lanes_per_stream says, no literal fast loop,
// DECODE_BLOCK_THREADS per block.  Both models keep 32 groups per SM resident, so decode_max_blocks_per_sm_v2(16) x
// decode_groups_per_block_v2(16) is the blend model's residency too.
void launch_decode_v2(int lanes_per_stream, bool blend, const DecodeParams &p, uint32_t n_blocks, cudaStream_t st);
void launch_decode_blend(const DecodeParams &p, const RecParams *r, uint32_t n_blocks, cudaStream_t st);   // its blend kernels (r: recording)
int decode_max_blocks_per_sm_v2(int lanes_per_stream);
int decode_groups_per_block_v2(int lanes_per_stream);
void launch_encode_model(const EncodeParams &p, uint32_t n_blocks, cudaStream_t st);   // groups of 16 lanes
void launch_encode_flush_mux(const EncodeParams &p, cudaStream_t st);                  // reverse rANS + mux/CRC (2 launches)
int encode_max_blocks_per_sm();
// the encoder's model pass under the blend model (dv_encode.cu built with DV_BLEND)
void launch_encode_model_blend(const EncodeParams &p, uint32_t n_blocks, cudaStream_t st);
void launch_rcp15_init(uint64_t *tab, cudaStream_t st);
// model selection: the cost-only model passes (no logs: EncodeParams::cost_tab / tally), the fan-out of n streams to n x C
// virtual streams (candidate-major) and the per-stream argmin
void launch_encode_tally(const EncodeParams &p, uint32_t n_blocks, cudaStream_t st);
void launch_encode_tally_blend(const EncodeParams &p, uint32_t n_blocks, cudaStream_t st);
void launch_auto_fanout(const uint64_t *in_off, const uint64_t *in_len, uint64_t n, uint32_t n_cands, uint64_t *v_off, uint64_t *v_len,
                        uint32_t *v_pm, cudaStream_t st);
void launch_auto_select(const uint64_t *tally, const int32_t *v_status, uint64_t n, uint32_t n_cands, uint32_t *chosen, uint64_t *cost,
                        cudaStream_t st);
// per-context mixing values: the binned cost pass over the n x k fan-out (BinParams), the kernel that builds each stream's
// mixed record from the per-entry winners, and the choice between the best uniform record and the mixed one (dv_encode.cu)
void launch_encode_bins(const EncodeParams &p, const BinParams &b, uint32_t n_blocks, cudaStream_t st);
void launch_encode_bins_blend(const EncodeParams &p, const BinParams &b, uint32_t n_blocks, cudaStream_t st);
void launch_mixmap_map(const uint64_t *best, uint64_t n, const MixValues &vals, uint8_t *records, uint32_t *mix_idx, cudaStream_t st);
void launch_mixmap_select(const uint64_t *tally, const int32_t *v_status, const uint64_t *x_tally, const int32_t *x_status, uint64_t n,
                          const MixValues &vals, const uint8_t *records, uint32_t *rec_idx, uint32_t *chosen, uint64_t *cost, uint8_t *mixing,
                          cudaStream_t st);
// decoding to command lists: the recording decoder (16 lanes per stream, either model) and the pack kernel that finishes the
// blobs (dv_kernels.cu)
void launch_decode_v2_rec(bool blend, const DecodeParams &p, const RecParams &r, uint32_t n_blocks, cudaStream_t st);
void launch_pack_cmds(const DecodeParams &p, const RecParams &r, cudaStream_t st);

// replaying command lists to raw bytes (dv_replay.cu): list i is blobs[blob_off[i] .. +blob_len[i]), its bytes go to
// out[out_off[i] .. +out_cap[i]); window 10..24 for every list, or 0 for each list's header window (clamped to 10..24)
struct ReplayParams {
    const uint8_t *blobs; const uint64_t *blob_off, *blob_len;
    uint8_t *out; const uint64_t *out_off, *out_cap; uint64_t *out_len; int32_t *status;
    uint32_t n_lists; int32_t window;
    uint32_t *work_counter; const uint8_t *tables;
};
void launch_replay_cmds(const ReplayParams &p, int sm_count, cudaStream_t st);   // one launch, persistent warps
}  // namespace dv
