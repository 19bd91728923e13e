// dv_kernels.h -- host-visible launch wrappers of the divANS kernels.
#pragma once
#include "dv_common.cuh"

namespace dv {
constexpr int DECODE_BLOCK_THREADS = 64;

// Resident blocks per SM of a stream kernel (register-limited; the kernels use ~2.3 KB of shared memory per block, so no
// shared-memory carve-out preference is set).
template <typename K> static inline int stream_kernel_blocks_per_sm(K kernel, int threads, size_t dyn_smem) {
    int nb = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, threads, dyn_smem);
    return nb;
}

void launch_frame(const FrameParams &p, uint8_t *payload, uint64_t payload_cap_bytes, cudaStream_t st);   // frame + payload scan + demux (3 launches)
// v2 engine (dv2_kernels.cu), lanes_per_stream = 16 (two streams per warp) or 8 (four)
void launch_decode_v2(int lanes_per_stream, const DecodeParams &p, uint32_t n_blocks, cudaStream_t st);
int decode_max_blocks_per_sm_v2(int lanes_per_stream);
int decode_groups_per_block_v2(int lanes_per_stream);
void launch_encode_model(const EncodeParams &p, uint32_t n_blocks, cudaStream_t st);   // groups of 16 lanes
void launch_encode_flush_mux(const EncodeParams &p, cudaStream_t st);                  // reverse rANS + mux/CRC (2 launches)
int encode_max_blocks_per_sm();
// the reference's feature="blend" probability model (dv_blend.cuh, dv_kernels.cu): 16 lanes per stream, no literal fast loop
void launch_decode16_blend(const DecodeParams &p, uint32_t n_blocks, cudaStream_t st);
int decode_max_blocks_per_sm16_blend();
void launch_encode_model_blend(const EncodeParams &p, uint32_t n_blocks, cudaStream_t st);
void launch_rcp15_init(uint64_t *tab, cudaStream_t st);
}  // namespace dv
