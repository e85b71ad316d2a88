// Launch geometry of the separator kernels, shared by the engine (sep_engine.cu) and the kernel tests
// (tests/kernels/kernel_harness.cu), so that the tests launch every kernel exactly as the engine does.
#pragma once
#include <algorithm>
#include <utility>

#include "sep_kernels.cuh"
#include "hop_kernels.cuh"

namespace l2h {

// front_many_kernel / back_many_kernel: `workers` CTAs (clusters) walk (stream, chunk-of-frames) items, each stream's T
// frames cut into as many chunks as there are workers per stream
struct ChunkWalk { int chunk, n_chunks, workers; };
static inline ChunkWalk chunk_walk(int B, int T, int max_workers) {
    const int per_stream = std::max(1, max_workers / B);
    const int chunk = (T + per_stream - 1) / per_stream;
    const int n_chunks = (T + chunk - 1) / chunk;
    return {chunk, n_chunks, std::min(max_workers, B * n_chunks)};
}
// one CTA per SM (150 KB of filters)
static inline ChunkWalk front_many_walk(int B, int T) { return chunk_walk(B, T, NUM_SMS); }
// clusters of BACK_CL, as many as stay resident together (3 CTAs of 72 KB per SM)
static inline ChunkWalk back_many_walk(int B, int T) { return chunk_walk(B, T, NUM_SMS * 3 / BACK_CL); }

// grids of the mid-section kernels: persistent over (stream, row tile) items, as many CTAs per SM as their shared memory
// allows (fused 225 KB -> 1, mid_a 107 KB -> 2, mid_b 68 KB -> 3, mid_c 50 KB -> 4)
static inline int mid_items(int B) { return B * ((NF + MID_RT - 1) / MID_RT); }
static inline dim3 mid_grid_for(int B, int ctas_per_sm) { return dim3(std::min(NUM_SMS * ctas_per_sm, mid_items(B))); }
// many streams: the section is throughput-bound and one fused CTA per SM (8 warps) cannot hide its own latencies; the
// three smaller kernels run 2-4 CTAs per SM (same arithmetic, +3 small global round trips)
static inline bool mid_split_for_throughput(int B) { return mid_items(B) > NUM_SMS; }

// CTAs of attn_cluster_kernel the current device holds at once
static inline int attn_cluster_resident() {
    static int wave[64] = {};
    return resident_ctas(wave, attn_cluster_kernel, 256, 0);
}
// few frames in flight -> split every head's 50-row window over 8-CTA clusters while they all fit in one wave
static inline int attn_splits(int B, int T) {
    return (B * T * NHEAD * ATT_CL <= attn_cluster_resident()) ? ATT_CL : 1;
}

// dynamic shared memory of the separator kernels that address records, in their form for Map (cudaFuncSetAttribute
// applies to the current device)
template <class Map>
static inline cudaError_t set_sep_smem() {
    const std::pair<const void*, size_t> kernels[] = {
        {(const void*)qkv_kernel_t<Map>, QKV_SMEM},          {(const void*)qkv_many_kernel_t<Map>, QKV_MANY_SMEM},
        {(const void*)attn_out_kernel_t<Map>, AOUT_SMEM},    {(const void*)back_kernel_t<Map>, BACK_SMEM},
        {(const void*)back_many_kernel_t<Map>, BACK_MANY_SMEM}, {(const void*)front_kernel_t<Map>, FRONT_SMEM},
        {(const void*)front_many_kernel_t<Map>, FRONT_SMEM}, {(const void*)mid_kernel_t<Map>, MID_SMEM},
        {(const void*)mid_b_kernel_t<Map>, MID_B_SMEM},      {(const void*)front1_kernel_t<Map>, FRONT1_SMEM}};
    for (const auto& k : kernels)
        if (cudaError_t e = cudaFuncSetAttribute(k.first, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k.second)) return e;
    return cudaSuccess;
}

}  // namespace l2h
