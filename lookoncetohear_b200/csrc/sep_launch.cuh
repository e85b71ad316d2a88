// Launch geometry of the separator kernels, shared by the engine (sep_engine.cu) and the kernel tests
// (tests/kernels/kernel_harness.cu), so that the tests launch every kernel exactly as the engine does.  A kernel launched
// from more than one place has one launcher here, the only place that states its grid, block, dynamic shared memory and
// cluster shape; it takes the kernel's own arguments in the kernel's order, after what only the geometry needs.
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

// dynamic shared memory of mid_a_kernel and mid_c_kernel, which address no records (one form serves every call)
static inline cudaError_t set_mid_split_smem() {
    cudaError_t e = cudaFuncSetAttribute(mid_a_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MID_A_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(mid_c_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MID_C_SMEM);
    return e;
}

// tail_kernel: 16 CTAs per cluster is a non-portable size.  Sets the dynamic shared memory and the non-portable cluster
// size of both Map forms on the current device and returns how many clusters the device can hold at once (0: it cannot
// be scheduled, and callers keep the separate kernels).  Clears the error state it may leave.
static inline int set_tail_attrs() {
    int ncl = 0;
    if (cudaFuncSetAttribute(tail_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TAIL_SMEM) == cudaSuccess &&
        cudaFuncSetAttribute(tail_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess) {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(TAIL_CL, 1); cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = TAIL_SMEM;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = TAIL_CL; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        if (cudaOccupancyMaxActiveClusters(&ncl, tail_kernel, &cfg) != cudaSuccess) ncl = 0;
    }
    if (ncl > 0 &&      // the slot-list form: same resources, so the same cluster count
        (cudaFuncSetAttribute(tail_kernel_t<Records>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TAIL_SMEM) != cudaSuccess ||
         cudaFuncSetAttribute(tail_kernel_t<Records>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess))
        ncl = 0;
    cudaGetLastError();
    return ncl;
}

// front_kernel: grid (T + gate, B), the T frames and, with gate = 1, each stream's speaker-gate memo CTA
template <class Map>
inline cudaError_t launch_front(bool pdl, cudaStream_t st, int B, int gate, const float* x, int64_t x_bstride, int64_t x_cstride,
                                int x_len, float* X, float* state, Map recs, const SepWeights& w, int T, int pos_rel, const float* emb,
                                float* spk_pre, int frame_k, int frames_total, int sample_off, const uint8_t* active) {
    return launch_k(pdl, front_kernel_t<Map>, dim3(T + gate, B), dim3(256), FRONT_SMEM, st, x, x_bstride, x_cstride, x_len, X, state,
                    recs, w, T, pos_rel, emb, spk_pre, frame_k, frames_total, sample_off, active);
}
// front_many_kernel: g.workers CTAs walk the chunks, then `gate` speaker-gate CTAs per stream
template <class Map>
inline cudaError_t launch_front_many(bool pdl, cudaStream_t st, int gate, const ChunkWalk& g, const float* x, int64_t x_bstride,
                                     int64_t x_cstride, int x_len, float* X, float* state, Map recs, const SepWeights& w, int T,
                                     int pos_rel, const float* emb, float* spk_pre, int n_streams, const uint8_t* active) {
    return launch_k(pdl, front_many_kernel_t<Map>, dim3(g.workers + gate * n_streams, 1), dim3(256), FRONT_SMEM, st, x, x_bstride,
                    x_cstride, x_len, X, state, recs, w, T, pos_rel, emb, spk_pre, g.chunk, g.n_chunks, n_streams, g.workers, active);
}
// front1_kernel: grid (TAIL_TILES + gate, B), the frame's 13 bin tiles and, with gate = 1, the speaker-gate CTA
template <class Map>
inline cudaError_t launch_front1(bool pdl, cudaStream_t st, int B, int gate, const float* x, int64_t x_bstride, int64_t x_cstride,
                                 int x_len, float* X, float* state, Map recs, const SepWeights& w, const BlockWeights& w0, float* GX,
                                 int pos_rel, const float* emb, float* spk_pre, const uint8_t* active) {
    return launch_k(pdl, front1_kernel_t<Map>, dim3(TAIL_TILES + gate, B), dim3(256), FRONT1_SMEM, st, x, x_bstride, x_cstride, x_len,
                    X, state, recs, w, w0, GX, pos_rel, emb, spk_pre, active);
}
// the middle section in one kernel, persistent over (stream, row tile) items, one CTA per SM
template <class Map>
inline cudaError_t launch_mid(bool pdl, cudaStream_t st, const float* Y, float* X, float* QKV, float* state, Map recs, int blk,
                              const BlockWeights& w, int n_streams, const uint8_t* active) {
    return launch_k(pdl, mid_kernel_t<Map>, mid_grid_for(n_streams, 1), dim3(256), MID_SMEM, st, Y, X, QKV, state, recs, blk, w,
                    n_streams, active);
}
// the middle section in three kernels, each persistent over (stream, row tile) items
inline cudaError_t launch_mid_a(bool pdl, cudaStream_t st, const float* Y, float* X, float* GI, const BlockWeights& w, int n_streams,
                                int64_t hop_stride, int n_hops) {
    return launch_k(pdl, mid_a_kernel, mid_grid_for(n_streams, 2), dim3(256), MID_A_SMEM, st, Y, X, GI, w, n_streams, hop_stride, n_hops);
}
template <class Map>
inline cudaError_t launch_mid_b(bool pdl, cudaStream_t st, const float* GI, float* Hn, int64_t hop_stride, int n_hops, float* state,
                                Map recs, int blk, const BlockWeights& w, int n_streams, const uint8_t* active) {
    return launch_k(pdl, mid_b_kernel_t<Map>, mid_grid_for(n_streams, 3), dim3(256), MID_B_SMEM, st, GI, Hn, hop_stride, n_hops, state,
                    recs, blk, w, n_streams, active);
}
inline cudaError_t launch_mid_c(bool pdl, cudaStream_t st, const float* Hn, float* X, float* QKV, const BlockWeights& w, int n_streams,
                                int64_t hop_stride, int n_hops) {
    return launch_k(pdl, mid_c_kernel, mid_grid_for(n_streams, 4), dim3(256), MID_C_SMEM, st, Hn, X, QKV, w, n_streams, hop_stride, n_hops);
}
// tail_kernel: one cluster of TAIL_CL CTAs per stream, grid (TAIL_CL, B); set_tail_attrs() must have returned > 0
template <class Map>
inline cudaError_t launch_tail(bool pdl, cudaStream_t st, int B, const float* Y, float* X, float* state, Map recs, int blk,
                               const BlockWeights& w, const NextIh& nx, int apply_gate, int frame_k, const uint8_t* active) {
    return launch_cluster(pdl, dim3(TAIL_CL, 1, 1), tail_kernel_t<Map>, dim3(TAIL_CL, B), dim3(256), TAIL_SMEM, st, Y, X, state, recs,
                          blk, w, nx, apply_gate, frame_k, active);
}
// lstm_cell_rows_kernel: one thread per (row, hidden unit)
template <class Map>
inline cudaError_t launch_lstm_cell_rows(bool pdl, cudaStream_t st, const float* gates, float* state, Map recs, int blk, float* Hout,
                                         int64_t rows, const uint8_t* active) {
    return launch_k(pdl, lstm_cell_rows_kernel_t<Map>, dim3((unsigned)((rows * 64 + 255) / 256)), dim3(256), 0, st, gates, state, recs,
                    blk, Hout, (int)rows, active);
}
// qkv_kernel: grid (T, B); the projections run inside (pre == nullptr) or are given, with less shared memory
template <class Map>
inline cudaError_t launch_qkv(bool pdl, cudaStream_t st, int B, const float* X, const float* pre, float* Q, float* Kall, float* Vall,
                              float* state, Map recs, int blk, const BlockWeights& w, int T, int frame_k, const uint8_t* active) {
    return launch_k(pdl, qkv_kernel_t<Map>, dim3(T, B), dim3(QKV_THREADS), pre ? QKV_PRE_SMEM : QKV_SMEM, st, X, pre, Q, Kall, Vall,
                    state, recs, blk, w, T, frame_k, active);
}
// qkv_many_kernel: `ctas` persistent CTAs walk the frames
template <class Map>
inline cudaError_t launch_qkv_many(bool pdl, cudaStream_t st, int ctas, const float* pre, float* Q, float* Kall, float* Vall,
                                   float* state, Map recs, int blk, const BlockWeights& w, int T, int n_frames, const uint8_t* active) {
    return launch_k(pdl, qkv_many_kernel_t<Map>, dim3(ctas), dim3(QKV_THREADS), QKV_MANY_SMEM, st, pre, Q, Kall, Vall, state, recs, blk,
                    w, T, n_frames, active);
}
template <class Map>
inline cudaError_t launch_kv_gather(bool pdl, cudaStream_t st, int B, const float* state, Map recs, int blk, float* Kall, float* Vall,
                                    int T) {
    return launch_k(pdl, kv_gather_kernel_t<Map>, dim3(ATT - 1, B * NHEAD), dim3(128), 0, st, state, recs, blk, Kall, Vall, T);
}
// attn_kernel (a CTA per query frame and head), attn_tile_kernel (ATT_TQ query frames per CTA; the linear scratch only, no
// frame_k) or attn_cluster_kernel (each window split over an ATT_CL-CTA cluster)
enum class AttnForm { query, tile, cluster };
template <class Map>
inline cudaError_t launch_attention(AttnForm form, bool pdl, cudaStream_t st, int B, const float* Q, const float* Kall,
                                    const float* Vall, const float* state, Map recs, int blk, float* Z, int T, int frame_k) {
    if (form == AttnForm::cluster)
        return launch_cluster(pdl, dim3(1, ATT_CL, 1), attn_cluster_kernel_t<Map>, dim3(T, NHEAD * ATT_CL, B), dim3(256), 0, st, Q, Kall,
                              Vall, state, recs, blk, Z, T, frame_k);
    if (form == AttnForm::tile)
        return launch_k(pdl, attn_tile_kernel, dim3((T + ATT_TQ - 1) / ATT_TQ, NHEAD, B), dim3(256), 0, st, Q, Kall, Vall, Z, T);
    return launch_k(pdl, attn_kernel_t<Map>, dim3(T, NHEAD, B), dim3(256), 0, st, Q, Kall, Vall, state, recs, blk, Z, T, frame_k);
}
template <class Map>
inline cudaError_t launch_attn_out(bool pdl, cudaStream_t st, int B, const float* Z, float* X, const float* state, Map recs,
                                   const BlockWeights& w, int apply_gate, int T) {
    return launch_k(pdl, attn_out_kernel_t<Map>, dim3(T, B), dim3(256), AOUT_SMEM, st, Z, X, state, recs, w, apply_gate, T);
}
template <class Map>
inline cudaError_t launch_ln_frame_res(bool pdl, cudaStream_t st, int B, const float* P, float* X, const float* state, Map recs,
                                       const BlockWeights& w, int apply_gate, int T) {
    return launch_k(pdl, ln_frame_res_kernel_t<Map>, dim3(T, B), dim3(256), 0, st, P, X, state, recs, w, apply_gate, T);
}
// back_kernel: a cluster of BACK_CL per frame and stream
template <class Map>
inline cudaError_t launch_back(bool pdl, cudaStream_t st, int B, const float* X, float* y, int64_t y_bstride, int64_t y_cstride,
                               int y_len, float* state, Map recs, const SepWeights& w, int T, int pos_rel, int frame_k, int frames_total,
                               int sample_off, int64_t hist_stride, const uint8_t* active) {
    return launch_cluster(pdl, dim3(BACK_CL, 1, 1), back_kernel_t<Map>, dim3(BACK_CL * T, B), dim3(256), BACK_SMEM, st, X, y, y_bstride,
                          y_cstride, y_len, state, recs, w, T, pos_rel, frame_k, frames_total, sample_off, hist_stride, active);
}
// back_many_kernel: g.workers clusters of BACK_CL walk the chunks
template <class Map>
inline cudaError_t launch_back_many(bool pdl, cudaStream_t st, const ChunkWalk& g, const float* X, float* y, int64_t y_bstride,
                                    int64_t y_cstride, int y_len, float* state, Map recs, const SepWeights& w, int T, int pos_rel,
                                    int n_streams, const uint8_t* active) {
    return launch_cluster(pdl, dim3(BACK_CL, 1, 1), back_many_kernel_t<Map>, dim3(BACK_CL * g.workers, 1), dim3(256), BACK_MANY_SMEM,
                          st, X, y, y_bstride, y_cstride, y_len, state, recs, w, T, pos_rel, g.chunk, g.n_chunks, n_streams, active);
}

// The slot-list helpers.  gather_h_kernel / scatter_hc_kernel copy blocks b0 .. b0 + n_blocks - 1 of the records, between
// the state and the copies Hg, Cg [blocks][n_streams][97][64] (Cg may be null for the gather): the kernels address
// block blk of a record from the state pointer they get, so a pointer b0 blocks further makes their block 0 block b0;
// one thread per float4 of a block's h (and c).
inline dim3 hc_copy_grid(int n_blocks, int n_streams) {
    return dim3((unsigned)(((int64_t)n_blocks * n_streams * FC / 4 + 255) / 256));
}
inline cudaError_t launch_gather_h(cudaStream_t st, int b0, const float* state, Records recs, int n_blocks, int n_streams, float* Hg,
                                   float* Cg) {
    const int64_t o = (int64_t)b0 * n_streams * FC;
    return launch_k(false, gather_h_kernel, hc_copy_grid(n_blocks, n_streams), dim3(256), 0, st, state + b0 * BK_STRIDE, recs,
                    n_blocks, n_streams, Hg + o, Cg ? Cg + o : nullptr);
}
inline cudaError_t launch_scatter_hc(cudaStream_t st, int b0, float* state, Records recs, int n_blocks, int n_streams, const float* Hg,
                                     const float* Cg) {
    const int64_t o = (int64_t)b0 * n_streams * FC;
    return launch_k(false, scatter_hc_kernel, hc_copy_grid(n_blocks, n_streams), dim3(256), 0, st, state + b0 * BK_STRIDE, recs,
                    n_blocks, n_streams, Hg + o, Cg + o);
}
// inter_gate_mask_kernel: grid (T, B)
inline cudaError_t launch_inter_gate_mask(cudaStream_t st, int B, float* gx, Records recs, int T) {
    return launch_k(false, inter_gate_mask_kernel, dim3(T, B), dim3(256), 0, st, gx, recs, T);
}
// inter_h_last_kernel: one CTA per row; Hg = the block's part of gather_h_kernel's copy
inline cudaError_t launch_inter_h_last(cudaStream_t st, int B, const float* Y, float* Hg, Records recs, int T) {
    return launch_k(false, inter_h_last_kernel, dim3(B), dim3(256), 0, st, Y, Hg, recs, T);
}

// The state kernels (l2h_sep_state_init, l2h_sep_state_reset_streams, l2h_sep_stream_dev and the pipelined graph).  Their
// launchers sit here rather than beside the kernels in sep_kernels.cuh: defined there, they changed the code nvcc
// generated for kernels that do not use them.
// state_init_kernel: the whole state of B records of `stride` floats, 592 CTAs of 256 threads
inline cudaError_t launch_state_init(cudaStream_t st, float* state, int64_t stride, int B) {
    const int64_t total = (int64_t)(sizeof(StateHeader) / 4) + (int64_t)B * stride;
    return launch_k(false, state_init_kernel, dim3(592), dim3(256), 0, st, state, total, stride, B);
}
// reset_streams_kernel over the host list slots[0 .. n-1]: one launch per RESET_MAX_SLOTS of them, each of ~2 CTAs per SM
// over all its records (each record is 6 MB of stores)
inline cudaError_t launch_reset_streams(cudaStream_t st, float* state, int64_t sstride, const int32_t* slots, int n) {
    for (int i0 = 0; i0 < n; i0 += RESET_MAX_SLOTS) {
        const int k = std::min(RESET_MAX_SLOTS, n - i0);
        SlotList sl{};
        std::copy(slots + i0, slots + i0 + k, sl.s);
        const unsigned per_rec = (unsigned)std::max(1, 2 * NUM_SMS / k);
        if (cudaError_t e = launch_k(false, reset_streams_kernel, dim3(per_rec, k), dim3(256), 0, st, state, sstride, sl)) return e;
    }
    return cudaSuccess;
}
// advance_header_kernel, the pipelined graph's last node: the header and each of the n_streams dense records advance by
// `frames` frames and one call.  One CTA of 256 threads.
inline cudaError_t launch_advance_header(cudaStream_t st, float* state, int64_t sstride, int n_streams, int frames) {
    return launch_k(false, advance_header_kernel, dim3(1), dim3(256), 0, st, state, sstride, n_streams, frames);
}
// set_clip_base_kernel: one thread
inline cudaError_t launch_set_clip_base(cudaStream_t st, float* state) {
    return launch_k(false, set_clip_base_kernel, dim3(1), dim3(1), 0, st, state);
}

}  // namespace l2h
