// Host side of umma_gemm (csrc/umma_gemm.cu): problem description, tile-shape selection, launch; bf16 hi/lo plane
// preparation for the B operands.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <algorithm>
#include <cstring>
#include <string>
#include "umma_gemm.cuh"

namespace l2h {
namespace umma {

// fp32 activation tensor seen as (channel, position, seq_inner, seq_outer); strides in floats
struct ASource {
    const float* base = nullptr;
    int64_t channels = 0;
    int64_t n_pos = 1, pos_stride = 0;
    int64_t n_inner = 1, inner_stride = 0;
    int64_t n_outer = 1, outer_stride = 0;
};

// bf16 hi/lo planes of a B operand: K-major [plane][z][N][ld >= K] or MN-major [plane][z][K][ld >= N]
struct BPlanes {
    const __nv_bfloat16* base = nullptr;
    int64_t ld = 0;            // row stride in elements (multiple of 8)
    int64_t z_stride = 0;      // elements between batch entries
    int64_t plane_stride = 0;  // elements between the hi and the lo plane
    int nz = 1;
    bool mn_major = false;
};

struct GemmDesc {
    ASource a0, a1;
    KChunk chunks[MAX_CHUNKS];
    int n_chunks = 0;
    int rows_per_seq = 0, nseq = 1;   // M space (rows = nseq * rows_per_seq)
    int pos_bias = 0;
    BPlanes b;
    bool b_by_seq = false;            // B batch index = sequence index (attention)
    int N = 0, K = 0;                 // K = extent of B along k (zero fill beyond)
    int passes = 3;
    float* C = nullptr;
    const float* R = nullptr;
    int64_t ldc = 0, c_seq_stride = 0, c_inner_stride = 0;
    int c_inner = 0;
    const float* bias = nullptr;
    const float* prelu = nullptr;     // scalar PReLU slope, or
    const float* prelu_vec = nullptr; // one slope per column (at most one of the two)
    const float* ln_g = nullptr;
    const float* ln_b = nullptr;
    float alpha = 1.f;
    bool pdl = false;                 // launch with the programmatic-serialization attribute (kernel chains)
};

inline void set_plain_chunks(GemmDesc& g, int K, bool ln = false) {
    g.n_chunks = (K + KC - 1) / KC;
    for (int j = 0; j < g.n_chunks; ++j) { g.chunks[j].c0 = (short)(j * KC); g.chunks[j].dp = 0; g.chunks[j].flags = ln ? 2 : 0; }
}
// windows of `w` consecutive positions x `C` channels (C a multiple of 64): k = dp*C + c
inline void set_window_chunks(GemmDesc& g, int C, int w, bool ln = false) {
    const int cpr = C / KC;
    g.n_chunks = cpr * w;
    for (int j = 0; j < g.n_chunks; ++j) { g.chunks[j].c0 = (short)((j % cpr) * KC); g.chunks[j].dp = (signed char)(j / cpr); g.chunks[j].flags = ln ? 2 : 0; }
}

cudaError_t configure();                 // per-device kernel attributes; call outside stream capture before the first launch
cudaError_t launch(const GemmDesc& g, cudaStream_t st, std::string* why = nullptr);
// fp32 matrix (any strides) -> bf16 hi/lo planes: hi[r*ld + c] + lo[r*ld + c] ~= src[r*row_stride + c*col_stride]
cudaError_t split_planes(const float* src, int64_t row_stride, int64_t col_stride, int rows, int cols, int64_t ld,
                         __nv_bfloat16* hi, __nv_bfloat16* lo, cudaStream_t st);

}  // namespace umma
}  // namespace l2h
