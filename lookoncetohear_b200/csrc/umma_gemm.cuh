// umma_gemm: the dense contractions of both networks on the Hopper tensor cores (wgmma).
//
//     C[m, n] = epi( alpha * sum_k A(m)[k] * B[n][k] + bias[n] )          (fp32 in, fp32 out)
//
// One persistent CTA per SM, 128-row tiles:
//   * operands arrive through TENSOR-MAP TMA (cp.async.bulk.tensor, SASS UTMALDG) with 128-byte swizzle:
//     the fp32 activation tile [128 rows x 64 k] into a staging ring, the weight tile (bf16, split on the host
//     side of the engine into hi/lo planes) straight into the operand ring;
//   * a converter warpgroup (thread = row) turns the staged fp32 rows into bf16 hi/lo operand tiles in the
//     canonical K-major SWIZZLE_128B layout (optionally applying LayerNorm over the 64 channels of the row first
//     -- nn.LayerNorm semantics -- so that LN -> Linear pairs are one kernel);
//   * two math warpgroups, 64 rows each, issue wgmma (bf16 x bf16 -> fp32, M = 64, N = BN in {64, 128}) with the
//     accumulators in registers.  passes = 3 gives fp32-grade products from three bf16 MMAs
//     (a_hi*b_hi + a_lo*b_hi + a_hi*b_lo, relative error ~2^-16 per product: the "bf16x3" split); passes = 2 drops the
//     b_lo term (bf16 weights, activations still split: the offline bf16 configuration); passes = 1 is plain bf16;
//   * the same warpgroups then apply bias / PReLU / residual / scale and store fp32 rows (transposed through shared
//     memory so that every warp store writes whole 128-byte lines); the TMA warp and the converter keep filling the
//     operand ring for the next tile meanwhile.
//
// "Rows" (the M space) are (sequence, position) pairs described by a 4-D tensor map (channel, position,
// seq_inner, seq_outer); a k-chunk of 64 channels may come from a position offset `dp` (overlapping windows: the
// enrollment net's unfold / ConvTranspose1d become plain GEMMs, out-of-range positions are zero-filled by TMA)
// and from one of two source tensors (concatenated K).  B is K-major [n][k] or MN-major [k][n] (attention P.V).
//
// Reference call sites this replaces (addmm / conv / bmm): tfgridnet_causal.py:510-516, :524-538, :547-551,
// :583-588; tfgridnet_orig/tfgridnet.py:117-125 (espnet2 GridNetBlock GEMMs and the T x T attention products).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include "common.cuh"

namespace l2h {
namespace umma {

constexpr int BM = 128;          // rows per tile: two math warpgroups of 64
constexpr int KC = 64;           // k-chunk: 64 bf16 = one 128-byte swizzle row
constexpr int NTHREADS = 416;    // warps 0-3: converter, 4-7 and 8-11: math (rows 0-63, 64-127), warp 12: TMA
constexpr int MAX_NSTG = 2;      // fp32 staging ring slots (32 KB each)
constexpr int STG_BYTES = BM * KC * 4;
constexpr int OPA_PLANE = BM * KC * 2;   // 16 KB per bf16 plane
constexpr int MAX_CHUNKS = 96;

struct KChunk {
    short c0;             // first channel of the chunk inside the source row
    signed char dp;       // position offset of the chunk (windows)
    unsigned char flags;  // bit0: source tensor 1, bit1: LayerNorm over the 64 channels
};

struct Params {
    CUtensorMap tmA0, tmA1, tmB;
    KChunk chunks[MAX_CHUNKS];
    int n_chunks;
    int P_TILE, S_TILE;        // positions x sequences per tile (P_TILE * S_TILE <= 128)
    int rows_per_seq, nseq;    // valid M space
    int seq_inner;             // sequence -> tensor-map coordinates (seq % seq_inner, seq / seq_inner)
    int pos_bias;              // added to every position coordinate (may be negative: zero-filled halo)
    int N, BN, n_tiles_n, passes, b_mn_major, b_by_seq;
    int nop;                   // operand ring slots
    int nstg;                  // fp32 staging ring slots (1 or 2)
    int vec_ok;                // C/R rows 16-byte aligned: float4 epilogue accesses
    int b_resident;            // all k-chunks of the B tile stay in shared memory for the CTA's whole life
    // epilogue
    float* C;
    const float* R;
    long long ldc, c_seq_stride, c_inner_stride;
    int c_inner;
    const float* bias;
    const float* prelu;
    const float* prelu_vec;
    const float* ln_g;
    const float* ln_b;
    float alpha;
};

}  // namespace umma
}  // namespace l2h
