// rows_gemm: C[m, n] = epi( sum_k A(m)[k] * Wt[k][n] + bias[n] ),  fp32 on the CUDA cores with
// paired fp32 FMAs.  "Rows" are (stream, frame, freq-bin) activations: M is huge or tiny, K and N are
// small (64..512), so W^T lives in shared memory and A streams through once.
//
// A rows may be overlapping windows of a [seq][pos][lda] tensor (the enrollment net's unfold /
// ConvTranspose1d become plain GEMMs this way): row m -> seq = m / a_rows_per_seq,
// p = m % a_rows_per_seq, address A + seq*a_seq_stride + p*lda, K contiguous floats.
//
// Optional prologue: LayerNorm over the K==64 channels of each row (nn.LayerNorm semantics:
// biased variance, eps inside the sqrt).  Epilogues: bias | bias+PReLU | bias+residual.
#pragma once
#include <algorithm>
#include <cstdlib>
#include "common.cuh"

namespace l2h {

struct GemmArgs {
    const float* A;
    int64_t lda;
    int a_rows_per_seq;      // 0 => plain row-major
    int64_t a_seq_stride;
    const float* Wt;         // [K][N]
    const float* bias;       // [N] or null
    float* C;
    int64_t ldc;
    int c_rows_per_seq;      // 0 => plain; else row m -> (seq = m / c_rows_per_seq, p = m % c_rows_per_seq)
    int64_t c_seq_stride;    //   offset = (seq / c_inner)*c_seq_stride + (seq % c_inner)*c_inner_stride + p*ldc
    int c_inner;             //   (c_inner <= 1 => offset = seq*c_seq_stride + p*ldc)
    int64_t c_inner_stride;
    const float* R;          // residual, indexed like C (may alias C); null => none
    const float* ln_g;       // LN prologue (requires K == 64); null => none
    const float* ln_b;
    const float* prelu;      // scalar slope pointer; null => none
    const float* prelu_vec;  // per-output-column slopes [N]; null => none
    int M, N, K;
};

constexpr int GK = 64;  // K tile

template <int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
rows_gemm_kernel(const GemmArgs g) {
    constexpr int NT = (BM / TM) * (BN / TN);
    constexpr int APAD = 4;
    extern __shared__ __align__(16) float smem[];
    float* As = smem;                      // [GK][BM + APAD]  (transposed: k-major)
    float* Bs = smem + GK * (BM + APAD);   // [GK][BN]

    TraceScope trace_(TK_GEMM, g.A);
    griddep_launch();
    const int tid = threadIdx.x;
    const int m0 = blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    const int tx = tid % (BN / TN);
    const int ty = tid / (BN / TN);

    float2 acc[TM][TN / 2];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN / 2; ++j) acc[i][j] = make_float2(0.f, 0.f);

    griddep_wait();
    for (int k0 = 0; k0 < g.K; k0 += GK) {
        // ---- A tile: 16 lanes per row, one float4 each (64 floats / row) ------------------
        for (int r = tid / 16; r < BM; r += NT / 16) {
            const int m = m0 + r;
            const int c4 = tid % 16;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m < g.M) {
                const float* ap;
                if (g.a_rows_per_seq > 0) {
                    const int seq = m / g.a_rows_per_seq, p = m % g.a_rows_per_seq;
                    ap = g.A + (int64_t)seq * g.a_seq_stride + (int64_t)p * g.lda;
                } else {
                    ap = g.A + (int64_t)m * g.lda;
                }
                v = *reinterpret_cast<const float4*>(ap + k0 + c4 * 4);
            }
            if (g.ln_g != nullptr) {   // LayerNorm over the 64 channels held by these 16 lanes
                float s = v.x + v.y + v.z + v.w;
#pragma unroll
                for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
                const float mu = s * (1.f / 64.f);
                const float dx = v.x - mu, dy = v.y - mu, dz = v.z - mu, dw = v.w - mu;
                float q = dx * dx + dy * dy + dz * dz + dw * dw;
#pragma unroll
                for (int o = 8; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
                const float rs = rsqrtf(q * (1.f / 64.f) + 1e-5f);
                const float4 gg = *reinterpret_cast<const float4*>(g.ln_g + c4 * 4);
                const float4 bb = *reinterpret_cast<const float4*>(g.ln_b + c4 * 4);
                v.x = dx * rs * gg.x + bb.x;
                v.y = dy * rs * gg.y + bb.y;
                v.z = dz * rs * gg.z + bb.z;
                v.w = dw * rs * gg.w + bb.w;
            }
            As[(c4 * 4 + 0) * (BM + APAD) + r] = v.x;
            As[(c4 * 4 + 1) * (BM + APAD) + r] = v.y;
            As[(c4 * 4 + 2) * (BM + APAD) + r] = v.z;
            As[(c4 * 4 + 3) * (BM + APAD) + r] = v.w;
        }
        // ---- B tile: Wt[k0 .. k0+63][n0 .. n0+BN) -----------------------------------------
        for (int i = tid; i < GK * (BN / 4); i += NT) {
            const int kk = i / (BN / 4), c4 = i % (BN / 4);
            *reinterpret_cast<float4*>(Bs + kk * BN + c4 * 4) =
                *reinterpret_cast<const float4*>(g.Wt + (int64_t)(k0 + kk) * g.N + n0 + c4 * 4);
        }
        __syncthreads();
#pragma unroll 8
        for (int kk = 0; kk < GK; ++kk) {
            float a[TM];
            float2 b[TN / 2];
            if constexpr (TM % 4 == 0) {
#pragma unroll
                for (int i = 0; i < TM; i += 4) {
                    const float4 t = *reinterpret_cast<const float4*>(As + kk * (BM + APAD) + ty * TM + i);
                    a[i] = t.x; a[i + 1] = t.y; a[i + 2] = t.z; a[i + 3] = t.w;
                }
            } else {
#pragma unroll
                for (int i = 0; i < TM; i += 2) {
                    const float2 t = *reinterpret_cast<const float2*>(As + kk * (BM + APAD) + ty * TM + i);
                    a[i] = t.x; a[i + 1] = t.y;
                }
            }
#pragma unroll
            for (int j = 0; j < TN; j += 4) {
                const float4 t = *reinterpret_cast<const float4*>(Bs + kk * BN + tx * TN + j);
                b[j / 2] = make_float2(t.x, t.y);
                b[j / 2 + 1] = make_float2(t.z, t.w);
            }
#pragma unroll
            for (int i = 0; i < TM; ++i) {
                const float2 aa = make_float2(a[i], a[i]);
#pragma unroll
                for (int j = 0; j < TN / 2; ++j) acc[i][j] = ffma2(aa, b[j], acc[i][j]);
            }
        }
        __syncthreads();
    }

    // ---- epilogue -----------------------------------------------------------------------
    const float slope = g.prelu ? __ldg(g.prelu) : 0.f;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int m = m0 + ty * TM + i;
        if (m >= g.M) continue;
        int64_t coff;
        if (g.c_rows_per_seq > 0) {
            const int seq = m / g.c_rows_per_seq, p = m % g.c_rows_per_seq;
            if (g.c_inner > 1)
                coff = (int64_t)(seq / g.c_inner) * g.c_seq_stride + (int64_t)(seq % g.c_inner) * g.c_inner_stride +
                       (int64_t)p * g.ldc;
            else
                coff = (int64_t)seq * g.c_seq_stride + (int64_t)p * g.ldc;
        } else {
            coff = (int64_t)m * g.ldc;
        }
#pragma unroll
        for (int j = 0; j < TN; j += 4) {
            const int n = n0 + tx * TN + j;
            float4 o = make_float4(acc[i][j / 2].x, acc[i][j / 2].y, acc[i][j / 2 + 1].x, acc[i][j / 2 + 1].y);
            if (g.bias) {
                const float4 bb = *reinterpret_cast<const float4*>(g.bias + n);
                o.x += bb.x; o.y += bb.y; o.z += bb.z; o.w += bb.w;
            }
            if (g.prelu) {
                o.x = prelu(o.x, slope); o.y = prelu(o.y, slope);
                o.z = prelu(o.z, slope); o.w = prelu(o.w, slope);
            }
            if (g.prelu_vec) {
                const float4 sv = *reinterpret_cast<const float4*>(g.prelu_vec + n);
                o.x = prelu(o.x, sv.x); o.y = prelu(o.y, sv.y);
                o.z = prelu(o.z, sv.z); o.w = prelu(o.w, sv.w);
            }
            if (g.R) {
                const float4 rr = *reinterpret_cast<const float4*>(g.R + coff + n);
                o.x += rr.x; o.y += rr.y; o.z += rr.z; o.w += rr.w;
            }
            *reinterpret_cast<float4*>(g.C + coff + n) = o;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Large-M variant.  Persistent CTAs keep the whole k-major weight slab W^T[K][BN] resident in shared
// memory and stream 128-row tiles of A through it in 64-deep k chunks; each thread owns an 8 x TN
// register tile (TN = BN/16), fed by 2 + TN/4 LDS.128 per k for 8*TN/2 FMA pairs -- twice the FMAs per
// shared-memory instruction of the small-tile kernel and no weight re-loads per row tile.
// Same GemmArgs contract (windowed A rows, LN prologue for K == 64, bias / PReLU / residual epilogues).
template <int BN>
__global__ void __launch_bounds__(256)
rows_gemm_big_kernel(const GemmArgs g, int n_row_tiles) {
    constexpr int BM = 128, TN = BN / 16, APAD = 4;
    extern __shared__ __align__(16) float smem[];
    float* Bs = smem;                               // [K][BN]
    float* As = smem + (size_t)g.K * BN;            // [GK][BM + APAD]   one k chunk, k-major
    griddep_launch();
    const int tid = threadIdx.x;
    const int n0 = blockIdx.y * BN;
    const int tx = tid & 15, ty = tid >> 4;
    // weight slab (independent of the chain)
    for (int i = tid; i < g.K * (BN / 4); i += 256) {
        const int kk = i / (BN / 4), c4 = i % (BN / 4);
        *reinterpret_cast<float4*>(Bs + kk * BN + c4 * 4) =
            __ldg(reinterpret_cast<const float4*>(g.Wt + (int64_t)kk * g.N + n0 + c4 * 4));
    }
    griddep_wait();
    const float slope = g.prelu ? __ldg(g.prelu) : 0.f;
    for (int tile = blockIdx.x; tile < n_row_tiles; tile += gridDim.x) {
        const int m0 = tile * BM;
        float2 acc[8][TN / 2];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < TN / 2; ++j) acc[i][j] = make_float2(0.f, 0.f);
        for (int k0 = 0; k0 < g.K; k0 += GK) {
            __syncthreads();                        // previous chunk fully consumed (and Bs written, first time)
            for (int r = tid >> 4; r < BM; r += 16) {
                const int m = m0 + r, c4 = tid & 15;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (m < g.M) {
                    const float* ap;
                    if (g.a_rows_per_seq > 0) {
                        const int seq = m / g.a_rows_per_seq, p = m % g.a_rows_per_seq;
                        ap = g.A + (int64_t)seq * g.a_seq_stride + (int64_t)p * g.lda;
                    } else {
                        ap = g.A + (int64_t)m * g.lda;
                    }
                    v = *reinterpret_cast<const float4*>(ap + k0 + c4 * 4);
                }
                if (g.ln_g != nullptr) {
                    float s = v.x + v.y + v.z + v.w;
#pragma unroll
                    for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
                    const float mu = s * (1.f / 64.f);
                    const float dx = v.x - mu, dy = v.y - mu, dz = v.z - mu, dw = v.w - mu;
                    float q = dx * dx + dy * dy + dz * dz + dw * dw;
#pragma unroll
                    for (int o = 8; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
                    const float rs = rsqrtf(q * (1.f / 64.f) + 1e-5f);
                    const float4 gg = *reinterpret_cast<const float4*>(g.ln_g + c4 * 4);
                    const float4 bb = *reinterpret_cast<const float4*>(g.ln_b + c4 * 4);
                    v.x = dx * rs * gg.x + bb.x; v.y = dy * rs * gg.y + bb.y;
                    v.z = dz * rs * gg.z + bb.z; v.w = dw * rs * gg.w + bb.w;
                }
                As[(c4 * 4 + 0) * (BM + APAD) + r] = v.x;
                As[(c4 * 4 + 1) * (BM + APAD) + r] = v.y;
                As[(c4 * 4 + 2) * (BM + APAD) + r] = v.z;
                As[(c4 * 4 + 3) * (BM + APAD) + r] = v.w;
            }
            __syncthreads();
            const float* bsk = Bs + (size_t)k0 * BN;
#pragma unroll 4
            for (int kk = 0; kk < GK; ++kk) {
                // rows ty*4..+3 and 64+ty*4..+3 ; cols tx*(TN/2)..  and BN/2 + tx*(TN/2).. (conflict-free float4 reads)
                const float4 a0 = *reinterpret_cast<const float4*>(As + kk * (BM + APAD) + ty * 4);
                const float4 a1 = *reinterpret_cast<const float4*>(As + kk * (BM + APAD) + 64 + ty * 4);
                const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                float2 b[TN / 2];
                if constexpr (TN == 8) {
                    const float4 b0 = *reinterpret_cast<const float4*>(bsk + kk * BN + tx * 4);
                    const float4 b1 = *reinterpret_cast<const float4*>(bsk + kk * BN + BN / 2 + tx * 4);
                    b[0] = make_float2(b0.x, b0.y); b[1] = make_float2(b0.z, b0.w);
                    b[2] = make_float2(b1.x, b1.y); b[3] = make_float2(b1.z, b1.w);
                } else {
                    const float2 b0 = *reinterpret_cast<const float2*>(bsk + kk * BN + tx * 2);
                    const float2 b1 = *reinterpret_cast<const float2*>(bsk + kk * BN + BN / 2 + tx * 2);
                    b[0] = b0; b[1] = b1;
                }
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float2 aa = make_float2(av[i], av[i]);
#pragma unroll
                    for (int j = 0; j < TN / 2; ++j) acc[i][j] = ffma2(aa, b[j], acc[i][j]);
                }
            }
        }
        // epilogue: thread's rows m0 + {ty*4+i, 64+ty*4+i}; column groups {tx*(TN/2), BN/2 + tx*(TN/2)}
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
            if (m >= g.M) continue;
            int64_t coff;
            if (g.c_rows_per_seq > 0) {
                const int seq = m / g.c_rows_per_seq, p = m % g.c_rows_per_seq;
                if (g.c_inner > 1)
                    coff = (int64_t)(seq / g.c_inner) * g.c_seq_stride + (int64_t)(seq % g.c_inner) * g.c_inner_stride + (int64_t)p * g.ldc;
                else
                    coff = (int64_t)seq * g.c_seq_stride + (int64_t)p * g.ldc;
            } else {
                coff = (int64_t)m * g.ldc;
            }
#pragma unroll
            for (int hgrp = 0; hgrp < 2; ++hgrp) {
                const int n = n0 + hgrp * (BN / 2) + tx * (TN / 2);
                {   // TN == 8: one float4 (2 float2) per half; TN == 4: one float2 per half
                    if constexpr (TN == 8) {
                        float4 o = make_float4(acc[i][hgrp * 2].x, acc[i][hgrp * 2].y, acc[i][hgrp * 2 + 1].x, acc[i][hgrp * 2 + 1].y);
                        if (g.bias) { const float4 bb = *reinterpret_cast<const float4*>(g.bias + n); o.x += bb.x; o.y += bb.y; o.z += bb.z; o.w += bb.w; }
                        if (g.prelu) { o.x = prelu(o.x, slope); o.y = prelu(o.y, slope); o.z = prelu(o.z, slope); o.w = prelu(o.w, slope); }
                        if (g.prelu_vec) { const float4 sv = *reinterpret_cast<const float4*>(g.prelu_vec + n); o.x = prelu(o.x, sv.x); o.y = prelu(o.y, sv.y); o.z = prelu(o.z, sv.z); o.w = prelu(o.w, sv.w); }
                        if (g.R) { const float4 rr = *reinterpret_cast<const float4*>(g.R + coff + n); o.x += rr.x; o.y += rr.y; o.z += rr.z; o.w += rr.w; }
                        *reinterpret_cast<float4*>(g.C + coff + n) = o;
                    } else {
                        float2 o = acc[i][hgrp];
                        if (g.bias) { const float2 bb = *reinterpret_cast<const float2*>(g.bias + n); o.x += bb.x; o.y += bb.y; }
                        if (g.prelu) { o.x = prelu(o.x, slope); o.y = prelu(o.y, slope); }
                        if (g.prelu_vec) { const float2 sv = *reinterpret_cast<const float2*>(g.prelu_vec + n); o.x = prelu(o.x, sv.x); o.y = prelu(o.y, sv.y); }
                        if (g.R) { const float2 rr = *reinterpret_cast<const float2*>(g.R + coff + n); o.x += rr.x; o.y += rr.y; }
                        *reinterpret_cast<float2*>(g.C + coff + n) = o;
                    }
                }
            }
        }
    }
}

template <int BN>
inline cudaError_t launch_rows_gemm_big(const GemmArgs& g, cudaStream_t st, bool pdl) {
    const size_t smem = ((size_t)g.K * BN + (size_t)GK * (128 + 4)) * sizeof(float);
    const int n_row_tiles = (g.M + 127) / 128;
    const int col_tiles = g.N / BN;
    // resident CTAs per SM: the 128-column variant holds 105 registers x 256 threads -> two; the 64-column variant
    // three (as far as shared memory allows).  The grid must not exceed what is resident (a second wave of a
    // persistent kernel doubles its time), and the row tiles are dealt out
    // evenly: every CTA takes ceil(tiles / gx_max) of them.
    const int by_smem = (smem <= 72 * 1024) ? 3 : (smem <= 110 * 1024 ? 2 : 1);
    const int per_sm = std::min(by_smem, BN == 128 ? 2 : 3);
    int gx = std::max(1, (NUM_SMS * per_sm) / col_tiles);
    if (gx > n_row_tiles) gx = n_row_tiles;
    const int per_cta = (n_row_tiles + gx - 1) / gx;
    gx = (n_row_tiles + per_cta - 1) / per_cta;
    return launch_k(pdl, rows_gemm_big_kernel<BN>, dim3(gx, col_tiles), dim3(256), smem, st, g, n_row_tiles);
}

template <int BM, int BN, int TM, int TN>
inline cudaError_t configure_rows_gemm_cfg() {
    const size_t smem = (size_t)(GK * (BM + 4) + GK * BN) * sizeof(float);
    return cudaFuncSetAttribute(rows_gemm_kernel<BM, BN, TM, TN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)smem);
}

// call once per process before the first launch (and outside stream capture)
inline cudaError_t configure_rows_gemm() {
    cudaError_t e = configure_rows_gemm_cfg<16, 64, 2, 4>();
    if (e == cudaSuccess) e = configure_rows_gemm_cfg<64, 128, 4, 8>();
    if (e == cudaSuccess) e = configure_rows_gemm_cfg<64, 64, 4, 4>();
    if (e == cudaSuccess) e = cudaFuncSetAttribute(rows_gemm_big_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(rows_gemm_big_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    return e;
}

template <int BM, int BN, int TM, int TN>
inline cudaError_t launch_rows_gemm_cfg(const GemmArgs& g, cudaStream_t st, bool pdl) {
    constexpr int NT = (BM / TM) * (BN / TN);
    const size_t smem = (size_t)(GK * (BM + 4) + GK * BN) * sizeof(float);
    dim3 grid((g.M + BM - 1) / BM, g.N / BN);
    return launch_k(pdl, rows_gemm_kernel<BM, BN, TM, TN>, grid, dim3(NT), smem, st, g);
}

// The kernel launch_rows_gemm runs for a problem (none: the problem is refused).
enum class RowsGemmForm { none, tile16x64, tile64x64, tile64x128, big64, big128 };

// Pick a tile by problem size: small M (one streaming frame = 97 rows) wants many small CTAs,
// large M wants the 64x128 tile.  N must be a multiple of 64; K a multiple of 64.
// `shape`: 0 = by size (below); 1 = 64x64 tiles, 2 = the persistent 128-row form, whatever M is (the pipelined graph's 4-hop
// batches of 388 rows: fewer, fatter CTAs compete less with the other stages' kernels)
inline RowsGemmForm rows_gemm_form(const GemmArgs& g, int shape) {
    if (g.N % 64 != 0 || g.K % 64 != 0 || g.M <= 0) return RowsGemmForm::none;
    if (g.ln_g && g.K != 64) return RowsGemmForm::none;
    if (shape == 1) return RowsGemmForm::tile64x64;
    if (g.M <= 2048 && shape == 0) return RowsGemmForm::tile16x64;
    {   // large M: persistent kernel with the weight slab resident in shared memory (when it fits)
        const int bn = (g.N % 128 == 0) ? 128 : 64;
        const size_t smem = ((size_t)g.K * bn + (size_t)GK * 132) * sizeof(float);
        if (smem <= 200 * 1024) return bn == 128 ? RowsGemmForm::big128 : RowsGemmForm::big64;
    }
    return g.N % 128 == 0 ? RowsGemmForm::tile64x128 : RowsGemmForm::tile64x64;
}

inline cudaError_t launch_rows_gemm(const GemmArgs& g, cudaStream_t st, bool pdl = false, int shape = 0) {
    switch (rows_gemm_form(g, shape)) {
        case RowsGemmForm::tile16x64: return launch_rows_gemm_cfg<16, 64, 2, 4>(g, st, pdl);      // 128 threads
        case RowsGemmForm::tile64x64: return launch_rows_gemm_cfg<64, 64, 4, 4>(g, st, pdl);      // 256 threads
        case RowsGemmForm::tile64x128: return launch_rows_gemm_cfg<64, 128, 4, 8>(g, st, pdl);    // 256 threads
        case RowsGemmForm::big64: return launch_rows_gemm_big<64>(g, st, pdl);
        case RowsGemmForm::big128: return launch_rows_gemm_big<128>(g, st, pdl);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace l2h
