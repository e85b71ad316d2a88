// mid_kernel: for one-frame calls (T == 1) everything between the intra BiLSTM and the attention
// is ROW-LOCAL (one row = one frequency bin of one stream):
//     X1 = X + Y W_l1^T + b                      intra Linear(128->64) + residual   (tfgridnet_causal.py:513-516)
//     g  = W_ih LN(X1) + W_hh h + b ; (h,c) cell   inter LSTM, one step, carried state   (:521-532)
//     X2 = X1 + h' W_l2^T + b                     inter Linear(64->64) + residual      (:534-538)
//     P  = PReLU(X2 W_qkv^T + b)                  the three attention projections      (:547-551, :354-387)
// The generic chain runs this as four row-GEMMs + one recurrence launch + the GEMM half of
// qkv_kernel.  Here one CTA keeps all the weight matrices (205 KB, one packed buffer) in shared memory --
// loaded BEFORE griddepcontrol.wait, i.e. while the 97-step intra recurrence is still running -- and
// pushes tiles of 8 rows through the whole section.  Persistent: grid = min(#tiles, #SMs) CTAs, each
// loading the weights ONCE and looping over (stream, row-tile) items.
//
// Tiling (v2).  With only 8 rows per tile the activations are the broadcast operand, and a broadcast
// LDS costs one shared-memory wavefront per 4 B per lane whatever its width,
// so a warp computing R rows x C columns per lane gets 32 R C / (R + C) FMAs per wavefront: v1 (C = 1,
// R = 2 or 8) was bound by the shared-memory pipe.  v2 splits K across KQ adjacent lanes instead of giving every lane its own
// column: a lane accumulates 8 rows x C = 4 or 8 columns over K/KQ values of k, the KQ partial tiles are
// summed by a shuffle reduce-scatter, and every lane ends up owning 8 C / KQ finished outputs for the
// epilogue.  Weights and activations are stored in k-slices padded by 4 floats so that the 8 lanes of a
// quarter-warp (one LDS.128 phase) hit 32 distinct banks.
#pragma once
#include <algorithm>
#include "common.cuh"
#include "sep_kernels.cuh"

namespace l2h {

constexpr int MID_RT = 8;
// phase geometry: K, N, C (columns per lane), KQ (k-slices = lanes per column group), KS = K / KQ
constexpr int M1_K = 128, M1_N = 64, M1_C = 4, M1_KQ = 16, M1_KS = 8;        // intra linear
constexpr int M3_K = 64, M3_N = 256, M3_C = 8, M3_KQ = 8, M3_KS = 8;         // LN(X1) x W_ih and h x W_hh (two products)
constexpr int M5_K = 64, M5_N = 64, M5_C = 4, M5_KQ = 16, M5_KS = 4;         // inter linear
constexpr int M6_K = 64, M6_N = NQKV, M6_C = 4, M6_KQ = 8, M6_KS = 8;        // q|k|v projections
__host__ __device__ constexpr int mid_wslice(int ks, int n) { return ks * n + 4; }
__host__ __device__ constexpr int mid_aslice(int ks) { return ks * MID_RT + 4; }
// BlockWeights::mid_pack: the five matrices k-sliced, in the order the split kernels need them contiguous
constexpr int MID_W1 = 0;
constexpr int MID_W3A = MID_W1 + M1_KQ * mid_wslice(M1_KS, M1_N);            // W_ih
constexpr int MID_W3B = MID_W3A + M3_KQ * mid_wslice(M3_KS, M3_N);           // W_hh
constexpr int MID_W5 = MID_W3B + M3_KQ * mid_wslice(M3_KS, M3_N);
constexpr int MID_W6 = MID_W5 + M5_KQ * mid_wslice(M5_KS, M5_N);
constexpr int MID_PACK = MID_W6 + M6_KQ * mid_wslice(M6_KS, M6_N);           // floats in BlockWeights::mid_pack
constexpr int MID_A1 = M1_KQ * mid_aslice(M1_KS), MID_A3 = M3_KQ * mid_aslice(M3_KS);
constexpr int MID_A5 = M5_KQ * mid_aslice(M5_KS), MID_A6 = M6_KQ * mid_aslice(M6_KS);
constexpr size_t MID_SMEM = (size_t)(MID_PACK + MID_A1 + 2 * MID_A3 + MID_A5 + MID_A6 + MID_RT * 64) * sizeof(float);
constexpr size_t MID_A_SMEM = (size_t)((MID_W3B - MID_W1) + MID_A1 + MID_A3 + MID_RT * 64) * sizeof(float);
constexpr size_t MID_B_SMEM = (size_t)((MID_W5 - MID_W3B) + MID_A3) * sizeof(float);
constexpr size_t MID_C_SMEM = (size_t)((MID_PACK - MID_W5) + MID_A5 + MID_A6) * sizeof(float);
static_assert(MID_SMEM <= 227 * 1024, "mid_kernel shared memory");
static_assert((MID_W3A % 4) == 0 && (MID_W3B % 4) == 0 && (MID_W5 % 4) == 0 && (MID_W6 % 4) == 0 && (MID_PACK % 4) == 0, "16-byte slices");

// index of activation (k, row r) in a k-sliced tile
__host__ __device__ constexpr int mid_aidx(int ks, int k, int r) { return (k / ks) * (ks * MID_RT + 4) + (k % ks) * MID_RT + r; }
// index of weight (k, n) in a k-sliced [K][N] matrix
__host__ __device__ constexpr int mid_widx(int ks, int n_cols, int k, int n) { return (k / ks) * (ks * n_cols + 4) + (k % ks) * n_cols + n; }

// host: BlockWeights::mid_pack (MID_PACK floats, padding zeroed) from the five matrices as the engine stores them, W^T
// [K][N]: wl1_t [128][64], wih2_t and whh2_t [64][256] (gate column j*4 + q), wl2_t [64][64], wqkv_t [64][NQKV]
inline void mid_pack_weights(const float* wl1_t, const float* wih2_t, const float* whh2_t, const float* wl2_t, const float* wqkv_t,
                             float* dst) {
    std::fill(dst, dst + MID_PACK, 0.f);
    for (int k = 0; k < M1_K; ++k)
        for (int n = 0; n < M1_N; ++n) dst[MID_W1 + mid_widx(M1_KS, M1_N, k, n)] = wl1_t[(int64_t)k * 64 + n];
    for (int k = 0; k < M3_K; ++k)
        for (int n = 0; n < M3_N; ++n) {
            dst[MID_W3A + mid_widx(M3_KS, M3_N, k, n)] = wih2_t[(int64_t)k * 256 + n];
            dst[MID_W3B + mid_widx(M3_KS, M3_N, k, n)] = whh2_t[(int64_t)k * 256 + n];
        }
    for (int k = 0; k < M5_K; ++k)
        for (int n = 0; n < M5_N; ++n) dst[MID_W5 + mid_widx(M5_KS, M5_N, k, n)] = wl2_t[(int64_t)k * 64 + n];
    for (int k = 0; k < M6_K; ++k)
        for (int n = 0; n < M6_N; ++n) dst[MID_W6 + mid_widx(M6_KS, M6_N, k, n)] = wqkv_t[(int64_t)k * NQKV + n];
}

// sum v[] over the KQ adjacent lanes of a group; lane kq keeps the kq-th chunk of NV / KQ values in v[0 ..)
template <int HALF, int BIT, int NV>
__device__ __forceinline__ void lane_rs_stage(float (&v)[NV], int kq) {
    if constexpr (BIT >= 1) {
        const bool upper = (kq & BIT) != 0;
#pragma unroll
        for (int i = 0; i < HALF; ++i) {
            const float send = upper ? v[i] : v[i + HALF];
            const float keep = upper ? v[i + HALF] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, BIT);
        }
        lane_rs_stage<HALF / 2, BIT / 2, NV>(v, kq);
    }
}
template <int NV, int KQ>
__device__ __forceinline__ void lane_reduce_scatter(float (&v)[NV], int kq) {
    lane_rs_stage<NV / 2, KQ / 2, NV>(v, kq);
}

// partial products of one lane: 8 rows x C columns over its k-slice, then the group reduce-scatter.
// Values are ordered row-major (v = r * C + c), so lane kq ends with rows/columns [kq * 8C/KQ, ...).
template <int C, int KQ, int KS, int N>
__device__ __forceinline__ void mid_mm(const float* __restrict__ Wp, const float* __restrict__ Ap, int cg, int kq,
                                       float (&v)[MID_RT * C]) {
    float2 acc[C][4];
#pragma unroll
    for (int c = 0; c < C; ++c)
#pragma unroll
        for (int p = 0; p < 4; ++p) acc[c][p] = make_float2(0.f, 0.f);
    const float* wp = Wp + kq * mid_wslice(KS, N) + cg * C;
    const float* ap = Ap + kq * mid_aslice(KS);
#pragma unroll
    for (int kk = 0; kk < KS; ++kk) {
        const float4 a0 = *reinterpret_cast<const float4*>(ap + kk * MID_RT);
        const float4 a1 = *reinterpret_cast<const float4*>(ap + kk * MID_RT + 4);
        const float2 ar[4] = {make_float2(a0.x, a0.y), make_float2(a0.z, a0.w), make_float2(a1.x, a1.y), make_float2(a1.z, a1.w)};
        float wv[C];
#pragma unroll
        for (int c4 = 0; c4 < C / 4; ++c4) {
            const float4 t = *reinterpret_cast<const float4*>(wp + kk * N + c4 * 4);
            wv[c4 * 4] = t.x; wv[c4 * 4 + 1] = t.y; wv[c4 * 4 + 2] = t.z; wv[c4 * 4 + 3] = t.w;
        }
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const float2 ww = make_float2(wv[c], wv[c]);
#pragma unroll
            for (int p = 0; p < 4; ++p) acc[c][p] = ffma2(ww, ar[p], acc[c][p]);
        }
    }
#pragma unroll
    for (int r = 0; r < MID_RT; ++r)
#pragma unroll
        for (int c = 0; c < C; ++c) v[r * C + c] = (r & 1) ? acc[c][r >> 1].y : acc[c][r >> 1].x;
    lane_reduce_scatter<MID_RT * C, KQ>(v, kq);
}

// Shared-memory tiles of one mid section (carved from the dynamic shared memory after the packed weights)
struct MidSmem {
    float *Wp, *A1, *A3, *A3h, *A5, *A6, *x1s;
    __device__ __forceinline__ explicit MidSmem(float* sm)
        : Wp(sm), A1(sm + MID_PACK), A3(A1 + MID_A1), A3h(A3 + MID_A3), A5(A3h + MID_A3), A6(A5 + MID_A5), x1s(A6 + MID_A6) {}
};

// The section's small parameter vectors, staged in shared memory before the dependency wait: every one of them would
// otherwise be a first-touch global load in the middle of the tile's latency chain (6 exposed L2 round trips per tile).
constexpr int MV_BL1 = 0, MV_LN2G = 64, MV_LN2B = 128, MV_B2 = 192, MV_BL2 = 448, MV_BQKV = 512, MV_SLOPES = 624, MV_TOTAL = 628;
__device__ __forceinline__ void mid_stage_vecs(float* vs, const BlockWeights& w, int tid) {
    for (int i = tid; i < MV_TOTAL; i += 256) {
        const float* src = i < MV_LN2G ? w.bl1 + i : i < MV_LN2B ? w.ln2_g + (i - MV_LN2G) : i < MV_B2 ? w.ln2_b + (i - MV_LN2B)
                         : i < MV_BL2 ? w.b2 + (i - MV_B2) : i < MV_BQKV ? w.bl2 + (i - MV_BL2) : i < MV_SLOPES ? w.bqkv + (i - MV_BQKV)
                         : w.slopes + (i - MV_SLOPES);
        vs[i] = __ldg(src);
    }
}

// One tile of MID_RT rows through the whole section.  Yrows/Xin: the tile's rows of the BiLSTM output / the block input
// (global); X2out / Pout: where the tile's rows of X2 (row stride 64) and of the projections (row stride NQKV) go --
// global for mid_kernel, the caller's shared memory for tail_kernel (hop_kernels.cuh); Xin may alias X2out.
// hst/cst: the stream's carried (h, c) of this block, [97][64].  vs: the vectors staged by mid_stage_vecs (visible to all
// threads after the first barrier in here).  The caller has waited for the weights.
// The carried-state half of the inter-LSTM step of a tile, h_prev W_hh (lane (jp, kq = row) keeps gates of hidden units 2jp, 2jp+1 of
// row kq: hv[0..7]) and the tile's old cell state.  It reads only what the PREVIOUS hop left, so tail_kernel runs it before the
// dependency wait, under the recurrence that is still going.  Needs W_hh (MID_W3B) in shared memory; ends with a barrier pending
// (the caller's next barrier separates it from the next writer of A3h).
__device__ __forceinline__ void mid_h_product(const MidSmem& S, const float* hst, const float* cst, int r0, int nr, int tid,
                                              float (&hv)[8], float2& cold) {
    if (tid < 128) {
        const int r = tid >> 4, k4 = tid & 15;
        const float4 v = (r < nr) ? *reinterpret_cast<const float4*>(hst + (r0 + r) * 64 + k4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        S.A3h[mid_aidx(M3_KS, k4 * 4 + 0, r)] = v.x; S.A3h[mid_aidx(M3_KS, k4 * 4 + 1, r)] = v.y;
        S.A3h[mid_aidx(M3_KS, k4 * 4 + 2, r)] = v.z; S.A3h[mid_aidx(M3_KS, k4 * 4 + 3, r)] = v.w;
    }
    cold = ((tid & 7) < nr) ? *reinterpret_cast<const float2*>(cst + (r0 + (tid & 7)) * 64 + (tid >> 3) * 2) : make_float2(0.f, 0.f);
    __syncthreads();
    float v[MID_RT * M3_C];
    mid_mm<M3_C, M3_KQ, M3_KS, M3_N>(S.Wp + MID_W3B, S.A3h, tid >> 3, tid & 7, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) hv[i] = v[i];
}

// PRE_H: the h W_hh product and the old cell state come from mid_h_product (hv_in, cold_in) instead of being computed here.
// store_hc = false: the new (h, c) are computed but not written back (a stream that skips this hop).
template <bool PRE_H = false>
__device__ __forceinline__ void mid_tile(const MidSmem& S, const float* Yrows, const float* Xin, float* X2out, float* Pout,
                                         float* hst, float* cst, int r0, int nr, const float* vs, int tid, bool store_hc,
                                         const float* hv_in = nullptr, float2 cold_in = make_float2(0.f, 0.f)) {
    float* Wp = S.Wp; float* A1 = S.A1; float* A3 = S.A3; float* A3h = S.A3h; float* A5 = S.A5; float* A6 = S.A6; float* x1s = S.x1s;
    // ---- tile loads: Y -> A1, h -> A3h ------------------------------------------------------------
    {
        const int r = tid >> 5, k4 = tid & 31;
        const float4 v = (r < nr) ? *reinterpret_cast<const float4*>(Yrows + (int64_t)r * 128 + k4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        A1[mid_aidx(M1_KS, k4 * 4 + 0, r)] = v.x; A1[mid_aidx(M1_KS, k4 * 4 + 1, r)] = v.y;
        A1[mid_aidx(M1_KS, k4 * 4 + 2, r)] = v.z; A1[mid_aidx(M1_KS, k4 * 4 + 3, r)] = v.w;
    }
    if (!PRE_H && tid < 128) {
        const int r = tid >> 4, k4 = tid & 15;
        const float4 v = (r < nr) ? *reinterpret_cast<const float4*>(hst + (r0 + r) * 64 + k4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        A3h[mid_aidx(M3_KS, k4 * 4 + 0, r)] = v.x; A3h[mid_aidx(M3_KS, k4 * 4 + 1, r)] = v.y;
        A3h[mid_aidx(M3_KS, k4 * 4 + 2, r)] = v.z; A3h[mid_aidx(M3_KS, k4 * 4 + 3, r)] = v.w;
    }
    // the two other chain inputs of this thread, requested now: the residual of phase 1 and the cell state of phase 4
    const int r1 = (tid & 15) >> 1, n1 = (tid >> 4) * 4 + (tid & 1) * 2;
    const float2 xo = (r1 < nr) ? *reinterpret_cast<const float2*>(Xin + (int64_t)r1 * 64 + n1) : make_float2(0.f, 0.f);
    float2 cold = cold_in;
    if (!PRE_H) cold = ((tid & 7) < nr) ? *reinterpret_cast<const float2*>(cst + (r0 + (tid & 7)) * 64 + (tid >> 3) * 2) : make_float2(0.f, 0.f);
    __syncthreads();
    // ---- phase 1: X1 = X + Y W1 + b ;  lane (cg, kq) finishes row kq/2, columns cg*4 + (kq&1)*2 + {0,1}
    float2 x1v;
    {
        float v[MID_RT * M1_C];
        mid_mm<M1_C, M1_KQ, M1_KS, M1_N>(Wp + MID_W1, A1, tid >> 4, tid & 15, v);
        const float2 bias = *reinterpret_cast<const float2*>(vs + MV_BL1 + n1);
        x1v = make_float2(xo.x + v[0] + bias.x, xo.y + v[1] + bias.y);
        *reinterpret_cast<float2*>(x1s + r1 * 64 + n1) = x1v;
    }
    __syncthreads();
    // ---- phase 2: LayerNorm over channels, one warp per row -> A3 ------------------------------------
    {
        const int r = tid >> 5, lane = tid & 31;
        const float v0 = x1s[r * 64 + lane], v1 = x1s[r * 64 + lane + 32];
        const float mu = warp_sum(v0 + v1) * (1.f / 64.f);
        const float d0 = v0 - mu, d1 = v1 - mu;
        const float rs = rsqrtf(warp_sum(d0 * d0 + d1 * d1) * (1.f / 64.f) + 1e-5f);
        A3[mid_aidx(M3_KS, lane, r)] = d0 * rs * vs[MV_LN2G + lane] + vs[MV_LN2B + lane];
        A3[mid_aidx(M3_KS, lane + 32, r)] = d1 * rs * vs[MV_LN2G + lane + 32] + vs[MV_LN2B + lane + 32];
    }
    __syncthreads();
    // ---- phase 3 + 4: gates and LSTM cell; lane (jp, kq) finishes row kq, hidden units 2jp, 2jp+1 ----
    {
        // two K = 64 products, combined as (x W_ih + b) + h W_hh: the arithmetic of mid_a_kernel + mid_b_kernel
        float u[MID_RT * M3_C], v[MID_RT * M3_C];
        const int jp = tid >> 3, r = tid & 7;
        mid_mm<M3_C, M3_KQ, M3_KS, M3_N>(Wp + MID_W3A, A3, jp, r, u);
        if (PRE_H) {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = hv_in[i];
        } else {
            mid_mm<M3_C, M3_KQ, M3_KS, M3_N>(Wp + MID_W3B, A3h, jp, r, v);
        }
        const float4 ba = *reinterpret_cast<const float4*>(vs + MV_B2 + jp * 8);
        const float4 bb = *reinterpret_cast<const float4*>(vs + MV_B2 + jp * 8 + 4);
        const float4 ga = make_float4(u[0] + ba.x, u[1] + ba.y, u[2] + ba.z, u[3] + ba.w);
        const float4 gb = make_float4(u[4] + bb.x, u[5] + bb.y, u[6] + bb.z, u[7] + bb.w);
        const float gi0 = fast_sigmoid(v[0] + ga.x), gf0 = fast_sigmoid(v[1] + ga.y), gg0 = fast_tanh(v[2] + ga.z), go0 = fast_sigmoid(v[3] + ga.w);
        const float gi1 = fast_sigmoid(v[4] + gb.x), gf1 = fast_sigmoid(v[5] + gb.y), gg1 = fast_tanh(v[6] + gb.z), go1 = fast_sigmoid(v[7] + gb.w);
        const float c0 = gf0 * cold.x + gi0 * gg0, c1 = gf1 * cold.y + gi1 * gg1;
        const float h0 = go0 * fast_tanh(c0), h1 = go1 * fast_tanh(c1);
        if (store_hc && r < nr) {
            *reinterpret_cast<float2*>(cst + (r0 + r) * 64 + jp * 2) = make_float2(c0, c1);
            *reinterpret_cast<float2*>(hst + (r0 + r) * 64 + jp * 2) = make_float2(h0, h1);
        }
        A5[mid_aidx(M5_KS, jp * 2, r)] = h0;
        A5[mid_aidx(M5_KS, jp * 2 + 1, r)] = h1;
    }
    __syncthreads();
    // ---- phase 5: X2 = X1 + h' W_l2 + b ; same lane -> output mapping as phase 1 -------------------
    {
        float v[MID_RT * M5_C];
        mid_mm<M5_C, M5_KQ, M5_KS, M5_N>(Wp + MID_W5, A5, tid >> 4, tid & 15, v);
        const float2 bias = *reinterpret_cast<const float2*>(vs + MV_BL2 + n1);
        const float2 x2v = make_float2(x1v.x + v[0] + bias.x, x1v.y + v[1] + bias.y);
        if (r1 < nr) *reinterpret_cast<float2*>(X2out + (int64_t)r1 * 64 + n1) = x2v;
        A6[mid_aidx(M6_KS, n1, r1)] = x2v.x;
        A6[mid_aidx(M6_KS, n1 + 1, r1)] = x2v.y;
    }
    __syncthreads();
    // ---- phase 6: P = PReLU(X2 W_qkv + b); lane (cg < 28, kq) finishes row kq, columns cg*4 .. +3 ----
    if (tid < (M6_N / M6_C) * M6_KQ) {
        float v[MID_RT * M6_C];
        const int cg = tid >> 3, r = tid & 7;
        mid_mm<M6_C, M6_KQ, M6_KS, M6_N>(Wp + MID_W6, A6, cg, r, v);
        const float4 bias = *reinterpret_cast<const float4*>(vs + MV_BQKV + cg * 4);
        const float slope = vs[MV_SLOPES + (cg < 6 ? 0 : (cg < 12 ? 1 : 2))];
        if (r < nr)
            *reinterpret_cast<float4*>(Pout + (int64_t)r * NQKV + cg * 4) =
                make_float4(prelu(v[0] + bias.x, slope), prelu(v[1] + bias.y, slope), prelu(v[2] + bias.z, slope),
                            prelu(v[3] + bias.w, slope));
    }
}

template <class Map>
__global__ void __launch_bounds__(256)
mid_kernel_t(const float* __restrict__ Y, float* X, float* __restrict__ QKV, float* __restrict__ state,
             Map recs, int blk, BlockWeights w, int n_streams, const uint8_t* __restrict__ active) {
    extern __shared__ __align__(16) float sm[];
    const MidSmem S(sm);
    __shared__ __align__(8) unsigned long long wbar;
    __shared__ __align__(16) float vs[MV_TOTAL];
    TraceScope trace_(TK_MID, Y);
    griddep_launch();
    const int tid = threadIdx.x;
    constexpr int TILES = (NF + MID_RT - 1) / MID_RT;       // row tiles per stream
    mid_stage_vecs(vs, w, tid);
    // ---- weights -> smem: TMA bulk copies (independent of the chain, so issued before the wait) ------
    if (tid == 0) {
        mbar_init(&wbar, 1);
        mbar_fence_init();
        mbar_expect_tx(&wbar, MID_PACK * 4);
        tma_load_1d(S.Wp + MID_W1, w.mid_pack + MID_W1, (MID_W3B - MID_W1) * 4, &wbar);
        tma_load_1d(S.Wp + MID_W3B, w.mid_pack + MID_W3B, (MID_W5 - MID_W3B) * 4, &wbar);
        tma_load_1d(S.Wp + MID_W5, w.mid_pack + MID_W5, (MID_PACK - MID_W5) * 4, &wbar);
    }
    __syncthreads();
    griddep_wait();
    mbar_wait(&wbar, 0);
    for (int item = blockIdx.x; item < n_streams * TILES; item += gridDim.x) {
        const int b = item / TILES;
        const int r0 = (item % TILES) * MID_RT;
        const int nr = min(MID_RT, NF - r0);
        __syncthreads();                    // the previous item's tiles are fully consumed
        float* sb = stream_rec(state, recs, b) + ST_BLK + (int64_t)blk * BK_STRIDE;
        const int64_t row0 = (int64_t)b * NF + r0;
        mid_tile(S, Y + row0 * 128, X + row0 * 64, X + row0 * 64, QKV + row0 * NQKV, sb + BK_H, sb + BK_C, r0, nr, vs, tid,
                 stream_active(recs, active, b));
    }
}

// ---- the same section as three kernels (wavefront-pipelined one-hop streams, sep_engine.cu) ----------
// Only the W_hh product and the cell carry state from hop to hop; in the pipeline that part is the stage every
// hop of a block has to pass through one after the other, so it is kept as small as possible:
//   mid_a  X1 = X + Y W_l1 + b ; GI = LN(X1) W_ih + b        no carried state: runs on the BiLSTM lanes
//   mid_b  g = GI + h W_hh ; (h, c) cell ; H' = h'            the serial stage: 64 KB of weights, K = 64
//   mid_c  X2 = X1 + H' W_l2 + b ; P = PReLU(X2 W_qkv + b)   no carried state: runs on the qkv lanes
__global__ void __launch_bounds__(256)
mid_a_kernel(const float* __restrict__ Y, float* __restrict__ X, float* __restrict__ GI, BlockWeights w, int n_streams,
             int64_t hop_stride, int n_hops) {      // n_hops hops per launch: the buffers of hop j sit j * hop_stride floats further
    extern __shared__ __align__(16) float sm[];
    float* W1 = sm;                                   // intra linear, k-sliced
    float* W3a = W1 + (MID_W3A - MID_W1);             // W_ih, k-sliced
    float* A1 = W1 + (MID_W3B - MID_W1);
    float* A3 = A1 + MID_A1;                          // LN(X1), k-sliced
    float* x1s = A3 + MID_A3;
    __shared__ __align__(8) unsigned long long wbar;
    TraceScope trace_(TK_MID_A, Y);
    griddep_launch();
    const int tid = threadIdx.x;
    constexpr int TILES = (NF + MID_RT - 1) / MID_RT;
    if (tid == 0) {
        mbar_init(&wbar, 1);
        mbar_fence_init();
        mbar_expect_tx(&wbar, (MID_W3B - MID_W1) * 4);
        tma_load_1d(W1, w.mid_pack + MID_W1, (MID_W3B - MID_W1) * 4, &wbar);
    }
    __syncthreads();
    griddep_wait();
    const float* Y0 = Y; float* X0 = X; float* GI0 = GI;
    for (int item = blockIdx.x; item < n_hops * n_streams * TILES; item += gridDim.x) {
        const int hop = item / (n_streams * TILES), it_h = item % (n_streams * TILES);
        Y = Y0 + (int64_t)hop * hop_stride; X = X0 + (int64_t)hop * hop_stride; GI = GI0 + (int64_t)hop * hop_stride;
        const int b = it_h / TILES;
        const int r0 = (it_h % TILES) * MID_RT;
        const int nr = min(MID_RT, NF - r0);
        __syncthreads();
        const int64_t row0 = (int64_t)b * NF + r0;
        {
            const int r = tid >> 5, k4 = tid & 31;
            const float4 v = (r < nr) ? *reinterpret_cast<const float4*>(Y + (row0 + r) * 128 + k4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
            A1[mid_aidx(M1_KS, k4 * 4 + 0, r)] = v.x; A1[mid_aidx(M1_KS, k4 * 4 + 1, r)] = v.y;
            A1[mid_aidx(M1_KS, k4 * 4 + 2, r)] = v.z; A1[mid_aidx(M1_KS, k4 * 4 + 3, r)] = v.w;
        }
        mbar_wait(&wbar, 0);
        __syncthreads();
        {
            const int r1 = (tid & 15) >> 1, n1 = (tid >> 4) * 4 + (tid & 1) * 2;
            float v[MID_RT * M1_C];
            mid_mm<M1_C, M1_KQ, M1_KS, M1_N>(W1, A1, tid >> 4, tid & 15, v);
            const float2 bias = __ldg(reinterpret_cast<const float2*>(w.bl1 + n1));
            const float2 xo = (r1 < nr) ? *reinterpret_cast<const float2*>(X + (row0 + r1) * 64 + n1) : make_float2(0.f, 0.f);
            const float2 x1v = make_float2(xo.x + v[0] + bias.x, xo.y + v[1] + bias.y);
            *reinterpret_cast<float2*>(x1s + r1 * 64 + n1) = x1v;
            if (r1 < nr) *reinterpret_cast<float2*>(X + (row0 + r1) * 64 + n1) = x1v;
        }
        __syncthreads();
        {
            const int r = tid >> 5, lane = tid & 31;
            const float v0 = x1s[r * 64 + lane], v1 = x1s[r * 64 + lane + 32];
            const float mu = warp_sum(v0 + v1) * (1.f / 64.f);
            const float d0 = v0 - mu, d1 = v1 - mu;
            const float rs = rsqrtf(warp_sum(d0 * d0 + d1 * d1) * (1.f / 64.f) + 1e-5f);
            A3[mid_aidx(M3_KS, lane, r)] = d0 * rs * __ldg(w.ln2_g + lane) + __ldg(w.ln2_b + lane);
            A3[mid_aidx(M3_KS, lane + 32, r)] = d1 * rs * __ldg(w.ln2_g + lane + 32) + __ldg(w.ln2_b + lane + 32);
        }
        __syncthreads();
        {
            float v[MID_RT * M3_C];
            const int jp = tid >> 3, r = tid & 7;
            mid_mm<M3_C, M3_KQ, M3_KS, M3_N>(W3a, A3, jp, r, v);
            const float4 ba = __ldg(reinterpret_cast<const float4*>(w.b2 + jp * 8));
            const float4 bb = __ldg(reinterpret_cast<const float4*>(w.b2 + jp * 8 + 4));
            if (r < nr) {
                float4* gp = reinterpret_cast<float4*>(GI + (row0 + r) * 256 + jp * 8);
                gp[0] = make_float4(v[0] + ba.x, v[1] + ba.y, v[2] + ba.z, v[3] + ba.w);
                gp[1] = make_float4(v[4] + bb.x, v[5] + bb.y, v[6] + bb.z, v[7] + bb.w);
            }
        }
    }
}

// n_hops consecutive hops per launch (GI / Hn of hop j at + j * hop_stride floats): h stays in shared memory and c in
// registers between them, the state is read before the first and written after the last.
template <class Map>
__global__ void __launch_bounds__(256)
mid_b_kernel_t(const float* __restrict__ GI, float* __restrict__ Hn, int64_t hop_stride, int n_hops, float* __restrict__ state,
               Map recs, int blk, BlockWeights w, int n_streams, const uint8_t* __restrict__ active) {
    extern __shared__ __align__(16) float sm[];
    float* W3b = sm;                                  // W_hh, k-sliced
    float* A3 = W3b + (MID_W5 - MID_W3B);             // h, k-sliced
    __shared__ __align__(8) unsigned long long wbar;
    TraceScope trace_(TK_MID_B, GI);
    griddep_launch();
    const int tid = threadIdx.x;
    constexpr int TILES = (NF + MID_RT - 1) / MID_RT;
    if (tid == 0) {
        mbar_init(&wbar, 1);
        mbar_fence_init();
        mbar_expect_tx(&wbar, (MID_W5 - MID_W3B) * 4);
        tma_load_1d(W3b, w.mid_pack + MID_W3B, (MID_W5 - MID_W3B) * 4, &wbar);
    }
    __syncthreads();
    griddep_wait();
    for (int item = blockIdx.x; item < n_streams * TILES; item += gridDim.x) {
        const int b = item / TILES;
        const int r0 = (item % TILES) * MID_RT;
        const int nr = min(MID_RT, NF - r0);
        __syncthreads();
        float* sb = stream_rec(state, recs, b) + ST_BLK + (int64_t)blk * BK_STRIDE;
        float* hst = sb + BK_H;
        float* cst = sb + BK_C;
        const int64_t row0 = (int64_t)b * NF + r0;
        if (tid < 128) {
            const int r = tid >> 4, k4 = tid & 15;
            const float4 v = (r < nr) ? *reinterpret_cast<const float4*>(hst + (r0 + r) * 64 + k4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
            A3[mid_aidx(M3_KS, k4 * 4 + 0, r)] = v.x; A3[mid_aidx(M3_KS, k4 * 4 + 1, r)] = v.y;
            A3[mid_aidx(M3_KS, k4 * 4 + 2, r)] = v.z; A3[mid_aidx(M3_KS, k4 * 4 + 3, r)] = v.w;
        }
        const int jp = tid >> 3, r = tid & 7;
        const bool live = r < nr;
        // this lane's cell state and input-side gate pre-activations: loaded now, used after the product
        float2 cc = live ? *reinterpret_cast<const float2*>(cst + (r0 + r) * 64 + jp * 2) : make_float2(0.f, 0.f);
        float2 hh = make_float2(0.f, 0.f);
        const float4* gp = reinterpret_cast<const float4*>(GI + (row0 + r) * 256 + jp * 8);
        float4 ga = make_float4(0.f, 0.f, 0.f, 0.f), gb = ga;
        if (live) { ga = gp[0]; gb = gp[1]; }
        mbar_wait(&wbar, 0);
        for (int j = 0; j < n_hops; ++j) {
            __syncthreads();                          // h of this hop is in A3
            float4 na = make_float4(0.f, 0.f, 0.f, 0.f), nb = na;      // the next hop's input-side gates, in flight during the product
            if (live && j + 1 < n_hops) {
                const float4* np = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(gp) + (int64_t)(j + 1) * hop_stride);
                na = np[0]; nb = np[1];
            }
            float v[MID_RT * M3_C];
            mid_mm<M3_C, M3_KQ, M3_KS, M3_N>(W3b, A3, jp, r, v);
            const float gi0 = fast_sigmoid(v[0] + ga.x), gf0 = fast_sigmoid(v[1] + ga.y), gg0 = fast_tanh(v[2] + ga.z), go0 = fast_sigmoid(v[3] + ga.w);
            const float gi1 = fast_sigmoid(v[4] + gb.x), gf1 = fast_sigmoid(v[5] + gb.y), gg1 = fast_tanh(v[6] + gb.z), go1 = fast_sigmoid(v[7] + gb.w);
            cc = make_float2(gf0 * cc.x + gi0 * gg0, gf1 * cc.y + gi1 * gg1);
            hh = make_float2(go0 * fast_tanh(cc.x), go1 * fast_tanh(cc.y));
            if (live) *reinterpret_cast<float2*>(Hn + (int64_t)j * hop_stride + (row0 + r) * 64 + jp * 2) = hh;
            ga = na; gb = nb;
            if (j + 1 < n_hops) {
                __syncthreads();                      // every lane has read the old h
                A3[mid_aidx(M3_KS, jp * 2, r)] = hh.x;
                A3[mid_aidx(M3_KS, jp * 2 + 1, r)] = hh.y;
            }
        }
        if (live && stream_active(recs, active, b)) {
            *reinterpret_cast<float2*>(cst + (r0 + r) * 64 + jp * 2) = cc;
            *reinterpret_cast<float2*>(hst + (r0 + r) * 64 + jp * 2) = hh;
        }
    }
}

__global__ void __launch_bounds__(256)
mid_c_kernel(const float* __restrict__ Hn, float* __restrict__ X, float* __restrict__ QKV, BlockWeights w, int n_streams,
             int64_t hop_stride, int n_hops) {
    extern __shared__ __align__(16) float sm[];
    float* W5 = sm;                                   // inter linear | q|k|v projections, k-sliced
    float* W6 = W5 + (MID_W6 - MID_W5);
    float* A5 = W5 + (MID_PACK - MID_W5);
    float* A6 = A5 + MID_A5;
    __shared__ __align__(8) unsigned long long wbar;
    TraceScope trace_(TK_MID_C, Hn);
    griddep_launch();
    const int tid = threadIdx.x;
    constexpr int TILES = (NF + MID_RT - 1) / MID_RT;
    if (tid == 0) {
        mbar_init(&wbar, 1);
        mbar_fence_init();
        mbar_expect_tx(&wbar, (MID_PACK - MID_W5) * 4);
        tma_load_1d(W5, w.mid_pack + MID_W5, (MID_PACK - MID_W5) * 4, &wbar);
    }
    __syncthreads();
    griddep_wait();
    const float* Hn0 = Hn; float* X0 = X; float* QKV0 = QKV;
    for (int item = blockIdx.x; item < n_hops * n_streams * TILES; item += gridDim.x) {
        const int hop = item / (n_streams * TILES), it_h = item % (n_streams * TILES);
        Hn = Hn0 + (int64_t)hop * hop_stride; X = X0 + (int64_t)hop * hop_stride; QKV = QKV0 + (int64_t)hop * hop_stride;
        const int b = it_h / TILES;
        const int r0 = (it_h % TILES) * MID_RT;
        const int nr = min(MID_RT, NF - r0);
        __syncthreads();
        const int64_t row0 = (int64_t)b * NF + r0;
        if (tid < 128) {
            const int r = tid >> 4, k4 = tid & 15;
            const float4 v = (r < nr) ? *reinterpret_cast<const float4*>(Hn + (row0 + r) * 64 + k4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
            A5[mid_aidx(M5_KS, k4 * 4 + 0, r)] = v.x; A5[mid_aidx(M5_KS, k4 * 4 + 1, r)] = v.y;
            A5[mid_aidx(M5_KS, k4 * 4 + 2, r)] = v.z; A5[mid_aidx(M5_KS, k4 * 4 + 3, r)] = v.w;
        }
        const int r1 = (tid & 15) >> 1, n1 = (tid >> 4) * 4 + (tid & 1) * 2;
        const float2 x1v = (r1 < nr) ? *reinterpret_cast<const float2*>(X + (row0 + r1) * 64 + n1) : make_float2(0.f, 0.f);
        mbar_wait(&wbar, 0);
        __syncthreads();
        {
            float v[MID_RT * M5_C];
            mid_mm<M5_C, M5_KQ, M5_KS, M5_N>(W5, A5, tid >> 4, tid & 15, v);
            const float2 bias = __ldg(reinterpret_cast<const float2*>(w.bl2 + n1));
            const float2 x2v = make_float2(x1v.x + v[0] + bias.x, x1v.y + v[1] + bias.y);
            if (r1 < nr) *reinterpret_cast<float2*>(X + (row0 + r1) * 64 + n1) = x2v;
            A6[mid_aidx(M6_KS, n1, r1)] = x2v.x;
            A6[mid_aidx(M6_KS, n1 + 1, r1)] = x2v.y;
        }
        __syncthreads();
        if (tid < (M6_N / M6_C) * M6_KQ) {
            float v[MID_RT * M6_C];
            const int cg = tid >> 3, r = tid & 7;
            mid_mm<M6_C, M6_KQ, M6_KS, M6_N>(W6, A6, cg, r, v);
            const float4 bias = __ldg(reinterpret_cast<const float4*>(w.bqkv + cg * 4));
            const float slope = __ldg(w.slopes + (cg < 6 ? 0 : (cg < 12 ? 1 : 2)));
            if (r < nr)
                *reinterpret_cast<float4*>(QKV + (row0 + r) * NQKV + cg * 4) =
                    make_float4(prelu(v[0] + bias.x, slope), prelu(v[1] + bias.y, slope), prelu(v[2] + bias.z, slope),
                                prelu(v[3] + bias.w, slope));
        }
    }
}

// the dense forms (call row b = record b); the `_t<Records>` forms serve slot-list calls (l2h_sep_forward_slots)
constexpr auto mid_kernel = mid_kernel_t<int64_t>;
constexpr auto mid_b_kernel = mid_b_kernel_t<int64_t>;

}  // namespace l2h
