// tail_kernel: for a one-hop call of a few streams (the latency path: one 8 ms chunk) everything of a block that follows
// the intra BiLSTM runs as ONE kernel, one thread-block cluster of 16 CTAs per stream:
//
//   phase M   the row-local middle (mid_kernel.cuh: intra Linear + residual, inter-LSTM step, inter Linear + residual,
//             Q|K|V projections) on 13 row tiles of 8 frequency bins, one tile per CTA, weights resident in shared memory
//   phase Q   LayerNorm over (F, E) per head of Q, K, V: every tile CTA reduces its rows to (mean, M2), the cluster
//             combines the 13 partials (Chan) through distributed shared memory; K and V go to the ring slot of this
//             frame, Q stays in shared memory                                                   (tfgridnet_causal.py:547-562)
//   phase A   attention over the 50-frame window: CTA (head h = rank / 4, part = rank % 4) scores its 12-13 ring rows
//             against Q_h (gathered from the tile CTAs) and reduces them to an un-normalised partial (max, sum, o[1552]) (:563-581)
//   phase O   every tile CTA merges the four partials of each head for ITS rows, applies Linear(64->64) + PReLU, the
//             cluster combines the LayerNorm(6208) statistics, + residual (+ speaker gate after block 0)          (:583-588, :250)
//   phase G   (blocks 0, 1) the input projection of the NEXT block's intra BiLSTM for the CTA's rows:
//             GX = LN(x) W_ih^T + b, with W_ih (128 KB) brought by TMA into the shared memory the mid weights occupied (:505-512)
//
// Replaces mid_kernel + qkv_kernel + attn_cluster_kernel + attn_out_kernel + the next rows_gemm launch: 5 launches and
// 4 global round trips become one launch with 5 cluster barriers (tools/cluster16_probe.cu times one).
// The 16-CTA cluster is a non-portable size: the engine asks cudaOccupancyMaxActiveClusters first and keeps the separate
// kernels when it cannot be scheduled.
#pragma once
#include "mid_kernel.cuh"

namespace l2h {

constexpr int TAIL_CL = 16;
constexpr int TAIL_TILES = (NF + MID_RT - 1) / MID_RT;        // 13
constexpr int TAIL_PARTS = TAIL_CL / NHEAD;                   // 4 CTAs share one head's window
static_assert(TAIL_TILES <= TAIL_CL && TAIL_PARTS * NHEAD == TAIL_CL, "cluster geometry");
// buffers that live in the shared memory of the intra-Linear weights (dead after phase 1 of the mid section)
constexpr int TL_WP = 0;                                      // [64][64]   W_p^T (k, n), by TMA after phase M
constexpr int TL_PS = TL_WP + 64 * 64;                        // [8][112]   projections of the tile
constexpr int TL_X2 = TL_PS + MID_RT * NQKV;                  // [8][64]    X2 (residual of phase O)
constexpr int TL_QN = TL_X2 + MID_RT * 64;                    // [4][8*6]   normalised Q of the tile's rows, per head
constexpr int TL_QS = TL_QN + NHEAD * MID_RT * QE;            // [584]      Q of this CTA's head (phase A)
constexpr int TL_OS = TL_QS + QK_LD;                          // [1552]     partial attention output
constexpr int TL_END = TL_OS + V_DIM;
static_assert(TL_END <= MID_W3A && TL_PS % 4 == 0 && TL_X2 % 4 == 0 && TL_QN % 4 == 0 && TL_QS % 4 == 0 && TL_OS % 4 == 0, "alias region");
static_assert(64 * 512 <= MID_PACK - MID_W3A, "next block's W_ih fits behind the alias region");
constexpr size_t TAIL_SMEM = MID_SMEM;

struct NextIh {                 // the next block's intra input projection (null wih_t: last block, no phase G)
    const float* ln_g; const float* ln_b; const float* wih_t; const float* bias; float* GX;
};

__device__ __forceinline__ int tail_rows(int p) { return min(MID_RT, NF - p * MID_RT); }

// Input projection of an intra BiLSTM for one tile of MID_RT rows: GX[r][0..511] = LN(x[r]) W_ih^T + b.
// xrows: the tile's rows [8][64] in shared memory (all 8 rows defined); xn: [64][8] scratch; wih: W_ih^T [64][512] in shared
// memory (its TMA has completed); (g0, g1, b0, b1): LayerNorm gamma / beta of channels lane, lane + 32; bias: b[2 tid .. +1].
// Thread t owns gate columns 2t, 2t+1 for all 8 rows (row pairs as float2 FMA pairs).  Ends without a barrier.
__device__ __forceinline__ void ih_rows_tile(const float* xrows, float* xn, const float* wih, float g0, float g1, float b0, float b1,
                                             float2 bias, float* gx_rows, int nr, int tid) {
    const int warp = tid >> 5, lane = tid & 31;
    {                                              // LayerNorm over channels: one warp per row, k-major result
        const int r = warp;
        const float v0 = xrows[r * 64 + lane], v1 = xrows[r * 64 + lane + 32];
        const float m = warp_sum(v0 + v1) * (1.f / 64.f);
        const float d0 = v0 - m, d1 = v1 - m;
        const float rstd = rsqrtf(warp_sum(d0 * d0 + d1 * d1) * (1.f / 64.f) + 1e-5f);
        xn[lane * MID_RT + r] = d0 * rstd * g0 + b0;
        xn[(lane + 32) * MID_RT + r] = d1 * rstd * g1 + b1;
    }
    __syncthreads();
    float2 acc[2][4];
#pragma unroll
    for (int c = 0; c < 2; ++c)
#pragma unroll
        for (int p = 0; p < 4; ++p) acc[c][p] = make_float2(0.f, 0.f);
#pragma unroll 8
    for (int k = 0; k < 64; ++k) {
        const float2 wv = *reinterpret_cast<const float2*>(wih + k * 512 + 2 * tid);
        const float4 xa = *reinterpret_cast<const float4*>(xn + k * MID_RT);
        const float4 xb = *reinterpret_cast<const float4*>(xn + k * MID_RT + 4);
        const float2 xr2[4] = {make_float2(xa.x, xa.y), make_float2(xa.z, xa.w), make_float2(xb.x, xb.y), make_float2(xb.z, xb.w)};
        const float2 w0 = make_float2(wv.x, wv.x), w1 = make_float2(wv.y, wv.y);
#pragma unroll
        for (int p = 0; p < 4; ++p) { acc[0][p] = ffma2(w0, xr2[p], acc[0][p]); acc[1][p] = ffma2(w1, xr2[p], acc[1][p]); }
    }
    float* gx = gx_rows + 2 * tid;
#pragma unroll
    for (int r = 0; r < MID_RT; ++r) {
        if (r < nr) {
            const float v0 = (r & 1) ? acc[0][r >> 1].y : acc[0][r >> 1].x;
            const float v1 = (r & 1) ? acc[1][r >> 1].y : acc[1][r >> 1].x;
            *reinterpret_cast<float2*>(gx + (int64_t)r * 512) = make_float2(v0 + bias.x, v1 + bias.y);
        }
    }
}

// (which, head, e, d) of projection column col of the 112
__device__ __forceinline__ void tail_col(int col, int& which, int& h, int& e, int& d) {
    which = (col < 24) ? 0 : (col < 48 ? 1 : 2);
    d = (which == 2) ? VD : QE;
    const int cc = col - (which == 2 ? 48 : which * 24);
    h = cc / d; e = cc % d;
}

template <class Map>
__global__ void __launch_bounds__(256)
tail_kernel_t(const float* __restrict__ Y, float* X, float* __restrict__ state, Map recs, int blk, BlockWeights w,
              NextIh nx, int apply_gate, int frame_k, const uint8_t* __restrict__ active) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(16) float sm[];
    const MidSmem S(sm);
    float* wps = sm + TL_WP; float* Ps = sm + TL_PS; float* x2s = sm + TL_X2; float* qn = sm + TL_QN;
    float* qs = sm + TL_QS; float* os = sm + TL_OS;
    float* Zs = S.A1;                       // [8][64] merged attention output of the tile (phase O); A1 is dead after phase 1
    float* xn = S.A1 + MID_RT * 64;         // [64][8] LN(x_out), k-major (phase G)
    float* wih = sm + MID_W3A;              // [64][512] next block's W_ih^T (phase G)
    __shared__ __align__(8) unsigned long long wbar, pbar, gbar;
    __shared__ __align__(16) float vs[MV_TOTAL];
    __shared__ float qstat[12][2];          // per (which, head): mean, M2 of this tile's rows
    __shared__ float gstat[12][2];          // ... combined: mean, rstd
    __shared__ float sc[16];
    __shared__ float ml[2];                 // phase A: this CTA's running max and sum
    __shared__ float pmx[TAIL_CL], psum[TAIL_CL], coef[TAIL_CL];
    __shared__ float pstat[2], fin[2];
    __shared__ float red[32];

    TraceScope trace_(TK_TAIL, Y);
    griddep_launch();
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int rk = (int)cluster.block_rank(), b = blockIdx.y;
    const bool has_tile = rk < TAIL_TILES;
    const int r0 = rk * MID_RT, nr = has_tile ? tail_rows(rk) : 0;
    float* st = stream_rec(state, recs, b);
    float* sb = st + ST_BLK + (int64_t)blk * BK_STRIDE;
    const bool has_next = nx.wih_t != nullptr;
    const bool live = stream_active(recs, active, b);          // false: the stream skips this hop, its record is not written
    if (tid == 0) {
        mbar_init(&wbar, 1); mbar_init(&pbar, 1); mbar_init(&gbar, 1);
        mbar_fence_init();
        if (has_tile) {                    // weights: independent of the chain, so before the dependency wait
            mbar_expect_tx(&wbar, MID_PACK * 4);
            tma_load_1d(S.Wp + MID_W1, w.mid_pack + MID_W1, (MID_W3B - MID_W1) * 4, &wbar);
            tma_load_1d(S.Wp + MID_W3B, w.mid_pack + MID_W3B, (MID_W5 - MID_W3B) * 4, &wbar);
            tma_load_1d(S.Wp + MID_W5, w.mid_pack + MID_W5, (MID_PACK - MID_W5) * 4, &wbar);
        }
    }
    // ---- every parameter this thread will need, requested before the dependency wait (registers / the staged vectors) -----
    const int n_o = tid & 63, rp = tid >> 6;               // phase O: this thread finishes rows rp and rp + 4, column n_o
    const bool ok0 = rp < nr, ok1 = rp + 4 < nr;
    float ng[4], nb[4];                                    // LayerNorm gamma / beta of the <= 4 projection elements it normalises
    float og0 = 0.f, ob0 = 0.f, og1 = 0.f, ob1 = 0.f, bp_n = 0.f, slope_p = 0.f;
    float gg0 = 0.f, gg1 = 0.f, gb0 = 0.f, gb1 = 0.f;      // phase G: the next block's LayerNorm, channels lane and lane + 32
    float2 gbias = make_float2(0.f, 0.f);
    if (has_tile) {
        mid_stage_vecs(vs, w, tid);
#pragma unroll
        for (int it = 0; it < 4; ++it) {
            const int idx = tid + 256 * it;
            ng[it] = 0.f; nb[it] = 0.f;
            if (idx < nr * NQKV) {
                int which, h, e, d;
                tail_col(idx % NQKV, which, h, e, d);
                const int i = (r0 + idx / NQKV) * d + e;
                ng[it] = __ldg((which == 0 ? w.lnq_g : (which == 1 ? w.lnk_g : w.lnv_g)) + i);
                nb[it] = __ldg((which == 0 ? w.lnq_b : (which == 1 ? w.lnk_b : w.lnv_b)) + i);
            }
        }
        if (ok0) { og0 = __ldg(w.lnp_g + (r0 + rp) * 64 + n_o); ob0 = __ldg(w.lnp_b + (r0 + rp) * 64 + n_o); }
        if (ok1) { og1 = __ldg(w.lnp_g + (r0 + rp + 4) * 64 + n_o); ob1 = __ldg(w.lnp_b + (r0 + rp + 4) * 64 + n_o); }
        bp_n = __ldg(w.bp + n_o); slope_p = __ldg(w.slopes + 3);
        if (has_next) {
            gg0 = __ldg(nx.ln_g + lane); gg1 = __ldg(nx.ln_g + lane + 32);
            gb0 = __ldg(nx.ln_b + lane); gb1 = __ldg(nx.ln_b + lane + 32);
            gbias = __ldg(reinterpret_cast<const float2*>(nx.bias + 2 * tid));
        }
    }
    __syncthreads();
    // the carried-state half of the inter-LSTM step (h_prev W_hh, old c): inputs of the PREVIOUS hop only -> before the dependency wait
    float hv[8];
    float2 cold = make_float2(0.f, 0.f);
    if (has_tile) {
        mbar_wait(&wbar, 0);
        mid_h_product(S, sb + BK_H, sb + BK_C, r0, nr, tid, hv, cold);
    }
    griddep_wait();
    const long long pos = rec_pos(st) + frame_k;
    trace_.mark(0);

    // ---- phase M ------------------------------------------------------------------------------------------------
    float gate0 = 1.f, gate1 = 1.f;
    if (has_tile) {
        if (apply_gate) {                  // the speaker gate of this thread's two outputs (front_kernel's memo CTA wrote it)
            if (ok0) gate0 = st[ST_GATE + (r0 + rp) * 64 + n_o];
            if (ok1) gate1 = st[ST_GATE + (r0 + rp + 4) * 64 + n_o];
        }
        const int64_t row0 = (int64_t)b * NF + r0;
        mid_tile<true>(S, Y + row0 * 128, X + row0 * 64, x2s, Ps, sb + BK_H, sb + BK_C, r0, nr, vs, tid, live, hv, cold);
        __syncthreads();
        if (tid == 0) {                    // the mid weights are dead: W_p (and the next block's W_ih) take their place
            fence_proxy_async();
            mbar_expect_tx(&pbar, 64 * 64 * 4);
            tma_load_1d(wps, w.wp_t, 64 * 64 * 4, &pbar);
            if (has_next) {
                mbar_expect_tx(&gbar, 64 * 512 * 4);
                tma_load_1d(wih, nx.wih_t, 64 * 512 * 4, &gbar);
            }
        }
    }
    trace_.mark(1);
    // ---- phase Q: partial LayerNorm statistics of the tile: 16 lanes per (which, head) group ----------------------------
    if (tid < 12 * 16) {
        const int g = tid >> 4, l16 = tid & 15;
        const int which = g >> 2, h = g & 3;
        const int d = (which == 2) ? VD : QE;
        const int col0 = (which == 2) ? (48 + h * VD) : (which * 24 + h * QE);
        const int n = nr * d;                              // <= 128
        float v[8];
        float s = 0.f;
#pragma unroll
        for (int it = 0; it < 8; ++it) {
            const int i = l16 + 16 * it;
            v[it] = (i < n) ? Ps[(i / d) * NQKV + col0 + i % d] : 0.f;
            s += v[it];
        }
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        const float mean = (n > 0) ? s / (float)n : 0.f;
        float q = 0.f;
#pragma unroll
        for (int it = 0; it < 8; ++it) { const float dv = (l16 + 16 * it < n) ? v[it] - mean : 0.f; q += dv * dv; }
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
        if (l16 == 0) { qstat[g][0] = mean; qstat[g][1] = q; }
    }
    trace_.mark(2);
    cluster.sync();                                                                    // #1: partial statistics visible
    trace_.mark(3);
    // phase A's ring rows that do not depend on this hop are requested now (they arrive while the statistics are combined)
    const int ah = rk / TAIL_PARTS, part = rk % TAIL_PARTS;
    constexpr int a_base = ATT / TAIL_PARTS, a_rem = ATT % TAIL_PARTS;     // 12 rows each, the first 2 parts take 13
    const int j0 = part * a_base + min(part, a_rem), na = a_base + (part < a_rem ? 1 : 0);
    const float* kb = sb + BK_K + (int64_t)ah * RING * QK_LD;
    const float* vb = sb + BK_V + (int64_t)ah * RING * V_DIM;
    const long long p0 = pos - (ATT - 1) + j0;
    const int first = (int)(((p0 % RING) + RING) % RING);
    const bool newest_here = (part == TAIL_PARTS - 1);      // the window's last row is the one this launch writes
    const int na_old = newest_here ? na - 1 : na;
    float4 kv[2][5];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        const int r = warp + 8 * rr;
        const float4* kr = reinterpret_cast<const float4*>(kb + (int64_t)((first + r) % RING) * QK_LD);
#pragma unroll
        for (int u = 0; u < 5; ++u) {
            const int i = lane + 32 * u;
            kv[rr][u] = (r < na_old && i < QK_LD / 4) ? __ldcg(kr + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    float4 vpre[7], vpre_b[7];                              // value rows 0..6 of this CTA's share: column tid and (threads < 132) tid + 256
    const bool has_b = tid + 256 < V_DIM / 4;
#pragma unroll
    for (int j = 0; j < 7; ++j) {
        const float4* vr = reinterpret_cast<const float4*>(vb + (int64_t)((first + j) % RING) * V_DIM);
        vpre[j] = __ldcg(vr + tid);
        vpre_b[j] = has_b ? __ldcg(vr + tid + 256) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (tid < 12) {
        const int d = ((tid >> 2) == 2) ? VD : QE;
        float mp[TAIL_TILES], m2[TAIL_TILES];
#pragma unroll
        for (int p = 0; p < TAIL_TILES; ++p) {
            const float* ps = cluster.map_shared_rank(&qstat[0][0], p);
            mp[p] = ps[tid * 2]; m2[p] = ps[tid * 2 + 1];
        }
        float mean = 0.f;
#pragma unroll
        for (int p = 0; p < TAIL_TILES; ++p) mean += (float)(tail_rows(p) * d) * mp[p];
        mean /= (float)(NF * d);
        float M2 = 0.f;
#pragma unroll
        for (int p = 0; p < TAIL_TILES; ++p) { const float dm = mp[p] - mean; M2 += m2[p] + (float)(tail_rows(p) * d) * dm * dm; }
        gstat[tid][0] = mean;
        gstat[tid][1] = rsqrtf(M2 / (float)(NF * d) + 1e-5f);
    }
    __syncthreads();
    // normalise the tile: Q -> shared memory (gathered by the attention CTAs), K | V -> this frame's ring slot
    const int slot = (int)(pos % RING);
    if (has_tile) {
#pragma unroll
        for (int it = 0; it < 4; ++it) {
            const int idx = tid + 256 * it;
            if (idx < nr * NQKV) {
                const int r = idx / NQKV;
                int which, h, e, d;
                tail_col(idx % NQKV, which, h, e, d);
                const int g = which * 4 + h, i = (r0 + r) * d + e;
                const float v = (Ps[idx] - gstat[g][0]) * gstat[g][1] * ng[it] + nb[it];
                if (which == 0) qn[h * (MID_RT * QE) + r * QE + e] = v;
                else if (live && which == 1) sb[BK_K + ((int64_t)h * RING + slot) * QK_LD + i] = v;
                else if (live) sb[BK_V + ((int64_t)h * RING + slot) * V_DIM + i] = v;
            }
        }
        if (live && rk == TAIL_TILES - 1 && tid < 2 * NHEAD)          // the two pad columns 582, 583 of the K row
            sb[BK_K + ((int64_t)(tid >> 1) * RING + slot) * QK_LD + QK_DIM + (tid & 1)] = 0.f;
    }
    trace_.mark(4);
    cluster.sync();                                                                    // #2: ring row and Q complete
    trace_.mark(5);
    // ---- phase A: this CTA's share of the 50-row window of head ah ------------------------------------------------------
    {
        for (int i = tid; i < QK_LD; i += 256) {
            float v = 0.f;
            if (i < QK_DIM) {
                const int p = i / (MID_RT * QE);
                v = cluster.map_shared_rank(qn, p)[ah * (MID_RT * QE) + (i - p * (MID_RT * QE))];
            }
            qs[i] = v;
        }
        if (newest_here) {                                 // the row written during this launch: the last part's last row
            static_assert(TAIL_PARTS - 1 >= a_rem, "the last part holds a_base rows");
            constexpr int r = a_base - 1;
            if (warp == (r & 7)) {
                const float4* kr = reinterpret_cast<const float4*>(kb + (int64_t)((first + r) % RING) * QK_LD);
#pragma unroll
                for (int u = 0; u < 5; ++u) {
                    const int i = lane + 32 * u;
                    kv[r >> 3][u] = (i < QK_LD / 4) ? __ldcg(kr + i) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
        }
        __syncthreads();
        const float scale = rsqrtf((float)QK_DIM);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {                 // one warp per key row
            const int r = warp + 8 * rr;
            if (r < na) {
                float s = 0.f;
#pragma unroll
                for (int u = 0; u < 5; ++u) {
                    const int i = lane + 32 * u;
                    if (i < QK_LD / 4) {
                        const float4 qv = reinterpret_cast<const float4*>(qs)[i];
                        s += kv[rr][u].x * qv.x + kv[rr][u].y * qv.y + kv[rr][u].z * qv.z + kv[rr][u].w * qv.w;
                    }
                }
                s = warp_sum(s);
                if (lane == 0) sc[r] = s * scale;
            }
        }
        __syncthreads();
        if (warp == 0) {
            const float a0 = (lane < na) ? sc[lane] : -INFINITY;
            const float mx = warp_max(a0);
            const float e0 = (lane < na) ? __expf(a0 - mx) : 0.f;
            const float lsum = warp_sum(e0);
            if (lane < na) sc[lane] = e0;
            if (lane == 0) { ml[0] = mx; ml[1] = lsum; }
        }
        // rows 7 .. na-1 of both columns in ONE batch of loads (they contain the row written during this launch)
        float4 v2[6], v2b[6];
#pragma unroll
        for (int j = 0; j < 6; ++j) {
            const float4* vr = reinterpret_cast<const float4*>(vb + (int64_t)((first + 7 + j) % RING) * V_DIM);
            v2[j] = (7 + j < na) ? __ldcg(vr + tid) : make_float4(0.f, 0.f, 0.f, 0.f);
            v2b[j] = (has_b && 7 + j < na) ? __ldcg(vr + tid + 256) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        __syncthreads();
        {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f), accb = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int j = 0; j < 7; ++j) {
                const float p = sc[j];                     // na >= 12 > 7
                acc.x = fmaf(p, vpre[j].x, acc.x); acc.y = fmaf(p, vpre[j].y, acc.y);
                acc.z = fmaf(p, vpre[j].z, acc.z); acc.w = fmaf(p, vpre[j].w, acc.w);
                accb.x = fmaf(p, vpre_b[j].x, accb.x); accb.y = fmaf(p, vpre_b[j].y, accb.y);
                accb.z = fmaf(p, vpre_b[j].z, accb.z); accb.w = fmaf(p, vpre_b[j].w, accb.w);
            }
#pragma unroll
            for (int j = 0; j < 6; ++j) {
                const float p = (7 + j < na) ? sc[7 + j] : 0.f;
                acc.x = fmaf(p, v2[j].x, acc.x); acc.y = fmaf(p, v2[j].y, acc.y);
                acc.z = fmaf(p, v2[j].z, acc.z); acc.w = fmaf(p, v2[j].w, acc.w);
                accb.x = fmaf(p, v2b[j].x, accb.x); accb.y = fmaf(p, v2b[j].y, accb.y);
                accb.z = fmaf(p, v2b[j].z, accb.z); accb.w = fmaf(p, v2b[j].w, accb.w);
            }
            reinterpret_cast<float4*>(os)[tid] = acc;
            if (has_b) reinterpret_cast<float4*>(os)[tid + 256] = accb;
        }
    }
    trace_.mark(6);
    cluster.sync();                                                                    // #3: every partial complete
    trace_.mark(7);
    // ---- phase O: merge the heads for the tile's rows, Linear + PReLU, LayerNorm(6208), residual ------------------------
    float pv0 = 0.f, pv1 = 0.f;
    if (has_tile) {
        if (tid < TAIL_CL) {
            const float* pml = cluster.map_shared_rank(ml, tid);
            pmx[tid] = pml[0]; psum[tid] = pml[1];
        }
        float4 zv[TAIL_PARTS];                              // Z[r][h*16 + c4*4 ..] = sum_p coef * o_p[(r0 + r)*16 + c4*4 ..]
        const int zr = tid >> 4, zh = (tid >> 2) & 3, zc = tid & 3;
        if (tid < 128 && zr < nr) {
#pragma unroll
            for (int p = 0; p < TAIL_PARTS; ++p)
                zv[p] = reinterpret_cast<const float4*>(cluster.map_shared_rank(os, zh * TAIL_PARTS + p))[(r0 + zr) * (VD / 4) + zc];
        }
        __syncthreads();
        if (tid < NHEAD) {
            float mstar = -INFINITY, den = 0.f, wgt[TAIL_PARTS];
#pragma unroll
            for (int p = 0; p < TAIL_PARTS; ++p) mstar = fmaxf(mstar, pmx[tid * TAIL_PARTS + p]);
#pragma unroll
            for (int p = 0; p < TAIL_PARTS; ++p) { wgt[p] = __expf(pmx[tid * TAIL_PARTS + p] - mstar); den += wgt[p] * psum[tid * TAIL_PARTS + p]; }
            const float inv = 1.f / den;
#pragma unroll
            for (int p = 0; p < TAIL_PARTS; ++p) coef[tid * TAIL_PARTS + p] = wgt[p] * inv;
        }
        __syncthreads();
        if (tid < 128) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            if (zr < nr) {
#pragma unroll
                for (int p = 0; p < TAIL_PARTS; ++p) {
                    const float cf = coef[zh * TAIL_PARTS + p];
                    acc.x = fmaf(cf, zv[p].x, acc.x); acc.y = fmaf(cf, zv[p].y, acc.y);
                    acc.z = fmaf(cf, zv[p].z, acc.z); acc.w = fmaf(cf, zv[p].w, acc.w);
                }
            }
            *reinterpret_cast<float4*>(Zs + zr * 64 + zh * VD + zc * 4) = acc;
        }
        mbar_wait(&pbar, 0);
        __syncthreads();
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;      // two partial sums per row: shorter dependency chains
#pragma unroll 8
        for (int k = 0; k < 64; k += 2) {
            const float w0 = wps[k * 64 + n_o], w1 = wps[(k + 1) * 64 + n_o];
            const float2 z0 = *reinterpret_cast<const float2*>(Zs + rp * 64 + k);
            const float2 z1 = *reinterpret_cast<const float2*>(Zs + (rp + 4) * 64 + k);
            a0 = fmaf(z0.x, w0, a0); a1 = fmaf(z0.y, w1, a1);
            a2 = fmaf(z1.x, w0, a2); a3 = fmaf(z1.y, w1, a3);
        }
        pv0 = prelu((a0 + a1) + bp_n, slope_p);
        pv1 = prelu((a2 + a3) + bp_n, slope_p);
        const float cnt = (float)(nr * 64);
        const float mean = block_sum((ok0 ? pv0 : 0.f) + (ok1 ? pv1 : 0.f), red) / cnt;
        const float d0 = ok0 ? pv0 - mean : 0.f, d1 = ok1 ? pv1 - mean : 0.f;
        const float M2 = block_sum(d0 * d0 + d1 * d1, red);
        if (tid == 0) { pstat[0] = mean; pstat[1] = M2; }
    }
    trace_.mark(8);
    cluster.sync();                                                                    // #4: LayerNorm partials visible
    trace_.mark(9);
    if (has_tile && warp == 0) {
        float mp = 0.f, m2 = 0.f, np = 0.f;
        if (lane < TAIL_TILES) {
            const float* ps = cluster.map_shared_rank(pstat, lane);
            mp = ps[0]; m2 = ps[1]; np = (float)(tail_rows(lane) * 64);
        }
        const float mean = warp_sum(np * mp) * (1.f / FC);
        const float dm = mp - mean;
        const float M2 = warp_sum(m2 + np * dm * dm);
        if (lane == 0) { fin[0] = mean; fin[1] = rsqrtf(M2 * (1.f / FC) + 1e-5f); }
    }
    __syncthreads();
    cluster.barrier_arrive();              // #5 (arrive): this CTA reads no peer's shared memory from here on
    if (has_tile) {
        const float mu = fin[0], rs = fin[1];
        float* xr = X + ((int64_t)b * NF + r0) * 64;
        float xo0 = 0.f, xo1 = 0.f;
        if (ok0) {
            xo0 = (x2s[rp * 64 + n_o] + (pv0 - mu) * rs * og0 + ob0) * gate0;
            xr[rp * 64 + n_o] = xo0;
        }
        if (ok1) {
            xo1 = (x2s[(rp + 4) * 64 + n_o] + (pv1 - mu) * rs * og1 + ob1) * gate1;
            xr[(rp + 4) * 64 + n_o] = xo1;
        }
        trace_.mark(10);
        // ---- phase G: GX rows of the next block = LN(x_out) W_ih^T + b ---------------------------------------------------
        if (has_next) {
            x2s[rp * 64 + n_o] = xo0;                      // each thread overwrites the two entries only it read
            x2s[(rp + 4) * 64 + n_o] = xo1;
            __syncthreads();
            mbar_wait(&gbar, 0);
            ih_rows_tile(x2s, xn, wih, gg0, gg1, gb0, gb1, gbias, nx.GX + ((int64_t)b * NF + r0) * 512, nr, tid);
        }
    }
    trace_.mark(11);
    cluster.barrier_wait();                // #5 (wait): nobody leaves while a peer may still read its shared memory
}

// ------------------------------------------------------------------------------------------------------------------
// front1_kernel: the head of a one-hop call on the latency path.  front_kernel runs a frame in ONE CTA (150 KB of analysis
// filters for 194 dot products, then a 3x3 conv, all on one SM) and is followed by
// the W_ih GEMM launch of block 0.  Here the frame is 13 row tiles of 8 bins like tail_kernel's: CTA p computes the
// spectrum only for the bins its conv rows touch (f0-1 .. f0+8: 20 filter rows instead of 194), the conv for its rows, and
// block 0's input projection GX = LN(x) W_ih^T + b for them (W_ih arrives by TMA meanwhile).  One more CTA (blockIdx.x == 13)
// is the speaker-gate memo of front_kernel.  grid (14, B), 256 threads.       (tfgridnet_causal.py:229-248, :505-512)
constexpr int F1_NB = MID_RT + 2;                      // bins per CTA with the conv halo
constexpr size_t FRONT1_SMEM = (size_t)(64 * 512) * sizeof(float);

template <class Map>
__global__ void __launch_bounds__(256)
front1_kernel_t(const float* __restrict__ x, int64_t x_bstride, int64_t x_cstride, int x_len, float* __restrict__ X,
                float* __restrict__ state, Map recs, SepWeights w, BlockWeights w0, float* __restrict__ GX, int pos_rel,
                const float* __restrict__ emb, float* __restrict__ spk_pre, const uint8_t* __restrict__ active) {
    extern __shared__ __align__(16) float wih[];       // [64][512] block 0's W_ih^T
    __shared__ __align__(16) float xs[NMIC][NFFT];      // the frame's samples (reused as scratch by the gate CTA: >= 288 floats)
    __shared__ float U[3][4][F1_NB];                    // [frame t-2..t][ch][halo + bin], zero outside 0..96
    __shared__ __align__(16) float xrows[MID_RT * 64];
    __shared__ __align__(16) float xn[64 * MID_RT];
    __shared__ __align__(8) unsigned long long gbar;
    TraceScope trace_(TK_FRONT, X);
    griddep_launch();
    const int p = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (p == TAIL_TILES) {                 // the extra CTA of this stream: speaker-gate memo
        griddep_wait();
        spk_gate_cta(emb, spk_pre, state, recs, w, b, &xs[0][0], active);
        return;
    }
    const int f0 = p * MID_RT, nr = tail_rows(p);
    if (tid == 0) {
        mbar_init(&gbar, 1);
        mbar_fence_init();
        mbar_expect_tx(&gbar, 64 * 512 * 4);
        tma_load_1d(wih, w0.wih1_t, 64 * 512 * 4, &gbar);
    }
    // parameters this thread needs later, requested now
    const int o = tid & 63, fq = tid >> 6;              // conv: output channel o, rows fq and fq + 4
    float wr[36];
#pragma unroll
    for (int k = 0; k < 36; ++k) wr[k] = __ldg(w.wc + o * 36 + k);
    const float bc = __ldg(w.bc + o);
    const float gg0 = __ldg(w0.ln1_g + lane), gg1 = __ldg(w0.ln1_g + lane + 32);
    const float gb0 = __ldg(w0.ln1_b + lane), gb1 = __ldg(w0.ln1_b + lane + 32);
    const float2 gbias = __ldg(reinterpret_cast<const float2*>(w0.b1 + 2 * tid));
    // the filter values of this warp's outputs: item = (bin slot, re|im) -> filterbank row ri*97 + fb; lanes split the 192 taps
    constexpr int ITEMS = 2 * F1_NB;                    // 20
    constexpr int PER_WARP = (ITEMS + 7) / 8;           // 3
    float fw[PER_WARP][NFFT / 32];
#pragma unroll
    for (int q = 0; q < PER_WARP; ++q) {
        const int item = warp + 8 * q;
        const int fb = f0 - 1 + item / 2, ri = item & 1;
        const bool live = item < ITEMS && fb >= 0 && fb < NF;
#pragma unroll
        for (int u = 0; u < NFFT / 32; ++u) fw[q][u] = live ? __ldg(w.wat + (lane + 32 * u) * 196 + ri * NF + fb) : 0.f;
    }
    __syncthreads();
    griddep_wait();
    const StateHeader* hdr = reinterpret_cast<const StateHeader*>(state);
    float* st = stream_rec(state, recs, b);
    const int par = rec_par(st);
    const float* cb = st + ST_CONV + par * (2 * 4 * NF);
    float* cb_next = st + ST_CONV + (par ^ 1) * (2 * 4 * NF);
    // samples of the frame: x[s0 .. s0 + 191] (zero past the end: the look-ahead padding of net.py:8-18,56-58)
    const int s0 = pos_rel ? (int)(hdr->pos - hdr->clip_base) * HOP : 0;
    const int xl = row_len(recs, b, 1, x_len, LOOKAHEAD);
    for (int i = tid; i < NMIC * NFFT; i += 256) {
        const int m = i / NFFT, n = i % NFFT, sidx = s0 + n;
        xs[m][n] = (sidx < xl) ? x[(int64_t)b * x_bstride + (int64_t)m * x_cstride + sidx] : 0.f;
    }
    // the two history frames of the conv come from the tails the previous call left
    for (int i = tid; i < 2 * 4 * F1_NB; i += 256) {
        const int fr = i / (4 * F1_NB), c = (i / F1_NB) % 4, sl = i % F1_NB, fb = f0 - 1 + sl;
        U[fr][c][sl] = (fb >= 0 && fb < NF) ? cb[(fr * 4 + c) * NF + fb] : 0.f;
    }
    __syncthreads();
    trace_.mark(0);
    // spectrum of this frame for the CTA's bins: channels [Re m0, Re m1, Im m0, Im m1]
#pragma unroll
    for (int q = 0; q < PER_WARP; ++q) {
        const int item = warp + 8 * q;
        if (item < ITEMS) {
            float a0 = 0.f, a1 = 0.f;
#pragma unroll
            for (int u = 0; u < NFFT / 32; ++u) {
                a0 = fmaf(fw[q][u], xs[0][lane + 32 * u], a0);
                a1 = fmaf(fw[q][u], xs[1][lane + 32 * u], a1);
            }
            a0 = warp_sum(a0); a1 = warp_sum(a1);
            if (lane == 0) {
                const int sl = item / 2, ri = item & 1;
                U[2][ri * 2 + 0][sl] = a0;              // zero for bins outside 0..96 (their filter values were zeroed)
                U[2][ri * 2 + 1][sl] = a1;
            }
        }
    }
    __syncthreads();
    trace_.mark(1);
    // conv: X[f][o] = b_o + sum_{c,i,j} Wc[o][c][i][j] * U[i][c][f-1+j]   (slot of bin f-1+j = (f - f0) + j)
    {
        float acc0 = bc, acc1 = bc;
#pragma unroll
        for (int c = 0; c < 4; ++c)
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
                for (int j = 0; j < 3; ++j) {
                    acc0 = fmaf(wr[c * 9 + i * 3 + j], U[i][c][fq + j], acc0);
                    acc1 = fmaf(wr[c * 9 + i * 3 + j], U[i][c][fq + 4 + j], acc1);
                }
        const bool ok0 = fq < nr, ok1 = fq + 4 < nr;
        xrows[fq * 64 + o] = ok0 ? acc0 : 0.f;
        xrows[(fq + 4) * 64 + o] = ok1 ? acc1 : 0.f;
        float* xr = X + ((int64_t)b * NF + f0) * 64;
        if (ok0) xr[fq * 64 + o] = acc0;
        if (ok1) xr[(fq + 4) * 64 + o] = acc1;
    }
    // next conv tails = spectrogram rows of frames t-1, t (own bins)
    if (stream_active(recs, active, b)) {
        for (int i = tid; i < 2 * 4 * nr; i += 256) {
            const int fr = i / (4 * nr), c = (i / nr) % 4, r = i % nr;
            cb_next[(fr * 4 + c) * NF + f0 + r] = U[1 + fr][c][1 + r];
        }
    }
    __syncthreads();
    trace_.mark(2);
    mbar_wait(&gbar, 0);
    ih_rows_tile(xrows, xn, wih, gg0, gg1, gb0, gb1, gbias, GX + ((int64_t)b * NF + f0) * 512, nr, tid);
}

// the dense forms (call row b = record b); the `_t<Records>` forms serve slot-list calls (l2h_sep_forward_slots)
constexpr auto tail_kernel = tail_kernel_t<int64_t>;
constexpr auto front1_kernel = front1_kernel_t<int64_t>;

}  // namespace l2h
