// tc_lstm: the LSTM recurrence for MANY sequences on the tensor cores (throughput regime: offline batches,
// enrollment; the few-sequence latency regime keeps lstm.cuh's CUDA-core kernels).
//
// Per step and direction the recurrent product is gates^T[256 x NS] = W_hh[256 x 64] . h^T[64 x NS]: "swap-AB" --
// the 256 gate rows are the MMA's M dimension (four M = 64 wgmma tiles, W_hh bf16 hi/lo resident in shared memory for
// the CTA's whole life), the CTA's NS = 32 sequences are its N dimension.  Products are bf16x3 split
// (W_hi h_hi + W_lo h_hi + W_hi h_lo; `passes` = 2 drops the W_lo term for the bf16 configuration, `passes` = 1 keeps
// only W_hi h_hi: plain bf16), accumulators in the
// registers of the CTA's single warpgroup.  A step:
//   1. wgmma of the four gate tiles (48 MMAs of N = 32); meanwhile the input projection gx of this step is in flight
//      (loaded at the end of the previous step; coalesced float4: the four gates of a unit are adjacent columns);
//   2. the accumulators go to a padded shared-memory exchange tile [sequence][gate column];
//   3. thread (warp w, lane l) owns the (sequence n = w + 4k, unit j = l + 32jj) pairs: the four gate pre-activations of
//      a pair are one float4 of the tile; activations, cell update (c in registers), h out as fp32 rows (the layer's
//      output) and as bf16 hi/lo into the K-major SWIZZLE_128B h^T operand tile of the next step.
// Two CTAs per SM overlap one CTA's MMAs with the other's element-wise work.
// Reference semantics: torch.nn.LSTM cell, gate order i,f,g,o (tfgridnet_causal.py:336-346, :512, :529).
//
// With FX (tc_lstm_x, separator, 64 input channels) the INPUT PROJECTION is inside too:
//     gates^T = W_ih . LN(x_t)^T + W_hh . h^T + b
// so the [rows x 512] projection never exists in HBM.  W_ih hi/lo planes sit next to W_hh in shared memory; during the
// cell stage of step s the threads LayerNorm the 32 input rows of step s+1 (4 threads per row, prefetched one further
// step ahead) and split them to bf16 hi/lo into the x^T operand tile.
#pragma once
#include "lstm.cuh"
#include "umma_ptx.cuh"

namespace l2h {
namespace tcl {

constexpr int NS = 32;                 // sequences per CTA (= MMA N)
constexpr int NTHREADS = 128;          // one warpgroup
constexpr int XLD = 260;               // padded row of the exchange tile (words): conflict-free fragment stores, 16-byte aligned rows
constexpr size_t W_BYTES = 2 * 256 * 128;                    // hi + lo planes, 256 rows x 128 B
constexpr size_t H_BYTES = 2 * NS * 128;                     // h^T (or x^T) hi + lo
constexpr size_t X_BYTES = (size_t)NS * XLD * 4;             // [NS][XLD]
constexpr size_t SMEM = 1024 + W_BYTES + H_BYTES + X_BYTES;
constexpr size_t XSMEM = 1024 + 2 * W_BYTES + 2 * H_BYTES + X_BYTES;

struct LstmXArgs {
    LstmArgs l;                       // gx / gx_ld unused with the projection inside; row addressing, out, whh, state
    const float* x;                   // [rows][x_ld] input activations (row addressing = l's strides)
    long long x_ld;
    const __nv_bfloat16* wih_hi;      // [ndir*256 (dir*256 + j*4+q)][64] K-major bf16 planes (the GEMM's B operand planes)
    const __nv_bfloat16* wih_lo;
    const float* bias;                // [ndir*256]  b_ih + b_hh
    const float* ln_g;                // [64] LayerNorm over the input channels (nn.LayerNorm semantics)
    const float* ln_b;
    // or null: [outer index] device step counts (an entry outside [0, L] counts as 0).  Steps s >= steps[o] of the
    // sequences of outer index o get gates i = -inf, f = +inf, g = 0, so c passes through them unchanged and the final c
    // is the one steps[o] steps leave (one direction: the separator's inter LSTM in ragged slot-list calls)
    const int32_t* steps;
};

L2H_DEVINL float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
constexpr float LOG2E = 1.4426950408889634f;
L2H_DEVINL float sigm(float x) { return rcp_approx(1.f + ex2_ftz(-LOG2E * x)); }
L2H_DEVINL float tanh_g(float x) { return fmaf(2.f, rcp_approx(1.f + ex2_ftz(-2.f * LOG2E * x)), -1.f); }

// element (row n, k = j) of a K-major SWIZZLE_128B [NS][64] operand tile, as bf16 hi and lo planes
L2H_DEVINL void put_split(unsigned base, int n, int j, float v) {
    const __nv_bfloat16 hh = __float2bfloat16_rn(v);
    const __nv_bfloat16 hl = __float2bfloat16_rn(v - __bfloat162float(hh));
    const unsigned off = base + (unsigned)n * 128u + ((((unsigned)j >> 3) ^ (unsigned)(n & 7)) << 4) + ((unsigned)j & 7u) * 2u;
    asm volatile("st.shared.b16 [%0], %1;" ::"r"(off), "h"(*reinterpret_cast<const unsigned short*>(&hh)) : "memory");
    asm volatile("st.shared.b16 [%0], %1;" ::"r"(off + NS * 128), "h"(*reinterpret_cast<const unsigned short*>(&hl)) : "memory");
}

template <bool FX, bool STEPS = false>
static __global__ void __launch_bounds__(NTHREADS, FX ? 1 : 2)
tc_lstm_kernel(const LstmXArgs xa, int passes) {
    const LstmArgs& a = xa.l;
    extern __shared__ uint8_t smem_raw[];
    __shared__ long long in_row[NS], out_row[NS], hc_off[NS];
    __shared__ int n_steps[STEPS ? NS : 1];       // STEPS: the sequence's own step count (LstmXArgs::steps)
    __shared__ float lng[64], lnb[64];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int dir = blockIdx.y, seq0 = blockIdx.x * NS;
    const unsigned sm0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const unsigned whh_sm = sm0, wih_sm = sm0 + (unsigned)W_BYTES;
    const unsigned h_sm = sm0 + (unsigned)((FX ? 2 : 1) * W_BYTES), x_sm = h_sm + (unsigned)H_BYTES;
    float* xt = reinterpret_cast<float*>(smem_raw + (sm0 - smem_u32(smem_raw)) + (FX ? 2 * (W_BYTES + H_BYTES) : W_BYTES + H_BYTES));
    griddep_launch();
    // sequence -> first row of gx / x / out (in rows), state offset; -1: no such sequence
    const bool same_out = (a.out_outer_stride | a.out_inner_stride | a.out_step_stride) == 0;
    const long long o_outer = same_out ? a.outer_stride : a.out_outer_stride, o_inner = same_out ? a.inner_stride : a.out_inner_stride;
    const long long o_step = same_out ? a.step_stride : a.out_step_stride;
    if (tid < NS) {
        const int seq = seq0 + tid;
        if (seq < a.nseq) {
            const long long o = seq / a.inner_count, i = seq % a.inner_count;
            in_row[tid] = o * a.outer_stride + i * a.inner_stride;
            out_row[tid] = o * o_outer + i * o_inner;
            hc_off[tid] = o * a.hc_outer_stride + i * 64;
            if constexpr (STEPS) {
                const int k = xa.steps[o];
                n_steps[tid] = (unsigned)k <= (unsigned)a.L ? k : 0;
            }
        } else {
            in_row[tid] = -1; out_row[tid] = -1; hc_off[tid] = -1;
            if constexpr (STEPS) n_steps[tid] = 0;
        }
    }
    if (FX && tid < 64) { lng[tid] = __ldg(xa.ln_g + tid); lnb[tid] = __ldg(xa.ln_b + tid); }
    // W_hh of this direction: fp32 [256 (j*4+q)][64] -> bf16 hi/lo, K-major SWIZZLE_128B rows; W_ih: the bf16 planes the
    // tensor-core GEMM uses, copied into the same layout (weights only: before the dependency wait)
    for (int row = tid; row < 256; row += NTHREADS) {
        const float4* src = reinterpret_cast<const float4*>(a.whh + ((size_t)dir * 256 + row) * 64);
        const unsigned dst = whh_sm + (unsigned)row * 128u;
#pragma unroll
        for (unsigned c = 0; c < 8; ++c) {
            const float4 v0 = __ldg(src + 2 * c), v1 = __ldg(src + 2 * c + 1);
            const float f[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
            unsigned hi[4], lo[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const __nv_bfloat162 h2 = __floats2bfloat162_rn(f[2 * e], f[2 * e + 1]);
                hi[e] = *reinterpret_cast<const unsigned*>(&h2);
                const float2 hf = __bfloat1622float2(h2);
                lo[e] = umma::pack_bf16x2(f[2 * e] - hf.x, f[2 * e + 1] - hf.y);
            }
            const unsigned sw = (c ^ (unsigned)(row & 7)) << 4;
            asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(dst + sw), "r"(hi[0]), "r"(hi[1]), "r"(hi[2]), "r"(hi[3]) : "memory");
            asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(dst + sw + 256 * 128), "r"(lo[0]), "r"(lo[1]), "r"(lo[2]), "r"(lo[3]) : "memory");
            if (FX) {
                const uint4 wh = __ldg(reinterpret_cast<const uint4*>(xa.wih_hi + ((size_t)dir * 256 + row) * 64) + c);
                const uint4 wl = __ldg(reinterpret_cast<const uint4*>(xa.wih_lo + ((size_t)dir * 256 + row) * 64) + c);
                const unsigned dsti = wih_sm + (unsigned)row * 128u + sw;
                asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(dsti), "r"(wh.x), "r"(wh.y), "r"(wh.z), "r"(wh.w) : "memory");
                asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(dsti + 256 * 128), "r"(wl.x), "r"(wl.y), "r"(wl.z), "r"(wl.w) : "memory");
            }
        }
    }
    __syncthreads();
    griddep_wait();

    const long long sgn = dir ? -1 : 1;
    long long st = dir ? (long long)(a.L - 1) : 0;
    // input rows (FX): thread (xn = tid / 4, xq = tid % 4) handles channels 16 xq .. 16 xq + 15 of sequence xn
    const int xn = tid >> 2, xq = tid & 3;
    float xv[16];
    auto load_x = [&](long long step) {
        const long long row = in_row[xn];
        if (row >= 0 && step >= 0 && step < a.L) {
            const float4* p = reinterpret_cast<const float4*>(xa.x + (row + step * a.step_stride) * xa.x_ld + 16 * xq);
#pragma unroll
            for (int i = 0; i < 4; ++i) { const float4 v = __ldg(p + i); xv[4 * i] = v.x; xv[4 * i + 1] = v.y; xv[4 * i + 2] = v.z; xv[4 * i + 3] = v.w; }
        } else {
#pragma unroll
            for (int i = 0; i < 16; ++i) xv[i] = 0.f;
        }
    };
    auto put_x = [&]() {                      // LayerNorm over the 64 channels (4 lanes), split, store K-major swizzled
        float sum = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) sum += xv[i];
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        const float mu = sum * (1.f / 64.f);
        float qq = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) { const float d = xv[i] - mu; qq = fmaf(d, d, qq); }
        qq += __shfl_xor_sync(0xffffffffu, qq, 1);
        qq += __shfl_xor_sync(0xffffffffu, qq, 2);
        const float rs = rsqrtf(qq * (1.f / 64.f) + 1e-5f);
        unsigned hi[8], lo[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int c0 = 16 * xq + 2 * e;
            const float y0 = fmaf((xv[2 * e] - mu) * rs, lng[c0], lnb[c0]), y1 = fmaf((xv[2 * e + 1] - mu) * rs, lng[c0 + 1], lnb[c0 + 1]);
            const __nv_bfloat162 h2 = __floats2bfloat162_rn(y0, y1);
            hi[e] = *reinterpret_cast<const unsigned*>(&h2);
            const float2 hf = __bfloat1622float2(h2);
            lo[e] = umma::pack_bf16x2(y0 - hf.x, y1 - hf.y);
        }
        const unsigned base = x_sm + (unsigned)xn * 128u;
#pragma unroll
        for (unsigned c = 0; c < 2; ++c) {    // 16-byte chunks 2 xq + c of row xn
            const unsigned off = base + (((2u * (unsigned)xq + c) ^ (unsigned)(xn & 7)) << 4);
            asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(off), "r"(hi[4 * c]), "r"(hi[4 * c + 1]), "r"(hi[4 * c + 2]), "r"(hi[4 * c + 3]) : "memory");
            asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(off + NS * 128), "r"(lo[4 * c]), "r"(lo[4 * c + 1]), "r"(lo[4 * c + 2]), "r"(lo[4 * c + 3]) : "memory");
        }
    };
    // gx of a step for this thread's pairs (the four gates of a unit are adjacent columns j*4 + q)
    float4 g_in[8][2];
    auto load_gx = [&](long long step) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const long long row = in_row[warp + 4 * k];
#pragma unroll
            for (int jj = 0; jj < 2; ++jj)
                g_in[k][jj] = row >= 0 ? __ldg(reinterpret_cast<const float4*>(a.gx + (row + step * a.step_stride) * a.gx_ld + dir * 256 + 4 * (lane + 32 * jj)))
                                       : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    float4 bias4[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
    if (FX) {
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) bias4[jj] = __ldg(reinterpret_cast<const float4*>(xa.bias + dir * 256) + lane + 32 * jj);
    }

    // initial state
    float c[8][2];
#pragma unroll
    for (int k = 0; k < 8; ++k)
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
            const int n = warp + 4 * k, j = lane + 32 * jj;
            float h0 = 0.f, c0 = 0.f;
            if (a.h_state != nullptr && hc_off[n] >= 0) { h0 = a.h_state[hc_off[n] + j]; c0 = a.c_state[hc_off[n] + j]; }
            c[k][jj] = c0;
            put_split(h_sm, n, j, h0);
        }
    if (FX) { load_x(st); put_x(); load_x(st + sgn); }
    else load_gx(st);
    fence_proxy_async();                       // generic-proxy operand writes -> visible to the tensor core
    __syncthreads();

    for (int s = 0; s < a.L; ++s) {
        float acc[4][16];
        umma::wg_fence();
#pragma unroll
        for (int mt = 0; mt < 4; ++mt) {
#pragma unroll
            for (int part = FX ? 0 : 1; part < 2; ++part) {             // 0: W_ih . x^T, 1: W_hh . h^T
                const unsigned wb = (part == 0 ? wih_sm : whh_sm) + (unsigned)mt * 8192u;
                const unsigned bb = part == 0 ? x_sm : h_sm;
                const unsigned long long w_hi = umma::smem_desc(wb, 16, 1024), w_lo = umma::smem_desc(wb + 256 * 128, 16, 1024);
                const unsigned long long b_hi = umma::smem_desc(bb, 16, 1024), b_lo = umma::smem_desc(bb + NS * 128, 16, 1024);
                for (int ps = 0; ps < 3; ++ps) {
                    if (ps == 1 && passes < 3) continue;            // W_lo term only for the fp32-grade split
                    if (ps == 2 && passes < 2) continue;            // h_lo / x_lo term: not for plain bf16
                    const unsigned long long da = (ps == 1) ? w_lo : w_hi, db = (ps == 2) ? b_lo : b_hi;
#pragma unroll
                    for (unsigned kk = 0; kk < 4; ++kk)
                        umma::wgmma_bf16<32, 0>(acc[mt], da + kk * 2, db + kk * 2, (part != (FX ? 0 : 1) || ps != 0 || kk != 0) ? 1 : 0);
                }
            }
        }
        umma::wg_commit();
        umma::wg_wait<0>();
#pragma unroll
        for (int mt = 0; mt < 4; ++mt) {
            umma::wg_fence_regs(acc[mt]);
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int pcol = mt * 64 + 16 * warp + (lane >> 2) + 8 * (e >> 1), n = 8 * i + 2 * (lane & 3) + (e & 1);
                    xt[n * XLD + pcol] = acc[mt][4 * i + e];
                }
        }
        __syncthreads();                       // every MMA of the step is complete, the exchange tile is written
        if (FX && s + 1 < a.L) {               // operand tile of step s+1, then the rows of step s+2
            put_x();
            load_x(st + 2 * sgn);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k)
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
                const int n = warp + 4 * k, j = lane + 32 * jj;
                float4 g = *reinterpret_cast<const float4*>(xt + n * XLD + 4 * j);     // i, f, g, o
                const float4 add = FX ? bias4[jj] : g_in[k][jj];
                g.x += add.x; g.y += add.y; g.z += add.z; g.w += add.w;
                if constexpr (STEPS) {
                    if (st >= n_steps[n]) { g.x = -INFINITY; g.y = INFINITY; g.z = 0.f; }
                }
                const float cc = sigm(g.y) * c[k][jj] + sigm(g.x) * tanh_g(g.z);
                c[k][jj] = cc;
                const float h = sigm(g.w) * (__fdividef(2.f, 1.f + ex2_ftz(-2.f * LOG2E * cc)) - 1.f);
                const long long orow = out_row[n];
                if (orow >= 0) a.out[(orow + st * o_step) * a.out_ld + dir * 64 + j] = h;
                put_split(h_sm, n, j, h);
                if (s + 1 == a.L && a.h_state != nullptr && hc_off[n] >= 0) {
                    a.h_state[hc_off[n] + j] = h;
                    a.c_state[hc_off[n] + j] = cc;
                }
            }
        if (!FX && s + 1 < a.L) load_gx(st + sgn);      // in flight during the next step's MMAs
        fence_proxy_async();
        __syncthreads();                       // h^T (and x^T) of step s+1 complete; the exchange tile is free again
        st += sgn;
    }
}

}  // namespace tcl

// (static: every translation unit that includes this header owns its copy of the kernel and configures it itself)
static inline cudaError_t configure_tc_lstm() {
    cudaError_t e = cudaFuncSetAttribute(tcl::tc_lstm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tcl::SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tcl::tc_lstm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tcl::XSMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tcl::tc_lstm_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tcl::XSMEM);
    return e;
}
// ... with the input projection (and its LayerNorm) inside
static inline cudaError_t launch_tc_lstm_x(const tcl::LstmXArgs& xa, int passes, cudaStream_t st, bool pdl = false) {
    if (xa.l.nseq <= 0 || xa.l.L <= 0 || !lstm_state_ok(xa.l) || passes < 1 || passes > 3) return cudaErrorInvalidValue;
    if ((xa.x_ld & 3) != 0 || (reinterpret_cast<uintptr_t>(xa.x) & 15) != 0 || (reinterpret_cast<uintptr_t>(xa.bias) & 15) != 0)
        return cudaErrorInvalidValue;
    if (xa.steps != nullptr && xa.l.ndir != 1) return cudaErrorInvalidValue;
    dim3 grid((xa.l.nseq + tcl::NS - 1) / tcl::NS, xa.l.ndir);
    if (xa.steps != nullptr) return launch_k(pdl, tcl::tc_lstm_kernel<true, true>, grid, dim3(tcl::NTHREADS), tcl::XSMEM, st, xa, passes);
    return launch_k(pdl, tcl::tc_lstm_kernel<true>, grid, dim3(tcl::NTHREADS), tcl::XSMEM, st, xa, passes);
}
// many sequences: the recurrence on the tensor cores
static inline cudaError_t launch_tc_lstm(const LstmArgs& a, int passes, cudaStream_t st, bool pdl = false) {
    if (a.nseq <= 0 || a.L <= 0 || !lstm_state_ok(a) || passes < 1 || passes > 3) return cudaErrorInvalidValue;
    if ((a.gx_ld & 3) != 0 || (reinterpret_cast<uintptr_t>(a.gx) & 15) != 0) return cudaErrorInvalidValue;   // float4 gate loads
    tcl::LstmXArgs xa{};
    xa.l = a;
    dim3 grid((a.nseq + tcl::NS - 1) / tcl::NS, a.ndir);
    return launch_k(pdl, tcl::tc_lstm_kernel<false>, grid, dim3(tcl::NTHREADS), tcl::SMEM, st, xa, passes);
}

}  // namespace l2h
