// lstm_rec: the serial part of every LSTM in both networks (hidden size 64).
//
// The input projection W_ih x + b_ih + b_hh for all steps is a rows_gemm done beforehand
// ("gx", gate columns packed as j*4 + q with q in {i,f,g,o}: thread tid of this kernel owns
// column tid).  What is left is, per step, a 256x64 mat-vec with W_hh, the cell update and
// one barrier -- a latency chain.  One CTA (128 threads: hidden unit x k-half) runs NSEQ independent
// sequences in lock-step with its W_hh slice in registers and h broadcast through shared memory; the
// FMAs are paired (float2) along k.  lstm_rec3_kernel: few sequences (latency), lstm_rec4_kernel: many
// sequences, the step written stage by stage across the CTA's sequences (throughput).
//
// Row addressing (rows of gx / out are activation rows of the [B,T,F,C] tensors):
//   seq -> (o = seq / inner_count, i = seq % inner_count)
//   row(seq, s) = o*outer_stride + i*inner_stride + s*step_stride
// intra (along F): inner_count=1, outer_stride=F(+pad), step_stride=1
// inter (along T): inner_count=F, outer_stride=T*F, inner_stride=1, step_stride=F
//
// Reference semantics: torch.nn.LSTM cell, gate order i,f,g,o
// (tfgridnet_causal.py:336-346, used :512 and :529).
#pragma once
#include <cstdlib>
#include "common.cuh"

namespace l2h {

struct LstmArgs {
    const float* gx;       // rows x gx_ld; direction d uses columns [d*256, d*256+256)
    int64_t gx_ld;
    float* out;            // rows x out_ld; direction d writes columns [d*64, d*64+64)
    int64_t out_ld;
    const float* whh;      // [ndir][256 (j*4+q)][64]
    float* h_state;        // carried state (read at start, written at end) or null; one direction only (ndir == 1):
    float* c_state;        //   element (seq, j) at (seq/inner_count)*hc_outer_stride + (seq%inner_count)*64 + j
    int64_t hc_outer_stride;
    int nseq, L;
    int inner_count;
    int64_t outer_stride, inner_stride, step_stride;
    // rows of `out` may follow a different (e.g. zero-padded) layout; all zero => same as gx rows
    int64_t out_outer_stride, out_inner_stride, out_step_stride;
    int ndir;              // 1 or 2; direction 1 runs the steps in reverse
};

// PRE = true: the whole input projection of the sequence (L x 1 KB) is brought in up front by TMA bulk
// copies (one per step row) -- no per-step async bookkeeping at all; used when it fits (short L).
// PRE = false: 8-stage cp.async ring refilled four rows (one group) at a time.
constexpr int L3_STAGES = 8;

template <int NSEQ, bool PRE>
__global__ void __launch_bounds__(128, PRE ? 1 : 2)
lstm_rec3_kernel(const LstmArgs a) {
    extern __shared__ __align__(16) float gdyn[];            // PRE: [NSEQ][L][256]
    __shared__ __align__(16) float hbuf[2][NSEQ][64];
    __shared__ __align__(16) float gring[PRE ? 1 : L3_STAGES][PRE ? 1 : NSEQ][PRE ? 4 : 256];
    __shared__ __align__(8) unsigned long long gbar;

    TraceScope trace_(TK_LSTM, a.gx);
    griddep_launch();
    const int tid = threadIdx.x;
    const int dir = blockIdx.y;
    const int seq0 = blockIdx.x * NSEQ;
    const int j = tid >> 1, kh = tid & 1;

    float2 w[4][16];                      // rows j*4+q, k in [32 kh, 32 kh + 32)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float4* wp = reinterpret_cast<const float4*>(a.whh + ((int64_t)dir * 256 + j * 4 + q) * 64 + 32 * kh);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float4 t = __ldg(wp + k);
            w[q][2 * k] = make_float2(t.x, t.y);
            w[q][2 * k + 1] = make_float2(t.z, t.w);
        }
    }
    if (PRE && tid == 0) { mbar_init(&gbar, 1); mbar_fence_init(); }
    __syncthreads();
    griddep_wait();

    const bool own_out = (a.out_outer_stride | a.out_inner_stride | a.out_step_stride) != 0;
    const int64_t o_step = (own_out ? a.out_step_stride : a.step_stride) * a.out_ld;
    const int sgn = (dir == 0) ? 1 : -1;
    const int first = (dir == 0) ? 0 : a.L - 1;
    const int64_t g_step = a.step_stride * a.gx_ld * sgn;

    float c[NSEQ];
    bool valid[NSEQ];
    float* outp[NSEQ];
    int64_t hc[NSEQ];
    const float* grow[NSEQ];              // &gx[row(seq, first)][dir*256]
#pragma unroll
    for (int s = 0; s < NSEQ; ++s) {
        const int seq = seq0 + s;
        valid[s] = seq < a.nseq;
        const int sq = valid[s] ? seq : 0;
        const int so = sq / a.inner_count, si = sq % a.inner_count;
        const int64_t gb = (int64_t)so * a.outer_stride + (int64_t)si * a.inner_stride;
        const int64_t ob = own_out ? (int64_t)so * a.out_outer_stride + (int64_t)si * a.out_inner_stride : gb;
        grow[s] = a.gx + (gb + (int64_t)first * a.step_stride) * a.gx_ld + dir * 256;
        outp[s] = a.out + ob * a.out_ld + (int64_t)first * o_step + dir * 64 + j;
        hc[s] = (int64_t)so * a.hc_outer_stride + (int64_t)si * 64 + j;
        c[s] = (a.c_state != nullptr && valid[s]) ? a.c_state[hc[s]] : 0.f;
        if (kh == 0) hbuf[0][s][j] = (a.h_state != nullptr && valid[s]) ? a.h_state[hc[s]] : 0.f;
    }

    if (PRE) {
        // one 1 KB bulk copy per (sequence, step): row of iteration `it` lands at gdyn[s][it][:]
        int nrows = 0;
#pragma unroll
        for (int s = 0; s < NSEQ; ++s) nrows += valid[s] ? a.L : 0;
        if (tid == 0) mbar_expect_tx(&gbar, (unsigned)nrows * 1024u);
        __syncthreads();
#pragma unroll
        for (int s = 0; s < NSEQ; ++s)
            if (valid[s])
                for (int it = tid; it < a.L; it += 128)
                    tma_load_1d(gdyn + ((int64_t)s * a.L + it) * 256, grow[s] + (int64_t)it * g_step, 1024, &gbar);
        mbar_wait(&gbar, 0);
    }
    // ring refill: group g = rows 4g .. 4g+3 -> stages (g % 2)*4 .. +3 ; 64 x 16 B chunks per row
    auto issue_group = [&](int g) {
        if (!PRE) {
#pragma unroll
            for (int s = 0; s < NSEQ; ++s) {
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const int idx = tid + 128 * u, r = idx >> 6, chunk = idx & 63;
                    const int it = 4 * g + r;
                    if (valid[s] && it < a.L)
                        cp_async16(&gring[(g % 2) * 4 + r][s][chunk * 4], grow[s] + (int64_t)it * g_step + chunk * 4);
                }
            }
            cp_async_commit();
        }
    };
    if (!PRE) {
        issue_group(0);
        cp_async_wait<0>();
    }
    __syncthreads();

    const float LOG2E = 1.4426950408889634f;
    const float S0 = kh ? -2.f * LOG2E : -LOG2E, A0 = kh ? 2.f : 1.f, B0 = kh ? -1.f : 0.f;
    trace_.mark(0);

    int cur = 0;
    for (int it = 0; it < a.L; ++it) {
        if (!PRE && (it & 3) == 0) issue_group((it >> 2) + 1);      // overwrites the group consumed 4 steps ago
#pragma unroll
        for (int s = 0; s < NSEQ; ++s) {
            const float* gr = PRE ? gdyn + ((int64_t)s * a.L + it) * 256 : &gring[it % L3_STAGES][s][0];
            const float2 g2 = *reinterpret_cast<const float2*>(gr + j * 4 + 2 * kh);   // this lane adds gx of gates 2kh, 2kh+1
            const float4* hp = reinterpret_cast<const float4*>(&hbuf[cur][s][32 * kh]);
            float2 acc[4][2];
#pragma unroll
            for (int q = 0; q < 4; ++q) { acc[q][0] = make_float2(0.f, 0.f); acc[q][1] = make_float2(0.f, 0.f); }
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float4 h4 = hp[k];
                const float2 hA = make_float2(h4.x, h4.y), hB = make_float2(h4.z, h4.w);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    acc[q][0] = ffma2(w[q][2 * k], hA, acc[q][0]);
                    acc[q][1] = ffma2(w[q][2 * k + 1], hB, acc[q][1]);
                }
            }
            float p[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float gadd = ((q >> 1) == kh) ? ((q & 1) ? g2.y : g2.x) : 0.f;
                const float t = ((acc[q][0].x + acc[q][0].y) + (acc[q][1].x + acc[q][1].y)) + gadd;
                p[q] = t + __shfl_xor_sync(0xffffffffu, t, 1);
            }
            // lane kh = 0 activates (i, f); lane kh = 1 activates (g, o)
            const float x0 = kh ? p[2] : p[0], x1 = kh ? p[3] : p[1];
            const float v0 = __fdividef(A0, 1.f + ex2_ftz(S0 * x0)) + B0;
            const float v1 = __fdividef(1.f, 1.f + ex2_ftz(-LOG2E * x1));
            const float og = __shfl_xor_sync(0xffffffffu, v0, 1);
            const float oo = __shfl_xor_sync(0xffffffffu, v1, 1);
            c[s] = v1 * c[s] + v0 * og;                  // meaningful on kh == 0 lanes: f*c + i*g
            const float h = oo * (__fdividef(2.f, 1.f + ex2_ftz(-2.f * LOG2E * c[s])) - 1.f);
            if (kh == 0) {
                hbuf[cur ^ 1][s][j] = h;
                if (valid[s]) *outp[s] = h;
            }
            outp[s] += sgn * o_step;
        }
        cur ^= 1;
        if (!PRE && (it & 3) == 3) cp_async_wait<0>();    // the next four rows (issued 4 steps ago) have landed
        __syncthreads();
    }
    trace_.mark(1);
    if (a.h_state != nullptr) {
#pragma unroll
        for (int s = 0; s < NSEQ; ++s) {
            if (valid[s] && kh == 0) {
                a.h_state[hc[s]] = hbuf[cur][s][j];
                a.c_state[hc[s]] = c[s];
            }
        }
    }
}

// ---- variant 4: variant 3's thread layout, throughput mode --------------------------------------
// With many sequences per CTA, variant 3's time per (sequence, step) does not fall with the number of sequences
// the CTA holds: 214-226 registers leave the
// scheduler no room to overlap the sequences' dependent chains.  Here the step is written stage by stage
// ACROSS the CTA's sequences (all dot products, then all reductions, then all activations) with one
// accumulator pair per gate, so NSEQ independent chains are in flight at every stage.
template <int NSEQ>
__global__ void __launch_bounds__(128, 2)
lstm_rec4_kernel(const LstmArgs a) {
    __shared__ __align__(16) float hbuf[2][NSEQ][64];
    extern __shared__ __align__(16) float gring[];          // [L3_STAGES][NSEQ][256]

    griddep_launch();
    const int tid = threadIdx.x;
    const int dir = blockIdx.y;
    const int seq0 = blockIdx.x * NSEQ;
    const int j = tid >> 1, kh = tid & 1;

    float2 w[4][16];                      // rows j*4+q, k in [32 kh, 32 kh + 32)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float4* wp = reinterpret_cast<const float4*>(a.whh + ((int64_t)dir * 256 + j * 4 + q) * 64 + 32 * kh);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float4 t = __ldg(wp + k);
            w[q][2 * k] = make_float2(t.x, t.y);
            w[q][2 * k + 1] = make_float2(t.z, t.w);
        }
    }
    griddep_wait();

    const bool own_out = (a.out_outer_stride | a.out_inner_stride | a.out_step_stride) != 0;
    const int64_t o_step = (own_out ? a.out_step_stride : a.step_stride) * a.out_ld;
    const int sgn = (dir == 0) ? 1 : -1;
    const int first = (dir == 0) ? 0 : a.L - 1;
    const int64_t g_step = a.step_stride * a.gx_ld * sgn;

    float c[NSEQ];
    bool valid[NSEQ];
    float* outp[NSEQ];
    int64_t hc[NSEQ];
    const float* grow[NSEQ];
#pragma unroll
    for (int s = 0; s < NSEQ; ++s) {
        const int seq = seq0 + s;
        valid[s] = seq < a.nseq;
        const int sq = valid[s] ? seq : 0;
        const int so = sq / a.inner_count, si = sq % a.inner_count;
        const int64_t gb = (int64_t)so * a.outer_stride + (int64_t)si * a.inner_stride;
        const int64_t ob = own_out ? (int64_t)so * a.out_outer_stride + (int64_t)si * a.out_inner_stride : gb;
        grow[s] = a.gx + (gb + (int64_t)first * a.step_stride) * a.gx_ld + dir * 256;
        outp[s] = a.out + ob * a.out_ld + (int64_t)first * o_step + dir * 64 + j;
        hc[s] = (int64_t)so * a.hc_outer_stride + (int64_t)si * 64 + j;
        c[s] = (a.c_state != nullptr && valid[s]) ? a.c_state[hc[s]] : 0.f;
        if (kh == 0) hbuf[0][s][j] = (a.h_state != nullptr && valid[s]) ? a.h_state[hc[s]] : 0.f;
    }
    auto issue_group = [&](int g) {       // rows 4g .. 4g+3 -> stages (g % 2)*4 .. +3 ; 64 x 16 B chunks per row
#pragma unroll
        for (int s = 0; s < NSEQ; ++s) {
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int idx = tid + 128 * u, r = idx >> 6, chunk = idx & 63;
                const int it = 4 * g + r;
                if (valid[s] && it < a.L)
                    cp_async16(&gring[(((g % 2) * 4 + r) * NSEQ + s) * 256 + chunk * 4], grow[s] + (int64_t)it * g_step + chunk * 4);
            }
        }
        cp_async_commit();
    };
    issue_group(0);
    cp_async_wait<0>();
    __syncthreads();

    const float LOG2E = 1.4426950408889634f;
    const float S0 = kh ? -2.f * LOG2E : -LOG2E, A0 = kh ? 2.f : 1.f, B0 = kh ? -1.f : 0.f;

    int cur = 0;
    for (int it = 0; it < a.L; ++it) {
        if ((it & 3) == 0) issue_group((it >> 2) + 1);              // overwrites the group consumed 4 steps ago
        // stage A: all dot products (4 NSEQ independent FMA-pair chains)
        float2 acc[NSEQ][4];
        float2 g2[NSEQ];
#pragma unroll
        for (int s = 0; s < NSEQ; ++s) {
            g2[s] = *reinterpret_cast<const float2*>(&gring[((it % L3_STAGES) * NSEQ + s) * 256 + j * 4 + 2 * kh]);
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[s][q] = make_float2(0.f, 0.f);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float4 h4[NSEQ];
#pragma unroll
            for (int s = 0; s < NSEQ; ++s) h4[s] = *reinterpret_cast<const float4*>(&hbuf[cur][s][32 * kh + 4 * k]);
#pragma unroll
            for (int s = 0; s < NSEQ; ++s) {
                const float2 hA = make_float2(h4[s].x, h4[s].y);
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[s][q] = ffma2(w[q][2 * k], hA, acc[s][q]);
            }
#pragma unroll
            for (int s = 0; s < NSEQ; ++s) {
                const float2 hB = make_float2(h4[s].z, h4[s].w);
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[s][q] = ffma2(w[q][2 * k + 1], hB, acc[s][q]);
            }
        }
        // stage B: k-half reduction; lane kh adds gx of gates 2kh, 2kh+1
        float p[NSEQ][4];
#pragma unroll
        for (int s = 0; s < NSEQ; ++s) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float gadd = ((q >> 1) == kh) ? ((q & 1) ? g2[s].y : g2[s].x) : 0.f;
                p[s][q] = (acc[s][q].x + acc[s][q].y) + gadd;
            }
        }
#pragma unroll
        for (int s = 0; s < NSEQ; ++s) {
#pragma unroll
            for (int q = 0; q < 4; ++q) p[s][q] += __shfl_xor_sync(0xffffffffu, p[s][q], 1);
        }
        // stage C: lane kh = 0 activates (i, f); lane kh = 1 activates (g, o)
        float v0[NSEQ], v1[NSEQ], e0[NSEQ], e1[NSEQ];
#pragma unroll
        for (int s = 0; s < NSEQ; ++s) {
            e0[s] = ex2_ftz(S0 * (kh ? p[s][2] : p[s][0]));
            e1[s] = ex2_ftz(-LOG2E * (kh ? p[s][3] : p[s][1]));
        }
#pragma unroll
        for (int s = 0; s < NSEQ; ++s) {
            v0[s] = __fdividef(A0, 1.f + e0[s]) + B0;
            v1[s] = __fdividef(1.f, 1.f + e1[s]);
        }
        float og[NSEQ], oo[NSEQ];
#pragma unroll
        for (int s = 0; s < NSEQ; ++s) {
            og[s] = __shfl_xor_sync(0xffffffffu, v0[s], 1);
            oo[s] = __shfl_xor_sync(0xffffffffu, v1[s], 1);
        }
        float ec[NSEQ];
#pragma unroll
        for (int s = 0; s < NSEQ; ++s) {
            c[s] = v1[s] * c[s] + v0[s] * og[s];        // meaningful on kh == 0 lanes: f*c + i*g
            ec[s] = ex2_ftz(-2.f * LOG2E * c[s]);
        }
#pragma unroll
        for (int s = 0; s < NSEQ; ++s) {
            const float h = oo[s] * (__fdividef(2.f, 1.f + ec[s]) - 1.f);
            if (kh == 0) {
                hbuf[cur ^ 1][s][j] = h;
                if (valid[s]) *outp[s] = h;
            }
            outp[s] += sgn * o_step;
        }
        cur ^= 1;
        if ((it & 3) == 3) cp_async_wait<0>();          // the next four rows (issued 4 steps ago) have landed
        __syncthreads();
    }
    if (a.h_state != nullptr) {
#pragma unroll
        for (int s = 0; s < NSEQ; ++s) {
            if (valid[s] && kh == 0) {
                a.h_state[hc[s]] = hbuf[cur][s][j];
                a.c_state[hc[s]] = c[s];
            }
        }
    }
}

constexpr size_t lstm_rec4_smem(int nseq) { return (size_t)L3_STAGES * nseq * 256 * sizeof(float); }

inline cudaError_t configure_lstm() {
    cudaError_t e = cudaFuncSetAttribute(lstm_rec3_kernel<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    return e;
}

// the state slot of a sequence has no direction term: a bidirectional call with carried state would have both
// directions read and write the same (h, c)
inline bool lstm_state_ok(const LstmArgs& a) {
    return (a.ndir == 1 || a.ndir == 2) && (a.h_state == nullptr || a.ndir == 1) && ((a.h_state == nullptr) == (a.c_state == nullptr));
}

// `form_nseq` > 0: choose the kernel (and its sequences per CTA) as for that many sequences, so that a call over a subset of
// a larger batch runs exactly the arithmetic the whole batch would (sep_engine.cu: block 0 of a targets call)
inline cudaError_t launch_lstm_rec(const LstmArgs& a, cudaStream_t st, bool pdl = false, int form_nseq = 0) {
    if (a.nseq <= 0 || a.L <= 0 || !lstm_state_ok(a)) return cudaErrorInvalidValue;
    const int fseq = form_nseq > 0 ? form_nseq : a.nseq;
    const int ctas1 = fseq * a.ndir;
    if (ctas1 <= NUM_SMS && (size_t)a.L * 1024 <= 200 * 1024)      // latency mode: one sequence per CTA, preloaded
        return launch_k(pdl, lstm_rec3_kernel<1, true>, dim3(a.nseq, a.ndir), dim3(128), (size_t)a.L * 1024, st, a);
    // many sequences: NSEQ per CTA in lock-step (stage by stage), at most 4: more sequences per CTA only while one sequence
    // per CTA (resp. two) would not fit the device in one wave.  (Six per CTA would need 226 registers; not kept.)
    static int wave1[64] = {}, wave2[64] = {};
    int per = 1;
    if ((int64_t)fseq * a.ndir > resident_ctas(wave1, lstm_rec3_kernel<1, false>, 128, 0)) {
        per = 2;
        if ((int64_t)((fseq + 1) / 2) * a.ndir > resident_ctas(wave2, lstm_rec4_kernel<2>, 128, lstm_rec4_smem(2))) per = 4;
    }
    dim3 grid((a.nseq + per - 1) / per, a.ndir);
    if (per == 2) return launch_k(pdl, lstm_rec4_kernel<2>, grid, dim3(128), lstm_rec4_smem(2), st, a);   // many sequences: stage by stage
    if (per == 4) return launch_k(pdl, lstm_rec4_kernel<4>, grid, dim3(128), lstm_rec4_smem(4), st, a);
    return launch_k(pdl, lstm_rec3_kernel<1, false>, grid, dim3(128), 0, st, a);
}

}  // namespace l2h
