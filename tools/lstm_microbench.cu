// Micro-benchmark of LSTM recurrence step variants (one CTA = one sequence, one direction).
// Build:  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/lstm_microbench tools/lstm_microbench.cu
// Prints ns per recurrent step for each variant (timing only; E* variants change the math).
#include <cstdio>
#include <vector>
#include "../lookoncetohear_b200/csrc/lstm.cuh"
using namespace l2h;

// experimental copy of variant 1 with switches
template <bool RING, bool STG, bool TANHC, bool ACT, bool BAR8>
__global__ void __launch_bounds__(256, 2)
exp_kernel(const float* __restrict__ gx, float* __restrict__ out, const float* __restrict__ whh, int L) {
    __shared__ __align__(16) float hbuf[2][64];
    __shared__ __align__(16) float gs[8][256];
    const int tid = threadIdx.x, j = tid >> 2, q = tid & 3;
    float2 w[32];
    const float4* wp = reinterpret_cast<const float4*>(whh + (int64_t)tid * 64);
#pragma unroll
    for (int k = 0; k < 16; ++k) { const float4 t = __ldg(wp + k); w[2*k] = make_float2(t.x, t.y); w[2*k+1] = make_float2(t.z, t.w); }
    if (q == 0) hbuf[0][j] = 0.f;
    float c = 0.f;
    auto issue = [&](int it) {
        if (RING) { if (tid < 64 && it < L) cp_async16(&gs[it % 8][tid * 4], gx + (int64_t)it * 256 + tid * 4); cp_async_commit(); }
    };
    if (RING) { for (int it = 0; it < 8 - 1; ++it) issue(it); cp_async_wait<8 - 2>(); }
    __syncthreads();
    const float S = (q == 2) ? -2.f * 1.4426950408889634f : -1.4426950408889634f;
    const float Aa = (q == 2) ? 2.f : 1.f, Bc = (q == 2) ? -1.f : 0.f;
    const int qbase = (tid & 31) & ~3;
    int cur = 0;
    float* op = out + j;
    for (int it = 0; it < L; ++it) {
        issue(it + 8 - 1);
        const float g0 = RING ? gs[it % 8][tid] : 0.01f * (float)(tid & 7);
        const float4* hp = reinterpret_cast<const float4*>(&hbuf[cur][0]);
        float2 a0 = make_float2(g0, 0.f), a1 = make_float2(0.f, 0.f), a2 = a1, a3 = a1;
#pragma unroll
        for (int k = 0; k < 16; k += 2) {
            const float4 h4 = hp[k], h5 = hp[k + 1];
            a0 = ffma2(w[2*k], make_float2(h4.x, h4.y), a0); a1 = ffma2(w[2*k+1], make_float2(h4.z, h4.w), a1);
            a2 = ffma2(w[2*k+2], make_float2(h5.x, h5.y), a2); a3 = ffma2(w[2*k+3], make_float2(h5.z, h5.w), a3);
        }
        const float pre = ((a0.x + a0.y) + (a1.x + a1.y)) + ((a2.x + a2.y) + (a3.x + a3.y));
        const float act = ACT ? __fdividef(Aa, 1.f + ex2_ftz(S * pre)) + Bc : pre * 0.01f;
        const float gi = __shfl_sync(0xffffffffu, act, qbase + 0), gf = __shfl_sync(0xffffffffu, act, qbase + 1);
        const float gg = __shfl_sync(0xffffffffu, act, qbase + 2), go = __shfl_sync(0xffffffffu, act, qbase + 3);
        c = gf * c + gi * gg;
        const float h = TANHC ? go * (__fdividef(2.f, 1.f + ex2_ftz(-2.f * 1.4426950408889634f * c)) - 1.f) : go * c * 0.5f;
        if (q == 0) { hbuf[cur ^ 1][j] = h; if (STG) *op = h; }
        op += 128;
        cur ^= 1;
        if (RING) cp_async_wait<8 - 2>();
        if (BAR8) __syncthreads();
        else asm volatile("bar.sync 1, 256;");
    }
    if (!STG && q == 0) out[j] = hbuf[cur][j] + c;
}

template <typename F>
float time_it(F f, int iters = 20) {
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    f(); f(); cudaDeviceSynchronize();
    cudaEventRecord(a);
    for (int i = 0; i < iters; ++i) f();
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    return ms / iters;
}

int main() {
    const int L = 970;
    float *gx, *out, *whh;
    cudaMalloc(&gx, (size_t)L * 512 * 4); cudaMalloc(&out, (size_t)L * 128 * 4 + 4096); cudaMalloc(&whh, 2 * 256 * 64 * 4);
    std::vector<float> hw(2 * 256 * 64), hg((size_t)L * 512);
    for (size_t i = 0; i < hw.size(); ++i) hw[i] = 0.05f * (float)((int)(i * 2654435761u % 200) - 100) / 100.f;
    for (size_t i = 0; i < hg.size(); ++i) hg[i] = 0.5f * (float)((int)(i * 40503u % 200) - 100) / 100.f;
    cudaMemcpy(whh, hw.data(), hw.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(gx, hg.data(), hg.size() * 4, cudaMemcpyHostToDevice);
    LstmArgs a{};
    a.gx = gx; a.gx_ld = 512; a.out = out; a.out_ld = 128; a.whh = whh; a.nseq = 1; a.L = L; a.inner_count = 1;
    a.outer_stride = L; a.inner_stride = 0; a.step_stride = 1; a.ndir = 2;
    auto rep = [&](const char* name, float ms) { printf("%-46s %8.1f ns/step\n", name, 1e6f * ms / L); };
    rep("v3 lstm_rec3_kernel<1,ring> (128 thr, unit x k-half)", time_it([&] { lstm_rec3_kernel<1, false><<<dim3(1, 2), 128>>>(a); }));
    {
        cudaFuncSetAttribute(lstm_rec3_kernel<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        LstmArgs b = a; b.L = 194; b.outer_stride = 194;
        float ms = time_it([&] { lstm_rec3_kernel<1, true><<<dim3(1, 2), 128, 194 * 1024>>>(b); });
        printf("%-46s %8.1f ns/step (L=194, incl. preload + launch)\n", "v3 lstm_rec3_kernel<1,preload>", 1e6f * ms / 194);
        b.L = 97; b.outer_stride = 97;
        ms = time_it([&] { lstm_rec3_kernel<1, true><<<dim3(1, 2), 128, 97 * 1024>>>(b); });
        printf("%-46s %8.2f us per launch (L=97, both directions)\n", "v3 preload, the T=1 intra launch", 1e3f * ms);
    }
    a.nseq = 4;  a.outer_stride = L / 4; a.L = L / 4;
    { float ms = time_it([&] { lstm_rec3_kernel<4, false><<<dim3(1, 2), 128>>>(a); }); printf("%-46s %8.1f ns/step (4 seqs in lock-step)\n", "v3 NSEQ=4", 1e6f * ms / (L / 4)); }
    rep("exp: full (ring, stg, tanh, act, bar0)", time_it([&] { exp_kernel<true, true, true, true, true><<<1, 256>>>(gx, out, whh, L); }));
    rep("exp: no ring (gx const)", time_it([&] { exp_kernel<false, true, true, true, true><<<1, 256>>>(gx, out, whh, L); }));
    rep("exp: no per-step STG", time_it([&] { exp_kernel<true, false, true, true, true><<<1, 256>>>(gx, out, whh, L); }));
    rep("exp: no tanh(c) MUFUs", time_it([&] { exp_kernel<true, true, false, true, true><<<1, 256>>>(gx, out, whh, L); }));
    rep("exp: no gate MUFUs", time_it([&] { exp_kernel<true, true, true, false, true><<<1, 256>>>(gx, out, whh, L); }));
    rep("exp: no MUFU at all", time_it([&] { exp_kernel<true, true, false, false, true><<<1, 256>>>(gx, out, whh, L); }));
    rep("exp: nothing but FMA+shfl+bar", time_it([&] { exp_kernel<false, false, false, false, true><<<1, 256>>>(gx, out, whh, L); }));
    rep("exp: full with named barrier", time_it([&] { exp_kernel<true, true, true, true, false><<<1, 256>>>(gx, out, whh, L); }));
    printf("%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
