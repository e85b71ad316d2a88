// How fast can ONE CTA stage a contiguous block from (L2-resident) global memory into shared memory?
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/copy_microbench tools/copy_microbench.cu
#include <cstdio>
#include "../lookoncetohear_b200/csrc/common.cuh"
using namespace l2h;

template <int MODE>
__global__ void __launch_bounds__(256) copy_kernel(const float* __restrict__ src, float* __restrict__ out, int bytes, int reps) {
    extern __shared__ __align__(128) float sm[];
    __shared__ __align__(8) unsigned long long bar;
    const int tid = threadIdx.x;
    if (tid == 0) { mbar_init(&bar, 1); mbar_fence_init(); }
    __syncthreads();
    float acc = 0.f;
    unsigned phase = 0;
    for (int r = 0; r < reps; ++r) {
        if (MODE == 0) {            // one bulk copy
            if (tid == 0) { mbar_expect_tx(&bar, bytes); tma_load_1d(sm, src, bytes, &bar); }
            mbar_wait(&bar, phase); phase ^= 1;
        } else if (MODE == 1) {     // 2 KB bulk copies from all threads
            if (tid == 0) mbar_expect_tx(&bar, bytes);
            __syncthreads();
            tma_load_split(sm, src, bytes, &bar, tid, 256);
            mbar_wait(&bar, phase); phase ^= 1;
        } else if (MODE == 2) {     // LDG.128 -> STS.128 loop
            for (int i = tid; i < bytes / 16; i += 256) reinterpret_cast<float4*>(sm)[i] = __ldg(reinterpret_cast<const float4*>(src) + i);
        } else if (MODE == 3) {     // cp.async 16 B, all in flight
            for (int i = tid; i < bytes / 16; i += 256) cp_async16(reinterpret_cast<float4*>(sm) + i, reinterpret_cast<const float4*>(src) + i);
            cp_async_commit(); cp_async_wait<0>();
        } else if (MODE == 4) {     // LDG.128 x8 batched -> STS
            for (int i0 = tid; i0 < bytes / 16; i0 += 256 * 8) {
                float4 v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) { const int i = i0 + 256 * u; v[u] = (i < bytes / 16) ? __ldg(reinterpret_cast<const float4*>(src) + i) : make_float4(0, 0, 0, 0); }
#pragma unroll
                for (int u = 0; u < 8; ++u) { const int i = i0 + 256 * u; if (i < bytes / 16) reinterpret_cast<float4*>(sm)[i] = v[u]; }
            }
        }
        __syncthreads();
        acc += sm[(tid * 37 + r) % (bytes / 4)];
        __syncthreads();
    }
    out[tid] = acc;
}

template <int MODE>
void run(const char* name, const float* src, float* out, int bytes) {
    cudaFuncSetAttribute(copy_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    const int reps = 200;
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    copy_kernel<MODE><<<1, 256, bytes>>>(src, out, bytes, 10);
    cudaDeviceSynchronize();
    cudaEventRecord(a);
    copy_kernel<MODE><<<1, 256, bytes>>>(src, out, bytes, reps);
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    printf("%-34s %7d B  %7.2f us/copy  %7.1f GB/s  (%s)\n", name, bytes, 1e3f * ms / reps, bytes / (1e6f * ms / reps) , cudaGetErrorString(cudaGetLastError()));
}

int main() {
    float *src, *out; cudaMalloc(&src, 1 << 20); cudaMalloc(&out, 4096); cudaMemset(src, 0, 1 << 20);
    for (int bytes : {24832, 75776, 150528}) {
        run<0>("one cp.async.bulk", src, out, bytes);
        run<1>("2 KB cp.async.bulk x N threads", src, out, bytes);
        run<2>("LDG.128 -> STS.128 loop", src, out, bytes);
        run<3>("cp.async 16 B, all in flight", src, out, bytes);
        run<4>("LDG.128 x8 batched -> STS", src, out, bytes);
    }
    return 0;
}
