// Probe: can a 16-CTA (non-portable) cluster with ~226 KB of shared memory per CTA be scheduled, and what do a
// cluster barrier and a DSMEM gather cost at that size?   nvcc -gencode arch=compute_90a,code=sm_90a -o cluster16_probe cluster16_probe.cu
#include <cooperative_groups.h>
#include <cstdio>
#include <cuda_runtime.h>
namespace cg = cooperative_groups;

__global__ void __launch_bounds__(256) probe(unsigned long long* out, int iters) {
    extern __shared__ float sm[];
    cg::cluster_group cl = cg::this_cluster();
    const int rk = cl.block_rank(), n = cl.num_blocks();
    sm[threadIdx.x] = (float)(rk * 1000 + threadIdx.x);
    cl.sync();
    unsigned long long t0, t1, t2;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (int i = 0; i < iters; ++i) cl.sync();
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    float acc = 0.f;
    for (int i = 0; i < iters; ++i) {
        for (int p = 0; p < n; ++p) acc += cl.map_shared_rank(sm, p)[(threadIdx.x + i) & 255];
        cl.sync();
    }
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t2));
    if (threadIdx.x == 0 && rk == 0) { out[0] = t1 - t0; out[1] = t2 - t1; out[2] = (unsigned long long)acc; }
    cl.sync();
}

int main() {
    for (int csz : {8, 16}) {
        for (size_t smem : {(size_t)64 * 1024, (size_t)226 * 1024}) {
            cudaFuncSetAttribute(probe, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            cudaFuncSetAttribute(probe, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
            cudaLaunchConfig_t cfg{};
            cfg.gridDim = dim3(csz); cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = smem;
            cudaLaunchAttribute at[1];
            at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = csz; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
            cfg.attrs = at; cfg.numAttrs = 1;
            int ncl = -1;
            cudaError_t e = cudaOccupancyMaxActiveClusters(&ncl, probe, &cfg);
            unsigned long long* d; cudaMalloc(&d, 64);
            const int iters = 200;
            cudaError_t le = cudaLaunchKernelEx(&cfg, probe, d, iters);
            cudaError_t se = cudaDeviceSynchronize();
            unsigned long long h[3] = {0, 0, 0};
            cudaMemcpy(h, d, 24, cudaMemcpyDeviceToHost);
            printf("cluster %2d smem %3zu KB: occupancy query %s -> %d clusters; launch %s, sync %s; cluster.sync %.0f ns; gather(%d peers)+sync %.0f ns\n",
                   csz, smem / 1024, cudaGetErrorString(e), ncl, cudaGetErrorString(le), cudaGetErrorString(se), (double)h[0] / iters, csz, (double)h[1] / iters);
            cudaFree(d);
            cudaGetLastError();
        }
    }
    return 0;
}
