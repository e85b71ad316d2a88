// Shared device helpers for the lookonce engine (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace l2h {

#define L2H_DEVINL __device__ __forceinline__

// SMs of an H100 SXM: the grid size of the persistent and work-splitting kernels (a smaller part only queues a wave)
constexpr int NUM_SMS = 132;

// ---- d.xy = a.xy * b.xy + c.xy: two fp32 FMAs (Hopper has no packed fp32 FMA; the kernels keep their pairwise form) ----
L2H_DEVINL float2 ffma2(float2 a, float2 b, float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

L2H_DEVINL float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
L2H_DEVINL float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Block-wide sum for blockDim.x <= 1024 (red must hold 32 floats). All threads get the result.
L2H_DEVINL float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();                 // protect red from a previous use
    if (lane == 0) red[warp] = v;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    float t = (lane < nw) ? red[lane] : 0.f;
    t = warp_sum(t);
    return t;
}

// sigmoid / tanh through ex2.approx + rcp.approx (abs err ~1e-7; MUFU.TANH's 5e-4 is too coarse
// for the 1e-3 rel-L2 gate across 97 recurrent steps x 3 blocks).
L2H_DEVINL float fast_sigmoid(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
L2H_DEVINL float fast_tanh(float x) { return 2.f * __fdividef(1.f, 1.f + __expf(-2.f * x)) - 1.f; }

// 2^x, flush-to-zero (plain ex2.approx carries extra denormal-range fix-up instructions)
L2H_DEVINL float ex2_ftz(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

L2H_DEVINL float prelu(float x, float a) { return x >= 0.f ? x : a * x; }

// cp.async 16 B (LDGSTS)
L2H_DEVINL void cp_async16(void* smem, const void* gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem));
}
L2H_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
L2H_DEVINL void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

// ---- TMA bulk copy (cp.async.bulk, SASS UBLKCP) + mbarrier: one instruction stages a whole
// contiguous tile (weights, a frame's rows) in shared memory at full L2 bandwidth, instead of a
// latency-bound LDG->STS loop.  Addresses and sizes must be multiples of 16 bytes.
L2H_DEVINL unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
L2H_DEVINL void mbar_init(unsigned long long* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
L2H_DEVINL void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
L2H_DEVINL void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
L2H_DEVINL void tma_load_1d(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// Stage a contiguous block with ONE bulk copy issued by thread 0 (fewer instructions and barrier arrivals than a
// loop of smaller bulk copies or an LDG.128 -> STS.128 loop).
// Called by all threads (uniform call sites); the caller arms the barrier with the byte total.
L2H_DEVINL void tma_load_split(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar,
                               int tid, int /*nthreads*/) {
    if (tid == 0) tma_load_1d(dst_smem, src_gmem, bytes, bar);
}
// order earlier generic-proxy accesses of shared memory before later async-proxy (TMA) writes to it
L2H_DEVINL void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
L2H_DEVINL void mbar_wait(unsigned long long* bar, unsigned phase) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}" ::"r"(smem_u32(bar)), "r"(phase) : "memory");
}

// Programmatic dependent launch (PDL): a kernel launched with the programmatic-serialization
// attribute may start while its predecessor drains; griddep_wait() blocks until the predecessor
// grid has completed and flushed.  Every kernel of a chain calls griddep_launch() first (lets the
// successor's CTAs become resident early and run their weight-only prologue) and griddep_wait()
// before touching anything an earlier kernel wrote -- on every path, so completion stays
// transitive.  Both are no-ops for launches without the attribute.
L2H_DEVINL void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
L2H_DEVINL void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

}  // namespace l2h

#include <utility>
namespace l2h {

// ---- pipeline tracing (diagnostics; off unless the host sets g_trace) ---------------------------------------
// Thread 0 of CTA (0,0,0) of an instrumented kernel records %globaltimer at entry and at exit, the SM it ran on, a
// kernel id and the low bits of one activation pointer (every hop owns a workspace slot, so the pointer says which
// hop the launch belongs to).  tools/pipe_trace.py turns the records into a per-stage timeline of the pipelined graph.
struct TraceRec { unsigned long long t0, t1; unsigned long long ptr; unsigned int kernel, sm; };
static __device__ TraceRec* g_trace = nullptr;
static __device__ unsigned int g_trace_cap = 0;
static __device__ unsigned int g_trace_n = 0;
enum TraceKernel { TK_FRONT = 0, TK_GEMM, TK_LSTM, TK_MID_A, TK_MID_B, TK_MID_C, TK_QKV, TK_ATTN, TK_ATTN_OUT, TK_BACK, TK_MID, TK_TAIL };
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
struct TraceScope {
    TraceRec* rec;
    __device__ __forceinline__ TraceScope(int kernel, const void* ptr) : rec(nullptr) {
        if ((threadIdx.x | blockIdx.x | blockIdx.y | blockIdx.z) == 0 && g_trace != nullptr) {
            const unsigned int slot = atomicAdd(&g_trace_n, 1u);
            if (slot < g_trace_cap) {
                rec = g_trace + slot;
                unsigned int sm;
                asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
                rec->ptr = (unsigned long long)ptr; rec->kernel = (unsigned int)kernel; rec->sm = sm; rec->t1 = 0;
                unsigned long long* m = marks();
                for (int p = 0; p < TRACE_MARKS; ++p) m[p] = 0ull;
                rec->t0 = globaltimer_ns();
            }
        }
    }
    __device__ __forceinline__ ~TraceScope() {
        if (rec != nullptr) {
            rec->t1 = globaltimer_ns();
            // time stamps taken inside the kernel: one more record each (id 100 + 20 * kernel + point), slots reserved at once
            unsigned long long* m = marks();
            unsigned int cnt = 0;
            for (int p = 0; p < TRACE_MARKS; ++p) cnt += (m[p] != 0ull) ? 1u : 0u;
            if (cnt != 0u) {
                unsigned int slot = atomicAdd(&g_trace_n, cnt);
                for (int p = 0; p < TRACE_MARKS; ++p) {
                    if (m[p] == 0ull) continue;
                    if (slot < g_trace_cap) {
                        TraceRec* r = g_trace + slot;
                        r->ptr = rec->ptr; r->kernel = 100u + (unsigned int)TRACE_MARKS * rec->kernel + (unsigned int)p; r->sm = rec->sm; r->t0 = r->t1 = m[p];
                    }
                    ++slot;
                }
            }
        }
    }
    static constexpr int TRACE_MARKS = 20;
    static __device__ __forceinline__ unsigned long long* marks() {
        __shared__ unsigned long long m[TRACE_MARKS];
        return m;
    }
    // a time stamp inside the kernel (the recording thread only; kept in shared memory until the kernel ends)
    __device__ __forceinline__ void mark(int point) {
        if (rec != nullptr) marks()[point] = globaltimer_ns();
    }
};

// How many CTAs of `kernel` (with `threads` threads and `smem` bytes of dynamic shared memory) the CURRENT device holds
// at once: occupancy per SM x SM count, cached per device in `cache` (one array per call site, 0 = not asked yet).  The
// one-wave limit of the persistent and work-splitting launches: a persistent grid larger than this runs a second wave.
template <typename... KArgs>
inline int resident_ctas(int (&cache)[64], void (*kernel)(KArgs...), int threads, size_t smem) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) { cudaGetLastError(); return NUM_SMS; }
    if (cache[dev] == 0) {
        int sms = 0, per = 0;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = NUM_SMS;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, kernel, threads, smem) != cudaSuccess || per <= 0) per = 1;
        cudaGetLastError();
        cache[dev] = per * sms;
    }
    return cache[dev];
}

// every kernel launch the engines issue goes through launch_k / launch_cluster / umma::launch: this counter makes the
// "kernels launched" figure of the C ABI exact for directly launched chains (graph replays count their kernel nodes)
inline thread_local long long g_launches = 0;

// host: launch with (or without) the PDL attribute
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(bool pdl, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                            Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    ++g_launches;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// same, as thread-block clusters of `cluster` CTAs (distributed shared memory between them)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_cluster(bool pdl, dim3 cluster, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                  cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cluster.x; attr[0].val.clusterDim.y = cluster.y; attr[0].val.clusterDim.z = cluster.z;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 2 : 1;
    ++g_launches;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
}  // namespace l2h
