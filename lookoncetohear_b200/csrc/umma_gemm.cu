// umma_gemm.cu: the wgmma GEMM kernel (umma_gemm.cuh) and its host side -- tensor maps (cuTensorMapEncodeTiled
// through the runtime's driver entry point, so the library does not link libcuda), shared-memory plan, launch.
#include "umma_host.cuh"
#include "umma_kernel.cuh"

namespace l2h {
namespace umma {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            f = nullptr;
        return reinterpret_cast<EncodeTiledFn>(f);
    }();
    return fn;
}

// 4-D tiled map with 128-byte swizzle; dims/strides in ELEMENTS (stride[0] is implicit 1), zero fill out of range
inline cudaError_t make_tmap4(CUtensorMap* m, CUtensorMapDataType dt, int elem_bytes, const void* base, const int64_t dims[4],
                              const int64_t strides[4], const int box[4]) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return cudaErrorNotSupported;
    cuuint64_t d[4], s[3];
    cuuint32_t b[4], es[4] = {1, 1, 1, 1};
    for (int i = 0; i < 4; ++i) { d[i] = (cuuint64_t)std::max<int64_t>(1, dims[i]); b[i] = (cuuint32_t)box[i]; }
    for (int i = 1; i < 4; ++i) {
        s[i - 1] = (cuuint64_t)strides[i] * elem_bytes;
        if (d[i] == 1 && s[i - 1] == 0) s[i - 1] = (cuuint64_t)16;        // size-1 dims still need a legal stride
        if (s[i - 1] % 16 != 0) return cudaErrorInvalidValue;
    }
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return cudaErrorInvalidValue;
    const CUresult r = fn(m, dt, 4, const_cast<void*>(base), d, s, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

// column tile: 64 for N <= 64, else 128 (the wgmma shapes the kernel is built for; the accumulators of a 64 x 128 tile
// are 64 registers per thread).  Columns beyond N are zero-filled by TMA and never stored.
inline int pick_bn(int N) { return N <= 64 ? 64 : 128; }

constexpr size_t SMEM_LIMIT = 227 * 1024 - 2048;      // dynamic shared memory budget (static barriers etc. come on top)
constexpr size_t EPI_BYTES = 8 * 2048;                // epilogue transpose buffers

cudaError_t configure() {
    static thread_local int done_dev = -1;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (done_dev == dev) return cudaSuccess;
    for (auto k : {umma_gemm_kernel<64, 0>, umma_gemm_kernel<64, 1>, umma_gemm_kernel<128, 0>, umma_gemm_kernel<128, 1>})
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_LIMIT);
    if (e == cudaSuccess) done_dev = dev;
    return e;
}

inline int sm_count() {
    static thread_local int n = 0, ndev = -1;
    int dev = 0;
    cudaGetDevice(&dev);
    if (ndev != dev) { cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); ndev = dev; }
    return n > 0 ? n : 132;
}

struct Plan { int BN, resident, nstg, nop; size_t smem; bool ok; };

// shared-memory plan for a column tile of BN: resident weight slab when it fits next to two staging slots and two
// A operand slots (small K), else A and B stream through a ring of operand slots together
inline Plan plan_for(const GemmDesc& g, int BN) {
    Plan pl{BN, 0, 2, 0, 0, false};
    const int planes_a = g.passes > 1 ? 2 : 1, planes = g.passes > 2 ? 2 : 1;
    const size_t opA = (size_t)planes_a * OPA_PLANE;
    const size_t opB = (size_t)planes * (g.b.mn_major ? (size_t)((BN + 63) / 64) * 8192 : (size_t)BN * 128);
    const size_t fixed = 1024 + EPI_BYTES;
    if (!g.b_by_seq && fixed + 2 * STG_BYTES + 2 * opA + (size_t)g.n_chunks * opB <= SMEM_LIMIT) {
        pl.resident = 1;
        const size_t left = SMEM_LIMIT - fixed - 2 * STG_BYTES - (size_t)g.n_chunks * opB;
        pl.nop = (int)std::min<size_t>(4, left / opA);
        pl.smem = fixed + 2 * STG_BYTES + (size_t)pl.nop * opA + (size_t)g.n_chunks * opB;
        pl.ok = true;
        return pl;
    }
    const size_t op = opA + opB;
    int nop = (int)((SMEM_LIMIT - fixed - 2 * STG_BYTES) / op);
    if (nop < 2) { pl.nstg = 1; nop = (int)((SMEM_LIMIT - fixed - STG_BYTES) / op); }
    pl.nop = std::min(nop, 4);
    pl.smem = fixed + (size_t)pl.nstg * STG_BYTES + (size_t)pl.nop * op;
    pl.ok = nop >= 1;
    return pl;
}

// what launch() decides before it encodes the tensor maps: tile shape, shared-memory plan, persistent grid, epilogue width
struct LaunchPlan { Plan pl; int P_TILE, S_TILE, n_tiles_n, grid, vec_ok; long long m_tiles; };

// null, or why the problem cannot be launched
inline const char* plan_launch(const GemmDesc& g, LaunchPlan& L) {
    {   // rows per tile = P_TILE positions x S_TILE sequences: pick the shape that wastes the fewest of the 128 rows
        const bool flat = g.a0.n_outer == 1 && (!g.a1.base || g.a1.n_outer == 1) && !g.b_by_seq;
        const int cand[3][2] = {{BM, 1}, {std::min(g.rows_per_seq, BM), std::max(1, BM / std::max(1, std::min(g.rows_per_seq, BM)))}, {1, BM}};
        double best = -1.0;
        for (int i = 0; i < 3; ++i) {
            const int P = cand[i][0], S = cand[i][1];
            if (S > 1 && !flat) continue;
            const long long pt = (g.rows_per_seq + P - 1) / P, stl = (g.nseq + S - 1) / S;
            const double eff = (double)g.rows_per_seq * g.nseq / ((double)pt * stl * BM);
            if (eff > best + 1e-9) { best = eff; L.P_TILE = P; L.S_TILE = S; }
        }
    }
    Plan pl = plan_for(g, pick_bn(g.N));
    if ((!pl.ok || (!pl.resident && pl.nop < 2)) && pl.BN > 64) pl = plan_for(g, 64);   // keep two operand slots
    if (!pl.ok) return "operand tile does not fit shared memory";
    L.pl = pl;
    L.n_tiles_n = (g.N + pl.BN - 1) / pl.BN;
    const int p_tiles = (g.rows_per_seq + L.P_TILE - 1) / L.P_TILE, s_tiles = (g.nseq + L.S_TILE - 1) / L.S_TILE;
    L.m_tiles = (long long)p_tiles * s_tiles;
    if (L.m_tiles * L.n_tiles_n > 0x7fffffff) return "too many tiles";
    // persistent grid: `groups` CTAs per column tile, every group member gets the same number of row tiles (+-1)
    const int sms = sm_count();
    long long groups = std::max(1, sms / L.n_tiles_n);
    groups = std::min(groups, L.m_tiles);
    const long long per = (L.m_tiles + groups - 1) / groups;
    groups = (L.m_tiles + per - 1) / per;
    L.grid = (int)groups * L.n_tiles_n;
    // float4 epilogue accesses: C / R rows and the per-column operands 16-byte aligned
    L.vec_ok = (g.ldc % 4 == 0 && g.c_seq_stride % 4 == 0 && g.c_inner_stride % 4 == 0 && (reinterpret_cast<uintptr_t>(g.C) & 15) == 0 &&
                (reinterpret_cast<uintptr_t>(g.R) & 15) == 0 && (reinterpret_cast<uintptr_t>(g.bias) & 15) == 0 &&
                (reinterpret_cast<uintptr_t>(g.prelu_vec) & 15) == 0) ? 1 : 0;
    return nullptr;
}

cudaError_t launch(const GemmDesc& g, cudaStream_t st, std::string* why) {
    auto bad = [&](const char* m) { if (why) *why = m; return cudaErrorInvalidValue; };
    if (g.n_chunks <= 0 || g.n_chunks > MAX_CHUNKS) return bad("k-chunk count");
    if (g.N <= 0 || g.rows_per_seq <= 0 || g.nseq <= 0) return bad("empty problem");
    if (g.passes < 1 || g.passes > 3) return bad("passes must be 1, 2 or 3");
    if (g.prelu && g.prelu_vec) return bad("scalar and vector PReLU slopes are exclusive");
    LaunchPlan lp;
    if (const char* m = plan_launch(g, lp)) return bad(m);
    const Plan& pl = lp.pl;
    cudaError_t e = configure();
    if (e != cudaSuccess) return e;
    Params p;
    memset(&p, 0, sizeof(p));
    memcpy(p.chunks, g.chunks, sizeof(KChunk) * g.n_chunks);
    p.n_chunks = g.n_chunks;
    p.P_TILE = lp.P_TILE; p.S_TILE = lp.S_TILE;
    p.rows_per_seq = g.rows_per_seq; p.nseq = g.nseq;
    p.seq_inner = (int)g.a0.n_inner;
    p.pos_bias = g.pos_bias;
    p.N = g.N; p.BN = pl.BN; p.n_tiles_n = lp.n_tiles_n;
    p.passes = g.passes; p.b_mn_major = g.b.mn_major ? 1 : 0; p.b_by_seq = g.b_by_seq ? 1 : 0;
    p.b_resident = pl.resident; p.nstg = pl.nstg; p.nop = pl.nop;
    const size_t smem = pl.smem;
    const int planes = g.passes > 2 ? 2 : 1;      // B planes the tensor map exposes
    // ---- tensor maps ----
    {
        const int tile_box[4] = {32, p.P_TILE, p.S_TILE, 1};
        const ASource* srcs[2] = {&g.a0, g.a1.base ? &g.a1 : &g.a0};
        CUtensorMap* maps[2] = {&p.tmA0, &p.tmA1};
        for (int i = 0; i < 2; ++i) {
            const ASource& a = *srcs[i];
            const int64_t dims[4] = {a.channels, a.n_pos, a.n_inner, a.n_outer};
            const int64_t strides[4] = {1, a.pos_stride, a.inner_stride, a.outer_stride};
            e = make_tmap4(maps[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, a.base, dims, strides, tile_box);
            if (e != cudaSuccess) return bad("A tensor map");
        }
        const BPlanes& b = g.b;
        if (!b.mn_major) {
            const int64_t dims[4] = {g.K, g.N, b.nz, planes};
            const int64_t strides[4] = {1, b.ld, b.z_stride, b.plane_stride};
            const int box[4] = {KC, p.BN, 1, 1};
            e = make_tmap4(&p.tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, b.base, dims, strides, box);
        } else {
            const int64_t dims[4] = {g.N, g.K, b.nz, planes};
            const int64_t strides[4] = {1, b.ld, b.z_stride, b.plane_stride};
            const int box[4] = {64, KC, 1, 1};
            e = make_tmap4(&p.tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, b.base, dims, strides, box);
        }
        if (e != cudaSuccess) return bad("B tensor map");
    }
    p.C = g.C; p.R = g.R; p.ldc = g.ldc; p.c_seq_stride = g.c_seq_stride; p.c_inner_stride = g.c_inner_stride; p.c_inner = g.c_inner;
    p.bias = g.bias; p.prelu = g.prelu; p.prelu_vec = g.prelu_vec; p.ln_g = g.ln_g; p.ln_b = g.ln_b; p.alpha = g.alpha;
    p.vec_ok = lp.vec_ok;
    const int grid = lp.grid;
    ++g_launches;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(NTHREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = g.pdl ? 1 : 0;
    if (p.BN == 64) return p.b_mn_major ? cudaLaunchKernelEx(&cfg, umma_gemm_kernel<64, 1>, p) : cudaLaunchKernelEx(&cfg, umma_gemm_kernel<64, 0>, p);
    return p.b_mn_major ? cudaLaunchKernelEx(&cfg, umma_gemm_kernel<128, 1>, p) : cudaLaunchKernelEx(&cfg, umma_gemm_kernel<128, 0>, p);
}

// ---- B operand preparation: fp32 matrix (any strides) -> bf16 hi/lo planes [2][rows][cols] ---------------------
__global__ void split_planes_kernel(const float* __restrict__ src, int64_t row_stride, int64_t col_stride, int rows, int cols,
                                    int64_t ld, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)rows * cols) return;
    const int r = (int)(i / cols), c = (int)(i % cols);
    const float a = src[(int64_t)r * row_stride + (int64_t)c * col_stride];
    const __nv_bfloat16 h = __float2bfloat16_rn(a);
    hi[(int64_t)r * ld + c] = h;
    lo[(int64_t)r * ld + c] = __float2bfloat16_rn(a - __bfloat162float(h));
}

cudaError_t split_planes(const float* src, int64_t row_stride, int64_t col_stride, int rows, int cols, int64_t ld,
                                __nv_bfloat16* hi, __nv_bfloat16* lo, cudaStream_t st) {
    const int64_t n = (int64_t)rows * cols;
    split_planes_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, row_stride, col_stride, rows, cols, ld, hi, lo);
    return cudaGetLastError();
}

}  // namespace umma
}  // namespace l2h
