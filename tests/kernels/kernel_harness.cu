// Test-only C entry points into the engine's tensor-core GEMM (umma::launch) and LSTM recurrences (lstm.cuh,
// tc_lstm.cuh), so that tests/test_umma_gemm_gpu.py and tests/test_lstm_kernels_gpu.py can drive each kernel directly
// with arbitrary shapes and compare it element by element with a float64 reference.
//
// The argument structs below are plain C (mirrored with ctypes in the tests); every function fills the engine's own
// descriptor and calls the engine's own launcher.  Built by lookoncetohear_b200/build.py as lib/libl2h_kernel_harness.so
// with hidden visibility, so this library's copy of the l2h symbols never binds to the product library's copy.
#include <cstdio>
#include "umma_gemm.cu"
#include "tc_lstm.cuh"

#define KH_API extern "C" __attribute__((visibility("default")))

using namespace l2h;

struct KhASource {
    const float* base;
    int64_t channels, n_pos, pos_stride, n_inner, inner_stride, n_outer, outer_stride;
};

struct KhGemm {
    KhASource a0, a1;
    int32_t n_chunks;
    int32_t chunk_c0[umma::MAX_CHUNKS], chunk_dp[umma::MAX_CHUNKS], chunk_flags[umma::MAX_CHUNKS];
    int32_t rows_per_seq, nseq, pos_bias;
    const void* b_base;                      // bf16 planes
    int64_t b_ld, b_z_stride, b_plane_stride;
    int32_t b_nz, b_mn_major, b_by_seq;
    int32_t N, K, passes;
    float* C;
    const float* R;
    int64_t ldc, c_seq_stride, c_inner_stride;
    int32_t c_inner;
    float alpha;
    const float *bias, *prelu, *prelu_vec, *ln_g, *ln_b;
};

// the launch plan umma::launch picks for a problem (umma::plan_launch)
struct KhPlan {
    int32_t BN, b_resident, nop, nstg, P_TILE, S_TILE, grid, n_tiles_n, vec_ok;
    int64_t smem, m_tiles;
};

struct KhLstm {
    const float* gx;
    int64_t gx_ld;
    float* out;
    int64_t out_ld;
    const float* whh;
    float* h_state;
    float* c_state;
    int64_t hc_outer_stride;
    int32_t nseq, L, inner_count, ndir;
    int64_t outer_stride, inner_stride, step_stride;
    int64_t out_outer_stride, out_inner_stride, out_step_stride;
    // tc_lstm_x only
    const float* x;
    int64_t x_ld;
    const void* wih_hi;
    const void* wih_lo;
    const float *bias, *ln_g, *ln_b;
};

enum KhLstmVariant {
    KH_LSTM_AUTO = 0,       // launch_lstm_rec's own choice
    KH_LSTM_REC3_PRE = 1,   // lstm_rec3_kernel<1, true>
    KH_LSTM_REC3_RING = 2,  // lstm_rec3_kernel<1, false>
    KH_LSTM_REC4_2 = 3,     // lstm_rec4_kernel<2>
    KH_LSTM_REC4_4 = 4,     // lstm_rec4_kernel<4>
    KH_LSTM_TC = 5,         // launch_tc_lstm
    KH_LSTM_TC_X = 6,       // launch_tc_lstm_x
};

static void put_why(char* why, int why_len, const char* m) {
    if (why && why_len > 0) snprintf(why, (size_t)why_len, "%s", m ? m : "");
}

static umma::ASource to_asrc(const KhASource& s) {
    umma::ASource a;
    a.base = s.base; a.channels = s.channels; a.n_pos = s.n_pos; a.pos_stride = s.pos_stride;
    a.n_inner = s.n_inner; a.inner_stride = s.inner_stride; a.n_outer = s.n_outer; a.outer_stride = s.outer_stride;
    return a;
}

static umma::GemmDesc to_desc(const KhGemm& k) {
    umma::GemmDesc g;
    g.a0 = to_asrc(k.a0);
    g.a1 = to_asrc(k.a1);
    g.n_chunks = k.n_chunks;
    for (int j = 0; j < umma::MAX_CHUNKS && j < k.n_chunks; ++j) {
        g.chunks[j].c0 = (short)k.chunk_c0[j];
        g.chunks[j].dp = (signed char)k.chunk_dp[j];
        g.chunks[j].flags = (unsigned char)k.chunk_flags[j];
    }
    g.rows_per_seq = k.rows_per_seq; g.nseq = k.nseq; g.pos_bias = k.pos_bias;
    g.b.base = static_cast<const __nv_bfloat16*>(k.b_base);
    g.b.ld = k.b_ld; g.b.z_stride = k.b_z_stride; g.b.plane_stride = k.b_plane_stride; g.b.nz = k.b_nz;
    g.b.mn_major = k.b_mn_major != 0;
    g.b_by_seq = k.b_by_seq != 0;
    g.N = k.N; g.K = k.K; g.passes = k.passes;
    g.C = k.C; g.R = k.R; g.ldc = k.ldc; g.c_seq_stride = k.c_seq_stride; g.c_inner_stride = k.c_inner_stride; g.c_inner = k.c_inner;
    g.bias = k.bias; g.prelu = k.prelu; g.prelu_vec = k.prelu_vec; g.ln_g = k.ln_g; g.ln_b = k.ln_b; g.alpha = k.alpha;
    return g;
}

static LstmArgs to_lstm(const KhLstm& k) {
    LstmArgs a{};
    a.gx = k.gx; a.gx_ld = k.gx_ld; a.out = k.out; a.out_ld = k.out_ld; a.whh = k.whh;
    a.h_state = k.h_state; a.c_state = k.c_state; a.hc_outer_stride = k.hc_outer_stride;
    a.nseq = k.nseq; a.L = k.L; a.inner_count = k.inner_count; a.ndir = k.ndir;
    a.outer_stride = k.outer_stride; a.inner_stride = k.inner_stride; a.step_stride = k.step_stride;
    a.out_outer_stride = k.out_outer_stride; a.out_inner_stride = k.out_inner_stride; a.out_step_stride = k.out_step_stride;
    return a;
}

KH_API int kh_sizeof_asource() { return (int)sizeof(KhASource); }
KH_API int kh_sizeof_gemm() { return (int)sizeof(KhGemm); }
KH_API int kh_sizeof_plan() { return (int)sizeof(KhPlan); }
KH_API int kh_sizeof_lstm() { return (int)sizeof(KhLstm); }

// kernels this library has launched on the calling thread (umma::launch and launch_k count every launch)
KH_API long long kh_launch_count() { return g_launches; }

// the plan umma::launch would use (host-only arithmetic: without a device the grid assumes 132 SMs); 0 if planned
static int fill_plan(const umma::GemmDesc& g, KhPlan* plan) {
    memset(plan, 0, sizeof(*plan));
    umma::LaunchPlan lp;
    if (!(g.n_chunks > 0 && g.n_chunks <= umma::MAX_CHUNKS && g.N > 0 && g.rows_per_seq > 0 && g.nseq > 0 &&
          g.passes >= 1 && g.passes <= 3 && umma::plan_launch(g, lp) == nullptr))
        return (int)cudaErrorInvalidValue;
    plan->BN = lp.pl.BN; plan->b_resident = lp.pl.resident; plan->nop = lp.pl.nop; plan->nstg = lp.pl.nstg;
    plan->P_TILE = lp.P_TILE; plan->S_TILE = lp.S_TILE; plan->grid = lp.grid; plan->n_tiles_n = lp.n_tiles_n;
    plan->vec_ok = lp.vec_ok; plan->smem = (int64_t)lp.pl.smem; plan->m_tiles = lp.m_tiles;
    return 0;
}

KH_API int kh_gemm_plan(const KhGemm* k, KhPlan* plan) { return fill_plan(to_desc(*k), plan); }

// plan (may be null) is filled whenever the problem passes umma::plan_launch, also when the launch itself fails
KH_API int kh_gemm(const KhGemm* k, KhPlan* plan, char* why, int why_len, void* stream) {
    put_why(why, why_len, nullptr);
    const umma::GemmDesc g = to_desc(*k);
    if (plan) fill_plan(g, plan);
    std::string w;
    const cudaError_t e = umma::launch(g, static_cast<cudaStream_t>(stream), &w);
    put_why(why, why_len, w.c_str());
    return (int)e;
}

KH_API int kh_split_planes(const float* src, int64_t row_stride, int64_t col_stride, int rows, int cols, int64_t ld,
                           void* hi, void* lo, void* stream) {
    return (int)umma::split_planes(src, row_stride, col_stride, rows, cols, ld, static_cast<__nv_bfloat16*>(hi),
                                   static_cast<__nv_bfloat16*>(lo), static_cast<cudaStream_t>(stream));
}

// `passes` applies to the tensor-core variants only
KH_API int kh_lstm(const KhLstm* k, int variant, int passes, char* why, int why_len, void* stream) {
    put_why(why, why_len, nullptr);
    static thread_local int configured_dev = -1;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return (int)e;
    if (configured_dev != dev) {
        e = configure_lstm();
        if (e == cudaSuccess) e = configure_tc_lstm();
        if (e != cudaSuccess) { put_why(why, why_len, "kernel attributes"); return (int)e; }
        configured_dev = dev;
    }
    const LstmArgs a = to_lstm(*k);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    // the forced kernels get the launchers' own argument checks
    if (variant >= KH_LSTM_REC3_PRE && variant <= KH_LSTM_REC4_4 && (a.nseq <= 0 || a.L <= 0 || !lstm_state_ok(a))) {
        put_why(why, why_len, "refused by the launcher's checks");
        return (int)cudaErrorInvalidValue;
    }
    switch (variant) {
        case KH_LSTM_AUTO: e = launch_lstm_rec(a, st); break;
        case KH_LSTM_REC3_PRE:
            if ((size_t)a.L * 1024 > 200 * 1024) { put_why(why, why_len, "L too long for the preloaded kernel"); return (int)cudaErrorInvalidValue; }
            e = launch_k(false, lstm_rec3_kernel<1, true>, dim3(a.nseq, a.ndir), dim3(128), (size_t)a.L * 1024, st, a);
            break;
        case KH_LSTM_REC3_RING: e = launch_k(false, lstm_rec3_kernel<1, false>, dim3(a.nseq, a.ndir), dim3(128), 0, st, a); break;
        case KH_LSTM_REC4_2:
            e = launch_k(false, lstm_rec4_kernel<2>, dim3((a.nseq + 1) / 2, a.ndir), dim3(128), lstm_rec4_smem(2), st, a);
            break;
        case KH_LSTM_REC4_4:
            e = launch_k(false, lstm_rec4_kernel<4>, dim3((a.nseq + 3) / 4, a.ndir), dim3(128), lstm_rec4_smem(4), st, a);
            break;
        case KH_LSTM_TC: e = launch_tc_lstm(a, passes, st); break;
        case KH_LSTM_TC_X: {
            tcl::LstmXArgs xa{};
            xa.l = a; xa.x = k->x; xa.x_ld = k->x_ld;
            xa.wih_hi = static_cast<const __nv_bfloat16*>(k->wih_hi); xa.wih_lo = static_cast<const __nv_bfloat16*>(k->wih_lo);
            xa.bias = k->bias; xa.ln_g = k->ln_g; xa.ln_b = k->ln_b;
            e = launch_tc_lstm_x(xa, passes, st);
            break;
        }
        default: put_why(why, why_len, "unknown variant"); return (int)cudaErrorInvalidValue;
    }
    if (e != cudaSuccess) put_why(why, why_len, cudaGetErrorString(e));
    return (int)e;
}
