// Test-only C entry points into the engine's tensor-core GEMM (umma::launch), LSTM recurrences (lstm.cuh,
// tc_lstm.cuh), the separator's attention section (sep_kernels.cuh), its front and back (sep_kernels.cuh,
// hop_kernels.cuh), its CUDA-core rows GEMM (gemm.cuh), its one-hop middle section (mid_kernel.cuh: mid_kernel, mid_a,
// mid_b, mid_c), the fused one-hop tail of a block (hop_kernels.cuh: tail_kernel, both record maps), the tensor-core
// chain's cell kernel (sep_kernels.cuh: lstm_cell_rows), the enrollment network's own kernels (embed_kernels.cuh: estd,
// efront, egn_apply, eqkv_ln, softmax_rows, eattn_out, ehead, einter_mask, eput_lens), the several-target kernels
// (targets_kernels.cuh: target_lists, spk_gate, gate_fanout) and the slot-list helpers (sep_kernels.cuh: gather_h,
// scatter_hc, inter_gate_mask, inter_h_last), the kernels that own a separator state's records (sep_kernels.cuh:
// state_init, reset_streams, advance_header, set_clip_base; targets_kernels.cuh: join_start, history_put, history_get,
// move_lead), the enrollment-from-capture kernels (embed_kernels.cuh: eslot_rows, eput_rows, and estd / efront over the
// capture ring's XRing map), so that the kernel-level tests (tests/test_*_kernels_gpu.py) can drive each kernel directly
// with arbitrary shapes and compare it element by element with a float64 or exact reference.
//
// The argument structs below are plain C (mirrored with ctypes in the tests); every function checks its arguments, fills
// the engine's own descriptor and calls the engine's own launcher.  Built by
// lookoncetohear_b200/build.py as lib/libl2h_kernel_harness.so with hidden visibility, so this library's copy of the
// l2h symbols never binds to the product library's copy.
#include <cstdio>
#include "umma_gemm.cu"
#include "gemm.cuh"
#include "tc_lstm.cuh"
#include "sep_launch.cuh"
#include "embed_kernels.cuh"
#include "targets_kernels.cuh"      // last, as in the engine

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
    const int32_t* steps;       // KH_LSTM_TC_X only (LstmXArgs::steps); must be null for the other variants
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

// 16-CTA tail_kernel clusters the configured device holds at once (set_tail_attrs; 0: tail_kernel cannot be scheduled)
static thread_local int tail_clusters = 0;

// the dynamic shared memory of every kernel launched here that needs more than the default, set once per device (the
// separator's dense forms with the engine's own list, and both forms of tail_kernel)
static cudaError_t configure() {
    static thread_local int configured_dev = -1;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess || configured_dev == dev) return e;
    e = configure_lstm();
    if (e == cudaSuccess) e = configure_tc_lstm();
    if (e == cudaSuccess) e = configure_rows_gemm();
    if (e == cudaSuccess) e = set_sep_smem<int64_t>();
    if (e == cudaSuccess) e = set_mid_split_smem();
    if (e == cudaSuccess) e = cudaFuncSetAttribute(emb::eattn_out_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)emb::EAOUT_SMEM);
    if (e == cudaSuccess) tail_clusters = set_tail_attrs();
    if (e == cudaSuccess) configured_dev = dev;
    return e;
}

// `passes` applies to the tensor-core variants only
KH_API int kh_lstm(const KhLstm* k, int variant, int passes, char* why, int why_len, void* stream) {
    put_why(why, why_len, nullptr);
    cudaError_t e = configure();
    if (e != cudaSuccess) { put_why(why, why_len, "kernel attributes"); return (int)e; }
    const LstmArgs a = to_lstm(*k);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (k->steps != nullptr && variant != KH_LSTM_TC_X) { put_why(why, why_len, "steps apply to tc_x only"); return (int)cudaErrorInvalidValue; }
    static const LstmRec forced[] = {LstmRec::rec3_pre, LstmRec::rec3_ring, LstmRec::rec4_2, LstmRec::rec4_4};   // KH_LSTM_REC*
    switch (variant) {
        case KH_LSTM_AUTO: e = launch_lstm_rec(a, st); break;
        case KH_LSTM_REC3_PRE: case KH_LSTM_REC3_RING: case KH_LSTM_REC4_2: case KH_LSTM_REC4_4: {
            // the forced kernels get the launcher's own argument checks
            const char* no = (a.nseq <= 0 || a.L <= 0 || !lstm_state_ok(a)) ? "refused by the launcher's checks"
                             : (variant == KH_LSTM_REC3_PRE && !lstm_rec_preloads(a.L)) ? "L too long for the preloaded kernel" : nullptr;
            if (no) { put_why(why, why_len, no); return (int)cudaErrorInvalidValue; }
            e = launch_lstm_variant(forced[variant - KH_LSTM_REC3_PRE], a, st, false);
            break;
        }
        case KH_LSTM_TC: e = launch_tc_lstm(a, passes, st); break;
        case KH_LSTM_TC_X: {
            tcl::LstmXArgs xa{};
            xa.l = a; xa.x = k->x; xa.x_ld = k->x_ld;
            xa.wih_hi = static_cast<const __nv_bfloat16*>(k->wih_hi); xa.wih_lo = static_cast<const __nv_bfloat16*>(k->wih_lo);
            xa.bias = k->bias; xa.ln_g = k->ln_g; xa.ln_b = k->ln_b; xa.steps = k->steps;
            e = launch_tc_lstm_x(xa, passes, st);
            break;
        }
        default: put_why(why, why_len, "unknown variant"); return (int)cudaErrorInvalidValue;
    }
    if (e != cudaSuccess) put_why(why, why_len, cudaGetErrorString(e));
    return (int)e;
}

// ---- the separator's attention section (sep_kernels.cuh) -------------------------------------------------------------
// The fields of BlockWeights that qkv_kernel, qkv_many_kernel, attn_out_kernel and ln_frame_res_kernel read.  The four
// Q/K LayerNorm vectors are read as QK_LD (584) floats: 582 values and 2 floats of padding.
struct KhSepWeights {
    const float *wqkv_t, *bqkv, *slopes;
    const float *lnq_g, *lnq_b, *lnk_g, *lnk_b, *lnv_g, *lnv_b;
    const float *wp_t, *bp, *lnp_g, *lnp_b;
};

enum KhAttnForm { KH_ATTN_QUERY = 0, KH_ATTN_TILE = 1, KH_ATTN_CLUSTER = 2 };   // attn_kernel, attn_tile_kernel, attn_cluster_kernel

static BlockWeights to_block(const KhSepWeights& k) {
    BlockWeights w{};
    w.wqkv_t = k.wqkv_t; w.bqkv = k.bqkv; w.slopes = k.slopes;
    w.lnq_g = k.lnq_g; w.lnq_b = k.lnq_b; w.lnk_g = k.lnk_g; w.lnk_b = k.lnk_b; w.lnv_g = k.lnv_g; w.lnv_b = k.lnv_b;
    w.wp_t = k.wp_t; w.bp = k.bp; w.lnp_g = k.lnp_g; w.lnp_b = k.lnp_b;
    return w;
}

KH_API int kh_sizeof_sep_weights() { return (int)sizeof(KhSepWeights); }

// RING, QK_LD, QK_DIM, V_DIM, ATT, ST_GATE, ST_BLK, BK_K, BK_V, BK_H, BK_C, BK_STRIDE, ST_POS, ST_CALLS,
// sizeof(StateHeader), stream_stride(n_blocks), ST_EMB, ST_GEN, ST_CONV, ST_DECONV, ST_ISTFT; returns the count written (21)
KH_API int kh_sep_layout(int n_blocks, int64_t* out) {
    const int64_t v[] = {RING, QK_LD, QK_DIM, V_DIM, ATT, ST_GATE, ST_BLK, BK_K, BK_V, BK_H, BK_C, BK_STRIDE, ST_POS, ST_CALLS,
                         (int64_t)sizeof(StateHeader), stream_stride(n_blocks), ST_EMB, ST_GEN, ST_CONV, ST_DECONV, ST_ISTFT};
    const int n = (int)(sizeof(v) / sizeof(v[0]));
    for (int i = 0; i < n; ++i) out[i] = v[i];
    return n;
}

// CTAs of attn_cluster_kernel the current device holds at once: the engine splits a call's windows over 8-CTA
// clusters while B * T * NHEAD * ATT_CL fits in this (attn_splits)
KH_API int kh_attn_cluster_resident() { return attn_cluster_resident(); }

// qkv_kernel: grid (T, B).  pre == nullptr: the Linear 64 -> 112 (+ bias + PReLU) runs inside, from X [B][T][97][64];
// otherwise pre holds the projections [B][T][97][112].
KH_API int kh_qkv(const KhSepWeights* w, const float* X, const float* pre, float* Q, float* Kall, float* Vall, float* state,
                  int64_t sstride, int blk, int B, int T, int frame_k, const uint8_t* active, void* stream) {
    if (B <= 0 || T <= 0 || frame_k < 0) return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    return (int)launch_qkv(false, static_cast<cudaStream_t>(stream), B, X, pre, Q, Kall, Vall, state, sstride, blk, to_block(*w), T,
                           frame_k, active);
}

// qkv_many_kernel over frames 0 .. n_frames-1 (frame fi = stream fi / T, row fi % T) with `grid` persistent CTAs
KH_API int kh_qkv_many(const KhSepWeights* w, const float* pre, float* Q, float* Kall, float* Vall, float* state,
                       int64_t sstride, int blk, int T, int grid, int n_frames, const uint8_t* active, void* stream) {
    if (T <= 0 || grid <= 0 || n_frames <= 0) return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    return (int)launch_qkv_many(false, static_cast<cudaStream_t>(stream), grid, pre, Q, Kall, Vall, state, sstride, blk, to_block(*w),
                                T, n_frames, active);
}

// kv_gather_kernel: grid (ATT - 1, B * NHEAD), 128 threads
KH_API int kh_kv_gather(const float* state, int64_t sstride, int blk, float* Kall, float* Vall, int B, int T, void* stream) {
    if (B <= 0 || T <= 1) return (int)cudaErrorInvalidValue;
    return (int)launch_kv_gather(false, static_cast<cudaStream_t>(stream), B, state, sstride, blk, Kall, Vall, T);
}

// One attention form: T == 1 reads the ring (window of frame clock + frame_k), T > 1 the linear scratch.  The tile form
// reads the scratch only; the engine never launches it with T == 1, and it has no frame_k.
KH_API int kh_attention(int form, const float* Q, const float* Kall, const float* Vall, const float* state, int64_t sstride,
                        int blk, float* Z, int B, int T, int frame_k, void* stream) {
    if (B <= 0 || T <= 0 || frame_k < 0 || (T > 1 && frame_k != 0)) return (int)cudaErrorInvalidValue;
    if (form < KH_ATTN_QUERY || form > KH_ATTN_CLUSTER || (form == KH_ATTN_TILE && T == 1)) return (int)cudaErrorInvalidValue;
    static const AttnForm forms[] = {AttnForm::query, AttnForm::tile, AttnForm::cluster};      // by KhAttnForm
    return (int)launch_attention(forms[form], false, static_cast<cudaStream_t>(stream), B, Q, Kall, Vall, state, sstride, blk, Z, T,
                                 frame_k);
}

// attn_out_kernel: grid (T, B); X [B][T][97][64] updated in place; the gate is ST_GATE of each stream's record
KH_API int kh_attn_out(const KhSepWeights* w, const float* Z, float* X, const float* state, int64_t sstride, int B, int T,
                       int apply_gate, void* stream) {
    if (B <= 0 || T <= 0) return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    return (int)launch_attn_out(false, static_cast<cudaStream_t>(stream), B, Z, X, state, sstride, to_block(*w), apply_gate, T);
}

// ln_frame_res_kernel: grid (T, B); P [B][T][97][64] = the projection after PReLU
KH_API int kh_ln_frame_res(const KhSepWeights* w, const float* P, float* X, const float* state, int64_t sstride, int B, int T,
                           int apply_gate, void* stream) {
    if (B <= 0 || T <= 0) return (int)cudaErrorInvalidValue;
    return (int)launch_ln_frame_res(false, static_cast<cudaStream_t>(stream), B, P, X, state, sstride, to_block(*w), apply_gate, T);
}

// ---- the separator's front and back (sep_kernels.cuh, hop_kernels.cuh) ----------------------------------------------
// The SepWeights fields, and for front1_kernel the block-0 fields of its input projection.
struct KhSepFrontBack {
    const float *wat, *ws, *wc, *bc, *we, *be, *lne_g, *lne_b, *wd, *bd;
    int32_t gen;
    const float *ln1_g, *ln1_b, *wih1_t, *b1;
};

static SepWeights to_sep(const KhSepFrontBack& k) {
    SepWeights w{};
    w.wat = k.wat; w.ws = k.ws; w.wc = k.wc; w.bc = k.bc; w.we = k.we; w.be = k.be; w.lne_g = k.lne_g; w.lne_b = k.lne_b;
    w.wd = k.wd; w.bd = k.bd; w.gen = k.gen;
    return w;
}

KH_API int kh_sizeof_sep_front_back() { return (int)sizeof(KhSepFrontBack); }

// front_kernel.  frames_total <= 1: an ordinary call of T frames, grid (T + 1, B).  frames_total > 1: hop frame_k of a
// group of frames_total one-frame calls of the pipelined graph (T must be 1): grid (frame_k == 0 ? 2 : 1, B), samples
// from offset frame_k * 128 -- only hop 0 carries the speaker-gate CTA.
KH_API int kh_front(const KhSepFrontBack* w, const float* x, int64_t x_bstride, int64_t x_cstride, int x_len, float* X,
                    float* state, int64_t sstride, int B, int T, int pos_rel, const float* emb, float* spk_pre, int frame_k,
                    int frames_total, const uint8_t* active, void* stream) {
    const bool group = frames_total > 1;
    if (B <= 0 || T <= 0 || (group && (T != 1 || frame_k < 0 || frame_k >= frames_total)) || (!group && frame_k != 0))
        return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    return (int)launch_front(false, static_cast<cudaStream_t>(stream), B, group ? (frame_k == 0 ? 1 : 0) : 1, x, x_bstride, x_cstride,
                             x_len, X, state, sstride, to_sep(*w), T, pos_rel, emb, spk_pre, group ? frame_k : 0,
                             group ? frames_total : 1, group ? frame_k * HOP : 0, active);
}

// the engine's front_many_kernel geometry for (B, T) (sep_launch.cuh)
KH_API void kh_front_many_geometry(int B, int T, int* chunk, int* n_workers) {
    const ChunkWalk g = front_many_walk(B, T);
    *chunk = g.chunk; *n_workers = g.workers;
}

// front_many_kernel: n_workers CTAs walk the (stream, chunk-of-`chunk`-frames) items, then one speaker-gate CTA per stream
KH_API int kh_front_many(const KhSepFrontBack* w, const float* x, int64_t x_bstride, int64_t x_cstride, int x_len, float* X,
                         float* state, int64_t sstride, int B, int T, int pos_rel, const float* emb, float* spk_pre, int chunk,
                         int n_workers, const uint8_t* active, void* stream) {
    if (B <= 0 || T <= 0 || chunk <= 0 || n_workers <= 0) return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    const ChunkWalk g{chunk, (T + chunk - 1) / chunk, n_workers};
    return (int)launch_front_many(false, static_cast<cudaStream_t>(stream), 1, g, x, x_bstride, x_cstride, x_len, X, state, sstride,
                                  to_sep(*w), T, pos_rel, emb, spk_pre, B, active);
}

// front1_kernel: one frame as 13 tiles of 8 bins plus the speaker-gate CTA, grid (14, B); GX [B][97][512]
KH_API int kh_front1(const KhSepFrontBack* w, const float* x, int64_t x_bstride, int64_t x_cstride, int x_len, float* X,
                     float* GX, float* state, int64_t sstride, int B, int pos_rel, const float* emb, float* spk_pre,
                     const uint8_t* active, void* stream) {
    if (B <= 0) return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    BlockWeights w0{};
    w0.ln1_g = w->ln1_g; w0.ln1_b = w->ln1_b; w0.wih1_t = w->wih1_t; w0.b1 = w->b1;
    return (int)launch_front1(false, static_cast<cudaStream_t>(stream), B, 1, x, x_bstride, x_cstride, x_len, X, state, sstride,
                              to_sep(*w), w0, GX, pos_rel, emb, spk_pre, active);
}

// back_kernel in clusters of BACK_CL.  frames_total <= 1: an ordinary call of T frames, grid (4 T, B); it advances the
// clocks.  frames_total > 1: hop frame_k of a pipelined group (T must be 1), grid (4, B), samples from offset
// frame_k * 128, X = this hop's rows with the previous hops' hist_stride floats apart; it advances no clock.
KH_API int kh_back(const KhSepFrontBack* w, const float* X, float* y, int64_t y_bstride, int64_t y_cstride, int y_len,
                   float* state, int64_t sstride, int B, int T, int pos_rel, int frame_k, int frames_total, int64_t hist_stride,
                   const uint8_t* active, void* stream) {
    const bool group = frames_total > 1;
    if (B <= 0 || T <= 0 || (group && (T != 1 || frame_k < 0 || frame_k >= frames_total)) || (!group && frame_k != 0))
        return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    return (int)launch_back(false, static_cast<cudaStream_t>(stream), B, X, y, y_bstride, y_cstride, y_len, state, sstride, to_sep(*w),
                            T, pos_rel, group ? frame_k : 0, group ? frames_total : 1, group ? frame_k * HOP : 0,
                            group ? hist_stride : 0, active);
}

// the engine's back_many_kernel geometry for (B, T) (sep_launch.cuh)
KH_API void kh_back_many_geometry(int B, int T, int* chunk, int* n_cl) {
    const ChunkWalk g = back_many_walk(B, T);
    *chunk = g.chunk; *n_cl = g.workers;
}

// back_many_kernel: n_cl clusters of BACK_CL walk the (stream, chunk-of-`chunk`-frames) items; it advances the clocks
KH_API int kh_back_many(const KhSepFrontBack* w, const float* X, float* y, int64_t y_bstride, int64_t y_cstride, int y_len,
                        float* state, int64_t sstride, int B, int T, int pos_rel, int chunk, int n_cl, const uint8_t* active,
                        void* stream) {
    if (B <= 0 || T <= 0 || chunk <= 0 || n_cl <= 0) return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    const ChunkWalk g{chunk, (T + chunk - 1) / chunk, n_cl};
    return (int)launch_back_many(false, static_cast<cudaStream_t>(stream), g, X, y, y_bstride, y_cstride, y_len, state, sstride,
                                 to_sep(*w), T, pos_rel, B, active);
}

// ---- the separator's CUDA-core rows GEMM (gemm.cuh) -------------------------------------------------------------------
// GemmArgs field for field
struct KhRowsGemm {
    const float* A;
    int64_t lda;
    int32_t a_rows_per_seq;
    int64_t a_seq_stride;
    const float *Wt, *bias;
    float* C;
    int64_t ldc;
    int32_t c_rows_per_seq;
    int64_t c_seq_stride;
    int32_t c_inner;
    int64_t c_inner_stride;
    const float *R, *ln_g, *ln_b, *prelu, *prelu_vec;
    int32_t M, N, K;
};

static GemmArgs to_rows_gemm(const KhRowsGemm& k) {
    GemmArgs g{};
    g.A = k.A; g.lda = k.lda; g.a_rows_per_seq = k.a_rows_per_seq; g.a_seq_stride = k.a_seq_stride;
    g.Wt = k.Wt; g.bias = k.bias; g.C = k.C; g.ldc = k.ldc;
    g.c_rows_per_seq = k.c_rows_per_seq; g.c_seq_stride = k.c_seq_stride; g.c_inner = k.c_inner; g.c_inner_stride = k.c_inner_stride;
    g.R = k.R; g.ln_g = k.ln_g; g.ln_b = k.ln_b; g.prelu = k.prelu; g.prelu_vec = k.prelu_vec;
    g.M = k.M; g.N = k.N; g.K = k.K;
    return g;
}

KH_API int kh_sizeof_rows_gemm() { return (int)sizeof(KhRowsGemm); }

// the kernel launch_rows_gemm runs for (M, N, K, shape) without a LayerNorm prologue, as RowsGemmForm (0: refused)
KH_API int kh_rows_gemm_form(int M, int N, int K, int shape) {
    GemmArgs g{};
    g.M = M; g.N = N; g.K = K;
    return (int)rows_gemm_form(g, shape);
}

// launch_rows_gemm(g, stream, no PDL, shape); *form (may be null) = the kernel it chose (RowsGemmForm)
KH_API int kh_rows_gemm(const KhRowsGemm* k, int shape, int* form, void* stream) {
    const GemmArgs g = to_rows_gemm(*k);
    if (form) *form = (int)rows_gemm_form(g, shape);
    if (shape < 0 || shape > 2 || g.A == nullptr || g.Wt == nullptr || g.C == nullptr || g.lda < g.K) return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    return (int)launch_rows_gemm(g, static_cast<cudaStream_t>(stream), false, shape);
}

// ---- the separator's one-hop middle section (mid_kernel.cuh) and the tensor-core chain's cell (sep_kernels.cuh) -------
// The fields of BlockWeights that mid_kernel, mid_a, mid_b and mid_c read.
struct KhMidWeights {
    const float *mid_pack, *bl1, *ln2_g, *ln2_b, *b2, *bl2, *bqkv, *slopes;
};

static BlockWeights to_mid(const KhMidWeights& k) {
    BlockWeights w{};
    w.mid_pack = k.mid_pack; w.bl1 = k.bl1; w.ln2_g = k.ln2_g; w.ln2_b = k.ln2_b; w.b2 = k.b2; w.bl2 = k.bl2; w.bqkv = k.bqkv;
    w.slopes = k.slopes;
    return w;
}

KH_API int kh_sizeof_mid_weights() { return (int)sizeof(KhMidWeights); }

// MID_PACK, MID_RT, MID_W1, MID_W3A, MID_W3B, MID_W5, MID_W6, MID_SMEM, MID_A_SMEM, MID_B_SMEM, MID_C_SMEM (bytes), NUM_SMS;
// returns the count written (12)
KH_API int kh_mid_layout(int64_t* out) {
    const int64_t v[] = {MID_PACK, MID_RT, MID_W1, MID_W3A, MID_W3B, MID_W5, MID_W6, (int64_t)MID_SMEM, (int64_t)MID_A_SMEM,
                         (int64_t)MID_B_SMEM, (int64_t)MID_C_SMEM, NUM_SMS};
    const int n = (int)(sizeof(v) / sizeof(v[0]));
    for (int i = 0; i < n; ++i) out[i] = v[i];
    return n;
}

// the engine's k-sliced packing (host arrays; dst holds MID_PACK floats)
KH_API void kh_mid_pack(const float* wl1_t, const float* wih2_t, const float* whh2_t, const float* wl2_t, const float* wqkv_t,
                        float* dst) {
    mid_pack_weights(wl1_t, wih2_t, whh2_t, wl2_t, wqkv_t, dst);
}

// mid_kernel over B streams' [B][97] rows of Y [..][128], X [..][64] (updated in place) and QKV [..][112]; the carried
// (h, c) of block blk of record b at state + header + b * sstride
KH_API int kh_mid(const KhMidWeights* w, const float* Y, float* X, float* QKV, float* state, int64_t sstride, int blk, int B,
                  const uint8_t* active, void* stream) {
    if (B <= 0 || blk < 0 || sstride <= 0) return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    return (int)launch_mid(false, static_cast<cudaStream_t>(stream), Y, X, QKV, state, sstride, blk, to_mid(*w), B, active);
}

// mid_a / mid_b / mid_c over n_hops hops whose buffers sit hop_stride floats apart
KH_API int kh_mid_a(const KhMidWeights* w, const float* Y, float* X, float* GI, int B, int64_t hop_stride, int n_hops, void* stream) {
    if (B <= 0 || n_hops <= 0 || hop_stride < 0) return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    return (int)launch_mid_a(false, static_cast<cudaStream_t>(stream), Y, X, GI, to_mid(*w), B, hop_stride, n_hops);
}

KH_API int kh_mid_b(const KhMidWeights* w, const float* GI, float* Hn, int64_t hop_stride, int n_hops, float* state, int64_t sstride,
                    int blk, int B, const uint8_t* active, void* stream) {
    if (B <= 0 || n_hops <= 0 || hop_stride < 0 || blk < 0 || sstride <= 0) return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    return (int)launch_mid_b(false, static_cast<cudaStream_t>(stream), GI, Hn, hop_stride, n_hops, state, sstride, blk, to_mid(*w), B,
                             active);
}

KH_API int kh_mid_c(const KhMidWeights* w, const float* Hn, float* X, float* QKV, int B, int64_t hop_stride, int n_hops, void* stream) {
    if (B <= 0 || n_hops <= 0 || hop_stride < 0) return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    return (int)launch_mid_c(false, static_cast<cudaStream_t>(stream), Hn, X, QKV, to_mid(*w), B, hop_stride, n_hops);
}

// lstm_cell_rows_kernel: gates [rows][256] (column j*4 + q), row r = stream r / 97, bin r % 97; Hout [rows][64]
KH_API int kh_lstm_cell_rows(const float* gates, float* state, int64_t sstride, int blk, float* Hout, int64_t rows,
                             const uint8_t* active, void* stream) {
    if (rows <= 0 || rows * 64 > 0x7fffffff || blk < 0 || sstride <= 0) return (int)cudaErrorInvalidValue;
    return (int)launch_lstm_cell_rows(false, static_cast<cudaStream_t>(stream), gates, state, sstride, blk, Hout, rows, active);
}

// ---- the fused one-hop tail of a block (hop_kernels.cuh: tail_kernel) -------------------------------------------------
// The fields of BlockWeights that tail_kernel reads (the middle section's, slopes[3] = the output PReLU, the Q/K/V
// LayerNorms with the Q/K vectors read as QK_LD floats, the output projection and its LayerNorm), and the next block's
// input projection (NextIh; nx_wih_t == null: no next block, GX untouched).
struct KhTailWeights {
    const float *mid_pack, *bl1, *ln2_g, *ln2_b, *b2, *bl2, *bqkv, *slopes;
    const float *lnq_g, *lnq_b, *lnk_g, *lnk_b, *lnv_g, *lnv_b;
    const float *wp_t, *bp, *lnp_g, *lnp_b;
    const float *nx_ln_g, *nx_ln_b, *nx_wih_t, *nx_bias;
};

static BlockWeights to_tail(const KhTailWeights& k) {
    BlockWeights w{};
    w.mid_pack = k.mid_pack; w.bl1 = k.bl1; w.ln2_g = k.ln2_g; w.ln2_b = k.ln2_b; w.b2 = k.b2; w.bl2 = k.bl2; w.bqkv = k.bqkv;
    w.slopes = k.slopes;
    w.lnq_g = k.lnq_g; w.lnq_b = k.lnq_b; w.lnk_g = k.lnk_g; w.lnk_b = k.lnk_b; w.lnv_g = k.lnv_g; w.lnv_b = k.lnv_b;
    w.wp_t = k.wp_t; w.bp = k.bp; w.lnp_g = k.lnp_g; w.lnp_b = k.lnp_b;
    return w;
}

static NextIh to_next(const KhTailWeights& k, float* GX) {
    NextIh nx{};
    if (k.nx_wih_t != nullptr) { nx.ln_g = k.nx_ln_g; nx.ln_b = k.nx_ln_b; nx.wih_t = k.nx_wih_t; nx.bias = k.nx_bias; nx.GX = GX; }
    return nx;
}

KH_API int kh_sizeof_tail_weights() { return (int)sizeof(KhTailWeights); }

// 16-CTA tail_kernel clusters the current device holds at once (set_tail_attrs): the engine fuses a block's tail while
// the call's rows fit in one wave of them
KH_API int kh_tail_clusters() { return configure() == cudaSuccess ? tail_clusters : 0; }

// tail_kernel, dense map: row b of Y [B][97][128], X [B][97][64] (updated in place) and GX [B][97][512] is record b at
// state + header + b * sstride; block blk
KH_API int kh_tail(const KhTailWeights* w, const float* Y, float* X, float* GX, float* state, int64_t sstride, int blk, int B,
                   int apply_gate, int frame_k, const uint8_t* active, void* stream) {
    if (B <= 0 || blk < 0 || sstride <= 0 || frame_k < 0 || (w->nx_wih_t != nullptr && GX == nullptr)) return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    if (tail_clusters <= 0) return (int)cudaErrorInvalidConfiguration;
    return (int)launch_tail(false, static_cast<cudaStream_t>(stream), B, Y, X, state, sstride, blk, to_tail(*w), to_next(*w, GX), apply_gate,
                            frame_k, active);
}

// tail_kernel_t<Records>: row b is record slots[b] of a state of `batch` records of sstride floats; hops (device, [B]) may
// be null; the call is one frame
KH_API int kh_tail_slots(const KhTailWeights* w, const float* Y, float* X, float* GX, float* state, int64_t sstride,
                         const int32_t* slots, int batch, const int32_t* hops, int blk, int B, int apply_gate, void* stream) {
    if (B <= 0 || batch <= 0 || blk < 0 || sstride <= 0 || slots == nullptr || (w->nx_wih_t != nullptr && GX == nullptr))
        return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    if (tail_clusters <= 0) return (int)cudaErrorInvalidConfiguration;
    const Records recs{sstride, slots, batch, hops, 1};
    return (int)launch_tail(false, static_cast<cudaStream_t>(stream), B, Y, X, state, recs, blk, to_tail(*w), to_next(*w, GX), apply_gate,
                            0, nullptr);
}

// ---- the enrollment network's own kernels (embed_kernels.cuh) --------------------------------------------------------
// Launched through embed_forward_impl's launchers.  Every `lens` (device, [B] int32) may be null: the equal-length path.
// The fields of EmbWeights that estd / efront / egn_apply / ehead read, and of EmbBlockWeights that eqkv_ln and eattn_out
// read.
struct KhEmbWeights {
    const float *dft, *wc, *bc, *gn_g, *gn_b, *lnh_g, *lnh_b;
};

struct KhEmbBlock {
    const float *gq, *bq, *gk, *bk, *gv, *bv;
    const float *wp_t, *bp, *slope_p, *gp, *bpn;
};

static emb::EmbWeights to_emb(const KhEmbWeights& k) {
    emb::EmbWeights w{};
    w.dft = k.dft; w.wc = k.wc; w.bc = k.bc; w.gn_g = k.gn_g; w.gn_b = k.gn_b; w.lnh_g = k.lnh_g; w.lnh_b = k.lnh_b;
    return w;
}

static emb::EmbBlockWeights to_emb_block(const KhEmbBlock& k) {
    emb::EmbBlockWeights w{};
    w.gq = k.gq; w.bq = k.bq; w.gk = k.gk; w.bk = k.bk; w.gv = k.gv; w.bv = k.bv;
    w.wp_t = k.wp_t; w.bp = k.bp; w.slope_p = k.slope_p; w.gp = k.gp; w.bpn = k.bpn;
    return w;
}

KH_API int kh_sizeof_emb_weights() { return (int)sizeof(KhEmbWeights); }
KH_API int kh_sizeof_emb_block() { return (int)sizeof(KhEmbBlock); }

// NFFT, HOP, NF, CH, QK, VDIM, FC, NQKV, DFT_LD, EAOUT_SMEM, LENS_PER_LAUNCH; returns the count written (11)
KH_API int kh_embed_layout(int64_t* out) {
    const int64_t v[] = {emb::NFFT, emb::HOP, emb::NF, emb::CH, emb::QK, emb::VDIM, emb::FC, emb::NQKV, emb::DFT_LD,
                         (int64_t)emb::EAOUT_SMEM, emb::LENS_PER_LAUNCH};
    const int n = (int)(sizeof(v) / sizeof(v[0]));
    for (int i = 0; i < n; ++i) out[i] = v[i];
    return n;
}

// estd_kernel: grid B, 256 threads; x [B][2][N]
KH_API int kh_estd(const float* x, int N, const int32_t* lens, float* inv_std, int B, void* stream) {
    if (B <= 0 || N <= 0) return (int)cudaErrorInvalidValue;
    return (int)emb::launch_estd(static_cast<cudaStream_t>(stream), B, x, N, lens, inv_std);
}

// efront_kernel: grid (T, B), 256 threads; the caller zeroes gn_sums [B][2] (double)
KH_API int kh_efront(const KhEmbWeights* w, const float* x, int N, const int32_t* lens, const float* inv_std, float* X,
                     double* gn_sums, int B, int T, void* stream) {
    if (B <= 0 || T <= 0) return (int)cudaErrorInvalidValue;
    return (int)emb::launch_efront(static_cast<cudaStream_t>(stream), B, x, N, lens, inv_std, X, gn_sums, to_emb(*w), T);
}

// egn_apply_kernel: ceil(total4 / 256) CTAs of 256 threads
KH_API int kh_egn_apply(const KhEmbWeights* w, float* X, const double* gn_sums, int64_t per_b, int64_t total4,
                        const int32_t* lens, void* stream) {
    if (per_b <= 0 || total4 <= 0) return (int)cudaErrorInvalidValue;
    return (int)emb::launch_egn_apply(static_cast<cudaStream_t>(stream), X, gn_sums, per_b, total4, lens, to_emb(*w));
}

// eqkv_ln_kernel: grid (T, B), 384 threads; QKV [B][T][65][128]
KH_API int kh_eqkv_ln(const KhEmbBlock* w, const float* QKV, float* Qn, void* Kp, void* Vp, int64_t k_plane, int64_t v_plane,
                      int B, int T, int Tp, void* stream) {
    if (B <= 0 || T <= 0 || Tp < T) return (int)cudaErrorInvalidValue;
    return (int)emb::launch_eqkv_ln(static_cast<cudaStream_t>(stream), B, QKV, Qn, static_cast<__nv_bfloat16*>(Kp),
                                    static_cast<__nv_bfloat16*>(Vp), k_plane, v_plane, to_emb_block(*w), T, Tp);
}

// softmax_rows_kernel: one CTA of 128 threads per row, Z * rows_per_z rows
KH_API int kh_softmax_rows(float* S, int64_t ld, int n, int rows_per_z, int64_t z_stride, int Z, const int32_t* lens,
                           void* stream) {
    if (Z <= 0 || rows_per_z <= 0 || n <= 0 || ld < n) return (int)cudaErrorInvalidValue;
    return (int)emb::launch_softmax_rows(static_cast<cudaStream_t>(stream), Z, S, ld, n, rows_per_z, z_stride, lens);
}

// the engine's eattn_out_kernel grid for (T, B)
KH_API int kh_eattn_out_grid(int T, int B) { return emb::eattn_out_ctas(T, B); }

// eattn_out_kernel with `grid` persistent CTAs over frames 0 .. n_frames-1 (frame item = b * T + t)
KH_API int kh_eattn_out(const KhEmbBlock* w, const float* O, float* X, int T, int Tp, int n_frames, int grid, void* stream) {
    if (T <= 0 || Tp < T || n_frames <= 0 || grid <= 0) return (int)cudaErrorInvalidValue;
    if (cudaError_t e = configure()) return (int)e;
    return (int)emb::launch_eattn_out(static_cast<cudaStream_t>(stream), grid, O, X, to_emb_block(*w), T, Tp, n_frames);
}

// ehead_kernel: grid B, 256 threads; HD [B][T][256]
KH_API int kh_ehead(const KhEmbWeights* w, const float* HD, float* out, int B, int T, const int32_t* lens, void* stream) {
    if (B <= 0 || T <= 0) return (int)cudaErrorInvalidValue;
    return (int)emb::launch_ehead(static_cast<cudaStream_t>(stream), B, HD, out, to_emb(*w), T, lens);
}

// einter_mask_kernel: grid (NF, B), 128 threads; gx [(b*NF + f)][steps][512]
KH_API int kh_einter_mask(float* gx, const int32_t* lens, int B, int steps, void* stream) {
    if (B <= 0 || steps <= 0 || lens == nullptr) return (int)cudaErrorInvalidValue;
    return (int)emb::launch_einter_mask(static_cast<cudaStream_t>(stream), B, gx, lens, steps);
}

// eput_lens_kernel: the host lengths lens_host[0 .. n-1] to dst, one launch per block of LENS_PER_LAUNCH, as the engine loops
KH_API int kh_eput_lens(int32_t* dst, const int32_t* lens_host, int n, void* stream) {
    if (n <= 0) return (int)cudaErrorInvalidValue;
    return (int)emb::launch_eput_lens(static_cast<cudaStream_t>(stream), dst, lens_host, n);
}

// ---- the several-target kernels (targets_kernels.cuh) and the slot-list helpers (sep_kernels.cuh) --------------------
// Records field for field: row b is record slots[b] of a state of `batch` records of `stride` floats; hops (device, one
// entry per row) may be null
struct KhRecords {
    int64_t stride;
    const int32_t* slots;
    int32_t batch;
    const int32_t* hops;
    int32_t frames;
};

static Records to_records(const KhRecords& k) { return Records{k.stride, k.slots, k.batch, k.hops, k.frames}; }
static bool records_ok(const KhRecords* r) { return r && r->stride > 0 && r->slots != nullptr && r->batch > 0 && r->frames > 0; }

KH_API int kh_sizeof_records() { return (int)sizeof(KhRecords); }

// target_lists_kernel over n listeners and `rows` target rows (n <= rows): records + offsets (the rows call) or groups
// (offsets and records null, K targets per group); lists = 5 rows + 1 int32, laid out as launch_target_lists states
KH_API int kh_target_lists(const int32_t* records, const int32_t* offsets, const int32_t* groups, const int32_t* hops, int n, int K,
                           int rows, int batch, int32_t* lists, void* stream) {
    const bool by_rows = records != nullptr && offsets != nullptr && groups == nullptr;
    const bool by_groups = records == nullptr && offsets == nullptr && groups != nullptr && K > 0;
    if (!(by_rows || by_groups) || n <= 0 || rows < n || batch <= 0 || lists == nullptr) return (int)cudaErrorInvalidValue;
    return (int)launch_target_lists(static_cast<cudaStream_t>(stream), records, offsets, groups, hops, n, K, rows, batch, lists);
}

// spk_gate_kernel over `rows` rows: recs == null -> the dense map (row r = record r, sstride floats apart), otherwise the
// Records map (sstride unused).  emb [rows][256], spk_pre [rows][6208].
KH_API int kh_spk_gate(const KhSepFrontBack* w, const float* emb, float* spk_pre, float* state, int64_t sstride, const KhRecords* recs,
                       int rows, void* stream) {
    if (rows <= 0 || (recs == nullptr && sstride <= 0) || (recs != nullptr && !records_ok(recs))) return (int)cudaErrorInvalidValue;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (recs == nullptr) return (int)launch_spk_gate(false, st, rows, emb, spk_pre, state, sstride, to_sep(*w));
    return (int)launch_spk_gate(false, st, rows, emb, spk_pre, state, to_records(*recs), to_sep(*w));
}

// gate_fanout_kernel: X [rows][T][97][64] from X0 [mixtures][T][97][64]; the dense map (recs == null: owner must be null,
// row r is mixture r / n_targets) or the Records map with an owner list
KH_API int kh_gate_fanout(const float* X0, float* X, const float* state, int64_t sstride, const KhRecords* recs, const int32_t* owner,
                          int n_targets, int T, int apply_gate, int rows, void* stream) {
    const bool dense = recs == nullptr && owner == nullptr && sstride > 0 && n_targets > 0;
    const bool listed = recs != nullptr && owner != nullptr && records_ok(recs);
    if (!(dense || listed) || rows <= 0 || T <= 0) return (int)cudaErrorInvalidValue;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (dense) return (int)launch_gate_fanout(false, st, rows, X0, X, state, sstride, owner, n_targets, T, apply_gate);
    return (int)launch_gate_fanout(false, st, rows, X0, X, state, to_records(*recs), owner, n_targets, T, apply_gate);
}

// gather_h_kernel over blocks b0 .. b0 + n_blocks - 1 of B rows' records into Hg (Cg: may be null), each
// [b0 + n_blocks][B][97][64]
KH_API int kh_gather_h(const float* state, const KhRecords* recs, int b0, int n_blocks, int B, float* Hg, float* Cg, void* stream) {
    if (!records_ok(recs) || b0 < 0 || n_blocks <= 0 || B <= 0 || Hg == nullptr) return (int)cudaErrorInvalidValue;
    return (int)launch_gather_h(static_cast<cudaStream_t>(stream), b0, state, to_records(*recs), n_blocks, B, Hg, Cg);
}

// scatter_hc_kernel: the inverse copy, into the records of the rows that store
KH_API int kh_scatter_hc(float* state, const KhRecords* recs, int b0, int n_blocks, int B, const float* Hg, const float* Cg,
                         void* stream) {
    if (!records_ok(recs) || b0 < 0 || n_blocks <= 0 || B <= 0 || Hg == nullptr || Cg == nullptr) return (int)cudaErrorInvalidValue;
    return (int)launch_scatter_hc(static_cast<cudaStream_t>(stream), b0, state, to_records(*recs), n_blocks, B, Hg, Cg);
}

// inter_gate_mask_kernel: gx [B][T][97][256], T = recs->frames
KH_API int kh_inter_gate_mask(float* gx, const KhRecords* recs, int B, void* stream) {
    if (!records_ok(recs) || B <= 0) return (int)cudaErrorInvalidValue;
    return (int)launch_inter_gate_mask(static_cast<cudaStream_t>(stream), B, gx, to_records(*recs), recs->frames);
}

// inter_h_last_kernel: Y [B][T][97][64] -> Hg [B][97][64], T = recs->frames
KH_API int kh_inter_h_last(const float* Y, float* Hg, const KhRecords* recs, int B, void* stream) {
    if (!records_ok(recs) || B <= 0) return (int)cudaErrorInvalidValue;
    return (int)launch_inter_h_last(static_cast<cudaStream_t>(stream), B, Y, Hg, to_records(*recs), recs->frames);
}

// ---- the kernels that own a separator state's records (sep_kernels.cuh, targets_kernels.cuh) -------------------------
// RESET_MAX_SLOTS, MOVE_MAX_PAIRS, SLOT_ROWS_PER_LAUNCH, MIN_SAMPLES (embed_kernels.cuh), EC_HEAD; returns the count
// written (5)
KH_API int kh_state_limits(int64_t* out) {
    const int64_t v[] = {RESET_MAX_SLOTS, MOVE_MAX_PAIRS, emb::SLOT_ROWS_PER_LAUNCH, emb::MIN_SAMPLES, EC_HEAD};
    const int n = (int)(sizeof(v) / sizeof(v[0]));
    for (int i = 0; i < n; ++i) out[i] = v[i];
    return n;
}

// state_init_kernel over a state of B records of `stride` floats
KH_API int kh_state_init(float* state, int64_t stride, int B, void* stream) {
    if (state == nullptr || stride <= 0 || B <= 0) return (int)cudaErrorInvalidValue;
    return (int)launch_state_init(static_cast<cudaStream_t>(stream), state, stride, B);
}

// reset_streams_kernel over the host list slots_host[0 .. n-1], each in [0, batch); records sstride floats apart, a
// multiple of 4 that holds at least the SPK floats of the embedding
static bool slots_in(const int32_t* s, int n, int batch) {
    for (int i = 0; i < n; ++i)
        if (s[i] < 0 || s[i] >= batch) return false;
    return true;
}
KH_API int kh_reset_streams(float* state, int64_t sstride, int batch, const int32_t* slots_host, int n, void* stream) {
    if (state == nullptr || slots_host == nullptr || sstride < SPK || sstride % 4 != 0 || batch <= 0 || n <= 0 ||
        !slots_in(slots_host, n, batch))
        return (int)cudaErrorInvalidValue;
    return (int)launch_reset_streams(static_cast<cudaStream_t>(stream), state, sstride, slots_host, n);
}

// advance_header_kernel: the header and the n_streams dense records advance by `frames` frames and one call
KH_API int kh_advance_header(float* state, int64_t sstride, int n_streams, int frames, void* stream) {
    if (state == nullptr || sstride <= 0 || n_streams <= 0) return (int)cudaErrorInvalidValue;
    return (int)launch_advance_header(static_cast<cudaStream_t>(stream), state, sstride, n_streams, frames);
}

// set_clip_base_kernel: header clip_base = header pos
KH_API int kh_set_clip_base(float* state, void* stream) {
    if (state == nullptr) return (int)cudaErrorInvalidValue;
    return (int)launch_set_clip_base(static_cast<cudaStream_t>(stream), state);
}

// move_lead_kernel over the host pairs from_host[i] -> to_host[i], i < n, each in [0, batch); records ss floats apart
KH_API int kh_move_lead(float* state, int64_t ss, int batch, const int32_t* from_host, const int32_t* to_host, int n, void* stream) {
    if (state == nullptr || from_host == nullptr || to_host == nullptr || ss < ST_BLK + BK_STRIDE || ss % 4 != 0 || batch <= 0 ||
        n <= 0 || !slots_in(from_host, n, batch) || !slots_in(to_host, n, batch))
        return (int)cudaErrorInvalidValue;
    return (int)launch_move_lead(static_cast<cudaStream_t>(stream), state, ss, from_host, to_host, n);
}

// join_start_kernel over J rows (device lists records and leads, any values); lists = 3 J int32: rec, used, owner;
// used_out (device, J) may be null
KH_API int kh_join_start(float* state, int64_t ss, int batch, const int32_t* records, const int32_t* leads, int w_max, int J,
                         int32_t* lists, int32_t* used_out, void* stream) {
    if (state == nullptr || records == nullptr || leads == nullptr || lists == nullptr || ss <= 0 || ss % 4 != 0 || batch <= 0 ||
        J <= 0 || w_max < 0)
        return (int)cudaErrorInvalidValue;
    return (int)launch_join_start(static_cast<cudaStream_t>(stream), J, state, ss, batch, records, leads, w_max, lists, used_out);
}

// history_put_kernel over M listeners: X0 [M][T][97][64] into hist [batch][F][97][64]; `lead` maps listener i to its lead
// record (lead->slots) and its hop count (lead->hops), with lead->frames = T
KH_API int kh_history_put(const float* X0, const float* state, const KhRecords* lead, float* hist, int F, int M, void* stream) {
    if (!records_ok(lead) || X0 == nullptr || hist == nullptr || F <= 0 || M <= 0) return (int)cudaErrorInvalidValue;
    return (int)launch_history_put(false, static_cast<cudaStream_t>(stream), M, X0, state, to_records(*lead), hist, F, lead->frames);
}

// history_get_kernel over J rows: X0 [J][T][97][64] from hist; `recs` is the join's row map (slots = rec, hops = used,
// frames = T); leads[j] must lie in [0, batch) for every row that stores
KH_API int kh_history_get(const float* hist, int F, const float* state, const KhRecords* recs, const int32_t* leads, float* X0, int J,
                          void* stream) {
    if (!records_ok(recs) || hist == nullptr || leads == nullptr || X0 == nullptr || F <= 0 || J <= 0) return (int)cudaErrorInvalidValue;
    return (int)launch_history_get(false, static_cast<cudaStream_t>(stream), J, hist, F, state, to_records(*recs), leads, X0,
                                   recs->frames);
}

// ---- enrollment from a capture (embed_kernels.cuh) -------------------------------------------------------------------
// eslot_rows_kernel over n rows: slots from the host list (each in [0, n_slots), as the engine requires) or the device
// list (any values), exactly one of them; lens_host any values; capture [n_slots][2][EC_HEAD + capacity]
KH_API int kh_eslot_rows(const int32_t* slots_host, const int32_t* slots_dev, const int32_t* lens_host, int n, const float* capture,
                         int n_slots, int capacity, int32_t* slots_out, int32_t* lens, int32_t* used, void* stream) {
    if ((slots_host == nullptr) == (slots_dev == nullptr) || lens_host == nullptr || capture == nullptr || n <= 0 || n_slots <= 0 ||
        capacity <= 0 || capacity > INT32_MAX - EC_HEAD || (slots_host != nullptr && !slots_in(slots_host, n, n_slots)))
        return (int)cudaErrorInvalidValue;
    return (int)emb::launch_eslot_rows(static_cast<cudaStream_t>(stream), slots_host, slots_dev, lens_host, n, capture,
                                       EC_HEAD + (int64_t)capacity, n_slots, capacity, slots_out, lens, used);
}

// eput_rows_kernel: src [B][256] to the dst rows of live rows, row_stride floats apart
KH_API int kh_eput_rows(const float* src, float* dst, int64_t row_stride, const int32_t* used, int B, void* stream) {
    if (src == nullptr || dst == nullptr || used == nullptr || row_stride < 256 || B <= 0) return (int)cudaErrorInvalidValue;
    return (int)emb::launch_eput_rows(static_cast<cudaStream_t>(stream), B, src, dst, row_stride, used);
}

// estd_kernel / efront_kernel over the capture ring (XRing): utterance b is the last lens[b] samples of slot slots[b]
// (device lists: slots in [0, n_slots), lens[b] in [MIN_SAMPLES, capacity], as eslot_rows leaves them); used[b] == 0
// marks a row that is not live
static emb::XRing to_ring(const float* capture, int capacity, const int32_t* slots, const int32_t* used) {
    return emb::XRing{capture, EC_HEAD + (int64_t)capacity, capacity, slots, used};
}
KH_API int kh_estd_ring(const float* capture, int capacity, const int32_t* slots, const int32_t* used, int N, const int32_t* lens,
                        float* inv_std, int B, void* stream) {
    if (capture == nullptr || slots == nullptr || used == nullptr || lens == nullptr || capacity <= 0 || N <= 0 || B <= 0)
        return (int)cudaErrorInvalidValue;
    return (int)emb::launch_estd_map(static_cast<cudaStream_t>(stream), B, to_ring(capture, capacity, slots, used), N, lens, inv_std);
}
KH_API int kh_efront_ring(const KhEmbWeights* w, const float* capture, int capacity, const int32_t* slots, const int32_t* used, int N,
                          const int32_t* lens, const float* inv_std, float* X, double* gn_sums, int B, int T, void* stream) {
    if (capture == nullptr || slots == nullptr || used == nullptr || lens == nullptr || capacity <= 0 || N <= 0 || B <= 0 || T <= 0)
        return (int)cudaErrorInvalidValue;
    return (int)emb::launch_efront_map(static_cast<cudaStream_t>(stream), B, to_ring(capture, capacity, slots, used), N, lens, inv_std,
                                       X, gn_sums, to_emb(*w), T);
}
