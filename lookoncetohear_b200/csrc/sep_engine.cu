// Separation engine: weight packing, state, the per-call kernel chain and the C ABI
// (include/lookonce_b200.h).  Host side of the hot path = this file; no torch anywhere.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <tuple>
#include <type_traits>
#include <string>
#include <vector>

#include "../../include/lookonce_b200.h"
#include "host_errors.h"
#include "weight_pack.h"
#include "gemm.cuh"
#include "umma_host.cuh"
#include "tc_lstm.cuh"
#include "lstm.cuh"
#include "sep_launch.cuh"
#include "targets_kernels.cuh"

namespace l2h {

thread_local std::string g_err;
int fail(int code, const std::string& msg) {
    g_err = msg;
    return code;
}

// (sequence, direction) pairs from which the recurrence runs on the tensor cores (tc_lstm: 32 sequences per CTA; CUDA cores:
// up to 4 per CTA).  The threshold was chosen with an earlier tensor-core recurrence on another GPU and has not been
// re-measured for the wgmma kernel on the H100; tools/offline_split_experiment.py measures the split (option "tc_lstm_min").
constexpr int TCL_MIN_SEQDIRS = 4096;

struct SepEngine {
    l2h_sep_config cfg;
    int n_blocks;
    WeightPack pack;                // packed weights; pack.device also owns the streams, events and cached graphs below
    int64_t weight_gen = 0;         // bumped by every commit
    std::vector<int64_t> plane_of;      // per block: plane offsets (pack.plane) of wih1, wl1, wih2, wl2, wqkv, [wih2|whh2], wp
    bool fuse_ih = false;               // many sequences: W_ih + LayerNorm inside the tensor-core recurrence (option "fuse_ih", default off)
    int tc_passes = 3;                  // 3 = bf16x3 split products (fp32 configs); 2 = bf16 weights x split activations (option
                                        // "bf16" = 1: the offline bf16 configuration); 1 = plain bf16 operands ("bf16" = 2)
    SepWeights w;
    std::vector<BlockWeights> bw;
    // CUDA-graph cache of whole kernel chains (the T=1 streaming chain is ~30 tiny kernels:
    // launch-bound unless replayed as a graph)
    struct CachedGraph { cudaGraphExec_t exec; int kernels; };   // kernels = kernel nodes, for the launch counter
    std::map<std::vector<int64_t>, CachedGraph> graphs;
    TraceRec* trace_dev = nullptr;                  // device trace buffer (l2h_sep_trace_start)
    int trace_cap = 0;
    int64_t launch_count = 0;                       // kernels launched so far (graph replays counted by their kernel nodes)
    cudaStream_t cap_stream = nullptr;
    struct MidSrc { int64_t wl1, wih2, whh2t, wl2, wqkv, dst, slopes, slope_vec; };
    std::vector<MidSrc> mid_src;   // per block: host offsets the packed mid_kernel weights are derived from at commit
    cudaStream_t pipe_streams[128] = {};
    std::vector<cudaEvent_t> pipe_events;
    int64_t pipe_budget = 0; // bytes the pipelined workspace may take (min(24 GB, half of the free memory at first use))
    int pipe_frames = 0;     // one-hop chains per pipelined graph (<= PIPE_MAX_FRAMES); 0 = auto: as many as a 24 GB workspace holds
    int pipe_alanes = 12;    // BiLSTM (stage A) hops in flight per block (<= PIPE_LANES)
    int pipe_gemm_shape = 0; // tile shape of the pipelined W_ih GEMM (gemm.cuh: launch_rows_gemm), option "pipeline_gemm_shape"
    int pipe_midb_hops = 4;       // pipeline: consecutive hops one mid_b launch takes (<= PIPE_MIDB_MAX)
    int pipe_pdl = 0;             // pipeline: stages launched with programmatic dependent launch (bit mask; 16 = mid_b)
    int pipe_qlanes = 3;     // qkv hops in flight per block (<= PIPE_QLANES)
    int pipe_clanes = 2;     // mid_c hops in flight per block (<= PIPE_CLANES)
    int pipe_tlanes = 3;     // attention hops in flight per block (<= PIPE_TLANES)
    int pipe_olanes = 4;     // attn_out hops in flight per block (<= PIPE_OLANES)
    int pipe_flanes = 6;     // front_kernel hops in flight (<= PIPE_FLANES)
    int pipe_blanes = 6;     // back_kernel hops in flight (<= PIPE_BLANES)
    bool use_pipe = true;    // wavefront pipelining of one-frame calls inside a multi-frame graph (option "pipeline")
    int tcl_min_seqdirs = TCL_MIN_SEQDIRS;  // (sequence, direction) pairs from which the recurrence runs on the tensor cores (option "tc_lstm_min")
    int tc_pdl = 7;              // programmatic dependent launch around the tensor-core GEMMs of many-row calls: bit 0 the many-stream mid section, bit 1 W_ih and the out projection + its LayerNorm kernel, bit 2 the persistent qkv kernel (PDL on EVERY kernel of that chain parks early-launched dependents on the SMs the big kernels need; option "tc_pdl")
    bool use_back_many = true;   // calls of several frames: front_many_kernel / back_many_kernel (one CTA / cluster per chunk of frames) instead of one per frame (option "back_many")
    bool use_tail = true;    // one-hop calls of a few streams: mid + qkv + attention + attn_out (+ next W_ih) as ONE 16-CTA cluster kernel (option "fused_tail")
    bool use_pdl = true;     // programmatic dependent launch between the kernels of a chain (option "pdl")
};

static void build_layout(SepEngine* e) {
    WeightPack& pk = e->pack;
    auto transposed = [&](const std::string& name, int rows, int cols, int ld_out) {
        // reference [rows][cols] -> packed [cols][ld_out] (k-major)
        const int64_t o = pk.alloc((int64_t)cols * ld_out);
        pk.repacked(name, (int64_t)rows * cols, [o, rows, cols, ld_out](const float* s, float* d) {
            for (int r = 0; r < rows; ++r)
                for (int c = 0; c < cols; ++c) d[o + (int64_t)c * ld_out + r] = s[(int64_t)r * cols + c];
        });
        return o;
    };
    const std::string P = "tfgridnet.";

    // STFT filterbanks [194][1][192]
    pk.bind(&e->w.wat, transposed(P + "enc.filterbank._filters", NROW, NFFT, 196));
    pk.bind(&e->w.ws, pk.plain(P + "dec.filterbank._filters", (int64_t)NROW * NFFT));
    pk.bind(&e->w.wc, pk.plain(P + "conv.0.weight", 64 * 36));
    pk.bind(&e->w.bc, pk.plain(P + "conv.0.bias", 64));
    pk.bind(&e->w.we, pk.plain(P + "embed_to_feats_proj.0.weight", (int64_t)FC * SPK));
    pk.bind(&e->w.be, pk.plain(P + "embed_to_feats_proj.0.bias", FC));
    pk.bind(&e->w.lne_g, pk.plain(P + "embed_to_feats_proj.1.weight", FC));
    pk.bind(&e->w.lne_b, pk.plain(P + "embed_to_feats_proj.1.bias", FC));
    pk.bind(&e->w.wd, pk.plain(P + "deconv.weight", 64 * 36));
    pk.bind(&e->w.bd, pk.plain(P + "deconv.bias", 4));

    e->bw.resize(e->n_blocks);
    for (int b = 0; b < e->n_blocks; ++b) {
        BlockWeights& W = e->bw[b];
        const std::string B = P + "blocks." + std::to_string(b) + ".";
        pk.bind(&W.ln1_g, pk.plain(B + "intra_norm.norm.weight", 64));
        pk.bind(&W.ln1_b, pk.plain(B + "intra_norm.norm.bias", 64));
        pk.bind(&W.ln2_g, pk.plain(B + "inter_norm.norm.weight", 64));
        pk.bind(&W.ln2_b, pk.plain(B + "inter_norm.norm.bias", 64));
        // LSTM input weights [256][64] -> Wt[k][dirofs + p], p = j*4+q
        auto ih = [&](const std::string& name, int64_t base, int ld, int dirofs) {
            pk.repacked(name, 256 * 64, [base, ld, dirofs](const float* s, float* d) {
                for (int p = 0; p < 256; ++p) {
                    const int r = perm_row(p);
                    for (int k = 0; k < 64; ++k) d[base + (int64_t)k * ld + dirofs + p] = s[r * 64 + k];
                }
            });
        };
        auto hh = [&](const std::string& name, int64_t base) {
            pk.repacked(name, 256 * 64, [base](const float* s, float* d) {
                for (int p = 0; p < 256; ++p) memcpy(d + base + (int64_t)p * 64, s + perm_row(p) * 64, 64 * sizeof(float));
            });
        };
        auto bias = [&](const std::string& name, int64_t base) {
            pk.accumulate(name, base, 256, [base](const float* s, float* d) {
                for (int p = 0; p < 256; ++p) d[base + p] += s[perm_row(p)];
            });
        };
        const int64_t wih1 = pk.alloc(64 * 512), b1 = pk.alloc(512), whh1 = pk.alloc(2 * 256 * 64);
        ih(B + "intra_rnn.weight_ih_l0", wih1, 512, 0);
        ih(B + "intra_rnn.weight_ih_l0_reverse", wih1, 512, 256);
        hh(B + "intra_rnn.weight_hh_l0", whh1);
        hh(B + "intra_rnn.weight_hh_l0_reverse", whh1 + 256 * 64);
        bias(B + "intra_rnn.bias_ih_l0", b1);
        bias(B + "intra_rnn.bias_hh_l0", b1);
        bias(B + "intra_rnn.bias_ih_l0_reverse", b1 + 256);
        bias(B + "intra_rnn.bias_hh_l0_reverse", b1 + 256);
        pk.bind(&W.wih1_t, wih1); pk.bind(&W.b1, b1); pk.bind(&W.whh1, whh1);
        const int64_t wl1 = transposed(B + "intra_linear.weight", 64, 128, 64);
        pk.bind(&W.wl1_t, wl1);
        pk.bind(&W.bl1, pk.plain(B + "intra_linear.bias", 64));
        const int64_t wih2 = pk.alloc(64 * 256), b2 = pk.alloc(256), whh2 = pk.alloc(256 * 64), whh2t = pk.alloc(64 * 256);
        ih(B + "inter_rnn.weight_ih_l0", wih2, 256, 0);
        pk.repacked(B + "inter_rnn.weight_hh_l0", 256 * 64, [whh2, whh2t](const float* s, float* d) {
            for (int p = 0; p < 256; ++p) {
                const int r = perm_row(p);
                memcpy(d + whh2 + (int64_t)p * 64, s + r * 64, 64 * sizeof(float));
                for (int k = 0; k < 64; ++k) d[whh2t + (int64_t)k * 256 + p] = s[r * 64 + k];
            }
        });
        pk.bind(&W.whh2_t, whh2t);
        bias(B + "inter_rnn.bias_ih_l0", b2);
        bias(B + "inter_rnn.bias_hh_l0", b2);
        pk.bind(&W.wih2_t, wih2); pk.bind(&W.b2, b2); pk.bind(&W.whh2, whh2);
        const int64_t wl2 = transposed(B + "inter_linear.weight", 64, 64, 64);
        pk.bind(&W.wl2_t, wl2);
        pk.bind(&W.bl2, pk.plain(B + "inter_linear.bias", 64));
        // Q | K | V projections -> one [64][112] k-major matrix
        const int64_t wqkv = pk.alloc(64 * NQKV), bqkv = pk.alloc(NQKV), slopes = pk.alloc(4);
        auto proj = [&](const std::string& mod, int rows, int col0, int slope_idx) {
            pk.repacked(B + mod + ".0.weight", (int64_t)rows * 64, [wqkv, rows, col0](const float* s, float* d) {
                for (int r = 0; r < rows; ++r)
                    for (int k = 0; k < 64; ++k) d[wqkv + (int64_t)k * NQKV + col0 + r] = s[r * 64 + k];
            });
            pk.repacked(B + mod + ".0.bias", rows, [bqkv, rows, col0](const float* s, float* d) {
                memcpy(d + bqkv + col0, s, rows * sizeof(float));
            });
            pk.repacked(B + mod + ".1.weight", 1, [slopes, slope_idx](const float* s, float* d) { d[slopes + slope_idx] = s[0]; });
        };
        proj("attn_conv_Q", NHEAD * QE, 0, 0);
        proj("attn_conv_K", NHEAD * QE, NHEAD * QE, 1);
        proj("attn_conv_V", NHEAD * VD, 2 * NHEAD * QE, 2);
        pk.bind(&W.wqkv_t, wqkv); pk.bind(&W.bqkv, bqkv); pk.bind(&W.slopes, slopes);
        const int64_t slope_vec = pk.alloc(NQKV);
        pk.bind(&W.slope_vec, slope_vec);
        const int64_t midp = pk.alloc(MID_PACK);
        pk.bind(&W.mid_pack, midp);
        e->mid_src.push_back({wl1, wih2, whh2t, wl2, wqkv, midp, slopes, slope_vec});
        pk.bind(&W.lnq_g, pk.plain(B + "attn_conv_Q.3.norm.weight", QK_DIM));
        pk.bind(&W.lnq_b, pk.plain(B + "attn_conv_Q.3.norm.bias", QK_DIM));
        pk.bind(&W.lnk_g, pk.plain(B + "attn_conv_K.3.norm.weight", QK_DIM));
        pk.bind(&W.lnk_b, pk.plain(B + "attn_conv_K.3.norm.bias", QK_DIM));
        pk.bind(&W.lnv_g, pk.plain(B + "attn_conv_V.3.norm.weight", V_DIM));
        pk.bind(&W.lnv_b, pk.plain(B + "attn_conv_V.3.norm.bias", V_DIM));
        const int64_t wp = transposed(B + "attn_concat_proj.0.weight", 64, 64, 64);
        pk.bind(&W.wp_t, wp);
        pk.bind(&W.bp, pk.plain(B + "attn_concat_proj.0.bias", 64));
        pk.repacked(B + "attn_concat_proj.1.weight", 1, [slopes](const float* s, float* d) { d[slopes + 3] = s[0]; });
        pk.bind(&W.lnp_g, pk.plain(B + "attn_concat_proj.3.norm.weight", FC));
        pk.bind(&W.lnp_b, pk.plain(B + "attn_concat_proj.3.norm.bias", FC));
        // tensor-core B operands of this block, in PL_* order
        auto reg = [&](int64_t wt, int K, int N, int ld) { e->plane_of.push_back(pk.plane(wt, K, N, ld)); };
        reg(wih1, 64, 512, 64); reg(wl1, 128, 64, 128); reg(wih2, 64, 256, 64); reg(wl2, 64, 64, 64); reg(wqkv, 64, NQKV, 64);
        reg(wih2, 64, 256, 128);
        pk.plane(whh2t, 64, 256, 128, 64);      // [W_ih | W_hh]: k = [x | h], one plane
        reg(wp, 64, 64, 64);
    }
}

// ---- the call's form: predicates shared by the chain (chain_form), the workspace and the entry points ------------------
constexpr int64_t TC_MIN_ROWS = 2048;      // calls of more rows run their dense contractions on the tensor cores: below this
                                           // the 16-row CUDA-core tiles win (one streaming frame = 97 rows)
// many rows (whole utterances, offline batches, many streams): the dense contractions run on the tensor cores
static bool tc_form(int B, int T) { return (int64_t)B * T * NF > TC_MIN_ROWS; }
// one-frame calls: the row-local middle of every block runs as fused kernels (mid_kernel.cuh).  (Taps want the
// intermediate activations of the generic chain, so they keep it.)
static bool row_mid_form(int T, uint32_t flags) { return T == 1 && !(flags & L2H_FLAG_TAPS); }
// both: the middle as tensor-core GEMMs and the cell update
static bool tc_mid_form(int B, int T, uint32_t flags) { return tc_form(B, T) && row_mid_form(T, flags); }

// ---- workspace carve-up (floats) ---------------------------------------------------------------
struct Workspace {
    int64_t X, GX, Y, Z, Q, KALL, VALL, PRE, QKVRAW, TAPS, HG, LISTS, total;
};

static Workspace carve(int n_blocks, int B, int T, uint32_t flags) {
    Workspace ws;
    const int64_t rows = (int64_t)B * T * NF;
    int64_t cur = 0;
    auto alloc = [&](int64_t n) { int64_t o = cur; cur = (cur + n + 31) & ~int64_t(31); return o; };
    ws.X = alloc(rows * 64);
    ws.GX = alloc(rows * 512);
    ws.Y = alloc(rows * 128);
    ws.Z = alloc(rows * 64);
    ws.Q = alloc((int64_t)B * NHEAD * T * QK_LD);
    ws.KALL = alloc(T > 1 ? (int64_t)B * NHEAD * (ATT - 1 + T) * QK_LD : 0);
    ws.VALL = alloc(T > 1 ? (int64_t)B * NHEAD * (ATT - 1 + T) * V_DIM : 0);
    ws.PRE = alloc((int64_t)B * FC);
    ws.QKVRAW = alloc(rows * NQKV);
    ws.TAPS = alloc((flags & L2H_FLAG_TAPS) ? (int64_t)(1 + 3 * n_blocks) * rows * 64 : 0);
    // the listed records' carried inter-LSTM state of every block for a slot-list call (gather_h_kernel): h for one-hop
    // calls in the tensor-core form, h and c ([n_blocks][B][97][64] each) for every multi-hop call
    ws.HG = alloc((T > 1 ? 2 : tc_mid_form(B, T, flags) ? 1 : 0) * (int64_t)n_blocks * B * FC);
    // a call over listed groups or target rows (l2h_sep_forward_targets_groups / _rows): the lists target_lists_kernel
    // builds, five int32 per target row and one more (records, hops, owners, the leads of at most B listeners, the clamped
    // offsets).  Reserved for every call, so that one size query serves every kind of call.
    ws.LISTS = alloc(5 * (int64_t)B + 1);
    ws.total = (cur + 511) & ~int64_t(511);      // a multiple of one GX row: pipelined hops address their slots as rows of one tensor
    return ws;
}

// cudaFuncSetAttribute applies to the CURRENT device: keep one flag per device ordinal
static bool g_attr_done[64] = {};
static int g_tail_clusters[64] = {};     // how many 16-CTA tail_kernel clusters the device can hold at once (0: cannot be scheduled)
static int set_attrs() {
    int dev_ord = 0;
    CK(cudaGetDevice(&dev_ord));
    if (dev_ord < 0 || dev_ord >= 64) return fail(1, "device ordinal out of range");
    if (g_attr_done[dev_ord]) return 0;
    CK(set_sep_smem<int64_t>());
    CK(set_sep_smem<Records>());      // the slot-list forms (l2h_sep_forward_slots)
    CK(set_mid_split_smem());
    CK(configure_rows_gemm());
    CK(configure_lstm());
    CK(umma::configure());
    CK(configure_tc_lstm());
    g_tail_clusters[dev_ord] = set_tail_attrs();
    g_attr_done[dev_ord] = true;
    return 0;
}


// ---- dense contractions on the tensor cores (csrc/umma_gemm.cuh) for calls with many rows --------------------------
enum { PL_IH1 = 0, PL_L1, PL_IH2, PL_L2, PL_QKV, PL_CAT, PL_P, PL_PER_BLOCK };

static umma::BPlanes tc_planes(const SepEngine* e, int blk, int which, int ld) {
    return e->pack.bplanes(e->plane_of[(size_t)blk * PL_PER_BLOCK + which], ld);
}

// C[rows][N] = epi(LN?(A[rows][lda, first K]) W^T + bias) (+ R), plain row-major rows
static int tc_rows_gemm(SepEngine* e, int blk, int which, const float* A, int64_t lda, int K, int N, const float* ln_g, const float* ln_b,
                        const float* bias, const float* prelu_vec, const float* R, float* C, int64_t ldc, int64_t rows, cudaStream_t st,
                        bool pdl, const float* prelu_scalar = nullptr) {
    umma::GemmDesc g;
    g.a0.base = A; g.a0.channels = K; g.a0.n_pos = rows; g.a0.pos_stride = lda;
    umma::set_plain_chunks(g, K, ln_g != nullptr);
    g.ln_g = ln_g; g.ln_b = ln_b;
    g.rows_per_seq = (int)rows; g.nseq = 1;
    g.b = tc_planes(e, blk, which, K); g.N = N; g.K = K; g.passes = e->tc_passes;
    g.bias = bias; g.prelu_vec = prelu_vec; g.prelu = prelu_scalar; g.R = R; g.C = C; g.ldc = ldc;
    g.pdl = pdl;
    std::string why;
    const cudaError_t ce = umma::launch(g, st, &why);
    if (ce != cudaSuccess) return fail(3, std::string("umma_gemm: ") + cudaGetErrorString(ce) + " " + why);
    return 0;
}

struct Profiler {                      // per-kernel device times via CUDA events on the launching stream
    std::vector<cudaEvent_t> ev;
    std::vector<const char*> names;
    int used = 0;
    int mark(const char* name, cudaStream_t st) {
        if (used == (int)ev.size()) { cudaEvent_t e; CK(cudaEventCreate(&e)); ev.push_back(e); }
        CK(cudaEventRecord(ev[used++], st));
        names.push_back(name);
        return 0;
    }
};

struct ChainArgs {
    const float* x; int64_t xbs, xcs; int x_len;
    const float* emb; float* state;
    float* y; int64_t ybs, ycs; int y_len;
    int B, T; float* wsp; size_t ws_bytes; uint32_t flags; int pos_rel;
    Profiler* prof = nullptr;
    const uint8_t* active = nullptr;     // one-hop calls: [B] device mask of the streams that advance (null: all)
    const int32_t* slots = nullptr;      // [B] device list, row b -> record slots[b] (null: row b -> record b); with targets > 1
                                         // the [B / targets] group list of l2h_sep_forward_targets_groups; with targets == 0
                                         // the [B] record list of l2h_sep_forward_targets_rows
    int state_batch = 0;                 // records in the state (slot lists only)
    const int32_t* hops = nullptr;       // slot lists: [B] device list of the frames each row advances (null: all T); per group
                                         // or listener (one per mixture) with targets != 1
    int targets = 1;                     // l2h_sep_forward_targets: rows per mixture (B counts target rows; x has B / targets);
                                         // 0: per listener, from `offsets`
    const int32_t* offsets = nullptr;    // targets == 0: [calls + 1] device list, mixture i owns target rows offsets[i] ..
    int calls = 0;                       // offsets[i+1]-1 (l2h_sep_forward_targets_rows); calls: the mixtures
    float* hist = nullptr;               // a block-0 history [state_batch][hist_frames][97*64]: listed rows calls write their
    int hist_frames = 0;                 // leads' frames into it, joins replay frames from it
    const int32_t* leads = nullptr;      // a join (l2h_sep_join_targets): [B] device list, row j replays the history of leads[j]
    int32_t* used = nullptr;             // ... and writes the frames it replays here (may be null)
    int join_frames = 0;                 // ... at most this many (0: a cold join)
};

// few streams, one hop (the latency path): everything after the BiLSTM as one 16-CTA cluster kernel per stream, while all
// B clusters of the launch are resident at once
static bool tail_fits(const SepEngine* e, int B) {
    int dev_ord = 0;
    cudaGetDevice(&dev_ord);
    return e->use_tail && dev_ord >= 0 && dev_ord < 64 && B <= g_tail_clusters[dev_ord];
}

// The form of one call, chosen once from its rows (B, T), its flags and the engine's options.  Block 0 of a targets call
// runs these same forms over the mixtures' rows; grids follow the rows of the block being launched.
struct RecForm {
    bool tc;       // the recurrence on the tensor cores (enough sequences to fill the GPU with 32-sequence CTAs), else lstm.cuh
    bool fused;    // ... with LayerNorm and W_ih inside the recurrence kernel (tc_lstm_x_kernel, option "fuse_ih")
};
struct ChainForm {
    bool row_mid, tc, tc_mid, fused_tail;
    bool mid_split;     // row_mid: mid_a / mid_b / mid_c instead of one mid_kernel (mid_split_for_throughput)
    bool walkers;       // front_many_kernel / back_many_kernel: CTAs (clusters) walk (stream, chunk-of-frames) items
    bool qkv_many;      // many frames: the persistent qkv_many_kernel, on at most qkv_ctas CTAs (one wave)
    int qkv_ctas;
    AttnForm attn;      // clusters while they fit one wave (attn_splits), else attn_tile_kernel where enough query tiles fill the
                        // GPU (one pass over 57 rows serves 8 queries), else attn_kernel
    RecForm intra, inter;
    // programmatic dependent launch pays on the latency chain of a few rows; with many rows early-launched dependents park
    // on the SMs the big kernels need, so tensor-core chains take it only where option "tc_pdl" asks: bit 0 the many-stream
    // mid section, bit 1 W_ih and the out projection + its LayerNorm kernel, bit 2 the persistent qkv kernel
    bool pdl, mid_pdl, gemm_pdl, qkv_pdl;
};

template <class Map>
static ChainForm chain_form(const SepEngine* e, int B, int T, uint32_t flags, bool profiled) {
    ChainForm f{};
    f.row_mid = row_mid_form(T, flags);
    f.tc = tc_form(B, T);
    f.tc_mid = tc_mid_form(B, T, flags);
    f.fused_tail = f.row_mid && !f.tc && tail_fits(e, B);
    f.mid_split = mid_split_for_throughput(B);
    f.walkers = (T > 1 || f.tc) && e->use_back_many;
    f.qkv_many = f.tc && (int64_t)B * T >= NUM_SMS;
    if (f.qkv_many) {
        static int wave[64] = {};
        f.qkv_ctas = resident_ctas(wave, qkv_many_kernel_t<Map>, QKV_THREADS, QKV_MANY_SMEM);
    }
    const bool attn_tiled = T > 1 && (int64_t)B * NHEAD * ((T + ATT_TQ - 1) / ATT_TQ) >= NUM_SMS;
    f.attn = attn_splits(B, T) > 1 ? AttnForm::cluster : attn_tiled ? AttnForm::tile : AttnForm::query;
    const auto rec = [e](int64_t seqdirs) { const bool tc = seqdirs >= e->tcl_min_seqdirs; return RecForm{tc, tc && e->fuse_ih}; };
    f.intra = rec((int64_t)B * T * 2);      // (stream, frame) sequences over F, both directions
    f.inter = rec((int64_t)B * NF);         // (stream, bin) sequences over T
    f.pdl = e->use_pdl && !profiled && !(flags & L2H_FLAG_TAPS) && !f.tc;
    f.mid_pdl = (e->tc_pdl & 1) != 0 && !profiled;
    f.gemm_pdl = (e->tc_pdl & 2) != 0 && !profiled;
    f.qkv_pdl = (e->tc_pdl & 4) != 0 && !profiled;
    return f;
}

// The rows one block runs over: the call's, or for block 0 of a targets call the mixtures' (Chain::rows_of)
template <class Map>
struct BlockRows {
    int B;              // streams
    int64_t rows;       // B * T * 97
    int64_t ss;         // record stride
    Map recs;           // record map
    float* X;           // the block's input and output
    bool ih_written;    // GX holds the intra input projection already: front1_kernel / the previous tail_kernel wrote it
    int gate;           // 1: this block's attn_out (tail_kernel) builds the speaker gate
};

#define MARK(name) do { if (a.prof) { if (int _rc = a.prof->mark(name, st)) return _rc; } } while (0)

// One call's chain: its arguments, form and workspace, and the steps enqueue_chain_t takes in several places or in one
// record map's form only
template <class Map>
struct Chain {
    static constexpr bool slots = std::is_same_v<Map, Records>;
    SepEngine* e; const ChainArgs& a; cudaStream_t st; const ChainForm& f; Map recs;
    int K;              // targets per mixture; 0: per listener (l2h_sep_forward_targets_rows)
    int M;              // mixtures: the rows of block 0 when the chain fans out
    bool fans;          // several targets per mixture: block 0 runs over the M mixtures, fan_out() makes the target rows
    int64_t ss;         // record stride
    Map lead;           // fans: the record map of block 0's rows, the mixtures' lead records (rows_of)
    int64_t lead_ss;    // ... and its record stride
    float *X, *GX, *Y, *Z, *Q, *KALL, *VALL, *PRE, *QKVRAW, *TAPS, *HG, *CG, *sbase;
    float* X0;          // fans: block 0's input and output, the mixtures' rows
    int32_t* lists;     // listed groups or rows: the lists target_lists() builds (target_lists_kernel), B entries each:
                        // the target rows' records, their hops, their owners, then the M leads and the M + 1 row offsets
    bool joins;         // a join (l2h_sep_join_targets): no front and no block 0; X0 holds frames of the leads' histories
    int tap = 0;

    Chain(SepEngine* e_, const ChainArgs& a_, cudaStream_t st_, const ChainForm& f_, Map recs_, const Workspace& ws)
        : e(e_), a(a_), st(st_), f(f_), recs(recs_), K(a_.targets), M(K > 0 ? a_.B / K : a_.calls), fans(K != 1),
          ss(stream_stride(e_->n_blocks)), joins(a_.leads != nullptr) {
        float* w = a.wsp;
        X = w + ws.X; GX = w + ws.GX; Y = w + ws.Y; Z = w + ws.Z; Q = w + ws.Q; KALL = w + ws.KALL; VALL = w + ws.VALL;
        PRE = w + ws.PRE; QKVRAW = w + ws.QKVRAW; TAPS = w + ws.TAPS; HG = w + ws.HG;
        CG = HG + (int64_t)e->n_blocks * a.B * FC;
        lists = reinterpret_cast<int32_t*>(w + ws.LISTS);
        sbase = a.state + sizeof(StateHeader) / 4;
        if constexpr (slots) { lead = Records{ss, lists + 3 * (int64_t)a.B, a.state_batch, a.hops, a.T}; lead_ss = ss; }
        else { lead = recs * K; lead_ss = ss * K; }
        // block 0's rows go in room of GX that block 0 leaves unused; with more than 8/9 as many mixtures as target rows
        // (many single-target listeners) there is none, and they go in X, which fan_out() moves to GX before fanning out
        const int64_t rows0 = (int64_t)M * a.T * NF;
        X0 = rows0 * (512 + 64) <= (int64_t)a.B * a.T * NF * 512 ? GX + rows0 * 512 : X;
    }

    // Several targets per mixture (l2h_sep_forward_targets): B counts target rows, K per mixture, row i*K + k = target k of
    // mixture i.  The front and block 0 do not depend on the speaker (its gate applies after block 0), so they run once
    // per mixture: over M = B / K rows, on the lead records i*K (record stride K*ss), without the gate, into X0.
    // fan_out() then builds every target row's gate memo and its gated copy of block 0's output in X, and blocks 1 ..
    // n_blocks-1 and the back run over all B rows.  Every form was chosen for the B rows, and block 0 runs those same
    // forms, so a target row gets the arithmetic of a dense call with its mixture duplicated.
    // Over listed groups or rows (l2h_sep_forward_targets_groups / _rows) block 0's map is the lead list target_lists()
    // builds, with the listeners' hop counts, and the target rows' map is its record list: a listener's rows need not be
    // K, adjacent or in order.
    BlockRows<Map> rows_of(int b) const {
        const bool lead_rows = fans && b == 0;
        BlockRows<Map> r{lead_rows ? M : a.B, 0, lead_rows ? lead_ss : ss, lead_rows ? lead : recs, lead_rows ? X0 : X,
                         f.fused_tail && !fans_out_before(b), (b == 0 && e->n_blocks > 1 && !fans) ? 1 : 0};
        r.rows = (int64_t)r.B * a.T * NF;
        return r;
    }
    bool fans_out_before(int b) const { return fans && b == 1; }      // b == n_blocks: before the back
    int fan_out() {
        const float* x0 = X0;
        if (X0 == X) {      // block 0 ran in X: GX is free after it
            CK(cudaMemcpyAsync(GX, X, (size_t)M * a.T * FC * sizeof(float), cudaMemcpyDeviceToDevice, st));
            x0 = GX;
        }
        const int32_t* owner = nullptr;      // dense targets: row r belongs to mixture r / K
        if constexpr (slots) {
            owner = lists + 2 * (int64_t)a.B;
            // a rows call with a history: block 0's frames of every lead into its ring
            if (a.hist && !joins) CK(launch_history_put(f.pdl, st, M, x0, a.state, lead, a.hist, a.hist_frames, a.T));
        }
        // a join built its rows' gate memos before the chain (enqueue_join)
        if (!joins) CK(launch_spk_gate(f.pdl, st, a.B, a.emb, PRE, a.state, recs, e->w));
        CK(launch_gate_fanout(f.pdl, st, a.B, x0, X, (const float*)a.state, recs, owner, K, a.T, e->n_blocks > 1 ? 1 : 0));
        MARK("gate_fanout");
        return 0;
    }
    // listed groups or rows: the target rows' lists and the leads, before any kernel reads them
    int target_lists() {
        if constexpr (slots) {
            if (joins) {      // the lists and the fresh records are join_start_kernel's (enqueue_join); here block 0's output
                              // of the replayed frames, from the leads' histories
                CK(launch_history_get(f.pdl, st, a.B, a.hist, a.hist_frames, a.state, recs, a.leads, X0, a.T));
                MARK("history_get");
            } else if (fans) {
                CK(launch_target_lists(st, a.offsets ? a.slots : nullptr, a.offsets, a.offsets ? nullptr : a.slots, a.hops, M, K, a.B,
                                       a.state_batch, lists));
                MARK("target_lists");
            }
        }
        return 0;
    }

    int do_tap() {
        if (a.flags & L2H_FLAG_TAPS) {
            const int64_t rows = (int64_t)a.B * a.T * NF;
            CK(cudaMemcpyAsync(TAPS + (int64_t)tap * rows * 64, X, rows * 64 * sizeof(float), cudaMemcpyDeviceToDevice, st));
            ++tap;
        }
        return 0;
    }

    // block b's dense layer `which` over R's rows, on the tensor cores or as the CUDA-core rows GEMM:
    // LN -> W_ih (PL_IH1, PL_IH2: X -> GX) or Linear + residual (PL_L1, PL_L2: Y -> X)
    int dense(int b, int which, const BlockRows<Map>& R, bool pdl) {
        const BlockWeights& W = e->bw[b];
        GemmArgs g{};
        switch (which) {
            case PL_IH1:
                g.A = R.X; g.lda = 64; g.Wt = W.wih1_t; g.bias = W.b1; g.C = GX; g.ldc = 512; g.ln_g = W.ln1_g; g.ln_b = W.ln1_b; g.N = 512;
                g.K = 64; break;
            case PL_L1: g.A = Y; g.lda = 128; g.Wt = W.wl1_t; g.bias = W.bl1; g.C = R.X; g.ldc = 64; g.R = R.X; g.N = 64; g.K = 128; break;
            case PL_IH2:
                g.A = R.X; g.lda = 64; g.Wt = W.wih2_t; g.bias = W.b2; g.C = GX; g.ldc = 256; g.ln_g = W.ln2_g; g.ln_b = W.ln2_b; g.N = 256;
                g.K = 64; break;
            default: g.A = Y; g.lda = 64; g.Wt = W.wl2_t; g.bias = W.bl2; g.C = R.X; g.ldc = 64; g.R = R.X; g.N = 64; g.K = 64; break;
        }
        if (f.tc) return tc_rows_gemm(e, b, which, g.A, g.lda, g.K, g.N, g.ln_g, g.ln_b, g.bias, nullptr, g.R, g.C, g.ldc, R.rows, st, pdl);
        g.M = (int)R.rows;
        CK(launch_rows_gemm(g, st, pdl));
        return 0;
    }

    // LayerNorm + W_ih + the recurrence of block b's intra (PL_IH1) or inter (PL_IH2) LSTM: one tensor-core kernel
    // (no [rows x 512] projection in HBM), or the projection (unless written already), the ragged rows' gate mask and the
    // recurrence
    int ln_ih_recurrence(int b, const BlockRows<Map>& R, int which, const LstmArgs& l) {
        const bool inter = which == PL_IH2;
        const RecForm rf = inter ? f.inter : f.intra;
        const BlockWeights& W = e->bw[b];
        if (rf.fused) {
            tcl::LstmXArgs xa{};
            xa.l = l; xa.x = R.X; xa.x_ld = 64;
            xa.wih_hi = e->pack.planes + e->plane_of[(size_t)b * PL_PER_BLOCK + which]; xa.wih_lo = xa.wih_hi + e->pack.planes_total;
            xa.bias = inter ? W.b2 : W.b1; xa.ln_g = inter ? W.ln2_g : W.ln1_g; xa.ln_b = inter ? W.ln2_b : W.ln1_b;
            if constexpr (slots) { if (inter) xa.steps = R.recs.hops; }      // ragged rows: masked inside
            CK(launch_tc_lstm_x(xa, e->tc_passes, st, false));
            MARK(inter ? "gemm_ih_inter" : "gemm_ih_intra");
        } else {
            if (!R.ih_written) {      // a tensor-core chain's intra W_ih takes "tc_pdl" bit 1
                if (int rc = dense(b, which, R, f.tc && !inter ? f.gemm_pdl : f.pdl)) return rc;
            }
            MARK(inter ? "gemm_ih_inter" : "gemm_ih_intra");
            if constexpr (slots) {
                if (inter && R.recs.hops) CK(launch_inter_gate_mask(st, R.B, GX, R.recs, a.T));
            }
            if (rf.tc) CK(launch_tc_lstm(l, e->tc_passes, st, f.pdl));
            else CK(launch_lstm_rec(l, st, f.pdl, l.nseq / R.B * a.B));      // the form of the call's sequences
        }
        MARK(inter ? "lstm_inter" : "lstm_intra");
        return 0;
    }

    // Slot lists: one-hop tensor-core chains read the listed records' h of every block for the inter-step GEMMs, and
    // multi-hop calls carry their (h, c) through the inter recurrences, from a copy in the workspace (HG, CG) that
    // gather_hc() takes before block 0 and scatter_hc() stores back after the last block's inter recurrence.  Block b's
    // part holds the rows of rows_of(b) (inter_hc): over listed groups or rows, block 0's part holds the lead rows.
    // hc_copy: gather_h_kernel or scatter_hc_kernel over the blocks from b0 on that share rows_of(b0)'s record map
    // (launch_gather_h / launch_scatter_hc: block b0 of the records, block b0's part of HG and CG).
    int hc_copy(bool scatter, int b0) {
        const BlockRows<Map> R = rows_of(b0);
        const int nb = (fans && b0 == 0) ? 1 : e->n_blocks - b0;
        if (scatter) CK(launch_scatter_hc(st, b0, a.state, R.recs, nb, R.B, HG, CG));
        else CK(launch_gather_h(st, b0, a.state, R.recs, nb, R.B, HG, a.T > 1 ? CG : nullptr));
        return 0;
    }
    int gather_hc() {
        if constexpr (slots) {
            if (f.tc_mid || a.T > 1) {
                if (!joins) { if (int rc = hc_copy(false, 0)) return rc; }
                if (fans && e->n_blocks > 1) { if (int rc = hc_copy(false, 1)) return rc; }
            }
        }
        return 0;
    }
    void inter_hc(LstmArgs& l, int b, const BlockRows<Map>& R) const {      // where block b's inter recurrence carries (h, c)
        if constexpr (slots) {
            l.h_state = HG + (int64_t)b * R.B * FC;
            l.c_state = CG + (int64_t)b * R.B * FC;
            l.hc_outer_stride = FC;
        } else {
            l.h_state = sbase + ST_BLK + (int64_t)b * BK_STRIDE + BK_H;
            l.c_state = sbase + ST_BLK + (int64_t)b * BK_STRIDE + BK_C;
            l.hc_outer_stride = R.ss;
        }
    }
    int h_last(int b, const BlockRows<Map>& R) {      // a ragged row's h is that of its own last frame
        if constexpr (slots) {
            if (R.recs.hops)
                CK(launch_inter_h_last(st, R.B, Y, HG + (int64_t)b * R.B * FC, R.recs, a.T));
        }
        return 0;
    }
    int scatter_hc() {
        if constexpr (slots) {
            if (!joins) { if (int rc = hc_copy(true, 0)) return rc; }
            if (fans && e->n_blocks > 1) { if (int rc = hc_copy(true, 1)) return rc; }
        }
        return 0;
    }
};

// Map: the record stride (dense calls) or Records (slot-list calls), see row_record in sep_kernels.cuh
template <class Map>
static int enqueue_chain_t(SepEngine* e, const ChainArgs& a, cudaStream_t st, Map recs) {
    const int T = a.T;
    if (!e->pack.committed) return fail(4, "weights not committed");
    if (a.B <= 0 || T <= 0) return fail(1, "batch and frames must be positive");
    const Workspace ws = carve(e->n_blocks, a.B, T, a.flags);
    if ((size_t)ws.total * sizeof(float) > a.ws_bytes) return fail(1, "workspace too small");
    if (int rc = set_attrs()) return rc;
    if ((int64_t)a.B * T * NF > 0x7fffffff / 2) return fail(1, "batch*frames too large for one call; split the batch");
    const ChainForm f = chain_form<Map>(e, a.B, T, a.flags, a.prof != nullptr);
    Chain<Map> c(e, a, st, f, recs, ws);
    MARK("start");
    if (int rc = c.target_lists()) return rc;
    if (int rc = c.gather_hc()) return rc;
    const BlockRows<Map> R0 = c.rows_of(0);           // the front runs over block 0's rows
    const int gate_ctas = c.fans ? 0 : 1;             // the front's speaker-gate memo CTAs (one per row); fan_out() builds them here
    if (c.joins) {
        // a join starts at block 1: target_lists() filled block 0's output from the histories
    } else if (f.fused_tail) {      // the frame as 13 row tiles: spectrum of the tile's bins, conv, and block 0's input projection
        CK(launch_front1(false, st, R0.B, gate_ctas, a.x, a.xbs, a.xcs, a.x_len, R0.X, a.state, R0.recs, e->w, e->bw[0], c.GX, a.pos_rel,
                         a.emb, c.PRE, a.active));
    } else if (f.walkers) {
        CK(launch_front_many(false, st, gate_ctas, front_many_walk(R0.B, T), a.x, a.xbs, a.xcs, a.x_len, R0.X, a.state, R0.recs, e->w, T,
                             a.pos_rel, a.emb, c.PRE, R0.B, a.active));
    } else {
        CK(launch_front(false, st, R0.B, gate_ctas, a.x, a.xbs, a.xcs, a.x_len, R0.X, a.state, R0.recs, e->w, T, a.pos_rel, a.emb, c.PRE,
                        0, 1, 0, a.active));
    }
    MARK("front");
    if (int rc = c.do_tap()) return rc;

    for (int b = c.joins ? 1 : 0; b < e->n_blocks; ++b) {
        if (c.fans_out_before(b)) { if (int rc = c.fan_out()) return rc; }
        const BlockRows<Map> R = c.rows_of(b);
        const BlockWeights& W = e->bw[b];
        // ---- intra: LN -> W_ih (both directions) -> BiLSTM over F -> Linear -> +res ------------
        LstmArgs l{};
        l.gx = c.GX; l.gx_ld = 512; l.out = c.Y; l.out_ld = 128; l.whh = W.whh1;
        l.nseq = R.B * T; l.L = NF; l.inner_count = 1; l.outer_stride = NF; l.inner_stride = 0; l.step_stride = 1;
        l.ndir = 2;
        if (int rc = c.ln_ih_recurrence(b, R, PL_IH1, l)) return rc;
        if (f.tc_mid) {
            // many streams, one hop: the row-local middle of the block as four tensor-core GEMMs and the cell update.
            // The inter-LSTM step is ONE GEMM over the concatenated k = [LN(x) | h_prev] (h read in place from the
            // per-stream state records through a strided tensor map) against [W_ih | W_hh].
            if (int rc = c.dense(b, PL_L1, R, f.mid_pdl)) return rc;
            {
                umma::GemmDesc q;
                q.a0.base = R.X; q.a0.channels = 64; q.a0.n_pos = NF; q.a0.pos_stride = 64; q.a0.n_inner = R.B; q.a0.inner_stride = (int64_t)NF * 64;
                q.a1.base = c.sbase + ST_BLK + (int64_t)b * BK_STRIDE + BK_H;
                q.a1.channels = 64; q.a1.n_pos = NF; q.a1.pos_stride = 64; q.a1.n_inner = R.B; q.a1.inner_stride = R.ss;
                if (a.slots) { q.a1.base = c.HG + (int64_t)b * R.B * FC; q.a1.inner_stride = FC; }      // gathered by gather_hc()
                q.n_chunks = 2;
                q.chunks[0].c0 = 0; q.chunks[0].dp = 0; q.chunks[0].flags = 2;      // x: LayerNorm
                q.chunks[1].c0 = 0; q.chunks[1].dp = 0; q.chunks[1].flags = 1;      // h: second source
                q.ln_g = W.ln2_g; q.ln_b = W.ln2_b;
                q.rows_per_seq = NF; q.nseq = R.B;
                q.b = tc_planes(e, b, PL_CAT, 128); q.N = 256; q.K = 128; q.passes = e->tc_passes;
                q.bias = W.b2; q.C = c.GX; q.ldc = 256; q.c_seq_stride = (int64_t)NF * 256;
                q.pdl = f.mid_pdl;
                std::string why;
                const cudaError_t ce = umma::launch(q, st, &why);
                if (ce != cudaSuccess) return fail(3, std::string("umma_gemm (inter step): ") + cudaGetErrorString(ce) + " " + why);
            }
            CK(launch_lstm_cell_rows(f.mid_pdl, st, c.GX, a.state, R.recs, b, c.Y, R.rows, a.active));
            if (int rc = c.dense(b, PL_L2, R, f.mid_pdl)) return rc;
            if (int rc = tc_rows_gemm(e, b, PL_QKV, R.X, 64, 64, NQKV, nullptr, nullptr, W.bqkv, W.slope_vec, nullptr, c.QKVRAW, NQKV, R.rows,
                                      st, f.mid_pdl)) return rc;
            MARK("mid");
        } else if (f.row_mid && f.mid_split) {
            float* GI = c.GX; float* HN = c.GX + R.rows * 256;         // the BiLSTM is done with GX
            CK(launch_mid_a(f.pdl, st, c.Y, R.X, GI, W, R.B, 0, 1));
            CK(launch_mid_b(f.pdl, st, GI, HN, 0, 1, a.state, R.recs, b, W, R.B, a.active));
            CK(launch_mid_c(f.pdl, st, HN, R.X, c.QKVRAW, W, R.B, 0, 1));
            MARK("mid");
        } else if (f.fused_tail) {
            NextIh nx{};      // the next block's input projection, where that block reads it from GX
            if (b + 1 < e->n_blocks && c.rows_of(b + 1).ih_written) {
                const BlockWeights& Wn = e->bw[b + 1];
                nx.ln_g = Wn.ln1_g; nx.ln_b = Wn.ln1_b; nx.wih_t = Wn.wih1_t; nx.bias = Wn.b1; nx.GX = c.GX;
            }
            CK(launch_tail(f.pdl, st, R.B, c.Y, R.X, a.state, R.recs, b, W, nx, R.gate, 0, a.active));
            MARK("tail");
            if (int rc = c.do_tap()) return rc;
            continue;
        } else if (f.row_mid) {
            CK(launch_mid(f.pdl, st, c.Y, R.X, c.QKVRAW, a.state, R.recs, b, W, R.B, a.active));
            MARK("mid");
        } else {
            if (int rc = c.dense(b, PL_L1, R, f.pdl)) return rc;
            MARK("gemm_lin_intra");
            if (int rc = c.do_tap()) return rc;
            // ---- inter: LN -> W_ih -> LSTM over T with carried (h, c) -> Linear -> +res ------------
            l = LstmArgs{};
            l.gx = c.GX; l.gx_ld = 256; l.out = c.Y; l.out_ld = 64; l.whh = W.whh2;
            c.inter_hc(l, b, R);
            l.nseq = R.B * NF; l.L = T; l.inner_count = NF; l.outer_stride = (int64_t)T * NF; l.inner_stride = 1;
            l.step_stride = NF; l.ndir = 1;
            if (int rc = c.ln_ih_recurrence(b, R, PL_IH2, l)) return rc;
            if (int rc = c.h_last(b, R)) return rc;
            if (b == e->n_blocks - 1) { if (int rc = c.scatter_hc()) return rc; }
            if (int rc = c.dense(b, PL_L2, R, f.pdl)) return rc;
            MARK("gemm_lin_inter");
            if (int rc = c.do_tap()) return rc;
        }
        // ---- attention --------------------------------------------------------------------------
        if (T > 1) {
            CK(launch_kv_gather(f.pdl, st, R.B, a.state, R.recs, b, c.KALL, c.VALL, T));
            MARK("kv_gather");
        }
        if (f.tc && !f.tc_mid) {      // Q|K|V projections of all rows as one tensor-core GEMM (+ bias + PReLU per column)
            if (int rc = tc_rows_gemm(e, b, PL_QKV, R.X, 64, 64, NQKV, nullptr, nullptr, W.bqkv, W.slope_vec, nullptr, c.QKVRAW, NQKV, R.rows,
                                      st, false)) return rc;
        }
        if (f.qkv_many) {      // many frames: persistent form (LayerNorm parameters staged once per CTA), one wave
            const int grid_q = (int)std::min<int64_t>(f.qkv_ctas, (int64_t)R.B * T);
            CK(launch_qkv_many(f.qkv_pdl, st, grid_q, c.QKVRAW, c.Q, c.KALL, c.VALL, a.state, R.recs, b, W, T, R.B * T, a.active));
        } else {
            const bool pre = f.tc || f.row_mid;      // the projections are in QKVRAW already
            CK(launch_qkv(f.pdl, st, R.B, R.X, pre ? c.QKVRAW : nullptr, c.Q, c.KALL, c.VALL, a.state, R.recs, b, W, T, 0, a.active));
        }
        MARK("qkv");
        CK(launch_attention(f.attn, f.pdl, st, R.B, c.Q, c.KALL, c.VALL, a.state, R.recs, b, c.Z, T, 0));
        MARK("attn");
        if (f.tc) {      // Linear(64->64) + PReLU of all rows on the tensor cores, then LayerNorm(6208) + residual (+ gate) per frame
            if (int rc = tc_rows_gemm(e, b, PL_P, c.Z, 64, 64, 64, nullptr, nullptr, W.bp, nullptr, nullptr, c.Y, 64, R.rows, st, f.gemm_pdl,
                                      W.slopes + 3)) return rc;
            CK(launch_ln_frame_res(f.gemm_pdl, st, R.B, c.Y, R.X, a.state, R.recs, W, R.gate, T));
        } else {
            CK(launch_attn_out(f.pdl, st, R.B, c.Z, R.X, a.state, R.recs, W, R.gate, T));
        }
        MARK("attn_out");
        if (int rc = c.do_tap()) return rc;
    }
    if (c.fans_out_before(e->n_blocks)) { if (int rc = c.fan_out()) return rc; }
    if (f.walkers) {
        CK(launch_back_many(f.pdl, st, back_many_walk(a.B, T), c.X, a.y, a.ybs, a.ycs, a.y_len, a.state, recs, e->w, T, a.pos_rel, a.B,
                            a.active));
    } else {
        CK(launch_back(f.pdl, st, a.B, c.X, a.y, a.ybs, a.ycs, a.y_len, a.state, recs, e->w, T, a.pos_rel, 0, 1, 0, 0, a.active));
    }
    MARK("back");
    return 0;
}
#undef MARK

static int enqueue_chain(SepEngine* e, const ChainArgs& a, cudaStream_t st) {
    const int64_t ss = stream_stride(e->n_blocks);
    if (a.slots && a.targets != 1) {     // listed groups or rows: the target rows' record (and hop) lists that
                                         // Chain::target_lists builds in the workspace at the start of the call
        const int32_t* lists = reinterpret_cast<const int32_t*>(a.wsp + carve(e->n_blocks, a.B, a.T, a.flags).LISTS);
        return enqueue_chain_t(e, a, st, Records{ss, lists, a.state_batch, a.hops ? lists + a.B : nullptr, a.T});
    }
    if (a.slots) return enqueue_chain_t(e, a, st, Records{ss, a.slots, a.state_batch, a.hops, a.T});
    return enqueue_chain_t(e, a, st, ss);
}

// A join (l2h_sep_join_targets, rows a.B = J, frames a.T = max(1, a.join_frames)): the rows' fresh records at their leads'
// clocks and the rows' lists (join_start_kernel), their gate memos, and, when frames are replayed, the chain from block 1
// over them (Chain::joins) as a ragged listed-rows call: row j advances its used[j] frames.
static int enqueue_join(SepEngine* e, const ChainArgs& a, cudaStream_t st) {
    if (!e->pack.committed) return fail(4, "weights not committed");
    const Workspace ws = carve(e->n_blocks, a.B, a.T, a.flags);
    if ((size_t)ws.total * sizeof(float) > a.ws_bytes) return fail(1, "workspace too small");
    if (int rc = set_attrs()) return rc;
    const int64_t ss = stream_stride(e->n_blocks);
    int32_t* lists = reinterpret_cast<int32_t*>(a.wsp + ws.LISTS);
    CK(launch_join_start(st, a.B, a.state, ss, a.state_batch, a.slots, a.leads, a.join_frames, lists, a.used));
    CK(launch_spk_gate(false, st, a.B, a.emb, a.wsp + ws.PRE, a.state, Records{ss, lists, a.state_batch, nullptr, a.T}, e->w));
    if (a.join_frames == 0) return 0;      // a cold join
    return enqueue_chain_t(e, a, st, Records{ss, lists, a.state_batch, lists + a.B, a.T});
}

static int enqueue_call(SepEngine* e, const ChainArgs& a, cudaStream_t st) {
    return a.leads ? enqueue_join(e, a, st) : enqueue_chain(e, a, st);
}

// ---- wavefront pipeline over (block, frame) for one-frame calls ---------------------------------------
// Work item (block b, hop t) depends only on (b-1, t) and (b, t-1) (SURVEY.md 3.3), and inside a block
// only part of the work carries state from hop to hop:
//   A   = W_ih GEMM + 97-step BiLSTM + mid_a needs X_t only           -> PIPE_LANES hops of it run side by side
//   B1  = mid_b (inter-LSTM step)            carries (h, c)            -> serial per block
//   Bc  = mid_c (inter Linear + Q|K|V)       needs h'_t, X_t only
//   B2a = qkv + attention                    carries the K/V rings     -> serial per block
//   B2b = attn_out                           needs Z_t, X_t only
// A graph of K consecutive one-hop chains is captured on 1 + 3*(PIPE_LANES+3) + 1 streams with event edges
// for exactly these dependencies; hops flow through the stages like a systolic wavefront and the
// steady-state cost per hop is the slowest SERIAL stage instead of the whole chain.  Every hop owns a
// workspace slot; state addressing uses each stream's own clock (pos + frame_k, the parity of its calls); the
// clocks advance once, at the last hop of the graph.  The arithmetic and its order per stream are unchanged: results are
// bit-identical to running the hops one after the other (tests/test_sep_gpu.py).
constexpr int PIPE_MAX_FRAMES = 500;
constexpr int PIPE_LANES = 16;     // max hops of stage A (BiLSTM) in flight per block (engine->pipe_alanes used)
constexpr int PIPE_FLANES = 8;     // max front_kernel lanes (frames of a group do not depend on each other there)
constexpr int PIPE_BLANES = 6;     // max back_kernel lanes
constexpr int PIPE_BASE = 1 + PIPE_FLANES + PIPE_BLANES;
constexpr int PIPE_QLANES = 4;     // max qkv lanes (hops write different ring rows; RING - ATT = 6 may run ahead of the attention)
constexpr int PIPE_CLANES = 3;     // max mid_c lanes (no hop-to-hop dependency, not bound by the ring guard)
constexpr int PIPE_TLANES = 4;     // max attention lanes (attention only reads the rings)
constexpr int PIPE_OLANES = 4;     // max attn_out lanes (no hop-to-hop dependency)
constexpr int PIPE_PER_BLOCK = PIPE_LANES + 1 + PIPE_QLANES + PIPE_TLANES + PIPE_OLANES + PIPE_CLANES;   // A lanes, B1 (mid), Bq lanes (qkv), Ba lanes (attention), Bo lanes (attn_out)
constexpr int PIPE_STREAMS = PIPE_BASE + 3 * PIPE_PER_BLOCK;
constexpr int PIPE_MIDB_MAX = 8;   // max hops per mid_b launch
constexpr int PIPE_QKV_AHEAD = RING - ATT;         // qkv of hop t+3 overwrites a ring row hop t's attention still reads
static_assert(PIPE_STREAMS <= 128, "pipe_streams[]");

static int64_t pipe_slot_floats(SepEngine* e, int B) { return carve(e->n_blocks, B, 1, 0).total; }
// hops per pipelined graph: fill + drain cost one chain latency per graph, so as many as possible -- every hop
// in flight owns a workspace slot (350 KB per stream), which is what bounds it for many streams
static int pipe_frames_for(SepEngine* e, int B) {
    if (e->pipe_frames > 0) return e->pipe_frames;
    // every hop in flight owns a workspace slot: at most 24 GB of them, and never more than half of what the device
    // has free right now (the state, the caller's buffers and other tenants need room too)
    if (e->pipe_budget == 0) {               // asked once per handle: cudaMemGetInfo costs tens of microseconds per call
        e->pipe_budget = (int64_t)24 << 30;
        size_t free_b = 0, total_b = 0;
        if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess && free_b > 0) e->pipe_budget = std::min<int64_t>(e->pipe_budget, (int64_t)(free_b / 2));
    }
    const int64_t fit = e->pipe_budget / (pipe_slot_floats(e, B) * (int64_t)sizeof(float));
    return (int)std::max<int64_t>(2, std::min<int64_t>(PIPE_MAX_FRAMES, fit));
}
static int enqueue_pipeline(SepEngine* e, const ChainArgs& a, int K, cudaStream_t origin) {
    if (e->n_blocks != 3) return fail(1, "pipeline graph is specialised to 3 blocks");
    const int B = a.B;
    const Workspace ws = carve(e->n_blocks, B, 1, 0);
    const int64_t slot = ws.total;
    if ((size_t)slot * K * sizeof(float) > a.ws_bytes) return fail(1, "workspace too small for the pipelined stream");
    const int64_t ss = stream_stride(e->n_blocks);
    const int rows = B * NF;
    const AttnForm attn = attn_splits(B, 1) > 1 ? AttnForm::cluster : AttnForm::query;
    // programmatic dependent launch, per stage: the kernel's prologue (weight staging) overlaps its stream predecessor's
    // tail; every kernel reaches griddepcontrol.wait before it touches activations or state.  Off by default: a parked
    // dependent holds shared memory and CTA slots the running kernels need, on the serial stage too (mid_b -> mid_b of the
    // next batch): its 13 CTAs would sit on half an SM each while mid_a walks its batch
    const int ppdl = e->pipe_pdl;         // stage bit mask (bits: include/lookonce_b200.h, l2h_sep_set_option)
    const bool many = mid_split_for_throughput(B);
    float* state = a.state;
    const uint8_t* all_active = nullptr;      // every stream of a pipelined graph advances
    for (int i = 0; i < PIPE_STREAMS; ++i)
        if (!e->pipe_streams[i]) CK(cudaStreamCreateWithFlags(&e->pipe_streams[i], cudaStreamNonBlocking));
    size_t ev_used = 0;
    auto next_event = [&](cudaEvent_t* out) -> int {
        if (ev_used == e->pipe_events.size()) {
            cudaEvent_t ev;
            CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
            e->pipe_events.push_back(ev);
        }
        *out = e->pipe_events[ev_used++];
        return 0;
    };
    auto edge = [&](cudaStream_t from, cudaStream_t to) -> int {     // `to` continues after everything enqueued on `from`
        if (from == to) return 0;
        cudaEvent_t ev;
        if (int rc = next_event(&ev)) return rc;
        CK(cudaEventRecord(ev, from));
        CK(cudaStreamWaitEvent(to, ev, 0));
        return 0;
    };
    // stream map: [0] capture origin (fork / join / header advance), front lanes, back lanes, then per block:
    // PIPE_LANES x A, B1, B2a, B2b
    auto sFront = [&](int k) { return e->pipe_streams[1 + k % e->pipe_flanes]; };
    auto sBackL = [&](int k) { return e->pipe_streams[1 + PIPE_FLANES + k % e->pipe_blanes]; };
    auto sA = [&](int b, int lane) { return e->pipe_streams[PIPE_BASE + b * PIPE_PER_BLOCK + lane]; };
    auto sB1 = [&](int b) { return e->pipe_streams[PIPE_BASE + b * PIPE_PER_BLOCK + PIPE_LANES]; };
    auto sBq = [&](int b, int k) { return e->pipe_streams[PIPE_BASE + b * PIPE_PER_BLOCK + PIPE_LANES + 1 + k % e->pipe_qlanes]; };
    auto sBa = [&](int b, int k) { return e->pipe_streams[PIPE_BASE + b * PIPE_PER_BLOCK + PIPE_LANES + 1 + PIPE_QLANES + k % e->pipe_tlanes]; };
    auto sBo = [&](int b, int k) {
        return e->pipe_streams[PIPE_BASE + b * PIPE_PER_BLOCK + PIPE_LANES + 1 + PIPE_QLANES + PIPE_TLANES + k % e->pipe_olanes];
    };
    auto sBc = [&](int b, int k) {
        return e->pipe_streams[PIPE_BASE + b * PIPE_PER_BLOCK + PIPE_LANES + 1 + PIPE_QLANES + PIPE_TLANES + PIPE_OLANES + k % e->pipe_clanes];
    };
    // events: stage A (BiLSTM [+ mid_a]) done, qkv done, attention done, attn_out done -- per block and hop
    std::vector<std::vector<cudaEvent_t>> a_done(3, std::vector<cudaEvent_t>(K, nullptr));
    std::vector<std::vector<cudaEvent_t>> qkv_done(3, std::vector<cudaEvent_t>(K, nullptr));
    std::vector<std::vector<cudaEvent_t>> att_done(3, std::vector<cudaEvent_t>(K, nullptr));
    std::vector<std::vector<cudaEvent_t>> out_done(3, std::vector<cudaEvent_t>(K, nullptr));
    auto record = [&](cudaEvent_t* ev, cudaStream_t s) -> int {
        if (int rc = next_event(ev)) return rc;
        CK(cudaEventRecord(*ev, s));
        return 0;
    };
    for (int i = 1; i < PIPE_STREAMS; ++i)                             // fork: bring the worker streams into the capture
        if (int rc = edge(origin, e->pipe_streams[i])) return rc;
    // The serial stage (mid_b) takes `mb` consecutive hops per launch: its launch overhead and its 64 KB of
    // weights are paid once per batch, h stays in shared memory and c in registers from hop to hop.  A batch waits
    // for stage A of all its hops; the upstream block is that far ahead anyway once the pipeline is full.
    const int mb = many ? 1 : std::max(1, std::min(e->pipe_midb_hops, PIPE_MIDB_MAX));
    float* PRE = a.wsp + ws.PRE;                                       // speaker-gate scratch: front stream only
    for (int k0 = 0; k0 < K; k0 += mb) {
        const int k1 = std::min(K, k0 + mb);                           // this batch: hops [k0, k1)
        for (int b = 0; b < 3; ++b) {
            const BlockWeights& W = e->bw[b];
            // ---- stage A of the batch: ONE launch each of W_ih GEMM, BiLSTM and mid_a for its hops [k0, k1) (the hops'
            // workspace slots are `slot` floats apart: strided rows / sequences / hop index inside the kernels) ------------
            {
                const int nh = k1 - k0;
                float* wsp = a.wsp + (int64_t)k0 * slot;
                float* X = wsp + ws.X; float* GX = wsp + ws.GX; float* Y = wsp + ws.Y;
                cudaStream_t st_a = sA(b, (k0 / mb) % e->pipe_alanes);
                for (int k = k0; k < k1; ++k) {
                    if (b == 0) {
                        // x / y are the group's buffers; hop k works at sample offset k*128 (plus, with pos_rel, the clip
                        // position the device derives from the state header)
                        cudaStream_t sF = sFront(k);
                        // the speaker-gate memo CTA (blockIdx.x == 1) rides with hop 0 only: one builder of ST_GATE per group
                        CK(launch_front((ppdl & 1) != 0, sF, B, k == 0 ? 1 : 0, a.x, a.xbs, a.xcs, a.x_len, a.wsp + (int64_t)k * slot + ws.X,
                                        state, ss, e->w, 1, a.pos_rel, a.emb, PRE, k, K, k * HOP, all_active));
                        if (k == 0) {                  // ... and every attn_out lane of block 0 (the gate's only reader) waits for it once
                            cudaEvent_t gate_ev;
                            if (int rc = record(&gate_ev, sF)) return rc;
                            for (int ln = 0; ln < e->pipe_olanes; ++ln) CK(cudaStreamWaitEvent(sBo(0, ln), gate_ev, 0));
                        }
                        if (int rc = edge(sF, st_a)) return rc;
                    } else {
                        CK(cudaStreamWaitEvent(st_a, out_done[b - 1][k], 0));
                    }
                }
                GemmArgs g{};
                g.A = X; g.lda = 64; g.a_rows_per_seq = rows; g.a_seq_stride = slot;
                g.Wt = W.wih1_t; g.bias = W.b1; g.C = GX; g.ldc = 512; g.c_rows_per_seq = rows; g.c_seq_stride = slot;
                g.ln_g = W.ln1_g; g.ln_b = W.ln1_b; g.M = rows * nh; g.N = 512; g.K = 64;
                CK(launch_rows_gemm(g, st_a, (ppdl & 2) != 0, e->pipe_gemm_shape));
                LstmArgs l{};
                l.gx = GX; l.gx_ld = 512; l.out = Y; l.out_ld = 128; l.whh = W.whh1;
                l.nseq = B * nh; l.L = NF; l.inner_count = B; l.outer_stride = slot / 512; l.inner_stride = NF; l.step_stride = 1;
                l.out_outer_stride = slot / 128; l.out_inner_stride = NF; l.out_step_stride = 1; l.ndir = 2;
                CK(launch_lstm_rec(l, st_a, (ppdl & 4) != 0));
                // only the W_hh product + cell (mid_b) is serial per block; the rest rides on the parallel lanes.
                // GI / H' live in the hop's GX slot, which the BiLSTM has finished with.  One CTA per (stream, row
                // tile) walks the batch's hops: its 100 KB of weights are staged once per batch, not once per hop.
                CK(launch_mid_a((ppdl & 8) != 0, st_a, Y, X, GX, W, B, slot, nh));
                cudaEvent_t ev_a;
                if (int rc = record(&ev_a, st_a)) return rc;
                for (int k = k0; k < k1; ++k) a_done[b][k] = ev_a;
            }
            // ---- the serial stage: one launch for the batch ----------------------------------------------------
            CK(cudaStreamWaitEvent(sB1(b), a_done[b][k0], 0));
            {
                float* wsp = a.wsp + (int64_t)k0 * slot;
                float* GI = wsp + ws.GX; float* HN = GI + (int64_t)rows * 256;
                CK(launch_mid_b((ppdl & 16) != 0, sB1(b), GI, HN, slot, k1 - k0, state, ss, b, W, B, all_active));
            }
            cudaEvent_t midb_done;
            if (int rc = record(&midb_done, sB1(b))) return rc;
            // ---- mid_c for the whole batch (one launch), then per hop: qkv -> attention -> attn_out (lanes, ring guards) ----
            cudaStream_t st_c = sBc(b, k0 / mb);
            float* wsp0 = a.wsp + (int64_t)k0 * slot;
            CK(cudaStreamWaitEvent(st_c, midb_done, 0));
            CK(launch_mid_c((ppdl & 32) != 0, st_c, wsp0 + ws.GX + (int64_t)rows * 256, wsp0 + ws.X, wsp0 + ws.QKVRAW, W, B, slot,
                            k1 - k0));      // as mid_a: a CTA walks the hops of its tile
            cudaEvent_t midc_done;
            if (int rc = record(&midc_done, st_c)) return rc;
            for (int k = k0; k < k1; ++k) {
                float* wsp = a.wsp + (int64_t)k * slot;
                float* X = wsp + ws.X; float* Z = wsp + ws.Z; float* Q = wsp + ws.Q; float* QKVRAW = wsp + ws.QKVRAW;
                cudaStream_t st_q = sBq(b, k);
                CK(cudaStreamWaitEvent(st_q, midc_done, 0));
                // the ring row this hop's K/V overwrite was last read by the attention of hop k-3: it and every earlier
                // attention (one per attention lane) must be done
                for (int d = 0; d < e->pipe_tlanes && k - PIPE_QKV_AHEAD - 1 - d >= 0; ++d)
                    CK(cudaStreamWaitEvent(st_q, att_done[b][k - PIPE_QKV_AHEAD - 1 - d], 0));
                CK(launch_qkv((ppdl & 64) != 0, st_q, B, X, QKVRAW, Q, nullptr, nullptr, state, ss, b, W, 1, k, all_active));
                if (int rc = record(&qkv_done[b][k], st_q)) return rc;
                // the attention reads this hop's ring row and the 49 before it: the other qkv lanes' latest hops must be in
                cudaStream_t st_t = sBa(b, k);
                for (int d = 0; d < e->pipe_qlanes && d <= k; ++d) CK(cudaStreamWaitEvent(st_t, qkv_done[b][k - d], 0));
                CK(launch_attention(attn, (ppdl & 128) != 0, st_t, B, Q, nullptr, nullptr, state, ss, b, Z, 1, k));
                if (int rc = record(&att_done[b][k], st_t)) return rc;
                CK(cudaStreamWaitEvent(sBo(b, k), att_done[b][k], 0));
                CK(launch_attn_out((ppdl & 256) != 0, sBo(b, k), B, Z, X, state, ss, W, b == 0 ? 1 : 0, 1));
                if (int rc = record(&out_done[b][k], sBo(b, k))) return rc;
            }
        }
        for (int k = k0; k < k1; ++k) {
            float* X = a.wsp + (int64_t)k * slot + ws.X;
            cudaStream_t sBack = sBackL(k);
            // this hop's output and the three before it (deconv / overlap-add context) sit on different attn_out lanes
            for (int d = 0; d <= 3 && d <= k; ++d) CK(cudaStreamWaitEvent(sBack, out_done[2][k - d], 0));
            CK(launch_back((ppdl & 512) != 0, sBack, B, X, a.y, a.ybs, a.ycs, a.y_len, state, ss, e->w, 1, a.pos_rel, k, K, k * HOP, slot,
                           all_active));
        }
    }
    for (int i = 1; i < PIPE_STREAMS; ++i)                             // join
        if (int rc = edge(e->pipe_streams[i], origin)) return rc;
    advance_header_kernel<<<1, 256, 0, origin>>>(state, ss, B, K);       // every clock: pos += K, calls += 1, after every hop of the group
    CK(cudaGetLastError());
    return 0;
}

// kernel nodes of a captured graph (for the launch counter)
static int count_kernel_nodes(cudaGraph_t graph) {
    size_t n = 0;
    if (cudaGraphGetNodes(graph, nullptr, &n) != cudaSuccess || n == 0) return 0;
    std::vector<cudaGraphNode_t> nodes(n);
    if (cudaGraphGetNodes(graph, nodes.data(), &n) != cudaSuccess) return 0;
    int k = 0;
    for (size_t i = 0; i < n; ++i) {
        cudaGraphNodeType t;
        if (cudaGraphNodeGetType(nodes[i], &t) == cudaSuccess && t == cudaGraphNodeTypeKernel) ++k;
    }
    return k;
}

static void drop_graphs(SepEngine* e) {
    for (auto& kv : e->graphs) cudaGraphExecDestroy(kv.second.exec);
    e->graphs.clear();
}

// cache key of a chain graph: every argument its kernels bake in (`t`: frames, or -hops for the pipelined form)
static std::vector<int64_t> graph_key(const ChainArgs& a, int t) {
    return {(int64_t)a.x, a.xbs, a.xcs, a.x_len, (int64_t)a.emb, (int64_t)a.state, (int64_t)a.y,
            a.ybs, a.ycs, a.y_len, a.B, t, (int64_t)a.wsp, (int64_t)a.flags, a.pos_rel, (int64_t)a.active,
            (int64_t)a.slots, a.state_batch, (int64_t)a.hops, a.targets, (int64_t)a.offsets, a.calls,
            (int64_t)a.hist, a.hist_frames, (int64_t)a.leads, (int64_t)a.used, a.join_frames};
}

// Launch the graph cached under `key` on `st`.  The first time a key is seen, `enqueue(cap)` is captured on the private
// stream `cap` (made on first use) and instantiated; at most 32 graphs are kept.
template <class Enqueue>
static int run_graph(SepEngine* e, const std::vector<int64_t>& key, cudaStream_t& cap, cudaStream_t st, Enqueue enqueue) {
    auto it = e->graphs.find(key);
    if (it == e->graphs.end()) {
        if (!e->pack.committed) return fail(4, "weights not committed");
        if (int rc = set_attrs()) return rc;
        if (!cap) CK(cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking));
        if (e->graphs.size() >= 32) drop_graphs(e);
        CK(cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal));
        const int rc = enqueue(cap);
        cudaGraph_t graph = nullptr;
        const cudaError_t ce = cudaStreamEndCapture(cap, &graph);
        if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
        if (ce != cudaSuccess) return fail(3, std::string("cudaStreamEndCapture: ") + cudaGetErrorString(ce));
        cudaGraphExec_t exec = nullptr;
        const int nk = count_kernel_nodes(graph);
        CK(cudaGraphInstantiate(&exec, graph, 0));
        cudaGraphDestroy(graph);
        it = e->graphs.emplace(key, SepEngine::CachedGraph{exec, nk}).first;
    }
    CK(cudaGraphLaunch(it->second.exec, st));
    e->launch_count += it->second.kernels;
    return 0;
}

// K chained one-frame calls as one pipelined graph
static int run_pipeline(SepEngine* e, const ChainArgs& a, int K, cudaStream_t st) {
    return run_graph(e, graph_key(a, -K), e->pipe_streams[0], st, [&](cudaStream_t origin) { return enqueue_pipeline(e, a, K, origin); });
}

// Launch the chain directly, or replay it from a cached CUDA graph (graph launches go to the caller's stream).
static int run_chain(SepEngine* e, const ChainArgs& a, cudaStream_t st, bool use_graph) {
    if (!use_graph || (a.flags & L2H_FLAG_TAPS)) {
        const long long before = g_launches;
        const int rc = enqueue_call(e, a, st);
        e->launch_count += g_launches - before;
        return rc;
    }
    return run_graph(e, graph_key(a, a.T), e->cap_stream, st, [&](cudaStream_t cs) { return enqueue_call(e, a, cs); });
}

}  // namespace l2h

using namespace l2h;

extern "C" {

int l2h_abi_version(void) { return L2H_ABI_VERSION; }
const char* l2h_last_error(void) { return g_err.c_str(); }

int l2h_sep_create(const l2h_sep_config* c, void** handle) {
    if (!c || !handle) return fail(1, "null argument");
    if (c->stft_chunk_size != HOP || c->stft_pad_size != LOOKAHEAD || c->embed_dim != SPK || c->num_ch != NMIC ||
        c->D != CH || c->L != NHEAD || c->I != 1 || c->J != 1 || c->H != HID || c->local_atten_len != ATT ||
        !c->use_attn || !c->lookahead || !c->chunk_causal || c->num_src != NSRC || c->B < 1 || c->B > 16)
        return fail(1, "unsupported configuration: the kernels are specialised to configs/tsh.json "
                       "(chunk 128, pad 64, embed 256, 2 ch, D 64, H 64, 4 heads, I=J=1, window 50, 2 src)");
    SepEngine* e = new SepEngine();
    e->cfg = *c;
    e->n_blocks = c->B;
    build_layout(e);
    *handle = e;
    return 0;
}

// everything the handle owns on its device: cached graphs, capture / pipeline streams, events, the weight buffers
static void release_device_resources(SepEngine* e) {
    int cur = -1;
    const int dev = e->pack.device;
    const bool sw = dev >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != dev;
    if (sw) cudaSetDevice(dev);
    drop_graphs(e);
    if (e->cap_stream) { cudaStreamDestroy(e->cap_stream); e->cap_stream = nullptr; }
    for (auto& ps : e->pipe_streams) if (ps) { cudaStreamDestroy(ps); ps = nullptr; }
    for (auto& ev : e->pipe_events) cudaEventDestroy(ev);
    e->pipe_events.clear();
    if (e->trace_dev) { cudaFree(e->trace_dev); e->trace_dev = nullptr; e->trace_cap = 0; }
    e->pack.release();
    if (sw) cudaSetDevice(cur);
}

// a handle is bound to the device that was current at its last commit (INTEGRATION.md: one handle per device)
static int check_device(SepEngine* e) {
    int cur = -1;
    CK(cudaGetDevice(&cur));
    const int dev = e->pack.device;
    if (dev >= 0 && cur != dev)
        return fail(1, "this handle's weights live on device " + std::to_string(dev) + " but device " + std::to_string(cur) +
                       " is current: commit the weights again with the new device current (Net.to(device) does), or use one handle per device");
    return 0;
}

int l2h_sep_destroy(void* handle) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e) return 0;
    release_device_resources(e);
    delete e;
    return 0;
}

int l2h_sep_load_weight(void* handle, const char* name, const float* data, int64_t numel) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !name || !data) return fail(1, "null argument");
    return e->pack.load(name, data, numel);
}

int l2h_sep_weights_expected(void* handle, int32_t* n_expected, int32_t* n_loaded) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e) return fail(1, "null handle");
    e->pack.counts(n_expected, n_loaded);
    return 0;
}

int l2h_sep_weight_info(void* handle, int32_t index, const char** name, int64_t* numel) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e) return fail(1, "null handle");
    return e->pack.info(index, name, numel);       // the name is valid until l2h_sep_destroy
}

int l2h_sep_commit_weights(void* handle, void* stream) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e) return fail(1, "null handle");
    if (int rc = e->pack.finish()) return rc;
    float* h = e->pack.host.data();
    for (const auto& m : e->mid_src)        // per-column PReLU slopes of the fused Q|K|V projection
        for (int n = 0; n < NQKV; ++n) h[m.slope_vec + n] = h[m.slopes + (n < NHEAD * QE ? 0 : (n < 2 * NHEAD * QE ? 1 : 2))];
    for (const auto& m : e->mid_src)        // k-sliced, bank-padded copies for mid_kernel (layout: mid_kernel.cuh)
        mid_pack_weights(h + m.wl1, h + m.wih2, h + m.whh2t, h + m.wl2, h + m.wqkv, h + m.dst);
    int cur = -1;
    CK(cudaGetDevice(&cur));
    if (e->pack.dev != nullptr && e->pack.device != cur)    // the module moved to another GPU: everything device-side is rebuilt there
        release_device_resources(e);
    if (int rc = e->pack.upload(static_cast<cudaStream_t>(stream))) return rc;
    e->w.gen = (int)(++e->weight_gen & 0x7fffff) + 1;      // never 0 (= a freshly initialised state)
    drop_graphs(e);                                         // cached graphs carry the old generation in their kernel arguments
    return 0;
}

int l2h_sep_state_offsets(void* handle, int64_t* out, int32_t n) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !out) return fail(1, "null argument");
    const int64_t v[L2H_STATE_OFFSETS] = {RING, QK_LD, QK_DIM, V_DIM, ATT, ST_EMB, ST_GATE, ST_CONV, ST_DECONV, ST_ISTFT, ST_BLK,
                                          BK_K, BK_V, BK_H, BK_C, BK_STRIDE, ST_POS, ST_CALLS};
    if (n < 16) return fail(1, "need room for at least 16 values");      // 16: the layout before the per-stream clocks
    for (int i = 0; i < std::min<int>(n, L2H_STATE_OFFSETS); ++i) out[i] = v[i];
    return 0;
}

int l2h_sep_state_layout(void* handle, int64_t* header_bytes, int64_t* stride_floats) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e) return fail(1, "null handle");
    if (header_bytes) *header_bytes = sizeof(StateHeader);
    if (stride_floats) *stride_floats = stream_stride(e->n_blocks);
    return 0;
}

int l2h_sep_state_bytes(void* handle, int32_t batch, size_t* bytes) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !bytes || batch <= 0) return fail(1, "bad argument");
    *bytes = sizeof(StateHeader) + (size_t)batch * stream_stride(e->n_blocks) * sizeof(float);
    return 0;
}

int l2h_sep_state_init(void* handle, void* state, int32_t batch, void* stream) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !state || batch <= 0) return fail(1, "bad argument");
    const int64_t ss = stream_stride(e->n_blocks);
    const int64_t total = sizeof(StateHeader) / 4 + (int64_t)batch * ss;
    state_init_kernel<<<592, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<float*>(state), total, ss, batch);
    CK(cudaGetLastError());
    e->launch_count += 1;
    return 0;
}

// slot lists of the stream-record calls: every slot in [0, batch), none twice
static int check_slots(const int32_t* slots, int32_t n, int32_t batch, const char* what) {
    std::vector<char> seen((size_t)batch, 0);
    for (int32_t i = 0; i < n; ++i) {
        const int32_t s = slots[i];
        if (s < 0 || s >= batch)
            return fail(1, std::string(what) + ": slot " + std::to_string(s) + " outside [0, " + std::to_string(batch) + ")");
        if (seen[(size_t)s]) return fail(1, std::string(what) + ": slot " + std::to_string(s) + " listed twice");
        seen[(size_t)s] = 1;
    }
    return 0;
}

int l2h_sep_state_reset_streams(void* handle, void* state, int32_t batch, const int32_t* slots_host, int32_t n, void* stream) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !state || !slots_host) return fail(1, "null argument");
    if (batch <= 0 || n <= 0 || n > batch) return fail(1, "batch and the slot count must be positive, slots at most batch");
    if (int rc = check_slots(slots_host, n, batch, "reset_streams")) return rc;
    if (int rc = check_device(e)) return rc;
    const int64_t ss = stream_stride(e->n_blocks);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    for (int32_t i0 = 0; i0 < n; i0 += RESET_MAX_SLOTS) {       // one launch for up to RESET_MAX_SLOTS records
        const int32_t k = std::min<int32_t>(RESET_MAX_SLOTS, n - i0);
        SlotList sl{};
        std::copy(slots_host + i0, slots_host + i0 + k, sl.s);
        // ~2 CTAs per SM over all records: each record is 6 MB of stores
        const unsigned per_rec = (unsigned)std::max(1, 2 * NUM_SMS / k);
        reset_streams_kernel<<<dim3(per_rec, k), 256, 0, st>>>(static_cast<float*>(state), ss, sl);
        CK(cudaGetLastError());
        e->launch_count += 1;
    }
    return 0;
}

int l2h_sep_state_copy_streams(void* handle, void* dst_state, int32_t dst_batch, const int32_t* dst_slots_host,
                               const void* src_state, int32_t src_batch, const int32_t* src_slots_host, int32_t n, void* stream) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !dst_state || !src_state || !dst_slots_host || !src_slots_host) return fail(1, "null argument");
    if (dst_batch <= 0 || src_batch <= 0 || n <= 0 || n > dst_batch) return fail(1, "batches and the slot count must be positive");
    if (int rc = check_slots(dst_slots_host, n, dst_batch, "copy_streams (destination)")) return rc;
    for (int32_t i = 0; i < n; ++i)
        if (src_slots_host[i] < 0 || src_slots_host[i] >= src_batch)
            return fail(1, "copy_streams: source slot " + std::to_string(src_slots_host[i]) + " outside [0, " + std::to_string(src_batch) + ")");
    if (dst_state == src_state) {         // within one state: no record may be both read and overwritten
        std::vector<char> src_used((size_t)src_batch, 0);
        for (int32_t i = 0; i < n; ++i) src_used[(size_t)src_slots_host[i]] = 1;
        for (int32_t i = 0; i < n; ++i)
            if (src_used[(size_t)dst_slots_host[i]])
                return fail(1, "copy_streams: slot " + std::to_string(dst_slots_host[i]) + " is both a source and a destination");
    }
    if (int rc = check_device(e)) return rc;
    const int64_t ss = stream_stride(e->n_blocks);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* dst = static_cast<float*>(dst_state) + sizeof(StateHeader) / 4;
    const float* src = static_cast<const float*>(src_state) + sizeof(StateHeader) / 4;
    for (int32_t i = 0; i < n; ++i) {
        float* d = dst + (int64_t)dst_slots_host[i] * ss;
        // the whole record, its clock included; then the gate memo is invalidated (generation 0 is never a handle's):
        // weight generations are per handle, so a memo built by another handle must not be trusted
        CK(cudaMemcpyAsync(d, src + (int64_t)src_slots_host[i] * ss, (size_t)ss * sizeof(float), cudaMemcpyDeviceToDevice, st));
        CK(cudaMemsetAsync(d + ST_GEN, 0, sizeof(float), st));
    }
    return 0;
}

int l2h_sep_state_move_lead(void* handle, void* state, int32_t batch, const int32_t* old_host, const int32_t* new_host, int32_t n,
                            void* stream) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !state || !old_host || !new_host) return fail(1, "null argument");
    if (batch <= 0 || n <= 0 || n > batch) return fail(1, "batch and the record count must be positive, records at most batch");
    if (int rc = check_slots(old_host, n, batch, "move_lead (old leads)")) return rc;
    if (int rc = check_slots(new_host, n, batch, "move_lead (new leads)")) return rc;
    std::vector<char> is_old((size_t)batch, 0);
    for (int32_t i = 0; i < n; ++i) is_old[(size_t)old_host[i]] = 1;
    for (int32_t i = 0; i < n; ++i)
        if (is_old[(size_t)new_host[i]])
            return fail(1, "move_lead: record " + std::to_string(new_host[i]) + " is both an old and a new lead");
    if (int rc = check_device(e)) return rc;
    const int64_t ss = stream_stride(e->n_blocks);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* rec = static_cast<float*>(state) + sizeof(StateHeader) / 4;
    // the clocks, as the work queued before this call leaves them: a lead moves only between records of one listener
    std::vector<long long> clk(2 * (size_t)n);
    for (int32_t i = 0; i < n; ++i) {
        CK(cudaMemcpyAsync(&clk[2 * i], rec + (int64_t)old_host[i] * ss + ST_POS, sizeof(long long), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(&clk[2 * i + 1], rec + (int64_t)new_host[i] * ss + ST_POS, sizeof(long long), cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));
    for (int32_t i = 0; i < n; ++i)
        if (clk[2 * i] != clk[2 * i + 1])
            return fail(1, "move_lead: records " + std::to_string(old_host[i]) + " and " + std::to_string(new_host[i]) +
                               " have different clocks (" + std::to_string(clk[2 * i]) + " and " + std::to_string(clk[2 * i + 1]) +
                               " frames)");
    for (int32_t i0 = 0; i0 < n; i0 += MOVE_MAX_PAIRS) {
        const int32_t k = std::min<int32_t>(MOVE_MAX_PAIRS, n - i0);
        PairList pl{};
        std::copy(old_host + i0, old_host + i0 + k, pl.from);
        std::copy(new_host + i0, new_host + i0 + k, pl.to);
        const unsigned per_rec = (unsigned)std::max(1, 2 * NUM_SMS / k);      // as reset_streams: ~2 CTAs per SM over all records
        move_lead_kernel<<<dim3(per_rec, k), 256, 0, st>>>(static_cast<float*>(state), ss, pl);
        CK(cudaGetLastError());
        e->launch_count += 1;
    }
    return 0;
}

int l2h_sep_workspace_bytes(void* handle, int32_t batch, int32_t frames, uint32_t flags, size_t* bytes) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !bytes || batch <= 0 || frames <= 0) return fail(1, "bad argument");
    *bytes = (size_t)carve(e->n_blocks, batch, frames, flags).total * sizeof(float);
    return 0;
}

int l2h_sep_tap_info(void* handle, int32_t batch, int32_t frames, int64_t* off, int32_t* n_stages) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e) return fail(1, "null handle");
    if (off) *off = carve(e->n_blocks, batch, frames, L2H_FLAG_TAPS).TAPS;
    if (n_stages) *n_stages = 1 + 3 * e->n_blocks;
    return 0;
}

int l2h_sep_launches_per_forward(void* handle, int32_t frames, int32_t* n) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !n) return fail(1, "bad argument");
    // one l2h_sep_forward: a one-hop call is 6 kernels per block (gemm, bilstm, mid, qkv, attn, attn_out; 8 with many
    // streams, where the mid section runs as three kernels), a multi-hop call 10.  Streams of one-hop calls go through
    // the pipelined graph instead -- l2h_sep_launch_count has the exact figure for everything this handle launched.
    if (frames == 1 && tail_fits(e, 1))
        *n = 1 + e->n_blocks * 2 + 1;       // front1, (BiLSTM, tail_kernel) per block, back
    else
        *n = 1 + e->n_blocks * (frames == 1 ? 6 : 10) + 1;
    return 0;
}

int l2h_sep_trace_start(void* handle, int32_t capacity) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || capacity < 0) return fail(1, "bad argument");
    CK(cudaDeviceSynchronize());
    TraceRec* none = nullptr;
    unsigned int zero = 0;
    CK(cudaMemcpyToSymbol(g_trace, &none, sizeof(none)));
    if (e->trace_dev) { cudaFree(e->trace_dev); e->trace_dev = nullptr; e->trace_cap = 0; }
    if (capacity == 0) return 0;                       // tracing off
    CK(cudaMalloc(&e->trace_dev, (size_t)capacity * sizeof(TraceRec)));
    CK(cudaMemset(e->trace_dev, 0, (size_t)capacity * sizeof(TraceRec)));
    e->trace_cap = capacity;
    const unsigned int cap = (unsigned int)capacity;
    CK(cudaMemcpyToSymbol(g_trace_n, &zero, sizeof(zero)));
    CK(cudaMemcpyToSymbol(g_trace_cap, &cap, sizeof(cap)));
    CK(cudaMemcpyToSymbol(g_trace, &e->trace_dev, sizeof(e->trace_dev)));
    return 0;
}

int l2h_sep_trace_read(void* handle, void* records_host, int32_t max_records, int32_t* n_records) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !n_records) return fail(1, "bad argument");
    CK(cudaDeviceSynchronize());
    unsigned int n = 0;
    CK(cudaMemcpyFromSymbol(&n, g_trace_n, sizeof(n)));
    n = std::min<unsigned int>(n, (unsigned int)e->trace_cap);
    *n_records = (int32_t)n;
    const unsigned int take = std::min<unsigned int>(n, (unsigned int)std::max(0, max_records));
    if (records_host && take) CK(cudaMemcpy(records_host, e->trace_dev, (size_t)take * sizeof(TraceRec), cudaMemcpyDeviceToHost));
    unsigned int zero = 0;
    CK(cudaMemcpyToSymbol(g_trace_n, &zero, sizeof(zero)));   // the next run starts a fresh trace
    return 0;
}

int l2h_sep_launch_count(void* handle, int64_t* kernels, int32_t reset) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e) return fail(1, "null handle");
    if (kernels) *kernels = e->launch_count;
    if (reset) e->launch_count = 0;
    return 0;
}

int l2h_sep_forward(void* handle, const float* x, int64_t xbs, int64_t xcs, int32_t x_len, const float* emb,
                    void* state, float* y, int64_t ybs, int64_t ycs, int32_t y_len, int32_t batch, int32_t frames,
                    void* ws, size_t ws_bytes, uint32_t flags, void* stream) {
    return l2h_sep_forward_active(handle, x, xbs, xcs, x_len, emb, state, y, ybs, ycs, y_len, batch, frames, ws, ws_bytes, flags,
                                  stream, nullptr);
}

int l2h_sep_forward_active(void* handle, const float* x, int64_t xbs, int64_t xcs, int32_t x_len, const float* emb,
                           void* state, float* y, int64_t ybs, int64_t ycs, int32_t y_len, int32_t batch, int32_t frames,
                           void* ws, size_t ws_bytes, uint32_t flags, void* stream, const uint8_t* active_dev) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (active_dev && frames != 1) return fail(1, "an activity mask needs a one-hop call (frames == 1)");
    if (active_dev && (flags & L2H_FLAG_TAPS)) return fail(1, "an activity mask cannot be combined with L2H_FLAG_TAPS");
    if (e) { if (int rc_dev = check_device(e)) return rc_dev; }
    if (!e || !x || !emb || !state || !y || !ws) return fail(1, "null argument");
    ChainArgs a{x, xbs, xcs, x_len, emb, static_cast<float*>(state), y, ybs, ycs, y_len, batch, frames,
                static_cast<float*>(ws), ws_bytes, flags & ~L2H_FLAG_GRAPH, 0};
    a.active = active_dev;
    return run_chain(e, a, static_cast<cudaStream_t>(stream), (flags & L2H_FLAG_GRAPH) != 0);
}

int l2h_sep_forward_targets(void* handle, const float* x, int64_t xbs, int64_t xcs, int32_t x_len, const float* emb,
                            void* state, float* y, int64_t ybs, int64_t ycs, int32_t y_len, int32_t batch, int32_t n_targets,
                            int32_t frames, void* ws, size_t ws_bytes, uint32_t flags, void* stream) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !x || !emb || !state || !y || !ws) return fail(1, "null argument");
    if (batch <= 0 || n_targets <= 0 || frames <= 0)
        return fail(1, "a targets call needs batch, n_targets and frames > 0 (batch = " + std::to_string(batch) + ", n_targets = " +
                           std::to_string(n_targets) + ", frames = " + std::to_string(frames) + ")");
    if ((int64_t)batch * n_targets * frames * NF > 0x7fffffff / 2)
        return fail(1, "batch*n_targets*frames too large for one call; split the batch");
    if (flags & L2H_FLAG_TAPS) return fail(1, "a targets call cannot be combined with L2H_FLAG_TAPS");
    if (int rc_dev = check_device(e)) return rc_dev;
    ChainArgs a{x, xbs, xcs, x_len, emb, static_cast<float*>(state), y, ybs, ycs, y_len, batch * n_targets, frames,
                static_cast<float*>(ws), ws_bytes, flags & ~L2H_FLAG_GRAPH, 0};
    a.targets = n_targets;
    return run_chain(e, a, static_cast<cudaStream_t>(stream), (flags & L2H_FLAG_GRAPH) != 0);
}

int l2h_sep_forward_targets_groups(void* handle, const float* x, int64_t xbs, int64_t xcs, int32_t x_len, const float* emb,
                                   void* state, int32_t state_batch, const int32_t* groups_dev, const int32_t* hops_dev, int32_t n,
                                   int32_t n_targets, int32_t frames, float* y, int64_t ybs, int64_t ycs, int32_t y_len, void* ws,
                                   size_t ws_bytes, uint32_t flags, void* stream) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !x || !emb || !state || !y || !ws || !groups_dev) return fail(1, "null argument");
    if (n <= 0 || n_targets <= 0 || frames <= 0)
        return fail(1, "a groups call needs n, n_targets and frames > 0 (n = " + std::to_string(n) + ", n_targets = " +
                           std::to_string(n_targets) + ", frames = " + std::to_string(frames) + ")");
    if (state_batch <= 0 || state_batch % n_targets != 0)
        return fail(1, "a groups call needs a state of groups of n_targets records (state_batch = " + std::to_string(state_batch) +
                           ", n_targets = " + std::to_string(n_targets) + ")");
    if (n > state_batch / n_targets)
        return fail(1, "a group list needs n <= state_batch / n_targets groups (n = " + std::to_string(n) + ", groups = " +
                           std::to_string(state_batch / n_targets) + ")");
    if ((int64_t)n * n_targets * frames * NF > 0x7fffffff / 2) return fail(1, "n*n_targets*frames too large for one call; split the list");
    if (flags & L2H_FLAG_TAPS) return fail(1, "a groups call cannot be combined with L2H_FLAG_TAPS");
    if (int rc_dev = check_device(e)) return rc_dev;
    ChainArgs a{x, xbs, xcs, x_len, emb, static_cast<float*>(state), y, ybs, ycs, y_len, n * n_targets, frames,
                static_cast<float*>(ws), ws_bytes, flags & ~L2H_FLAG_GRAPH, 0};
    a.slots = groups_dev;
    a.state_batch = state_batch;
    a.hops = hops_dev;
    a.targets = n_targets;
    return run_chain(e, a, static_cast<cudaStream_t>(stream), (flags & L2H_FLAG_GRAPH) != 0);
}

static int targets_rows(void* handle, const float* x, int64_t xbs, int64_t xcs, int32_t x_len, const float* emb, void* state,
                        int32_t state_batch, const int32_t* records_dev, const int32_t* offsets_dev, const int32_t* hops_dev,
                        int32_t n, int32_t n_rows, int32_t frames, float* y, int64_t ybs, int64_t ycs, int32_t y_len, void* ws,
                        size_t ws_bytes, uint32_t flags, void* stream, float* hist, int32_t hist_frames) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !x || !emb || !state || !y || !ws || !records_dev || !offsets_dev) return fail(1, "null argument");
    if (n <= 0 || n_rows <= 0 || frames <= 0)
        return fail(1, "a target rows call needs n, n_rows and frames > 0 (n = " + std::to_string(n) + ", n_rows = " +
                           std::to_string(n_rows) + ", frames = " + std::to_string(frames) + ")");
    if (n_rows > state_batch)
        return fail(1, "a target rows call needs n_rows <= state_batch (n_rows = " + std::to_string(n_rows) + ", state_batch = " +
                           std::to_string(state_batch) + ")");
    if (n > n_rows)      // the mixtures' rows of the front and block 0 live in the workspace of the n_rows target rows
        return fail(1, "a target rows call needs n <= n_rows (n = " + std::to_string(n) + ", n_rows = " + std::to_string(n_rows) + ")");
    if ((int64_t)n_rows * frames * NF > 0x7fffffff / 2) return fail(1, "n_rows*frames too large for one call; split the rows");
    if (flags & L2H_FLAG_TAPS) return fail(1, "a target rows call cannot be combined with L2H_FLAG_TAPS");
    if (int rc_dev = check_device(e)) return rc_dev;
    ChainArgs a{x, xbs, xcs, x_len, emb, static_cast<float*>(state), y, ybs, ycs, y_len, n_rows, frames,
                static_cast<float*>(ws), ws_bytes, flags & ~L2H_FLAG_GRAPH, 0};
    a.slots = records_dev;
    a.state_batch = state_batch;
    a.hops = hops_dev;
    a.targets = 0;
    a.offsets = offsets_dev;
    a.calls = n;
    a.hist = hist;
    a.hist_frames = hist_frames;
    return run_chain(e, a, static_cast<cudaStream_t>(stream), (flags & L2H_FLAG_GRAPH) != 0);
}

int l2h_sep_forward_targets_rows(void* handle, const float* x, int64_t xbs, int64_t xcs, int32_t x_len, const float* emb,
                                 void* state, int32_t state_batch, const int32_t* records_dev, const int32_t* offsets_dev,
                                 const int32_t* hops_dev, int32_t n, int32_t n_rows, int32_t frames, float* y, int64_t ybs,
                                 int64_t ycs, int32_t y_len, void* ws, size_t ws_bytes, uint32_t flags, void* stream) {
    return targets_rows(handle, x, xbs, xcs, x_len, emb, state, state_batch, records_dev, offsets_dev, hops_dev, n, n_rows, frames, y,
                        ybs, ycs, y_len, ws, ws_bytes, flags, stream, nullptr, 0);
}

int l2h_sep_forward_targets_rows_history(void* handle, const float* x, int64_t xbs, int64_t xcs, int32_t x_len, const float* emb,
                                         void* state, int32_t state_batch, const int32_t* records_dev, const int32_t* offsets_dev,
                                         const int32_t* hops_dev, int32_t n, int32_t n_rows, int32_t frames, float* y, int64_t ybs,
                                         int64_t ycs, int32_t y_len, void* ws, size_t ws_bytes, uint32_t flags, void* stream,
                                         float* hist_dev, int32_t hist_frames) {
    if (!hist_dev) return fail(1, "null argument: hist_dev");
    if (hist_frames < 1) return fail(1, "a history needs hist_frames >= 1 (hist_frames = " + std::to_string(hist_frames) + ")");
    return targets_rows(handle, x, xbs, xcs, x_len, emb, state, state_batch, records_dev, offsets_dev, hops_dev, n, n_rows, frames, y,
                        ybs, ycs, y_len, ws, ws_bytes, flags, stream, hist_dev, hist_frames);
}

int l2h_sep_join_targets(void* handle, const int32_t* records_dev, const int32_t* leads_dev, const float* emb, int32_t J, void* state,
                         int32_t state_batch, const float* hist_dev, int32_t hist_frames, int32_t frames, float* y, int64_t ybs,
                         int64_t ycs, int32_t* used_dev, void* ws, size_t ws_bytes, uint32_t flags, void* stream) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !records_dev || !leads_dev || !emb || !state || !ws) return fail(1, "null argument");
    if (J <= 0 || J > state_batch)
        return fail(1, "a join needs 0 < J <= state_batch (J = " + std::to_string(J) + ", state_batch = " + std::to_string(state_batch) +
                           ")");
    if (frames < 0) return fail(1, "a join needs frames >= 0 (frames = " + std::to_string(frames) + ")");
    if (hist_dev && hist_frames < 1)
        return fail(1, "a history needs hist_frames >= 1 (hist_frames = " + std::to_string(hist_frames) + ")");
    const int replay = hist_dev ? std::min(frames, hist_frames) : 0;      // the most frames a row replays
    if (replay > 0 && !y) return fail(1, "null argument: y_dev (the join replays frames)");
    if ((int64_t)J * replay * NF > 0x7fffffff / 2) return fail(1, "J*frames too large for one call; split the rows");
    if (flags & L2H_FLAG_TAPS) return fail(1, "a join cannot be combined with L2H_FLAG_TAPS");
    if (int rc_dev = check_device(e)) return rc_dev;
    ChainArgs a{nullptr, 0, 0, 0, emb, static_cast<float*>(state), y, ybs, ycs, HOP * replay, J, std::max(1, replay),
                static_cast<float*>(ws), ws_bytes, flags & ~L2H_FLAG_GRAPH, 0};
    a.slots = records_dev;
    a.state_batch = state_batch;
    a.targets = 0;
    a.calls = J;
    a.hist = const_cast<float*>(hist_dev);
    a.hist_frames = hist_dev ? hist_frames : 0;
    a.leads = leads_dev;
    a.used = used_dev;
    a.join_frames = replay;
    return run_chain(e, a, static_cast<cudaStream_t>(stream), (flags & L2H_FLAG_GRAPH) != 0);
}

int l2h_sep_forward_slots(void* handle, const float* x, int64_t xbs, int64_t xcs, int32_t x_len, const float* emb,
                          void* state, int32_t state_batch, const int32_t* slots_dev, int32_t n, float* y, int64_t ybs,
                          int64_t ycs, int32_t y_len, void* ws, size_t ws_bytes, uint32_t flags, void* stream) {
    return l2h_sep_forward_slots_frames(handle, x, xbs, xcs, x_len, emb, state, state_batch, slots_dev, n, 1, y, ybs, ycs,
                                        y_len, ws, ws_bytes, flags, stream);
}

int l2h_sep_forward_slots_frames(void* handle, const float* x, int64_t xbs, int64_t xcs, int32_t x_len, const float* emb,
                                 void* state, int32_t state_batch, const int32_t* slots_dev, int32_t n, int32_t frames,
                                 float* y, int64_t ybs, int64_t ycs, int32_t y_len, void* ws, size_t ws_bytes,
                                 uint32_t flags, void* stream) {
    return l2h_sep_forward_slots_hops(handle, x, xbs, xcs, x_len, emb, state, state_batch, slots_dev, nullptr, n, frames, y,
                                      ybs, ycs, y_len, ws, ws_bytes, flags, stream);
}

int l2h_sep_forward_slots_hops(void* handle, const float* x, int64_t xbs, int64_t xcs, int32_t x_len, const float* emb,
                               void* state, int32_t state_batch, const int32_t* slots_dev, const int32_t* hops_dev,
                               int32_t n, int32_t frames, float* y, int64_t ybs, int64_t ycs, int32_t y_len, void* ws,
                               size_t ws_bytes, uint32_t flags, void* stream) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !x || !emb || !state || !y || !ws || !slots_dev) return fail(1, "null argument");
    if (state_batch <= 0 || n <= 0 || n > state_batch)
        return fail(1, "a slot list needs 0 < n <= state_batch (n = " + std::to_string(n) + ", state_batch = " +
                           std::to_string(state_batch) + ")");
    if (frames <= 0) return fail(1, "a slot-list call needs frames > 0 (frames = " + std::to_string(frames) + ")");
    if (flags & L2H_FLAG_TAPS) return fail(1, "a slot list cannot be combined with L2H_FLAG_TAPS");
    if (int rc_dev = check_device(e)) return rc_dev;
    ChainArgs a{x, xbs, xcs, x_len, emb, static_cast<float*>(state), y, ybs, ycs, y_len, n, frames,
                static_cast<float*>(ws), ws_bytes, flags & ~L2H_FLAG_GRAPH, 0};
    a.slots = slots_dev;
    a.state_batch = state_batch;
    a.hops = hops_dev;
    return run_chain(e, a, static_cast<cudaStream_t>(stream), (flags & L2H_FLAG_GRAPH) != 0);
}

// One-hop calls are pipelined over hops (wavefront graph) only for FEW streams: with many streams every kernel of a hop
// already fills the GPU, the dense stages run on the tensor cores (enqueue_chain) and the hops replay one chain graph.
static bool pipeline_applies(const SepEngine* e, int batch, int cpc, int n_calls) {
    return cpc == 1 && e->use_pipe && e->n_blocks == 3 && n_calls > 1 && !tc_form(batch, 1);
}

int l2h_sep_stream_host(void* handle, const float* x_host, int32_t x_len, const float* emb, void* state,
                        float* y_host, int32_t y_len, int32_t batch, int32_t n_calls, int32_t cpc,
                        float* x_stage, float* y_stage, void* ws, size_t ws_bytes, void* stream) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (e) { if (int rc_dev = check_device(e)) return rc_dev; }
    if (!e || !x_host || !emb || !state || !y_host || !x_stage || !y_stage || !ws) return fail(1, "null argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // hops moved per host<->device round: one call's worth, or (one-hop calls, pipelining on) a group of up to
    // PIPE_MAX_FRAMES hops that then run as ONE wavefront-pipelined graph of one-hop chains
    const bool pipe = pipeline_applies(e, batch, cpc, n_calls);
    int group = cpc;
    if (pipe) {
        const int64_t slot = pipe_slot_floats(e, batch);
        group = (int)std::min<int64_t>(std::min(pipe_frames_for(e, batch), n_calls), (int64_t)(ws_bytes / sizeof(float)) / slot);
        if (group < 2) group = 1;
    }
    const int hops_total = n_calls * cpc;
    const int in_len = HOP * group + LOOKAHEAD, out_len = HOP * group;      // staging strides
    for (int h0 = 0; h0 < hops_total; h0 += group) {
        const int hops = std::min(group, hops_total - h0);
        const int s0 = h0 * HOP;
        int n_in = std::min(x_len - s0, HOP * hops + LOOKAHEAD);
        if (n_in <= 0) return fail(1, "x_host shorter than n_calls * chunks_per_call * 128 samples");
        CK(cudaMemcpy2DAsync(x_stage, in_len * sizeof(float), x_host + s0, (size_t)x_len * sizeof(float),
                             (size_t)n_in * sizeof(float), (size_t)batch * NMIC, cudaMemcpyHostToDevice, st));
        // (a short last round changes the sizes and therefore the graph key: at most two graphs)
        ChainArgs a{x_stage, (int64_t)NMIC * in_len, in_len, n_in, emb, static_cast<float*>(state), y_stage,
                    (int64_t)NSRC * out_len, out_len, HOP * hops, batch, pipe ? 1 : hops, static_cast<float*>(ws), ws_bytes, 0, 0};
        int rc = (pipe && hops > 1) ? run_pipeline(e, a, hops, st) : run_chain(e, a, st, true);
        if (rc) return rc;
        const int n_out = std::min(y_len - s0, HOP * hops);
        if (n_out > 0)
            CK(cudaMemcpy2DAsync(y_host + s0, (size_t)y_len * sizeof(float), y_stage, out_len * sizeof(float),
                                 (size_t)n_out * sizeof(float), (size_t)batch * NSRC, cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));
    return 0;
}

int l2h_sep_stream_dev(void* handle, const float* x_dev, int32_t x_len, const float* emb, void* state,
                       float* y_dev, int32_t y_len, int32_t batch, int32_t n_calls, int32_t cpc, void* ws,
                       size_t ws_bytes, void* stream) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (e) { if (int rc_dev = check_device(e)) return rc_dev; }
    if (!e || !x_dev || !emb || !state || !y_dev || !ws) return fail(1, "null argument");
    if (n_calls <= 0 || cpc <= 0) return fail(1, "n_calls and chunks_per_call must be positive");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    set_clip_base_kernel<<<1, 1, 0, st>>>(static_cast<float*>(state));
    CK(cudaGetLastError());
    e->launch_count += 1;
    ChainArgs a{x_dev, (int64_t)NMIC * x_len, x_len, x_len, emb, static_cast<float*>(state), y_dev,
                (int64_t)NSRC * y_len, y_len, y_len, batch, cpc, static_cast<float*>(ws), ws_bytes, 0, 1};
    if (pipeline_applies(e, batch, cpc, n_calls)) {
        // groups of up to PIPE_MAX_FRAMES one-frame calls, each group one wavefront-pipelined graph
        const int64_t slot = pipe_slot_floats(e, batch);
        int kmax = (int)std::min<int64_t>(pipe_frames_for(e, batch), (int64_t)(ws_bytes / sizeof(float)) / slot);
        if (kmax >= 2) {
            int done = 0;
            while (done < n_calls) {
                const int K = std::min(kmax, n_calls - done);
                if (K == 1) { if (int rc = run_chain(e, a, st, true)) return rc; }
                else if (int rc = run_pipeline(e, a, K, st)) return rc;
                done += K;
            }
            return 0;
        }
    }
    for (int i = 0; i < n_calls; ++i)
        if (int rc = run_chain(e, a, st, true)) return rc;
    return 0;
}

int l2h_sep_stream_workspace_bytes(void* handle, int32_t batch, int32_t chunks_per_call, size_t* bytes) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !bytes || batch <= 0 || chunks_per_call <= 0) return fail(1, "bad argument");
    if (pipeline_applies(e, batch, chunks_per_call, 2))
        *bytes = (size_t)pipe_slot_floats(e, batch) * pipe_frames_for(e, batch) * sizeof(float);
    else
        *bytes = (size_t)carve(e->n_blocks, batch, chunks_per_call, 0).total * sizeof(float);
    return 0;
}

int l2h_sep_set_option(void* handle, const char* name, int32_t value) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !name) return fail(1, "bad argument");
    const std::string n(name);
    if (n == "defaults") {                      // pipeline settings back to the built-in defaults
        const SepEngine d{};
        e->pipe_alanes = d.pipe_alanes; e->pipe_qlanes = d.pipe_qlanes; e->pipe_clanes = d.pipe_clanes; e->pipe_tlanes = d.pipe_tlanes;
        e->pipe_olanes = d.pipe_olanes; e->pipe_flanes = d.pipe_flanes; e->pipe_blanes = d.pipe_blanes;
        e->pipe_frames = d.pipe_frames; e->pipe_pdl = d.pipe_pdl; e->pipe_midb_hops = d.pipe_midb_hops;
    }
    else if (n == "pipeline") e->use_pipe = value != 0;
    else if (n == "pipeline_frames") e->pipe_frames = value <= 0 ? 0 : std::max(2, std::min(PIPE_MAX_FRAMES, (int)value));
    else if (n == "pipeline_lanes") e->pipe_alanes = std::max(1, std::min(PIPE_LANES, (int)value));
    else if (n == "pipeline_pdl") e->pipe_pdl = value;
    else if (n == "pipeline_gemm_shape") e->pipe_gemm_shape = std::max(0, std::min(2, (int)value));
    else if (n == "pipeline_midb_hops") e->pipe_midb_hops = std::max(1, std::min(PIPE_MIDB_MAX, (int)value));
    else if (n == "pipeline_qkv_lanes") e->pipe_qlanes = std::max(1, std::min(PIPE_QLANES, (int)value));
    else if (n == "pipeline_midc_lanes") e->pipe_clanes = std::max(1, std::min(PIPE_CLANES, (int)value));
    else if (n == "pipeline_attn_lanes") e->pipe_tlanes = std::max(1, std::min(PIPE_TLANES, (int)value));
    else if (n == "pipeline_out_lanes") e->pipe_olanes = std::max(1, std::min(PIPE_OLANES, (int)value));
    else if (n == "pipeline_front_lanes") e->pipe_flanes = std::max(1, std::min(PIPE_FLANES, (int)value));
    else if (n == "pipeline_back_lanes") e->pipe_blanes = std::max(1, std::min(PIPE_BLANES, (int)value));
    else if (n == "pdl") e->use_pdl = value != 0;
    else if (n == "fused_tail") e->use_tail = value != 0;
    else if (n == "back_many") e->use_back_many = value != 0;
    else if (n == "tc_pdl") e->tc_pdl = (int)value;
    else if (n == "tc_lstm_min") e->tcl_min_seqdirs = std::max(1, (int)value);
    else if (n == "fuse_ih") e->fuse_ih = value != 0;
    else if (n == "bf16") e->tc_passes = value == 0 ? 3 : (value == 2 ? 1 : 2);   // 1: bf16 weights x split activations; 2: plain bf16 both
    else return fail(2, "unknown option: " + n);
    drop_graphs(e);                             // cached graphs were built with the old setting
    return 0;
}

int l2h_sep_pipeline_frames(void* handle, int32_t* frames) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (!e || !frames) return fail(1, "bad argument");
    *frames = (e->use_pipe && e->n_blocks == 3) ? pipe_frames_for(e, 1) : 1;
    return 0;
}

int l2h_sep_profile(void* handle, const float* x_dev, int32_t x_len, const float* emb, void* state, float* y_dev,
                    int32_t batch, int32_t frames, void* ws, size_t ws_bytes, int32_t iters, const char** names,
                    float* ms_total, int32_t* counts, int32_t* n_names, void* stream) {
    SepEngine* e = static_cast<SepEngine*>(handle);
    if (e) { if (int rc_dev = check_device(e)) return rc_dev; }
    if (!e || !x_dev || !emb || !state || !y_dev || !ws || !names || !ms_total || !counts || !n_names)
        return fail(1, "null argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Profiler prof;
    std::vector<std::string> order;
    std::map<std::string, std::pair<double, int>> acc;
    const int out_len = HOP * frames;
    for (int it = -2; it < iters; ++it) {           // two untimed warm-up chains
        prof.used = 0;
        prof.names.clear();
        ChainArgs a{x_dev, (int64_t)NMIC * x_len, x_len, x_len, emb, static_cast<float*>(state), y_dev,
                    (int64_t)NSRC * out_len, out_len, out_len, batch, frames, static_cast<float*>(ws), ws_bytes, 0, 0};
        a.prof = &prof;
        if (int rc = enqueue_chain(e, a, st)) return rc;
        CK(cudaStreamSynchronize(st));
        if (it < 0) continue;
        for (int i = 1; i < prof.used; ++i) {
            float ms = 0.f;
            CK(cudaEventElapsedTime(&ms, prof.ev[i - 1], prof.ev[i]));
            const std::string nm = prof.names[i];
            if (!acc.count(nm)) order.push_back(nm);
            acc[nm].first += ms;
            acc[nm].second += 1;
        }
    }
    for (auto ev : prof.ev) cudaEventDestroy(ev);
    static std::vector<std::string> keep;            // storage for the returned C strings
    keep = order;
    int n = 0;
    for (auto& nm : keep) {
        if (n >= 64) break;
        names[n] = nm.c_str();
        ms_total[n] = (float)acc[nm].first;
        counts[n] = acc[nm].second;
        ++n;
    }
    *n_names = n;
    return 0;
}

}  // extern "C"
