// Enrollment engine: weight packing, the kernel chain and the C ABI (include/lookonce_b200.h).
// Reference path: EmbedTFGridNet.forward, reference src/models/tfgridnet_orig/tfgridnet.py:100-127
// (trunk = espnet2 TF-GridNet block, SURVEY.md Appendix B).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/lookonce_b200.h"
#include "host_errors.h"
#include "weight_pack.h"
#include "embed_kernels.cuh"
#include "lstm.cuh"
#include "umma_host.cuh"
#include "tc_lstm.cuh"

namespace l2h {

using namespace emb;

struct EmbedEngine {
    l2h_embed_config cfg;
    int n_blocks;
    // packed weights; every tensor-core B operand also as bf16 hi/lo planes [2][N][K] (csrc/umma_host.cuh: split_planes)
    WeightPack pack;
    EmbWeights w;
    std::vector<EmbBlockWeights> bw;
    // plane offsets (pack.plane) of the head Linear and, per block, of both W_ih, both ConvTranspose1d and Q|K|V
    int64_t head_plane = 0;
    struct BlockPlanes { int64_t ih1, l1, ih2, l2, qkv; };
    std::vector<BlockPlanes> bplanes;
    int attrs_dev = -1;
    int passes = 3;                 // 3: bf16x3 split products (fp32-grade), 2: bf16 weights x split activations, 1: plain bf16
    int tcl_min_seqdirs = 2048;     // (sequence, direction) pairs from which a recurrence runs on the tensor cores (option "tc_lstm_min")
};

static void build_layout(EmbedEngine* e) {
    WeightPack& pk = e->pack;
    // DFT table generated here (torch.stft: periodic Hann, onesided, not normalised)
    const int64_t dft = pk.alloc(NFFT * DFT_LD);
    for (int n = 0; n < NFFT; ++n) {
        const double win = 0.5 - 0.5 * std::cos(2.0 * M_PI * n / NFFT);
        for (int k = 0; k < NF; ++k) {
            const double ang = 2.0 * M_PI * k * n / NFFT;
            pk.host[dft + n * DFT_LD + k] = (float)(win * std::cos(ang));
            pk.host[dft + n * DFT_LD + NF + k] = (float)(-win * std::sin(ang));
        }
    }
    pk.bind(&e->w.dft, dft);
    pk.bind(&e->w.wc, pk.plain("conv.0.weight", 64 * 36));
    pk.bind(&e->w.bc, pk.plain("conv.0.bias", 64));
    pk.bind(&e->w.gn_g, pk.plain("conv.1.weight", 64));
    pk.bind(&e->w.gn_b, pk.plain("conv.1.bias", 64));
    pk.ignore("deconv.weight", 64 * 2 * 9);
    pk.ignore("deconv.bias", 2);
    {   // head Linear [256][4160 (c*65+f)] -> [4160 (f*64+c)][256]
        const int64_t o = pk.alloc((int64_t)FC * 256);
        pk.repacked("embed_proj.0.weight", (int64_t)256 * FC, [o](const float* src, float* d) {
            for (int n = 0; n < 256; ++n)
                for (int c = 0; c < CH; ++c)
                    for (int f = 0; f < NF; ++f) d[o + (int64_t)(f * 64 + c) * 256 + n] = src[(int64_t)n * FC + c * NF + f];
        });
        pk.bind(&e->w.wh_t, o);
        e->head_plane = pk.plane(o, FC, 256, FC);
    }
    pk.bind(&e->w.bh, pk.plain("embed_proj.0.bias", 256));
    pk.bind(&e->w.lnh_g, pk.plain("embed_proj.1.weight", 256));
    pk.bind(&e->w.lnh_b, pk.plain("embed_proj.1.bias", 256));

    e->bw.resize(e->n_blocks);
    e->bplanes.resize(e->n_blocks);
    for (int b = 0; b < e->n_blocks; ++b) {
        EmbBlockWeights& W = e->bw[b];
        EmbedEngine::BlockPlanes& PL = e->bplanes[b];
        const std::string B = "blocks." + std::to_string(b) + ".";
        auto rnn = [&](const std::string& nm, const float** ln_g, const float** ln_b, const float** wih, const float** bb,
                       const float** whh, const float** wl, const float** bl, int64_t& p_ih, int64_t& p_l) {
            pk.bind(ln_g, pk.plain(B + nm + "_norm.gamma", 64));
            pk.bind(ln_b, pk.plain(B + nm + "_norm.beta", 64));
            const int64_t o_ih = pk.alloc(256 * 512), o_b = pk.alloc(512), o_hh = pk.alloc(2 * 256 * 64);
            for (int dir = 0; dir < 2; ++dir) {
                const std::string sfx = dir ? "_reverse" : "";
                pk.repacked(B + nm + "_rnn.weight_ih_l0" + sfx, 256 * 256, [o_ih, dir](const float* src, float* d) {
                    for (int p = 0; p < 256; ++p) {     // [256 rows][256 = c*4+k] -> [k*64+c][dir*256+p]
                        const int r = perm_row(p);
                        for (int c = 0; c < 64; ++c)
                            for (int k = 0; k < 4; ++k)
                                d[o_ih + (int64_t)(k * 64 + c) * 512 + dir * 256 + p] = src[(int64_t)r * 256 + c * 4 + k];
                    }
                });
                pk.repacked(B + nm + "_rnn.weight_hh_l0" + sfx, 256 * 64, [o_hh, dir](const float* src, float* d) {
                    for (int p = 0; p < 256; ++p)
                        memcpy(d + o_hh + (int64_t)(dir * 256 + p) * 64, src + perm_row(p) * 64, 64 * sizeof(float));
                });
                const int64_t ob = o_b + dir * 256;
                for (const char* bn : {"_rnn.bias_ih_l0", "_rnn.bias_hh_l0"})
                    pk.accumulate(B + nm + bn + sfx, ob, 256, [ob](const float* src, float* d) {
                        for (int p = 0; p < 256; ++p) d[ob + p] += src[perm_row(p)];
                    });
            }
            pk.bind(wih, o_ih); pk.bind(bb, o_b); pk.bind(whh, o_hh);
            p_ih = pk.plane(o_ih, 256, 512, 256);
            {   // ConvTranspose1d weight [128 h][64 c][4 k] -> [(kk*128+h)][c] with k = 3-kk
                const int64_t o = pk.alloc(512 * 64);
                pk.repacked(B + nm + "_linear.weight", 128 * 64 * 4, [o](const float* src, float* d) {
                    for (int kk = 0; kk < 4; ++kk)
                        for (int h = 0; h < 128; ++h)
                            for (int c = 0; c < 64; ++c) d[o + (int64_t)(kk * 128 + h) * 64 + c] = src[((int64_t)h * 64 + c) * 4 + (3 - kk)];
                });
                pk.bind(wl, o);
                p_l = pk.plane(o, 512, 64, 512);
            }
            pk.bind(bl, pk.plain(B + nm + "_linear.bias", 64));
        };
        rnn("intra", &W.ln1_g, &W.ln1_b, &W.wih1_t, &W.b1, &W.whh1, &W.wl1_t, &W.bl1, PL.ih1, PL.l1);
        rnn("inter", &W.ln2_g, &W.ln2_b, &W.wih2_t, &W.b2, &W.whh2, &W.wl2_t, &W.bl2, PL.ih2, PL.l2);
        const int64_t wqkv = pk.alloc(64 * NQKV), bqkv = pk.alloc(NQKV), sl = pk.alloc(NQKV);
        const int64_t gq = pk.alloc(NH * QK), bq = pk.alloc(NH * QK), gk = pk.alloc(NH * QK), bk = pk.alloc(NH * QK);
        const int64_t gv = pk.alloc(NH * VDIM), bv = pk.alloc(NH * VDIM);
        for (int h = 0; h < NH; ++h) {
            struct Br { const char* nm; int d; int col0; int64_t g; int64_t bt; };
            const Br brs[3] = {{"attn_conv_Q_", QE, h * QE, gq, bq}, {"attn_conv_K_", QE, 32 + h * QE, gk, bk},
                               {"attn_conv_V_", VD, 64 + h * VD, gv, bv}};
            for (const Br& br : brs) {
                const std::string M = B + br.nm + std::to_string(h);
                const int d = br.d, col0 = br.col0;
                pk.repacked(M + ".0.weight", d * 64, [wqkv, d, col0](const float* src, float* dd) {
                    for (int r = 0; r < d; ++r)
                        for (int k = 0; k < 64; ++k) dd[wqkv + (int64_t)k * NQKV + col0 + r] = src[r * 64 + k];
                });
                pk.repacked(M + ".0.bias", d, [bqkv, d, col0](const float* src, float* dd) { memcpy(dd + bqkv + col0, src, d * sizeof(float)); });
                pk.repacked(M + ".1.weight", 1, [sl, d, col0](const float* src, float* dd) { for (int r = 0; r < d; ++r) dd[sl + col0 + r] = src[0]; });
                // gamma/beta [1][d][1][65] -> per head [(f*d + e)]
                for (int gb = 0; gb < 2; ++gb) {
                    const int64_t base = (gb == 0 ? br.g : br.bt) + (int64_t)h * NF * d;
                    pk.repacked(M + (gb == 0 ? ".2.gamma" : ".2.beta"), d * NF, [base, d](const float* src, float* dd) {
                        for (int e2 = 0; e2 < d; ++e2)
                            for (int f = 0; f < NF; ++f) dd[base + f * d + e2] = src[e2 * NF + f];
                    });
                }
            }
        }
        pk.bind(&W.wqkv_t, wqkv); pk.bind(&W.bqkv, bqkv); pk.bind(&W.slope_qkv, sl);
        pk.bind(&W.gq, gq); pk.bind(&W.bq, bq); pk.bind(&W.gk, gk); pk.bind(&W.bk, bk); pk.bind(&W.gv, gv); pk.bind(&W.bv, bv);
        PL.qkv = pk.plane(wqkv, 64, NQKV, 64);
        {   // concat proj [64][64][1][1] -> [k][n]
            const int64_t o = pk.alloc(64 * 64);
            pk.repacked(B + "attn_concat_proj.0.weight", 64 * 64, [o](const float* src, float* d) {
                for (int n = 0; n < 64; ++n)
                    for (int k = 0; k < 64; ++k) d[o + (int64_t)k * 64 + n] = src[n * 64 + k];
            });
            pk.bind(&W.wp_t, o);
        }
        pk.bind(&W.bp, pk.plain(B + "attn_concat_proj.0.bias", 64));
        pk.bind(&W.slope_p, pk.plain(B + "attn_concat_proj.1.weight", 1));
        for (int gb = 0; gb < 2; ++gb) {   // [1][64][1][65] -> (f*64 + c)
            const int64_t o = pk.alloc(FC);
            pk.repacked(B + (gb == 0 ? "attn_concat_proj.2.gamma" : "attn_concat_proj.2.beta"), FC, [o](const float* src, float* d) {
                for (int c = 0; c < CH; ++c)
                    for (int f = 0; f < NF; ++f) d[o + f * 64 + c] = src[c * NF + f];
            });
            pk.bind(gb == 0 ? &W.gp : &W.bpn, o);
        }
    }
}

struct EWs { int64_t INV, GN, X, GX, HC, QKV, QN, KP, VP, S, O, HD, LENS, total; int T, Tp; };

static EWs ecarve(int B, int N) {
    EWs w;
    const int T = 1 + N / HOP, Tp = (T + 63) & ~63;
    w.T = T; w.Tp = Tp;
    const int64_t rows = (int64_t)B * T * NF;
    int64_t cur = 0;
    auto alloc = [&](int64_t n) { int64_t o = cur; cur = (cur + n + 31) & ~int64_t(31); return o; };
    w.INV = alloc(B);
    w.GN = alloc(4 * B);                       // 2 doubles per utterance
    w.X = alloc(rows * 64);
    const int64_t seq_rows = std::max((int64_t)B * T * (NF - KS + 1), (int64_t)B * NF * (T - KS + 1));
    w.GX = alloc(seq_rows * 512);
    w.HC = alloc(seq_rows * 128);
    w.QKV = alloc(rows * NQKV);
    w.QN = alloc((int64_t)B * NH * Tp * QK);
    w.KP = alloc((int64_t)B * NH * Tp * QK);    // two bf16 planes = one float per element
    w.VP = alloc((int64_t)B * NH * Tp * VDIM);
    w.S = alloc((int64_t)B * NH * T * Tp);
    w.O = alloc((int64_t)B * NH * Tp * VDIM);
    w.HD = alloc((int64_t)B * T * 256);
    w.LENS = alloc(B);                         // int32 per utterance: the device copy of the lengths of a mixed batch
    w.total = cur;
    return w;
}

#define CKU(expr)                                                                                  \
    do {                                                                                           \
        std::string _why;                                                                          \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess)                                                                     \
            return fail(3, std::string(#expr) + ": " + cudaGetErrorString(_e) + " " + _why);       \
    } while (0)

// The shortest utterance: T = 1 + n / HOP >= KS frames for the 4-frame unfold.
constexpr int MIN_SAMPLES = HOP * (KS - 1);

// x [B][2][N]; utterance b is x[b, :, :lens_host[b]] (lens_host null: every utterance is N long).  Every argument is
// checked before the committed-weights check and before any device work.
static int embed_forward_impl(EmbedEngine* e, const float* x, float* out, int B, int N, const int32_t* lens_host, float* wsp,
                              size_t ws_bytes, cudaStream_t st) {
    if (B <= 0) return fail(1, "need batch >= 1");
    if (N < MIN_SAMPLES) return fail(1, "utterance too short for the 4-frame unfold: need at least 192 samples");
    bool mixed = false;                        // some utterance shorter than N: the padded-frame path
    if (lens_host != nullptr)
        for (int b = 0; b < B; ++b) {
            if (lens_host[b] < MIN_SAMPLES || lens_host[b] > N)
                return fail(1, "length " + std::to_string(lens_host[b]) + " of utterance " + std::to_string(b) + " is outside [192, n_max = " +
                                   std::to_string(N) + "]");
            mixed |= lens_host[b] != N;
        }
    const EWs ws = ecarve(B, N);
    if ((size_t)ws.total * sizeof(float) > ws_bytes) return fail(1, "workspace too small");
    const int T = ws.T, Tp = ws.Tp;
    const int64_t rows = (int64_t)B * T * NF;
    if (rows * 2 > 0x7fffffff) return fail(1, "batch too large for one call; split it (l2h_embed_max_batch)");
    if (!e->pack.committed) return fail(4, "weights not committed");
    int cur_dev = -1;
    CK(cudaGetDevice(&cur_dev));
    if (cur_dev != e->pack.device)
        return fail(1, "this handle's weights live on device " + std::to_string(e->pack.device) + " but device " + std::to_string(cur_dev) +
                       " is current: commit the weights again with the new device current (EmbedTFGridNet.to(device) does), or use one "
                       "handle per device");
    if (e->attrs_dev != cur_dev) {
        CK(configure_lstm());
        CK(configure_tc_lstm());
        CK(umma::configure());
        CK(cudaFuncSetAttribute(eattn_out_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)EAOUT_SMEM));
        e->attrs_dev = cur_dev;
    }
    float* INV = wsp + ws.INV; double* GN = reinterpret_cast<double*>(wsp + ws.GN);
    float* X = wsp + ws.X; float* GX = wsp + ws.GX; float* HC = wsp + ws.HC;
    float* QKV = wsp + ws.QKV; float* QN = wsp + ws.QN;
    __nv_bfloat16* KP = reinterpret_cast<__nv_bfloat16*>(wsp + ws.KP);
    __nv_bfloat16* VP = reinterpret_cast<__nv_bfloat16*>(wsp + ws.VP);
    float* S = wsp + ws.S; float* O = wsp + ws.O; float* HD = wsp + ws.HD;
    const int Z = B * NH;
    const int64_t k_plane = (int64_t)Z * Tp * QK, v_plane = (int64_t)Z * Tp * VDIM;
    const int passes = e->passes;
    const WeightPack& pk = e->pack;

    // lengths on the device only for a mixed batch; equal lengths run exactly the equal-length path
    int32_t* lens = nullptr;
    if (mixed) {
        lens = reinterpret_cast<int32_t*>(wsp + ws.LENS);
        CK(launch_eput_lens(st, lens, lens_host, B));
    }

    CK(launch_estd(st, B, x, N, lens, INV));
    CK(cudaMemsetAsync(GN, 0, sizeof(double) * 2 * B, st));
    CK(launch_efront(st, B, x, N, lens, INV, X, GN, e->w, T));
    {
        const int64_t per_b = (int64_t)T * NF * CH, total4 = (int64_t)B * per_b / 4;
        CK(launch_egn_apply(st, X, GN, per_b, total4, lens, e->w));
    }

    for (int blk = 0; blk < e->n_blocks; ++blk) {
        const EmbBlockWeights& W = e->bw[blk];
        const EmbedEngine::BlockPlanes& PL = e->bplanes[blk];
        for (int path = 0; path < 2; ++path) {          // 0: intra (along F), 1: inter (along T)
            const bool inter = path == 1;
            const int Ls = inter ? T : NF;               // positions per sequence
            const int steps = Ls - KS + 1;
            const int nseq = inter ? B * NF : B * T;
            // ---- LN + unfold(ks=4) + W_ih of both directions: one tensor-core GEMM.  Rows = (sequence, window start);
            // the four taps are four k-chunks read at position offsets 0..3 of X itself (no unfolded copy, no LN pass,
            // no transposed copy for the inter path: the tensor map strides do it) --------------------------------------
            umma::GemmDesc g;
            g.a0.base = X; g.a0.channels = 64;
            if (!inter) { g.a0.n_pos = NF; g.a0.pos_stride = 64; g.a0.n_inner = nseq; g.a0.inner_stride = (int64_t)NF * 64; }
            else {
                g.a0.n_pos = T; g.a0.pos_stride = (int64_t)NF * 64; g.a0.n_inner = NF; g.a0.inner_stride = 64;
                g.a0.n_outer = B; g.a0.outer_stride = (int64_t)T * NF * 64;
            }
            umma::set_window_chunks(g, 64, KS, true);
            g.ln_g = inter ? W.ln2_g : W.ln1_g; g.ln_b = inter ? W.ln2_b : W.ln1_b;
            g.rows_per_seq = steps; g.nseq = nseq;
            g.b = pk.bplanes(inter ? PL.ih2 : PL.ih1, 256); g.N = 512; g.K = 256; g.passes = passes;
            g.bias = inter ? W.b2 : W.b1; g.C = GX; g.ldc = 512; g.c_seq_stride = (int64_t)steps * 512;
            CKU(umma::launch(g, st, &_why));
            // windows past an utterance's own frames: zero state, zero h
            if (inter && lens != nullptr) CK(launch_einter_mask(st, B, GX, lens, steps));
            LstmArgs l{};
            l.gx = GX; l.gx_ld = 512; l.out = HC; l.out_ld = 128; l.whh = inter ? W.whh2 : W.whh1;
            l.nseq = nseq; l.L = steps; l.inner_count = 1; l.outer_stride = steps; l.inner_stride = 0; l.step_stride = 1;
            l.ndir = 2;
            if ((int64_t)l.nseq * l.ndir >= e->tcl_min_seqdirs) CK(launch_tc_lstm(l, passes, st));   // many sequences: recurrence on the tensor cores
            else CK(launch_lstm_rec(l, st));
            // ---- ConvTranspose1d(128->64, k=4) + residual: output position p reads h rows p-3 .. p; rows outside the
            // sequence are the zero-filled halo of the tensor map ----------------------------------------------------
            umma::GemmDesc c;
            c.a0.base = HC; c.a0.channels = 128; c.a0.n_pos = steps; c.a0.pos_stride = 128;
            if (!inter) { c.a0.n_inner = nseq; c.a0.inner_stride = (int64_t)steps * 128; }
            else { c.a0.n_inner = NF; c.a0.inner_stride = (int64_t)steps * 128; c.a0.n_outer = B; c.a0.outer_stride = (int64_t)NF * steps * 128; }
            umma::set_window_chunks(c, 128, KS, false);
            c.pos_bias = -(KS - 1);
            c.rows_per_seq = Ls; c.nseq = nseq;
            c.b = pk.bplanes(inter ? PL.l2 : PL.l1, 512); c.N = 64; c.K = 512; c.passes = passes;
            c.bias = inter ? W.bl2 : W.bl1; c.C = X; c.R = X;
            if (!inter) { c.ldc = 64; c.c_seq_stride = (int64_t)NF * 64; }                 // row ((b,t), f) -> X[b][t][f]
            else { c.ldc = (int64_t)NF * 64; c.c_inner = NF; c.c_seq_stride = (int64_t)T * NF * 64; c.c_inner_stride = 64; }   // ((b,f), t)
            CKU(umma::launch(c, st, &_why));
        }
        // ---- full self-attention over frames ------------------------------------------------
        {
            umma::GemmDesc g;                          // Q|K|V 1x1 convs of all heads + PReLU
            g.a0.base = X; g.a0.channels = 64; g.a0.n_pos = rows; g.a0.pos_stride = 64;
            umma::set_plain_chunks(g, 64);
            g.rows_per_seq = (int)rows; g.nseq = 1;
            g.b = pk.bplanes(PL.qkv, 64); g.N = NQKV; g.K = 64; g.passes = passes;
            g.bias = W.bqkv; g.prelu_vec = W.slope_qkv; g.C = QKV; g.ldc = NQKV; g.c_seq_stride = 0;
            CKU(umma::launch(g, st, &_why));
        }
        CK(launch_eqkv_ln(st, B, QKV, QN, KP, VP, k_plane, v_plane, W, T, Tp));
        {
            umma::GemmDesc g;                          // S = Q K^T / sqrt(520), per (utterance, head)
            g.a0.base = QN; g.a0.channels = QK; g.a0.n_pos = T; g.a0.pos_stride = QK; g.a0.n_inner = Z; g.a0.inner_stride = (int64_t)Tp * QK;
            umma::set_plain_chunks(g, QK);
            g.rows_per_seq = T; g.nseq = Z; g.b_by_seq = true;
            g.b.base = KP; g.b.ld = QK; g.b.z_stride = (int64_t)Tp * QK; g.b.plane_stride = k_plane; g.b.nz = Z;
            g.N = T; g.K = QK; g.passes = passes; g.alpha = 1.f / sqrtf((float)QK);
            g.C = S; g.ldc = Tp; g.c_seq_stride = (int64_t)T * Tp;
            CKU(umma::launch(g, st, &_why));
        }
        CK(launch_softmax_rows(st, Z, S, Tp, T, T, (int64_t)T * Tp, lens));
        {
            umma::GemmDesc g;                          // O = P V (V is the MN-major B operand: [frame][f*16+c])
            g.a0.base = S; g.a0.channels = T; g.a0.n_pos = T; g.a0.pos_stride = Tp; g.a0.n_inner = Z; g.a0.inner_stride = (int64_t)T * Tp;
            umma::set_plain_chunks(g, T);
            g.rows_per_seq = T; g.nseq = Z; g.b_by_seq = true;
            g.b.base = VP; g.b.ld = VDIM; g.b.z_stride = (int64_t)Tp * VDIM; g.b.plane_stride = v_plane; g.b.nz = Z; g.b.mn_major = true;
            g.N = VDIM; g.K = T; g.passes = passes;
            g.C = O; g.ldc = VDIM; g.c_seq_stride = (int64_t)Tp * VDIM;
            CKU(umma::launch(g, st, &_why));
        }
        CK(launch_eattn_out(st, eattn_out_ctas(T, B), O, X, W, T, Tp, T * B));
    }
    // ---- head: Linear(4160 -> 256) over rows (b,t) [features f*64+c], LN, mean over T -----------
    {
        umma::GemmDesc g;
        g.a0.base = X; g.a0.channels = FC; g.a0.n_pos = (int64_t)B * T; g.a0.pos_stride = FC;
        umma::set_plain_chunks(g, FC);
        g.rows_per_seq = B * T; g.nseq = 1;
        g.b = pk.bplanes(e->head_plane, FC); g.N = 256; g.K = FC; g.passes = passes;
        g.bias = e->w.bh; g.C = HD; g.ldc = 256;
        CKU(umma::launch(g, st, &_why));
    }
    CK(launch_ehead(st, B, HD, out, e->w, T, lens));
    return 0;
}

}  // namespace l2h

using namespace l2h;

extern "C" {

int l2h_embed_create(const l2h_embed_config* c, void** handle) {
    if (!c || !handle) return fail(1, "null argument");
    if (c->embed_dim != 256 || c->num_ch != 2 || c->n_fft != emb::NFFT || c->stride != emb::HOP || c->num_blocks < 1 ||
        c->num_blocks > 16)
        return fail(1, "unsupported configuration: the kernels are specialised to configs/embed.json "
                       "(embed 256, 2 ch, n_fft 128, stride 64)");
    EmbedEngine* e = new EmbedEngine();
    e->cfg = *c;
    e->n_blocks = c->num_blocks;
    build_layout(e);
    *handle = e;
    return 0;
}

int l2h_embed_destroy(void* handle) {
    EmbedEngine* e = static_cast<EmbedEngine*>(handle);
    if (!e) return 0;
    e->pack.release();
    delete e;
    return 0;
}

int l2h_embed_load_weight(void* handle, const char* name, const float* data, int64_t numel) {
    EmbedEngine* e = static_cast<EmbedEngine*>(handle);
    if (!e || !name || !data) return fail(1, "null argument");
    return e->pack.load(name, data, numel);
}

int l2h_embed_weights_expected(void* handle, int32_t* n_expected, int32_t* n_loaded) {
    EmbedEngine* e = static_cast<EmbedEngine*>(handle);
    if (!e) return fail(1, "null handle");
    e->pack.counts(n_expected, n_loaded);
    return 0;
}

// the handle is bound to the device current here: a commit on another device releases the old buffers and rebuilds them
int l2h_embed_commit_weights(void* handle, void* stream) {
    EmbedEngine* e = static_cast<EmbedEngine*>(handle);
    if (!e) return fail(1, "null handle");
    if (int rc = e->pack.finish()) return rc;
    return e->pack.upload(static_cast<cudaStream_t>(stream));
}

int l2h_embed_set_option(void* handle, const char* name, int32_t value) {
    EmbedEngine* e = static_cast<EmbedEngine*>(handle);
    if (!e || !name) return fail(1, "bad argument");
    const std::string n(name);
    if (n == "bf16") e->passes = value == 0 ? 3 : (value == 2 ? 1 : 2);   // 0 (default): bf16x3 split, fp32-grade; 1: bf16 weights x
                                                                          // split activations; 2: plain bf16 operands
    else if (n == "tc_lstm_min") e->tcl_min_seqdirs = std::max(1, (int)value);
    else return fail(2, "unknown option: " + n);
    return 0;
}

int l2h_embed_workspace_bytes(void* handle, int32_t batch, int32_t n_samples, size_t* bytes) {
    if (!handle || !bytes || batch <= 0 || n_samples < emb::NFFT) return fail(1, "bad argument");
    *bytes = (size_t)ecarve(batch, n_samples).total * sizeof(float);
    return 0;
}

int l2h_embed_max_batch(void* handle, int32_t n_samples, int32_t* max_batch) {
    if (!handle || !max_batch || n_samples < emb::NFFT) return fail(1, "bad argument");
    const double per = (double)ecarve(1, n_samples).total * sizeof(float);
    const int64_t rows1 = (int64_t)(1 + n_samples / emb::HOP) * emb::NF;
    int64_t nb = (int64_t)(24e9 / per);                       // keep the workspace under ~24 GB
    nb = std::min<int64_t>(nb, (int64_t)(0x3fffffff / (rows1 * 4)));   // int32 row indices in the GEMMs
    *max_batch = (int32_t)std::max<int64_t>(1, nb);
    return 0;
}

int l2h_embed_forward_lengths(void* handle, const float* x_dev, int32_t n_max, const int32_t* lengths_host, int32_t batch,
                              float* emb_dev, void* ws, size_t ws_bytes, void* stream) {
    EmbedEngine* e = static_cast<EmbedEngine*>(handle);
    if (!e || !x_dev || !emb_dev || !ws) return fail(1, "null argument");
    return embed_forward_impl(e, x_dev, emb_dev, batch, n_max, lengths_host, static_cast<float*>(ws), ws_bytes,
                              static_cast<cudaStream_t>(stream));
}

int l2h_embed_forward(void* handle, const float* x_dev, float* emb_dev, int32_t batch, int32_t n_samples, void* ws,
                      size_t ws_bytes, void* stream) {
    return l2h_embed_forward_lengths(handle, x_dev, n_samples, nullptr, batch, emb_dev, ws, ws_bytes, stream);
}

}  // extern "C"
