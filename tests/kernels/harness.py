"""ctypes mirrors of tests/kernels/kernel_harness.cu and the float64 references the kernel-level tests compare with.

The references restate, in float64, both the exact operation (fp32 inputs, exact arithmetic) and the bf16 hi/lo split the
tensor-core kernels are meant to compute:  x = hi + lo with hi = rn_bf16(x), lo = rn_bf16(x - hi) (x - hi is exact in
fp32), and a product of `passes` terms
    passes = 1:  a_hi b_hi                          (plain bf16)
    passes = 2:  a_hi b_hi + a_lo b_hi              (bf16 "weights" b, split activations a)
    passes = 3:  a_hi b_hi + a_lo b_hi + a_hi b_lo  (bf16x3: fp32-grade)
with a = the activation (GEMM: the A row; recurrence: h or LN(x)) and b = the weight, so passes = 2 always means
bf16 weights times split activations.
"""
import ctypes
import math

import numpy as np
import torch

from lookoncetohear_b200 import build as _build

MAX_CHUNKS = 96
KC = 64

LSTM_VARIANTS = {"auto": 0, "rec3_pre": 1, "rec3_ring": 2, "rec4_2": 3, "rec4_4": 4, "tc": 5, "tc_x": 6}


class ASource(ctypes.Structure):
    _fields_ = [("base", ctypes.c_void_p), ("channels", ctypes.c_int64), ("n_pos", ctypes.c_int64),
                ("pos_stride", ctypes.c_int64), ("n_inner", ctypes.c_int64), ("inner_stride", ctypes.c_int64),
                ("n_outer", ctypes.c_int64), ("outer_stride", ctypes.c_int64)]


class Gemm(ctypes.Structure):
    _fields_ = [("a0", ASource), ("a1", ASource), ("n_chunks", ctypes.c_int32),
                ("chunk_c0", ctypes.c_int32 * MAX_CHUNKS), ("chunk_dp", ctypes.c_int32 * MAX_CHUNKS),
                ("chunk_flags", ctypes.c_int32 * MAX_CHUNKS),
                ("rows_per_seq", ctypes.c_int32), ("nseq", ctypes.c_int32), ("pos_bias", ctypes.c_int32),
                ("b_base", ctypes.c_void_p), ("b_ld", ctypes.c_int64), ("b_z_stride", ctypes.c_int64),
                ("b_plane_stride", ctypes.c_int64), ("b_nz", ctypes.c_int32), ("b_mn_major", ctypes.c_int32),
                ("b_by_seq", ctypes.c_int32), ("N", ctypes.c_int32), ("K", ctypes.c_int32), ("passes", ctypes.c_int32),
                ("C", ctypes.c_void_p), ("R", ctypes.c_void_p), ("ldc", ctypes.c_int64), ("c_seq_stride", ctypes.c_int64),
                ("c_inner_stride", ctypes.c_int64), ("c_inner", ctypes.c_int32), ("alpha", ctypes.c_float),
                ("bias", ctypes.c_void_p), ("prelu", ctypes.c_void_p), ("prelu_vec", ctypes.c_void_p),
                ("ln_g", ctypes.c_void_p), ("ln_b", ctypes.c_void_p)]


class Plan(ctypes.Structure):
    _fields_ = [("BN", ctypes.c_int32), ("b_resident", ctypes.c_int32), ("nop", ctypes.c_int32), ("nstg", ctypes.c_int32),
                ("P_TILE", ctypes.c_int32), ("S_TILE", ctypes.c_int32), ("grid", ctypes.c_int32),
                ("n_tiles_n", ctypes.c_int32), ("vec_ok", ctypes.c_int32), ("smem", ctypes.c_int64),
                ("m_tiles", ctypes.c_int64)]


class Lstm(ctypes.Structure):
    _fields_ = [("gx", ctypes.c_void_p), ("gx_ld", ctypes.c_int64), ("out", ctypes.c_void_p), ("out_ld", ctypes.c_int64),
                ("whh", ctypes.c_void_p), ("h_state", ctypes.c_void_p), ("c_state", ctypes.c_void_p),
                ("hc_outer_stride", ctypes.c_int64), ("nseq", ctypes.c_int32), ("L", ctypes.c_int32),
                ("inner_count", ctypes.c_int32), ("ndir", ctypes.c_int32), ("outer_stride", ctypes.c_int64),
                ("inner_stride", ctypes.c_int64), ("step_stride", ctypes.c_int64), ("out_outer_stride", ctypes.c_int64),
                ("out_inner_stride", ctypes.c_int64), ("out_step_stride", ctypes.c_int64),
                ("x", ctypes.c_void_p), ("x_ld", ctypes.c_int64), ("wih_hi", ctypes.c_void_p), ("wih_lo", ctypes.c_void_p),
                ("bias", ctypes.c_void_p), ("ln_g", ctypes.c_void_p), ("ln_b", ctypes.c_void_p), ("steps", ctypes.c_void_p)]


class SepWeights(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("wqkv_t", "bqkv", "slopes", "lnq_g", "lnq_b", "lnk_g", "lnk_b", "lnv_g", "lnv_b",
                                                "wp_t", "bp", "lnp_g", "lnp_b")]


class SepFrontBack(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("wat", "ws", "wc", "bc", "we", "be", "lne_g", "lne_b", "wd", "bd")] + \
               [("gen", ctypes.c_int32)] + [(n, ctypes.c_void_p) for n in ("ln1_g", "ln1_b", "wih1_t", "b1")]


class EmbWeights(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("dft", "wc", "bc", "gn_g", "gn_b", "lnh_g", "lnh_b")]


class EmbBlock(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("gq", "bq", "gk", "bk", "gv", "bv", "wp_t", "bp", "slope_p", "gp", "bpn")]


class RowsGemm(ctypes.Structure):
    """GemmArgs (gemm.cuh) field for field"""
    _fields_ = [("A", ctypes.c_void_p), ("lda", ctypes.c_int64), ("a_rows_per_seq", ctypes.c_int32),
                ("a_seq_stride", ctypes.c_int64), ("Wt", ctypes.c_void_p), ("bias", ctypes.c_void_p), ("C", ctypes.c_void_p),
                ("ldc", ctypes.c_int64), ("c_rows_per_seq", ctypes.c_int32), ("c_seq_stride", ctypes.c_int64),
                ("c_inner", ctypes.c_int32), ("c_inner_stride", ctypes.c_int64)] + \
               [(n, ctypes.c_void_p) for n in ("R", "ln_g", "ln_b", "prelu", "prelu_vec")] + \
               [("M", ctypes.c_int32), ("N", ctypes.c_int32), ("K", ctypes.c_int32)]


class MidWeights(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("mid_pack", "bl1", "ln2_g", "ln2_b", "b2", "bl2", "bqkv", "slopes")]


class TailWeights(ctypes.Structure):
    """KhTailWeights: the fields of BlockWeights that tail_kernel reads, then the next block's input projection (nx_wih_t
    null: no next block)"""
    _fields_ = [(n, ctypes.c_void_p) for n in ("mid_pack", "bl1", "ln2_g", "ln2_b", "b2", "bl2", "bqkv", "slopes", "lnq_g",
                                                "lnq_b", "lnk_g", "lnk_b", "lnv_g", "lnv_b", "wp_t", "bp", "lnp_g", "lnp_b",
                                                "nx_ln_g", "nx_ln_b", "nx_wih_t", "nx_bias")]


class Records(ctypes.Structure):
    """KhRecords = Records (sep_kernels.cuh): row b is record slots[b] of `batch` records of `stride` floats"""
    _fields_ = [("stride", ctypes.c_int64), ("slots", ctypes.c_void_p), ("batch", ctypes.c_int32), ("hops", ctypes.c_void_p),
                ("frames", ctypes.c_int32)]


MIRRORS = {"kh_sizeof_asource": ASource, "kh_sizeof_gemm": Gemm, "kh_sizeof_plan": Plan, "kh_sizeof_lstm": Lstm,
           "kh_sizeof_sep_weights": SepWeights, "kh_sizeof_sep_front_back": SepFrontBack,
           "kh_sizeof_emb_weights": EmbWeights, "kh_sizeof_emb_block": EmbBlock, "kh_sizeof_rows_gemm": RowsGemm,
           "kh_sizeof_mid_weights": MidWeights, "kh_sizeof_tail_weights": TailWeights, "kh_sizeof_records": Records}
MID_SYMBOLS = ("kh_rows_gemm", "kh_rows_gemm_form", "kh_mid_layout", "kh_mid_pack", "kh_mid", "kh_mid_a", "kh_mid_b",
               "kh_mid_c", "kh_lstm_cell_rows")
TAIL_SYMBOLS = ("kh_tail_clusters", "kh_tail", "kh_tail_slots")
TARGETS_SYMBOLS = ("kh_target_lists", "kh_spk_gate", "kh_gate_fanout", "kh_gather_h", "kh_scatter_hc", "kh_inter_gate_mask",
                   "kh_inter_h_last")
EMBED_SYMBOLS = ("kh_embed_layout", "kh_estd", "kh_efront", "kh_egn_apply", "kh_eqkv_ln", "kh_softmax_rows",
                 "kh_eattn_out_grid", "kh_eattn_out", "kh_ehead", "kh_einter_mask", "kh_eput_lens")
SYMBOLS = ("kh_gemm", "kh_gemm_plan", "kh_split_planes", "kh_lstm", "kh_launch_count", "kh_sep_layout", "kh_qkv",
           "kh_qkv_many", "kh_kv_gather", "kh_attention", "kh_attn_out", "kh_ln_frame_res",
           "kh_attn_cluster_resident", "kh_front", "kh_front_many", "kh_front_many_geometry", "kh_front1", "kh_back",
           "kh_back_many", "kh_back_many_geometry") + EMBED_SYMBOLS + MID_SYMBOLS + TAIL_SYMBOLS + TARGETS_SYMBOLS + tuple(MIRRORS)
EMBED_LAYOUT_NAMES = ("NFFT", "HOP", "NF", "CH", "QK", "VDIM", "FC", "NQKV", "DFT_LD", "EAOUT_SMEM", "LENS_PER_LAUNCH")

ATTN_FORMS = {"query": 0, "tile": 1, "cluster": 2}
SEP_LAYOUT_NAMES = ("RING", "QK_LD", "QK_DIM", "V_DIM", "ATT", "ST_GATE", "ST_BLK", "BK_K", "BK_V", "BK_H", "BK_C",
                    "BK_STRIDE", "ST_POS", "ST_CALLS", "HEADER_BYTES", "STREAM_STRIDE", "ST_EMB", "ST_GEN", "ST_CONV",
                    "ST_DECONV", "ST_ISTFT")

_lib = None


def lib():
    """Build the harness if its sources changed (a no-op after build()) and load it."""
    global _lib
    if _lib is None:
        L = ctypes.CDLL(_build.build_harness())
        for s in MIRRORS:
            getattr(L, s).restype = ctypes.c_int
        L.kh_launch_count.restype = ctypes.c_longlong
        L.kh_gemm.restype = ctypes.c_int
        L.kh_gemm.argtypes = [ctypes.POINTER(Gemm), ctypes.POINTER(Plan), ctypes.c_char_p, ctypes.c_int, ctypes.c_void_p]
        L.kh_gemm_plan.restype = ctypes.c_int
        L.kh_gemm_plan.argtypes = [ctypes.POINTER(Gemm), ctypes.POINTER(Plan)]
        L.kh_split_planes.restype = ctypes.c_int
        L.kh_split_planes.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
                                      ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.kh_lstm.restype = ctypes.c_int
        L.kh_lstm.argtypes = [ctypes.POINTER(Lstm), ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_int, ctypes.c_void_p]
        P, I, I64, W = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.POINTER(SepWeights)
        sigs = {
            "kh_sep_layout": [I, ctypes.POINTER(ctypes.c_int64)],
            "kh_attn_cluster_resident": [],
            "kh_qkv": [W, P, P, P, P, P, P, I64, I, I, I, I, P, P],
            "kh_qkv_many": [W, P, P, P, P, P, I64, I, I, I, I, P, P],
            "kh_kv_gather": [P, I64, I, P, P, I, I, P],
            "kh_attention": [I, P, P, P, P, I64, I, P, I, I, I, P],
            "kh_attn_out": [W, P, P, P, I64, I, I, I, P],
            "kh_ln_frame_res": [W, P, P, P, I64, I, I, I, P],
        }
        FB, IP = ctypes.POINTER(SepFrontBack), ctypes.POINTER(ctypes.c_int)
        sigs.update({
            "kh_front": [FB, P, I64, I64, I, P, P, I64, I, I, I, P, P, I, I, P, P],
            "kh_front_many": [FB, P, I64, I64, I, P, P, I64, I, I, I, P, P, I, I, P, P],
            "kh_front1": [FB, P, I64, I64, I, P, P, P, I64, I, I, P, P, P, P],
            "kh_back": [FB, P, P, I64, I64, I, P, I64, I, I, I, I, I, I64, P, P],
            "kh_back_many": [FB, P, P, I64, I64, I, P, I64, I, I, I, I, I, P, P],
        })
        for s in ("kh_front_many_geometry", "kh_back_many_geometry"):
            getattr(L, s).restype = None
            getattr(L, s).argtypes = [I, I, IP, IP]
        EW, EB = ctypes.POINTER(EmbWeights), ctypes.POINTER(EmbBlock)
        sigs.update({
            "kh_embed_layout": [ctypes.POINTER(ctypes.c_int64)],
            "kh_estd": [P, I, P, P, I, P],
            "kh_efront": [EW, P, I, P, P, P, P, I, I, P],
            "kh_egn_apply": [EW, P, P, I64, I64, P, P],
            "kh_eqkv_ln": [EB, P, P, P, P, I64, I64, I, I, I, P],
            "kh_softmax_rows": [P, I64, I, I, I64, I, P, P],
            "kh_eattn_out_grid": [I, I],
            "kh_eattn_out": [EB, P, P, I, I, I, I, P],
            "kh_ehead": [EW, P, P, I, I, P, P],
            "kh_einter_mask": [P, P, I, I, P],
            "kh_eput_lens": [P, P, I, P],
        })
        MW = ctypes.POINTER(MidWeights)
        sigs.update({
            "kh_rows_gemm": [ctypes.POINTER(RowsGemm), I, IP, P],
            "kh_rows_gemm_form": [I, I, I, I],
            "kh_mid_layout": [ctypes.POINTER(ctypes.c_int64)],
            "kh_mid": [MW, P, P, P, P, I64, I, I, P, P],
            "kh_mid_a": [MW, P, P, P, I, I64, I, P],
            "kh_mid_b": [MW, P, P, I64, I, P, I64, I, I, P, P],
            "kh_mid_c": [MW, P, P, P, I, I64, I, P],
            "kh_lstm_cell_rows": [P, P, I64, I, P, I64, P, P],
        })
        TW = ctypes.POINTER(TailWeights)
        sigs.update({
            "kh_tail_clusters": [],
            "kh_tail": [TW, P, P, P, P, I64, I, I, I, I, P, P],
            "kh_tail_slots": [TW, P, P, P, P, I64, P, I, P, I, I, I, P],
        })
        RP = ctypes.POINTER(Records)
        sigs.update({
            "kh_target_lists": [P, P, P, P, I, I, I, I, P, P],
            "kh_spk_gate": [FB, P, P, P, I64, RP, I, P],
            "kh_gate_fanout": [P, P, P, I64, RP, P, I, I, I, I, P],
            "kh_gather_h": [P, RP, I, I, I, P, P, P],
            "kh_scatter_hc": [P, RP, I, I, I, P, P, P],
            "kh_inter_gate_mask": [P, RP, I, P],
            "kh_inter_h_last": [P, P, RP, I, P],
        })
        L.kh_mid_pack.restype = None
        L.kh_mid_pack.argtypes = [P] * 6
        for s, args in sigs.items():
            getattr(L, s).restype = ctypes.c_int
            getattr(L, s).argtypes = args
        _lib = L
    return _lib


def ptr(t):
    return None if t is None else t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def gemm(desc):
    """(cudaError_t, plan, why) of one kh_gemm call."""
    plan, why = Plan(), ctypes.create_string_buffer(256)
    rc = lib().kh_gemm(ctypes.byref(desc), ctypes.byref(plan), why, 256, stream())
    return rc, plan, why.value.decode()


def gemm_plan(desc):
    """the plan umma::launch would use for `desc` (no launch, no device needed), or None if it refuses the problem"""
    plan = Plan()
    return plan if lib().kh_gemm_plan(ctypes.byref(desc), ctypes.byref(plan)) == 0 else None


def lstm(args, variant, passes=3):
    why = ctypes.create_string_buffer(256)
    rc = lib().kh_lstm(ctypes.byref(args), LSTM_VARIANTS[variant], passes, why, 256, stream())
    return rc, why.value.decode()


def sep_layout(n_blocks):
    """kh_sep_layout as {name: value} (SEP_LAYOUT_NAMES): offsets in floats, HEADER_BYTES in bytes"""
    out = (ctypes.c_int64 * 32)()
    n = lib().kh_sep_layout(n_blocks, out)
    return dict(zip(SEP_LAYOUT_NAMES, list(out)[:n]))


def qkv(w, X, pre, Q, K, V, state, sstride, blk, B, T, frame_k=0, active=None):
    return lib().kh_qkv(ctypes.byref(w), ptr(X), ptr(pre), ptr(Q), ptr(K), ptr(V), ptr(state), sstride, blk, B, T, frame_k,
                        ptr(active), stream())


def qkv_many(w, pre, Q, K, V, state, sstride, blk, T, grid, n_frames, active=None):
    return lib().kh_qkv_many(ctypes.byref(w), ptr(pre), ptr(Q), ptr(K), ptr(V), ptr(state), sstride, blk, T, grid, n_frames,
                             ptr(active), stream())


def kv_gather(state, sstride, blk, K, V, B, T):
    return lib().kh_kv_gather(ptr(state), sstride, blk, ptr(K), ptr(V), B, T, stream())


def attention(form, Q, K, V, state, sstride, blk, Z, B, T, frame_k=0):
    return lib().kh_attention(ATTN_FORMS[form], ptr(Q), ptr(K), ptr(V), ptr(state), sstride, blk, ptr(Z), B, T, frame_k,
                              stream())


def attn_out(w, Z, X, state, sstride, B, T, apply_gate):
    return lib().kh_attn_out(ctypes.byref(w), ptr(Z), ptr(X), ptr(state), sstride, B, T, apply_gate, stream())


def ln_frame_res(w, P, X, state, sstride, B, T, apply_gate):
    return lib().kh_ln_frame_res(ctypes.byref(w), ptr(P), ptr(X), ptr(state), sstride, B, T, apply_gate, stream())


# x, y: [B][2][n] (any strides along the first two dimensions); x_len / y_len count samples of the last dimension
def front(w, x, x_len, X, state, sstride, B, T, pos_rel, emb, spk_pre, frame_k=0, frames_total=1, active=None):
    return lib().kh_front(ctypes.byref(w), ptr(x), x.stride(0), x.stride(1), x_len, ptr(X), ptr(state), sstride, B, T, pos_rel,
                          ptr(emb), ptr(spk_pre), frame_k, frames_total, ptr(active), stream())


def front_many_geometry(B, T):
    """(chunk, n_workers) the engine launches front_many_kernel with"""
    c, n = ctypes.c_int(), ctypes.c_int()
    lib().kh_front_many_geometry(B, T, ctypes.byref(c), ctypes.byref(n))
    return c.value, n.value


def front_many(w, x, x_len, X, state, sstride, B, T, pos_rel, emb, spk_pre, chunk, n_workers, active=None):
    return lib().kh_front_many(ctypes.byref(w), ptr(x), x.stride(0), x.stride(1), x_len, ptr(X), ptr(state), sstride, B, T,
                               pos_rel, ptr(emb), ptr(spk_pre), chunk, n_workers, ptr(active), stream())


def front1(w, x, x_len, X, GX, state, sstride, B, pos_rel, emb, spk_pre, active=None):
    return lib().kh_front1(ctypes.byref(w), ptr(x), x.stride(0), x.stride(1), x_len, ptr(X), ptr(GX), ptr(state), sstride, B,
                           pos_rel, ptr(emb), ptr(spk_pre), ptr(active), stream())


def back(w, X, y, y_len, state, sstride, B, T, pos_rel, frame_k=0, frames_total=1, hist_stride=0, active=None):
    return lib().kh_back(ctypes.byref(w), ptr(X), ptr(y), y.stride(0), y.stride(1), y_len, ptr(state), sstride, B, T, pos_rel,
                         frame_k, frames_total, hist_stride, ptr(active), stream())


def back_many_geometry(B, T):
    """(chunk, n_cl) the engine launches back_many_kernel with"""
    c, n = ctypes.c_int(), ctypes.c_int()
    lib().kh_back_many_geometry(B, T, ctypes.byref(c), ctypes.byref(n))
    return c.value, n.value


def back_many(w, X, y, y_len, state, sstride, B, T, pos_rel, chunk, n_cl, active=None):
    return lib().kh_back_many(ctypes.byref(w), ptr(X), ptr(y), y.stride(0), y.stride(1), y_len, ptr(state), sstride, B, T,
                              pos_rel, chunk, n_cl, ptr(active), stream())


# ---- float64 references ---------------------------------------------------------------------------------------------
def split_bf16(x):
    """bf16 hi/lo planes of fp32 x, as the kernels form them (round to nearest even; x - hi exact in fp32)."""
    x = x.float()
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi, lo


def split_product(a, b, passes):
    """float64 emulation of sum_k a[m,k] b[n,k] with the split terms of `passes` (a, b fp32 [M,K], [N,K])."""
    ah, al = (t.double() for t in split_bf16(a))
    bh, bl = (t.double() for t in split_bf16(b))
    out = ah @ bh.T
    if passes >= 2:
        out = out + al @ bh.T
    if passes >= 3:
        out = out + ah @ bl.T
    return out


def layer_norm64(x, g, b, eps=1e-5, unbiased=False):
    """LayerNorm over the last dimension: biased variance, eps inside the sqrt (unbiased=True: a mutated reference)"""
    x = x.double()
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    if unbiased:
        var = var * x.shape[-1] / (x.shape[-1] - 1)
    return (x - mu) / torch.sqrt(var + eps) * g.double() + b.double()


# ---- the separator's attention section (tfgridnet_causal.py:540-588; oracle/restate.py::sep_block) ------------------
# Shapes: NF = 97 bins, CH = 64 channels, NHEAD = 4 heads, QE = 6 (Q/K features per bin and head), VD = 16 (V), a
# window of ATT = 50 frames.  Q/K rows are QK_DIM = 582 = 97*6 values (element f*6 + e), stored QK_LD = 584 wide; V rows
# are V_DIM = 1552 = 97*16 values (f*16 + c).  The mutated references (keyword flags) restate the plausible mistakes a
# kernel could make; the tests show that each one is far outside the bound the kernels meet.
NF, CH, NHEAD, QE, VD, ATT, RING = 97, 64, 4, 6, 16, 50, 56
QK_DIM, QK_LD, V_DIM, FC, NQKV = NF * QE, 584, NF * VD, NF * CH, 2 * 4 * 6 + 4 * 16


def prelu64(x, a):
    return torch.where(x >= 0, x, a * x)


def qkv_proj64(X, wqkv_t, bqkv, slopes, swap_qk_slopes=False):
    """Linear 64 -> 112 + bias + PReLU (slope slopes[0] on the Q columns 0..23, [1] on K 24..47, [2] on V 48..111) of
    X [..., 97, 64] -> [..., 97, 112] (tfgridnet_causal.py:354-387: attn_conv_Q/K/V, layers .0 and .1)"""
    s = slopes.double()
    sq, sk = (s[1], s[0]) if swap_qk_slopes else (s[0], s[1])
    a = torch.cat([sq.expand(24), sk.expand(24), s[2].expand(64)])
    return prelu64(X.double() @ wqkv_t.double() + bqkv.double(), a)


def qkv_ln64(P, lnq, lnk, lnv, unbiased=False, heads_transposed=False):
    """head split + LayerNorm over (F, E) per (Q/K/V, head) of projections P [N, 97, 112] -> Q, K [N, 4, 582] and
    V [N, 4, 1552].  Head h of Q owns columns h*6 + e, element i = f*6 + e (K: 24 + h*6 + e; V: 48 + h*16 + c).
    lnq / lnk / lnv: (gain, bias), of at least 582 / 1552 values.  heads_transposed: column e*4 + h (a mutant)."""
    N = P.shape[0]
    out = []
    for d, c0, (g, b) in ((QE, 0, lnq), (QE, 24, lnk), (VD, 48, lnv)):
        cols = P[:, :, c0:c0 + NHEAD * d].double()
        y = cols.view(N, NF, d, NHEAD).permute(0, 3, 1, 2) if heads_transposed else cols.view(N, NF, NHEAD, d).permute(0, 2, 1, 3)
        n = NF * d
        out.append(layer_norm64(y.reshape(N, NHEAD, n), g[:n], b[:n], unbiased=unbiased))
    return tuple(out)


def window_mask(qframes, kframes, lo=-(ATT - 1), hi=0, mask_before_start=False):
    """[T, n] bool: query frame qframes[t] attends to key frame kframes[j] iff qframes[t] + lo <= kframes[j] <=
    qframes[t] + hi -- the model's window is the 50 frames ending at the query's (lo = -49, hi = 0).  Frames before the
    stream start are zero rows that TAKE PART in the softmax (the reference's zero-initialised K_buf / V_buf);
    mask_before_start=True leaves them out instead (a mutant)."""
    q = torch.as_tensor(qframes, dtype=torch.int64)[:, None]
    k = torch.as_tensor(kframes, dtype=torch.int64)[None, :]
    w = (k >= q + lo) & (k <= q + hi)
    return w & (k >= 0) if mask_before_start else w


def attention64(q, K, V, window, scale=1.0 / QK_DIM ** 0.5):
    """softmax(q . k * scale) V over each query's window: q [T, H, >=582], K [n, H, >=582] and V [n, H, 1552] the rows
    of n frames, window [T, n] (window_mask) -> [T, H, 1552]"""
    s = torch.einsum("thd,nhd->htn", q[..., :QK_DIM].double(), K[..., :QK_DIM].double()) * scale
    s = s.masked_fill(~window[None], float("-inf"))
    return torch.einsum("htn,nhd->thd", torch.softmax(s, dim=-1), V.double())


def merge_heads64(o, transposed=False):
    """head outputs o [N, 4, 1552] (feature f*16 + c) -> Z [N, 97, 64] with channel h*16 + c of bin f
    (tfgridnet_causal.py:575-581); transposed: channel c*4 + h (a mutant)"""
    N = o.shape[0]
    z = o.double().view(N, NHEAD, NF, VD).permute(0, 2, 1, 3)          # [N, 97, 4, 16]
    if transposed:
        z = z.transpose(2, 3)
    return z.reshape(N, NF, CH)


def ln_frame_res64(P, X, g, b, gate=None, per_bin=False, gate_first=False, unbiased=False):
    """X + LayerNorm over the frame's 6208 values (f, c) of P [N, 97, 64], times the speaker gate [N, 97, 64] if given
    (tfgridnet_causal.py:583-588, :250-251).  Mutants: per_bin (LayerNorm over each bin's 64 values), gate_first
    (X * gate + LN), unbiased (variance over n - 1)."""
    N = P.shape[0]
    if per_bin:
        y = layer_norm64(P, g.view(NF, CH), b.view(NF, CH), unbiased=unbiased)
    else:
        y = layer_norm64(P.reshape(N, FC), g, b, unbiased=unbiased).view(N, NF, CH)
    x = X.double()
    if gate is None:
        return x + y
    gate = gate.double().view(N, NF, CH)
    return x * gate + y if gate_first else (x + y) * gate


def attn_out64(Z, X, wp_t, bp, slope, g, b, gate=None, **mutant):
    """Linear 64 -> 64 + bias + PReLU (slopes[3]) of Z [N, 97, 64], then ln_frame_res64"""
    return ln_frame_res64(prelu64(Z.double() @ wp_t.double() + bp.double(), float(slope)), X, g, b, gate, **mutant)


class Ring:
    """Where the kernels keep a stream's K/V history (sep_layout.h): frame n of head h lives in slot n mod RING of the
    block's K ring (and V ring), at ST_BLK + blk*BK_STRIDE + BK_K (BK_V) + (h*RING + slot) * row floats of the stream's
    record.  The attention window of frame n is frames n-49 .. n; the other RING - ATT slots ("spare": frames n-55 ..
    n-50) hold rows that later hops of the pipelined graph may already have overwritten."""

    def __init__(self, lay):
        self.lay = lay
        assert lay["RING"] == RING and lay["ATT"] == ATT and lay["QK_LD"] == QK_LD and lay["V_DIM"] == V_DIM

    @staticmethod
    def slot(n):
        return n % RING                                  # Python's % is non-negative: frame -1 -> slot 55

    def row(self, blk, which, h, n):
        """offset (floats) of frame n's row of head h inside a stream record; which = 'k' or 'v'"""
        base = self.lay["ST_BLK"] + blk * self.lay["BK_STRIDE"]
        if which == "k":
            return base + self.lay["BK_K"] + (h * RING + self.slot(n)) * QK_LD
        return base + self.lay["BK_V"] + (h * RING + self.slot(n)) * V_DIM

    @staticmethod
    def window(n, lo=-(ATT - 1), hi=0):
        return list(range(n + lo, n + hi + 1))

    @staticmethod
    def spare(n):
        return list(range(n - RING + 1, n - ATT + 1))


def lstm_ref(gx, whh, nseq, L, ndir, row_of, h0=None, c0=None):
    """float64 LSTM over the packed gate layout of lstm.cuh: gx [rows][ndir*256] (column d*256 + j*4 + q, q = i, f, g, o),
    whh [ndir][256][64].  row_of(seq [nseq], step) -> gx rows.  Direction 1 runs the steps in reverse.  h0 / c0
    [nseq][64] (direction 0 only).  Returns h [ndir][L][nseq][64] indexed by step, and the final (h, c) per direction."""
    gx = gx.double()
    seqs = torch.arange(nseq)
    hs = torch.zeros(ndir, L, nseq, 64, dtype=torch.float64)
    finals = []
    for d in range(ndir):
        h = torch.zeros(nseq, 64, dtype=torch.float64) if h0 is None or d else h0.double().clone()
        c = torch.zeros(nseq, 64, dtype=torch.float64) if c0 is None or d else c0.double().clone()
        w = whh[d]
        for s in (range(L) if d == 0 else range(L - 1, -1, -1)):
            g = (gx[row_of(seqs, s), d * 256:(d + 1) * 256] + h @ w.double().T).view(nseq, 64, 4)
            i, f, gg, o = torch.sigmoid(g[..., 0]), torch.sigmoid(g[..., 1]), torch.tanh(g[..., 2]), torch.sigmoid(g[..., 3])
            c = f * c + i * gg
            h = o * torch.tanh(c)
            hs[d, s] = h
        finals.append((h, c))
    return hs, finals


def packed_from_torch(w):
    """torch.nn.LSTM gate rows (q*64 + j) -> the packed rows of lstm.cuh (j*4 + q)."""
    return w.view(4, 64, *w.shape[1:]).transpose(0, 1).reshape(w.shape)


# ---- the separator's front and back (tfgridnet_causal.py:229-273; oracle/restate.py::sep_core) -----------------------
# One stream at a time.  Frame t of a call covers samples s0 + 128 t .. + 191 (128 new samples and the 64-sample
# look-ahead); the spectrum has channels [Re m0, Re m1, Im m0, Im m1] and bins f = 0..96; the conv reads the two frames
# before the call from the conv tail [2][4][97] and zero-pads in F; the transposed conv reads the deconv tail [2][97][64];
# the synthesis of frame t-1 comes from the iSTFT tail [2 ears][194].  Each reference returns, next to every value, an
# element-wise bound on the fp32 rounding error of a kernel that computes it: u sqrt(n) sum |terms| for each sum of n
# terms (with the bounds of its inputs carried through), u = 2^-24.  The mutant flags restate plausible kernel mistakes.
HOP, NFFT, LOOKAHEAD, NROW, SPK = 128, 192, 64, 194, 256
U32 = 2.0 ** -24
# A LayerNorm's own rounding, relative to a normalised value: the variance is a block sum of <= 25 sequential terms per
# thread and an 8-level tree (<= 33 roundings of positive terms, 17 u on its square root), rsqrtf adds <= 2 ulp (4 u)
# and the final multiply-add 3 roundings: at most this many u (the 64-value LayerNorms of front1_kernel round less)
LN_U = 24


def frames64(x, x_len, s0, T):
    """[2, T, 192] float64: frame t of mic m = x[m, s0 + 128 t + n], zero outside [0, x_len) (x [2][>= x_len])"""
    idx = s0 + HOP * torch.arange(T)[:, None] + torch.arange(NFFT)[None, :]
    ok = (idx >= 0) & (idx < x_len)
    out = torch.zeros(x.shape[0], T, NFFT, dtype=torch.float64)
    out[:, ok] = x[:, idx[ok]].double()
    return out


def _pad_f(u, clamp=False):
    """[..., 97, ...] with F on dim -2 (X-like) -> zero-padded (or edge-clamped: a mutant) to 99 bins"""
    lo, hi = (u[..., :1, :], u[..., -1:, :]) if clamp else (torch.zeros_like(u[..., :1, :]),) * 2
    return torch.cat([lo, u, hi], dim=-2)


def front64(x, x_len, s0, T, conv_tail, Wa, Wc, bc, shift=0, reim_interleaved=False, conv_flip_time=False,
            edge_clamp=False):
    """STFT analysis, channel regroup and the causal 3x3 conv of one stream (tfgridnet_causal.py:229-242).
    x [2][n] (fp32), conv_tail [2][4][97] (frames -2, -1), Wa [194][192] analysis filters, Wc [64][4][3][3], bc [64].
    Returns X [T][97][64], the new conv tail [2][4][97] (spectra of the call's last two frames) and their bounds.
    Mutants: shift (frames one hop late), reim_interleaved (channels [Re m0, Im m0, Re m1, Im m1]), conv_flip_time
    (kernel rows i -> 2 - i), edge_clamp (bins -1 and 97 copy bins 0 and 96)."""
    fr = frames64(x, x_len, s0 + HOP * shift, T)
    Wa = Wa.double()
    S, Sa = fr @ Wa.T, fr.abs() @ Wa.abs().T                              # [2, T, 194]
    order = [0, 2, 1, 3] if reim_interleaved else [0, 1, 2, 3]              # channel ri*2 + m (mutant: m*2 + ri)

    def regroup(s):
        u = torch.stack([s[0, :, :NF], s[1, :, :NF], s[0, :, NF:], s[1, :, NF:]], dim=1)   # [T, 4, 97]
        return u[:, order]
    tail = conv_tail.double()
    Up = torch.cat([tail, regroup(S)])                                      # [T + 2, 4, 97]
    Ua = torch.cat([tail.abs(), regroup(Sa)])
    Ue = torch.cat([torch.zeros_like(tail), regroup(Sa) * (U32 * math.sqrt(NFFT))])     # bound of each spectrum value
    W = Wc.double()
    if conv_flip_time:
        W = W.flip(2)
    X = torch.zeros(T, NF, CH, dtype=torch.float64) + bc.double()
    Xa = torch.zeros_like(X) + bc.double().abs()
    Xe = torch.zeros_like(X)
    pads = [_pad_f(u.transpose(1, 2), edge_clamp) for u in (Up, Ua, Ue)]  # [T + 2, 99, 4]
    for i in range(3):
        for j in range(3):
            w = W[:, :, i, j]
            X = X + pads[0][i:i + T, j:j + NF] @ w.T
            Xa = Xa + pads[1][i:i + T, j:j + NF] @ w.abs().T
            Xe = Xe + pads[2][i:i + T, j:j + NF] @ w.abs().T
    return dict(X=X, X_bound=Xe + U32 * math.sqrt(37) * Xa, tail=Up[-2:], tail_bound=Ue[-2:])


def gate64(e, We, be, g, b, cf_order=False, unbiased=False):
    """speaker gate LN_6208(We e + be) (tfgridnet_causal.py:247-248), element c*97 + f stored at [f][c] -> ([97][64],
    bound).  Mutants: cf_order (element i stored at flat i), unbiased (variance over 6207)."""
    # each row is a 256-term dot product whose longest rounding chain is 8 products per lane, a 5-level warp tree and
    # the bias: 16 roundings; an error pe in p moves y by |g| (pe + mean pe) / sigma, and |g xh| mean pe / sigma more
    # through sigma
    p = We.double() @ e.double() + be.double()
    pe = U32 * math.sqrt(16) * (We.double().abs() @ e.double().abs() + be.double().abs())
    y = layer_norm64(p, g, b, unbiased=unbiased)
    sd = p.std(unbiased=False)
    gx = (g.double() * (p - p.mean()) / sd).abs()
    bound = (g.double().abs() * (pe + pe.mean()) + gx * pe.mean()) / sd + U32 * (LN_U * gx + 2 * b.double().abs())
    if cf_order:
        return y.view(NF, CH), bound.view(NF, CH)
    return y.view(CH, NF).T, bound.view(CH, NF).T



def ih64(X, g, b, wih_t, bias):
    """block 0's intra input projection LN_64(X) W_ih^T + b of X [97][64] -> ([97][512], bound); wih_t [64][512] and
    bias [512] in the packed column order d*256 + j*4 + q of lstm.cuh"""
    xn = layer_norm64(X, g, b)
    xh = (X.double() - X.double().mean(-1, keepdim=True)) / X.double().std(-1, unbiased=False, keepdim=True)
    W = wih_t.double()
    out = xn @ W + bias.double()
    bound = U32 * (math.sqrt(65) * (xn.abs() @ W.abs() + bias.double().abs()) + LN_U * ((g.double() * xh).abs() @ W.abs()))
    return out, bound


def back64(X, deconv_tail, istft_tail, Wd, bd, Ws, plain_conv=False, swap_ear_ri=False, ola="model", carry_istft=True):
    """causal 3x3 transposed conv, Re/Im regroup, synthesis and overlap-add of one stream (tfgridnet_causal.py:256-273,
    net.py:61).  X [T][97][64], deconv_tail [2][97][64] (frames -2, -1), istft_tail [2 ears][194] (frame -1), Wd
    [64][4][3][3] (c, o, i, j), bd [4], Ws [194][192] synthesis filters.  D[o,t,f] = bd[o] + sum Wd[c,o,i,j]
    Xp[c,t+2-i,f+1-j]; channel o = 2 ear + ri; output sample 128 t + n = w_t[n] (+ w_{t-1}[128 + n] for n < 64).
    Returns y [2][128 T], the new deconv tail [2][97][64], the new iSTFT tail [2][194] and bounds.
    Mutants: plain_conv (kernel flipped in both axes), swap_ear_ri (o = 2 ri + ear), ola = "dropped" (no tail added) or
    "wrong_half" (w_{t-1}[n] added), carry_istft=False (frame -1 synthesised from zeros)."""
    T = X.shape[0]
    Xp = torch.cat([deconv_tail.double(), X.double()])                     # [T + 2, 97, 64]
    Xpp, Xpa = _pad_f(Xp), _pad_f(Xp.abs())                                # [T + 2, 99, 64]
    W = Wd.double()
    if plain_conv:
        W = W.flip(2, 3)
    D = torch.zeros(4, T, NF, dtype=torch.float64) + bd.double()[:, None, None]
    Da = torch.zeros_like(D) + bd.double().abs()[:, None, None]
    for i in range(3):
        for j in range(3):
            D = D + torch.einsum("tfc,co->otf", Xpp[2 - i:2 - i + T, 2 - j:2 - j + NF], W[:, :, i, j])
            Da = Da + torch.einsum("tfc,co->otf", Xpa[2 - i:2 - i + T, 2 - j:2 - j + NF], W[:, :, i, j].abs())
    De = U32 * math.sqrt(4 * 9 * 64) * Da

    def regroup(d):                                                        # [4, T, 97] -> [2 ears, T, 194]
        pairs = [(0, 2), (1, 3)] if swap_ear_ri else [(0, 1), (2, 3)]
        return torch.stack([torch.cat([d[a], d[c]], dim=-1) for a, c in pairs])
    R, Ra, Re = regroup(D), regroup(D.abs()), regroup(De)
    tail = istft_tail.double() if carry_istft else torch.zeros(2, NROW, dtype=torch.float64)
    Rp = torch.cat([tail[:, None], R], dim=1)                              # [2, T + 1, 194]
    Rpa = torch.cat([istft_tail.double().abs()[:, None], Ra], dim=1)
    Rpe = torch.cat([torch.zeros(2, 1, NROW, dtype=torch.float64), Re], dim=1)
    Wsd = Ws.double()
    w = Rp @ Wsd                                                           # [2, T + 1, 192]
    wa = Rpa @ Wsd.abs()
    we = Rpe @ Wsd.abs()

    def ola_(v, mode):
        head = v[:, 1:, :HOP].clone()
        if mode == "model":
            head[..., :LOOKAHEAD] += v[:, :-1, HOP:]
        elif mode == "wrong_half":
            head[..., :LOOKAHEAD] += v[:, :-1, :LOOKAHEAD]
        return head.reshape(2, T * HOP)
    bound = ola_(we, "model") + U32 * math.sqrt(NROW + 2 * 4) * ola_(wa, "model")
    return dict(y=ola_(w, ola), y_bound=bound, deconv_tail=Xp[-2:], istft_tail=R[:, -1], istft_bound=Re[:, -1])


def pack_front_back(sd, pad=float("nan"), prefix="tfgridnet."):
    """the front / back weights of a state dict in the kernels' layouts (SepWeights): wat [192][196] (the analysis
    filters transposed, 2 pad columns = pad), ws [194][192], wc [64][36], wd [64][4][9], we [6208][256], be, and the
    gate LayerNorm's lne_g / lne_b in c*97 + f order (the model's own)"""
    g = lambda k: sd[prefix + k].detach().float()
    wa = g("enc.filterbank._filters")[:, 0]
    wat = torch.full((NFFT, NROW + 2), pad, dtype=torch.float32)
    wat[:, :NROW] = wa.T
    return dict(wat=wat, ws=g("dec.filterbank._filters")[:, 0].contiguous(), wc=g("conv.0.weight").reshape(CH, 36),
                bc=g("conv.0.bias"), we=g("embed_to_feats_proj.0.weight"), be=g("embed_to_feats_proj.0.bias"),
                lne_g=g("embed_to_feats_proj.1.weight"), lne_b=g("embed_to_feats_proj.1.bias"),
                wd=g("deconv.weight").reshape(CH, 4, 9), bd=g("deconv.bias"))


def unpack_front_back(p, prefix="tfgridnet."):
    """pack_front_back's inverse: the state-dict tensors"""
    return {prefix + "enc.filterbank._filters": p["wat"][:, :NROW].T.reshape(NROW, 1, NFFT),
            prefix + "dec.filterbank._filters": p["ws"].reshape(NROW, 1, NFFT),
            prefix + "conv.0.weight": p["wc"].reshape(CH, 4, 3, 3), prefix + "conv.0.bias": p["bc"],
            prefix + "embed_to_feats_proj.0.weight": p["we"], prefix + "embed_to_feats_proj.0.bias": p["be"],
            prefix + "embed_to_feats_proj.1.weight": p["lne_g"], prefix + "embed_to_feats_proj.1.bias": p["lne_b"],
            prefix + "deconv.weight": p["wd"].reshape(CH, 4, 3, 3), prefix + "deconv.bias": p["bd"]}


# ---- the enrollment network's own kernels (embed_kernels.cuh; tfgridnet.py:100-127, oracle/restate.py::embed_forward
# and embed_block) ----------------------------------------------------------------------------------------------------
# Activations [T][F = 65][C = 64] per utterance.  An utterance of n own samples has T_b = 1 + n // 64 frames; frames
# t >= T_b of a padded batch are padding.  Every reference takes float64 copies of the kernel's fp32 inputs and returns,
# next to every value, an element-wise bound on the kernel's fp32 rounding (u = 2^-24 per rounding, u sqrt(n) sum |terms|
# for a sum of n terms, input bounds carried through).  The keyword flags are the mutants: plausible kernel mistakes.
E_NFFT, E_HOP, E_NF, E_CH, E_NH, E_QE, E_VD = 128, 64, 65, 64, 4, 8, 16
E_QK, E_VDIM, E_FC, E_NQKV, E_DFT_LD, E_LENS_PER_LAUNCH = 520, 1040, 4160, 128, 132, 1000
E_PAD_GATES = (float("-inf"), float("-inf"), 0.0, 0.0)      # (i, f, g, o) of a padded inter window


def embed_layout():
    """kh_embed_layout as {name: value} (EMBED_LAYOUT_NAMES; EAOUT_SMEM in bytes)"""
    out = (ctypes.c_int64 * 16)()
    n = lib().kh_embed_layout(out)
    return dict(zip(EMBED_LAYOUT_NAMES, list(out)[:n]))


def estd(x, N, lens, inv_std, B):
    return lib().kh_estd(ptr(x), N, ptr(lens), ptr(inv_std), B, stream())


def efront(w, x, N, lens, inv_std, X, gn_sums, B, T):
    return lib().kh_efront(ctypes.byref(w), ptr(x), N, ptr(lens), ptr(inv_std), ptr(X), ptr(gn_sums), B, T, stream())


def egn_apply(w, X, gn_sums, per_b, total4, lens):
    return lib().kh_egn_apply(ctypes.byref(w), ptr(X), ptr(gn_sums), per_b, total4, ptr(lens), stream())


def eqkv_ln(w, QKV, Qn, Kp, Vp, k_plane, v_plane, B, T, Tp):
    return lib().kh_eqkv_ln(ctypes.byref(w), ptr(QKV), ptr(Qn), ptr(Kp), ptr(Vp), k_plane, v_plane, B, T, Tp, stream())


def softmax_rows(S, ld, n, rows_per_z, z_stride, Z, lens):
    return lib().kh_softmax_rows(ptr(S), ld, n, rows_per_z, z_stride, Z, ptr(lens), stream())


def eattn_out_grid(T, B):
    """the engine's eattn_out_kernel grid: min(T B, 4 CTAs per SM)"""
    return lib().kh_eattn_out_grid(T, B)


def eattn_out(w, O, X, T, Tp, n_frames, grid):
    return lib().kh_eattn_out(ctypes.byref(w), ptr(O), ptr(X), T, Tp, n_frames, grid, stream())


def ehead(w, HD, out, B, T, lens):
    return lib().kh_ehead(ctypes.byref(w), ptr(HD), ptr(out), B, T, ptr(lens), stream())


def einter_mask(gx, lens, B, steps):
    return lib().kh_einter_mask(ptr(gx), ptr(lens), B, steps, stream())


def eput_lens(dst, lens_host, n):
    arr = (ctypes.c_int32 * len(lens_host))(*lens_host)
    return lib().kh_eput_lens(ptr(dst), arr, n, stream())


def e_frames(n):
    return 1 + n // E_HOP


def _ln_bound64(y, g, b, chain, ye=None, dims=(-1,)):
    """LayerNorm (biased variance, eps 1e-5 inside the sqrt) of y over `dims`, and the bound on a kernel that computes it
    with fp32 two-pass statistics whose longest rounding chain is `chain` (the per-thread sums plus the reduction tree),
    rsqrtf (2 ulp = 4 u), the final (y - mu) rs g + b (3 roundings and |b|) and one more rounding for a residual add.
    ye: bounds on the inputs, carried through as in gate64 (|g| (ye + mean ye) + |g xh| mean ye) / sigma."""
    mu = y.mean(dims, keepdim=True)
    sd = torch.sqrt(((y - mu) ** 2).mean(dims, keepdim=True) + 1e-5)
    xh = (y - mu) / sd
    out = xh * g + b
    gx = (g * xh).abs()
    bound = U32 * ((0.5 * chain + 12) * gx + chain * y.abs().mean(dims, keepdim=True) / sd * g.abs() + 2 * b.abs())
    if ye is not None:
        m = ye.mean(dims, keepdim=True)
        bound = bound + (g.abs() * (ye + m) + gx * m) / sd
    return out, bound


def estd64(x, n, unbiased=True, mic0_only=False):
    """1 / std over the utterance's own 2n samples of both mics (x [2][>= n]), unbiased (tfgridnet.py:109-110), and its
    bound: the kernel sums in double, so one rounding to fp32.  Mutants: unbiased=False, mic0_only."""
    v = (x[:1, :n] if mic0_only else x[:, :n]).double().reshape(-1)
    inv = 1.0 / v.std(unbiased=unbiased)
    return inv, inv * (U32 + 1e-12)


def dft_table64(symmetric_hann=False):
    """[128][130]: window[n] (cos | -sin)(2 pi k n / 128), k = 0..64, with the periodic Hann window of torch.stft
    (symmetric_hann: the symmetric one, a mutant)"""
    n = torch.arange(E_NFFT, dtype=torch.float64)
    win = 0.5 - 0.5 * torch.cos(2 * math.pi * n / (E_NFFT - 1 if symmetric_hann else E_NFFT))
    ang = 2 * math.pi * n[:, None] * torch.arange(E_NF, dtype=torch.float64)[None, :] / E_NFFT
    return torch.cat([win[:, None] * torch.cos(ang), -win[:, None] * torch.sin(ang)], dim=1)


def efront64(x, n, T, inv, Wc, bc, edge_repeat=False, reflect_at=None, symmetric_hann=False, reim_interleaved=False,
             conv_flip_time=False):
    """the centred STFT (reflect padding about the utterance's own last sample n - 1, no edge repeat; periodic Hann) of
    x [2][>= n] * inv, channels [Re m0, Re m1, Im m0, Im m1], then Conv2d(4 -> 64, 3x3) zero-padded in T (frames outside
    [0, T_b)) and in F, for the T frames of the padded layout: rows t >= T_b are exactly zero.  Wc [64][4][3][3], bc [64].
    Returns X [T][65][64], its bound, and the GroupNorm sums (sum X, sum X^2 over the real frames) with their bounds.
    Mutants: edge_repeat (reflect with the edge sample repeated), reflect_at (reflect at another length, e.g. N),
    symmetric_hann, reim_interleaved ([Re m0, Im m0, Re m1, Im m1]), conv_flip_time."""
    Tb = e_frames(n)
    L = n if reflect_at is None else reflect_at
    s = E_HOP * torch.arange(Tb)[:, None] - E_NFFT // 2 + torch.arange(E_NFFT)[None, :]
    if edge_repeat:
        s = torch.where(s < 0, -s - 1, s)
        s = torch.where(s >= L, 2 * L - 1 - s, s)
    else:
        s = s.abs()
        s = torch.where(s >= L, 2 * (L - 1) - s, s)
    xs = x.double()[:, s] * float(inv)                                     # [2, Tb, 128]
    D = dft_table64(symmetric_hann)
    S, Sa = xs @ D, xs.abs() @ D.abs()                                     # [2, Tb, 130]
    order = [0, 2, 1, 3] if reim_interleaved else [0, 1, 2, 3]

    def regroup(v):
        u = torch.stack([v[0, :, :E_NF], v[1, :, :E_NF], v[0, :, E_NF:], v[1, :, E_NF:]])[order]     # [4, Tb, 65]
        p = torch.zeros(4, Tb + 2, E_NF + 2, dtype=torch.float64)
        p[:, 1:Tb + 1, 1:E_NF + 1] = u
        return p
    # the spectrum: 128 products (x * inv and the fp32 table each add one rounding per term)
    Up, Ua, Ue = regroup(S), regroup(Sa), regroup(Sa) * (U32 * (math.sqrt(E_NFFT) + 2))
    W = Wc.double().flip(2) if conv_flip_time else Wc.double()
    X = torch.zeros(T, E_NF, E_CH, dtype=torch.float64)
    Xa = torch.zeros_like(X)
    Xe = torch.zeros_like(X)
    X[:Tb] += bc.double()
    Xa[:Tb] += bc.double().abs()
    for i in range(3):
        for j in range(3):
            w = W[:, :, i, j]
            X[:Tb] += torch.einsum("ctf,oc->tfo", Up[:, i:i + Tb, j:j + E_NF], w)
            Xa[:Tb] += torch.einsum("ctf,oc->tfo", Ua[:, i:i + Tb, j:j + E_NF], w.abs())
            Xe[:Tb] += torch.einsum("ctf,oc->tfo", Ue[:, i:i + Tb, j:j + E_NF], w.abs())
    Xb = Xe + U32 * math.sqrt(37) * Xa
    r = X[:Tb]
    sums = torch.stack([r.sum(), (r * r).sum()])
    sums_bound = torch.stack([Xb[:Tb].sum(), (2 * r.abs() * Xb[:Tb] + Xb[:Tb] ** 2).sum()]) + 1e-12 * sums.abs()
    return dict(X=X, X_bound=Xb, sums=sums, sums_bound=sums_bound)


def egn64(X, sums, Tb, g, b, padded_count=False, unbiased=False):
    """GroupNorm(1 group) of one utterance X [T][65][64] from its sums (sum X, sum X^2 over the real frames): population
    variance over T_b 65 64 values, eps 1e-5, affine per channel; frames t >= T_b come back exactly as they are.  The
    kernel forms mean and variance in double and rounds them to fp32 once, then 4 fp32 roundings.
    Mutants: padded_count (count T 65 64), unbiased (variance over count - 1)."""
    X = X.double()
    T = X.shape[0]
    cnt = float((T if padded_count else Tb) * E_FC)
    mu = float(sums[0]) / cnt
    var = float(sums[1]) / cnt - mu * mu
    if unbiased:
        var = var * cnt / (cnt - 1)
    rs = 1.0 / math.sqrt(var + 1e-5)
    out, bound = X.clone(), torch.zeros_like(X)
    xh = (X[:Tb] - mu) * rs
    gg, bb = g.double(), b.double()
    out[:Tb] = xh * gg + bb
    bound[:Tb] = U32 * (5 * (xh * gg).abs() + abs(mu) * rs * gg.abs() + 2 * bb.abs())
    return out, bound


def eqkv_ln64(QKV, gq, bq, gk, bk, gv, bv, per_bin=False, heads_transposed=False, swap_qk_gains=False):
    """per head, the LayerNorm over (f, e) of the PReLU'd projections QKV [T][65][128] (columns Q h*8 + e | 32 + K h*8 + e
    | 64 + V h*16 + c), element f*d + e; gains / biases [4][65 d].  Returns {"Q", "K", "V"}: ([4][T][65 d], bound).
    The kernel's statistics: each lane sums 65 d / 32 values, then a 5-level warp tree.
    Mutants: per_bin (a LayerNorm over each bin's d values), heads_transposed (column e*4 + h), swap_qk_gains."""
    P = QKV.double()
    T = P.shape[0]
    if swap_qk_gains:
        (gq, bq), (gk, bk) = (gk, bk), (gq, bq)
    out = {}
    for name, d, c0, g, b in (("Q", E_QE, 0, gq, bq), ("K", E_QE, 32, gk, bk), ("V", E_VD, 64, gv, bv)):
        cols = P[:, :, c0:c0 + E_NH * d]
        y = (cols.view(T, E_NF, d, E_NH).permute(3, 0, 1, 2) if heads_transposed
             else cols.view(T, E_NF, E_NH, d).permute(2, 0, 1, 3))                    # [4, T, 65, d]
        g4, b4 = g.double().view(E_NH, 1, E_NF, d), b.double().view(E_NH, 1, E_NF, d)
        n = E_NF * d
        v, bound = _ln_bound64(y, g4, b4, n / 32 + 5, dims=(-1,) if per_bin else (-2, -1))
        out[name] = (v.reshape(E_NH, T, n), bound.reshape(E_NH, T, n))
    return out


def softmax_row_lens(Z, rows_per_z, lens, n, by_mod=False):
    """the column count of each of the Z rows_per_z rows of softmax_rows_kernel: the own frame count of utterance z / 4
    (lens None: n).  by_mod: utterance z % 4 (a mutant)."""
    z = torch.arange(Z * rows_per_z) // rows_per_z
    if lens is None:
        return torch.full_like(z, n)
    u = z % E_NH if by_mod else z // E_NH
    return torch.tensor([e_frames(int(lens[int(i)])) for i in u])


def softmax64(S, ncols, zero_pad=True):
    """softmax over the first ncols[r] columns of each row of S [rows][ld]; columns ncols[r] .. ld - 1 become exactly 0
    (zero_pad=False: left as they are, a mutant).  Bound of each weight p: its own __expf error (2 + 1.2 |s - max| ulp,
    plus the rounding of s - max) and the weighted mean of all of them (through the sum), plus the sum's rounding
    (n / 128 terms per thread and a 10-level tree) and the reciprocal and product."""
    S = S.double()
    ncols = torch.as_tensor(ncols)
    out = S.clone() if not zero_pad else torch.zeros_like(S)
    bound = torch.zeros_like(S)
    for n in ncols.unique().tolist():
        r = (ncols == n).nonzero()[:, 0]
        s = S[r, :n]
        d = s - s.max(1, keepdim=True).values
        p = torch.softmax(s, 1)
        re = U32 * (6 + 4.4 * d.abs())
        out[r, :n] = p
        bound[r, :n] = p * (re + (p * re).sum(1, keepdim=True) + U32 * (n / 128 + 14)) + 2.0 ** -126
    return out, bound


def eattn_out64(O, X, wp_t, bp, slope, gp, bpn, heads_cf=False, ignore_slope=False, ln_per_bin=False):
    """the attention output of one utterance's frames: gather heads O [T][4][1040] (feature f*16 + c) to channel h*16 + c
    of bin f, Linear 64 -> 64 (wp_t [64 in][64 out]) + bias, scalar PReLU, LayerNorm over the frame's 4160 values in
    (f*64 + c) order (gp, bpn [4160]), then the residual X [T][65][64].  Returns (X', bound).
    Mutants: heads_cf (channel c*4 + h), ignore_slope (no PReLU), ln_per_bin (LayerNorm over C per bin)."""
    T = O.shape[0]
    z = O.double().view(T, E_NH, E_NF, E_VD).permute(0, 2, 1, 3)               # [T, 65, 4, 16]
    if heads_cf:
        z = z.transpose(2, 3)
    Z = z.reshape(T, E_NF, E_CH)
    W, bpd = wp_t.double(), bp.double()
    P = Z @ W + bpd
    a = 1.0 if ignore_slope else float(slope)
    Pe = U32 * math.sqrt(65) * (Z.abs() @ W.abs() + bpd.abs()) * max(1.0, abs(a))
    P = prelu64(P, a)
    g, b = gp.double().view(E_NF, E_CH), bpn.double().view(E_NF, E_CH)
    if ln_per_bin:
        y, yb = _ln_bound64(P, g, b, 64 / 256 + 10, ye=Pe, dims=(-1,))
    else:
        y, yb = _ln_bound64(P, g, b, E_FC / 256 + 10, ye=Pe, dims=(-2, -1))
    out = X.double() + y
    return out, yb + U32 * out.abs()


def ehead64(HD, Tb, g, b, div_T=False, mean_before_ln=False):
    """LayerNorm(256) of each of the utterance's own T_b frames of HD [T][256], then their mean (tfgridnet.py:124-125),
    and its bound: the mean of the frames' LayerNorm bounds (8 values per lane, 5-level tree) plus the sum's rounding
    (T_b / 8 terms per warp, 8 warps, the division).  Mutants: div_T (the sum over T_b frames divided by the padded T),
    mean_before_ln (the LayerNorm of the mean frame)."""
    H = HD.double()
    T = H.shape[0]
    gd, bd = g.double(), b.double()
    if mean_before_ln:
        y, yb = _ln_bound64(H[:Tb].mean(0), gd, bd, 13)
        return y, yb
    y, yb = _ln_bound64(H[:Tb], gd, bd, 13)
    out = y.sum(0) / (T if div_T else Tb)
    bound = yb.sum(0) / Tb + U32 * (math.ceil(Tb / 8) + 9) * y.abs().sum(0) / Tb
    return out, bound


def einter_mask_expected(gx, lens, steps, start=3, fwd_only=False, pad=E_PAD_GATES):
    """what einter_mask_kernel leaves in gx [(b*65 + f)][steps][512] (columns dir*256 + j*4 + q, q = i, f, g, o): every
    unit's four gates of the windows s >= T_b - start of each (b, f) sequence become pad, in both directions; every other
    float is bit-unchanged.  Mutants: start = 4 or 2 (one window early / late), fwd_only, pad in another gate order."""
    out = gx.clone().view(len(lens), E_NF, steps, 2, 64, 4)
    p = torch.tensor(pad, dtype=gx.dtype)
    for b, n in enumerate(lens):
        s0 = max(0, e_frames(int(n)) - start)
        if fwd_only:
            out[b, :, s0:, 0] = p
        else:
            out[b, :, s0:] = p
    return out.view(gx.shape)


def pack_embed(sd, n_blocks=1):
    """the weights the enrollment kernels read, in the engine's packed layouts (embed_engine.cu: build_layout), as fp32:
    wc [64][36], bc, gn_g, gn_b, lnh_g, lnh_b, and per block i: wqkv_t [64][128] (columns Q h*8 + e | 32 + K h*8 + e |
    64 + V h*16 + c), bqkv, slope_qkv [128], gq / bq / gk / bk [4][520] and gv / bv [4][1040] in (f*d + e) order, wp_t
    [64 in][64 out], bp, slope_p [1], gp / bpn [4160] in (f*64 + c) order (keys "i.name")"""
    g = lambda k: sd[k].detach().float()
    out = dict(wc=g("conv.0.weight").reshape(E_CH, 36), bc=g("conv.0.bias"), gn_g=g("conv.1.weight"),
               gn_b=g("conv.1.bias"), lnh_g=g("embed_proj.1.weight"), lnh_b=g("embed_proj.1.bias"))
    for i in range(n_blocks):
        p = f"blocks.{i}."
        w = torch.zeros(E_CH, E_NQKV)
        bias, slope = torch.zeros(E_NQKV), torch.zeros(E_NQKV)
        ln = {k: torch.zeros(E_NH, E_NF * d) for k, d in (("gq", 8), ("bq", 8), ("gk", 8), ("bk", 8), ("gv", 16), ("bv", 16))}
        for h in range(E_NH):
            for nm, d, c0, gk, bk in (("Q", E_QE, h * E_QE, "gq", "bq"), ("K", E_QE, 32 + h * E_QE, "gk", "bk"),
                                      ("V", E_VD, 64 + h * E_VD, "gv", "bv")):
                m = f"{p}attn_conv_{nm}_{h}."
                w[:, c0:c0 + d] = g(m + "0.weight")[:, :, 0, 0].T
                bias[c0:c0 + d] = g(m + "0.bias")
                slope[c0:c0 + d] = g(m + "1.weight")[0]
                ln[gk][h] = g(m + "2.gamma")[0, :, 0, :].T.reshape(-1)
                ln[bk][h] = g(m + "2.beta")[0, :, 0, :].T.reshape(-1)
        out.update({f"{i}.wqkv_t": w, f"{i}.bqkv": bias, f"{i}.slope_qkv": slope})
        out.update({f"{i}.{k}": v for k, v in ln.items()})
        out[f"{i}.wp_t"] = g(p + "attn_concat_proj.0.weight")[:, :, 0, 0].T.contiguous()
        out[f"{i}.bp"] = g(p + "attn_concat_proj.0.bias")
        out[f"{i}.slope_p"] = g(p + "attn_concat_proj.1.weight").reshape(1)
        out[f"{i}.gp"] = g(p + "attn_concat_proj.2.gamma")[0, :, 0, :].T.reshape(-1).contiguous()
        out[f"{i}.bpn"] = g(p + "attn_concat_proj.2.beta")[0, :, 0, :].T.reshape(-1).contiguous()
    return out


def dft_table32(pad=float("nan")):
    """the engine's fp32 DFT table [128][132] (build_layout: periodic Hann, cos | -sin), its 2 pad columns = pad"""
    t = torch.full((E_NFFT, E_DFT_LD), pad, dtype=torch.float32)
    t[:, :2 * E_NF] = dft_table64().float()
    return t


def eattention64(X2, pk, blk=0, **mut):
    """the attention section of one utterance's T_b frames X2 [T_b][65][64] through the references (the Q|K|V projection,
    Q.K^T / sqrt(520), P.V and the GEMMs in float64): eqkv_ln64 -> softmax64 -> eattn_out64; mut goes to eattn_out64"""
    T = X2.shape[0]
    q = lambda k: pk[f"{blk}.{k}"]
    QKV = prelu64(X2.double() @ q("wqkv_t").double() + q("bqkv").double(), q("slope_qkv").double())
    r = eqkv_ln64(QKV, q("gq"), q("bq"), q("gk"), q("bk"), q("gv"), q("bv"))
    O = torch.zeros(T, E_NH, E_VDIM, dtype=torch.float64)
    for h in range(E_NH):
        S = r["Q"][0][h] @ r["K"][0][h].T / math.sqrt(E_QK)
        P, _ = softmax64(S, [T] * T)
        O[:, h] = P @ r["V"][0][h]
    return eattn_out64(O, X2, q("wp_t"), q("bp"), q("slope_p"), q("gp"), q("bpn"), **mut)[0]


# ---- the separator's CUDA-core rows GEMM (gemm.cuh) and its one-hop middle section (mid_kernel.cuh) -------------------
# The weights are in the engine's stored layout: W^T [K][N]; the inter-LSTM gates in unit-major columns j*4 + q
# (q = i, f, g, o); the Q|K|V projection's PReLU slopes by column group (Q 0-23, K 24-47, V 48-111).  Each reference
# returns, next to every value, an element-wise bound on the kernel's fp32 rounding: u = 2^-24, a sum of n terms within
# u sqrt(n) sum |terms|, input bounds carried through (a LayerNorm's through |g| / sigma, as in _ln_bound64).
ROWS_GEMM_FORMS = {0: None, 1: "tile16x64", 2: "tile64x64", 3: "tile64x128", 4: "big64", 5: "big128"}    # RowsGemmForm
MID_LAYOUT_NAMES = ("MID_PACK", "MID_RT", "MID_W1", "MID_W3A", "MID_W3B", "MID_W5", "MID_W6", "MID_SMEM", "MID_A_SMEM",
                    "MID_B_SMEM", "MID_C_SMEM", "NUM_SMS")
# (region, K, N, KS) of the five k-sliced matrices of BlockWeights::mid_pack (mid_kernel.cuh: M1 .. M6)
MID_MATRICES = (("MID_W1", 128, 64, 8), ("MID_W3A", 64, 256, 8), ("MID_W3B", 64, 256, 8), ("MID_W5", 64, 64, 4),
                ("MID_W6", 64, NQKV, 8))
SLOPE_GROUPS = (24, 48)          # first column of the K and of the V group


def rows_gemm(desc, shape=0):
    """(cudaError_t, RowsGemmForm name) of one kh_rows_gemm call"""
    form = ctypes.c_int()
    rc = lib().kh_rows_gemm(ctypes.byref(desc), shape, ctypes.byref(form), stream())
    return rc, ROWS_GEMM_FORMS[form.value]


def rows_gemm_form(M, N, K, shape=0):
    return ROWS_GEMM_FORMS[lib().kh_rows_gemm_form(M, N, K, shape)]


def mid_layout():
    """kh_mid_layout as {name: value} (MID_LAYOUT_NAMES; offsets in floats, *_SMEM in bytes)"""
    out = (ctypes.c_int64 * 16)()
    n = lib().kh_mid_layout(out)
    return dict(zip(MID_LAYOUT_NAMES, list(out)[:n]))


def mid_widx(ks, n_cols, k, n):
    """index of weight (k, n) in a k-sliced [K][N] matrix (mid_kernel.cuh: slices of ks rows padded by 4 floats)"""
    return (k // ks) * (ks * n_cols + 4) + (k % ks) * n_cols + n


def mid_pack(wl1_t, wih2_t, whh2_t, wl2_t, wqkv_t):
    """BlockWeights::mid_pack from the five W^T matrices, by the engine's own packing (kh_mid_pack; host memory)"""
    src = [t.detach().float().contiguous().cpu() for t in (wl1_t, wih2_t, whh2_t, wl2_t, wqkv_t)]
    dst = torch.full((mid_layout()["MID_PACK"],), float("nan"))
    lib().kh_mid_pack(*[t.data_ptr() for t in src], dst.data_ptr())
    return dst


def mid_unpack(packed, lay):
    """the five W^T matrices read back from a mid_pack through mid_widx"""
    out = []
    for region, K, N, ks in MID_MATRICES:
        k = torch.arange(K)[:, None]
        n = torch.arange(N)[None, :]
        out.append(packed[lay[region] + mid_widx(ks, N, k, n)])
    return out


def mid(w, Y, X, QKV, state, sstride, blk, B, active=None):
    return lib().kh_mid(ctypes.byref(w), ptr(Y), ptr(X), ptr(QKV), ptr(state), sstride, blk, B, ptr(active), stream())


def mid_a(w, Y, X, GI, B, hop_stride=0, n_hops=1):
    return lib().kh_mid_a(ctypes.byref(w), ptr(Y), ptr(X), ptr(GI), B, hop_stride, n_hops, stream())


def mid_b(w, GI, Hn, state, sstride, blk, B, hop_stride=0, n_hops=1, active=None):
    return lib().kh_mid_b(ctypes.byref(w), ptr(GI), ptr(Hn), hop_stride, n_hops, ptr(state), sstride, blk, B, ptr(active),
                          stream())


def mid_c(w, Hn, X, QKV, B, hop_stride=0, n_hops=1):
    return lib().kh_mid_c(ctypes.byref(w), ptr(Hn), ptr(X), ptr(QKV), B, hop_stride, n_hops, stream())


def lstm_cell_rows(gates, state, sstride, blk, Hout, rows, active=None):
    return lib().kh_lstm_cell_rows(ptr(gates), ptr(state), sstride, blk, ptr(Hout), rows, ptr(active), stream())


def rows_offsets(M, ld, rows_per_seq=0, seq_stride=0):
    """[M] offset (floats) of GEMM row m: m * ld, or windowed (seq = m / rows_per_seq, p = m % rows_per_seq) at
    seq * seq_stride + p * ld (gemm.cuh: a_rows_per_seq / c_rows_per_seq with c_inner <= 1)"""
    m = torch.arange(M, dtype=torch.int64)
    if rows_per_seq <= 0:
        return m * ld
    return (m // rows_per_seq) * seq_stride + (m % rows_per_seq) * ld


def _layer_norm_mut(x, g, b, unbiased=False, eps_outside=False, eps=1e-5):
    """layer_norm64 with the LayerNorm mutants: unbiased variance, eps added outside the sqrt"""
    x = x.double()
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    if unbiased:
        var = var * x.shape[-1] / (x.shape[-1] - 1)
    sd = torch.sqrt(var) + eps if eps_outside else torch.sqrt(var + eps)
    return (x - mu) / sd * g.double() + b.double()


def rows_gemm64(A, Wt, bias=None, ln=None, R=None, ln_chain=8, unbiased=False, eps_outside=False, no_transpose=False,
                drop_bias=False, drop_residual=False):
    """C = [LN(A)] W + bias [+ R] of the logical rows A [M][K] (fp32), Wt [K][N], ln = (g, b) over K = 64 channels, R
    [M][N] the residual.  ln_chain: the LayerNorm statistics' longest rounding chain (rows GEMM: 4 values per lane and a
    4-level shuffle tree = 8).  Mutants: unbiased / eps_outside (LayerNorm), no_transpose (W^T's memory read as W [N][K]),
    drop_bias, drop_residual.  Returns (C, bound)."""
    K, N = Wt.shape
    a = A.double()
    ae = torch.zeros_like(a)
    if ln is not None:
        g, b = ln[0].double(), ln[1].double()
        if unbiased or eps_outside:
            a = _layer_norm_mut(A, g, b, unbiased, eps_outside)
        else:
            a, ae = _ln_bound64(a, g, b, ln_chain)
    W = Wt.double().reshape(N, K).T if no_transpose else Wt.double()
    out = a @ W
    terms = a.abs() @ W.abs()
    if bias is not None and not drop_bias:
        out = out + bias.double()
        terms = terms + bias.double().abs()
    if R is not None and not drop_residual:
        out = out + R.double()
        terms = terms + R.double().abs()
    return out, ae @ W.abs() + U32 * (math.sqrt(K + 2) * terms + out.abs())


def _sigmoid_err(x, s):
    """__fdividef(1, 1 + __expf(-x)) (fast_sigmoid) and its ex2.approx.ftz form (lstm_cell_rows): __expf is within
    2 + 1.16 |x| ulp (CUDA C Programming Guide, intrinsic functions; the 1.16 |x| is the rounding of x log2 e), which
    moves s = 1 / (1 + e) by s (1 - s) times that relative error; 1 + e rounds once and __fdividef adds 2 ulp"""
    return s * (1 - s) * (2 + 1.16 * x.abs()) * 2.0 ** -23 + 5 * U32 * s


def _tanh_err(x, t):
    """fast_tanh = 2 fast_sigmoid(2x) - 1: twice the sigmoid's error at 2x, and the subtraction's rounding"""
    s = (t + 1) / 2
    return 2 * _sigmoid_err(2 * x, s) + U32


def cell64(G, Ge, c, ce, swap_if=False, drop_c=False):
    """one LSTM cell step from the gate pre-activations G [..][256] (column j*4 + q, q = i, f, g, o) with bounds Ge and
    the carried c [..][64] (bound ce): c' = f c + i g, h' = o tanh(c').  Mutants: swap_if (i and f exchanged), drop_c
    (c carried as 0).  Returns (h', bound, c', bound)."""
    G = G.double().view(*G.shape[:-1], 64, 4)
    Ge = Ge.double().view(*G.shape)
    c = torch.zeros_like(c.double()) if drop_c else c.double()
    qi, qf = (1, 0) if swap_if else (0, 1)
    xi, xf, xg, xo = G[..., qi], G[..., qf], G[..., 2], G[..., 3]
    ei, ef, eg, eo = Ge[..., qi], Ge[..., qf], Ge[..., 2], Ge[..., 3]
    i, f, g, o = torch.sigmoid(xi), torch.sigmoid(xf), torch.tanh(xg), torch.sigmoid(xo)
    ie = i * (1 - i) * ei + _sigmoid_err(xi, i)
    fe = f * (1 - f) * ef + _sigmoid_err(xf, f)
    ge = (1 - g * g) * eg + _tanh_err(xg, g)
    oe = o * (1 - o) * eo + _sigmoid_err(xo, o)
    c2 = f * c + i * g
    c2e = c.abs() * fe + f * ce + g.abs() * ie + i * ge + U32 * (2 * (f * c).abs() + 2 * (i * g).abs())
    t = torch.tanh(c2)
    h = o * t
    he = t.abs() * oe + o * ((1 - t * t) * c2e + _tanh_err(c2, t)) + U32 * h.abs()
    return h, he, c2, c2e


def lstm_cell64(gates, c, **mutant):
    """lstm_cell_rows_kernel of exact fp32 gates [rows][256] and c [rows][64]: (h', bound, c', bound)"""
    return cell64(gates, torch.zeros_like(gates.double()), c, torch.zeros_like(c.double()), **mutant)


def mid_a64(Y, X, p, drop_residual=False, drop_bias=False, unbiased=False, eps_outside=False):
    """X1 = X + Y W_l1 + b_l1 and GI = LN(X1) W_ih + b of rows Y [..][128], X [..][64]; p: the block's weights
    (wl1_t, bl1, ln2_g, ln2_b, wih2_t, b2, ...).  The LayerNorm's statistics: 2 values per lane, a 5-level warp tree.
    Returns (X1, bound, GI, bound)."""
    W1, b1 = p["wl1_t"].double(), p["bl1"].double()
    x = torch.zeros_like(X.double()) if drop_residual else X.double()
    X1 = x + Y.double() @ W1 + (0 if drop_bias else b1)
    X1e = U32 * (math.sqrt(130) * (X.double().abs() + Y.double().abs() @ W1.abs() + b1.abs()) + X1.abs())
    g, b = p["ln2_g"].double(), p["ln2_b"].double()
    if unbiased or eps_outside:
        xn, xne = _layer_norm_mut(X1, g, b, unbiased, eps_outside), torch.zeros_like(X1)
    else:
        xn, xne = _ln_bound64(X1, g, b, 6, ye=X1e)
    Wih, b2 = p["wih2_t"].double(), p["b2"].double()
    GI = xn @ Wih + b2
    GIe = xne @ Wih.abs() + U32 * (math.sqrt(66) * (xn.abs() @ Wih.abs() + b2.abs()) + GI.abs())
    return X1, X1e, GI, GIe


def mid_gates64(GI, GIe, h, he, p):
    """g = GI + h W_hh (the kernels' operand order: (h W_hh) + ((x W_ih) + b)) and its bound"""
    Whh = p["whh2_t"].double()
    G = GI.double() + h.double() @ Whh
    return G, GIe + he @ Whh.abs() + U32 * (math.sqrt(65) * (h.double().abs() @ Whh.abs() + GI.double().abs()) + G.abs())


def mid_c64(X1, X1e, H, He, p, drop_residual=False, drop_bias=False, slope_groups=SLOPE_GROUPS):
    """X2 = X1 + H W_l2 + b_l2 and P = PReLU(X2 W_qkv + b_qkv) with the slope of each column's group.  Mutants:
    drop_residual, drop_bias (b_l2), slope_groups (other group boundaries).  Returns (X2, bound, P, bound)."""
    W2, b2 = p["wl2_t"].double(), p["bl2"].double()
    x1 = torch.zeros_like(X1.double()) if drop_residual else X1.double()
    X2 = x1 + H.double() @ W2 + (0 if drop_bias else b2)
    X2e = X1e + He @ W2.abs() + U32 * (math.sqrt(66) * (X1.double().abs() + H.double().abs() @ W2.abs() + b2.abs()) + X2.abs())
    Wq, bq, s = p["wqkv_t"].double(), p["bqkv"].double(), p["slopes"].double()
    col = torch.arange(NQKV)
    a = torch.where(col < slope_groups[0], s[0], torch.where(col < slope_groups[1], s[1], s[2]))
    Z = X2 @ Wq + bq
    Ze = X2e @ Wq.abs() + U32 * (math.sqrt(65) * (X2.abs() @ Wq.abs() + bq.abs()) + Z.abs())
    P = prelu64(Z, a)
    return X2, X2e, P, Ze * torch.clamp(a.abs(), min=1.0) + U32 * P.abs()


def mid64(Y, X, h, c, p, swap_if=False, drop_c=False, whh_new_h=False, drop_residual=False, drop_bias=False,
          slope_groups=SLOPE_GROUPS, unbiased=False, eps_outside=False, hb=None, cb=None):
    """the one-hop middle section of rows Y [..][128], X [..][64] with the carried (h, c) [..][64]: X1 = X + Y W_l1 + b;
    the inter-LSTM step from LN(X1) and (h, c); X2 = X1 + h' W_l2 + b; P = PReLU(X2 W_qkv + b).  hb / cb: bounds of the
    carried (h, c) (None: exact).  Mutants: those of mid_a64, cell64 and mid_c64 (drop_residual / drop_bias apply to both
    Linears), whh_new_h (h W_hh taken from the new h: the state read after it was overwritten).  Returns a dict of X1, GI,
    h, c, X2, P and their bounds (key + "_b")."""
    X1, X1e, GI, GIe = mid_a64(Y, X, p, drop_residual, drop_bias, unbiased, eps_outside)
    zero = torch.zeros_like(h.double())
    hb = zero if hb is None else hb.double()
    cb = zero if cb is None else cb.double()
    G, Ge = mid_gates64(GI, GIe, h, hb, p)
    h2, h2e, c2, c2e = cell64(G, Ge, c, cb, swap_if, drop_c)
    if whh_new_h:
        G, Ge = mid_gates64(GI, GIe, h2.float(), zero, p)
        h2, h2e, c2, c2e = cell64(G, Ge, c, cb, swap_if, drop_c)
    X2, X2e, P, Pe = mid_c64(X1, X1e, h2, h2e, p, drop_residual, drop_bias, slope_groups)
    return dict(X1=X1, X1_b=X1e, GI=GI, GI_b=GIe, h=h2, h_b=h2e, c=c2, c_b=c2e, X2=X2, X2_b=X2e, P=P, P_b=Pe)


def mid_b64(GIs, h, c, p, GIe=None, no_advance=False, store_first=False):
    """mid_b_kernel over the hops of GIs [n_hops][..][256] from the carried (h, c): per hop g = GI + h W_hh, the cell,
    H'_j = h'.  GIe: the bounds of GIs (None: exact fp32 inputs).  Mutants: no_advance (every hop from the carried h),
    store_first (the state after the first hop is what is stored).  Returns (H' [n_hops][..][64], bounds, the stored
    (h, c) and their bounds)."""
    h = h.double()
    c = c.double()
    he, ce = torch.zeros_like(h), torch.zeros_like(c)
    h0 = h
    Hs, Hes, stored = [], [], None
    for j in range(GIs.shape[0]):
        gie = torch.zeros_like(GIs[j].double()) if GIe is None else GIe[j]
        hin, hine = (h0, torch.zeros_like(h0)) if no_advance else (h, he)
        G, Ge = mid_gates64(GIs[j], gie, hin, hine, p)
        h, he, c, ce = cell64(G, Ge, c, ce)
        Hs.append(h)
        Hes.append(he)
        if j == 0 and store_first:
            stored = (h, he, c, ce)
    if stored is None:
        stored = (h, he, c, ce)
    return torch.stack(Hs), torch.stack(Hes), stored


# ---- the fused one-hop tail of a block (hop_kernels.cuh: tail_kernel; tfgridnet_causal.py:518-588, :250, :505-512) ---
# tail_kernel runs, for one frame of each stream, the middle section (mid64), the Q/K/V LayerNorms, the 50-frame
# attention over the K/V ring, the output projection with its LayerNorm(6208), the residual, the speaker gate and the next
# block's input projection.  One 16-CTA cluster per stream: CTA p < 13 owns bins 8p .. 8p + 7 (the last tile: bin 96
# alone) and combines the LayerNorm statistics of all tiles from their (mean, M2); CTA r attends with head r / 4 over
# window rows TAIL_PART_ROWS[r % 4] .. TAIL_PART_ROWS[r % 4 + 1] - 1 (row j = frame pos - 49 + j; the last part's last
# row is the one this launch writes), and the tile CTAs merge each head's four partials by their maxima.
TAIL_CL, TAIL_TILES = 16, 13
TAIL_PART_ROWS = (0, 13, 26, 38, 50)
# the longest rounding chains of the kernel's LayerNorm statistics: phase Q sums 8 values per lane over a 4-level
# shuffle tree and combines 13 tiles one after the other; phase O sums 2 values per thread over a block tree (5 + 3
# levels) and 13 tiles over a 5-level warp tree
TAIL_Q_CHAIN, TAIL_O_CHAIN = 32, 24
# absolute error of a normalised Q/K/V value from everything before the statistics (the 64-term projection of X2, whose
# rows of low X1 spread carry the LayerNorm(64)'s amplified rounding, over the group's spread ~0.5), and of an output
# value from the attention and the projection (|score| ~ 1 or ~80, 50-row sums, a 64-term projection over the spread of
# the LayerNorm(6208)'s input)
TAIL_QKV_TOL, TAIL_X_TOL = 5e-5, 2e-4


def tail_clusters():
    """how many tail_kernel clusters the device holds at once (0: it cannot be scheduled)"""
    return lib().kh_tail_clusters()


def tail(w, Y, X, GX, state, sstride, blk, B, apply_gate, frame_k=0, active=None):
    return lib().kh_tail(ctypes.byref(w), ptr(Y), ptr(X), ptr(GX), ptr(state), sstride, blk, B, apply_gate, frame_k,
                         ptr(active), stream())


def tail_slots(w, Y, X, GX, state, sstride, slots, batch, hops, blk, B, apply_gate):
    return lib().kh_tail_slots(ctypes.byref(w), ptr(Y), ptr(X), ptr(GX), ptr(state), sstride, ptr(slots), batch, ptr(hops),
                               blk, B, apply_gate, stream())


def chan_ln64(y, g, b, d, tiles="exact"):
    """LayerNorm (biased variance, eps 1e-5 inside the sqrt) over y [97 * d] (element f*d + e), with the statistics
    combined from the 13 row tiles' (mean, M2) as tail_kernel combines them (Chan): mean = sum n_p m_p / N, M2 = sum
    (M2_p + n_p (m_p - mean)^2).  tiles="exact" equals layer_norm64.  Mutants: "equal" (every tile weighted as 8 rows,
    also the 1-row last tile), "no_between" (M2 without the between-tile term), "per_tile" (each tile normalised by its
    own statistics)."""
    y = y.double()
    t = y.view(NF, d)
    parts = [t[p * 8:(p + 1) * 8].reshape(-1) for p in range(TAIL_TILES)]
    if tiles == "per_tile":
        out = torch.cat([(q - q.mean()) / torch.sqrt(((q - q.mean()) ** 2).mean() + 1e-5) for q in parts])
        return out * g.double() + b.double()
    n = [float(q.numel()) for q in parts]
    wts = [8.0 * d] * len(parts) if tiles == "equal" else n
    N = float(NF * d)
    m = [q.mean() for q in parts]
    m2 = [((q - mq) ** 2).sum() for q, mq in zip(parts, m)]
    mean = sum(wp * mp for wp, mp in zip(wts, m)) / N
    M2 = sum(m2) if tiles == "no_between" else sum(a + wp * (mp - mean) ** 2 for a, wp, mp in zip(m2, wts, m))
    return (y - mean) / torch.sqrt(M2 / N + 1e-5) * g.double() + b.double()


def tail64(Y, X, h, c, p, hist_k, hist_v, gate=None, nxt=None, hist_tol=0.0, hb=None, cb=None, stale=None, shift=False,
           no_rescale=False, qkv_stats="exact", ln_per_tile=False, heads_transposed=False, gate_first=False, drop_gate=False,
           ih_from_x2=False, **mid_mutant):
    """tail_kernel for one stream at clock pos, in float64, with a bound on each output's fp32 error.
    Y [97][128] (the intra BiLSTM's output), X [97][64] (the block input), (h, c) [97][64] the carried inter-LSTM state
    (bounds hb / cb); p: the block weights (mid64's, lnq_g .. lnv_b of >= 582 / 1552 values, wp_t, bp, lnp_g, lnp_b);
    hist_k [50][4][>= 582] and hist_v [50][4][1552]: the K / V rows of frames pos - 50 .. pos - 1 (zero rows before the
    stream start; row 0 is read only by the shift mutant), exact up to hist_tol.  gate [97][64]: the speaker gate of the
    block output (None: no gate); nxt: the next block's (ln_g, ln_b, wih_t, bias) (None: no phase G).

    Bounds.  (h, c): mid64's element-wise bounds.  Q/K/V, per (Q/K/V, head) group: TAIL_QKV_TOL |g|max, plus the
    statistics' rounding chain TAIL_Q_CHAIN u |mean| / sigma |g|max (what a group of mean >> spread costs) and P's own
    rounding 4 u |P|max / sigma |g|max.  X: TAIL_X_TOL, twice the largest Q/K/V group bound and the window rows' hist_tol
    (a K/V or q error moves a score and so Z by about as much), and the LayerNorm(6208)'s chain TAIL_O_CHAIN u |mean| /
    sigma |g|max, times max(1, |gate|).  GX: ih64's bound, plus X's bound carried through the LayerNorm(64) and |W_ih|.

    Mutants: those of mid64 (keyword arguments), stale = (k [4][>= 582], v [4][1552]) the newest row read before this hop
    wrote it (the slot's old content), shift (the window one frame earlier: pos - 50 .. pos - 1), no_rescale (each part's
    partial taken with its own max, merged without exp(m_p - max)), qkv_stats = "equal" / "no_between" (chan_ln64),
    ln_per_tile (LayerNorm(6208) per row tile), heads_transposed (projection column c0 + e*4 + h), gate_first (X2 gate +
    LN), drop_gate, ih_from_x2 (phase G applied to X2).

    Returns a dict of X, K [4][582], V [4][1552], Q [4][582], h, c, X2, P, Z, GX (with nxt) and the bounds of X, K, V, Q,
    h, c and GX (key + "_b", the shape of the value)."""
    m = mid64(Y, X, h, c, p, hb=hb, cb=cb, **mid_mutant)
    P = m["P"]
    # phase Q: head split and LayerNorm over (F, E) per (Q/K/V, head)
    qkv, qkv_b = [], []
    for d, c0, key in ((QE, 0, "lnq"), (QE, 24, "lnk"), (VD, 48, "lnv")):
        n = NF * d
        g, b = p[key + "_g"][:n].double(), p[key + "_b"][:n].double()
        cols = P[:, c0:c0 + NHEAD * d]
        if heads_transposed:
            y = cols.reshape(NF, d, NHEAD).permute(2, 0, 1).reshape(NHEAD, n)
        else:
            y = cols.reshape(NF, NHEAD, d).permute(1, 0, 2).reshape(NHEAD, n)
        qkv.append(torch.stack([chan_ln64(y[hh], g, b, d, qkv_stats) for hh in range(NHEAD)]))
        mu, sd = y.mean(-1, keepdim=True), y.std(-1, unbiased=False, keepdim=True)
        tol = g.abs().max() * (TAIL_QKV_TOL + U32 * (TAIL_Q_CHAIN * mu.abs() + 4 * y.abs().max(-1, keepdim=True)[0]) / sd)
        qkv_b.append(tol.expand(NHEAD, n))
    (q, k, v), (qb, kb, vb) = qkv, qkv_b
    # phase A: the window of frames pos - 49 .. pos (shift: pos - 50 .. pos - 1)
    hk, hv = hist_k[..., :QK_DIM].double(), hist_v.double()
    k_new, v_new = (k, v) if stale is None else (stale[0][..., :QK_DIM].double(), stale[1].double())
    Kw, Vw = (hk, hv) if shift else (torch.cat([hk[1:], k_new[None]]), torch.cat([hv[1:], v_new[None]]))
    o = []
    for hh in range(NHEAD):
        s = Kw[:, hh] @ q[hh] / math.sqrt(QK_DIM)                         # [50]
        if no_rescale:
            e = torch.cat([torch.exp(s[a:z] - s[a:z].max()) for a, z in zip(TAIL_PART_ROWS[:-1], TAIL_PART_ROWS[1:])])
        else:
            e = torch.exp(s - s.max())
        o.append(e / e.sum() @ Vw[:, hh])
    Z = merge_heads64(torch.stack(o)[None])[0]
    # phase O: Linear + PReLU, LayerNorm(6208), residual, gate
    Pp = prelu64(Z @ p["wp_t"].double() + p["bp"].double(), float(p["slopes"][3]))
    lg, lb = p["lnp_g"].double(), p["lnp_b"].double()
    y = chan_ln64(Pp.reshape(FC), lg, lb, CH, "per_tile" if ln_per_tile else "exact").view(NF, CH)
    X2 = m["X2"]
    res = X2 + y
    xtol = TAIL_X_TOL + 2 * max(float(t.max()) for t in qkv_b) + 2 * hist_tol + \
        TAIL_O_CHAIN * U32 * float(Pp.mean().abs() / Pp.std(unbiased=False) * lg.abs().max())
    if gate is None or drop_gate:
        Xo = res
    else:
        gt = gate.double()
        Xo = X2 * gt + y if gate_first else res * gt
        xtol *= max(1.0, float(gt.abs().max()))
    Xb = torch.full_like(Xo, xtol)
    out = dict(X=Xo, X_b=Xb, K=k, K_b=kb, V=v, V_b=vb, Q=q, Q_b=qb, h=m["h"], h_b=m["h_b"], c=m["c"], c_b=m["c_b"], X2=X2,
               P=P, Z=Z)
    if nxt is not None:
        ng, nb, wih_t, bias = nxt
        src = X2 if ih_from_x2 else Xo
        GX, GXb = ih64(src, ng, nb, wih_t, bias)
        sd = src.std(-1, unbiased=False, keepdim=True)
        xh = (src - src.mean(-1, keepdim=True)) / sd
        carried = ((ng.double().abs() * 2 * xtol + (ng.double() * xh).abs() * xtol) / sd) @ wih_t.double().abs()
        out.update(GX=GX, GX_b=GXb + carried)
    return out


# tail64's mutants that need no data of their own (stale=(k, v) needs the slot's old rows), by name
TAIL_MUTANTS = {"shift": dict(shift=True), "no_rescale": dict(no_rescale=True), "qkv_equal_weights": dict(qkv_stats="equal"),
                "qkv_no_between": dict(qkv_stats="no_between"), "ln_per_tile": dict(ln_per_tile=True),
                "heads_transposed": dict(heads_transposed=True), "gate_first": dict(gate_first=True),
                "drop_gate": dict(drop_gate=True), "ih_from_x2": dict(ih_from_x2=True), "eps_outside": dict(eps_outside=True),
                "swap_if": dict(swap_if=True), "drop_c": dict(drop_c=True)}


def tail_chain64(Ys, Xs, h, c, p, hist_k, hist_v, gates=None, nxt=None, **mutant):
    """len(Ys) consecutive hops of tail64 on one stream: hop j runs at clock pos + j on Ys[j], Xs[j] and the (h, c) hop
    j - 1 left, and its window holds the K/V rows hops 0 .. j - 1 wrote (exact up to their bounds).  hist_k / hist_v: the
    rows of frames pos - 50 .. pos - 1.  Returns the list of tail64's outputs."""
    K, V = hist_k[..., :QK_DIM].double(), hist_v.double()
    hb = cb = None
    tol = 0.0
    outs = []
    for j in range(len(Ys)):
        r = tail64(Ys[j], Xs[j], h, c, p, K[j:j + ATT], V[j:j + ATT], None if gates is None else gates[j], nxt, tol, hb, cb,
                   **mutant)
        outs.append(r)
        K, V = torch.cat([K, r["K"][None]]), torch.cat([V, r["V"][None]])
        tol = max(tol, float(r["K_b"].max()), float(r["V_b"].max()))
        h, c, hb, cb = r["h"], r["c"], r["h_b"], r["c_b"]
    return outs


# ---- the several-target kernels (targets_kernels.cuh) and the slot-list helpers (sep_kernels.cuh) --------------------
# target_lists_kernel builds, at the start of a call over a state's listeners, which record each target row uses, the
# frames it advances, the listener that owns it, each listener's lead record and the clamped row offsets; spk_gate_kernel
# and gate_fanout_kernel give every target row its speaker-gate memo and its gated copy of block 0's output.  The slot-list
# helpers copy the listed records' carried inter-LSTM (h, c) to and from the workspace, and mask the frames a ragged row
# does not advance.  Every reference here is exact (integer lists, copies, one fp32 multiply per element).
INT_MAX = 2 ** 31 - 1
TARGET_LISTS_MUTANTS = ("no_carry", "no_clamp", "owner_off_by_one", "lead_unvalidated")
FANOUT_MUTANTS = ("owner_mod", "gate_unowned")


def records_map(stride, slots, batch, hops=None, frames=1):
    """a Records map over device int32 tensors slots [rows] and hops [rows] (or None)"""
    return Records(stride, ptr(slots), batch, ptr(hops), frames)


def _byref(s):
    return None if s is None else ctypes.byref(s)


def target_lists(records, offsets, groups, hops, n, K, rows, batch, lists):
    return lib().kh_target_lists(ptr(records), ptr(offsets), ptr(groups), ptr(hops), n, K, rows, batch, ptr(lists), stream())


def spk_gate(w, emb, spk_pre, state, sstride, recs, rows):
    """recs None: the dense map (row r = record r, sstride floats apart)"""
    return lib().kh_spk_gate(ctypes.byref(w), ptr(emb), ptr(spk_pre), ptr(state), sstride, _byref(recs), rows, stream())


def gate_fanout(X0, X, state, sstride, recs, owner, n_targets, T, apply_gate, rows):
    """recs and owner None: the dense map, row r of mixture r / n_targets"""
    return lib().kh_gate_fanout(ptr(X0), ptr(X), ptr(state), sstride, _byref(recs), ptr(owner), n_targets, T, apply_gate, rows,
                                stream())


def gather_h(state, recs, b0, n_blocks, B, Hg, Cg):
    return lib().kh_gather_h(ptr(state), ctypes.byref(recs), b0, n_blocks, B, ptr(Hg), ptr(Cg), stream())


def scatter_hc(state, recs, b0, n_blocks, B, Hg, Cg):
    return lib().kh_scatter_hc(ptr(state), ctypes.byref(recs), b0, n_blocks, B, ptr(Hg), ptr(Cg), stream())


def inter_gate_mask(gx, recs, B):
    return lib().kh_inter_gate_mask(ptr(gx), ctypes.byref(recs), B, stream())


def inter_h_last(Y, Hg, recs, B):
    return lib().kh_inter_h_last(ptr(Y), ptr(Hg), ctypes.byref(recs), B, stream())


def row_frames(hops, b, T):
    """the frames row b advances (sep_kernels.cuh row_frames): all T without hops, hops[b] if it lies in [0, T], else 0"""
    if hops is None:
        return T
    h = int(hops[b])
    return h if 0 <= h <= T else 0


def target_lists_ref(records, offsets, groups, hops, n, K, rows, batch, mutant=None):
    """target_lists_kernel of int lists: records + offsets (a rows call) or groups (K rows per group).  Returns rec, owner,
    lead, rec_hops (None without hops) and start (None without offsets).  Mutants (TARGET_LISTS_MUTANTS): no_carry (the
    running maximum restarts at every 1024-entry pass), no_clamp (offsets not clamped to [0, rows]),
    owner_off_by_one (the owner search counts start < r instead of <= r), lead_unvalidated (a listener whose lead record is
    invalid still stores through its other rows)."""
    def listed(i, r, first):
        if records is None:
            g = groups[i]
            return g * K + (r - first) if 0 <= g < batch // K else -1
        s = records[r] if 0 <= r < rows else -1              # (only the no_clamp mutant reads outside the list)
        return s if 0 <= s < batch else -1
    start = None
    if offsets is not None:
        start, run = [], (-math.inf if mutant == "no_clamp" else 0)
        for i in range(n + 1):
            if mutant == "no_carry" and i % 1024 == 0:
                run = 0
            v = offsets[i] if mutant == "no_clamp" else min(max(offsets[i], 0), rows)
            run = max(run, v)
            start.append(run)
    first = (lambda i: start[i]) if start is not None else (lambda i: i * K)
    lead = [listed(i, first(i), first(i)) if first(i) < first(i + 1) else -1 for i in range(n)]
    rec, owner = [], []
    for r in range(rows):
        if start is not None:                                 # the kernel's binary search over start[0 .. n]
            lo, hi = 0, n + 1
            while lo < hi:
                mid = (lo + hi) >> 1
                if (start[mid] < r) if mutant == "owner_off_by_one" else (start[mid] <= r):
                    lo = mid + 1
                else:
                    hi = mid
            i = lo - 1 if lo - 1 < n else -1
        else:
            i = r // K if r // K < n else -1
        owner.append(i)
        ok = i >= 0 and (mutant == "lead_unvalidated" or lead[i] >= 0)
        rec.append(listed(i, r, first(i)) if ok else -1)
    rec_hops = None if hops is None else [hops[i] if i >= 0 else 0 for i in owner]
    return dict(rec=rec, owner=owner, lead=lead, rec_hops=rec_hops, start=start)


def _partition(g, n, used):
    """n + 1 non-decreasing offsets from 0 to `used`, with empty listeners"""
    cuts = sorted(g.randrange(used + 1) for _ in range(n - 1))
    off = [0] + cuts + [used]
    for j in range(3, n, 7):                                  # every 7th listener from the 4th on empty
        off[j + 1] = off[j]
    return off


def target_lists_cases(T=3):
    """the target_lists_kernel problems the GPU test runs (and the CPU test shows every mutant differs on): name, the
    lists, n, K, rows, batch, and `catches`, the mutants that must differ from the reference on the case"""
    import random
    bad_records = (-1, None, INT_MAX, -INT_MAX)              # None: batch
    bad_hops = (-1, 0, T, T + 1, INT_MAX, -INT_MAX)
    cases = []

    def rows_case(name, n, rows, spare, seed, hops=True, edits=(), invalid_lead=False, catches=()):
        g = random.Random(seed)
        batch = rows + 7
        recs = g.sample(range(batch), rows)
        for j in range(5, rows, 37):                          # bad records: -1, batch, +-(2^31 - 1)
            b = bad_records[(j // 37) % 4]
            recs[j] = batch if b is None else b
        off = _partition(g, n, rows - spare)
        for kind, j in edits:
            if kind == "neg":
                off[j] = -5 - j
            elif kind == "above":
                off[j] = rows + 100
            elif kind == "dec":                              # below its predecessor (and below the running maximum)
                off[j] = max(off[j - 1] - 3, 0)
        if invalid_lead:                                      # the first listener of >= 2 valid rows: its lead invalid
            for i in range(n):
                a, z = off[i], off[i + 1]
                if 0 <= a and z - a >= 2 and z <= rows and off[i] == max(off[:i + 1]) and all(
                        0 <= recs[r] < batch for r in range(a + 1, z)):
                    recs[a] = -1
                    break
        hp = [g.choice(bad_hops) if g.random() < 0.3 else g.randrange(T + 1) for _ in range(n)] if hops else None
        cases.append(dict(name=name, records=recs, offsets=off, groups=None, hops=hp, n=n, K=0, rows=rows, batch=batch,
                          catches=set(catches) | {"owner_off_by_one"}))

    rows_case("rows_n1", 1, 1, 0, 1)
    rows_case("rows_n1_spare", 1, 8, 3, 2, invalid_lead=True, catches=("lead_unvalidated",))
    rows_case("rows_n31", 31, 100, 6, 3, invalid_lead=True, catches=("lead_unvalidated",))
    rows_case("rows_n31_bad", 31, 64, 0, 4, hops=False, edits=(("neg", 0), ("dec", 9), ("neg", 15), ("above", 29)),
              catches=("no_clamp",))
    rows_case("rows_n1023", 1023, 2048, 17, 5, edits=(("dec", 500), ("neg", 0)), invalid_lead=True,
              catches=("no_clamp", "lead_unvalidated"))
    rows_case("rows_n1024", 1024, 3000, 40, 6, hops=False, edits=(("dec", 1024),), catches=("no_carry",))
    rows_case("rows_n1025", 1025, 2100, 0, 7, edits=(("dec", 1024), ("dec", 1025)), catches=("no_carry",))
    rows_case("rows_n2500", 2500, 4096, 100, 8, edits=(("neg", 0), ("dec", 1024), ("dec", 2048), ("above", 2490)),
              invalid_lead=True, catches=("no_carry", "no_clamp", "lead_unvalidated"))

    def groups_case(name, n, K, n_groups, seed, hops=True):
        g = random.Random(seed)
        batch = n_groups * K                                  # the engine guarantees batch % K == 0
        grp = [g.randrange(n_groups) for _ in range(n)]
        for j in range(1, n, 5):                              # groups outside [0, batch / K)
            grp[j] = (-1, n_groups, INT_MAX, -INT_MAX)[(j // 5) % 4]
        hp = [g.choice(bad_hops) if g.random() < 0.3 else g.randrange(T + 1) for _ in range(n)] if hops else None
        cases.append(dict(name=name, records=None, offsets=None, groups=grp, hops=hp, n=n, K=K, rows=n * K, batch=batch,
                          catches=set()))

    groups_case("groups_n1_K2", 1, 2, 2, 11)
    groups_case("groups_n31_K3", 31, 3, 10, 12)
    groups_case("groups_n1500_K2", 1500, 2, 1500, 13, hops=False)
    return cases


def gate_fanout_ref(X0, gates, owner, K, apply_gate, mutant=None):
    """gate_fanout_kernel: X0 [mixtures][T][97][64] and gates [rows][97][64] (the gate of each target row's record) ->
    X [rows][T][97][64], row r = X0[i] (times the gate if apply_gate and i >= 0) with i = owner[r] (owner None: r / K),
    mixture 0 for i = -1; fp32 products, as the kernel's (exact).  Mutants (FANOUT_MUTANTS): owner_mod (owner r % K),
    gate_unowned (a row without owner gated too)."""
    rows = gates.shape[0]
    out = torch.empty((rows,) + tuple(X0.shape[1:]), dtype=torch.float32)
    for r in range(rows):
        i = (r % K if mutant == "owner_mod" else r // K) if owner is None else int(owner[r])
        v = X0[max(i, 0)].float()
        out[r] = v * gates[r].float()[None] if apply_gate and (i >= 0 or mutant == "gate_unowned") else v
    return out


# ---- binaural renderer (csrc/render.cu) and evaluation metrics (csrc/eval_metrics.cu) --------------------------------
U32 = 2.0 ** -24                    # unit roundoff of fp32
U64 = 2.0 ** -53                    # unit roundoff of float64
F32_EPS = 1.1920928955078125e-07    # torch.finfo(torch.float32).eps, torchmetrics' SI-SNR epsilon
FIR_MUTANTS = ("drop_chunk_tap", "tile_shift", "left_both", "src_se")
MIX_MUTANTS = ("peak_ear0", "noise_unnormalised")
METRICS_MUTANTS = ("no_centre", "one_pass", "f64_eps", "first_ear", "si_i_sign", "clamp_product")


def fir64(src, rir, exact=False, mutant=None):
    """fir_kernel: events [B, S, 2, N] = convolve(src[b, s], rir[b, s, ear])[:N] from src [B, S, N] and rir [B, S, 2, L],
    in float64 (fftconvolve).  exact: data whose products lie on the 2^-8 grid (integers, or halves times quarters),
    rounded to the nearest multiple of 2^-8 (+0.0, never -0.0), which is exact while every sum stays far below 2^45.  Mutants (FIR_MUTANTS): drop_chunk_tap (tap k of a 256-tap chunk with
    k % 256 == 255 left out), tile_shift (every tile's source window one sample early: y[o] = F[o - 1]), left_both (both
    ears with the left-ear response), src_se (event (s, ear) reads source row 2 s + ear of the flattened [B * S] sources,
    NaN past the last)."""
    from scipy.signal import fftconvolve
    src, rir = np.asarray(src, np.float64), np.asarray(rir, np.float64).copy()
    B, S, N = src.shape
    x = np.broadcast_to(src[:, :, None, :], (B, S, 2, N))
    if mutant == "src_se":
        flat = np.concatenate([src.reshape(B * S, N), np.full((2 * S, N), np.nan)])
        x = flat[np.arange(B)[:, None, None] * S + 2 * np.arange(S)[None, :, None] + np.arange(2)[None, None, :]]
    if mutant == "drop_chunk_tap":
        rir[..., 255::256] = 0.0
    if mutant == "left_both":
        rir[:, :, 1] = rir[:, :, 0]
    y = fftconvolve(x, rir, axes=-1)[..., :N]
    if exact:
        y = np.rint(y * 256.0) / 256.0 + 0.0
    if mutant == "tile_shift":
        y = np.concatenate([np.zeros_like(y[..., :1]), y[..., :-1]], axis=-1)
    return y


def fir_bound64(src, rir):
    """per-sample bound on one fp32 running sum of the L products: (L + 1) 2^-24 sum_k |h_k| |x_(o-k)|"""
    return (rir.shape[-1] + 1) * U32 * fir64(np.abs(src), np.abs(rir))


def mix64(ev, noise=None, scale=None, fp32=False, mutant=None):
    """mix_peak_kernel + mix_norm_kernel: (events [B, S, 2, N], mixture [B, 2, N], norm [B]) from the un-normalised events
    ev [B, S, 2, N], noise [B, 2, N] or None and scale [B] or None (= 1).
    fp32: the kernels' fp32 model -- the peak of |v| with v = fl(sc noise) (0 without noise) plus each event in order,
    nf = max(peak, 1), events fl32(e / nf), the mixture fl32(fl32(sc / nf) noise) plus each normalised event in order;
    otherwise the same in float64 (the reference's arithmetic).  Mutants (MIX_MUTANTS): peak_ear0 (the peak over ear 0
    only), noise_unnormalised (the mixture's noise not divided by nf)."""
    dt = np.float32 if fp32 else np.float64
    ev = np.asarray(ev).astype(dt)
    B, S, _, N = ev.shape
    sc = np.ones(B, dt) if scale is None else np.asarray(scale).astype(dt)
    nz = None if noise is None else np.asarray(noise).astype(dt)
    v = np.zeros((B, 2, N), dt) if nz is None else sc[:, None, None] * nz
    for s in range(S):
        v = v + ev[:, s]
    peak = np.abs(v[:, :1] if mutant == "peak_ear0" else v).reshape(B, -1).max(1)
    nf = np.maximum(peak, dt(1))
    e = ev / nf[:, None, None, None]
    m = np.zeros((B, 2, N), dt) if nz is None else (sc if mutant == "noise_unnormalised" else sc / nf)[:, None, None] * nz
    for s in range(S):
        m = m + e[:, s]
    return e, m, nf


def mix_bound64(e, noise, scale, nf):
    """per-sample bound on the kernel's fp32 mixture against sc noise / nf + sum_s e_s in float64 (e, nf: the kernel's
    own events and norm): one rounding for sc / nf, one for the product (none if fused with the first add), S for the
    adds: (S + 3) 2^-24 (|sc noise| / nf + sum |e_s|), the extra unit covering gamma_(S+2)'s slack"""
    S = e.shape[1]
    a = np.abs(np.asarray(e, np.float64)).sum(1)
    if noise is not None:
        sc = np.ones(len(nf)) if scale is None else np.asarray(scale, np.float64)
        a = a + np.abs(sc[:, None, None] * np.asarray(noise, np.float64)) / np.asarray(nf, np.float64)[:, None, None]
    return (S + 3) * U32 * a


def render_int_inputs(B, S, N, L, seed, noise=False):
    """integer-valued sources and responses (|x|, |h| <= 8 up to L = 4097, <= 4 beyond): every partial sum of the FIR and
    of the peak is an integer below 2^24, so the fp32 kernels are exact in any order.  noise: integer noise in [-8, 8]
    and power-of-two scales 2^-3 .. 2^2 (sc noise then stays on a 2^-3 grid: the peak's sums are exact too)."""
    rng = np.random.default_rng(seed)
    a = 8 if L <= 4097 else 4
    src = rng.integers(-a, a + 1, (B, S, N)).astype(np.float32)
    rir = rng.integers(-a, a + 1, (B, S, 2, L)).astype(np.float32)
    if not noise:
        return src, rir, None, None
    return src, rir, rng.integers(-8, 9, (B, 2, N)).astype(np.float32), (2.0 ** rng.integers(-3, 3, B)).astype(np.float32)


# (B, S, N, L, noise, mutants that must miss the exact comparison).  L on and around the 256-tap chunk edges, N on and
# around the 1024-sample tiles, below 4 and past 132 * 256 / 2 = 16896 (the mixing kernels' grid-stride loop), L > N.
RENDER_EXACT_CASES = (
    (1, 1, 1, 1, False, ("left_both",)),
    (2, 1, 3, 2, False, FIR_MUTANTS[1:]),
    (3, 4, 4, 255, False, FIR_MUTANTS[1:]),
    (2, 4, 5, 256, False, FIR_MUTANTS[1:]),
    (1, 1, 1023, 257, False, FIR_MUTANTS[:3]),
    (2, 2, 1024, 511, False, FIR_MUTANTS),
    (1, 4, 1025, 512, False, FIR_MUTANTS),
    (2, 1, 16896, 513, False, FIR_MUTANTS),
    (1, 2, 16897, 4096, False, FIR_MUTANTS),
    (1, 1, 80000, 4097, False, FIR_MUTANTS[:3]),
    (1, 1, 80000, 16384, False, FIR_MUTANTS[:3]),
    (300, 1, 1025, 257, False, FIR_MUTANTS),
    (7, 4, 3, 4096, False, FIR_MUTANTS[1:]),
    (2, 4, 1000, 16384, False, FIR_MUTANTS),
    (3, 4, 1025, 257, True, FIR_MUTANTS + ("noise_unnormalised",)),
    (2, 2, 17000, 300, True, FIR_MUTANTS + ("noise_unnormalised",)),
    (1, 1, 3, 5, True, ("left_both", "tile_shift", "noise_unnormalised")),
)


def render_peak_inputs(N=20000):
    """Four items of two events, a three-tap response, no noise: item 0's mixture peaks at exactly 1.0 (events unchanged),
    item 1's at -64 on ear 0's sample 0, item 2's stays below 1 (events unchanged), item 3's -- the last item's -- at 64
    on ear 1's last sample.  Every other |mixture| sample is at most 8."""
    rng = np.random.default_rng(11)
    src = rng.integers(-1, 2, (4, 2, N)).astype(np.float32)
    rir = rng.integers(-1, 2, (4, 2, 2, 3)).astype(np.float32)
    src[0], rir[0] = 0.0, 0.0
    src[0, 0, 5], rir[0, 0, 1, 0] = 1.0, 1.0
    src[1, 1, 0], rir[1, 1, 0, 0] = -8.0, 8.0
    src[2, 1] = 0.0
    src[2, 0] *= 0.5
    rir[2, 0] = (0.25, -0.25, 0.25)
    src[3, 0, -1], rir[3, 0, 1] = 8.0, (8.0, 0.0, 0.0)
    rir[3, 1, 1] = 0.0
    return src, rir


def si_snr64(p, t, mutant=None):
    """SI-SNR in dB over the last axis, centred and in float64, as oracle/restate.py::si_sdr (torchmetrics).  Mutants
    (METRICS_MUTANTS): no_centre, one_pass (raw sums: pt = spt - sp st / n, ..., noise = alpha^2 tt - 2 alpha pt + pp),
    f64_eps (float64's epsilon for float32's)."""
    p, t = np.asarray(p, np.float64), np.asarray(t, np.float64)
    eps = np.finfo(np.float64).eps if mutant == "f64_eps" else F32_EPS
    if mutant == "one_pass":
        n = p.shape[-1]
        sp, st = p.sum(-1), t.sum(-1)
        pt, tt, pp = (p * t).sum(-1) - sp * st / n, (t * t).sum(-1) - st * st / n, (p * p).sum(-1) - sp * sp / n
        alpha = (pt + eps) / (tt + eps)
        sig = alpha * alpha * tt
        return 10 * np.log10((sig + eps) / (np.maximum(sig - 2 * alpha * pt + pp, 0.0) + eps))
    if mutant != "no_centre":
        p, t = p - p.mean(-1, keepdims=True), t - t.mean(-1, keepdims=True)
    alpha = ((p * t).sum(-1, keepdims=True) + eps) / ((t * t).sum(-1, keepdims=True) + eps)
    ts = alpha * t
    r = ts - p
    return 10 * np.log10(((ts * ts).sum(-1) + eps) / ((r * r).sum(-1) + eps))


def si_snr_err64(p, t):
    """bound on the double-precision error, in dB, of SI-SNR computed in the centred order (means, centred sums and alpha,
    residual energy summed directly), from the centred signals alone, so it does not grow with a DC offset: the energies'
    relative errors stay below 4 (n + 2) u64 (1 + sqrt(sig / noise)) each (the sums' n u64, the residual's cancellation
    u64 (|alpha t~| + |p~|) per sample, through Cauchy-Schwarz), and 10 log10 turns a relative error r into 10 r / ln 10 dB"""
    p, t = np.asarray(p, np.float64), np.asarray(t, np.float64)
    n = p.shape[-1]
    p, t = p - p.mean(-1, keepdims=True), t - t.mean(-1, keepdims=True)
    alpha = ((p * t).sum(-1, keepdims=True) + F32_EPS) / ((t * t).sum(-1, keepdims=True) + F32_EPS)
    sig, noise = ((alpha * t) ** 2).sum(-1) + F32_EPS, ((alpha * t - p) ** 2).sum(-1) + F32_EPS
    return 10 / math.log(10) * 8 * (n + 2) * U64 * (1 + np.sqrt(sig / noise))


def cos64(x, y, mutant=None):
    """F.cosine_similarity over the last axis in float64: <x, y> / (max(|x|, 1e-8) max(|y|, 1e-8)).  Mutant
    clamp_product: <x, y> / max(|x| |y|, 1e-8)."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    nx, ny = np.sqrt((x * x).sum(-1)), np.sqrt((y * y).sum(-1))
    den = np.maximum(nx * ny, 1e-8) if mutant == "clamp_product" else np.maximum(nx, 1e-8) * np.maximum(ny, 1e-8)
    return (x * y).sum(-1) / den


def eval_metrics64(est, tgt, mix=None, emb=None, emb_gt=None, mutant=None):
    """eval_metrics_kernel in float64: est / tgt / mix [B, C, n], emb / emb_gt [B, D] -> ([B, 3] (mean over channels of
    SI-SNR(est, tgt), mean of SI-SNR(est, tgt) - SI-SNR(mix, tgt) (0 without mix), cosine (0 without embeddings)),
    [B, 3] bound on the kernel's error: its fp32 rounding plus si_snr_err64 of each term, or the cosine's double
    rounding 2 (D + 4) u64 (sum |x y| / den + |cos|)).  Mutants: METRICS_MUTANTS (first_ear: ear 0 instead of the mean;
    si_i_sign: si_snr_i negated)."""
    s = si_snr64(est, tgt, mutant)
    err = si_snr_err64(est, tgt)
    out, bound = np.zeros((s.shape[0], 3)), np.zeros((s.shape[0], 3))
    red = (lambda a: a[:, 0]) if mutant == "first_ear" else (lambda a: a.mean(1))
    out[:, 0], bound[:, 0] = red(s), err.mean(1)
    if mix is not None:
        out[:, 1] = red(s - si_snr64(mix, tgt, mutant)) * (-1 if mutant == "si_i_sign" else 1)
        bound[:, 1] = (err + si_snr_err64(mix, tgt)).mean(1)
    if emb is not None:
        x, y = np.asarray(emb, np.float64), np.asarray(emb_gt, np.float64)
        out[:, 2] = cos64(x, y, mutant)
        den = np.maximum(np.sqrt((x * x).sum(-1)), 1e-8) * np.maximum(np.sqrt((y * y).sum(-1)), 1e-8)
        bound[:, 2] = 2 * (x.shape[-1] + 4) * U64 * (np.abs(x * y).sum(-1) / den + np.abs(out[:, 2]))
    return out, U32 * (np.abs(out) + bound) + bound


def worst_ratio(got, ref, bound):
    """max |got - ref| / bound, where a zero bound asks for equality (inf if not met)"""
    d = np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bound > 0, d / np.where(bound > 0, bound, 1.0), np.where(d == 0, 0.0, np.inf))
    return float(r.max()) if r.size else 0.0


EMB_KINDS = ("random", "zero", "tiny", "parallel", "antiparallel", "huge", "tiny_vs_unit")


def metrics_inputs(B, C, n, seed, snr=(20.0,), dc=(0.0,), target="noise", mixture=True, D=None):
    """est, tgt, mix (or None), emb, emb_gt (or None), fp32.  The target: 0.1 N(0, 1) ("noise"), zeros ("silent") or one
    random constant per row ("constant").  Item b's estimate is dc_b 0.1 + 1.7 t + white noise at snr_b + 3 c dB on ear c
    (snr_b = snr[b % len(snr)], dc_b = dc[b // len(snr) % len(dc)], offsets in units of the target's RMS 0.1); the
    mixture t + 0.1 N(0, 1) + dc_b 0.05.  Embeddings of dimension D cycle through EMB_KINDS: zero (emb = 0), tiny (both
    of norm 1e-9), parallel (emb_gt = 3 emb), antiparallel (emb_gt = -emb / 2), huge (elements near 1e18),
    tiny_vs_unit (norms 1e-9 and 1)."""
    rng = np.random.default_rng(seed)
    if target == "noise":
        t = 0.1 * rng.standard_normal((B, C, n))
    elif target == "silent":
        t = np.zeros((B, C, n))
    else:
        t = np.broadcast_to(rng.uniform(-1, 1, (B, C, 1)), (B, C, n))
    t = t.astype(np.float32).astype(np.float64)
    sb = np.array([snr[b % len(snr)] for b in range(B)])[:, None] + 3.0 * np.arange(C)[None, :]
    db = np.array([dc[b // len(snr) % len(dc)] for b in range(B)])[:, None, None]
    w = 0.17 * 10.0 ** (-sb / 20)
    est = (db * 0.1 + 1.7 * t + w[:, :, None] * rng.standard_normal((B, C, n))).astype(np.float32)
    mix = (t + 0.1 * rng.standard_normal((B, C, n)) + db * 0.05).astype(np.float32) if mixture else None
    emb = emb_gt = None
    if D is not None:
        x, y = rng.standard_normal((B, D)), rng.standard_normal((B, D))
        for b in range(B):
            k = EMB_KINDS[b % len(EMB_KINDS)]
            nx = np.linalg.norm(x[b])
            if k == "zero":
                x[b] = 0.0
            elif k == "tiny":
                x[b], y[b] = x[b] * 1e-9 / nx, y[b] * 1e-9 / np.linalg.norm(y[b])
            elif k == "parallel":
                y[b] = 3.0 * x[b]
            elif k == "antiparallel":
                y[b] = -0.5 * x[b]
            elif k == "huge":
                x[b], y[b] = x[b] * 1e18, y[b] * 1e18
            elif k == "tiny_vs_unit":
                x[b], y[b] = x[b] * 1e-9 / nx, y[b] / np.linalg.norm(y[b])
        emb, emb_gt = x.astype(np.float32), y.astype(np.float32)
    return est, t.astype(np.float32), mix, emb, emb_gt


# (id, metrics_inputs arguments, mutants that must miss the bound by >= 10x on the case)
METRICS_CASES = (
    ("snr_sweep", dict(B=5, C=2, n=80000, seed=1, snr=(-30.0, 0.0, 30.0, 60.0, 90.0), D=256), ("first_ear", "si_i_sign")),
    ("dc_offsets", dict(B=8, C=2, n=80000, seed=2, snr=(60.0, 84.0), dc=(0.0, 1.0, 100.0, 1000.0), D=1000),
     ("no_centre", "one_pass", "first_ear", "si_i_sign", "clamp_product")),
    ("dc_long", dict(B=1, C=2, n=2 ** 20 + 3, seed=3, snr=(84.0,), dc=(1000.0,), D=257),
     ("no_centre", "one_pass", "first_ear", "si_i_sign")),
    ("one_ear", dict(B=5, C=1, n=257, seed=4, snr=(-10.0, 10.0, 40.0), dc=(0.0, 1.0), D=1), ("si_i_sign",)),
    ("three_ears", dict(B=5, C=3, n=255, seed=5, snr=(0.0, 25.0, 50.0), D=255), ("first_ear", "si_i_sign", "clamp_product")),
    ("n2", dict(B=1, C=2, n=2, seed=6, D=257), ()),
    ("n3_b300", dict(B=300, C=2, n=3, seed=7, snr=(-30.0, 0.0, 30.0, 90.0), D=1000), ("clamp_product",)),
    ("n256", dict(B=5, C=3, n=256, seed=8, snr=(10.0, 70.0), D=257), ("first_ear", "si_i_sign", "clamp_product")),
    ("silent_target", dict(B=2, C=2, n=1000, seed=9, target="silent", D=256), ("f64_eps",)),
    ("constant_target", dict(B=2, C=3, n=1001, seed=10, target="constant", dc=(100.0,), D=256), ("f64_eps",)),
    ("no_mixture", dict(B=5, C=2, n=2 ** 20 + 3, seed=11, snr=(90.0, 30.0), dc=(1.0, 1000.0), mixture=False, D=256),
     ("no_centre", "one_pass", "first_ear")),
    ("no_embeddings", dict(B=300, C=2, n=257, seed=12, snr=(-30.0, 0.0, 45.0, 90.0), dc=(0.0, 100.0)),
     ("no_centre", "first_ear", "si_i_sign")),
)
