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
                ("bias", ctypes.c_void_p), ("ln_g", ctypes.c_void_p), ("ln_b", ctypes.c_void_p)]


class SepWeights(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("wqkv_t", "bqkv", "slopes", "lnq_g", "lnq_b", "lnk_g", "lnk_b", "lnv_g", "lnv_b",
                                                "wp_t", "bp", "lnp_g", "lnp_b")]


class SepFrontBack(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in ("wat", "ws", "wc", "bc", "we", "be", "lne_g", "lne_b", "wd", "bd")] + \
               [("gen", ctypes.c_int32)] + [(n, ctypes.c_void_p) for n in ("ln1_g", "ln1_b", "wih1_t", "b1")]


MIRRORS = {"kh_sizeof_asource": ASource, "kh_sizeof_gemm": Gemm, "kh_sizeof_plan": Plan, "kh_sizeof_lstm": Lstm,
           "kh_sizeof_sep_weights": SepWeights, "kh_sizeof_sep_front_back": SepFrontBack}
SYMBOLS = ("kh_gemm", "kh_gemm_plan", "kh_split_planes", "kh_lstm", "kh_launch_count", "kh_sep_layout", "kh_qkv",
           "kh_qkv_many", "kh_kv_gather", "kh_attention", "kh_attn_out", "kh_ln_frame_res",
           "kh_attn_cluster_resident", "kh_front", "kh_front_many", "kh_front_many_geometry", "kh_front1", "kh_back",
           "kh_back_many", "kh_back_many_geometry") + tuple(MIRRORS)

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
