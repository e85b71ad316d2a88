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


MIRRORS = {"kh_sizeof_asource": ASource, "kh_sizeof_gemm": Gemm, "kh_sizeof_plan": Plan, "kh_sizeof_lstm": Lstm}
SYMBOLS = ("kh_gemm", "kh_gemm_plan", "kh_split_planes", "kh_lstm", "kh_launch_count") + tuple(MIRRORS)

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


def layer_norm64(x, g, b, eps=1e-5):
    x = x.double()
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * g.double() + b.double()


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
