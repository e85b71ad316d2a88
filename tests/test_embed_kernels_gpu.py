"""The enrollment network's own kernels (csrc/embed_kernels.cuh) launched directly, every kernel against float64.

estd_kernel, efront_kernel, egn_apply_kernel, eqkv_ln_kernel, softmax_rows_kernel, eattn_out_kernel, ehead_kernel,
einter_mask_kernel and eput_lens_kernel run through tests/kernels/kernel_harness.cu with embed_forward_impl's geometry
(eattn_out_kernel also with caller-chosen grids), on mixed-length batches (lengths 192 = the shortest, one inter window;
255; 256; 64 k + 63; the longest, not first in the batch) and on the equal-length path (lens null, N not a multiple of
64).  The references (kernels/harness.py: estd64, efront64, egn64, eqkv_ln64, softmax64, eattn_out64, ehead64,
einter_mask_expected) restate the model (tfgridnet.py:100-127, espnet2's GridNet block) for one utterance of its own
length; a CPU test pins them to oracle/restate.py.  Every float a kernel must not read or write holds a NaN sentinel:
x past each utterance's length, the DFT table's two pad columns, Q/K/V rows T .. Tp-1, O rows t >= T, HD rows
t >= T_b, the guard floats around every buffer.  Padded frames a kernel must leave alone must survive bit for bit.

Bounds (element-wise, computed by the references; u = 2^-24): estd one fp32 rounding of a double result; efront the
128-term DFT (plus the fp32 table and the scaled sample, u (sqrt(128) + 2)) carried through the 36-term conv plus bias
(u sqrt(37)); the GroupNorm sums carry those bounds (they are double atomics, so they are compared with a bound, not bit
for bit); egn_apply 5 fp32 roundings of the normalised value plus the fp32 mean; the LayerNorms (eqkv_ln, eattn_out,
ehead) their fp32 two-pass statistics (u per term of the longest per-thread chain plus the tree), rsqrtf (2 ulp) and
the affine, with the bounds of their inputs carried through; softmax_rows the __expf error, (2 + 1.2 |s - max|) ulp plus
the rounding of s - max, and the sum.  K and V come out as bf16 hi/lo planes: hi + lo is held to the bound plus the
split's own 2^-17, and hi to 2^-8 of the value.  einter_mask and eput_lens are exact.  Every kernel is also compared
with the mutated references that apply to it; each must miss by >= 10x the bound.
Measured on one NVIDIA H100 80GB HBM3 (700 W power limit): worst error / bound 0.57 (estd), 0.058 (efront), 0.001 (its
GroupNorm sums), 0.79 (egn_apply), 0.34 / 0.89 / 0.89 (eqkv_ln Q / K / V), 0.38 (softmax_rows), 0.82 (eattn_out),
0.065 (ehead); einter_mask and eput_lens exact.  Smallest mutant error / bound: 22 (egn_apply against the unbiased
variance over 74 880 values), 2650 (efront, symmetric Hann), 3800 (estd, biased); every other mutant misses by more than
10^5x.

Also here: the premise of the padded inter path (sigma(-inf) = 0 exactly, so h and c stay exactly 0 in masked windows)
on each recurrence kernel, and two chain-level checks through EmbedTFGridNet: a NaN-poisoned workspace, and one call of
more than LENS_PER_LAUNCH utterances.
"""
import ctypes
import math

import pytest
import torch

from kernels import harness as kh
from kernels.scaffold import Guarded, Ledger, bits, dev, is_sentinel, ratio, sentinel  # noqa: F401
from lookoncetohear_b200 import EmbedTFGridNet, _cabi, synth
from lookoncetohear_b200.configs import EMBED_PARAMS
from oracle import restate as rs

pytestmark = pytest.mark.gpu

NF, CH, FC, NH, QK, VDIM, HOP = kh.E_NF, kh.E_CH, kh.E_FC, kh.E_NH, kh.E_QK, kh.E_VDIM, kh.E_HOP
# mixed lengths: the shortest (T_b = 4: one inter window), 255, 256, 64 k + 63, the longest (not first)
LENS_MIXED = [1343, 192, 4000, 255, 256]
CASES = {"mixed": (LENS_MIXED, max(LENS_MIXED)), "equal": (None, 1100)}      # equal: N not a multiple of 64
LEDGER = Ledger()


@pytest.fixture(scope="module")
def w(dev):
    return Weights(dev)


@pytest.fixture(scope="module", autouse=True)
def summary():
    yield
    LEDGER.summary()


def lens_dev(lens, dev):
    return None if lens is None else torch.tensor(lens, dtype=torch.int32, device=dev)


def own(lens, N, B):
    return [N] * B if lens is None else list(lens)


# ---- weights ---------------------------------------------------------------------------------------------------------
class Weights:
    """a seeded EmbedTFGridNet's weights with random affine parameters, packed as the engine packs them (kh.pack_embed),
    and the engine's fp32 DFT table with NaN in its two pad columns"""

    def __init__(self, dev):
        torch.manual_seed(0)
        sd = {k: v.detach().clone() for k, v in EmbedTFGridNet(**EMBED_PARAMS).state_dict().items()}
        g = torch.Generator().manual_seed(1)
        for k, v in sd.items():
            if k.endswith((".gamma", "conv.1.weight", "embed_proj.1.weight")):
                sd[k] = 1 + 0.3 * torch.randn(v.shape, generator=g)
            elif k.endswith((".beta", "conv.1.bias", "embed_proj.1.bias")):
                sd[k] = 0.3 * torch.randn(v.shape, generator=g)
        sd["blocks.0.attn_concat_proj.1.weight"] = torch.tensor([-0.4])     # a slope far from 1
        self.sd = sd
        self.p = kh.pack_embed(sd)
        self.Wc = sd["conv.0.weight"]
        self.d = {k: v.contiguous().to(dev) for k, v in self.p.items()}
        self.d["dft"] = kh.dft_table32().to(dev)
        self.c = kh.EmbWeights()
        for k in ("dft", "wc", "bc", "gn_g", "gn_b", "lnh_g", "lnh_b"):
            setattr(self.c, k, self.d[k].data_ptr())
        self.cb = kh.EmbBlock()
        for k in ("gq", "bq", "gk", "bk", "gv", "bv", "wp_t", "bp", "slope_p", "gp", "bpn"):
            setattr(self.cb, k, self.d["0." + k].data_ptr())

    def b(self, k):
        return self.p["0." + k]


def signal(lens, N, dev, seed):
    """x [B][2][N] (CPU, real data everywhere) and its device copy with NaN past each utterance's length"""
    g = torch.Generator().manual_seed(seed)
    B = len(own(lens, N, 1)) if lens is not None else 2
    x = 0.7 * torch.randn(B, 2, N, generator=g)
    xd = x.clone()
    for b, n in enumerate(own(lens, N, B)):
        xd[b, :, n:] = float("nan")
    return x, xd.to(dev)


# ---- estd, efront, egn_apply -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_estd(case, dev):
    lens, N = CASES[case]
    x, xd = signal(lens, N, dev, 10)
    B = x.shape[0]
    inv = Guarded((B,), dev)
    assert kh.estd(xd, N, lens_dev(lens, dev), inv.t, B) == 0
    torch.cuda.synchronize()
    assert inv.ok()
    inv = inv.t
    err, mut = 0.0, {"biased": 0.0, "mic0": 0.0}
    for b, n in enumerate(own(lens, N, B)):
        ref, bound = kh.estd64(x[b], n)
        err = max(err, ratio(inv[b:b + 1], ref.view(1), bound.view(1)))
        mut["biased"] = max(mut["biased"], ratio(inv[b:b + 1], kh.estd64(x[b], n, unbiased=False)[0].view(1), bound.view(1)))
        mut["mic0"] = max(mut["mic0"], ratio(inv[b:b + 1], kh.estd64(x[b], n, mic0_only=True)[0].view(1), bound.view(1)))
    LEDGER.check("estd", err, mut)


@pytest.mark.parametrize("case", list(CASES))
def test_efront(case, dev, w):
    """every frame (t = 0 and t = T_b - 1 included) against efront64, rows t >= T_b exactly zero, and the GroupNorm sums
    of each utterance"""
    lens, N = CASES[case]
    x, xd = signal(lens, N, dev, 11)
    B, T = x.shape[0], kh.e_frames(N)
    inv = torch.stack([kh.estd64(x[b], n)[0] for b, n in enumerate(own(lens, N, B))]).float()
    X = Guarded((B, T, NF, CH), dev)
    gn = torch.zeros(2 * B + 2, dtype=torch.float64, device=dev)
    gn[2 * B:] = float("nan")
    assert kh.efront(w.c, xd, N, lens_dev(lens, dev), inv.to(dev), X.t, gn, B, T) == 0
    torch.cuda.synchronize()
    assert X.ok() and bool(gn[2 * B:].isnan().all())
    X = X.t
    muts = dict(edge_repeat=dict(edge_repeat=True), reflect_at_N=dict(reflect_at=N), symmetric_hann=dict(symmetric_hann=True),
                reim_interleaved=dict(reim_interleaved=True), conv_flip_time=dict(conv_flip_time=True))
    err, errs, mut = 0.0, 0.0, {k: 0.0 for k in muts}
    bc = w.p["bc"]
    for b, n in enumerate(own(lens, N, B)):
        ref = kh.efront64(x[b], n, T, inv[b], w.Wc, bc)
        err = max(err, ratio(X[b], ref["X"], ref["X_bound"]))
        errs = max(errs, ratio(gn[2 * b:2 * b + 2], ref["sums"], ref["sums_bound"]))
        assert bool((bits(X[b, kh.e_frames(n):]) == 0).all())
        for k, m in muts.items():
            mut[k] = max(mut[k], ratio(X[b], kh.efront64(x[b], n, T, inv[b], w.Wc, bc, **m)["X"], ref["X_bound"]))
    if lens is None:
        del mut["reflect_at_N"]                        # the same thing on the equal-length path
    LEDGER.check("efront", err, mut)
    LEDGER.check("efront GN sums", errs, {})


@pytest.mark.parametrize("case", list(CASES))
def test_egn_apply(case, dev, w):
    """total4 is not a multiple of 256 in either case; padded frames (random data here) must stay bit-identical"""
    lens, N = CASES[case]
    B, T = len(own(lens, N, 2)), kh.e_frames(N)
    g = torch.Generator().manual_seed(12)
    X0 = (1.5 * torch.randn(B, T, NF, CH, generator=g) + 0.3)
    total4 = B * T * FC // 4
    assert total4 % 256 != 0
    sums = torch.zeros(2 * B, dtype=torch.float64)
    for b, n in enumerate(own(lens, N, B)):
        r = X0[b, :kh.e_frames(n)].double()
        sums[2 * b], sums[2 * b + 1] = r.sum(), (r * r).sum()
    X = Guarded((B, T, NF, CH), dev, X0)
    assert kh.egn_apply(w.c, X.t, sums.to(dev), T * FC, total4, lens_dev(lens, dev)) == 0
    torch.cuda.synchronize()
    assert X.ok()
    X = X.t
    err, mut = 0.0, {"padded_count": 0.0, "unbiased": 0.0}
    for b, n in enumerate(own(lens, N, B)):
        Tb = kh.e_frames(n)
        ref, bound = kh.egn64(X0[b], sums[2 * b:2 * b + 2], Tb, w.p["gn_g"], w.p["gn_b"])
        err = max(err, ratio(X[b], ref, bound))
        assert torch.equal(bits(X[b, Tb:]).cpu(), bits(X0[b, Tb:]))
        for k in mut:
            m = kh.egn64(X0[b], sums[2 * b:2 * b + 2], Tb, w.p["gn_g"], w.p["gn_b"], **{k: True})[0]
            mut[k] = max(mut[k], ratio(X[b], m, bound))
    if lens is None:
        del mut["padded_count"]
    LEDGER.check("egn_apply", err, mut)


# ---- eqkv_ln ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,T,Tp", [(2, 40, 64), (1, 64, 64)], ids=["T40_Tp64", "T64"])
def test_eqkv_ln(B, T, Tp, dev, w):
    g = torch.Generator().manual_seed(13 + T)
    QKV = torch.randn(B, T, NF, kh.E_NQKV, generator=g) * 1.3 + 0.2
    Z = B * NH
    k_plane, v_plane = Z * Tp * QK, Z * Tp * VDIM
    Qg = Guarded((Z, Tp, QK), dev)
    Kg, Vg = Guarded((k_plane,), dev), Guarded((v_plane,), dev)         # two bf16 planes = one float per element
    Qn = Qg.t
    Kp, Vp = Kg.t.view(torch.bfloat16).view(2, Z, Tp, QK), Vg.t.view(torch.bfloat16).view(2, Z, Tp, VDIM)
    assert kh.eqkv_ln(w.cb, QKV.to(dev), Qn, Kp, Vp, k_plane, v_plane, B, T, Tp) == 0
    torch.cuda.synchronize()
    assert Qg.ok() and Kg.ok() and Vg.ok()
    assert is_sentinel(Qn[:, T:])
    for P, n in ((Kp, QK), (Vp, VDIM)):                            # rows T .. Tp-1 of both planes keep the sentinel
        fresh = sentinel(P.numel() // 2, dev).view(torch.int16).view(P.shape)
        assert torch.equal(P.view(torch.int16)[:, :, T:], fresh[:, :, T:])
    ln = [w.b(k) for k in ("gq", "bq", "gk", "bk", "gv", "bv")]
    muts = dict(per_bin=dict(per_bin=True), heads_transposed=dict(heads_transposed=True), swap_qk_gains=dict(swap_qk_gains=True))
    errs = {"Q": 0.0, "K": 0.0, "V": 0.0}
    mut = {k: 0.0 for k in muts}
    for b in range(B):
        ref = kh.eqkv_ln64(QKV[b], *ln)
        mrefs = {k: kh.eqkv_ln64(QKV[b], *ln, **m) for k, m in muts.items()}
        got = {"Q": Qn.view(B, NH, Tp, QK)[b, :, :T]}
        for name, P, n in (("K", Kp, QK), ("V", Vp, VDIM)):
            hi = P[0].view(B, NH, Tp, n)[b, :, :T].double().cpu()
            lo = P[1].view(B, NH, Tp, n)[b, :, :T].double().cpu()
            v = ref[name][0]
            assert bool(((hi - v).abs() <= 2.0 ** -8 * v.abs() + ref[name][1]).all()), name      # hi is the leading part
            got[name] = hi + lo
        for name in "QKV":
            v, bound = ref[name]
            if name != "Q":
                bound = bound + 2.0 ** -17 * v.abs()
            errs[name] = max(errs[name], ratio(got[name], v, bound))
            for k in muts:
                mut[k] = max(mut[k], ratio(got[name], mrefs[k][name][0], bound))
    for name in "QKV":
        LEDGER.check(f"eqkv_ln {name}", errs[name], mut if name == "V" else {})


# ---- softmax_rows ----------------------------------------------------------------------------------------------------
SOFTMAX = {
    # utterances of different T_b in one launch (z % 4 would pick another utterance's length), padded query rows
    "mixed": ([640, 192, 1343, 4000, 300], 4000, 3.0),
    "large_scores": ([640, 192, 1343, 4000, 300], 4000, 80.0),        # |s| up to about 80
    "equal_T1251": (None, 80000, 2.0),                                 # ld = Tp = 1280 at T = 1251
}


@pytest.mark.parametrize("case", list(SOFTMAX))
def test_softmax_rows(case, dev):
    lens, N, scale = SOFTMAX[case]
    T = kh.e_frames(N)
    Tp = (T + 63) // 64 * 64
    B = 1 if lens is None else len(lens)
    Z = B * NH
    g = torch.Generator().manual_seed(14)
    S0 = (torch.rand(Z * T, Tp, generator=g) * 2 - 1) * scale if scale > 10 else scale * torch.randn(Z * T, Tp, generator=g)
    S = Guarded((Z * T, Tp), dev, S0)
    assert kh.softmax_rows(S.t, Tp, T, T, T * Tp, Z, lens_dev(lens, dev)) == 0
    torch.cuda.synchronize()
    assert S.ok()
    S = S.t
    ncols = kh.softmax_row_lens(Z, T, lens, T)
    ref, bound = kh.softmax64(S0, ncols)
    mut = {"pad_not_zeroed": ratio(S, kh.softmax64(S0, ncols, zero_pad=False)[0], bound)}
    if lens is not None:
        mut["len_z_mod_NH"] = ratio(S, kh.softmax64(S0, kh.softmax_row_lens(Z, T, lens, T, by_mod=True))[0], bound)
    LEDGER.check("softmax_rows", ratio(S, ref, bound), mut)


# ---- eattn_out -------------------------------------------------------------------------------------------------------
EATTN = [(3, 9, 64, "engine"), (3, 9, 64, 1), (3, 9, 64, 7), (3, 9, 64, 40), (3, 200, 256, "engine")]


@pytest.mark.parametrize("B,T,Tp,grid", EATTN, ids=[f"B{b}_T{t}_grid{g}" for b, t, _, g in EATTN])
def test_eattn_out(B, T, Tp, grid, dev, w):
    """grid 7 and 1: a CTA walks frames of several utterances; 40 > 27 frames: CTAs with no frame.  O rows t >= T are NaN"""
    if grid == "engine":
        grid = kh.eattn_out_grid(T, B)
        assert grid == min(T * B, 132 * 4)
    g = torch.Generator().manual_seed(15 + T)
    O0 = torch.randn(B, NH, T, VDIM, generator=g)
    X0 = torch.randn(B, T, NF, CH, generator=g)
    O, X = Guarded((B, NH, Tp, VDIM), dev), Guarded((B, T, NF, CH), dev, X0)
    O.t[:, :, :T] = O0.to(dev)
    assert kh.eattn_out(w.cb, O.t, X.t, T, Tp, T * B, grid) == 0
    torch.cuda.synchronize()
    assert O.ok() and X.ok()
    X = X.t
    a = [w.b(k) for k in ("wp_t", "bp", "slope_p", "gp", "bpn")]
    muts = dict(heads_cf=dict(heads_cf=True), ignore_slope=dict(ignore_slope=True), ln_per_bin=dict(ln_per_bin=True))
    err, mut = 0.0, {k: 0.0 for k in muts}
    for b in range(B):
        Ob = O0[b].transpose(0, 1)                                   # [T][4][1040]
        ref, bound = kh.eattn_out64(Ob, X0[b], *a)
        err = max(err, ratio(X[b], ref, bound))
        for k, m in muts.items():
            mut[k] = max(mut[k], ratio(X[b], kh.eattn_out64(Ob, X0[b], *a, **m)[0], bound))
    LEDGER.check("eattn_out", err, mut)


# ---- ehead -----------------------------------------------------------------------------------------------------------
EHEAD = {"mixed": ([400, 1216, 192, 1200], 1216), "equal": (None, 13 * HOP + 5)}   # T_b 7, 20 (= T), 4, 19; T = 14


@pytest.mark.parametrize("case", list(EHEAD))
def test_ehead(case, dev, w):
    lens, N = EHEAD[case]
    T = kh.e_frames(N)
    B = len(own(lens, N, 2))
    g = torch.Generator().manual_seed(16)
    HD0 = torch.randn(B, T, 256, generator=g) * 2 + 0.5
    HDd = HD0.clone()
    for b, n in enumerate(own(lens, N, B)):
        HDd[b, kh.e_frames(n):] = float("nan")                       # never read
    out = Guarded((B, 256), dev)
    assert kh.ehead(w.c, HDd.to(dev), out.t, B, T, lens_dev(lens, dev)) == 0
    torch.cuda.synchronize()
    assert out.ok()
    out = out.t
    err, mut = 0.0, {"div_T": 0.0, "mean_before_ln": 0.0}
    for b, n in enumerate(own(lens, N, B)):
        Tb = kh.e_frames(n)
        ref, bound = kh.ehead64(HD0[b], Tb, w.p["lnh_g"], w.p["lnh_b"])
        err = max(err, ratio(out[b], ref, bound))
        for k in mut:
            mut[k] = max(mut[k], ratio(out[b], kh.ehead64(HD0[b], Tb, w.p["lnh_g"], w.p["lnh_b"], **{k: True})[0], bound))
    if lens is None:
        del mut["div_T"]
    LEDGER.check("ehead", err, mut)


# ---- einter_mask, eput_lens ------------------------------------------------------------------------------------------
def test_einter_mask(dev):
    """bit-exact, the longest utterance (4000 samples) untouched, the shortest (one inter window) fully masked"""
    lens, N = LENS_MIXED, max(LENS_MIXED)
    steps = kh.e_frames(N) - 3
    B = len(lens)
    g = torch.Generator().manual_seed(17)
    gx0 = torch.randn(B * NF, steps, 512, generator=g)
    gx = Guarded((B * NF, steps, 512), dev, gx0)
    assert kh.einter_mask(gx.t, lens_dev(lens, dev), B, steps) == 0
    torch.cuda.synchronize()
    assert gx.ok()
    got = gx.t.cpu()
    ref = kh.einter_mask_expected(gx0, lens, steps)
    assert torch.equal(bits(got), bits(ref))
    ilong = lens.index(N)
    assert torch.equal(bits(got.view(B, NF, -1)[ilong]), bits(gx0.view(B, NF, -1)[ilong]))
    for m in (dict(start=4), dict(start=2), dict(fwd_only=True), dict(pad=(float("-inf"), 0.0, float("-inf"), 0.0))):
        assert not torch.equal(bits(got), bits(kh.einter_mask_expected(gx0, lens, steps, **m))), m
    LEDGER.check("einter_mask", 0.0, {"start_Tb-4": math.inf, "start_Tb-2": math.inf, "fwd_only": math.inf,
                                      "gate_order": math.inf})


@pytest.mark.parametrize("n", [1, 1000, 1001])
def test_eput_lens(n, dev):
    lens = [192 + 37 * i for i in range(n)]
    dst = Guarded((n,), dev)
    n0 = kh.lib().kh_launch_count()
    assert kh.eput_lens(dst.t, lens, n) == 0
    torch.cuda.synchronize()
    assert kh.lib().kh_launch_count() - n0 == (n + kh.E_LENS_PER_LAUNCH - 1) // kh.E_LENS_PER_LAUNCH
    assert bits(dst.t).cpu().tolist() == lens
    assert dst.ok()


# ---- the -inf premise on the recurrences -----------------------------------------------------------------------------
RECURRENCES = [("rec3_pre", 3), ("rec3_ring", 3), ("rec4_2", 3), ("rec4_4", 3), ("tc", 1), ("tc", 2), ("tc", 3)]


@pytest.mark.parametrize("variant,passes", RECURRENCES, ids=[f"{v}_p{p}" for v, p in RECURRENCES])
def test_masked_windows_leave_zero_state(variant, passes, dev):
    """gate pre-activations of the inter path masked as einter_mask leaves them (the engine's layout: sequence (b, f),
    steps of one sequence contiguous, both directions): h is exactly 0 in every masked window, every output is finite,
    and the real windows equal, bit for bit, a run of the same variant over only the T_b - 3 real steps -- the reverse
    direction reaches its first real window in exactly zero state"""
    lens = [20 * HOP, 9 * HOP + 17, 4 * HOP]                      # T_b 21 (the longest), 10, 5
    B, L = len(lens), kh.e_frames(max(lens)) - 3
    g = torch.Generator().manual_seed(18)
    gx = kh.einter_mask_expected(0.8 * torch.randn(B * NF, L, 512, generator=g), lens, L)
    whh = ((torch.rand(2, 256, 64, generator=g) * 2 - 1) * 0.25).to(dev)

    def run(gx_, nseq, steps):
        gd = gx_.contiguous().to(dev)
        out = sentinel(nseq * steps * 128, dev).view(nseq, steps, 128)
        a = kh.Lstm()
        a.gx, a.gx_ld, a.out, a.out_ld, a.whh = gd.data_ptr(), 512, out.data_ptr(), 128, whh.data_ptr()
        a.nseq, a.L, a.inner_count, a.ndir = nseq, steps, 1, 2
        a.outer_stride, a.inner_stride, a.step_stride = steps, 0, 1
        rc, why = kh.lstm(a, variant, passes)
        torch.cuda.synchronize()
        assert rc == 0, why
        return out.cpu()

    full = run(gx, B * NF, L).view(B, NF, L, 128)
    assert bool(torch.isfinite(full).all())
    for b, n in enumerate(lens):
        real = kh.e_frames(n) - 3
        assert bool((full[b, :, real:] == 0).all()), (b, "h not exactly 0 in a masked window")
        alone = run(gx.view(B, NF, L, 512)[b, :, :real], NF, real)
        assert torch.equal(full[b, :, :real], alone.view(NF, real, 128)), (b, variant, passes)


# ---- the chain through EmbedTFGridNet --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def net(dev):
    torch.manual_seed(0)
    return EmbedTFGridNet(**EMBED_PARAMS).eval().to(dev)


def _ws_bytes(net, B, N):
    n = ctypes.c_size_t()
    _cabi.check(_cabi.lib().l2h_embed_workspace_bytes(net._engine(), B, N, ctypes.byref(n)))
    return n.value


@pytest.mark.parametrize("lens,N", [([4800, 192, 1343, 3000], 4800), (None, 1100)], ids=["mixed", "equal"])
def test_poisoned_workspace(net, dev, lens, N):
    """a workspace full of NaN (refilled before every call: a call reuses the buffer) gives the embedding of a zeroed
    one: no kernel of the chain reads workspace the chain has not written (rows T .. Tp-1, the padding of S, the tails of
    HC and GX)"""
    B = 2 if lens is None else len(lens)
    x = synth.enrollment(B, N, seed0=4100).to(dev)
    outs = {}
    for fill in (0x00, 0xFF):                                      # 0xFF bytes: NaN floats and doubles
        net._ws = torch.full((_ws_bytes(net, B, N) + 4096,), fill, dtype=torch.uint8, device=dev)
        with torch.no_grad():
            outs[fill] = net(x, lengths=lens).cpu()
    assert bool(torch.isfinite(outs[0xFF]).all())
    assert rs.rel_l2(outs[0xFF], outs[0x00]) <= 1e-6, rs.rel_l2(outs[0xFF], outs[0x00])
    net._ws = None


def test_more_than_one_lengths_block(dev):
    """one mixed-length call of 1003 utterances takes two eput_lens launches; each row equals the equal-length call of
    its length group (recurrences pinned to the tensor cores on both sides)"""
    torch.manual_seed(0)
    m = EmbedTFGridNet(**EMBED_PARAMS).eval().to(dev)
    m.set_option("tc_lstm_min", 1)
    n_utt = 1003
    lens = [(192, 255, 256)[i % 3] for i in range(n_utt)]
    x = synth.enrollment(n_utt, 256, seed0=4200).to(dev)
    with torch.no_grad():
        o = m(x, lengths=lens).cpu()
        assert bool(torch.isfinite(o).all())
        for n in (192, 255, 256):
            idx = [i for i, v in enumerate(lens) if v == n]
            r = m(x[idx, :, :n].contiguous()).cpu()
            for j, i in enumerate(idx):
                e = rs.rel_l2(o[i:i + 1], r[j:j + 1])
                assert e <= 1e-5, (i, n, e)
