"""The LSTM recurrences (csrc/lstm.cuh, csrc/tc_lstm.cuh) launched directly, every kernel against the float64 LSTM.

For each shape the reference runs once and every variant is compared with it: launch_lstm_rec's own choice, each
CUDA-core kernel forced (lstm_rec3_kernel<1,true/false>, lstm_rec4_kernel<2/4>), the tensor-core recurrence
(launch_tc_lstm) and the one with LayerNorm + W_ih inside (launch_tc_lstm_x, against LN + W_ih + W_hh in float64).
Shapes cover the intra layout (one sequence per row block, gaps between blocks) and the inter layout (inner_count = 97,
step_stride = 97), an output layout of its own, carried (h0, c0) state at a stride with gaps, both directions, and a
tensor-core tail CTA (4099 sequences).  h is checked at every step, the final (h, c) too; the output buffer's other
columns, its padding and the state gaps hold a NaN sentinel that must survive.

Bounds on |h - h64| (absolute): CUDA-core kernels and passes = 3 errors come from the approximate activations (~1e-7 each)
and fp32 (or bf16x3) products, carried over the steps.  On the same data the passes = 2 error must be >= 10x the
passes = 3 bound (the W_lo term is applied) and the passes = 1 error larger still (the h_lo / x_lo term is dropped).
Measured on one H100 80GB HBM3: worst error / bound 0.26 (CUDA core, 3.9e-7), 0.29 (tc_lstm, 5.8e-6), 0.45
(tc_lstm_x, 2.2e-5); passes = 2 error / passes = 3 bound >= 84x; RMS error passes 1 / passes 2 >= 1.39.
"""
from dataclasses import dataclass

import pytest
import torch

from kernels import harness as kh
from kernels.scaffold import SENSITIVITY, SENTINEL, dev, sentinel  # noqa: F401

pytestmark = pytest.mark.gpu

TOL = {"cuda": 1.5e-6, "tc": 2e-5, "tc_x": 5e-5}    # |h - h64| bound per family (passes = 3 for the tensor cores)


@dataclass
class S:
    nseq: int
    L: int
    ndir: int
    inter: bool
    own_out: bool = False
    state: bool = False

    @property
    def name(self):
        return (f"n{self.nseq}_L{self.L}_d{self.ndir}_{'inter' if self.inter else 'intra'}"
                f"{'_out' if self.own_out else ''}{'_state' if self.state else ''}")


def _layout(s):
    """row addressing (inner_count, outer, inner, step) of gx / x and of out; rows in each"""
    if s.inter:
        ic = 97
        n_out = (s.nseq + ic - 1) // ic
        g = (ic, s.L * ic, 1, ic)
        o = (ic, (s.L + 1) * ic, 1, ic) if s.own_out else g
        rows_g, rows_o = n_out * s.L * ic, n_out * (s.L + 1 if s.own_out else s.L) * ic
    else:
        ic = 1
        g = (1, s.L + 2, 0, 1)                       # two gap rows between sequences
        o = (1, s.L + 3, 0, 1) if s.own_out else g
        rows_g, rows_o = s.nseq * (s.L + 2), s.nseq * (o[1])
    return g, o, rows_g, rows_o


def _rows(lay, seqs, step):
    ic, outer, inner, st = lay
    return (seqs // ic) * outer + (seqs % ic) * inner + step * st


class Problem:
    def __init__(self, s, dev, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.s, self.dev = s, dev
        self.gl, self.ol, rows_g, rows_o = _layout(s)
        ic = self.gl[0]
        n_out = (s.nseq + ic - 1) // ic
        self.gx_ld = s.ndir * 256 + 4
        self.x_ld = 68
        x = torch.randn(rows_g, self.x_ld, generator=g)
        self.x = x
        self.ln_g = 1 + 0.2 * torch.randn(64, generator=g)
        self.ln_b = 0.2 * torch.randn(64, generator=g)
        self.wih = (torch.rand(s.ndir * 256, 64, generator=g) * 2 - 1) * 0.25
        self.bias = 0.3 * torch.randn(s.ndir * 256, generator=g)
        self.whh = (torch.rand(s.ndir, 256, 64, generator=g) * 2 - 1) * 0.25
        gx64 = kh.layer_norm64(x[:, :64], self.ln_g, self.ln_b) @ self.wih.double().T + self.bias.double()
        self.gx = torch.zeros(rows_g, self.gx_ld)
        self.gx[:, :s.ndir * 256] = gx64.float()
        self.out_ld = 136
        self.rows_o = rows_o
        self.hc_stride = ic * 64 + 16                # gaps between state records
        self.n_hc = n_out * self.hc_stride
        seqs = torch.arange(s.nseq)
        self.hc_idx = ((seqs // ic) * self.hc_stride + (seqs % ic) * 64)[:, None] + torch.arange(64)[None, :]
        self.h0 = self.c0 = None
        if s.state:
            self.h0 = 0.5 * torch.randn(s.nseq, 64, generator=g)
            self.c0 = 0.5 * torch.randn(s.nseq, 64, generator=g)
        self.ref, self.fin = kh.lstm_ref(self.gx, self.whh, s.nseq, s.L, s.ndir, lambda q, t: _rows(self.gl, q, t),
                                         self.h0, self.c0)
        # every element of `out` the problem owns
        steps = torch.arange(s.L)
        orow = _rows(self.ol, seqs[None, :], steps[:, None])                       # [L][nseq]
        self.out_idx = torch.stack([orow[..., None] * self.out_ld + d * 64 + torch.arange(64) for d in range(s.ndir)])
        self.d_gx, self.d_x, self.d_whh = self.gx.to(dev), x.to(dev), self.whh.to(dev)
        self.d_bias, self.d_lng, self.d_lnb = self.bias.to(dev), self.ln_g.to(dev), self.ln_b.to(dev)
        hi, lo = kh.split_bf16(self.wih)
        self.d_wih_hi, self.d_wih_lo = hi.to(dev), lo.to(dev)

    def run(self, variant, passes=3, h_state=True):
        s, dev = self.s, self.dev
        out = sentinel(self.rows_o * self.out_ld, dev)
        h = c = None
        if s.state and h_state:
            h = sentinel(self.n_hc, dev)
            c = h.clone()
            h[self.hc_idx.to(dev)] = self.h0.to(dev)
            c[self.hc_idx.to(dev)] = self.c0.to(dev)
        a = kh.Lstm()
        a.gx, a.gx_ld, a.out, a.out_ld, a.whh = self.d_gx.data_ptr(), self.gx_ld, out.data_ptr(), self.out_ld, self.d_whh.data_ptr()
        a.h_state, a.c_state, a.hc_outer_stride = kh.ptr(h), kh.ptr(c), self.hc_stride
        a.nseq, a.L, a.inner_count, a.ndir = s.nseq, s.L, self.gl[0], s.ndir
        a.outer_stride, a.inner_stride, a.step_stride = self.gl[1], self.gl[2], self.gl[3]
        if s.own_out:
            a.out_outer_stride, a.out_inner_stride, a.out_step_stride = self.ol[1], self.ol[2], self.ol[3]
        a.x, a.x_ld, a.wih_hi, a.wih_lo = self.d_x.data_ptr(), self.x_ld, self.d_wih_hi.data_ptr(), self.d_wih_lo.data_ptr()
        a.bias, a.ln_g, a.ln_b = self.d_bias.data_ptr(), self.d_lng.data_ptr(), self.d_lnb.data_ptr()
        rc, why = kh.lstm(a, variant, passes)
        torch.cuda.synchronize()
        return rc, why, a, out, h, c

    def check(self, variant, passes=3):
        """max |h - h64| over every step (and the final h, c); asserts the sentinels survived"""
        rc, why, _, out, h, c = self.run(variant, passes)
        assert rc == 0, (variant, why)
        oi = self.out_idx.to(self.dev)
        got = out[oi].double().cpu()                                      # [ndir][L][nseq][64]
        untouched = torch.ones_like(out, dtype=torch.bool)
        untouched[oi.reshape(-1)] = False
        assert bool((out.view(torch.int32)[untouched] == SENTINEL).all()), f"{variant}: out written outside the problem"
        assert bool(torch.isfinite(got).all()), variant
        err = float((got - self.ref).abs().max())
        self.rms = float((got - self.ref).pow(2).mean().sqrt())
        if self.s.state:
            hi = self.hc_idx.to(self.dev)
            gap = torch.ones_like(h, dtype=torch.bool)
            gap[hi.reshape(-1)] = False
            assert bool((h.view(torch.int32)[gap] == SENTINEL).all()) and bool((c.view(torch.int32)[gap] == SENTINEL).all())
            hf, cf = self.fin[0]
            err = max(err, float((h[hi].double().cpu() - hf).abs().max()))
            err = max(err, float(((c[hi].double().cpu() - cf).abs() / (1 + cf.abs())).max()))
        return err


SHAPES = [
    S(1, 1, 1, False, state=True),
    S(1, 2, 2, True),
    S(31, 2, 2, False, own_out=True),
    S(32, 97, 1, True, own_out=True, state=True),
    S(33, 500, 1, False, state=True),
    S(33, 97, 2, True),
    S(31, 500, 2, True, own_out=True),
    S(4099, 97, 1, True, state=True),
    S(4099, 2, 2, False, own_out=True),
]


@pytest.mark.parametrize("shape", SHAPES, ids=[s.name for s in SHAPES])
def test_recurrence_variants(shape, dev):
    p = Problem(shape, dev, seed=shape.nseq + shape.L)
    variants = ["auto", "rec3_ring", "rec4_2", "rec4_4", "tc", "tc_x"]
    if shape.L * 1024 <= 200 * 1024:
        variants.insert(1, "rec3_pre")
    errs = {}
    for v in variants:
        errs[v] = p.check(v)
    print(f"[{shape.name}] |h - h64| max: " + ", ".join(f"{v} {e:.2e}" for v, e in errs.items()))
    for v, e in errs.items():
        fam = v if v in ("tc", "tc_x") else "cuda"
        assert e <= TOL[fam], (v, e, TOL[fam])


SENS_SHAPES = [S(32, 97, 1, True, own_out=True, state=True), S(33, 97, 2, True)]


@pytest.mark.parametrize("shape", SENS_SHAPES, ids=[s.name for s in SENS_SHAPES])
@pytest.mark.parametrize("variant", ["tc", "tc_x"])
def test_tensor_core_pass_counts(variant, shape, dev):
    """passes 3 < 2 < 1 in error: the W_lo term is applied at 3 only, the h_lo (x_lo) term at 2 and 3.  Passes 2 and 1
    are ordered by the RMS error over all steps: dropping h_lo adds an error term independent of the dropped W_lo term
    (about sqrt(2) x the RMS), while the max over a few thousand values is too noisy to order them."""
    p = Problem(shape, dev, seed=7)
    e, rms = {}, {}
    for ps in (1, 2, 3):
        e[ps] = p.check(variant, ps)
        rms[ps] = p.rms
    print(f"[{variant} {shape.name}] |h - h64| by passes: max {e}, rms {rms}; passes-2 error / passes-3 bound "
          f"{e[2] / TOL[variant]:.1f}, rms 1 / rms 2 {rms[1] / rms[2]:.2f}")
    assert e[3] <= TOL[variant]
    assert e[2] >= SENSITIVITY * TOL[variant], e
    assert rms[1] > 1.15 * rms[2], rms


@pytest.mark.parametrize("variant", ["auto", "rec3_pre", "rec3_ring", "rec4_2", "rec4_4", "tc", "tc_x"])
def test_bidirectional_carried_state_refused(variant, dev):
    """The state slot of a sequence has no direction term: with ndir = 2 both directions would share it.  The
    launchers refuse the call and enqueue nothing."""
    p = Problem(S(33, 5, 2, False, state=True), dev, seed=3)
    n0 = kh.lib().kh_launch_count()
    rc, why, _, out, h, c = p.run(variant)
    assert rc != 0, variant
    assert kh.lib().kh_launch_count() == n0
    assert bool((out.view(torch.int32) == SENTINEL).all())
    hi = p.hc_idx.to(dev)
    assert torch.equal(h[hi].cpu(), p.h0) and torch.equal(c[hi].cpu(), p.c0)      # the state was not touched


def test_tc_passes_out_of_range_refused(dev):
    p = Problem(S(33, 3, 1, False), dev, seed=4)
    for v in ("tc", "tc_x"):
        for ps in (0, 4):
            n0 = kh.lib().kh_launch_count()
            rc, _, _, out, _, _ = p.run(v, ps)
            assert rc != 0 and kh.lib().kh_launch_count() == n0
            assert bool((out.view(torch.int32) == SENTINEL).all())
