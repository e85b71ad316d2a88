"""The separator's CUDA-core rows GEMM (csrc/gemm.cuh) launched directly through launch_rows_gemm, against float64.

The four dense layers of a block run as this GEMM whenever a call has at most 2048 rows: LayerNorm -> W_ih (K 64,
N 512 intra and N 256 inter) and the two Linears with the residual added in place (K 128 with lda 128, K 64).  They run
here at M in {97, 194, 1261, 2047, 2048}: one streaming frame of one stream up to the last size of the 16-row tile, with
ragged last tiles.  The wavefront pipeline's W_ih GEMM over a batch of hops reads windowed A rows and writes strided C
rows, a hop slot apart, under option pipeline_gemm_shape 0 / 1 / 2; it runs at M = 388 (4 hops of one stream) and
M = 2328 (4 hops of 6 streams) in every shape, and each launch reports which kernel ran: every reachable form
(rows_gemm_kernel<16,64,2,4>, rows_gemm_kernel<64,64,4,4>, rows_gemm_big_kernel<128>) is launched.

The reference (kernels/harness.py: rows_gemm64) is LayerNorm with biased variance and eps inside the sqrt, x W + b, then
the residual.  Each value has its own bound: u = 2^-24, u sqrt(n) sum |terms| for the n-term sum, the LayerNorm's
rounding carried through |g| / sigma.  The LayerNorm problems include a constant row, whose normalised row is exactly
ln_b (so its output is bit for bit that of a launch without the LayerNorm on the row ln_b), a row of mean 10^3 and unit
spread, and a row of spread 0.01 (where eps inside or outside the sqrt differs).  Every float the kernel must not write
holds the NaN sentinel 0x7FC0DEAD and must survive: rows past M, the guard floats after C, the gaps between hop slots;
every float it must not read is NaN too: A's padding columns (lda > K) and the hop slots' gaps.  All forms accumulate k in
order, then add the bias, then the residual, so every form gives the same bits on the same problem.

Mutants (each must miss the bound by >= 10x): the LayerNorm's variance unbiased, eps outside the sqrt, W^T's memory read
as W, the bias or the residual dropped, the rows offset by one 16-row tile.
Measured on one NVIDIA H100 80GB HBM3 (700 W power limit): worst error / bound 0.17 (LayerNorm -> W_ih, N 512 and
N 256), 0.38 (Linear K 128), 0.55 (Linear K 64), 0.19 (pipeline forms); the smallest mutant error / bound is 721 (eps
outside the sqrt, LayerNorm -> W_ih N 256).
"""
import math

import pytest
import torch

from kernels import harness as kh

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC0DEAD
SENSITIVITY = 10.0
GUARD = 1024
TILE = 16
REACHABLE = {"tile16x64", "tile64x64", "big128"}
WORST, MUTANT_MIN = {}, {}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    kh.lib()
    return torch.device("cuda", 0)


def sentinel(n, dev):
    return torch.full((n,), SENTINEL, dtype=torch.int32, device=dev).view(torch.float32)


def bits(t):
    return t.contiguous().view(torch.int32)


# kind -> (K, N, lda, LayerNorm, residual in place): the engine's four dense layers (sep_engine.cu: Chain::dense); the
# K 64 Linear takes lda 72 here so that its 8 padding columns (NaN) show any read past K
KINDS = {"ih_intra": (64, 512, 64, True, False), "ih_inter": (64, 256, 64, True, False),
         "lin_intra": (128, 64, 128, False, True), "lin_inter": (64, 64, 72, False, True)}


class Problem:
    def __init__(self, kind, M, seed, a_off=None, c_off=None, n_floats=None):
        """A [M][K] and, for the residual layers, R [M][N]; a_off / c_off: the rows' offsets in one buffer of n_floats
        (None: A and C in buffers of their own at M * lda / M * N)"""
        K, N, lda, ln, res = KINDS[kind]
        g = torch.Generator().manual_seed(seed)
        self.kind, self.M, self.K, self.N, self.lda, self.res = kind, M, K, N, lda, res
        self.A = torch.randn(M, K, generator=g)
        self.Wt = torch.randn(K, N, generator=g) / math.sqrt(K)
        self.bias = 0.3 * torch.randn(N, generator=g)
        self.ln = (1 + 0.2 * torch.randn(K, generator=g), 0.2 * torch.randn(K, generator=g)) if ln else None
        self.R = torch.randn(M, N, generator=g) if res else None
        if ln:
            self.A[0] = 0.75                                              # LN(row) = ln_b exactly
            self.A[1] = 0.5 + 0.01 * torch.randn(K, generator=g)          # spread 0.01
            self.A[M - 1] = 1000.0 + torch.randn(K, generator=g)          # mean 10^3, unit spread
        self.a_off = kh.rows_offsets(M, lda) if a_off is None else a_off
        self.c_off = kh.rows_offsets(M, N) if c_off is None else c_off
        self.shared = n_floats is not None
        self.n_a = n_floats if self.shared else M * lda
        self.n_c = n_floats if self.shared else M * N

    def ref(self, **mutant):
        return kh.rows_gemm64(self.A, self.Wt, self.bias, self.ln, self.R, **mutant)

    def run(self, dev, shape=0, windowed=None, ln=True, A=None):
        """one launch (ln=False: without the LayerNorm; A: other rows); asserts that nothing outside C's rows changed
        and that no NaN was read; returns (the form launched, C's rows [M][N])"""
        A = self.A if A is None else A
        abuf = sentinel(self.n_a + GUARD, dev)
        ai = (self.a_off[:, None] + torch.arange(self.K)[None, :]).to(dev)
        abuf[ai] = A.to(dev)
        cbuf = abuf if self.shared else sentinel(self.n_c + GUARD, dev)
        ci = (self.c_off[:, None] + torch.arange(self.N)[None, :]).to(dev)
        if self.res:
            cbuf[ci] = self.R.to(dev)
        before = cbuf.clone()
        abefore = abuf.clone()
        w = {k: v.to(dev) for k, v in (("Wt", self.Wt), ("bias", self.bias))}
        d = kh.RowsGemm()
        d.A, d.lda, d.Wt, d.bias, d.C, d.ldc = abuf.data_ptr(), self.lda, w["Wt"].data_ptr(), w["bias"].data_ptr(), \
            cbuf.data_ptr(), self.N
        if windowed is not None:
            rows, c_base, slot = windowed
            d.a_rows_per_seq, d.a_seq_stride = rows, slot
            d.c_rows_per_seq, d.c_seq_stride = rows, slot
            d.C = cbuf.data_ptr() + 4 * c_base
        if self.res:
            d.R = d.C
        lnd = None
        if self.ln is not None and ln:
            lnd = [t.to(dev) for t in self.ln]
            d.ln_g, d.ln_b = lnd[0].data_ptr(), lnd[1].data_ptr()
        d.M, d.N, d.K = self.M, self.N, self.K
        rc, form = kh.rows_gemm(d, shape)
        torch.cuda.synchronize()
        assert rc == 0, (self.kind, self.M, shape, rc)
        got = cbuf[ci].clone()
        exp = before.clone()
        exp[ci] = got
        assert torch.equal(bits(cbuf), bits(exp)), f"{self.kind} M={self.M} shape {shape}: C written outside its rows"
        if not self.shared:
            assert torch.equal(bits(abuf), bits(abefore)), "A written"
        assert bool(torch.isfinite(got).all()), "a NaN sentinel was read"
        return form, got


def ratio(got, ref, bound):
    return float(((got.double().cpu() - ref).abs() / bound).max())


def check(key, got, p):
    """got within the reference's per-element bound; every mutant misses it by >= SENSITIVITY x"""
    ref, bound = p.ref()
    r = ratio(got, ref, bound)
    WORST[key] = max(WORST.get(key, 0.0), r)
    names = ["no_transpose", "drop_bias"] + (["unbiased", "eps_outside"] if p.ln is not None else []) + \
            (["drop_residual"] if p.res else [])
    mut = {m: ratio(got, p.ref(**{m: True})[0], bound) for m in names}
    mut["tile_offset"] = ratio(got[TILE:], ref[:-TILE], bound[TILE:])
    MUTANT_MIN[key] = min(MUTANT_MIN.get(key, math.inf), min(mut.values()))
    print(f"[{key}] err / bound {r:.3f}; mutants / bound: " + ", ".join(f"{m} {v:.0f}" for m, v in mut.items()))
    assert r <= 1.0, (key, r)
    for m, v in mut.items():
        assert v >= SENSITIVITY, (key, m, v)


@pytest.mark.parametrize("M", [97, 194, 1261, 2047, 2048])
@pytest.mark.parametrize("kind", list(KINDS))
def test_dense_layers(kind, M, dev):
    p = Problem(kind, M, seed=M + len(kind))
    assert kh.rows_gemm_form(M, p.N, p.K) == "tile16x64"
    form, got = p.run(dev)
    assert form == "tile16x64"
    check(kind, got, p)
    if p.ln is not None:
        # the constant row's normalised row is exactly ln_b: bit for bit the launch without LayerNorm on ln_b
        A2 = p.A.clone()
        A2[0] = p.ln[1]
        _, got2 = p.run(dev, ln=False, A=A2)
        assert torch.equal(bits(got[0]), bits(got2[0]))


def _pipeline_problem(B, hops, seed):
    """the pipelined W_ih GEMM of `hops` hop slots of B streams: hop j's X rows at j * slot, its GX rows at
    j * slot + c_base (slot: a multiple of one GX row, as the engine's workspace)"""
    rows = B * kh.NF
    c_base = rows * 64 + 64
    slot = -(-(c_base + rows * 512 + 64) // 512) * 512
    M = rows * hops
    p = Problem("ih_intra", M, seed, a_off=kh.rows_offsets(M, 64, rows, slot),
                c_off=c_base + kh.rows_offsets(M, 512, rows, slot), n_floats=(hops + 1) * slot)
    return p, (rows, c_base, slot)


@pytest.mark.parametrize("B,hops", [(1, 4), (6, 4)], ids=["M388", "M2328"])
def test_pipeline_windowed_forms(B, hops, dev):
    """every pipeline_gemm_shape on windowed A / strided C; all forms give the same bits"""
    p, win = _pipeline_problem(B, hops, seed=B * 10 + hops)
    outs, forms = {}, set()
    for shape in (0, 1, 2):
        form, got = p.run(dev, shape, windowed=win)
        assert form == kh.rows_gemm_form(p.M, p.N, p.K, shape) and form in REACHABLE, (shape, form)
        forms.add(form)
        check(f"pipeline {form}", got, p)
        outs[shape] = got
    assert forms == ({"tile16x64", "tile64x64", "big128"} if p.M <= 2048 else {"tile64x64", "big128"})
    for shape in (1, 2):
        assert torch.equal(bits(outs[shape]), bits(outs[0])), f"shape {shape} differs from shape 0"


def test_forms_agree_on_plain_rows(dev):
    """the plain (not windowed) layout: the 16-row tile, the 64x64 tile and the persistent form, bit for bit"""
    p = Problem("ih_inter", 1261, seed=5)
    outs = {s: p.run(dev, s) for s in (0, 1, 2)}
    assert {f for f, _ in outs.values()} == {"tile16x64", "tile64x64", "big128"}
    for s in (1, 2):
        assert torch.equal(bits(outs[s][1]), bits(outs[0][1])), s


def test_summary(dev):
    print("worst error / bound: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(WORST.items())))
    print("smallest mutant error / bound: " + ", ".join(f"{k} {v:.0f}" for k, v in sorted(MUTANT_MIN.items())))
    assert all(v <= 1.0 for v in WORST.values()) and all(v >= SENSITIVITY for v in MUTANT_MIN.values())
