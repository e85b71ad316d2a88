"""umma_gemm_kernel (wgmma + TMA, csrc/umma_kernel.cuh) through umma::launch, element by element.

Every case is compared two ways:
  (a) with the exact float64 product of the same fp32 inputs:  |C - C64| <= tol_p (|A|.|B|)[m,n] + epilogue rounding,
      tol_p = the split's worst product error (passes 3: 5 2^-18, 2: 2^-9 + 2^-16, 1: 2^-8 + 2^-17) + fp32 accumulation;
  (b) (no LayerNorm chunk) with a float64 emulation of exactly the split terms of its pass count (tests/kernels/harness.py):
      the only difference left is fp32 accumulation, bounded by CB 2^-24 K^0.3 (|A|.|B|)[m,n] (measured: the error
      relative to |A|.|B| grows about as K^0.3 from K = 64 to 6144, slower than sqrt(K)).  Against the emulation of
      one pass fewer the same case must miss that bound by >= 20x: (b) sees a dropped split term, a misplaced tile,
      swizzle chunk or column.
The output buffer's padding, the columns beyond N and every element the problem does not own hold a NaN sentinel that
must survive; the A rows' padding beyond their channels and the B planes' padding are NaN, so only the TMA's zero fill
may stand in for them.  Each case asserts the launch plan (column tile, resident weight slab or operand ring, tile
shape, row tiles per CTA, float4 or element-wise epilogue) it is meant to exercise.

Measured on one H100 80GB HBM3: worst ratio of error to bound (a) 0.80 (ragged K = 33, passes = 2), (b) 0.48 over all
cases; the emulation of one pass fewer misses bound (b) by >= 29.6x (the closest: K = 6144).
"""
import math
from dataclasses import dataclass, field

import pytest
import torch

from kernels import harness as kh
from kernels.scaffold import SENTINEL, dev, sentinel  # noqa: F401

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TOL = {3: 5 * 2.0 ** -18, 2: 2.0 ** -9 + 2.0 ** -16, 1: 2.0 ** -8 + 2.0 ** -17}
CA = 4.0                       # fp32 accumulation term of bound (a), in units of 2^-24 sqrt(K)
CB = 5.0                       # bound (b), in units of 2^-24 K^0.3 (the measured growth of the accumulation error with K)
LN_TOL = 2.0 ** -19            # fp32 LayerNorm of the row, relative to the products (bound (a) of LN cases)
WRONG_MARGIN = 20.0


@dataclass
class G:
    name: str
    rows: int = 128            # rows_per_seq
    nseq: int = 1
    Ls: int = 0                # positions stored per sequence (default rows)
    C: int = 64                # channels of a source row (ragged K when not a multiple of 64)
    w: int = 1                 # window taps (chunk dp = 0 .. w-1)
    pos_bias: int = 0
    N: int = 64
    passes: int = 3
    ln: bool = False
    two_src: bool = False
    a1_ld: int = 0             # row stride of source 1 (floats), 0: C rounded up to 4
    n_inner: int = 0           # sequence split into (inner, outer); 0: all inner
    bias: bool = False
    prelu: bool = False        # scalar slope
    prelu_vec: bool = False
    res: bool = False
    inplace: bool = False      # R == C
    alpha: float = 1.0
    b_by_seq: bool = False
    mn_major: bool = False
    ldc_pad: int = 0
    c_inner: int = 0
    small_int: bool = False
    expect: dict = field(default_factory=dict)


def _chunks(c):
    if c.C % 64 != 0:
        assert c.w == 1 and not c.two_src
        n = (c.C + 63) // 64
        ch = [(j * 64, 0, 2 if c.ln else 0) for j in range(n)]
    else:
        cpr = c.C // 64
        ch = [((j % cpr) * 64, j // cpr, 2 if c.ln else 0) for j in range(cpr * c.w)]
        if c.two_src:
            ch += [(c0, dp, 1) for (c0, dp, _) in ch]
    return ch


def _rand(shape, g, small_int, scale=1.0):
    if small_int:
        return torch.randint(-4, 5, shape, generator=g).float()
    return (torch.rand(shape, generator=g) * 2 - 1) * (scale * math.sqrt(3.0))


def _row_offsets(c, ldc, width):
    """element offset of row (seq, pos) of C, the kernel's epilogue addressing"""
    seq = torch.arange(c.nseq).repeat_interleave(c.rows)
    pos = torch.arange(c.rows).repeat(c.nseq)
    if c.c_inner > 1:
        seq_stride = c.rows * ldc
        return (seq // c.c_inner) * seq_stride + (seq % c.c_inner) * width + pos * ldc, seq_stride, width
    return seq * (c.rows * ldc) + pos * ldc, c.rows * ldc, 0


def _epilogue(S, c, t):
    x = S * c.alpha
    if c.bias:
        x = x + t["bias"].double()
    if c.prelu or c.prelu_vec:
        sl = t["slope"].double()
        x = torch.where(x >= 0, x, x * sl)
    if c.res:
        x = x + t["R"].double()
    return x


def run_case(c, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    Ls = c.Ls or c.rows
    ld0 = (c.C + 3) // 4 * 4
    ld1 = c.a1_ld or ld0
    chunks = _chunks(c)
    nck = len(chunks)
    Kext = c.C * c.w * (2 if c.two_src else 1)
    Ktot = nck * 64
    nz = c.nseq if c.b_by_seq else 1
    M = c.nseq * c.rows
    # row padding beyond C is NaN (A) and so are the B planes' padding beyond N / K: the kernel must take the zeros of the
    # TMA's out-of-range fill, never the stored padding
    S0 = torch.full((c.nseq, Ls, ld0), float("nan"))
    S0[..., :c.C] = _rand((c.nseq, Ls, c.C), g, c.small_int)
    S1 = torch.full((c.nseq, Ls, ld1), float("nan"))
    S1[..., :c.C] = _rand((c.nseq, Ls, c.C), g, c.small_int)
    W = _rand((nz, c.N, Kext), g, c.small_int, 1.0 if c.small_int else 1.0 / math.sqrt(Kext))
    t = {"bias": _rand((c.N,), g, c.small_int), "ln_g": 1 + 0.2 * _rand((64,), g, False), "ln_b": 0.2 * _rand((64,), g, False)}
    if c.prelu:
        t["slope"] = torch.full((1,), 0.25)
    if c.prelu_vec:
        t["slope"] = 0.5 * _rand((c.N,), g, False)
    if c.res:
        t["R"] = _rand((M, c.N), g, c.small_int)

    # ---- the A rows the kernel sees, k = j*64 + c (float64 LN for the exact reference, none for the emulation)
    A = torch.zeros(M, Ktot, dtype=torch.float64)
    pos = torch.arange(c.rows)
    for j, (c0, dp, fl) in enumerate(chunks):
        src = S1 if fl & 1 else S0
        p = pos + dp + c.pos_bias
        ok = (p >= 0) & (p < Ls)
        v = torch.zeros(c.nseq, c.rows, 64, dtype=torch.float64)
        hi = min(c0 + 64, c.C)
        v[:, ok, :hi - c0] = src[:, p[ok], c0:hi].double()
        if fl & 2:
            v = kh.layer_norm64(v, t["ln_g"], t["ln_b"])
        A[:, j * 64:(j + 1) * 64] = v.reshape(M, 64)
    Wk = torch.zeros(nz, c.N, Ktot)
    Wk[..., :Kext] = W
    zrow = torch.arange(M) // c.rows if c.b_by_seq else torch.zeros(M, dtype=torch.long)

    def per_z(f):
        out = torch.empty(M, c.N, dtype=torch.float64)
        for z in range(nz):
            m = zrow == z
            out[m] = f(m, Wk[z])
        return out

    S64 = per_z(lambda m, w: A[m] @ w.double().T)
    P = per_z(lambda m, w: A[m].abs() @ w.double().abs().T)
    ref = _epilogue(S64, c, t)

    # ---- device operands
    d = {k: v.to(dev) for k, v in t.items()}
    dS0, dS1, dW = S0.to(dev), S1.to(dev), W.to(dev)
    if c.mn_major:
        ldb = (c.N + 7) // 8 * 8
        zs = Kext * ldb
    else:
        ldb = (Kext + 7) // 8 * 8
        zs = c.N * ldb
    planes = torch.full((2 * nz * zs,), float("nan"), dtype=torch.bfloat16, device=dev)
    st = kh.stream()
    for z in range(nz):
        hi_p, lo_p = planes[z * zs:], planes[nz * zs + z * zs:]
        if c.mn_major:
            rc = kh.lib().kh_split_planes(dW[z].data_ptr(), 1, Kext, Kext, c.N, ldb, hi_p.data_ptr(), lo_p.data_ptr(), st)
        else:
            rc = kh.lib().kh_split_planes(dW[z].data_ptr(), Kext, 1, c.N, Kext, ldb, hi_p.data_ptr(), lo_p.data_ptr(), st)
        assert rc == 0
    width = c.N + c.ldc_pad
    ldc = width * c.c_inner if c.c_inner > 1 else width
    off, seq_stride, inner_stride = _row_offsets(c, ldc, width)
    total = int(off.max()) + ldc + 64
    Cbuf = sentinel(total, dev)
    idx = (off[:, None] + torch.arange(c.N)[None, :]).to(dev)
    Rbuf = None
    if c.res:
        Rbuf = Cbuf if c.inplace else Cbuf.clone()
        Rbuf[idx] = d["R"]

    desc = kh.Gemm()
    for a, base, ld in ((desc.a0, dS0, ld0), (desc.a1, dS1 if c.two_src else None, ld1)):
        if base is None:
            continue
        n_inner = c.n_inner or c.nseq
        a.base, a.channels, a.n_pos, a.pos_stride = base.data_ptr(), c.C, Ls, ld
        a.n_inner, a.inner_stride = n_inner, Ls * ld
        a.n_outer, a.outer_stride = c.nseq // n_inner, n_inner * Ls * ld
    desc.n_chunks = nck
    for j, (c0, dp, fl) in enumerate(chunks):
        desc.chunk_c0[j], desc.chunk_dp[j], desc.chunk_flags[j] = c0, dp, fl
    desc.rows_per_seq, desc.nseq, desc.pos_bias = c.rows, c.nseq, c.pos_bias
    desc.b_base, desc.b_ld, desc.b_z_stride, desc.b_plane_stride = planes.data_ptr(), ldb, zs, nz * zs
    desc.b_nz, desc.b_mn_major, desc.b_by_seq = nz, int(c.mn_major), int(c.b_by_seq)
    desc.N, desc.K, desc.passes = c.N, Kext, c.passes
    desc.C, desc.R = Cbuf.data_ptr(), kh.ptr(Rbuf)
    desc.ldc, desc.c_seq_stride, desc.c_inner_stride, desc.c_inner = ldc, seq_stride, inner_stride, c.c_inner
    desc.alpha = c.alpha
    desc.bias = kh.ptr(d["bias"]) if c.bias else None
    desc.prelu = kh.ptr(d["slope"]) if c.prelu else None
    desc.prelu_vec = kh.ptr(d["slope"]) if c.prelu_vec else None
    if c.ln:
        desc.ln_g, desc.ln_b = d["ln_g"].data_ptr(), d["ln_b"].data_ptr()
    rc, plan, why = kh.gemm(desc)
    assert rc == 0, why
    torch.cuda.synchronize()
    got = Cbuf[idx].double().cpu()
    untouched = torch.ones(total, dtype=torch.bool, device=dev)
    untouched[idx.reshape(-1)] = False
    bits = Cbuf.view(torch.int32)[untouched]
    assert bool((bits == SENTINEL).all()), f"{c.name}: {int((bits != SENTINEL).sum())} elements outside the problem written"
    assert bool(torch.isfinite(got).all())

    # ---- plan expectations.  The float4 epilogue (vec_ok) is on exactly when every C / R row starts 16-byte aligned
    # (torch allocations are); with a ragged N it then mixes float4 groups and element-wise groups in one tile
    assert plan.vec_ok == int(ldc % 4 == 0 and seq_stride % 4 == 0 and inner_stride % 4 == 0), c.name
    for k, v in c.expect.items():
        have = {"tiles_per_cta": -(-plan.m_tiles // (plan.grid // plan.n_tiles_n))}.get(k, None)
        have = getattr(plan, k) if have is None else have
        assert (v(have) if callable(v) else have == v), f"{c.name}: plan {k} = {have}, expected {v}"

    # ---- (a) exact
    sl = torch.ones(1, dtype=torch.float64)
    if c.prelu or c.prelu_vec:
        sl = torch.maximum(sl, t["slope"].double().abs())
    epi = 4 * U * ((c.alpha * S64).abs() * sl + (t["bias"].double().abs() * sl if c.bias else 0)
                   + (t["R"].double().abs() if c.res else 0) + ref.abs())
    acc = U * math.sqrt(Ktot)
    bound_a = abs(c.alpha) * sl * (TOL[c.passes] + CA * acc + (LN_TOL if c.ln else 0.0)) * P + epi + 1e-30
    ratio_a = float(((got - ref).abs() / bound_a).max())
    res = {"a": ratio_a}
    if c.small_int and c.passes == 3 and not c.ln:
        assert torch.equal(got, ref), f"{c.name}: small-integer product not exact"
    # ---- (b) emulation of the split, and the sensitivity against one pass fewer
    if not c.ln:
        A32 = A.float()
        emu = {p: _epilogue(per_z(lambda m, w: kh.split_product(A32[m], w, p)), c, t)
               for p in range(max(1, c.passes - 1), c.passes + 1)}
        bound_b = abs(c.alpha) * sl * CB * U * Ktot ** 0.3 * P + epi + 1e-30
        res["b"] = float(((got - emu[c.passes]).abs() / bound_b).max())
        if c.passes > 1 and not c.small_int:          # small integers have no lo plane: every pass count agrees
            res["wrong"] = float(((got - emu[c.passes - 1]).abs() / bound_b).max())
    print(f"[{c.name}] plan BN={plan.BN} resident={plan.b_resident} nop={plan.nop} nstg={plan.nstg} vec_ok={plan.vec_ok} "
          f"tile={plan.P_TILE}x{plan.S_TILE} grid={plan.grid} m_tiles={plan.m_tiles} ratios {res}")
    assert res["a"] <= 1.0, (c.name, res)
    if "b" in res:
        assert res["b"] <= 1.0, (c.name, res)
    if "wrong" in res:
        assert res["wrong"] >= WRONG_MARGIN, (c.name, res)
    return res


CASES = [
    # the former standalone harness's correctness cases
    G("int_k64_n64_p1", rows=1000, small_int=True, passes=1),
    G("int_k64_n64_p3", rows=1000, small_int=True),
    G("rand_k64_n64_p3", rows=1000),
    G("rand_k64_n64_p1", rows=1000, passes=1),
    G("rand_k128_n256_p2_bias_res", rows=3000, C=128, N=256, passes=2, bias=True, res=True),
    G("win4_k256_n512_p2_ln", nseq=37, Ls=65, rows=62, w=4, N=512, passes=2, ln=True, bias=True),
    G("k256_n512_bias_prelu_vec", rows=3000, C=256, N=512, bias=True, prelu_vec=True),
    G("ln_k64_n256_res", rows=5000, N=256, ln=True, bias=True, res=True),
    G("ln_k64_n512", rows=2000, N=512, ln=True, bias=True),
    G("n112_k64_prelu_vec", rows=700, N=112, bias=True, prelu_vec=True),
    G("win4_short_seq_ln", nseq=37, Ls=65, rows=62, w=4, N=512, ln=True, bias=True,
      expect={"P_TILE": 62, "S_TILE": 2}),
    G("win4_halo", nseq=5, Ls=300, rows=303, C=128, w=4, pos_bias=-3, bias=True, res=True),
    G("win4_inner_outer", nseq=6, Ls=200, rows=197, w=4, N=512, ln=True, bias=True, n_inner=3,
      expect={"S_TILE": 1}),
    G("batched_k520_n300_alpha", nseq=3, Ls=300, rows=300, C=520, N=300, alpha=0.25, b_by_seq=True,
      expect={"b_resident": 0}),
    G("batched_mn_k300_n1040", nseq=3, Ls=150, rows=150, C=300, N=1040, b_by_seq=True, mn_major=True),
    G("mn_k128_n208", rows=400, C=128, N=208, bias=True, mn_major=True),
    G("two_src_ln_k128_n256", rows=1500, N=256, ln=True, bias=True, two_src=True),
    G("k4160_n256", rows=600, C=4160, N=256, bias=True, expect={"b_resident": 0, "nop": lambda v: v >= 2}),
    # two sources, the second at a record-sized row stride (the streaming state)
    G("two_src_strided_a1", rows=300, N=128, bias=True, two_src=True, a1_ld=1000),
    # flat multi-sequence tiles: 20 positions x 6 sequences per tile
    G("flat_20x6", nseq=50, rows=20, N=96, bias=True, res=True, expect={"P_TILE": 20, "S_TILE": 6}),
    # sequence index split into inner and outer, short sequences (tiles of one sequence)
    G("inner_outer_short", nseq=12, rows=40, Ls=40, N=64, n_inner=4, bias=True, expect={"S_TILE": 1}),
    # epilogue variants
    G("scalar_prelu_alpha", rows=257, N=192, alpha=-0.75, bias=True, prelu=True),
    G("scalar_prelu_ragged", rows=129, N=70, ldc_pad=2, bias=True, prelu=True, expect={"vec_ok": 1}),
    G("scalar_prelu_ragged_cold", rows=129, N=70, bias=True, prelu=True, expect={"vec_ok": 0}),
    G("residual_in_place", rows=300, N=128, bias=True, res=True, inplace=True),
    G("residual_in_place_ragged", rows=131, N=67, ldc_pad=1, res=True, inplace=True, expect={"vec_ok": 1}),
    G("residual_in_place_ragged_cold", rows=131, N=67, res=True, inplace=True, expect={"vec_ok": 0}),
    G("c_inner3", nseq=6, rows=50, N=64, bias=True, res=True, c_inner=3, ldc_pad=4, expect={"vec_ok": 1}),
    G("c_inner3_ragged", nseq=6, rows=50, N=102, bias=True, prelu_vec=True, c_inner=3, ldc_pad=2, expect={"vec_ok": 1}),
    G("c_inner3_odd", nseq=5, rows=33, N=100, bias=True, c_inner=3, ldc_pad=1, expect={"vec_ok": 0}),
    G("odd_ldc_cold_path", rows=200, N=128, ldc_pad=1, bias=True, prelu_vec=True, res=True, expect={"vec_ok": 0}),
    G("pad_ldc_vec", rows=200, N=128, ldc_pad=12, bias=True, res=True, expect={"vec_ok": 1}),
    # attention-shaped P.V: ragged K = T, MN-major B per sequence
    G("pv_T99", nseq=3, rows=99, C=99, N=260, b_by_seq=True, mn_major=True, alpha=0.5),
    G("pv_T1251", nseq=2, rows=1251, C=1251, N=130, b_by_seq=True, mn_major=True),
    # Q.K^T as the enrollment net runs it: N = T = 99 columns in rows padded to Tp = 128 (float4 epilogue, ragged N)
    G("qk_T99", nseq=2, rows=99, C=128, N=99, ldc_pad=29, b_by_seq=True, alpha=0.125, expect={"vec_ok": 1}),
    G("qk_T99_unpadded", nseq=2, rows=99, C=128, N=99, b_by_seq=True, expect={"vec_ok": 0}),
    # ragged K (TMA zero fill of the A channels and of B's k extent)
    G("ragged_k200", rows=300, C=200, N=128, bias=True),
    G("ragged_k33_p2", rows=300, C=33, N=64, passes=2),
]


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_gemm_case(case, dev):
    run_case(case, dev)


# column counts: BN = 64 / 128 and a ragged last tile, with rows padded to a multiple of 4 so the float4 epilogue is on.
# A ragged N then puts whole float4 groups and a partial group into one warp's 32 columns (N % 32 >= 4, e.g. 70, 102;
# N = 2 mod 4: 66, 130), which sends that warp to the element-wise path while the other warps of the tile stay on float4
@pytest.mark.parametrize("N", [1, 8, 63, 64, 65, 66, 70, 100, 102, 127, 128, 129, 130, 300, 1040])
def test_gemm_columns(N, dev):
    run_case(G(f"N{N}", rows=129, N=N, ldc_pad=(-N) % 4, bias=True, prelu_vec=True,
               expect={"BN": 64 if N <= 64 else 128, "vec_ok": 1}), dev, seed=N)


# ... and the same column counts with rows that are not 16-byte aligned: every column element-wise
@pytest.mark.parametrize("N", [1, 63, 65, 70, 102, 130])
def test_gemm_columns_unaligned_rows(N, dev):
    run_case(G(f"N{N}_cold", rows=129, N=N, ldc_pad=1 if N % 4 == 0 else 0, bias=True, prelu_vec=True, res=True,
               expect={"vec_ok": 0}), dev, seed=N)


# k-chunk counts on both sides of the resident-slab / operand-ring switch, for both column tiles: with bf16x3 the whole
# weight slab stays resident up to 2 chunks at BN = 128 and up to 5 at BN = 64 (test_kernels_cpu.py pins the switch)
@pytest.mark.parametrize("N", [64, 256])
@pytest.mark.parametrize("chunks", [1, 2, 3, 5, 6, 65, 96])
def test_gemm_k_chunks(chunks, N, dev):
    bn = 64 if N <= 64 else 128
    exp = {"BN": bn, "b_resident": int(chunks <= (2 if bn == 128 else 5))}
    if not exp["b_resident"]:
        exp["nop"] = lambda v: v >= 2
    run_case(G(f"K{chunks}x64_N{N}", rows=130, C=64 * chunks, N=N, bias=True, expect=exp), dev, seed=chunks)


# row counts: partial tiles, exact tiles, and 3 * 132 * 128 + 77 rows (every CTA walks several row tiles)
@pytest.mark.parametrize("rows", [1, 97, 127, 128, 129, 3 * 132 * 128 + 77])
def test_gemm_rows(rows, dev):
    exp = {"tiles_per_cta": lambda v: v >= 3} if rows > 50000 else {}
    run_case(G(f"rows{rows}", rows=rows, N=64, bias=True, res=True, expect=exp), dev, seed=rows)


@pytest.mark.parametrize("passes", [1, 2, 3])
def test_gemm_pass_counts_large_k(passes, dev):
    run_case(G(f"k1024_p{passes}", rows=256, C=1024, N=128, passes=passes), dev, seed=passes)


def test_split_planes_bit_exact(dev):
    """umma::split_planes equals the torch hi/lo split bit for bit, K-major and transposed, with row padding."""
    g = torch.Generator().manual_seed(5)
    for rows, cols, transposed in ((37, 131, False), (130, 75, True), (1, 1, False)):
        src = torch.randn(rows, cols, generator=g) * torch.logspace(-20, 20, cols)[None, :]
        src[0, 0] = 1 + 2 ** -8                           # a rounding tie
        ds = src.to(dev)
        if transposed:    # planes [cols][rows]: hi[r*ld + c] = src[c][r]
            R, Cc, rs, cs, want = cols, rows, 1, cols, src.T
        else:
            R, Cc, rs, cs, want = rows, cols, cols, 1, src
        ld = (Cc + 7) // 8 * 8
        hi = torch.zeros(R, ld, dtype=torch.bfloat16, device=dev)
        lo = torch.zeros(R, ld, dtype=torch.bfloat16, device=dev)
        assert kh.lib().kh_split_planes(ds.data_ptr(), rs, cs, R, Cc, ld, hi.data_ptr(), lo.data_ptr(), kh.stream()) == 0
        th, tl = kh.split_bf16(want.contiguous())
        assert torch.equal(hi[:, :Cc].cpu().view(torch.int16), th.view(torch.int16))
        assert torch.equal(lo[:, :Cc].cpu().view(torch.int16), tl.view(torch.int16))
        assert bool((hi[:, Cc:] == 0).all()) and bool((lo[:, Cc:] == 0).all())


def _valid_desc(dev, keep):
    A = torch.randn(256, 64, device=dev)
    planes = torch.zeros(2 * 64 * 64, dtype=torch.bfloat16, device=dev)
    C = sentinel(256 * 64, dev)
    s = torch.ones(64, device=dev)
    keep += [A, planes, C, s]
    d = kh.Gemm()
    d.a0.base, d.a0.channels, d.a0.n_pos, d.a0.pos_stride = A.data_ptr(), 64, 256, 64
    d.a0.n_inner, d.a0.n_outer = 1, 1
    d.n_chunks = 1
    d.rows_per_seq, d.nseq = 256, 1
    d.b_base, d.b_ld, d.b_z_stride, d.b_plane_stride, d.b_nz = planes.data_ptr(), 64, 64 * 64, 64 * 64, 1
    d.N, d.K, d.passes, d.C, d.ldc, d.c_seq_stride, d.alpha = 64, 64, 3, C.data_ptr(), 64, 256 * 64, 1.0
    return d, C, s


@pytest.mark.parametrize("what", ["chunks0", "chunks97", "passes0", "passes4", "unaligned_a", "unaligned_b", "both_prelu"])
def test_launch_refusals(what, dev):
    """umma::launch refuses a malformed problem with a reason and enqueues nothing."""
    keep = []
    d, C, s = _valid_desc(dev, keep)
    rc, _, why = kh.gemm(d)                               # the well-formed problem launches
    assert rc == 0, why
    torch.cuda.synchronize()
    C.view(torch.int32).fill_(SENTINEL)
    if what == "chunks0":
        d.n_chunks = 0
    elif what == "chunks97":
        d.n_chunks = 97
    elif what == "passes0":
        d.passes = 0
    elif what == "passes4":
        d.passes = 4
    elif what == "unaligned_a":
        d.a0.base += 4
    elif what == "unaligned_b":
        d.b_base += 2
    elif what == "both_prelu":
        d.prelu, d.prelu_vec = s.data_ptr(), s.data_ptr()
    n0 = kh.lib().kh_launch_count()
    rc, _, why = kh.gemm(d)
    torch.cuda.synchronize()
    assert rc != 0 and why, what
    assert kh.lib().kh_launch_count() == n0
    assert bool((C.view(torch.int32) == SENTINEL).all())
