"""The kernel harness library (tests/kernels/) and the float64 references the kernel-level GPU tests
(test_umma_gemm_gpu.py, test_lstm_kernels_gpu.py) rely on.  No device needed."""
import ctypes

import torch

from kernels import harness as kh


def test_harness_builds_and_exports():
    L = kh.lib()
    for s in kh.SYMBOLS:
        assert hasattr(L, s), s


def test_ctypes_mirrors_match_the_c_structs():
    L = kh.lib()
    for fn, cls in kh.MIRRORS.items():
        assert getattr(L, fn)() == ctypes.sizeof(cls), (fn, cls.__name__)


def _plan(n_chunks, N, passes=3, ldc=None):
    d = kh.Gemm()
    d.a0.channels, d.a0.n_pos, d.a0.n_inner, d.a0.n_outer = 64 * n_chunks, 130, 1, 1
    d.n_chunks, d.rows_per_seq, d.nseq, d.N, d.K, d.passes = n_chunks, 130, 1, N, 64 * n_chunks, passes
    d.ldc = N if ldc is None else ldc
    d.c_seq_stride = 130 * d.ldc
    return kh.gemm_plan(d)


def test_gemm_plan_resident_switch():
    """umma::launch's own plan (no device needed): with bf16x3 the weight slab stays resident in shared memory up to
    2 k-chunks at BN = 128 and up to 5 at BN = 64; beyond, A and B stream through a ring of at least two operand slots.
    test_umma_gemm_gpu.py runs k-chunk counts on both sides of both switch points."""
    for N, bn, last in ((256, 128, 2), (64, 64, 5)):
        for k in (1, last, last + 1, 65, 96):
            p = _plan(k, N)
            assert p is not None and p.BN == bn, (N, k)
            assert p.b_resident == int(k <= last), (N, k, p.b_resident)
            if not p.b_resident:
                assert p.nop >= 2, (N, k, p.nop)
    assert _plan(97, 64) is None and _plan(0, 64) is None and _plan(1, 64, passes=4) is None


def test_gemm_plan_vec_ok():
    """the float4 epilogue is chosen from the row alignment alone: a ragged N with padded rows keeps it"""
    assert _plan(1, 70, ldc=72).vec_ok == 1
    assert _plan(1, 70).vec_ok == 0
    assert _plan(1, 64).vec_ok == 1


def test_lstm_reference_equals_torch_lstm():
    """lstm_ref over the packed gate layout (columns j*4+q) equals torch.nn.LSTM in float64, both directions, with a
    carried (h0, c0) on the forward direction."""
    torch.manual_seed(0)
    nseq, L, F = 5, 7, 16
    for reverse in (False, True):
        m = torch.nn.LSTM(F, 64, batch_first=True).double()
        x = torch.randn(nseq, L, F, dtype=torch.float64)
        h0 = 0.5 * torch.randn(1, nseq, 64, dtype=torch.float64)
        c0 = 0.5 * torch.randn(1, nseq, 64, dtype=torch.float64)
        # lstm_ref carries state on direction 0 only: the reverse direction starts from zero
        with torch.no_grad():
            if reverse:
                want, (hn, cn) = m(x.flip(1))
                want = want.flip(1)
            else:
                want, (hn, cn) = m(x, (h0, c0))
        w_ih, w_hh = m.weight_ih_l0.detach(), m.weight_hh_l0.detach()
        b = (m.bias_ih_l0 + m.bias_hh_l0).detach()
        gx = (x.reshape(-1, F) @ w_ih.T + b)[:, _perm()]           # rows seq*L + step
        d = 1 if reverse else 0
        gx2 = torch.zeros(nseq * L, 512, dtype=torch.float64)
        gx2[:, d * 256:(d + 1) * 256] = gx
        whh = torch.zeros(2, 256, 64, dtype=torch.float64)
        whh[d] = kh.packed_from_torch(w_hh)
        hs, fin = kh.lstm_ref(gx2, whh, nseq, L, d + 1, lambda s, t: s * L + t,
                              h0=None if reverse else h0[0], c0=None if reverse else c0[0])
        got = hs[d].transpose(0, 1)                                    # [nseq][L][64]
        assert torch.allclose(got, want, rtol=0, atol=1e-12)
        assert torch.allclose(fin[d][0], hn[0], rtol=0, atol=1e-12)
        assert torch.allclose(fin[d][1], cn[0], rtol=0, atol=1e-12)


def _perm():
    return torch.tensor([q * 64 + j for j in range(64) for q in range(4)])


def test_packed_from_torch_is_the_gate_permutation():
    w = torch.arange(256 * 3, dtype=torch.float64).view(256, 3)
    assert torch.equal(kh.packed_from_torch(w), w[_perm()])


def test_bf16_split_reproduces_fp32():
    """hi = rn_bf16(x) (torch rounds to nearest even, like __float2bfloat16_rn), lo = rn_bf16(x - hi): hi + lo equals x
    to 2^-17 relative (lo carries 8 more significant bits), and |lo| <= 2^-9 |x|."""
    torch.manual_seed(1)
    x = torch.cat([torch.randn(100000), torch.randn(1000) * 1e-20, torch.randn(1000) * 1e20,
                   torch.tensor([1.0, -1.0, 0.0, 1 + 2 ** -8, 1 + 3 * 2 ** -8])])
    hi, lo = kh.split_bf16(x)
    r = hi.double() + lo.double()
    nz = x != 0
    rel = ((r - x.double()).abs() / x.double().abs())[nz]
    assert float(rel.max()) <= 2.0 ** -17
    assert bool(((lo.double().abs() <= 2.0 ** -8 * x.double().abs()) | ~nz).all())
    # round to nearest EVEN at ties (bf16 ulp at 1 is 2^-7): 1 + 2^-8 -> 1, 1 + 3 * 2^-8 -> 1 + 2^-6
    assert float(hi[-2]) == 1.0 and float(hi[-1]) == 1.0 + 2 ** -6


def test_split_product_passes():
    """passes = 3 is exact on small-integer inputs (every operand is its own hi); on general inputs each pass count is
    within its documented scale of the exact product and passes = 3 < 2 < 1 in error."""
    torch.manual_seed(2)
    a = torch.randint(-4, 5, (33, 200)).float()
    b = torch.randint(-4, 5, (17, 200)).float()
    exact = a.double() @ b.double().T
    assert torch.equal(kh.split_product(a, b, 3), exact)
    a, b = torch.randn(64, 256), torch.randn(48, 256)
    exact = a.double() @ b.double().T
    P = a.double().abs() @ b.double().abs().T
    err = {p: float(((kh.split_product(a, b, p) - exact).abs() / P).max()) for p in (1, 2, 3)}
    assert err[3] <= 3 * 2.0 ** -17 and err[2] <= 2.0 ** -8 and err[1] <= 2.0 ** -7
    assert err[3] < err[2] / 20 and err[2] < err[1]
