"""The float64 references of the renderer and evaluation-metrics kernels (kernels/harness.py: fir64, mix64, si_snr64,
cos64, eval_metrics64), pinned to the reference's own calls and to the restated oracle, and the cases
test_render_metrics_kernels_gpu.py runs: the integer-valued render inputs keep every partial sum exact in fp32, the
peak inputs peak where they say, and every mutant a case names misses it -- the exact comparison for the renderer, the
bound by >= 10x for the bounded checks.  No device needed."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from scipy.signal import convolve

from kernels import harness as kh
from oracle import restate as rs
from test_render_gpu import _reference

SENSITIVITY = 10.0


def _real_inputs(B, S, N, L, seed):
    rng = np.random.default_rng(seed)
    srcs = (0.4 * rng.standard_normal((B, S, N))).astype(np.float32)
    rirs = (rng.standard_normal((B, S, 2, L)) * np.exp(-np.arange(L) / max(L / 6, 1.0))).astype(np.float32)
    return srcs, rirs, (0.05 * rng.standard_normal((B, 2, N))).astype(np.float32), rng.uniform(0.5, 2.0, B).astype(np.float32)


@pytest.mark.parametrize("B,S,N,L", [(2, 3, 1600, 73), (1, 2, 501, 1), (2, 1, 409, 1500), (1, 1, 3000, 257)])
def test_fir64_is_the_references_convolve(B, S, N, L):
    srcs, rirs, _, _ = _real_inputs(B, S, N, L, 3 + L)
    y = kh.fir64(srcs, rirs)
    for b in range(B):
        for s in range(S):
            for ear in range(2):
                want = convolve(srcs[b, s].astype(np.float64), rirs[b, s, ear].astype(np.float64))[:N]
                assert np.abs(y[b, s, ear] - want).max() <= 1e-12 * max(1.0, np.abs(want).max())
    si, ri, _, _ = kh.render_int_inputs(B, S, N, L, 5)
    ye = kh.fir64(si, ri, exact=True)
    assert np.array_equal(ye, np.stack([[[np.convolve(si[b, s].astype(np.float64), ri[b, s, e].astype(np.float64))[:N]
                                          for e in range(2)] for s in range(S)] for b in range(B)]))
    assert not np.signbit(ye[ye == 0]).any()


@pytest.mark.parametrize("B,S,N,L,noise", [(2, 3, 1600, 73, True), (1, 2, 501, 1, False), (3, 4, 2000, 20, True)])
def test_mix64_is_the_references_mixing(B, S, N, L, noise):
    srcs, rirs, nz, sc = _real_inputs(B, S, N, L, 9)
    srcs *= 6.0                                                    # some items above 1, so the division is exercised
    if not noise:
        nz, sc = np.zeros_like(nz), np.ones_like(sc)
    e, m, nf = kh.mix64(kh.fir64(srcs, rirs), nz, sc)
    e_r, m_r, nf_r = _reference(srcs, rirs, nz, sc)
    assert np.abs(e - e_r).max() <= 1e-12 and np.abs(m - m_r).max() <= 1e-12 and np.abs(nf - nf_r).max() <= 1e-12 * nf_r.max()
    assert (nf_r > 1).any()


def test_si_snr64_is_the_oracle():
    g = torch.Generator().manual_seed(2)
    t = 0.1 * torch.randn(3, 2, 5000, generator=g, dtype=torch.float64)
    for dc in (0.0, 0.3, 100.0):
        p = dc + 1.7 * t + 1e-3 * torch.randn(3, 2, 5000, generator=g, dtype=torch.float64)
        assert np.abs(kh.si_snr64(p.numpy(), t.numpy()) - rs.si_sdr(p, t).numpy()).max() <= 1e-12 * 100
    z = torch.zeros(1, 1, 64, dtype=torch.float64)
    assert np.abs(kh.si_snr64(t[:1, :1, :64].numpy(), z.numpy()) - rs.si_sdr(t[:1, :1, :64], z).numpy()).max() <= 1e-12


def test_cos64_is_torch_cosine_similarity():
    est, tgt, mix, emb, emb_gt = kh.metrics_inputs(len(kh.EMB_KINDS) * 2, 1, 2, 0, D=257)
    want = F.cosine_similarity(torch.from_numpy(emb).double(), torch.from_numpy(emb_gt).double(), dim=-1).numpy()
    assert np.abs(kh.cos64(emb, emb_gt) - want).max() <= 1e-12
    assert kh.cos64(emb, emb_gt)[kh.EMB_KINDS.index("zero")] == 0.0


def _int_case(case):
    B, S, N, L, noise, names = case
    src, rir, nz, sc = kh.render_int_inputs(B, S, N, L, seed=B * 7919 + N * 31 + L, noise=noise)
    return src, rir, nz, sc, names


@pytest.mark.parametrize("case", kh.RENDER_EXACT_CASES, ids=lambda c: f"B{c[0]}_S{c[1]}_N{c[2]}_L{c[3]}{'_noise' if c[4] else ''}")
def test_render_exact_cases_are_exact_and_mutants_miss(case):
    """every partial sum is an integer (noise: a multiple of 2^-3) below 2^24 (2^21), so the kernels' fp32 sums are
    exact in any order; each named mutant changes the events, the norm or (noise_unnormalised) misses the mixture bound
    by >= 10x"""
    src, rir, nz, sc, names = _int_case(case)
    absF = kh.fir64(np.abs(src), np.abs(rir), exact=True)
    peak_terms = absF.sum(1) + (0 if nz is None else np.abs(sc[:, None, None] * nz))
    assert absF.max() < 2 ** 24 and peak_terms.max() < (2 ** 21 if nz is not None else 2 ** 24)
    F_ = kh.fir64(src, rir, exact=True)
    e, m, nf = kh.mix64(F_, nz, sc, fp32=True)
    for mut in names:
        if mut in kh.FIR_MUTANTS:
            e2, _, nf2 = kh.mix64(kh.fir64(src, rir, exact=True, mutant=mut), nz, sc, fp32=True)
            assert not (np.array_equal(e2, e) and np.array_equal(nf2, nf)), mut
        else:
            _, m2, _ = kh.mix64(F_, nz, sc, fp32=True, mutant=mut)
            want = sc[:, None, None] * nz.astype(np.float64) / nf[:, None, None] + e.astype(np.float64).sum(1)
            assert (np.abs(m2 - want) / kh.mix_bound64(e, nz, sc, nf)).max() >= SENSITIVITY, mut


def test_render_peak_inputs_peak_where_they_say():
    src, rir = kh.render_peak_inputs()
    e, m, nf = kh.mix64(kh.fir64(src, rir, exact=True), fp32=True)
    assert nf.tolist() == [1.0, 64.0, 1.0, 64.0]
    assert m[1, 0, 0] == -1.0 and m[3, 1, -1] == 1.0 and np.abs(m[0]).max() == 1.0 and 0 < np.abs(m[2]).max() < 1.0
    assert np.array_equal(e[[0, 2]], kh.fir64(src, rir, exact=True)[[0, 2]].astype(np.float32))
    _, _, nf2 = kh.mix64(kh.fir64(src, rir, exact=True), fp32=True, mutant="peak_ear0")
    assert nf2[3] != nf[3]


@pytest.mark.parametrize("case", kh.METRICS_CASES, ids=lambda c: c[0])
def test_metrics_mutants_miss_the_bound(case):
    _, args, names = case
    est, tgt, mix, emb, emb_gt = kh.metrics_inputs(**args)
    ref, bound = kh.eval_metrics64(est, tgt, mix, emb, emb_gt)
    assert np.isfinite(ref).all() and (bound[:, 0] > 0).all()
    assert (bound[:, 1] > 0).all() == (mix is not None) and (bound[:, 2] > 0).any() == (emb is not None)
    for mut in names:
        got, _ = kh.eval_metrics64(est, tgt, mix, emb, emb_gt, mutant=mut)
        assert kh.worst_ratio(got, ref, bound) >= SENSITIVITY, mut
