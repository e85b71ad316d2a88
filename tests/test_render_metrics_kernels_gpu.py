"""The binaural renderer's kernels (csrc/render.cu: fir_kernel, mix_peak_kernel, mix_norm_kernel, which
l2h_render_binaural launches in that order) and the evaluation epilogue (csrc/eval_metrics.cu: eval_metrics_kernel,
l2h_eval_metrics) called through the C ABI, every output sample against an exact or float64 reference of
kernels/harness.py (pinned by test_render_metrics_cpu.py).

Renderer, exact: integer-valued sources and responses (kh.render_int_inputs) keep every partial sum an integer below
2^24, so the fp32 FIR is exact in any order, with or without FMA.  Without noise the norm (the peak), the events
(fl32(F / nf): IEEE division) and the mixture (a sequential fp32 sum from 0) must match kh.mix64's fp32 model bit for
bit, at L on and around the 256-tap chunks (1 .. 16384, also L > N), N on and around the 1024-sample tiles, below 4 and
past 16896 (the mixing kernels' grid-stride loop), S = 1 and 4, B up to 300.  With integer noise and power-of-two
scales the norm and the events stay exact and the mixture must lie within kh.mix_bound64 (the noise product may be
fused).  The peak inputs put the peak at exactly 1.0 (events unchanged), at -64 on ear 0's sample 0, below 1 and on ear
1's last sample of the last item; NULL noise, noise with a NULL scale and a NULL norm pointer are covered.  Real-valued
data (the shapes of test_render_gpu.py and a 4096-tap response) are held to the per-sample bound of one fp32 running sum,
(L + 1) 2^-24 sum |h| |x|, carried through the norm and the division.  mix_peak_kernel's fmaxf drops a NaN where
torch's max would propagate it; no case feeds one.

Metrics: channels 1-3, n from 2 to 2^20 + 3, B up to 300, SNR -30 .. +90 dB, DC offsets of 0, 1, 100 and 1000 target
RMS, silent and constant targets, embeddings of D = 1 .. 1000 that are zero, of norm 1e-9, parallel, antiparallel and
near 1e18 (kh.METRICS_CASES).  Each figure must lie within its fp32 rounding plus kh.si_snr_err64 (the double-precision
error of the centred computation, which does not grow with the DC offset) or the cosine's double rounding.  A NULL
mixture must give si_snr_i exactly 0, NULL embeddings a similarity of exactly 0.

Every input, output and scratch buffer sits between GUARD floats holding the sentinel 0x7FC0DEAD: the guards must keep
it bit for bit, and a read outside an input would carry a NaN into the comparisons.  The Python wrappers refuse shapes
the kernels would read past.
Measured on one NVIDIA H100 80GB HBM3 (700 W power limit): worst error / bound 0.33 (FIR), 0.037 (norm), 0.45 (mixture),
0.98 (SI-SNR, where the bound is mostly the fp32 rounding of the result), 0.93 (si_snr_i), 0.88 (cosine); every exact
comparison holds bit for bit.  The smallest mutant error / bound of the bounded references is 100 (the one-pass
formula at n = 2^20 + 3, DC 1000 RMS); the one-pass kernel this file replaced missed the bound by 27x to 2e5x on the
cases with a DC offset.  The file runs in about 11 s.
"""
import numpy as np
import pytest
import torch

from kernels import harness as kh
from kernels.scaffold import Guarded, dev  # noqa: F401
from lookoncetohear_b200 import _cabi
from lookoncetohear_b200.metrics import eval_metrics
from lookoncetohear_b200.render import render_binaural

pytestmark = pytest.mark.gpu


def ptr(g):
    """the device pointer of a Guarded buffer, or NULL"""
    return None if g is None else g.t.data_ptr()


def render(src, rir, noise, scale, dev, norm=True):
    """l2h_render_binaural on guarded copies -> (events, mixture, norm or None) as numpy fp32; every guard intact"""
    B, S, N = src.shape
    g_src, g_rir, g_nz, g_sc = (None if x is None else Guarded(x.shape, dev, x) for x in (src, rir, noise, scale))
    ev, mix, scratch = Guarded((B, S, 2, N), dev), Guarded((B, 2, N), dev), Guarded((B,), dev)
    nrm = Guarded((B,), dev) if norm else None
    rc = _cabi.lib().l2h_render_binaural(ptr(g_src), ptr(g_rir), ptr(g_nz), ptr(g_sc), B, S, N, rir.shape[-1], ptr(ev),
                                         ptr(mix), ptr(nrm), ptr(scratch), torch.cuda.current_stream(dev).cuda_stream)
    assert rc == 0, _cabi.lib().l2h_last_error().decode()
    torch.cuda.synchronize(dev)
    for g in (g_src, g_rir, g_nz, g_sc, ev, mix, scratch, nrm):
        assert g is None or g.ok(), "a guard lost its sentinel"
    return ev.t.cpu().numpy(), mix.t.cpu().numpy(), nrm.t.cpu().numpy() if nrm else None


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def case_id(c):
    return f"B{c[0]}_S{c[1]}_N{c[2]}_L{c[3]}{'_noise' if c[4] else ''}"


# ---- renderer -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", kh.RENDER_EXACT_CASES, ids=case_id)
def test_render_integer_data_is_exact(case, dev):
    B, S, N, L, noise, _ = case
    src, rir, nz, sc = kh.render_int_inputs(B, S, N, L, seed=B * 7919 + N * 31 + L, noise=noise)
    e_r, m_r, nf_r = kh.mix64(kh.fir64(src, rir, exact=True), nz, sc, fp32=True)
    ev, mix, nrm = render(src, rir, nz, sc, dev)
    assert same_bits(nrm, nf_r), "norm"
    bad = np.argwhere(ev.view(np.int32) != e_r.view(np.int32))
    assert bad.size == 0, ("events differ at", bad[:5], ev[tuple(bad[0])], e_r[tuple(bad[0])])
    if nz is None:
        assert same_bits(mix, m_r), "mixture"
    else:
        want = sc[:, None, None] * nz.astype(np.float64) / nf_r.astype(np.float64)[:, None, None] + e_r.astype(np.float64).sum(1)
        r = kh.worst_ratio(mix, want, kh.mix_bound64(e_r, nz, sc, nf_r))
        print(f"render {case_id(case)}: mixture error / bound {r:.3g}")
        assert r <= 1.0


def test_render_peak_placement_and_null_paths(dev):
    """peaks at exactly 1.0, at -64 on sample 0, below 1 and on ear 1's last sample of the last item; then NULL noise
    scale (noise at scale 1) and a NULL norm pointer"""
    src, rir = kh.render_peak_inputs()
    e_r, m_r, nf_r = kh.mix64(kh.fir64(src, rir, exact=True), fp32=True)
    ev, mix, nrm = render(src, rir, None, None, dev)
    assert nrm.tolist() == [1.0, 64.0, 1.0, 64.0]
    assert same_bits(nrm, nf_r) and same_bits(ev, e_r) and same_bits(mix, m_r)
    ev2, mix2, nrm2 = render(src, rir, None, None, dev, norm=False)
    assert nrm2 is None and same_bits(ev2, e_r) and same_bits(mix2, m_r)

    B, S, N, L = 3, 2, 17001, 257
    src, rir, nz, _ = kh.render_int_inputs(B, S, N, L, seed=21, noise=True)
    e_r, _, nf_r = kh.mix64(kh.fir64(src, rir, exact=True), nz, None, fp32=True)
    ev, mix, nrm = render(src, rir, nz, None, dev, norm=False)
    assert same_bits(ev, e_r)
    want = nz.astype(np.float64) / nf_r.astype(np.float64)[:, None, None] + e_r.astype(np.float64).sum(1)
    assert kh.worst_ratio(mix, want, kh.mix_bound64(e_r, nz, None, nf_r)) <= 1.0


@pytest.mark.parametrize("B,S,N,L,gain", [(2, 3, 16000, 73, 1.0), (1, 2, 5001, 1, 0.2), (2, 1, 4096, 1500, 6.0),
                                          (3, 4, 80000, 200, 3.0), (2, 2, 20000, 4096, 3.0)])
def test_render_real_data_within_bounds(B, S, N, L, gain, dev):
    """FIR: |e nf - F64| <= (L + 1) 2^-24 sum |h| |x| + 2^-24 (|F64| + that); the norm within the peak's share of those
    bounds plus (S + 2) 2^-24 of its terms; the mixture within kh.mix_bound64 of the kernel's own events and norm"""
    rng = np.random.default_rng(7 + L)
    src = (gain * 0.2 * rng.standard_normal((B, S, N))).astype(np.float32)
    rir = (rng.standard_normal((B, S, 2, L)) * np.exp(-np.arange(L) / max(L / 6, 1.0))).astype(np.float32)
    nz = (0.05 * rng.standard_normal((B, 2, N))).astype(np.float32)
    sc = rng.uniform(0.5, 2.0, B).astype(np.float32)
    ev, mix, nrm = render(src, rir, nz, sc, dev)
    F64, fb = kh.fir64(src, rir), kh.fir_bound64(src, rir)
    nf = nrm.astype(np.float64)
    eb = fb + kh.U32 * (np.abs(F64) + fb)
    r_fir = kh.worst_ratio(ev.astype(np.float64) * nf[:, None, None, None], F64, eb)
    v = sc[:, None, None] * nz.astype(np.float64) + F64.sum(1)
    vb = fb.sum(1) + (S + 2) * kh.U32 * (np.abs(sc[:, None, None] * nz.astype(np.float64)) + np.abs(F64).sum(1) + fb.sum(1))
    peak64 = np.maximum(np.abs(v).reshape(B, -1).max(1), 1.0)
    r_norm = kh.worst_ratio(nf, peak64, vb.reshape(B, -1).max(1))
    want = sc[:, None, None] * nz.astype(np.float64) / nf[:, None, None] + ev.astype(np.float64).sum(1)
    r_mix = kh.worst_ratio(mix, want, kh.mix_bound64(ev, nz, sc, nrm))
    print(f"render real B{B} S{S} N{N} L{L}: fir {r_fir:.3g} norm {r_norm:.3g} mixture {r_mix:.3g} (error / bound)")
    assert r_fir <= 1.0 and r_norm <= 1.0 and r_mix <= 1.0
    if gain >= 3.0:
        assert (nf > 1.0).any()


def test_render_refuses_shapes_the_kernels_would_read_past(dev):
    src = torch.zeros(2, 3, 100, device=dev)
    rir = torch.zeros(2, 3, 2, 16, device=dev)
    noise, sc = torch.zeros(2, 2, 100, device=dev), torch.ones(2, device=dev)
    bad = [dict(srcs=src[0]), dict(rirs=rir[:, :2]), dict(rirs=rir[..., :0]), dict(rirs=rir[:, :, :1]),
           dict(rirs=rir[..., None]), dict(noise=noise[:, :, :99]), dict(noise=noise[:1]), dict(noise=noise[:, :1]),
           dict(noise_scale=sc[:1]), dict(noise_scale=torch.ones(3, device=dev))]
    for kw in bad:
        args = dict(srcs=src, rirs=rir, noise=noise, noise_scale=sc) | kw
        with pytest.raises(ValueError):
            render_binaural(args["srcs"], args["rirs"], args["noise"], args["noise_scale"])
    render_binaural(src, rir, noise, sc)                   # the well-formed call still runs
    torch.cuda.synchronize(dev)


# ---- evaluation metrics ---------------------------------------------------------------------------------------------
def metrics(est, tgt, mix, emb, emb_gt, dev):
    """l2h_eval_metrics on guarded copies -> [B, 3] numpy fp32; every guard intact"""
    B, C, n = est.shape
    ins = {k: Guarded(v.shape, dev, v) for k, v in dict(est=est, tgt=tgt, mix=mix, emb=emb, emb_gt=emb_gt).items() if v is not None}
    out = Guarded((B, 3), dev)
    p = lambda k: ptr(ins.get(k))
    rc = _cabi.lib().l2h_eval_metrics(p("est"), p("tgt"), p("mix"), B, C, n, p("emb"), p("emb_gt"),
                                      emb.shape[1] if emb is not None else 0, ptr(out), torch.cuda.current_stream(dev).cuda_stream)
    assert rc == 0, _cabi.lib().l2h_last_error().decode()
    torch.cuda.synchronize(dev)
    for g in list(ins.values()) + [out]:
        assert g.ok(), "a guard lost its sentinel"
    return out.t.cpu().numpy()


@pytest.mark.parametrize("case", kh.METRICS_CASES, ids=lambda c: c[0])
def test_metrics_within_bounds(case, dev):
    name, args, _ = case
    est, tgt, mix, emb, emb_gt = kh.metrics_inputs(**args)
    got = metrics(est, tgt, mix, emb, emb_gt, dev)
    ref, bound = kh.eval_metrics64(est, tgt, mix, emb, emb_gt)
    if mix is None:
        assert (got[:, 1] == 0).all() and not np.signbit(got[:, 1]).any()
    if emb is None:
        assert (got[:, 2] == 0).all() and not np.signbit(got[:, 2]).any()
    r = [kh.worst_ratio(got[:, k], ref[:, k], bound[:, k]) for k in range(3)]
    print(f"metrics {name}: error / bound sisnr {r[0]:.3g} si_snr_i {r[1]:.3g} cosine {r[2]:.3g}")
    assert max(r) <= 1.0, (r, got, ref)


def test_metrics_refuses_shapes_the_kernel_would_read_past(dev):
    out, tgt, mix = (torch.zeros(3, 2, 500, device=dev) for _ in range(3))
    emb = torch.ones(3, 1, 256, device=dev)
    bad = [dict(mixture=mix[:, :1]), dict(mixture=mix[:2]), dict(mixture=mix[..., :499]), dict(embedding_gt=None),
           dict(embedding=None), dict(embedding_gt=emb[..., :255]), dict(embedding=emb[..., :255]),
           dict(embedding_gt=torch.ones(3, 300, device=dev)), dict(embedding=emb[:2], embedding_gt=emb[:2]),
           dict(embedding=emb[..., :0], embedding_gt=emb[..., :0])]
    for kw in bad:
        args = dict(mixture=mix, embedding=emb, embedding_gt=emb) | kw
        with pytest.raises(ValueError):
            eval_metrics(out, tgt, args["mixture"], args["embedding"], args["embedding_gt"])
    m = eval_metrics(out, tgt, mix, emb, emb)              # the well-formed call still runs; [B, 1, D] is [B, D]
    assert m.shape == (3, 3)
    assert eval_metrics(out, tgt).shape == (3, 3)
