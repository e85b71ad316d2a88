"""GPU resampler (l2h_resample, lookoncetohear_b200.resample) against the float64 restatement oracle/resample.py, which
tests/test_resample_cpu.py pins to torchaudio.functional.resample; and render_binaural with responses at other rates."""
import numpy as np
import pytest
import torch

from lookoncetohear_b200 import resample
from lookoncetohear_b200.render import render_binaural
from oracle import resample as ors

pytestmark = pytest.mark.gpu

LENGTHS = [1, 7, 200, 2000, 80000]


def _check_rows(y, x, rates, new):
    """Every row of y: the oracle's resampled row, then zeros; rel-L2 and max-abs within 1e-5."""
    y = y.cpu().numpy().astype(np.float64)
    x = x.cpu().numpy().astype(np.float64)
    assert y.shape[-1] == max(ors.output_length(x.shape[-1], r, new) for r in rates)
    for r, (yr, xr) in enumerate(zip(y, x)):
        ref = ors.resample(xr, rates[r], new)
        got = yr[:ref.size]
        assert not yr[ref.size:].any(), f"row {r}: padding is not zero"
        scale = max(np.abs(ref).max(), 1e-30)
        assert np.linalg.norm(got - ref) <= 1e-5 * max(np.linalg.norm(ref), 1e-30), (r, rates[r])
        assert np.abs(got - ref).max() <= 1e-5 * scale, (r, rates[r])


@pytest.mark.parametrize("n", LENGTHS)
def test_mixed_rates_to_16k_match_oracle(n):
    rates = [44100, 48000, 8000, 22050, 16000, 44100]
    g = torch.Generator().manual_seed(n)
    x = torch.randn(len(rates), n, generator=g)
    y = resample(x.cuda(), rates, 16000)
    torch.cuda.synchronize()
    _check_rows(y, x, rates, 16000)
    assert torch.equal(y[4, :n].cpu(), x[4])                                  # orig == new: the row, bit for bit


@pytest.mark.parametrize("n", LENGTHS)
def test_16k_to_8k_matches_oracle(n):
    x = torch.randn(2, n, generator=torch.Generator().manual_seed(100 + n))
    y = resample(x.cuda(), 16000, 8000)
    assert y.shape == (2, ors.output_length(n, 16000, 8000))
    _check_rows(y, x, [16000, 16000], 8000)


def test_identity_returns_the_input():
    x = torch.randn(3, 2, 1001, device="cuda")
    assert resample(x, 16000, 16000) is x
    assert resample(x, torch.full((3, 2), 16000), 16000) is x


def test_leading_dims_per_item_rates_and_dtype():
    x = torch.randn(3, 2, 2, 555, dtype=torch.float64, generator=torch.Generator().manual_seed(5))
    per_item = torch.tensor([44100, 48000, 16000]).view(3, 1, 1)
    y = resample(x.cuda(), per_item, 16000)
    assert y.dtype == torch.float64 and y.shape == (3, 2, 2, 555)
    rates = per_item.expand(3, 2, 2).reshape(-1).tolist()
    _check_rows(y.reshape(12, -1), x.float().reshape(12, -1), rates, 16000)
    xs = torch.randn(4, 1200, device="cuda")[:, ::3]                            # strided rows
    _check_rows(resample(xs, 48000, 16000), xs, [48000] * 4, 16000)


def test_many_rows_and_many_rate_changes():
    """More distinct rates (16) and rate changes (768) than one launch takes, and more rows than one grid column
    (65535)."""
    distinct = [8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 7350, 9600, 14700, 19200,
                29400, 37800, 50000, 64000, 176400]
    alt = [distinct[(r * 7) % len(distinct)] for r in range(2000)]
    x = torch.randn(2000, 200, generator=torch.Generator().manual_seed(3))
    _check_rows(resample(x.cuda(), alt, 16000), x, alt, 16000)
    rows = 70000
    rates = [22050] * 40000 + [8000] * (rows - 40000)
    x = torch.randn(rows, 7, generator=torch.Generator().manual_seed(4))
    y = resample(x.cuda(), rates, 16000).cpu().double().numpy()
    xd = x.double().numpy()
    for rate, sl in ((22050, slice(0, 40000)), (8000, slice(40000, rows))):
        ref = ors.resample(xd[sl], rate, 16000)
        got = y[sl, :ref.shape[-1]]
        assert not y[sl, ref.shape[-1]:].any()
        assert np.linalg.norm(got - ref) <= 1e-5 * np.linalg.norm(ref)


def test_render_resamples_responses_per_item():
    rng = np.random.default_rng(11)
    B, S, N, L = 3, 2, 16000, 551
    rir_sr = [44100, 48000, 22050]
    srcs = (0.3 * rng.standard_normal((B, S, N))).astype(np.float32)
    rirs = (rng.standard_normal((B, S, 2, L)) * np.exp(-np.arange(L) / 90.0)).astype(np.float32)
    noise = (0.05 * rng.standard_normal((B, 2, N))).astype(np.float32)
    nscale = rng.uniform(0.5, 2.0, B).astype(np.float32)
    cu = lambda a: torch.from_numpy(a).cuda()
    got = render_binaural(cu(srcs), cu(rirs), cu(noise), cu(nscale), rir_sr=rir_sr, sr=16000)
    lens = [ors.output_length(L, r, 16000) for r in rir_sr]
    pre = np.zeros((B, S, 2, max(lens)), np.float32)                            # the oracle's responses, zero-padded
    for b in range(B):
        pre[b, ..., :lens[b]] = ors.resample(rirs[b], rir_sr[b], 16000)
    want = render_binaural(cu(srcs), cu(pre), cu(noise), cu(nscale))
    for g, w in zip(got, want):
        g, w = g.cpu().double().numpy(), w.cpu().double().numpy()
        assert np.linalg.norm(g - w) <= 1e-5 * np.linalg.norm(w)


def test_render_at_the_source_rate_is_unchanged():
    rng = np.random.default_rng(12)
    srcs = torch.from_numpy((0.1 * rng.standard_normal((2, 2, 3000))).astype(np.float32)).cuda()
    rirs = torch.from_numpy((0.1 * rng.standard_normal((2, 2, 2, 64))).astype(np.float32)).cuda()
    plain = render_binaural(srcs, rirs)
    for rate in (16000, [16000, 16000]):
        same = render_binaural(srcs, rirs, rir_sr=rate, sr=16000)
        assert all(torch.equal(a, b) for a, b in zip(plain, same))
    with pytest.raises(ValueError):
        render_binaural(srcs, rirs, rir_sr=[44100, 48000, 22050])
