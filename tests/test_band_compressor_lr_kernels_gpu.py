"""band_compressor_lr_kernel of csrc/resample.cu called through the C ABI (l2h_band_compressor_lr), every hop against the
float64 model of test_band_compressor_lr_cpu.py started from the kernel's own state at the hop's start, so errors cannot
compound across hops; instantiations (one per band count K and order N) from K = 1 to 16 in both orders, C = 1 to 3
channels.

Bounds: the output to 8 times the deviation of the same sections run in float32 from the same states (their roundoff,
per band, scaled by the band's largest gain) plus the ramp's and the sum's roundoff; the level P from that band error;
the detectors from P's error, 4 ulp, and either coefficient where P is within its error of S; the gains to 1e-4 dB.
Mutants of the model (the gain ramp one sample early, the level from channel 0 only) must miss their bounds by
SENSITIVITY in every hop that exercises them.  Every buffer is a Guarded one: the guards, the unlisted
slot's state row and the output rows of calls that store nothing keep the sentinel bit for bit.
"""
import numpy as np
import pytest
import torch
from scipy.signal import sosfilt

import test_band_compressor_cpu as bc
import test_band_compressor_lr_cpu as lr
from kernels.scaffold import Guarded, Ledger, bits, dev, is_sentinel, ratio  # noqa: F401
from lookoncetohear_b200 import BandCompressor, _cabi

pytestmark = pytest.mark.gpu
HOP = 128
U = 2.0 ** -24
LEDGER = Ledger()
ATTACK, RELEASE = float(np.float32(bc.ATTACK)), float(np.float32(bc.RELEASE))
CONFIGS = [(4, 1, 2), (8, 1, 1), (4, 2, 2), (8, 3, 3), (4, 5, 2), (8, 5, 2), (4, 8, 3), (8, 8, 1), (4, 11, 2),
           (8, 12, 2), (4, 16, 3), (8, 16, 2)]


def ints(values, dev):
    g = Guarded((len(values),), dev)
    g.t.view(torch.int32).copy_(torch.tensor(values, dtype=torch.int32))
    return g


def from_row(row, K, S):
    r = np.asarray(row, np.float32).astype(np.float64)
    C = r.shape[0]
    return {"prof": r[:, :K].copy(), "g": r[:, K:2 * K].copy(), "S": r[0, 2 * K:3 * K].copy(),
            "knee": r[0, 3 * K:4 * K].copy(), "slope": r[0, 4 * K:5 * K].copy(), "z": r[:, 5 * K:].reshape(C, K, S, 2).copy()}


def to_row(st):
    C, K = st["prof"].shape
    row = np.zeros((C, 5 * K + st["z"][0].size), np.float32)
    row[:, :K], row[:, K:2 * K], row[:, 5 * K:] = st["prof"], st["g"], st["z"].reshape(C, -1)
    row[0, 2 * K:3 * K], row[0, 3 * K:4 * K], row[0, 4 * K:5 * K] = st["S"], st["knee"], st["slope"]
    return row


def mutant_hop(st, x, bank, mutant):
    """the model's hop with one mutant: 'early' (the ramp one sample early) or 'unlinked' (channel 0's level only)"""
    m = {k: v.copy() for k, v in st.items()}
    band, ok = lr.lr_bands(m, x, bank)
    S = bc.detect(m["S"], band, ATTACK, RELEASE, mutant)[1] if ok else m["S"]
    g1 = bc.end_gains(m, S)
    gk = bc.ramp(m["g"], g1, mutant)
    return (np.where(gk == 0, 1.0, 10 ** (gk / 20)) * band).sum(1)


def hop_bound(st, x, bank, g1):
    """the bounds of one hop from st (see the module's docstring): the output's [C, 128], and P's [K] (the level's error
    from the bands' roundoff)"""
    C, K = st["prof"].shape
    m = {k: v.copy() for k, v in st.items()}
    band, _ = lr.lr_bands(m, x, bank)
    with np.errstate(invalid="ignore"):
        w = np.where(np.abs(x) < 2.0 ** 32, x, 0.0)
    dev_b = np.zeros((C, K))
    if bank.shape[1]:
        for c in range(C):
            for b in range(K):
                sos = np.concatenate([bank[b][:, :3], np.ones((bank.shape[1], 1)), bank[b][:, 3:]], 1)
                lo = sosfilt(sos.astype(np.float32), w[c].astype(np.float32), zi=st["z"][c, b].astype(np.float32))[0]
                dev_b[c, b] = np.abs(lo.astype(np.float64) - band[c, b]).max()
    gk = bc.ramp(st["g"], g1)
    lin = np.where(gk == 0, 1.0, 10 ** (gk / 20))
    d = 8 * dev_b
    eP = ((2 * np.abs(band) * d[..., None] + d[..., None] ** 2).mean(axis=(0, 2)) + 1e-6 * (band ** 2).mean(axis=(0, 2)))
    return (lin.max(-1) * d).sum(1)[:, None] + (lin * np.abs(band)).sum(1) * (1e-6 + (K + 2) * U), eP


@pytest.mark.parametrize("N,K,C", CONFIGS, ids=lambda v: str(v))
def test_band_compressor_lr(N, K, C, dev):
    edges = tuple(float(e) for e in np.geomspace(150.0, 7000.0, K - 1)) if K > 1 else ()
    bank = BandCompressor.design_lr(edges, N).double().numpy()
    S = bank.shape[1]
    sos = Guarded((max(1, bank.size),), dev, torch.from_numpy(np.resize(bank.astype(np.float32), max(1, bank.size))))
    rf = 5 * K + 2 * K * S
    state = Guarded((3, C, rf), dev)
    slots, listed = ints([2, 0], dev), (2, 0)
    for s in listed:
        state.t[s] = 0
    g = np.random.default_rng(N * 100 + K * 10 + C)
    errs, shown = {}, {"early": -np.inf}
    if C > 1:
        shown["unlinked"] = -np.inf
    for seg in range(4):
        for s in listed:
            st = from_row(state.t[s].cpu().numpy(), K, S)
            bc.set_profile(st, g.uniform(-10, 12, (C, K)), knees=g.uniform(-50, -30, K), ratios=g.uniform(1, 4, K))
            if seg == 3:
                st["prof"][:], st["slope"][:] = 0, 0                      # back to flat
            state.t[s] = torch.from_numpy(to_row(st))
        x = {s: bc.speech(C, 3, 100 * seg + s + K, db=float(g.uniform(-30, 0))) for s in listed}
        if seg == 1:
            x[2][0, 5] = np.nan                                       # not measured, staged as 0
            x[0][C - 1, HOP + 9] = -np.inf
        for h in range(3):
            y = Guarded((2, C, HOP), dev, torch.from_numpy(np.stack([x[s][:, h * HOP:(h + 1) * HOP] for s in listed]).astype(np.float32)))
            out = Guarded((2, C, HOP), dev)
            hops = ints([1, 1 if h != 2 else 0], dev)               # the third hop stores nothing in row 1
            before = {s: from_row(state.t[s].cpu().numpy(), K, S) for s in listed}
            rc = _cabi.lib().l2h_band_compressor_lr(y.t.data_ptr(), C * HOP, HOP, out.t.data_ptr(), C * HOP, HOP, 2, C, 1,
                                                    slots.t.data_ptr(), hops.t.data_ptr(), sos.t.data_ptr(), K, N,
                                                    state.t.data_ptr(), 3, ATTACK, RELEASE, None)
            assert rc == 0, _cabi.lib().l2h_last_error().decode()
            torch.cuda.synchronize(dev)
            for i, s in enumerate(listed):
                if h == 2 and i == 1:
                    assert is_sentinel(out.t[i]) and torch.equal(bits(state.t[s]), bits(torch.from_numpy(to_row(before[s])).to(dev)))
                    continue
                after = from_row(state.t[s].cpu().numpy(), K, S)
                xh = x[s][:, h * HOP:(h + 1) * HOP]
                m = {k: v.copy() for k, v in before[s].items()}
                band, ok = lr.lr_bands(m, xh, bank)
                P, Sw = bc.detect(m["S"], band, ATTACK, RELEASE) if ok else (m["S"], m["S"])
                yb, eP = hop_bound(before[s], xh, bank, after["g"])
                dS = np.abs(P - m["S"])
                eS = (max(ATTACK, RELEASE) * eP + 4 * 2.0 ** -23 * np.maximum(np.abs(Sw), np.abs(m["S"]))
                      + np.where(dS <= eP, abs(ATTACK - RELEASE) * (dS + eP), 0.0)) if ok else np.zeros(K)
                yw = lr.lr_hop_out(band, before[s]["g"], after["g"])
                got = out.t[i].cpu().numpy()
                e = {"y": ratio(got, yw, yb), "S": ratio(after["S"], Sw, eS),
                     "g": ratio(after["g"], bc.end_gains(before[s], after["S"]), 1e-4)}
                for k, v in e.items():
                    errs[k] = max(errs.get(k, 0.0), v)
                for mu in shown:
                    alt = mutant_hop(before[s], xh, bank, mu)
                    if ratio(alt, yw, yb) >= 1:                       # the hop exercises the mutant
                        shown[mu] = max(shown[mu], ratio(got, alt, yb))
            assert out.ok() and y.ok()
    assert is_sentinel(state.t[1]), "an unlisted slot"
    assert state.ok() and slots.ok() and sos.ok()
    LEDGER.check("lr compressor", errs, {m: v for m, v in shown.items() if v > -np.inf})


@pytest.mark.parametrize("N,K,C", [(8, 16, 4), (4, 5, 20)])
def test_refuses_staging_past_shared_memory(N, K, C, dev):
    S = N // 2 * (K - 1)
    state = Guarded((3, C, 5 * K + 2 * K * S), dev)
    y, out = Guarded((2, C, HOP), dev), Guarded((2, C, HOP), dev)
    sos, slots = Guarded((K * S * 5,), dev, torch.zeros(K * S * 5)), ints([2, 0], dev)
    rc = _cabi.lib().l2h_band_compressor_lr(y.t.data_ptr(), C * HOP, HOP, out.t.data_ptr(), C * HOP, HOP, 2, C, 1,
                                            slots.t.data_ptr(), None, sos.t.data_ptr(), K, N, state.t.data_ptr(), 3,
                                            ATTACK, RELEASE, None)
    assert rc == 2 and b"shared memory" in _cabi.lib().l2h_last_error()
    torch.cuda.synchronize(dev)
    assert is_sentinel(state.t) and is_sentinel(out.t) and state.ok() and out.ok()


def test_summary():
    LEDGER.summary()
