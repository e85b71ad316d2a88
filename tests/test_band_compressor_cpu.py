"""Host-side checks of the band compressor, no device: a float64 numpy model of the linked multiband compressor
(l2h_band_compressor, the reference of tests/test_band_compressor_gpu.py) with its own checks; the bank's design; the
layout; the argument errors of the three C entries, returned before anything is enqueued; the Python checks of
BandCompressor; the header; the exports."""
import ctypes
import math

import numpy as np
import pytest
import torch
from scipy.signal import firwin

from kernels.scaffold import SENSITIVITY, ratio
from lookoncetohear_b200 import BandCompressor
from serving_util import declaration, doc_before, header

HOP = 128
BIG = 2.0 ** 32
EDGES = (500.0, 1000.0, 2000.0, 4000.0)
ENTRIES = ("l2h_band_compressor_design", "l2h_band_compressor_layout", "l2h_band_compressor")


def coef(tau):
    return -math.expm1(-HOP / 16000 / tau)


ATTACK, RELEASE = coef(0.005), coef(0.08)


# ---- the model -------------------------------------------------------------------------------------------------------
def bank64(edges=EDGES, taps=129):
    """the bank in float64 from scipy's firwin: [K, taps]"""
    lp = [firwin(taps, e, fs=16000) for e in edges]
    delta = np.zeros(taps)
    delta[(taps - 1) // 2] = 1.0
    lo = [np.zeros(taps)] + lp
    hi = lp + [delta]
    return np.stack([h - l for h, l in zip(hi, lo)])


def model_state(C, K, L):
    """a fresh slot: per-ear profile and current gains (dB), the detectors, knees, slopes and each channel's history"""
    return {"prof": np.zeros((C, K)), "g": np.zeros((C, K)), "S": np.zeros(K), "knee": np.zeros(K),
            "slope": np.zeros(K), "hist": np.zeros((C, L - 1))}


def set_profile(st, gains, knees=0.0, ratios=1.0):
    K = st["S"].shape[0]
    st["prof"] = np.broadcast_to(np.asarray(gains, dtype=np.float64), st["prof"].shape).copy()
    st["knee"] = np.broadcast_to(np.asarray(knees, dtype=np.float64), (K,)).copy()
    st["slope"] = 1.0 - 1.0 / np.broadcast_to(np.asarray(ratios, dtype=np.float64), (K,))


# Mutants of the model, each a plausible kernel bug (model_hop(mutant=...)): the gain ramp one sample early, the
# detector's level from channel 0 only, the level not divided by C, the taps applied in reverse (a correlation), the
# second copy of the history rotation dropped (only histories longer than one thread's 128 samples), release for attack.
MUTANTS = ("early", "unlinked", "undivided", "reversed", "history", "attack")


def bands(st, x, bank, mutant=None):
    """the staged window [C, L - 1 + 128], the band signals [C, K, 128] and whether every sample is measured"""
    with np.errstate(invalid="ignore"):
        ok = np.abs(x) < BIG
    w = np.concatenate([st["hist"], np.where(ok, x, 0.0)], 1)
    taps = bank[:, ::-1] if mutant == "reversed" else bank
    band = np.stack([[np.convolve(w[c], taps[b], "valid") for b in range(len(taps))] for c in range(len(w))])
    return w, band, bool(ok.all())


def detect(S, band, attack=ATTACK, release=RELEASE, mutant=None):
    """the detectors after a measured hop: the linked level P [K] and the new S [K]"""
    if mutant == "unlinked":
        P = (band[:1] ** 2).mean(axis=(0, 2))
    elif mutant == "undivided":
        P = (band ** 2).sum(axis=(0, 2)) / HOP
    else:
        P = (band ** 2).mean(axis=(0, 2))
    up = np.where(P > S, release if mutant == "attack" else attack, release)
    return P, S + up * (P - S)


def end_gains(st, S):
    """each channel's band gains (dB) at the end of a hop whose detectors end at S"""
    with np.errstate(divide="ignore"):
        level = 10 * np.log10(S)
    R = st["slope"] * np.maximum(0.0, level - st["knee"])
    return np.clip(st["prof"] - R[None], -40.0, 40.0)


def ramp(g0, g1, mutant=None):
    """the dB gain of samples k = 1 .. 128 (k = 0 .. 127 for the early mutant), [..., 128]"""
    k = np.arange(HOP) + (mutant != "early")
    return g0[..., None] + (g1 - g0)[..., None] * k / HOP


def hop_out(w, band, g0, g1, mutant=None):
    """the hop's output from the gains at its start and end: the window delayed by D where both are 0 dB everywhere"""
    H = w.shape[1] - HOP
    if not g0.any() and not g1.any():
        return w[:, H - H // 2:H - H // 2 + HOP]
    gk = ramp(g0, g1, mutant)
    return (np.where(gk == 0, 1.0, 10 ** (gk / 20)) * band).sum(1)


def model_hop(st, x, bank, attack=ATTACK, release=RELEASE, mutant=None):
    """l2h_band_compressor on one hop of one slot: x [C, 128] float64 (float32 values), bank [K, L]; returns the hop's
    output and advances st"""
    w, band, ok = bands(st, x, bank, mutant)
    if ok:
        st["S"] = detect(st["S"], band, attack, release, mutant)[1]
    g0, g1 = st["g"], end_gains(st, st["S"])
    y = hop_out(w, band, g0, g1, mutant)
    hist = w[:, HOP:]
    if mutant == "history" and hist.shape[1] > HOP:
        hist = np.concatenate([hist[:, :HOP], st["hist"][:, HOP:]], 1)
    st["hist"], st["g"] = hist, g1
    return y


# ---- the kernel's state row and the error bound of one hop ----------------------------------------------------------
U = 2.0 ** -24                       # the unit roundoff of fp32
LOG2_10_20 = math.log2(10) / 20
LOG2_10_20_F32 = float(np.float32(LOG2_10_20))


def gamma(n):
    return n * U / (1 - n * U)


def from_row(row, K):
    """a slot's state rows [C, 5 K + L - 1] as the kernel keeps them (fp32) -> the model's state"""
    r = np.asarray(row, np.float32).astype(np.float64)
    return {"prof": r[:, :K].copy(), "g": r[:, K:2 * K].copy(), "S": r[0, 2 * K:3 * K].copy(),
            "knee": r[0, 3 * K:4 * K].copy(), "slope": r[0, 4 * K:5 * K].copy(), "hist": r[:, 5 * K:].copy()}


def to_row(st):
    """the model's state -> the kernel's fp32 rows; the head words only channel 0 keeps are 0 in the other channels"""
    C, K = st["prof"].shape
    row = np.zeros((C, 5 * K + st["hist"].shape[1]), np.float32)
    row[:, :K], row[:, K:2 * K], row[:, 5 * K:] = st["prof"], st["g"], st["hist"]
    row[0, 2 * K:3 * K], row[0, 3 * K:4 * K], row[0, 4 * K:5 * K] = st["S"], st["knee"], st["slope"]
    return row


def hop_bound(st, x, bank, S1, g1, attack=ATTACK, release=RELEASE):
    """The kernel's error bounds for one hop from state st, given the detectors S1 and gains g1 it ended the hop with:
    {"S": S1 against detect(), "g": g1 against end_gains(st, S1), "y": the output against hop_out(st g, g1)}.
      band: an L-term fp32 FMA chain, beta = gamma_L sum |h| |x|;
      P: 128 C squares of band signals within beta, summed at depth C + 8, then one scaling by fl(1 / (128 C));
      S: fmaf(coef, fl(P - S), S), and, where |P - S| is within P's error, either coefficient;
      g: 10 log10f(S1) (2 ulp), then the knee's difference, the slope's product and the profile's difference;
      y: gk = fmaf(fl(g1 - g0), k / 128, g0), exp2f (2 ulp) of fl(gk fl(log2(10) / 20)), then the K-term FMA band sum;
         0 where g0 and g1 are 0 dB everywhere (the delayed input)."""
    C = x.shape[0]
    K, L = bank.shape
    w, band, ok = bands(st, x, bank)
    aw = np.abs(w)
    beta = gamma(L) * np.stack([[np.convolve(aw[c], np.abs(bank[b]), "valid") for b in range(K)] for c in range(C)])
    out = {}
    if ok:
        P, S = detect(st["S"], band, attack, release)
        big = np.abs(band) + beta
        eP = ((2 * np.abs(band) * beta + beta ** 2).sum(axis=(0, 2)) + gamma(C + 8) * (big ** 2).sum(axis=(0, 2))) \
            / (HOP * C) * (1 + 3 * U) + 2 * U * P
        d = np.abs(P - st["S"])
        c = np.maximum(attack, release)
        eS = c * (eP * (1 + U) + U * d) + U * (np.abs(S) + c * eP) + np.where(d <= eP, abs(attack - release) * (d + eP), 0)
        out["S"] = eS
    else:
        out["S"] = np.zeros(K)                      # the detectors keep their bits
    with np.errstate(divide="ignore", invalid="ignore"):
        lg = np.where(S1 > 0, np.log10(np.where(S1 > 0, S1, 1.0)), 0.0)
    t = 10 * lg
    et = 10 * 2 * 2.0 ** -23 * np.abs(lg) + U * np.abs(t)
    R = np.where(S1 > 0, st["slope"] * np.maximum(0.0, t - st["knee"]), 0.0)      # 10 log10f(0) = -inf: R is 0
    eR = np.where(S1 > 0, np.abs(st["slope"]) * (et + U * np.abs(t - st["knee"])) + U * np.abs(R), 0.0)
    out["g"] = eR[None] + U * np.abs(st["prof"] - R[None]) * (R != 0)[None]
    g0 = st["g"]
    if not g0.any() and not g1.any():
        out["y"] = np.zeros((C, HOP))
        return out
    gk = ramp(g0, g1)
    egk = U * np.abs(g1 - g0)[..., None] + U * np.abs(gk)
    earg = LOG2_10_20 * egk + np.abs(gk) * (abs(LOG2_10_20_F32 - LOG2_10_20) + U * LOG2_10_20_F32)
    lin = np.where(gk == 0, 1.0, 10 ** (gk / 20))
    elin = lin * (math.log(2) * earg + 2.0 ** -22) * (1 + 4 * U)
    out["y"] = (lin * beta + np.abs(band) * elin).sum(1) + gamma(K) * ((lin + elin) * (np.abs(band) + beta)).sum(1)
    return out


def hop_errors(st, x, bank, got, mutant=None, attack=ATTACK, release=RELEASE):
    """error / bound of a hop run from state st, got = {"y", "S", "g", "hist"} (its output and the state it ended with),
    against the model or one of its mutants from st: S against detect(), g against end_gains() of got's S, y against
    hop_out() of st's and got's gains; the history must match bit for bit (inf where it does not)"""
    b = hop_bound(st, x, bank, got["S"], got["g"], attack, release)
    w, band, ok = bands(st, x, bank, mutant)
    S = detect(st["S"], band, attack, release, mutant)[1] if ok else st["S"]
    m = {k: v.copy() for k, v in st.items()}
    model_hop(m, x, bank, attack, release, mutant)
    return {"y": ratio(got["y"], hop_out(w, band, st["g"], got["g"], mutant), b["y"]),
            "S": ratio(got["S"], S, b["S"]), "g": ratio(got["g"], end_gains(st, got["S"]), b["g"]),
            "hist": 0.0 if np.array_equal(got["hist"], m["hist"]) else math.inf}


def model_run(x, ticks, bank, st=None, **kw):
    """x [C, 128 N] through one slot in ticks of the given hop counts: (y, state, the detector levels after every hop)"""
    st = st or model_state(x.shape[0], *bank.shape)
    ys, levels, h = [], [], 0
    for m in ticks:
        for _ in range(m):
            ys.append(model_hop(st, x[:, HOP * h:HOP * (h + 1)], bank, **kw))
            levels.append(st["S"].copy())
            h += 1
    return np.concatenate(ys, 1), st, np.array(levels)


def sine(C, hops, freq=1500.0, db=-30.0):
    """a sine in every channel, rounded to float32: at 1500 Hz a hop holds exactly 12 periods"""
    t = np.arange(HOP * hops) / 16000
    return np.tile(10 ** (db / 20) * np.sin(2 * np.pi * freq * t), (C, 1)).astype(np.float32).astype(np.float64)


def speech(C, hops, seed, db=0.0):
    """a seeded speech-like signal: partials across the bands and noise under a syllable envelope, the channels at
    different levels (an ILD), rounded to float32"""
    g = np.random.default_rng(seed)
    N = HOP * hops
    t = np.arange(N) / 16000
    env = np.repeat(g.uniform(0.2, 1.0, N // 1600 + 1), 1600)[:N]
    sig = env * (np.sin(2 * np.pi * 220 * t) + 0.7 * np.sin(2 * np.pi * 1300 * t) + 0.5 * np.sin(2 * np.pi * 3100 * t)
                 + 0.3 * g.standard_normal(N)) * 0.1 * 10 ** (db / 20)
    return np.stack([sig * (1.0 - 0.4 * c / max(C - 1, 1)) for c in range(C)]).astype(np.float32).astype(np.float64)


def cuts(hops, seed, hi=4):
    g = np.random.default_rng(seed)
    out = []
    while sum(out) < hops:
        out.append(int(min(g.integers(0, hi), hops - sum(out))))
    return out


BANK = bank64()


# ---- the model's own checks ------------------------------------------------------------------------------------------
def test_bank_sums_to_a_delay_and_separates_the_bands():
    delta = np.zeros(129)
    delta[64] = 1.0
    assert np.abs(BANK.sum(0) - delta).max() < 1e-12
    mids = (250.0, 700.0, 1400.0, 2800.0, 6000.0)
    n = np.arange(129)
    for b in range(5):
        resp = [20 * np.log10(abs(np.sum(BANK[b] * np.exp(-2j * np.pi * f / 16000 * n)))) for f in mids]
        for o in range(5):
            if o != b:
                assert resp[o] - resp[b] <= -47.0, (b, o, resp)


def test_fresh_slot_is_the_delayed_input():
    x = speech(2, 20, 1)
    y, st, _ = model_run(x, [20], BANK)
    assert np.array_equal(y[:, 64:], x[:, :-64]) and not y[:, :64].any()
    assert st["S"].min() > 0


def test_flat_six_db_doubles_the_delayed_input():
    x = speech(2, 30, 2)
    st = model_state(2, 5, 129)
    set_profile(st, 20 * math.log10(2.0))
    y, _, _ = model_run(x, [30], BANK, st=st)
    assert np.abs(y[:, HOP:] - 2 * x[:, HOP - 64:-64]).max() <= 1e-9 * np.abs(x).max()


def test_sine_in_band_2_settles_at_the_compressed_gain():
    """a 1500 Hz sine at -30 dBFS in both ears, band 2 at +10 dB with a -40 dBFS knee and ratio 2: its level reads
    -33.02 dBFS, its gain settles at 10 - 0.5 (-33.02 + 40) = 6.51 dB, and the output sits 6.50 dB above the input"""
    x = sine(2, 200)
    st = model_state(2, 5, 129)
    set_profile(st, [0, 0, 10, 0, 0], knees=-40.0, ratios=[1, 1, 2, 1, 1])
    y, st, _ = model_run(x, [200], BANK, st=st)
    level = 10 * math.log10(st["S"][2])
    assert abs(level - (-33.02)) < 0.01
    assert abs(st["g"][0, 2] - 6.51) < 0.05 and st["g"][0, 2] == st["g"][1, 2]
    n = np.arange(129)
    pass_db = 20 * np.log10(abs(np.sum(BANK[2] * np.exp(-2j * np.pi * 1500 / 16000 * n))))
    assert abs(pass_db - (-0.013)) < 0.001
    tail = slice(HOP * 150, None)
    rise = 20 * math.log10(np.sqrt((y[:, tail] ** 2).mean() / (x[:, tail] ** 2).mean()))
    assert abs(rise - 6.50) < 0.05


def test_attack_and_release_follow_their_time_constants():
    """the detector's distance to a steady level shrinks by exp(-8 ms / tau) per hop: attack when the level rises,
    release when it falls"""
    x = np.concatenate([sine(1, 60, db=-40.0), sine(1, 60, db=-20.0), sine(1, 300, db=-40.0)], 1)
    _, _, S = model_run(x, [420], BANK)
    s = S[:, 2]
    for lo, hi, tau, target in ((62, 68, 0.005, s[119]), (125, 250, 0.08, s[-1])):     # against the settled level
        ratio = (s[lo + 1:hi + 1] - target) / (s[lo:hi] - target)
        assert np.abs(ratio - math.exp(-0.008 / tau)).max() < 1e-3, tau
    # 1 / e of the way after tau: 0.625 hops for attack, 10 for release
    assert (s[61 + 10] - s[59]) / (s[100] - s[59]) > 0.99
    assert abs((s[120 + 10] - s[119]) / (s[400] - s[119]) - (1 - math.exp(-10 * 0.008 / 0.08))) < 0.02


def test_non_finite_hops_are_not_measured():
    x = speech(2, 40, 3)
    x[0, HOP * 20 + 5] = np.nan
    x[1, HOP * 27] = -np.inf
    x[0, HOP * 33 + 7] = 2.0 ** 32
    st = model_state(2, 5, 129)
    set_profile(st, [3, -2, 6, 9, 1], knees=-50.0, ratios=3.0)
    y, st, S = model_run(x, [40], BANK, st=st)
    for h in (20, 27, 33):
        assert np.array_equal(S[h], S[h - 1]), h
    assert np.isfinite(y).all() and all(np.isfinite(v).all() for v in st.values())


def test_cutting_into_ticks_changes_nothing():
    x = speech(2, 90, 4, db=-6.0)
    st0 = model_state(2, 5, 129)
    set_profile(st0, np.array([[0, 4, 8, 12, 6], [2, 6, 14, 20, 10]]), knees=-45.0, ratios=[1.5, 2, 2, 3, 2])
    runs = [model_run(x, t, BANK, st={k: v.copy() for k, v in st0.items()}) for t in ([90], cuts(90, 5), cuts(90, 6))]
    for y, st, _ in runs[1:]:
        assert np.array_equal(y, runs[0][0]) and all(np.array_equal(st[k], runs[0][1][k]) for k in st)


def random_bank(K, L, seed):
    """a seeded asymmetric bank [K, L] of fp32 values: unlike the designed one, it shows the order of the taps"""
    return np.random.default_rng(seed).uniform(-0.3, 0.3, (K, L)).astype(np.float32).astype(np.float64)


def test_state_row_round_trips():
    C, K, L = 3, 4, 37
    row = (np.arange(C * (5 * K + L - 1)).reshape(C, -1) * 0.37 - 5).astype(np.float32)
    row[1:, 2 * K:5 * K] = 0
    st = from_row(row, K)
    assert st["S"].tolist() == row[0, 2 * K:3 * K].tolist() and np.array_equal(st["hist"], row[:, 5 * K:])
    assert np.array_equal(to_row(st).view(np.int32), row.view(np.int32))


def mutant_case():
    """a hop of 2 channels through a random bank of 161 taps (a history of 160 samples): the detectors attack, every
    gain moves, and the channels differ"""
    C, K, L = 2, 4, 161
    bank = random_bank(K, L, 3)
    st = model_state(C, K, L)
    set_profile(st, np.array([[6, -3, 9, 2], [1, 4, -5, 8]]), knees=-60.0, ratios=[2, 3, 1.5, 4])
    st["S"], st["g"] = np.full(K, 1e-5), np.full((C, K), 3.0)
    x = speech(C, 3, 7, db=-3.0)
    st["hist"] = x[:, :L - 1].copy()
    return st, x[:, 2 * HOP:], bank


def test_bounds_are_zero_where_the_arithmetic_is_exact():
    st, x, bank = mutant_case()
    st["hist"][:] = 0
    st["S"][:] = 0
    b = hop_bound(st, np.zeros_like(x), bank, np.zeros(4), end_gains(st, np.zeros(4)))
    assert all(not v.any() for v in b.values())                  # silence: every band, level and gain is exact
    st["g"][:], st["prof"][:] = 0, 0
    b = hop_bound(st, x, bank, np.zeros(4), np.zeros((2, 4)))
    assert not b["y"].any() and not b["g"].any()                 # 0 dB at both ends: the delayed input


def test_mutants_miss_their_bounds():
    st, x, bank = mutant_case()
    m = {k: v.copy() for k, v in st.items()}
    y = model_hop(m, x, bank)
    got = {"y": y, "S": m["S"], "g": m["g"], "hist": m["hist"]}
    assert max(hop_errors(st, x, bank, got).values()) == 0
    for mutant in MUTANTS:
        assert max(hop_errors(st, x, bank, got, mutant).values()) >= SENSITIVITY, mutant


# ---- the library -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from lookoncetohear_b200 import build, _cabi
    build.build()
    return _cabi.lib()


def design(lib, edges, taps):
    e = (ctypes.c_float * max(1, len(edges)))(*edges)
    out = np.full((len(edges) + 1, taps), np.nan, dtype=np.float32)
    rc = lib.l2h_band_compressor_design(len(edges) + 1, e, taps, out.ctypes.data)
    return rc, out


@pytest.mark.parametrize("edges,taps", [(EDGES, 129), (EDGES, 97), ((), 33), ((1000.0,), 255),
                                        (tuple(450.0 * (k + 1) for k in range(15)), 129)])
def test_design_is_the_firwin_differences(lib, edges, taps):
    rc, got = design(lib, edges, taps)
    assert rc == 0
    want = bank64(edges, taps)
    delta = np.zeros(taps)
    delta[(taps - 1) // 2] = 1.0
    assert np.abs(got - want).max() < 1e-7
    assert np.abs(got.astype(np.float64).sum(0) - delta).max() < 1e-7
    assert np.array_equal(BandCompressor.design(edges, taps).numpy(), got)


def test_entries_exported_and_declared(lib):
    from lookoncetohear_b200 import _cabi
    hdr = header()
    for name in ENTRIES:
        assert hasattr(lib, name), name
        assert name in _cabi.declared_symbols(), name
        assert declaration(hdr, name)[0] is not None, name
    import lookoncetohear_b200 as pkg
    assert "BandCompressor" in pkg.__all__ and "BandCompressor" in pkg.__doc__


def test_layout(lib):
    row = ctypes.c_int32(-1)
    for C, K, L in ((1, 1, 33), (2, 5, 129), (2, 16, 255), (8, 5, 129)):
        assert lib.l2h_band_compressor_layout(C, K, L, ctypes.byref(row)) == 0 and row.value == 5 * K + L - 1
    assert lib.l2h_band_compressor_layout(2, 5, 129, None) == 1 and b"null" in lib.l2h_last_error()
    assert lib.l2h_band_compressor_layout(0, 5, 129, ctypes.byref(row)) == 1 and b"channels" in lib.l2h_last_error()
    for K in (0, 17, -1):
        assert lib.l2h_band_compressor_layout(2, K, 129, ctypes.byref(row)) == 1 and b"bands" in lib.l2h_last_error()
    for L in (31, 32, 128, 257, 0):
        assert lib.l2h_band_compressor_layout(2, 5, L, ctypes.byref(row)) == 1 and b"taps" in lib.l2h_last_error()
    assert lib.l2h_band_compressor_layout(40, 5, 129, ctypes.byref(row)) == 2
    assert b"shared memory" in lib.l2h_last_error()


def test_design_argument_errors(lib):
    out = np.zeros((5, 129), dtype=np.float32)
    e = (ctypes.c_float * 4)(*EDGES)
    assert lib.l2h_band_compressor_design(5, e, 129, None) == 1 and b"null" in lib.l2h_last_error()
    assert lib.l2h_band_compressor_design(5, None, 129, out.ctypes.data) == 1 and b"null" in lib.l2h_last_error()
    assert lib.l2h_band_compressor_design(1, None, 129, out.ctypes.data) == 0
    assert lib.l2h_band_compressor_design(17, e, 129, out.ctypes.data) == 1 and b"bands" in lib.l2h_last_error()
    assert lib.l2h_band_compressor_design(0, e, 129, out.ctypes.data) == 1 and b"bands" in lib.l2h_last_error()
    assert lib.l2h_band_compressor_design(5, e, 130, out.ctypes.data) == 1 and b"taps" in lib.l2h_last_error()
    for bad in ((500.0, 500.0, 2000.0, 4000.0), (1000.0, 500.0, 2000.0, 4000.0), (0.0, 1000.0, 2000.0, 4000.0),
                (500.0, 1000.0, 2000.0, 8000.0), (500.0, float("nan"), 2000.0, 4000.0), (-1.0, 1000.0, 2000.0, 4000.0)):
        rc, _ = design(lib, bad, 129)
        assert rc == 1 and b"edges" in lib.l2h_last_error(), bad


# argument errors: fake device addresses far apart, so only the argument under test is wrong
Y, OUT, SLOTS, TAPS, ST = (ctypes.c_void_p(a) for a in (0x1000000, 0x2000000, 0x4000000, 0x5000000, 0x6000000))


def _call(lib, y=Y, y_row=None, y_ch=None, out=OUT, o_row=None, o_ch=None, n=2, C=2, T=3, slots=SLOTS, hops=None,
          taps_dev=TAPS, K=5, L=129, st=ST, S=4, attack=0.8, release=0.1):
    y_ch = HOP * T if y_ch is None else y_ch
    o_ch = HOP * T if o_ch is None else o_ch
    y_row = C * y_ch if y_row is None else y_row
    o_row = C * o_ch if o_row is None else o_row
    return lib.l2h_band_compressor(y, y_row, y_ch, out, o_row, o_ch, n, C, T, slots, hops, taps_dev, K, L, st, S,
                                   attack, release, None)


def test_call_argument_errors(lib):
    for kw in ({"y": None}, {"out": None}, {"slots": None}, {"taps_dev": None}, {"st": None}):
        assert _call(lib, **kw) == 1, kw
        assert b"null" in lib.l2h_last_error()
    for kw in ({"n": 0}, {"C": 0}, {"T": 0}, {"S": 0}, {"n": -1}, {"T": -3}):
        assert _call(lib, **kw) == 1, kw
        assert b"positive" in lib.l2h_last_error(), kw
    assert _call(lib, n=5, S=4) == 1 and b"n <= n_slots" in lib.l2h_last_error()
    assert _call(lib, T=2 ** 24, y_ch=2 ** 31, o_ch=2 ** 31) == 1 and b"frames" in lib.l2h_last_error()
    for kw in ({"attack": 0.0}, {"attack": 1.5}, {"attack": float("nan")}, {"release": -0.1},
               {"release": float("inf")}):
        assert _call(lib, **kw) == 1 and b"attack" in lib.l2h_last_error(), kw
    for K in (0, 17):
        assert _call(lib, K=K) == 1 and b"bands" in lib.l2h_last_error(), K
    for L in (31, 130, 257):
        assert _call(lib, L=L) == 1 and b"taps" in lib.l2h_last_error(), L
    for kw in ({"y_ch": 383}, {"y_row": 2 * 384 - 1}, {"o_ch": 100}, {"o_row": 384}):
        assert _call(lib, **kw) == 1, kw
        assert b"stride" in lib.l2h_last_error(), kw
    for kw in ({"out": ctypes.c_void_p(0x1000000 + 4)}, {"out": Y, "o_row": 4 * 384},
               {"out": ctypes.c_void_p(0x1000000 + 4 * (2 * 2 * 384 - 1))}, {"out": ctypes.c_void_p(0x1000000 - 4)}):
        assert _call(lib, **kw) == 1, kw
        assert b"overlap" in lib.l2h_last_error(), kw
    assert _call(lib, C=40, n=1, S=1) == 2 and b"shared memory" in lib.l2h_last_error()


def test_header_documents_the_band_compressor():
    hdr = header()
    _, args = declaration(hdr, "l2h_band_compressor")
    assert args == ["y_dev", "y_row_stride", "y_ch_stride", "out_dev", "out_row_stride", "out_ch_stride", "n", "channels",
                    "frames", "slots_dev", "hops_dev", "taps_dev", "bands", "taps", "state_dev", "n_slots", "attack",
                    "release", "stream"]
    assert declaration(hdr, "l2h_band_compressor_layout")[1] == ["channels", "bands", "taps", "row_floats"]
    assert declaration(hdr, "l2h_band_compressor_design")[1] == ["bands", "edges_hz", "taps", "out"]
    doc = doc_before(hdr, hdr.index("int l2h_band_compressor_design("))
    for phrase in ("firwin", "delta[n - D]", "same for every channel", "interaural level differences", "-3.01",
                   "1 - exp(-0.008 / tau)", "clamp(gain_cb - R_b, -40, 40)", "bit for bit", "not measured",
                   "before anything is enqueued", "CUDA graph", "All zeros is a fresh slot", "stores nothing",
                   "y itself", "5 bands + taps - 1", "Uploads nothing", "shared memory"):
        assert phrase in doc, phrase
    assert "l2h_band_compressor" in hdr[:hdr.index("#ifndef")]


# ---- the Python checks -----------------------------------------------------------------------------------------------
def test_constructor_checks():
    for bad in ({"slots": 0}, {"channels": 0}, {"edges": (1000, 500)}, {"edges": (0, 500)}, {"edges": (500, 8000)},
                {"edges": tuple(range(100, 1700, 100))}, {"edges": "500"}, {"edges": (500, float("nan"))},
                {"taps": 128}, {"taps": 31}, {"taps": 257}, {"taps": 129.0}, {"attack": 0.0}, {"attack": -1.0},
                {"release": float("inf")}, {"release": True}, {"attack": "5ms"}):
        kw = {"slots": 4, "channels": 2, "device": "cuda"}
        kw.update(bad)
        with pytest.raises(ValueError):
            BandCompressor(**kw)
    with pytest.raises(RuntimeError, match="CUDA"):
        BandCompressor(4, 2, device="cpu")
    with pytest.raises(ValueError, match="shared memory"):
        BandCompressor(4, 40, device="cpu")


def test_per_hop_quantities(monkeypatch):
    got = {}
    monkeypatch.setattr(BandCompressor, "_allocate",
                        lambda self, row, device: (got.update(row=row), setattr(self, "state", torch.zeros(1))))
    cmp = BandCompressor(4, 2)
    assert got["row"] == 5 * 5 + 128 and cmp.delay == 64 and (cmp.bands, cmp.n_taps) == (5, 129)
    assert cmp.edges == EDGES and cmp.taps.shape == (5, 129)
    assert cmp.attack_coef == pytest.approx(ATTACK, rel=1e-15) and cmp.release_coef == pytest.approx(RELEASE, rel=1e-15)
    one = BandCompressor(4, 1, edges=(), taps=33)
    assert (one.bands, one.delay, got["row"]) == (1, 16, 5 + 32)


def _host_compressor(slots=4, C=2, K=5, L=129):
    """a BandCompressor whose state lives in host memory: the Python checks run, no engine call is reached"""
    cmp = BandCompressor.__new__(BandCompressor)
    cmp.n_slots, cmp.channels, cmp.bands, cmp.n_taps = slots, C, K, L
    cmp.state = torch.zeros(slots, C, 5 * K + L - 1)
    return cmp


def test_call_needs_cuda():
    with pytest.raises(RuntimeError, match="CUDA"):
        _host_compressor()(torch.zeros(2, 2, 256), [0, 1])


def test_set_profile_writes_the_documented_words():
    cmp, K = _host_compressor(), 5
    cmp.set_profile([2], [1, 2, 3, 4, 5], knees=-40.0, ratios=2.0)
    assert cmp.state[2, 0, :K].tolist() == [1, 2, 3, 4, 5] == cmp.state[2, 1, :K].tolist()
    assert cmp.state[2, 0, 3 * K:4 * K].tolist() == [-40.0] * K and cmp.state[2, 0, 4 * K:5 * K].tolist() == [0.5] * K
    assert not cmp.state[2, 1, 2 * K:].any() and not cmp.state[[0, 1, 3]].any()
    cmp.set_profile([0, 3], [[1, 1, 1, 1, 1], [2, 2, 2, 2, 2]], ratios=[[1, 1, 1, 1, 4], [1, 2, 1, 1, 1]])
    assert cmp.state[3, 1, :K].tolist() == [2] * K and cmp.state[0, 0, 4 * K + 4].item() == 0.75
    assert cmp.state[3, 0, 4 * K:5 * K].tolist() == [0, 0.5, 0, 0, 0]
    ears = torch.arange(2 * 2 * K, dtype=torch.float64).reshape(2, 2, K) - 10
    cmp.set_profile(torch.tensor([1, 2]), ears, knees=[-50, -40, -30, -20, -10])
    assert torch.equal(cmp.state[[1, 2], :, :K].double(), ears)
    assert cmp.state[1, 0, 3 * K:4 * K].tolist() == [-50, -40, -30, -20, -10]
    for bad in ({"gains": [1, 2, 3]}, {"gains": [[1] * 5] * 3}, {"gains": [41] * 5}, {"gains": [float("nan")] * 5},
                {"gains": 3.0}, {"knees": float("inf")}, {"knees": [0] * 4}, {"ratios": 0.5}, {"ratios": [1, 1, 1, 1, -2]},
                {"ratios": float("nan")}, {"gains": True}):
        kw = {"gains": [0.0] * 5}
        kw.update(bad)
        with pytest.raises(ValueError):
            cmp.set_profile([0, 1], **kw)
    for slots in ([], [4], [1, 1], [-1]):
        with pytest.raises(ValueError):
            cmp.set_profile(slots, [0.0] * 5)


def test_telemetry_views_and_reset():
    cmp, K = _host_compressor(), 5
    assert cmp.level.shape == (4, K) and bool((cmp.level == -math.inf).all())
    assert cmp.gain.shape == (4, 2, K) and not cmp.gain.any()
    cmp.state[1, 0, 2 * K + 3] = 0.5                               # a full-scale sine's mean square
    cmp.state[1, 1, K + 2] = -4.5
    assert cmp.level[1, 3].item() == pytest.approx(-3.0103, abs=1e-4) and cmp.gain[1, 1, 2].item() == -4.5
    cmp.set_profile([3], [1.0] * K)
    cmp.reset([1])
    assert not cmp.state[1].any() and cmp.state[3, 0, 0] == 1.0
