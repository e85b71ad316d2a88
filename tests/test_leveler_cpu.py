"""Host-side checks of the leveler, no device: a float64 numpy model of the gated, K-weighted leveler (l2h_leveler, the
reference of tests/test_leveler_gpu.py) with its own checks; the layout; the argument errors of both C entries, returned
before anything is enqueued; the Python checks of Leveler; the header; the exports."""
import ctypes
import math

import numpy as np
import pytest
import torch
from scipy.signal import lfilter

from kernels.scaffold import SENSITIVITY, ratio
from lookoncetohear_b200 import Leveler
from serving_util import declaration, doc_before, header

HOP, FLOATS = 128, 7
BIG = 2.0 ** 32
ENTRIES = ("l2h_leveler_layout", "l2h_leveler")
DEFAULTS = {"target": -20.0, "gate": -50.0, "relative": -20.0, "alpha": -math.expm1(-HOP / (3.0 * 16000)),
            "settle": 32, "min_gain": -12.0, "max_gain": 12.0, "rise": 3.0 * HOP / 16000, "fall": 10.0 * HOP / 16000}


# ---- the model -------------------------------------------------------------------------------------------------------
def k_weighting(rate):
    """the BS.1770 pre-filters at `rate` Hz from their analog prototypes: (shelf b, shelf a, high-pass b, high-pass a)"""
    K = math.tan(math.pi * 1681.974450955533 / rate)
    Q, Vh = 0.7071752369554196, 10 ** (3.999843853973347 / 20)
    Vb = Vh ** 0.4996667741545416
    a0 = 1 + K / Q + K * K
    sb = np.array([(Vh + Vb * K / Q + K * K) / a0, 2 * (K * K - Vh) / a0, (Vh - Vb * K / Q + K * K) / a0])
    sa = np.array([1.0, 2 * (K * K - 1) / a0, (1 - K / Q + K * K) / a0])
    K = math.tan(math.pi * 38.13547087602444 / rate)
    Q = 0.5003270373238773
    a0 = 1 + K / Q + K * K
    return sb, sa, np.array([1.0, -2.0, 1.0]), np.array([1.0, 2 * (K * K - 1) / a0, (1 - K / Q + K * K) / a0])


FILTERS = k_weighting(16000)


def lufs(power):
    with np.errstate(divide="ignore"):
        return -0.691 + 10 * np.log10(power)


def model_state(C):
    """a fresh row: each channel's shelf and high-pass states, the estimate, the gated hops and the gain (dB)"""
    return {"shelf": np.zeros((C, 2)), "hp": np.zeros((C, 2)), "E": 0.0, "n": 0, "g": 0.0}


FILTERS32 = tuple(f.astype(np.float32).astype(np.float64) for f in FILTERS)     # the coefficients lv_filters rounds
INT32_MAX = 2 ** 31 - 1

# Mutants of the model, each a plausible kernel bug (model_hop(mutant=...)): the gain ramp one sample early, the
# estimate's weight max(alpha, 1 / n), the relative gate ignored, d taken one hop after `settle`, the power of channel 0
# only, the rise clamp dropped.
MUTANTS = ("early", "weight", "relative", "settle", "channel0", "rise")


def measured(x):
    return bool(np.isfinite(x).all() and np.abs(x).max() < BIG)


def gain_step(g, E, n, before, p=DEFAULTS, mutant=None):
    """the gain (dB) at the end of a measured hop that started at g with `before` gated hops and ends with n and E"""
    settle = p["settle"] + (mutant == "settle")
    if n < settle:
        return g
    d = min(max(p["target"] - lufs(E), p["min_gain"]), p["max_gain"])
    if before < settle:
        return d
    return g + (max(d - g, -p["fall"]) if mutant == "rise" else min(max(d - g, -p["fall"]), p["rise"]))


def hop_out(x, g0, g1, mutant=None):
    k = np.arange(HOP) + (mutant != "early")
    gk = g0 + (g1 - g0) * k / HOP
    return x * np.where(gk == 0, 1.0, 10 ** (gk / 20))


def model_hop(st, x, p=DEFAULTS, coefs=FILTERS, mutant=None, gated=None):
    """l2h_leveler on one hop of one row: x [C, 128] float64 (float32 values), returns the leveled hop; advances st.
    coefs: the filters (FILTERS32: the kernel's fp32 coefficients); gated: the gates' decision, when not the model's.
    The gated-hop count saturates at INT32_MAX, and a negative count word counts as 0, as in the kernel."""
    g0 = st["g"]
    st["n"] = max(st["n"], 0)
    if measured(x):
        sb, sa, hb, ha = coefs
        u, st["shelf"] = lfilter(sb, sa, x, axis=1, zi=st["shelf"])
        w, st["hp"] = lfilter(hb, ha, u, axis=1, zi=st["hp"])
        P = float(((w[:1] if mutant == "channel0" else w) ** 2).sum()) / HOP
        L, before = lufs(P), st["n"]
        if gated is None:
            gated = L >= p["gate"] and (st["n"] == 0 or mutant == "relative" or L >= lufs(st["E"]) + p["relative"])
        if gated:
            n = max(st["n"], 1) if mutant == "weight" else st["n"] + 1
            st["E"] += max(p["alpha"], 1 / n) * (P - st["E"])
            st["n"] = min(st["n"] + 1, INT32_MAX)
        st["g"] = gain_step(st["g"], st["E"], st["n"], before, p, mutant)
    return hop_out(x, g0, st["g"], mutant)


# ---- the kernel's state row and the error bound of one hop ----------------------------------------------------------
U = 2.0 ** -24                       # the unit roundoff of fp32
LOG2_10_20 = math.log2(10) / 20
LOG2_10_20_F32 = float(np.float32(LOG2_10_20))


def from_row(row):
    """a row's state [C, 7] as the kernel keeps it (fp32) -> the model's state; the count word as the int32 it holds"""
    r = np.ascontiguousarray(row, np.float32)
    return {"E": float(r[0, 0]), "n": int(r[0, 1:2].view(np.int32)[0]), "g": float(r[0, 2]),
            "shelf": r[:, 3:5].astype(np.float64), "hp": r[:, 5:7].astype(np.float64)}


def to_row(st):
    C = st["shelf"].shape[0]
    row = np.zeros((C, FLOATS), np.float32)
    row[0, 0], row[0, 2] = st["E"], st["g"]
    row[0, 1:2].view(np.int32)[0] = st["n"]
    row[:, 3:5], row[:, 5:7] = st["shelf"], st["hp"]
    return row


def lufs_err(v, ev=0.0):
    """the error of the kernel's -0.691f + 10 log10f(v) at a v within ev of the float64 v: log10f's 2 ulp, the product's
    and the sum's roundings, -0.691f's own, and ev carried through the logarithm"""
    if v <= 0:
        return 0.0 if ev == 0 else math.inf
    lg = math.log10(v)
    return (10 * 10 / math.log(10) * ev / v if ev else 0.0) + 20 * 2.0 ** -23 * abs(lg) + U * abs(10 * lg) \
        + U * abs(lufs(v)) + abs(float(np.float32(-0.691)) + 0.691)


def filter_bound(st, x, coefs=FILTERS32):
    """The two sections in transposed direct form II, one fmaf per step as the kernel runs them: (the float64 states
    [C, 4], their error bounds, the per-channel sums of the squared weighted samples [C] and their bounds).  Each step's
    roundings (u |value| per rounded result) are carried to later steps through the powers of the sections' state
    matrix M, in absolute value: |M^m| stays small where |M|^m, with the high-pass's poles near 1, would not.  The
    error of u = fl(sb0 x + s1) enters as one of s1.  A thread accumulates channels c, c + 128, ... into one sum, so a
    channel's rounding terms are counted against its thread's running sum."""
    (sb0, sb1, sb2), (_, sa1, sa2), _, (_, ha1, ha2) = coefs
    M = np.array([[-sa1, 1, 0, 0], [-sa2, 0, 0, 0], [-2 - ha1, 0, -ha1, 1], [1 - ha2, 0, -ha2, 0]])
    Mp = [np.eye(4)]
    for _ in range(HOP):
        Mp.append(M @ Mp[-1])
    Mp = np.array(Mp)                                          # [HOP + 1, 4, 4]
    cM = np.abs(Mp[:, 0] + Mp[:, 2])                           # w = u + h1 = s1 + h1 + sb0 x: [HOP + 1, 4]
    C = len(x)
    s1, s2 = st["shelf"][:, 0].copy(), st["shelf"][:, 1].copy()
    h1, h2 = st["hp"][:, 0].copy(), st["hp"][:, 1].copy()
    a, b, W = np.zeros((C, HOP, 4)), np.zeros((C, HOP, 4)), np.zeros((C, HOP))
    for k in range(HOP):
        xk = x[:, k]
        u = sb0 * xk + s1
        inner = -sa1 * u + s2
        s1n = sb1 * xk + inner
        prod = -sa2 * u
        s2 = sb2 * xk + prod
        w = u + h1
        inner2 = -ha1 * w + h2
        h1n = -2 * u + inner2
        h2 = -ha2 * w + u
        a[:, k, 0] = U * np.abs(u)
        b[:, k] = np.stack([U * (np.abs(inner) + np.abs(s1n)), U * (np.abs(prod) + np.abs(s2)),
                            U * (np.abs(inner2) + np.abs(h1n) + abs(ha1) * np.abs(w)),
                            U * (np.abs(h2) + abs(ha2) * np.abs(w))], 1)
        s1, h1, W[:, k] = s1n, h1n, w
    j = np.arange(HOP)
    e = np.einsum("jst,cjt->cs", np.abs(Mp[HOP - j]), a) + np.einsum("jst,cjt->cs", np.abs(Mp[HOP - 1 - j]), b)
    lag = j[:, None] - j[None, :]                              # k - j
    Ta = np.where((lag > 0)[..., None], cM[np.clip(lag, 0, HOP)], 0.0)
    Tb = np.where((lag > 0)[..., None], cM[np.clip(lag - 1, 0, HOP)], 0.0)
    ew = np.einsum("kjs,cjs->ck", Ta, a) + np.einsum("kjs,cjs->ck", Tb, b) + a[:, :, 0] + U * np.abs(W)
    A = (W * W).sum(1)
    eA = (2 * np.abs(W) * ew + ew * ew).sum(1) + U * np.cumsum(W * W, 1).sum(1)
    for c in range(128, C):                                    # the sums of the thread's earlier channels
        eA[c] += HOP * U * (A[c % 128:c:128] + eA[c % 128:c:128]).sum()
    grow = 1 + 8 * U
    return np.stack([s1, s2, h1, h2], 1), e * grow, A, eA * grow


def hop_errors(st, x, p, got, mutant=None, coefs=FILTERS32):
    """error / bound of a hop run from state st, got = from_row() of the state it ended with plus its output "y", against
    the model or one of its mutants from st.  The count word must match exactly; where the float64 loudness lies within
    its bound of a gate, the kernel's branch (shown by its count, or by its estimate at a saturated count) is taken.
      filters: filter_bound's running bounds;  P: the per-channel sums within their bounds, summed over min(C, 128)
      thread sums from 0;  E: fmaf(w, fl(P - E), E), w = max(alpha, fl(1 / fl(n + 1))) within 2 roundings of 1 / (n + 1);
      g: from the kernel's own E, lufs_err, then the target's, d - g's and the step's roundings;
      y: from the kernel's own start and end gains: fmaf(fl(g1 - g0), k / 128, g0), exp2f (2 ulp), the product."""
    g0, n0 = st["g"], max(st["n"], 0)
    out = {}
    if not measured(x):
        same = got["E"] == st["E"] and got["n"] == n0 and got["g"] == g0 and \
            np.array_equal(got["shelf"], st["shelf"]) and np.array_equal(got["hp"], st["hp"])
        out["state"] = 0.0 if same else math.inf
        g1, eg = got["g"], 0.0
    else:
        ref, ef, A, eA = filter_bound(st, x, coefs)
        out["filters"] = ratio(np.concatenate([got["shelf"], got["hp"]], 1), ref, ef)
        m = min(len(x), 128)
        P, eP = A.sum() / HOP, (eA.sum() + gamma(m) * (A + eA).sum()) / HOP
        L, eL = lufs(P), lufs_err(P, eP)
        ambiguous = abs(L - p["gate"]) <= eL or (
            n0 > 0 and abs(L - lufs(st["E"]) - p["relative"]) <= eL + lufs_err(st["E"]) + U * abs(lufs(st["E"]) + p["relative"]))
        took = got["n"] != n0 if n0 < INT32_MAX else got["E"] != st["E"]
        mst = dict(st, shelf=st["shelf"].copy(), hp=st["hp"].copy())
        model_hop(mst, x, p, coefs, mutant, gated=took if ambiguous else None)
        out["n"] = 0.0 if got["n"] == mst["n"] else math.inf
        if mst["n"] != n0 or (n0 == INT32_MAX and mst["E"] != st["E"]):          # gated
            wgt = max(p["alpha"], 1 / (n0 + 1))
            d = abs(P - st["E"])
            eE = wgt * (eP + U * (d + eP)) + 2 * U * wgt * d + U * abs(mst["E"])
            if mutant == "channel0":
                eE += wgt * eP                                                   # its own P, not the bound's
            out["E"] = ratio(got["E"], mst["E"], eE * (1 + 4 * U))
        else:
            out["E"] = 0.0 if got["E"] == st["E"] else math.inf
        g1 = gain_step(g0, got["E"], mst["n"], n0, p, mutant)
        settle = p["settle"] + (mutant == "settle")
        eg = 0.0
        if mst["n"] >= settle:
            LE = lufs(got["E"])
            t = p["target"] - LE
            d = min(max(t, p["min_gain"]), p["max_gain"])
            eg = lufs_err(got["E"]) + U * abs(t)
            if n0 >= settle:
                eg += U * abs(d - g0) + U * abs(g1)
        out["g"] = ratio(got["g"], g1, eg * (1 + 4 * U))
    gk = g0 + (got["g"] - g0) * np.arange(1, HOP + 1) / HOP
    egk = U * abs(got["g"] - g0) + U * np.abs(gk)
    earg = LOG2_10_20 * egk + np.abs(gk) * (abs(LOG2_10_20_F32 - LOG2_10_20) + U * LOG2_10_20_F32)
    lin = np.where(gk == 0, 1.0, 10 ** (gk / 20))
    elin = lin * (math.log(2) * earg + 2.0 ** -22)
    y = hop_out(x, g0, got["g"], mutant)
    exact = g0 == 0 and got["g"] == 0                              # a gain of 0 dB is exactly 1
    out["y"] = ratio(got["y"], y, 0.0 if exact else (np.abs(x) * elin + U * np.abs(y)) * (1 + 4 * U))
    return out


def gamma(n):
    return n * U / (1 - n * U)


def model_run(x, ticks, p=DEFAULTS, st=None):
    """x [C, 128 N] through one row in ticks of the given hop counts: (y, state, the gain after every hop)"""
    st = st or model_state(x.shape[0])
    ys, gains, h = [], [], 0
    for m in ticks:
        for _ in range(m):
            ys.append(model_hop(st, x[:, HOP * h:HOP * (h + 1)], p))
            gains.append(st["g"])
            h += 1
    return np.concatenate(ys, 1), st, np.array(gains)


def voice(C, hops, seed, db=0.0, pause=None):
    """a seeded speech-like signal of `hops` hops at roughly `db` dB: bursts of partials and noise with a syllable
    envelope, quiet gaps in `pause` (a slice of hops), the channels at different levels (an ILD), rounded to float32"""
    g = np.random.default_rng(seed)
    N = HOP * hops
    t = np.arange(N) / 16000
    env = np.repeat(g.uniform(0.3, 1.0, N // 1600 + 1), 1600)[:N]
    sig = env * (np.sin(2 * np.pi * 180 * t) + 0.6 * np.sin(2 * np.pi * 1170 * t) + 0.3 * g.standard_normal(N)) * 0.1
    sig *= 10 ** (db / 20)
    if pause is not None:
        sig[HOP * pause.start:HOP * pause.stop] *= 1e-4
    return np.stack([sig * (1.0 - 0.3 * c / max(C - 1, 1)) for c in range(C)]).astype(np.float32).astype(np.float64)


def cuts(hops, seed, hi=4):
    g = np.random.default_rng(seed)
    out = []
    while sum(out) < hops:
        out.append(int(min(g.integers(0, hi), hops - sum(out))))
    return out


# ---- the model's own checks ------------------------------------------------------------------------------------------
def test_coefficients_reproduce_the_bs1770_table_at_48k():
    sb, sa, hb, ha = k_weighting(48000)
    assert np.abs(sb - [1.53512485958697, -2.69169618940638, 1.19839281085285]).max() < 1e-12
    assert np.abs(sa - [1.0, -1.69065929318241, 0.73248077421585]).max() < 1e-12
    assert np.abs(ha - [1.0, -1.99004745483398, 0.99007225036621]).max() < 1e-12
    assert list(hb) == [1.0, -2.0, 1.0]


@pytest.mark.parametrize("C,want", [(1, -2.970), (2, 0.040)])
def test_full_scale_997_hz_sine(C, want):
    """a full-scale 997 Hz sine at 16 kHz in every channel, past the filters' start: its K-weighted loudness"""
    N = HOP * 400
    x = np.tile(np.sin(2 * np.pi * 997 * np.arange(N) / 16000), (C, 1))
    sb, sa, hb, ha = FILTERS
    w = lfilter(hb, ha, lfilter(sb, sa, x, axis=1), axis=1)[:, HOP * 100:]
    assert abs(float(lufs((w ** 2).sum(0).mean())) - want) < 1e-3
    y, st, _ = model_run(x, [400])
    assert abs(lufs(st["E"]) - want) < 0.01                       # the estimate of the same hops


def test_gate_holds_the_estimate_through_pauses():
    """a voice with a long near-silent pause: the pause's hops fail the absolute gate, so neither the estimate nor the
    count moves, and the gain stays where it was; a hop 25 dB under the estimate fails the relative gate"""
    x = voice(2, 600, 1, db=-10.0, pause=slice(300, 450))
    _, st, gains = model_run(x, [305])                            # the filters' tail of the voice fades in the pause
    E, n, g = st["E"], st["n"], st["g"]
    assert 250 < n <= 305
    x2 = x[:, HOP * 305:HOP * 450]
    _, st2, g2 = model_run(x2, [145], st=dict(st, shelf=st["shelf"].copy(), hp=st["hp"].copy()))
    assert st2["n"] == n and st2["E"] == E
    # gain moves only toward the d of the held estimate, which it had reached or approaches monotonically
    d = min(max(-20.0 - lufs(E), -12.0), 12.0)
    assert np.all(np.diff(np.abs(g2 - d)) <= 1e-12) and abs(g2[0] - g) <= DEFAULTS["fall"] + 1e-12
    quiet = voice(2, 40, 2, db=-35.0)                              # ~25 dB under the estimate, over the absolute gate
    st3 = dict(st, shelf=st["shelf"].copy(), hp=st["hp"].copy())
    model_run(quiet, [40], st=st3)
    assert st3["n"] == n and st3["E"] == E


def test_settle_then_rise_and_fall():
    """the gain stays at 0 dB for the first settle - 1 gated hops, takes d in the hop of the settle-th, then follows a
    level change at exactly `rise` dB per hop upward and `fall` dB per hop downward"""
    p = dict(DEFAULTS, settle=10, alpha=0.05)                     # a short window: the estimate follows within hops
    x = voice(1, 2000, 3, db=5.0)                                  # about -20 LUFS
    x[:, HOP * 800:HOP * 1400] *= 10 ** (-10 / 20)                # 10 dB softer: the gain rises
    x[:, HOP * 1400:] *= 10 ** (16 / 20)                          # then 6 dB louder than the start: it falls
    _, st, g = model_run(x, [2000], p)
    assert np.all(g[:9] == 0) and g[9] != 0
    steps = np.diff(g)[9:]                                         # after the settling hop
    assert steps.max() <= p["rise"] + 1e-12 and steps.min() >= -p["fall"] - 1e-12
    assert np.isclose(steps[791:891], p["rise"]).sum() > 50          # rising at the rate limit
    assert np.isclose(steps[1391:1491], -p["fall"]).sum() > 50       # falling at the rate limit
    # a fresh row whose settle-th gated hop is the 10th takes d there exactly
    st2 = model_state(1)
    for h in range(10):
        model_hop(st2, x[:, HOP * h:HOP * (h + 1)], p)
    assert st2["n"] == 10 and st2["g"] == min(max(-20.0 - lufs(st2["E"]), -12.0), 12.0)


def test_non_finite_hops_are_not_measured():
    x = voice(2, 60, 4)
    x[0, HOP * 20 + 5] = np.nan
    x[1, HOP * 41] = np.inf
    x[0, HOP * 50 + 7] = 2.0 ** 32
    _, st_a, g_a = model_run(x, [60])
    keep = [h for h in range(60) if h not in (20, 41, 50)]
    y_b, st_b, _ = model_run(np.concatenate([x[:, HOP * h:HOP * (h + 1)] for h in keep], 1), [57])
    assert st_a["n"] == st_b["n"] and st_a["E"] == st_b["E"] and np.array_equal(st_a["hp"], st_b["hp"])
    assert g_a[20] == g_a[19] and g_a[41] == g_a[40]


def test_cutting_into_ticks_changes_nothing():
    x = voice(2, 700, 5, db=-14.0, pause=slice(200, 260))
    y, st, _ = model_run(x, [700])
    for seed in (6, 7):
        y2, st2, _ = model_run(x, cuts(700, seed))
        assert np.array_equal(y, y2)
        assert all(np.array_equal(st[k], st2[k]) for k in st)


def test_identity_at_zero_gain_range():
    x = voice(2, 100, 8)
    y, st, _ = model_run(x, [100], dict(DEFAULTS, min_gain=0.0, max_gain=0.0))
    assert np.array_equal(y, x) and st["g"] == 0 and st["n"] > 0


def test_state_row_round_trips():
    row = (np.arange(3 * FLOATS).reshape(3, FLOATS) * 0.37 - 2).astype(np.float32)
    row[1:, :3] = 0
    row[0, 1:2].view(np.int32)[0] = -5
    st = from_row(row)
    assert st["n"] == -5 and st["E"] == row[0, 0] and np.array_equal(st["hp"], row[:, 5:])
    assert np.array_equal(to_row(st).view(np.int32), row.view(np.int32))


P_MUT = dict(DEFAULTS, settle=4, alpha=float(np.float32(0.01)), rise=0.05, fall=0.05)


def mutant_cases():
    """mutant -> (state, hop): a gated, rate-limited hop of two channels at different levels (the ramp, the weight,
    channel 0's power, the rise clamp); a hop over the absolute gate and 30 dB under the estimate (the relative gate);
    the hop that reaches `settle` (d one hop late)"""
    x = voice(2, 40, 9, db=-6.0)
    st = model_state(2)
    model_run(x[:, :30 * HOP], [30], P_MUT, st)
    hop = x[:, 30 * HOP:31 * HOP]
    a = dict(st, n=5, g=-6.0, E=st["E"] * 0.5)
    b = dict(st, n=5, E=st["E"] * 1000)
    c = dict(st, n=P_MUT["settle"] - 1)
    return {"early": (a, hop), "weight": (a, hop), "channel0": (a, hop), "rise": (a, hop), "relative": (b, hop),
            "settle": (c, hop)}


def kernel_like(st, x, p):
    """the model's own hop as a kernel's result: its end state and output"""
    m = dict(st, shelf=st["shelf"].copy(), hp=st["hp"].copy())
    y = model_hop(m, x, p, FILTERS32)
    return dict(m, y=y)


def test_bounds_are_zero_where_the_arithmetic_is_exact():
    st, x = model_state(3), np.zeros((3, HOP))
    errs = hop_errors(st, x, P_MUT, kernel_like(st, x, P_MUT))
    assert all(v == 0 for v in errs.values())
    x = voice(3, 1, 4)                                            # 0 dB at both ends: the input itself
    got = kernel_like(st, x, P_MUT)
    assert np.array_equal(got["y"], x) and hop_errors(st, x, P_MUT, dict(got, y=x * (1 + U)))["y"] == math.inf


def test_mutants_miss_their_bounds():
    for mutant, (st, x) in mutant_cases().items():
        got = kernel_like(st, x, P_MUT)
        assert max(hop_errors(st, x, P_MUT, got).values()) < 1e-6, mutant      # lfilter's float64 roundings
        assert max(hop_errors(st, x, P_MUT, got, mutant).values()) >= SENSITIVITY, mutant


# ---- the library -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from lookoncetohear_b200 import build, _cabi
    build.build()
    return _cabi.lib()


def test_entries_exported_and_declared(lib):
    from lookoncetohear_b200 import _cabi
    hdr = header()
    for name in ENTRIES:
        assert hasattr(lib, name), name
        assert name in _cabi.declared_symbols(), name
        assert declaration(hdr, name)[0] is not None, name
    import lookoncetohear_b200 as pkg
    assert "Leveler" in pkg.__all__ and "Leveler" in pkg.__doc__


def test_layout(lib):
    row = ctypes.c_int32(-1)
    for C in (1, 2, 8, 1000):
        assert lib.l2h_leveler_layout(C, ctypes.byref(row)) == 0 and row.value == FLOATS
    assert lib.l2h_leveler_layout(2, None) == 1 and b"null" in lib.l2h_last_error()
    assert lib.l2h_leveler_layout(0, ctypes.byref(row)) == 1 and b"channels" in lib.l2h_last_error()


def test_header_documents_the_leveler():
    hdr = header()
    _, args = declaration(hdr, "l2h_leveler")
    assert args == ["y_dev", "y_row_stride", "y_ch_stride", "out_dev", "out_row_stride", "out_ch_stride", "n", "R",
                    "channels", "frames", "records_dev", "offsets_dev", "hops_dev", "state_dev", "n_rows", "target",
                    "gate", "relative", "alpha", "settle_hops", "min_gain", "max_gain", "rise_step", "fall_step", "stream"]
    assert declaration(hdr, "l2h_leveler_layout")[1] == ["channels", "row_floats"]
    doc = doc_before(hdr, hdr.index("int l2h_leveler_layout("))
    for phrase in ("one gain for all channels", "BS.1770", "libebur128", "-0.691 + 10 log10 P", "relative",
                   "max(alpha, 1 / (n + 1))", "settle_hops", "bit for bit", "not measured", "before anything is enqueued",
                   "CUDA graph", "All zeros is a fresh row", "stores nothing", "y itself", "no added delay"):
        assert phrase in doc, phrase
    assert "l2h_leveler" in hdr[:hdr.index("#ifndef")]


# argument errors: fake device addresses far apart, so only the argument under test is wrong
Y, OUT, LIST, ST = (ctypes.c_void_p(a) for a in (0x1000000, 0x2000000, 0x4000000, 0x5000000))
OK = {"target": -20.0, "gate": -50.0, "relative": -20.0, "alpha": 0.00266, "settle": 32, "min_gain": -12.0,
      "max_gain": 12.0, "rise": 0.024, "fall": 0.08}


def _call(lib, y=Y, y_row=None, y_ch=None, out=OUT, o_row=None, o_ch=None, n=2, R=3, C=2, T=3, records=LIST,
          offsets=LIST, hops=None, st=ST, rows=4, **kw):
    v = dict(OK, **kw)
    y_ch = HOP * T if y_ch is None else y_ch
    o_ch = HOP * T if o_ch is None else o_ch
    y_row = C * y_ch if y_row is None else y_row
    o_row = C * o_ch if o_row is None else o_row
    return lib.l2h_leveler(y, y_row, y_ch, out, o_row, o_ch, n, R, C, T, records, offsets, hops, st, rows, v["target"],
                           v["gate"], v["relative"], v["alpha"], v["settle"], v["min_gain"], v["max_gain"], v["rise"],
                           v["fall"], None)


def test_call_argument_errors(lib):
    for kw in ({"y": None}, {"out": None}, {"records": None}, {"st": None}):
        assert _call(lib, **kw) == 1, kw
        assert b"null" in lib.l2h_last_error()
    for kw in ({"n": 0}, {"R": 0}, {"C": 0}, {"T": 0}, {"rows": 0}, {"n": -1}, {"T": -3}):
        assert _call(lib, **kw) == 1, kw
        assert b"positive" in lib.l2h_last_error(), kw
    assert _call(lib, n=5, R=6, rows=4) == 1 and b"n <= n_slots" in lib.l2h_last_error()
    assert _call(lib, n=4, R=3) == 1 and b"n <= R" in lib.l2h_last_error()
    assert _call(lib, T=2 ** 24, y_ch=2 ** 31, o_ch=2 ** 31) == 1 and b"frames" in lib.l2h_last_error()
    for k in ("target", "gate", "relative", "min_gain", "max_gain"):
        for v in (float("nan"), float("inf"), -float("inf")):
            assert _call(lib, **{k: v}) == 1 and b"finite" in lib.l2h_last_error(), (k, v)
    assert _call(lib, relative=0.5) == 1 and b"relative" in lib.l2h_last_error()
    for a in (0.0, -0.1, 1.5, float("nan")):
        assert _call(lib, alpha=a) == 1 and b"alpha" in lib.l2h_last_error(), a
    for lo, hi in ((3.0, 2.0), (-41.0, 0.0), (0.0, 40.5)):
        assert _call(lib, min_gain=lo, max_gain=hi) == 1 and b"gain range" in lib.l2h_last_error(), (lo, hi)
    for kw in ({"rise": -0.1}, {"fall": -1.0}, {"rise": float("inf")}, {"fall": float("nan")}):
        assert _call(lib, **kw) == 1 and b"rise_step" in lib.l2h_last_error(), kw
    for s in (0, -5):
        assert _call(lib, settle=s) == 1 and b"settle_hops" in lib.l2h_last_error(), s
    for kw in ({"y_ch": 383}, {"y_row": 2 * 384 - 1}, {"o_ch": 100}, {"o_row": 384}):
        assert _call(lib, **kw) == 1, kw
        assert b"stride" in lib.l2h_last_error(), kw
    for kw in ({"out": ctypes.c_void_p(0x1000000 + 4)}, {"out": Y, "o_row": 4 * 384},
               {"out": ctypes.c_void_p(0x1000000 + 4 * (3 * 2 * 384 - 1))}, {"out": ctypes.c_void_p(0x1000000 - 4)}):
        assert _call(lib, **kw) == 1, kw
        assert b"overlap" in lib.l2h_last_error(), kw


# ---- the Python checks -----------------------------------------------------------------------------------------------
def test_constructor_checks():
    for bad in ({"rows": 0}, {"channels": 0}, {"target": float("nan")}, {"gate": float("inf")}, {"relative": 1.0},
                {"window": 0.0}, {"window": -1.0}, {"settle": 0.0}, {"settle": -0.1}, {"min_gain": 3.0, "max_gain": 1.0},
                {"min_gain": -41.0}, {"max_gain": 40.5}, {"rise": -1.0}, {"fall": -0.5}, {"target": True},
                {"fall": "10"}):
        kw = {"rows": 4, "channels": 2, "device": "cuda"}
        kw.update(bad)
        with pytest.raises(ValueError):
            Leveler(**kw)
    with pytest.raises(RuntimeError, match="CUDA"):
        Leveler(4, 2, device="cpu")


def test_per_hop_quantities(monkeypatch):
    """alpha, settle hops and dB steps from seconds and dB/s at 128 samples per hop of 16 kHz"""
    got = {}
    monkeypatch.setattr(Leveler, "_allocate", lambda self, row, device: got.update(row=row))
    lev = Leveler(4, 2)
    assert got["row"] == FLOATS
    assert lev.alpha == pytest.approx(DEFAULTS["alpha"], rel=1e-15) and lev.settle_hops == 32
    assert lev.rise_step == pytest.approx(0.024) and lev.fall_step == pytest.approx(0.08)
    assert (lev.target, lev.gate, lev.relative, lev.min_gain, lev.max_gain) == (-20.0, -50.0, -20.0, -12.0, 12.0)
    assert Leveler(4, 2, settle=0.001).settle_hops == 1 and Leveler(4, 2, window=1e-9).alpha == pytest.approx(1.0)


def _host_leveler(rows=4, C=2):
    """a Leveler whose state lives in host memory: the Python checks run, no engine call is reached"""
    lev = Leveler.__new__(Leveler)
    lev.n_slots, lev.channels = rows, C
    lev.state = torch.zeros(rows, C, FLOATS)
    return lev


def test_call_needs_cuda():
    lev = _host_leveler()
    with pytest.raises(RuntimeError, match="CUDA"):
        lev(torch.zeros(2, 2, 256), [0, 1])


def test_telemetry_views_and_reset():
    lev = _host_leveler()
    assert lev.loudness.tolist() == [-math.inf] * 4 and not lev.gain.any()
    lev.state[2, 0, 0] = 0.01                                     # E: -20 dB of power
    lev.state[2, 0, 1:2].view(torch.int32)[0] = 5
    lev.state[2, 0, 2] = -3.5
    lev.state[1, 0, 0] = 0.5                                      # an estimate with no gated hop reads -inf
    assert lev.loudness[2].item() == pytest.approx(-20.691, abs=1e-4)
    assert lev.loudness[[0, 1, 3]].tolist() == [-math.inf] * 3
    assert lev.gain.tolist() == [0.0, 0.0, -3.5, 0.0]
    lev.reset([2])
    assert not lev.state[2].any() and lev.state[1, 0, 0] == 0.5
