"""Host-side checks of the limiter, no device: a float64 numpy model of the look-ahead limiter (l2h_limiter, the reference
of tests/test_limiter_gpu.py) with its own checks; the layout; the argument errors of both C entries, returned before
anything is enqueued; the Python checks of Limiter; the header; the exports."""
import ctypes
import itertools
import math

import numpy as np
import pytest
import torch

from kernels.scaffold import SENSITIVITY, ratio
from lookoncetohear_b200 import Limiter
from serving_util import FAKE_DEV, declaration, doc_before, header

Q, MUTE, HEAD = 65536, 150 * 65536, 4
CEILING = float(np.float32(10 ** (-1 / 20)))
ENTRIES = ("l2h_limiter_layout", "l2h_limiter")


# ---- the model -------------------------------------------------------------------------------------------------------
def model_state(C, La):
    """a fresh slot: the delay line, the q and r histories, r of the last sample, the slot's ceiling (0: the call's), the
    samples limited and the dB of reduction at the last sample"""
    return {"xd": np.zeros((C, La)), "qh": np.zeros(La, np.int64), "rh": np.zeros(La, np.int64), "r": 0, "ceil": 0.0,
            "limited": 0, "db": 0.0}


FLT_MIN, FLT_MAX = float(np.finfo(np.float32).tiny), float(np.finfo(np.float32).max)
INT32_MAX = 2 ** 31 - 1
U = 2.0 ** -24

# Mutants of the model, each a plausible kernel bug (model_push(mutant=...)): the hold one sample short, the box one
# sample short, r carried in from 0, the slot's ceiling ignored, a non-finite sample's level taken as 0 instead of muting.
MUTANTS = ("hold", "box", "carry", "ceiling", "nonfinite")


def q_words(x, lim, mutant=None):
    """each sample's q [n] and where Q log2(p / ceiling) lies within 1e-9 of an integer, so that the device's double
    log2 may round the other way [n]"""
    finite = np.isfinite(x)
    p = np.abs(np.where(finite, x, 0.0)).max(0)
    q = np.zeros(p.shape, np.int64)
    near = np.zeros(p.shape, bool)
    over = p > lim
    v = Q * np.log2(p[over] / lim)
    q[over] = np.minimum(MUTE, np.ceil(v) + 1).astype(np.int64)
    near[over] = np.abs(v - np.round(v)) < 1e-9
    if mutant != "nonfinite":
        q[~finite.all(0)] = MUTE
    return q, near


def model_push(st, x, ceiling, La, step, mutant=None, q=None, trace=None):
    """l2h_limiter on one slot: x [C, n] float64 (float32 values) pushed, returns y [C, n]; advances st.  As in the
    kernel, the slot's ceiling applies where it is a positive normal float, history and r words count within [0, MUTE]
    and the count of limited samples saturates; q: the push's q words, when not the model's own; trace: a dict that
    receives the box sums a."""
    C, n = x.shape
    c = st["ceil"]
    lim = c if FLT_MIN <= c <= FLT_MAX and mutant != "ceiling" else ceiling
    if q is None:
        q = q_words(x, lim, mutant)[0]
    qa = np.concatenate([np.clip(st["qh"], 0, MUTE), q])
    s = np.lib.stride_tricks.sliding_window_view(qa, La + 1).max(1)                # q[k - La .. k]
    if mutant == "hold" and La:
        s = np.lib.stride_tricks.sliding_window_view(qa[1:], La).max(1)
    k = np.arange(n, dtype=np.int64)
    r_in = 0 if mutant == "carry" else min(max(st["r"], 0), MUTE)
    r = np.maximum(r_in - (k + 1) * step, np.maximum.accumulate(s + k * step) - k * step)
    ra = np.concatenate([np.clip(st["rh"], 0, MUTE), r])
    a = np.lib.stride_tricks.sliding_window_view(ra, La + 1).sum(1)                # r[k - La .. k]
    if mutant == "box" and La:
        a = np.lib.stride_tricks.sliding_window_view(ra[1:], La).sum(1)
    g = np.where(a >= MUTE * (La + 1), 0.0, 2.0 ** (-a / (Q * (La + 1))))
    xs = np.concatenate([st["xd"], x], 1)
    xd = xs[:, :n]
    y = np.where(np.isfinite(xd), g * np.where(np.isfinite(xd), xd, 0.0), 0.0)
    st.update(xd=xs[:, n:], qh=qa[n:], rh=ra[n:], r=int(r[-1]),
              limited=min(INT32_MAX, max(st["limited"], 0) + int((a > 0).sum())),
              db=float(a[-1] / (Q * (La + 1)) * 20 * math.log10(2)))
    if trace is not None:
        trace["a"] = a
    return y


def from_row(row, La):
    """a slot's state rows [C, 4 + 3 La] as the kernel keeps them (fp32) -> the model's state; int32 words as they are"""
    r = np.ascontiguousarray(row, np.float32)
    i = r.view(np.int32)
    return {"xd": r[:, HEAD:HEAD + La].astype(np.float64), "qh": i[0, HEAD + La:HEAD + 2 * La].astype(np.int64),
            "rh": i[0, HEAD + 2 * La:].astype(np.int64), "r": int(i[0, 0]), "ceil": float(r[0, 1]),
            "limited": int(i[0, 2]), "db": float(r[0, 3])}


def to_row(st, C):
    La = st["qh"].shape[0]
    row = np.zeros((C, HEAD + 3 * La), np.float32)
    i = row.view(np.int32)
    i[0, 0], row[0, 1], i[0, 2], row[0, 3] = st["r"], st["ceil"], st["limited"], st["db"]
    row[:, HEAD:HEAD + La] = st["xd"]
    i[0, HEAD + La:HEAD + 2 * La], i[0, HEAD + 2 * La:] = st["qh"], st["rh"]
    return row


def push_bound(x, xd, a, La):
    """the bound of each output sample of a push whose box sums are a [n] (the model's), its delayed inputs xd [C, n]:
    0 where a = 0 (the input itself), where a mutes (exactly 0) and where x is not finite (0); else the gain 2^-e as
    exp2f of the fraction's fp32 rounding (2 ulp) times 2^-floor(e), the product's rounding, and 2^-149 where ldexpf
    rounds a subnormal result"""
    e = a / (Q * (La + 1))
    f = e - np.floor(e)
    gf = 2.0 ** -f
    eg = gf * math.log(2) * (U * f + 2.0 ** -50) + 2.0 ** -23
    b = 2.0 ** -np.floor(e) * np.abs(np.where(np.isfinite(xd), xd, 0.0)) * (eg + U * gf) * (1 + 4 * U) + 2.0 ** -149
    return np.where((a == 0) | (a >= MUTE * (La + 1)) | ~np.isfinite(xd), 0.0, b)


def push_errors(st, x, ceiling, La, step, got, mutant=None):
    """error / bound of a push run from state st, got = from_row() of the state it ended with plus its output "y":
    every integer word and the delay line bit for bit (inf where one differs), y within push_bound and the reduction
    word within its double-to-float rounding.  Where q is within 1e-9 of a quantum's edge either q is accepted: the
    variant whose words match the kernel's is compared."""
    c = st["ceil"]
    lim = c if FLT_MIN <= c <= FLT_MAX and mutant != "ceiling" else ceiling
    q, near = q_words(x, lim, mutant)
    best = None
    for bump in itertools.product((0, 1), repeat=min(int(near.sum()), 4)):
        qv = q.copy()
        qv[np.flatnonzero(near)[:len(bump)]] -= np.array(bump, np.int64)
        m = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in st.items()}
        tr = {}
        y = model_push(m, x, ceiling, La, step, mutant, qv, tr)
        same = all(np.array_equal(got[k], m[k]) for k in ("qh", "rh")) and got["r"] == m["r"] and \
            got["limited"] == m["limited"] and np.float32(got["ceil"]).view(np.int32) == np.float32(st["ceil"]).view(np.int32)
        same = same and np.array_equal(np.asarray(got["xd"], np.float32).view(np.int32),
                                       np.asarray(m["xd"], np.float32).view(np.int32))
        xd = np.concatenate([st["xd"], x], 1)[:, :x.shape[1]]
        errs = {"words": 0.0 if same else math.inf,
                "y": ratio(got["y"], y, push_bound(x, xd, tr["a"], La)),
                "db": ratio(got["db"], m["db"], U * abs(m["db"]) * (1 + 2.0 ** -20))}
        if best is None or max(errs.values()) < max(best.values()):
            best = errs
    return best


def model_run(x, pushes, ceiling=CEILING, La=16, step=20):
    """x [C, N] in pushes of the given lengths through a fresh slot: (y [C, sum(pushes)], the final state)"""
    st, ys, pos = model_state(x.shape[0], La), [], 0
    for m in pushes:
        if m:
            ys.append(model_push(st, x[:, pos:pos + m], ceiling, La, step))
        pos += m
    return np.concatenate(ys, 1), st


def loud(C, N, seed, peak=6.9):
    """a seeded speech-like stereo signal: bursts of two partials and noise at levels up to `peak`, the channels at
    different levels (an ILD), rounded to float32"""
    g = np.random.default_rng(seed)
    t = np.arange(N) / 16000
    env = np.repeat(g.uniform(0.05, 1.0, N // 400 + 1), 400)[:N] * peak
    sig = env * (np.sin(2 * np.pi * 220 * t) + 0.5 * np.sin(2 * np.pi * 1330 * t) + 0.3 * g.standard_normal(N)) / 1.8
    return np.stack([sig * (0.6 + 0.4 * c / max(C - 1, 1)) for c in range(C)]).astype(np.float32).astype(np.float64)


def cuts(N, seed, hi=400):
    g = np.random.default_rng(seed)
    out = []
    while sum(out) < N:
        out.append(int(min(g.integers(0, hi), N - sum(out))))
    return out


# ---- the model's own checks ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("La", [0, 1, 16, 44])
def test_model_holds_the_ceiling_and_links_the_channels(La):
    x = loud(2, 16000, 1)
    y, st = model_run(x, [16000], La=La)
    assert np.abs(y).max() <= CEILING and np.abs(y).max() > 0.99 * CEILING
    xd = np.pad(x, ((0, 0), (La, 0)))[:, :16000]
    live = np.abs(xd[0]) > 1e-6
    assert np.abs(y[1][live] / y[0][live] - xd[1][live] / xd[0][live]).max() < 1e-12      # one gain for both channels
    assert st["limited"] > 0 and st["r"] >= 0


def test_model_is_transparent_below_the_ceiling():
    x = loud(2, 4000, 2, peak=0.5)
    assert np.abs(x).max() <= CEILING
    y, st = model_run(x, [1000, 3000], La=16)
    assert np.array_equal(y, np.pad(x, ((0, 0), (16, 0)))[:, :4000]) and st["limited"] == 0


def test_model_split_invariance():
    """the same stream cut into 400 random pushes (zeros included): the same output and state, exactly"""
    x = loud(2, 40000, 3)
    y, st = model_run(x, [40000], La=44, step=19)
    for seed in (4, 5):
        y2, st2 = model_run(x, cuts(40000, seed), La=44, step=19)
        assert np.array_equal(y, y2)
        assert all(np.array_equal(st[k], st2[k]) for k in st)


def test_state_row_round_trips():
    row = (np.arange(3 * (HEAD + 3 * 5)).reshape(3, -1) * 0.37 - 2).astype(np.float32)
    i = row.view(np.int32)
    i[0, 0], i[0, 2], i[0, HEAD + 5:] = -7, INT32_MAX - 3, np.arange(10) * 70000 - 3
    row[1:, :HEAD], row[1:, HEAD + 5:] = 0, 0
    st = from_row(row, 5)
    assert st["r"] == -7 and st["limited"] == INT32_MAX - 3 and st["qh"][0] == -3
    assert np.array_equal(to_row(st, 3).view(np.int32), i)


def mutant_case():
    """a push of 2 channels with peaks over the slot's own ceiling and a NaN, from a slot releasing a large r"""
    La = 8
    st = model_state(2, La)
    st.update(r=3 * Q, ceil=0.5, rh=np.full(La, 3 * Q), qh=np.full(La, Q))
    x = loud(2, 300, 11, peak=12.0)
    x[1, 250] = np.nan
    return st, x, La


def kernel_like(st, x, La, step=20):
    m = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in st.items()}
    y = model_push(m, x, CEILING, La, step)
    return dict(m, y=y, db=float(np.float32(m["db"])))


def test_bounds_are_zero_where_the_arithmetic_is_exact():
    st = model_state(2, 4)
    x = loud(2, 200, 12, peak=0.5)                                 # under the ceiling: a = 0, the input delayed
    assert not push_bound(x, x, np.zeros(200, np.int64), 4).any()
    assert not push_bound(x, x, np.full(200, MUTE * 5), 4).any()  # muted: exactly 0
    assert max(push_errors(st, x, CEILING, 4, 20, kernel_like(st, x, 4)).values()) == 0


def test_mutants_miss_their_bounds():
    st, x, La = mutant_case()
    got = kernel_like(st, x, La, 2000)
    assert max(push_errors(st, x, CEILING, La, 2000, got).values()) <= 1.0
    for mutant in MUTANTS:
        assert max(push_errors(st, x, CEILING, La, 2000, got, mutant).values()) >= SENSITIVITY, mutant


def test_model_release_and_mute():
    """a single peak: the reduction reaches it La samples ahead, then recovers by `step` quanta a sample; a NaN writes 0,
    mutes its own time step in every channel, and the state stays finite"""
    La, step = 8, 1000
    x = np.full((2, 400), 0.25)
    x[0, 50] = 4 * CEILING                                       # 2 octaves over: q = 2 Q + 1
    y, st = model_run(x, [400], La=La, step=step)
    assert abs(y[0, 50 + La]) <= CEILING and y[1, 50 + La] == pytest.approx(0.25 * CEILING / (4 * CEILING), rel=1e-4)
    assert np.array_equal(y[:, :50], np.pad(x, ((0, 0), (La, 0)))[:, :50])         # before the look-ahead: untouched
    assert st["r"] == 0 and st["limited"] == La + 1 + math.ceil((2 * Q + 1) / step) + La - 1
    x[1, 200] = np.nan
    y, st = model_run(x, [200, 200], La=La, step=step)
    assert y[1, 200 + La] == 0 and y[0, 200 + La] == 0 and np.isfinite(y).all()
    assert st["r"] == MUTE - (399 - 200 - La) * step and np.isfinite(st["db"])


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
    assert "Limiter" in pkg.__all__ and "Limiter" in pkg.__doc__


def test_layout(lib):
    row = ctypes.c_int32(-1)
    for C, La in ((1, 0), (2, 44), (2, 48), (8, 1000)):
        assert lib.l2h_limiter_layout(C, La, ctypes.byref(row)) == 0 and row.value == HEAD + 3 * La
    assert lib.l2h_limiter_layout(2, 44, None) == 1 and b"null" in lib.l2h_last_error()
    assert lib.l2h_limiter_layout(0, 44, ctypes.byref(row)) == 1 and b"channels" in lib.l2h_last_error()
    assert lib.l2h_limiter_layout(2, -1, ctypes.byref(row)) == 1 and b"negative" in lib.l2h_last_error()
    assert lib.l2h_limiter_layout(2, 3072, ctypes.byref(row)) == 2 and b"shared memory" in lib.l2h_last_error()
    assert lib.l2h_limiter_layout(2, 3071, ctypes.byref(row)) == 0


def test_header_documents_the_limiter():
    hdr = header()
    _, args = declaration(hdr, "l2h_limiter")
    assert args == ["x_dev", "x_row_stride", "x_ch_stride", "max_in", "counts_dev", "unit", "y_dev", "y_row_stride",
                    "y_ch_stride", "n", "channels", "slots_dev", "state_dev", "n_slots", "ceiling", "lookahead",
                    "release_step", "stream"]
    assert declaration(hdr, "l2h_limiter_layout")[1] == ["channels", "lookahead", "row_floats"]
    doc = doc_before(hdr, hdr.index("int l2h_limiter_layout("))
    for phrase in ("one gain for all channels", "after the up-resampler", "|y| <= ceiling exactly", "bit for bit",
                   "before anything is enqueued", "CUDA graph", "All zeros is a fresh slot", "stores nothing",
                   "not finite", "exceeds the kernel's shared memory", "Q = 65536"):
        assert phrase in doc, phrase
    assert "l2h_limiter" in hdr[:hdr.index("#ifndef")]


# argument errors: fake device addresses far apart, so only the argument under test is wrong
X, Y, LIST, ST = (ctypes.c_void_p(a) for a in (0x1000000, 0x2000000, 0x4000000, 0x5000000))


def _call(lib, x=X, x_row=None, x_ch=None, max_in=441, counts=LIST, unit=1, y=Y, y_row=None, y_ch=None, n=2, C=2,
          slots=LIST, st=ST, S=4, ceiling=CEILING, La=44, step=20):
    x_ch = max_in if x_ch is None else x_ch
    y_ch = max_in if y_ch is None else y_ch
    x_row = C * x_ch if x_row is None else x_row
    y_row = C * y_ch if y_row is None else y_row
    return lib.l2h_limiter(x, x_row, x_ch, max_in, counts, unit, y, y_row, y_ch, n, C, slots, st, S, ceiling, La, step,
                           None)


def test_call_argument_errors(lib):
    for kw in ({"x": None}, {"counts": None}, {"y": None}, {"slots": None}, {"st": None}):
        assert _call(lib, **kw) == 1, kw
        assert b"null" in lib.l2h_last_error()
    for kw in ({"n": 0}, {"C": 0}, {"max_in": 0}, {"unit": 0}, {"S": 0}, {"n": -1}, {"unit": -128}):
        assert _call(lib, **kw) == 1, kw
        assert b"positive" in lib.l2h_last_error(), kw
    assert _call(lib, n=5, S=4) == 1 and b"n <= n_slots" in lib.l2h_last_error()
    for c in (0.0, -1.0, 1e-39, float("inf"), float("nan")):
        assert _call(lib, ceiling=c) == 1 and b"ceiling" in lib.l2h_last_error(), c
    for step in (0, -1, MUTE + 1):
        assert _call(lib, step=step) == 1 and b"release_step" in lib.l2h_last_error(), step
    assert _call(lib, La=-1) == 1 and b"negative" in lib.l2h_last_error()
    assert _call(lib, max_in=6000) == 2 and b"shared memory" in lib.l2h_last_error()
    for kw in ({"x_ch": 440}, {"x_row": 2 * 441 - 1}, {"y_ch": 100}, {"y_row": 441}):
        assert _call(lib, **kw) == 1, kw
        assert b"stride" in lib.l2h_last_error(), kw
    for kw in ({"y": X}, {"y": ctypes.c_void_p(0x1000000 + 4 * (2 * 2 * 441 - 1))}, {"y": ctypes.c_void_p(0x1000000 - 4)}):
        assert _call(lib, **kw) == 1, kw
        assert b"overlap" in lib.l2h_last_error(), kw


def test_layout_errors_come_before_the_call(lib):
    """the call refuses a look-ahead or push its layout cannot stage with code 2, before reading any pointer"""
    assert _call(lib, La=3072, max_in=1) == 2
    assert _call(lib, C=8, La=1000, max_in=600, x=FAKE_DEV, y=ctypes.c_void_p(0x9000000)) == 2


# ---- the Python checks -----------------------------------------------------------------------------------------------
def test_constructor_checks():
    for bad in ({"slots": 0}, {"channels": 0}, {"rate": 0}, {"rate": 44100.5}, {"ceiling": 0.0}, {"ceiling": -1.0},
                {"ceiling": float("nan")}, {"ceiling": 1e39}, {"ceiling": 1e-50}, {"ceiling": True},
                {"lookahead": -0.001}, {"lookahead": float("inf")}, {"release": 0.0}, {"release": -3.0},
                {"release": float("inf")}, {"release": 1e12}, {"lookahead": 0.1}):
        kw = {"slots": 4, "channels": 2, "rate": 44100, "device": "cuda"}
        kw.update(bad)
        with pytest.raises(ValueError):
            Limiter(**kw)
    with pytest.raises(RuntimeError, match="CUDA"):
        Limiter(4, 2, 44100, device="cpu")


def test_samples_and_steps(monkeypatch):
    """La and the release step from seconds and dB/s: 1 ms is 44 samples at 44.1 kHz, 80 dB/s is 20 quanta a sample"""
    got = {}
    monkeypatch.setattr(Limiter, "_allocate", lambda self, row, device: got.update(row=row))
    lim = Limiter(4, 2, 44100)
    assert (lim.lookahead, lim.release_step, got["row"]) == (44, 20, HEAD + 3 * 44)
    assert lim.ceiling == CEILING
    assert Limiter(4, 2, 48000).lookahead == 48 and Limiter(4, 2, 16000, lookahead=0).lookahead == 0
    assert Limiter(4, 2, 16000, release=1e-3).release_step == 1                       # at least one quantum
    assert Limiter(4, 2, 16000, release=480.0).release_step == round(480 / (20 * math.log10(2)) * Q / 16000)


def _host_limiter(S=4, C=2, La=44):
    """a Limiter whose state lives in host memory: the Python checks run, no engine call is reached"""
    lim = Limiter.__new__(Limiter)
    lim.n_slots, lim.channels, lim.rate, lim.ceiling, lim.lookahead, lim.release_step = S, C, 44100, CEILING, La, 20
    lim.state = torch.zeros(S, C, HEAD + 3 * La)
    return lim


def test_call_needs_cuda():
    lim = _host_limiter()
    with pytest.raises(RuntimeError, match="CUDA"):
        lim(torch.zeros(2, 2, 441), [441, 441], [0, 1])


def test_set_ceiling_and_telemetry_views():
    lim = _host_limiter()
    lim.set_ceiling([2, 0], [0.5, 0.25])
    lim.set_ceiling([3], 1.0)
    assert lim.state[:, 0, 1].tolist() == [0.25, 0.0, 0.5, 1.0] and not lim.state[:, 1].any()
    lim.set_ceiling(torch.tensor([3]), 0)                                   # back to the default
    assert lim.state[3, 0, 1] == 0
    for slots, values in (([4], 0.5), ([-1], 0.5), ([1, 1], 0.5), ([], 0.5), ([0], -0.5), ([0], float("nan")),
                          ([0], float("inf")), ([0], 1e39), ([0], True), ([0, 1], [0.5]), ([0.5], 0.5)):
        with pytest.raises(ValueError):
            lim.set_ceiling(slots, values)
    lim.state[1, 0, 2:3].view(torch.int32)[0] = 1234
    lim.state[1, 0, 3] = 6.5
    assert lim.limited.tolist() == [0, 1234, 0, 0] and lim.limited.dtype == torch.int32
    assert lim.reduction.tolist() == [0.0, 6.5, 0.0, 0.0]
    lim.reset([1, 2])
    assert not lim.limited.any() and not lim.reduction.any() and lim.state[2, 0, 1] == 0
