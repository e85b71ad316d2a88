"""Host-side checks of the limiter, no device: a float64 numpy model of the look-ahead limiter (l2h_limiter, the reference
of tests/test_limiter_gpu.py) with its own checks; the layout; the argument errors of both C entries, returned before
anything is enqueued; the Python checks of Limiter; the header; the exports."""
import ctypes
import math

import numpy as np
import pytest
import torch

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


def model_push(st, x, ceiling, La, step):
    """l2h_limiter on one slot: x [C, n] float64 (float32 values) pushed, returns y [C, n]; advances st"""
    C, n = x.shape
    lim = st["ceil"] if st["ceil"] > 0 else ceiling
    finite = np.isfinite(x)
    p = np.abs(np.where(finite, x, 0.0)).max(0)
    q = np.zeros(n, np.int64)
    over = p > lim
    with np.errstate(divide="ignore"):
        q[over] = np.minimum(MUTE, np.ceil(Q * np.log2(p[over] / lim)) + 1).astype(np.int64)
    q[~finite.all(0)] = MUTE
    qa = np.concatenate([st["qh"], q])
    s = np.lib.stride_tricks.sliding_window_view(qa, La + 1).max(1)                # q[k - La .. k]
    k = np.arange(n, dtype=np.int64)
    r = np.maximum(st["r"] - (k + 1) * step, np.maximum.accumulate(s + k * step) - k * step)
    ra = np.concatenate([st["rh"], r])
    a = np.lib.stride_tricks.sliding_window_view(ra, La + 1).sum(1)                # r[k - La .. k]
    g = np.where(a >= MUTE * (La + 1), 0.0, 2.0 ** (-a / (Q * (La + 1))))
    xs = np.concatenate([st["xd"], x], 1)
    xd = xs[:, :n]
    y = np.where(np.isfinite(xd), g * np.where(np.isfinite(xd), xd, 0.0), 0.0)
    st.update(xd=xs[:, n:], qh=qa[n:], rh=ra[n:], r=int(r[-1]), limited=min(2 ** 31 - 1, st["limited"] + int((a > 0).sum())),
              db=float(a[-1] / (Q * (La + 1)) * 20 * math.log10(2)))
    return y


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
