"""Resampling without a GPU: the float64 restatement (oracle/resample.py) against torchaudio.functional.resample and its
fixture, and the argument checks of l2h_resample / lookoncetohear_b200.resample, which run before any CUDA call.  Also the
float64 models of the device's resamplers (whole signals, one push of whole periods, one packet), each with a per-sample
bound on the device's fp32 error and mutants that must miss it, the reference of test_stream_stage_kernels_gpu.py."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from oracle import resample as ors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAIRS = [(44100, 16000), (48000, 16000), (16000, 8000), (8000, 16000), (22050, 16000)]
LENGTHS = [1, 7, 200, 2000, 80000]


def rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.mark.parametrize("n", LENGTHS)
@pytest.mark.parametrize("orig,new", PAIRS)
def test_restatement_matches_torchaudio(orig, new, n):
    AF = pytest.importorskip("torchaudio.functional")
    x = np.random.default_rng(orig + n).standard_normal(n)
    y_ta = AF.resample(torch.from_numpy(x), orig, new).numpy()    # float64: torchaudio's filter is built in x's dtype
    y = ors.resample(x, orig, new)
    assert y.shape == y_ta.shape == (ors.output_length(n, orig, new),)
    assert rel(y, y_ta) <= 1e-6


def test_restatement_reproduces_fixture():
    g = np.load(os.path.join(ROOT, "tests", "golden", "resample_golden.npz"))
    xl = np.random.default_rng(int(g["long_seed"])).standard_normal(80000)
    np.testing.assert_allclose([xl.sum(), (xl ** 2).sum()], g["long_checksum"], rtol=1e-12)
    for orig, new in PAIRS:
        for n in LENGTHS[:-1]:
            ref = g[f"y_{orig}_{new}_{n}"]
            y = ors.resample(g[f"x_{n}"], orig, new)
            assert y.shape == ref.shape and rel(y, ref) <= 1e-6, (orig, new, n)
        y = ors.resample(xl, orig, new)
        key = f"y_{orig}_{new}_80000"
        assert y.size == int(g[key + "_len"])
        assert abs(np.linalg.norm(y) / float(g[key + "_norm"]) - 1) <= 1e-6
        assert rel(y[g[key + "_idx"]], g[key + "_val"]) <= 1e-6


def test_restatement_identity_and_lengths():
    x = np.random.default_rng(0).standard_normal((3, 101))
    assert np.array_equal(ors.resample(x, 16000, 16000), x)
    assert ors.resample(x, 44100, 16000).shape == (3, 37)                     # ceil(16000 * 101 / 44100)
    assert ors.output_length(80000, 16000, 8000) == 40000
    assert ors.output_length(1, 8000, 16000) == 2


# ---- the device's sample, in float64, and a bound on its error ---------------------------------------------------------
# rs_output (csrc/resample.cu) weighs the taps c - w .. c + w of output m (c = floor(m o / q), phase r = m o - c q) with
# u = r base / (o q) + (w - t) base / o, computed in fp64 and rounded to fp32, then h(u) = (base / o) sinc(u) cos^2(pi u / 12)
# in fp32 and the sum in fp32 fmaf.  The build has no --use_fast_math, so x / y is the IEEE division (0.5 ulp); the CUDA
# Math API documents sinpif and cospif at 1 ulp.  1 ulp of a value v is at most 2 u |v|, u = 2^-24.
U = 2.0 ** -24
WIDTH = 6
RS_MUTANTS = ("rolloff", "window", "taps", "phase", "u_fp32", "scale")
STREAM_MUTANTS = ("delay_plus", "delay_minus", "count_ignored", "history_shifted")
PACKET_MUTANTS = STREAM_MUTANTS + ("phase_word_ignored",)


def rs_filter(orig, new):
    """(o, q, w, base) of orig -> new Hz"""
    g = math.gcd(orig, new)
    o, q = orig // g, new // g
    base = min(o, q) * ors.ROLLOFF
    return o, q, math.ceil(WIDTH * o / base), base


def rs_weights(u, base, o, q, mutant=None):
    """the exact weights h(u) and their derivative dh/du"""
    rolloff = 0.985 / 0.99 if mutant == "rolloff" else 1.0
    b = base * rolloff
    v = u * rolloff
    half = 2 * WIDTH + (1 if mutant == "window" else 0)
    scale = b / (q if mutant == "scale" else o)
    live = np.abs(v) < WIDTH
    sinc = np.sinc(v)
    win = np.cos(np.pi * v / half) ** 2
    with np.errstate(divide="ignore", invalid="ignore"):
        dsinc = np.where(v == 0, 0.0, (np.cos(np.pi * v) - sinc) / v)
    dwin = -np.pi / half * np.sin(2 * np.pi * v / half)
    return np.where(live, scale * sinc * win, 0.0), np.where(live, scale * rolloff * (dsinc * win + sinc * dwin), 0.0)


def rs_samples(win, origin, jd, o, q, w, base, m_abs=None, mutant=None):
    """(y, bound): the outputs at positions jd (int64 array) of a signal whose input n sits at win[origin + n], as
    rs_delayed / resample_kernel compute them, in float64, and a per-output bound on the device's error.  Positions whose
    taps fall outside win must not be asked for.  m_abs: the outputs' absolute positions (the "u_fp32" mutant)."""
    jd = np.asarray(jd, np.int64)
    a = jd * o
    c = a // q
    r = a - c * q
    if mutant == "phase":
        r = r + 1
    t = np.arange(2 * w + 1)
    if jd.size == 0:
        return np.zeros(0), np.zeros(0)
    X = np.asarray(win, np.float64)[(origin + c - w)[:, None] + t[None, :]]
    u = (r[:, None] / (o * q) + (w - t)[None, :] / o) * base
    if mutant == "u_fp32":                            # u in fp32 from the absolute position instead of the remainder
        f = np.float32
        m = np.asarray(m_abs if m_abs is not None else jd, np.int64)[:, None]
        n = (m * o // q - w) + t[None, :]
        u = (f(base) * (m.astype(f) / f(q) - n.astype(f) / f(o))).astype(np.float64)
    h, dh = rs_weights(u, base, o, q, mutant)
    if mutant == "taps":
        h[:, 2 * w] = 0
    near = np.abs(u) < WIDTH * (1 + 4 * U)
    near[:, 0] = False                                 # tap 0 has u >= w base / o >= 6: it never enters the sum
    h[:, 0] = 0
    Xs = np.where(near, X, 0.0)                        # a word that never enters the sum (NaN, 3e38) weighs nothing
    y = (h * Xs).sum(1)
    # the weight's error: u's rounding to fp32 times |h'|, then the fp32 evaluation (sinc 6 u relative: sinpif, the fp32
    # pi, the product and the division; window: cospif of u / 6 with 1 / 6 rounded, the half and the sum; scale and two
    # products: 3 u), and near |u| = 6 the window's absolute error where the device may still take the tap
    du = U * np.abs(u) + 1e-12
    scale = base / o
    sinc_abs = np.abs(np.where(np.abs(u) < WIDTH * (1 + 4 * U), np.sinc(u), 0.0))
    cw = np.abs(np.cos(np.pi * u / WIDTH))
    win_err = 0.5 * (2 * U * cw + 2 * np.pi * U * np.abs(u) / WIDTH) + U * (0.5 + 0.5 * cw)
    E = np.abs(dh) * du * (1 + 1e-3) + np.abs(h) * 9 * U + scale * sinc_abs * win_err * (1 + 8 * U)
    E = np.where(near, E * (1 + 16 * U), 0.0)
    K = near.sum(1)
    gamma = K * U / (1 - K * U)
    ax = np.abs(Xs)
    bound = (ax * E).sum(1) + gamma * ((np.abs(h) + E) * ax).sum(1)
    return y, bound


def whole(x, orig, new, cap, mutant=None):
    """(y, bound) of resample_kernel for one row of n_in samples into `cap` outputs (zeros past n_out, equal rates a copy)"""
    x = np.asarray(x, np.float64)
    n_in = x.shape[-1]
    if orig == new:
        y = np.zeros(cap)
        y[:n_in] = x
        return y, np.zeros(cap)
    o, q, w, base = rs_filter(orig, new)
    n_out = min(cap, ors.output_length(n_in, orig, new))
    pad = np.concatenate([np.zeros(w + 1), x, np.zeros(w + 2)])
    m = np.arange(n_out)
    y, b = np.zeros(cap), np.zeros(cap)
    y[:n_out], b[:n_out] = rs_samples(pad, w + 1, m, o, q, w, base, m_abs=m, mutant=mutant)
    return y, b


def clamp_word(v, hi):
    """a count word stored as a float, clamped into [0, hi] (NaN: 0)"""
    v = float(np.float32(v))
    return hi if v >= hi else (int(v) if v > 0 else 0)


def stream_push(st, x, orig, new, block, keep, mutant=None):
    """resample_stream_kernel for one (row, channel) pushing h blocks x [h block] onto the state row st [H + keep]:
    (y [keep + h out_block], bound, new state row)"""
    o, q, w, base = rs_filter(orig, new)
    D = w * q // o + {"delay_plus": 1, "delay_minus": -1}.get(mutant, 0)
    H = -(-(w * q // o) * o // q) + w
    st = np.asarray(st, np.float64)
    before = D if mutant == "count_ignored" else clamp_word(st[0], w * q // o)
    win = np.concatenate([[0.0], st[1:H], np.asarray(x, np.float64)])
    n_new = len(x) // o * q
    j = np.arange(n_new)
    started = before + j >= D
    origin = H + (1 if mutant == "history_shifted" else 0)
    y, b = np.zeros(n_new), np.zeros(n_new)
    if started.any():
        ys, bs = rs_samples(np.concatenate([win, np.zeros(2 * w + 4)]), origin, (j - D)[started], o, q, w, base, mutant=mutant)
        y[started], b[started] = ys, bs
    out = np.concatenate([st[H:H + keep], y])
    new = np.concatenate([[min(w * q // o, before + n_new)], win[len(win) - H + 1:], out[n_new:]])
    return out, np.concatenate([np.zeros(keep), b]), new


def packet_push(st, x, orig, new, mutant=None):
    """resample_packets_kernel for one (row, channel) pushing n > 0 samples x onto st [2 + H]: (y [n_new], bound, new
    state row)"""
    o, q, w, base = rs_filter(orig, new)
    D0 = w * q // o
    D = D0 + {"delay_plus": 1, "delay_minus": -1}.get(mutant, 0)
    H = -(-(D0 + 1) * o // q) + w + 1
    st = np.asarray(st, np.float64)
    before = D if mutant == "count_ignored" else clamp_word(st[0], D0)
    p = 0 if mutant == "phase_word_ignored" else clamp_word(st[1], o - 1)
    n = len(x)
    j0 = p * q // o
    n_new = (p + n) * q // o - j0
    win = np.concatenate([st[2:2 + H], np.asarray(x, np.float64), np.zeros(2 * w + 4)])   # room for the mutants
    k = np.arange(n_new)
    started = before + k >= D
    origin = H - p + (1 if mutant == "history_shifted" else 0)
    y, b = np.zeros(n_new), np.zeros(n_new)
    if started.any():
        y[started], b[started] = rs_samples(win, origin, (j0 + k - D)[started], o, q, w, base, mutant=mutant)
    return y, b, np.concatenate([[min(D0, before + n_new), (p + n) % o], win[n:n + H]])


def _delayed(x, orig, new, D, n):
    z = ors.resample(x, orig, new)
    return np.concatenate([np.zeros(D), z])[:n]


@pytest.mark.parametrize("orig,new", [(48000, 16000), (16000, 44100), (44100, 16000), (16000, 8000), (16001, 16000)])
def test_models_are_the_delayed_whole_signal(orig, new):
    """ragged pushes through each one-push model equal oracle.resample delayed by D, to float64 rounding; the bound is
    0 before the stream starts and past n_out"""
    o, q, w, base = rs_filter(orig, new)
    D = w * q // o
    g = np.random.default_rng(orig)
    x = g.standard_normal(12 * o + 37)
    # whole-signal
    y, b = whole(x, orig, new, ors.output_length(len(x), orig, new) + 5)
    z = ors.resample(x, orig, new)
    assert np.allclose(y[:len(z)], z, rtol=0, atol=1e-12) and not y[len(z):].any() and not b[len(z):].any()
    assert (b[:len(z)] > 0).all() and b.max() < 1e-5
    # packets
    H = -(-(D + 1) * o // q) + w + 1
    st, got, fed = np.zeros(2 + H), [], 0
    for n in [1, o - 1, o, o + 1, 3, 2 * o + 5, 7]:
        n = min(n, len(x) - fed)
        if n <= 0:
            break
        yk, bk, st = packet_push(st, x[fed:fed + n], orig, new)
        got.append(yk)
        fed += n
    got = np.concatenate(got)
    assert len(got) == fed * q // o
    want = _delayed(x[:fed], orig, new, D, len(got))
    assert np.allclose(got, want, rtol=0, atol=1e-12)
    # whole periods
    if o <= 500:
        Hs = -(-D * o // q) + w
        st, got = np.zeros(Hs + 3), []
        for h in [1, 0, 2, 3, 1]:
            yk, bk, st = stream_push(st, x[len(got) and sum(len(a) - 3 for a in got) // q * o:][:h * o], orig, new, o, 3)
            got.append(yk)
        cat = np.concatenate([a[3:] for a in got])
        assert np.allclose(cat, _delayed(x, orig, new, D, len(cat)), rtol=0, atol=1e-12)
        assert not bk[:3].any()


def test_bound_covers_an_fp32_evaluation():
    """the kernel's arithmetic emulated in numpy float32 (its own sin / cos for sinpif / cospif) lies within the bound"""
    f = np.float32
    for orig, new in [(48000, 16000), (16000, 44100), (46200, 40000)]:
        o, q, w, base = rs_filter(orig, new)
        x = np.float32(np.random.default_rng(o).standard_normal(4 * o + 50)).astype(np.float64)
        y, b = whole(x, orig, new, ors.output_length(len(x), orig, new))
        pad = np.concatenate([np.zeros(w + 1), x, np.zeros(w + 2)])
        emu = []
        for m in range(len(y)):
            c, r = m * o // q, m * o % q
            u0 = r * (base / (o * q)) + w * (base / o)
            acc = f(0)
            for t in range(2 * w + 1):
                u = f(u0 - t * (base / o))
                if abs(u) < 6:
                    s = f(1) if u == 0 else f(np.sin(np.pi * np.float64(u))) / (f(3.14159265358979) * u)
                    wn = f(0.5) + f(0.5) * f(np.cos(np.pi * np.float64(u * (f(1) / f(6)))))
                    acc = f(np.float64(acc) + np.float64(f(f(base / o) * s) * wn) * pad[w + 1 + c - w + t])
            emu.append(acc)
        assert np.all(np.abs(np.array(emu, np.float64) - y) <= b), (orig, new)


@pytest.mark.parametrize("mutant", RS_MUTANTS)
def test_resample_mutants_miss_their_bound(mutant):
    from kernels.scaffold import SENSITIVITY, ratio
    x = np.float32(np.random.default_rng(5).standard_normal(60000)).astype(np.float64)
    for orig, new in [(44100, 16000)]:
        cap = ors.output_length(len(x), orig, new)
        y, b = whole(x, orig, new, cap)
        ym, _ = whole(x, orig, new, cap, mutant)
        assert ratio(ym, y, b) >= SENSITIVITY, mutant


@pytest.mark.parametrize("mutant", PACKET_MUTANTS)
def test_stream_mutants_miss_their_bound(mutant):
    from kernels.scaffold import SENSITIVITY, ratio
    orig, new = 44100, 16000
    o, q, w, base = rs_filter(orig, new)
    D = w * q // o
    H = -(-(D + 1) * o // q) + w + 1
    g = np.random.default_rng(6)
    st = np.concatenate([[2.0, 100.0], g.standard_normal(H)])      # started part-way, phase 100
    x = g.standard_normal(900)
    y, b, s1 = packet_push(st, x, orig, new)
    ym, _, s2 = packet_push(st, x, orig, new, mutant)
    assert len(ym) != len(y) or ratio(ym, y, b) >= SENSITIVITY or not np.array_equal(s1, s2)
    if mutant != "phase_word_ignored":
        Hs = -(-D * o // q) + w
        st = np.concatenate([[2.0], g.standard_normal(Hs - 1 + 4)])
        y, b, s1 = stream_push(st, x[:2 * o], orig, new, o, 4)
        ym, _, s2 = stream_push(st, x[:2 * o], orig, new, o, 4, mutant)
        assert ratio(ym, y, b) >= SENSITIVITY, mutant


@pytest.fixture(scope="module")
def lib():
    from lookoncetohear_b200 import _cabi, build
    build.build()
    return _cabi.lib()


def _call(lib, rates, new, n_in=200, cap=None, x_stride=None, y_stride=None, x=16, y=4096):
    """l2h_resample with placeholder device addresses: only for argument sets that must be refused before any launch."""
    arr = (ctypes.c_int32 * len(rates))(*rates)
    cap = 1000 if cap is None else cap
    return lib.l2h_resample(ctypes.c_void_p(x), n_in if x_stride is None else x_stride, n_in, len(rates), arr, new,
                            ctypes.c_void_p(y), cap if y_stride is None else y_stride, cap, None)


def test_abi_refuses_bad_rates(lib):
    assert _call(lib, [0], 16000) == 1 and b"orig_freq 0 is not positive" in lib.l2h_last_error()
    assert _call(lib, [44100, 44100, -16000], 16000) == 1 and b"row 2" in lib.l2h_last_error()
    assert _call(lib, [44100], 0) == 1 and b"new_freq 0" in lib.l2h_last_error()
    assert _call(lib, [44100], -8000) == 1
    # 50x downsampling: the input window of a 256-output tile no longer fits the kernel's shared memory
    assert _call(lib, [44100, 800000], 16000, cap=100000) == 2
    assert b"ratio 50/1 (800000 -> 16000 Hz) is too large" in lib.l2h_last_error()


def test_abi_refuses_small_capacity(lib):
    # 200 samples: 44100 -> 16000 gives ceil(16000 * 200 / 44100) = 73, 8000 -> 16000 gives 400
    assert _call(lib, [44100], 16000, cap=72) == 1 and b"73 output samples, capacity 72" in lib.l2h_last_error()
    assert _call(lib, [44100, 8000], 16000, cap=399) == 1 and b"row 1" in lib.l2h_last_error()
    assert _call(lib, [16000], 16000, cap=199) == 1                          # equal rates need n_in samples too


def test_abi_refuses_bad_sizes(lib):
    assert _call(lib, [44100], 16000, x=0) == 1 and b"bad argument" in lib.l2h_last_error()
    assert _call(lib, [44100], 16000, y=0) == 1
    assert _call(lib, [], 16000) == 1                                          # no rows
    assert _call(lib, [44100], 16000, x_stride=199) == 1                       # rows would overlap
    assert _call(lib, [44100], 16000, y_stride=999) == 1
    assert lib.l2h_resample(ctypes.c_void_p(16), 200, 200, 1, None, 16000, ctypes.c_void_p(4096), 100, 100, None) == 1


def test_python_refuses_other_methods_and_cpu_tensors():
    from lookoncetohear_b200 import resample
    x = torch.zeros(2, 100)
    for kw in ({"resampling_method": "sinc_interp_kaiser"}, {"lowpass_filter_width": 16}, {"rolloff": 0.95}, {"beta": 14.0}):
        with pytest.raises(ValueError, match="only torchaudio's default"):
            resample(x, 44100, 16000, **kw)
    with pytest.raises(ValueError):
        resample(x, 44100, 0)
    with pytest.raises(RuntimeError, match="CUDA"):
        resample(x, 44100, 16000)
