"""The jitter buffer (JitterBuffer, l2h_jitter_buffer) without a GPU: an exact model of its bookkeeping and a float64 model
of its concealment, over the kernel's own state layout (so the GPU tests can run one call of the model from the kernel's
state), checked against the rules of include/lookonce_b200.h; and the layout, the argument errors, the Python checks, the
header and the exports."""
import ctypes
import math

import numpy as np
import pytest
import torch

from lookoncetohear_b200 import JitterBuffer
from serving_util import FAKE_DEV, declaration, doc_before, header

HEAD, LOST, RECOVER, SEQ = 16, -1, 1 << 17, 1 << 16
U = 2.0 ** -24                                       # fp32 unit roundoff


def rnd(v):
    return int(math.floor(v + 0.5))


class Params:
    """the kernel's derived sizes of a jitter buffer (l2h_jitter_buffer header block)"""

    def __init__(self, rate, P, C=1, D=1, W=16, max_out=4):
        self.rate, self.P, self.C, self.D, self.W, self.R, self.max_out = rate, P, C, D, W, 2 * W, max_out
        self.tmin, self.tmax, self.wc = rnd(0.0025 * rate), rnd(0.015 * rate), rnd(0.020 * rate)
        self.H = self.wc + self.tmax
        self.lr, self.ga, self.gb = min(rnd(0.004 * rate), P), rnd(0.010 * rate), rnd(0.060 * rate)
        self.o_ring = HEAD + self.R
        self.o_hist = self.o_ring + self.R * P
        self.o_per = self.o_hist + self.H
        self.rf = self.o_per + self.tmax

    def fresh(self, slots=1):
        return np.zeros((slots, self.C, self.rf), dtype=np.float32)


def gain(k, p):
    return 1.0 if k < p.ga else (0.0 if k >= p.gb else (p.gb - k) / (p.gb - p.ga))


def clean(v):
    v = np.asarray(v, dtype=np.float32).copy()
    v[~(np.abs(v) < 2.0 ** 32)] = 0.0
    return v


def pitch(win, p, trace=None, force=None):
    """the lag of the period that ends win's last sample ([C, H] history), float64; `force` overrides it (a lag the
    kernel chose in a near tie); trace gets (lag, scores, bounds) per search"""
    s = win.astype(np.float64).sum(0)
    a = s[p.H - p.wc:]
    best, bt = -1.0, p.tmax
    scores, bounds = {}, {}
    g = (p.wc + p.C) * U / (1 - (p.wc + p.C) * U)
    for t in range(p.tmin, p.tmax + 1):
        b = s[p.H - p.wc - t:p.H - t]
        num, en = float(a @ b), float(b @ b)
        sc = num / math.sqrt(max(en, 2.0 ** -126)) if num > 0 else -1.0
        scores[t] = sc
        bounds[t] = g * float(np.abs(a) @ np.abs(b)) / math.sqrt(max(en, 2.0 ** -126)) + max(sc, 0) * (0.5 * g + 2 * U)
        if num > 0 and sc > best:
            best, bt = sc, t
    if trace is not None:
        trace.append((bt, scores, bounds))
    return bt if force is None else force


def model_call(st, x, seqs, cnt, p, force=None, trace=None):
    """One call of one row: st [C, rf] float32 (the slot's state, updated in place), x [C, M P], seqs [M], cnt.  Returns
    y [C, m P] float32 (each sample computed in float64, then rounded as the kernel stores it).  `force`: lags for the
    searches, in order."""
    w = st.view(np.int32)
    h = w[0]
    R, W, P, H = p.R, p.W, p.P, p.H
    force = list(force or [])
    tg = h[HEAD:HEAD + R].astype(np.int64).copy()
    started = int(h[0]) != 0
    next_ = min(max(int(h[1]), 0), SEQ - 1)
    pos = min(max(int(h[2]), 0), R - 1)
    pend = min(max(int(h[3]), 0), W)
    add = dict(lost=0, late=0, dup=0, dropped=0, restarts=0)

    def slot(d):
        return (pos + pend + d) % R

    def held(d):
        return tg[slot(d)] == ((next_ + d) & (SEQ - 1)) + 1

    far = max([d for d in range(W) if held(d)], default=-1)
    cp = [-1] * cnt
    for j in range(cnt):
        s = int(seqs[j])
        if s < 0 or s >= SEQ:
            continue
        if not started:
            started, next_ = True, s
        d = (s - next_) & (SEQ - 1)
        if d >= SEQ // 2:
            d -= SEQ
        recover = False
        if d < 0:
            add["late"] += 1
            continue
        if d < W:
            if held(d):
                add["dup"] += 1
                continue
        else:
            for e in range(W):
                add["dropped"] += int(held(e))
                tg[slot(e)] = 0
            add["restarts"] += 1
            next_, d, far, recover = s, 0, -1, True
        at = slot(d)
        tg[at] = s + 1
        cp = [-1 if c == at else c for c in cp]
        cp[j] = at
        far = max(far, d)
        while True:
            if held(0):
                t, recover = (next_ + 1) | (RECOVER if recover else 0), False
            elif far >= p.D + 1:
                t = LOST
                add["lost"] += 1
            else:
                break
            if pend == W:
                tg[pos] = 0
                pos, pend = (pos + 1) % R, pend - 1
                add["dropped"] += 1
            tg[(pos + pend) % R] = t
            pend, next_, far = pend + 1, (next_ + 1) & (SEQ - 1), far - 1
    n_out = min(pend, p.max_out)
    kinds, slots_out = [], []
    for k in range(n_out):
        at = (pos + k) % R
        t = int(tg[at])
        kinds.append(t if 1 <= (t & ~RECOVER) <= SEQ else LOST)
        slots_out.append(at)
        tg[at] = 0
    pos, pend = (pos + n_out) % R, pend - n_out
    nheld = sum(int(held(d)) for d in range(W))
    # the samples: stored packets into the ring, then each written packet
    ring = st[:, p.o_ring:p.o_hist].reshape(p.C, R, P)
    for j, at in enumerate(cp):
        if at >= 0:
            ring[:, at] = clean(x[:, j * P:(j + 1) * P])
    win = np.concatenate([st[:, p.o_hist:p.o_per], np.zeros((p.C, n_out * P), np.float32)], 1)
    per = st[:, p.o_per:p.o_per + p.tmax].copy()
    run, tau = min(max(int(h[4]), 0), p.gb), int(h[5])
    tau = tau if p.tmin <= tau <= p.tmax else 0
    i = np.arange(P)
    for k, (t, at) in enumerate(zip(kinds, slots_out)):
        base = k * P
        if tau == 0 and t != LOST and not t & RECOVER:
            win[:, H + base:H + base + P] = ring[:, at]
            continue
        if tau == 0:
            tau = pitch(win[:, base:base + H], p, trace, force.pop(0) if force else None)
            run = 0
            per[:, :tau] = win[:, base + H - tau:base + H]
            h[12] = tau
        g = np.array([gain(min(run + q, p.gb), p) for q in i])
        cont = g * per[:, (run + i) % tau].astype(np.float64)
        v = cont
        if t != LOST:
            r = ring[:, at].astype(np.float64)
            wgt = 0.5 - 0.5 * np.cos(np.pi * (i + 1) / (p.lr + 1))
            v = np.where(i < p.lr, cont + wgt * (r - cont), r)
            tau, run = 0, 0
        else:
            run = min(run + P, p.gb)
        win[:, H + base:H + base + P] = v.astype(np.float32)
    st[:, p.o_hist:p.o_per] = win[:, n_out * P:]
    st[:, p.o_per:p.o_per + p.tmax] = per
    h[HEAD:HEAD + R] = tg.astype(np.int32)
    h[0], h[1], h[2], h[3] = int(started), next_, pos, pend
    for k, name in zip(range(6, 11), ("lost", "late", "dup", "dropped", "restarts")):
        h[k] = min(max(int(h[k]), 0) + add[name], 2 ** 31 - 1)
    h[11] = nheld
    h[4], h[5] = (run if tau else 0), tau
    return win[:, H:H + n_out * P], n_out


def model_run(p, packets, arrivals, cuts, st=None):
    """arrivals (a list of sequence numbers, each naming packets[s % len]) cut into calls of cuts[k] packets: the
    concatenated output [C, N] and the final state"""
    st = p.fresh()[0] if st is None else st
    out, a = [], 0
    for c in cuts:
        seq = arrivals[a:a + c]
        x = np.concatenate([packets[s % len(packets)] for s in seq], 1) if seq else np.zeros((p.C, 0), np.float32)
        y, _ = model_call(st, x, seq, len(seq), p)
        out.append(y)
        a += c
    while True:                                      # the backlog: calls with count 0
        y, m = model_call(st, np.zeros((p.C, 0), np.float32), [], 0, p)
        if not m:
            break
        out.append(y)
    return np.concatenate(out, 1), st


def words(st):
    return st[0].view(np.int32)


def packets_of(p, n, seed):
    g = np.random.default_rng(seed)
    return [(0.3 * g.standard_normal((p.C, p.P))).astype(np.float32) for _ in range(n)]


def random_cuts(n, seed, hi=4):
    g = np.random.default_rng(seed)
    cuts, left = [], n
    while left:
        c = int(min(left, g.integers(0, hi + 1)))
        cuts.append(c)
        left -= c
    return cuts


def schedule(n, seed, loss=0.1, swap=0.1, dup=0.05, start=0):
    """a seeded arrival sequence of n packets from `start`: losses, neighbours swapped and duplicates"""
    g = np.random.default_rng(seed)
    seq = [(start + k) & (SEQ - 1) for k in range(n) if g.random() >= loss]
    for k in range(len(seq) - 1):
        if g.random() < swap:
            seq[k], seq[k + 1] = seq[k + 1], seq[k]
    out = []
    for s in seq:
        out.append(s)
        if g.random() < dup:
            out.append(s)
    return out


# ---- the release rules -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate,P", [(16000, 160), (44100, 441), (48000, 480)])
def test_perfect_network_is_bit_for_bit(rate, P):
    p = Params(rate, P, C=2)
    pk = packets_of(p, 40, 1)
    for seed in range(3):
        y, st = model_run(p, pk, list(range(40)), random_cuts(40, seed))
        assert np.array_equal(y.view(np.int32), np.concatenate(pk, 1).view(np.int32))
        assert words(st)[6:12].tolist() == [0, 0, 0, 0, 0, 0]


@pytest.mark.parametrize("D", [0, 1, 3])
def test_reordering_within_depth_gives_the_stream(D):
    p = Params(16000, 160, D=D)
    pk = packets_of(p, 30, 2)
    arr = list(range(30))
    for k in range(2, 26, 6):                        # packet k arrives D places late
        arr.insert(k + D, arr.pop(k))
    y, st = model_run(p, pk, arr, [1] * 30)
    assert np.array_equal(y, np.concatenate(pk, 1))
    assert words(st)[6] == 0 and words(st)[7] == 0


def test_reordering_beyond_depth_is_late_and_concealed():
    p = Params(16000, 160, D=1)
    pk = packets_of(p, 20, 3)
    arr = list(range(20))
    arr.insert(10, arr.pop(7))                       # packet 7 arrives three packets late: 8, 9 declare it lost first
    y, st = model_run(p, pk, arr, [1] * 20)
    w = words(st)
    assert (w[6], w[7]) == (1, 1)
    assert y.shape[1] == 20 * 160
    assert np.array_equal(y[:, :7 * 160], np.concatenate(pk[:7], 1))
    assert np.array_equal(y[:, 8 * 160 + p.lr:9 * 160], pk[8][:, p.lr:])     # after the fade, packet 8 as it was
    assert np.array_equal(y[:, 9 * 160:], np.concatenate(pk[9:], 1))


@pytest.mark.parametrize("rate,P,W,D", [(16000, 160, 16, 1), (44100, 441, 8, 0), (48000, 480, 16, 3)])
def test_cuts_and_max_out_change_nothing(rate, P, W, D):
    p0 = Params(rate, P, C=2, D=D, W=W, max_out=64)
    pk = packets_of(p0, 64, 4)
    arr = schedule(120, 5, loss=0.15, start=65500)
    want, st0 = model_run(p0, pk, arr, [1] * len(arr))
    # each call writes at least as many packets as it takes arrivals, so the backlog never fills
    for seed, mo, hi in ((0, 2, 1), (1, 3, 2), (2, 4, 3), (3, 7, 4)):
        p = Params(rate, P, C=2, D=D, W=W, max_out=mo)
        y, st = model_run(p, pk, arr, random_cuts(len(arr), seed, hi))
        assert np.array_equal(y.view(np.int32), want.view(np.int32)), (seed, mo)
        assert np.array_equal(words(st)[6:11], words(st0)[6:11])


def test_wrap_duplicates_and_restarts():
    p = Params(16000, 160, W=8)
    pk = packets_of(p, 16, 6)
    arr = [65533, 65535, 65535, 65534, 0, 2, 2, 1]   # a wrap, with two duplicates of held packets
    y, st = model_run(p, pk, arr, [3, 0, 5])
    w = words(st)
    assert np.array_equal(y, np.concatenate([pk[s % 16] for s in (65533, 65534, 65535, 0, 1, 2)], 1))
    assert (w[1], w[8], w[6], w[7]) == (3, 2, 0, 0)
    y, _ = model_run(p, pk, [2, 1], [2], st=st)      # released packets arriving again are late
    assert y.shape[1] == 0 and (words(st)[7], words(st)[8]) == (2, 2)
    arr2 = [6, 3000, 3001, 3003, 2999]               # 6 declares 3 and 4 lost and waits; the restart at 3000 drops it
    st_before = st.copy()
    y2, _ = model_run(p, pk, arr2, [5], st=st)
    w = words(st)
    assert (w[6], w[10], w[9], w[7]) == (2, 1, 1, 3)  # 3 and 4 lost, one restart, packet 6 dropped, 2999 late
    assert w[1] == 3002 and w[11] == 1               # 3003 waits for 3002 (depth 1)
    assert y2.shape[1] == 4 * 160                    # 3 and 4 concealed, then 3000 (faded in) and 3001
    assert np.array_equal(y2[:, 3 * 160:], pk[3001 % 16]) and st_before.shape == st.shape


RESTART_ARRIVALS, RESTART_CUTS = [0, 2, 3, 4, 5, 6, 1, 5000, 5001, 5002], [7, 1, 1, 1]


def restart_behind_a_backlog(max_out, C=1):
    """packets 0 .. 6 released by one call (1 arriving last, depth 8), then a restart at 5000 while they wait"""
    p = Params(16000, 160, C=C, D=8, W=16, max_out=max_out)
    pk = packets_of(p, 16, 13)
    y, st = model_run(p, pk, RESTART_ARRIVALS, RESTART_CUTS)
    return p, pk, y, st


def test_a_restart_keeps_the_decided_backlog():
    """a restart while released packets wait unwritten: they still play, bit for bit, under every max_out"""
    p, pk, want, st = restart_behind_a_backlog(16)
    assert np.array_equal(want[:, :7 * 160], np.concatenate(pk[:7], 1))
    assert (words(st)[10], words(st)[6], words(st)[9]) == (1, 0, 0)
    for mo in (1, 2, 3, 8):
        _, _, y, st2 = restart_behind_a_backlog(mo)
        assert np.array_equal(y.view(np.int32), want.view(np.int32)), mo
        assert np.array_equal(words(st2)[6:11], words(st)[6:11])


def test_backlog_overflow_drops_the_oldest():
    p = Params(16000, 160, W=4, max_out=1)
    pk = packets_of(p, 12, 7)
    st = p.fresh()[0]
    x = np.concatenate(pk, 1)
    y, m = model_call(st, x, list(range(12)), 12, p)
    assert m == 1 and words(st)[9] == 8               # 12 released, the backlog keeps 4: the 8 oldest go
    assert words(st)[3] == 3 and np.array_equal(y, pk[8])


# ---- the concealment -------------------------------------------------------------------------------------------------
def voiced(rate, f0, n, seed, C=2):
    """harmonics 1..6 of f0 with seeded amplitudes and phases, channel 1 a delayed, scaled copy"""
    g = np.random.default_rng(seed)
    t = np.arange(n) / rate
    amp, ph = g.uniform(0.2, 1, 6) / np.arange(1, 7), g.uniform(0, 2 * np.pi, 6)
    base = lambda d: sum(a * np.sin(2 * np.pi * f0 * (h + 1) * (t - d) + p) for h, (a, p) in enumerate(zip(amp, ph)))
    return np.stack([0.3 * base(0), 0.2 * base(3e-4)][:C]).astype(np.float32)


def lose(p, sig, first, count, total):
    """sig cut into packets, packets first .. first + count - 1 lost; the output of one call per arrival"""
    pk = [sig[:, k * p.P:(k + 1) * p.P] for k in range(total)]
    arr = [k for k in range(total) if not first <= k < first + count]
    y, st = model_run(p, pk, arr, [1] * len(arr))
    return y, st


@pytest.mark.parametrize("rate,P", [(16000, 160), (44100, 441), (48000, 480)])
def test_concealment_finds_the_period_and_beats_zero_fill(rate, P):
    p = Params(rate, P, C=2)
    for seed, f0 in enumerate((90.0, 140.0, 220.0, 350.0)):
        T0 = rate / f0
        total = 12
        sig = voiced(rate, f0, total * P, seed)
        y, st = lose(p, sig, 8, 1, total)
        tau = int(words(st)[12])
        assert abs(tau - round(tau / T0) * T0) <= 1.0, (f0, tau, T0)           # the period or a multiple of it
        # integer-period copy of the signal: e[k] = x[N - tau + (k mod tau)].  Each repeat drifts by |tau - m T0| <= 1
        # sample; harmonics of up to 6 f0 <= 2.1 kHz then lose coherence by at most 2 pi 2100 / rate rad per repeat, so
        # over one 10 ms packet (at most 4 repeats at 350 Hz) the error energy stays under 1/2 of zero-fill's
        seg = slice(8 * P, 9 * P)
        err = float(((y[:, seg].astype(np.float64) - sig[:, seg]) ** 2).sum())
        zero = float((sig[:, seg].astype(np.float64) ** 2).sum())
        assert err < 0.5 * zero, (f0, err / zero)


def test_integer_period_conceals_exactly():
    p = Params(16000, 160, C=2)
    sig = voiced(16000, 16000 / 100, 12 * 160, 9)    # period exactly 100 samples
    y, st = lose(p, sig, 8, 1, 12)
    assert int(words(st)[12]) % 100 == 0
    seg = slice(8 * 160, 9 * 160)
    # the repeat is the signal itself, up to the fp32 rounding of both: error energy below 2^-40 of zero-fill's
    err = float(((y[:, seg].astype(np.float64) - sig[:, seg]) ** 2).sum())
    assert err <= 2.0 ** -40 * float((sig[:, seg].astype(np.float64) ** 2).sum())


@pytest.mark.parametrize("rate,P", [(16000, 160), (44100, 441)])
def test_long_runs_go_silent_and_recovery_does_not_click(rate, P):
    p = Params(rate, P, C=2)
    total, first, count = 20, 6, 9                  # a 90 ms burst
    sig = voiced(rate, 150.0, total * P, 11)
    y, _ = lose(p, sig, first, count, total)
    run = y[:, first * P:(first + count) * P]
    assert np.all(run[:, p.gb:] == 0) and np.any(run[:, :p.ga] != 0)
    # after the silent run the packet fades in.  A step of v = e + w (r - e) is at most |de| + |dr| (each at most the
    # signal's largest step: e loops a period of it) plus the fade's largest weight step, pi / (2 (Lr + 1)), times
    # |r - e| <= 2 peak
    k0 = (first + count) * P
    seg = y[:, k0 - 1:k0 + p.lr + 1].astype(np.float64)
    peak = float(np.abs(sig).max())
    bound = 2 * float(np.abs(np.diff(sig, axis=1)).max()) + math.pi / (p.lr + 1) * peak
    assert float(np.abs(np.diff(seg, axis=1)).max()) <= bound
    # a one-packet loss recovers from the running concealment with the same bound on its steps
    y, _ = lose(p, sig, first, 1, total)
    seg = y[:, (first + 1) * P - 1:(first + 1) * P + p.lr + 1].astype(np.float64)
    assert float(np.abs(np.diff(seg, axis=1)).max()) <= bound


def test_bad_input_enters_as_zero():
    p = Params(16000, 160)
    pk = packets_of(p, 4, 12)
    pk[1][0, 3], pk[1][0, 7], pk[2][0, 0] = np.nan, 2.0 ** 33, np.inf
    y, _ = model_run(p, pk, [0, 1, 2, 3], [4])
    assert y[0, 160 + 3] == 0 and y[0, 160 + 7] == 0 and y[0, 320] == 0 and np.isfinite(y).all()


# ---- interfaces ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from lookoncetohear_b200 import _cabi, build
    build.build()
    return _cabi.lib()


def test_entries_exported_and_declared(lib):
    hdr = header()
    for name in ("l2h_jitter_buffer_layout", "l2h_jitter_buffer"):
        assert hasattr(lib, name)
        decl, _ = declaration(hdr, name)
        assert decl, name


def layout(lib, *args):
    v = ctypes.c_int32(-1)
    return lib.l2h_jitter_buffer_layout(*args, ctypes.byref(v)), v.value


@pytest.mark.parametrize("rate,P,W", [(16000, 160, 16), (44100, 441, 16), (48000, 480, 8), (8000, 80, 1)])
def test_layout(lib, rate, P, W):
    p = Params(rate, P, C=2, W=W)
    assert layout(lib, 2, rate, P, 0, W, 4) == (0, p.rf)


def test_layout_errors(lib):
    assert layout(lib, 0, 16000, 160, 1, 16, 4)[0] == 1
    assert layout(lib, 1, 7999, 160, 1, 16, 4)[0] == 1
    assert layout(lib, 1, 16000, 0, 1, 16, 4)[0] == 1          # packet < 1
    assert layout(lib, 1, 16000, 160, 16, 16, 4)[0] == 1       # depth >= window
    assert layout(lib, 1, 16000, 160, -1, 16, 4)[0] == 1
    assert layout(lib, 1, 16000, 160, 1, 0, 4)[0] == 1
    assert layout(lib, 1, 16000, 160, 1, 4097, 4)[0] == 1
    assert layout(lib, 1, 16000, 160, 1, 16, 0)[0] == 1
    assert layout(lib, 2, 48000, 480, 1, 16, 6)[0] == 0        # 2 (1680 + 6 * 480) + 1680 + 1440 + 38 = 12278 words
    assert layout(lib, 2, 48000, 480, 1, 16, 7)[0] == 2        # 13239 words: more than 48 KB
    assert layout(lib, 8, 192000, 160, 1, 16, 1)[0] == 2       # the history of 8 channels at 192 kHz
    assert lib.l2h_jitter_buffer_layout(1, 16000, 160, 1, 16, 4, None) == 1


def test_call_errors(lib):
    i32 = ctypes.c_void_p(0x20000)

    def call(x=FAKE_DEV, xr=320, xc=320, M=2, n=2, C=1, y=ctypes.c_void_p(0x100000), yr=640, yc=640, slots=i32,
             n_slots=4, depth=1):
        return lib.l2h_jitter_buffer(x, xr, xc, M, i32, i32, y, yr, yc, i32, n, C, slots, FAKE_DEV, n_slots, 16000, 160,
                                     depth, 16, 4, None)

    assert call(x=None) == 1 and call(slots=None) == 1
    assert call(n=0) == 1 and call(M=0) == 1 and call(n=5) == 1
    assert call(xr=300) == 1                         # rows overlap
    assert call(yr=600) == 1
    assert call(depth=16) == 1
    assert call(y=ctypes.c_void_p(0x10000 + 4 * 100)) == 1      # y overlaps x
    assert call(M=12000) == 2                        # the arrivals' ring slots do not fit the staging
    assert "l2h_jitter_buffer" in lib.l2h_last_error().decode()


def test_constructor_checks():
    with pytest.raises(ValueError):
        JitterBuffer(4, 2, 44100, 441, depth=16, window=16, device="cpu")
    with pytest.raises(ValueError):
        JitterBuffer(4, 2, 44100, 0, device="cpu")
    with pytest.raises(ValueError):
        JitterBuffer(4, 2, 4000, 40, device="cpu")
    with pytest.raises(ValueError):
        JitterBuffer(4, 2, 48000, 480, max_out=8, device="cpu")  # error 2 is a ValueError too
    with pytest.raises(ValueError):
        JitterBuffer(4, 0, 44100, 441, device="cpu")
    with pytest.raises(RuntimeError, match="CUDA"):
        JitterBuffer(4, 2, 44100, 441, device="cpu")


def test_call_needs_cuda():
    jb = JitterBuffer.__new__(JitterBuffer)
    jb.n_slots, jb.channels, jb.packet = 4, 2, 441
    jb.state = torch.zeros(4, 2, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        jb(torch.zeros(1, 2, 441), [[0]], [1], [0])


def test_header_documents_the_jitter_buffer():
    hdr = header()
    decl, args = declaration(hdr, "l2h_jitter_buffer")
    doc = doc_before(hdr, decl.start())
    for a in ("x_dev", "seqs_dev", "counts_dev", "y_dev", "out_counts_dev", "slots_dev"):
        assert a in args and a in doc, a
    for words_ in ("RFC 1982", "depth", "late", "duplicate", "dropped", "restarts", "lost", "bit for bit",
                   "l2h_resample_packets", "l2h_hop_fifo", "l2h_sep_forward_slots_hops", "Errors", "1 = ", "2 = "):
        assert words_ in doc, words_


def test_host_seqs_are_checked_where_pushed():
    """host sequence numbers are checked only for the packets a row pushes, so short rows may be padded with -1; with
    the counts on the device every entry is checked"""
    jb = JitterBuffer.__new__(JitterBuffer)
    jb.state = torch.zeros(1)
    assert jb._seqs([[5, -1], [3, 4]], 2, 2, [1, 2]).tolist() == [[5, -1], [3, 4]]
    for seqs, counts in (([[5, -1], [3, 4]], None), ([[5, -1], [3, 70000]], [1, 2]), ([[5, -1]], [1])):
        with pytest.raises(ValueError):
            jb._seqs(seqs, 2, 2, counts)
