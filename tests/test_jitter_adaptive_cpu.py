"""The jitter buffer with adaptive deadlines (JitterBuffer(deadline=(lo, hi)), l2h_jitter_buffer_adaptive) without a GPU:
an exact model of its bookkeeping, its lateness statistics and its per-slot deadline, and a float64 model of its
concealment, over the kernel's own state layout, built on the timed model of tests/test_jitter_deadline_cpu.py (so the
GPU tests can run one call of it from the kernel's state), checked against the rules of include/lookonce_b200.h; and the
layout, the argument errors, the Python checks, the header and the export."""
import ctypes
import math

import numpy as np
import pytest
import torch

import test_jitter_buffer_cpu as jm
import test_jitter_deadline_cpu as tm
from lookoncetohear_b200 import JitterBuffer
from serving_util import FAKE_DEV, declaration, doc_before, header

HEAD, LOST, RECOVER, SEQ = jm.HEAD, jm.LOST, jm.RECOVER, jm.SEQ
A_S, A_T, EXPIRED = tm.A_S, tm.A_T, tm.EXPIRED
BINS, STATS, UNIT, BIN_MAX = 64, 66, 1 << 24, 1 << 30
ser16, ser32, period, stall = tm.ser16, tm.ser32, tm.period, tm.stall


class Adapt:
    """an adaptive buffer's parameters: jm.Params plus the bounds, the bin width, r, the warm-up and the memory N"""

    def __init__(self, p, lo, hi, late_rate=0.02):
        self.p, self.lo, self.hi, self.late_rate = p, lo, hi, late_rate
        self.w = max(1, -(-hi // BINS))
        self.r = math.floor(late_rate * 65536.0 + 0.5)
        self.warm = min(math.ceil(1.0 / late_rate), 2 ** 31 - 1)
        T = period(p)
        self.N = max(1, (10_000_000 + T) // (2 * T))
        self.rf = p.rf + STATS
        self.o_stats = p.rf

    def fresh(self, slots=1):
        return np.zeros((slots, self.p.C, self.rf), dtype=np.float32)


def stats(st, a):
    """(bins [64] int64, k, deadline) of a slot's state"""
    s = st[0, a.o_stats:].view(np.int32)
    return s[:BINS].astype(np.int64), int(s[BINS]), int(s[BINS + 1])


def bin_of(l, a):
    return 0 if l < 0 else min(l // a.w, BINS - 1)


def update(h, k, bins, a):
    """the measured bins, in arrival order, into the histogram h (int64 [64], in place); returns k"""
    for b in bins:
        m = min(k, a.N - 1) + 1
        h -= h // m
        h[b] += UNIT // m
        k = min(k + 1, 2 ** 31 - 1)
    return k


def quantile_deadline(h, k, a):
    if k < a.warm:
        return a.hi
    total = int(h.sum())
    tail = 0
    tails = [0] * BINS
    for b in range(BINS - 1, -1, -1):
        tails[b] = tail
        tail += int(h[b])
    b = next(b for b in range(BINS) if tails[b] * 65536 <= a.r * total)
    return min(max((b + 1) * a.w, a.lo), a.hi)


def adaptive_call(st, x, seqs, cnt, a, now, arrivals=None, force=None, trace=None, lateness=None):
    """One adaptive call of one row at clock `now` (µs, any int, taken mod 2^32), as tm.timed_call: st [C, rf + 66]
    float32 updated in place, `arrivals` [cnt] ints or None.  Returns (y [C, m P] float32, m); `lateness` gets the
    lateness of each measured packet."""
    p = a.p
    w = st.view(np.int32)
    h = w[0]
    R, W, P, H = p.R, p.W, p.P, p.H
    force = list(force or [])
    tg = h[HEAD:HEAD + R].astype(np.int64).copy()
    started = int(h[0]) != 0
    next_ = min(max(int(h[1]), 0), SEQ - 1)
    pos = min(max(int(h[2]), 0), R - 1)
    pend = min(max(int(h[3]), 0), W)
    a_s, a_t, now = min(max(int(h[A_S]), 0), SEQ - 1), int(h[A_T]) & 0xFFFFFFFF, now & 0xFFFFFFFF
    add = dict(lost=0, late=0, dup=0, dropped=0, restarts=0, expired=0)
    measured = []

    def slot(d):
        return (pos + pend + d) % R

    def held(d):
        return tg[slot(d)] == ((next_ + d) & (SEQ - 1)) + 1

    def stalled():
        return ser16(next_ - a_s - 1) >= stall(p)

    def push(t):
        nonlocal pos, pend, next_, far
        if pend == W:
            tg[pos] = 0
            pos, pend = (pos + 1) % R, pend - 1
            add["dropped"] += 1
        tg[(pos + pend) % R] = t
        pend, next_, far = pend + 1, (next_ + 1) & (SEQ - 1), far - 1

    def measure(s, arr):
        l = ser32(arr - (a_t + ser16(s - a_s) * period(p)))
        measured.append(bin_of(l, a))
        if lateness is not None:
            lateness.append(l)

    far = max([d for d in range(W) if held(d)], default=-1)
    cp = [-1] * cnt
    for j in range(cnt):
        s = int(seqs[j])
        if s < 0 or s >= SEQ:
            continue
        arr = now
        if arrivals is not None:
            v = int(arrivals[j]) & 0xFFFFFFFF
            arr = v if ser32(v - now) < 0 else now
        first = not started
        if not started:
            started, next_, a_s = True, s, s
        d = ser16(s - next_)
        recover = False
        if d < 0:
            add["late"] += 1
            if not stalled():
                measure(s, arr)
            continue
        if d < W and not stalled():
            if held(d):
                add["dup"] += 1
                continue
            if not first:
                measure(s, arr)
        else:
            for e in range(W):
                add["dropped"] += int(held(e))
                tg[slot(e)] = 0
            add["restarts"] += 1
            next_, d, far, recover, a_s = s, 0, -1, True, s
        if ser16(s - a_s) >= 0:
            a_s, a_t = s, arr
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
            push(t)
    deadline = a.hi
    if started:                                      # the statistics and the slot's deadline
        sw = st[0, a.o_stats:].view(np.int32)
        hist = np.clip(sw[:BINS].astype(np.int64), 0, BIN_MAX)
        k = update(hist, max(int(sw[BINS]), 0), measured, a)
        deadline = quantile_deadline(hist, k, a)
        sw[:BINS], sw[BINS], sw[BINS + 1] = hist.astype(np.int32), k, deadline
    while started:                                   # the release rule once more at now, with the slot's deadline
        if held(0):
            t = next_ + 1
        elif far >= p.D + 1:
            t = LOST
            add["lost"] += 1
        elif not stalled() and ser32(now - (a_t + ser16(next_ - a_s) * period(p))) >= deadline:
            t = LOST
            add["lost"] += 1
            add["expired"] += 1
        else:
            break
        push(t)
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
    ring = st[:, p.o_ring:p.o_hist].reshape(p.C, R, P)
    for j, at in enumerate(cp):
        if at >= 0:
            ring[:, at] = jm.clean(x[:, j * P:(j + 1) * P])
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
            tau = jm.pitch(win[:, base:base + H], p, trace, force.pop(0) if force else None)
            run = 0
            per[:, :tau] = win[:, base + H - tau:base + H]
            h[12] = tau
        g = np.array([jm.gain(min(run + q, p.gb), p) for q in i])
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
    for k, name in zip((6, 7, 8, 9, 10, EXPIRED), ("lost", "late", "dup", "dropped", "restarts", "expired")):
        h[k] = min(max(int(h[k]), 0) + add[name], 2 ** 31 - 1)
    h[11] = nheld
    h[4], h[5] = (run if tau else 0), tau
    h[A_S], h[A_T] = a_s, ser32(a_t)
    return win[:, H:H + n_out * P], n_out


def adaptive_run(a, src, plan, st=None, check=None, lateness=None):
    """plan: (arrivals, now) or (arrivals, now, arrival times) per call, packet s being src(s) [C, P], or src[s % len]
    for a list.  Returns (the outputs per call, the out counts, the final state); check(st, m, k) runs after call k."""
    p = a.p
    st = a.fresh()[0] if st is None else st
    packet = src if callable(src) else (lambda s: src[s % len(src)])
    ys, ms = [], []
    for k, call in enumerate(plan):
        seq, now = call[0], call[1]
        times = call[2] if len(call) > 2 else None
        x = np.concatenate([packet(s) for s in seq], 1) if seq else np.zeros((p.C, 0), np.float32)
        y, m = adaptive_call(st, x, seq, len(seq), a, now, times, lateness=lateness)
        ys.append(y)
        ms.append(m)
        if check:
            check(st, m, k)
    return ys, ms, st


def timed_plan(arrive, t0=0, tick=tm.TICK, extra=2):
    """tm.ticked with each packet's own arrival time: (packets, now, arrival times) per tick"""
    items = sorted((t, s) for s, t in arrive.items() if t is not None)
    last = max(t for t, _ in items)
    plan, k = [], 0
    while True:
        now = k * tick
        got = [(t, s) for t, s in items if now - tick < t <= now]
        plan.append(([s for _, s in got], t0 + now, [t0 + t for t, _ in got]))
        if now >= last + extra * tick:
            return plan
        k += 1


def jittered(n, lat, T=10000, first=0, seed=0, gone=()):
    """arrival times of packets first .. first + n - 1 sent every T µs from 1000, packet k delayed by lat(k, rng) µs"""
    g = np.random.default_rng(seed)
    return {(first + k) & (SEQ - 1): None if k in gone else 1000 + k * T + int(lat(k, g)) for k in range(n)}


def gamma_lat(shape, scale, shift=2000):
    return lambda k, g: shift + g.gamma(shape, scale)


def words(st):
    return st[0].view(np.int32)


def cat(ys):
    return np.concatenate(ys, 1)


# ---- lo == hi: the timed buffer ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("rate,P,W,D", [(16000, 160, 16, 1), (44100, 441, 8, 0), (48000, 480, 16, 3)])
def test_equal_bounds_are_the_timed_buffer(rate, P, W, D):
    p = jm.Params(rate, P, C=2, D=D, W=W, max_out=4)
    T = period(p)
    pk = jm.packets_of(p, 64, 4)
    late = 0
    for seed, dl in enumerate((15000, 2 * T + 1000)):
        arrive = jittered(120, gamma_lat(2.0, 4000.0), T, first=65500, seed=seed, gone={30, 31, 50, 70, 71, 72, 73})
        for k in range(60, 60 + 12):             # an outage longer than S: stalls and a restart
            arrive[(65500 + k) & (SEQ - 1)] = None
        plan = tm.ticked(arrive, t0=2 ** 31 - 300000)
        a = Adapt(p, dl, dl)
        st0, st1 = p.fresh()[0], a.fresh()[0]
        for k, (seq, now) in enumerate(plan):
            x = np.concatenate([pk[s % 64] for s in seq], 1) if seq else np.zeros((p.C, 0), np.float32)
            want, m0 = tm.timed_call(st0, x, seq, len(seq), p, now, dl)
            # arrival times equal to now, or none at all
            got, m1 = adaptive_call(st1, x, seq, len(seq), a, now, [now] * len(seq) if k % 2 else None)
            assert m0 == m1 and np.array_equal(got.view(np.int32), want.view(np.int32)), k
            assert np.array_equal(st1[:, :p.rf].view(np.int32), st0.view(np.int32)), k
            assert stats(st1, a)[2] == (dl if words(st1)[0] else 0)
        assert words(st0)[EXPIRED] > 0 and words(st0)[10] > 0     # deadline releases and a restart
        late += int(words(st0)[7])
    assert late > 0


# ---- the statistics --------------------------------------------------------------------------------------------------
def test_warm_up_holds_hi():
    p = jm.Params(44100, 441, C=1, D=1, W=16, max_out=8)
    a = Adapt(p, 0, 60000, 0.05)
    assert a.warm == 20 and a.w == 938 and a.N == 500 and a.r == 3277
    plan = timed_plan(jittered(60, lambda k, g: 3000 + 100 * (k % 3), period(p)))
    seen = []

    def check(st, m, k):
        seen.append(stats(st, a)[1:])

    adaptive_run(a, jm.packets_of(p, 8, 1), plan, check=check)
    seen = [v for v in seen if v != (0, 0)]          # from the call that takes the first packet
    assert seen and all(dl == 60000 for k, dl in seen if k < 20)
    assert any(dl < 60000 for k, dl in seen if k >= 20)
    assert seen[-1][0] == 59 and seen[-1][1] < 10000             # the first packet is not measured


def test_the_update_is_a_mean_then_forgets():
    """the first N packets weigh equally (to the integer floors), later ones forget with memory N"""
    a = Adapt(jm.Params(16000, 160), 0, 6400)
    h = np.zeros(BINS, np.int64)
    k = update(h, 0, [3] * 10 + [5] * 10, a)
    assert k == 20 and abs(h[3] - UNIT // 2) <= 64 and abs(h[5] - UNIT // 2) <= 64 and abs(int(h.sum()) - UNIT) <= 64
    k = update(h, k, [7] * (a.N - 20), a)
    assert abs(h[3] - 10 * UNIT // a.N) <= 2 * a.N and abs(int(h.sum()) - UNIT) <= 64 * a.N
    h2 = h.copy()
    update(h2, 2 * a.N, [9] * a.N, a)
    assert abs(h2[3] / h[3] - (1 - 1 / a.N) ** a.N) < 0.01


def test_stationary_trace_finds_the_quantile(late_rate=0.02):
    """a seeded stationary trace of 20 000 packets, lateness a shifted gamma: the steady-state deadline lies within one
    bin of the float64 (1 - late_rate) quantile of the measured lateness, and the packets dropped as late are at most
    1.5 late_rate of those that arrived"""
    p = jm.Params(16000, 160, C=1, D=1, W=16, max_out=8)
    a = Adapt(p, 0, 64000, late_rate)
    T = period(p)
    arrive = jittered(20000, gamma_lat(2.0, 3000.0), T, seed=11)
    plan = timed_plan(arrive)
    lat, dls = [], []

    def check(st, m, k):
        dls.append(stats(st, a)[2])

    _, _, st = adaptive_run(a, [np.zeros((1, p.P), np.float32)], plan, check=check, lateness=lat)
    q = float(np.quantile(np.asarray(lat[len(lat) // 4:], np.float64), 1 - late_rate))
    steady = np.asarray(dls[len(dls) // 4:])
    med = float(np.median(steady))
    assert med - 2 * a.w <= q <= med + a.w, (q, med, a.w)
    assert words(st)[7] <= 1.5 * late_rate * 20000, (words(st)[7], late_rate)
    assert words(st)[10] == 0


def test_a_step_in_jitter_moves_the_deadline():
    """2 ms of jitter, then 30 ms, then 2 ms again: the deadline rises within a few N late_rate packets and falls back
    within a few N"""
    p = jm.Params(44100, 441, C=1, D=1, W=16, max_out=8)
    a = Adapt(p, 0, 64000, 0.02)
    T, N = period(p), a.N
    n1, n2, n3 = 2000, 1500, 3000

    def lat(k, g):
        return 2000 + (g.uniform(0, 30000) if n1 <= k < n1 + n2 else g.uniform(0, 2000))

    arrive = jittered(n1 + n2 + n3, lat, T, seed=5)
    plan = timed_plan(arrive)
    by_packet = {}

    def check(st, m, k):
        by_packet[max(plan[k][0], default=-1)] = stats(st, a)[2]

    adaptive_run(a, [np.zeros((1, p.P), np.float32)], plan, check=check)
    dl = np.full(n1 + n2 + n3, a.hi)                 # the deadline after the call that took packet s (or the last one)
    for s in range(n1 + n2 + n3):
        dl[s] = by_packet.get(s, dl[s - 1] if s else a.hi)
    low = np.median(dl[n1 - 500:n1])
    assert low <= 4 * a.w + 2000
    rise = int(np.argmax(dl[n1:] > low + 2 * a.w)), int(np.argmax(dl[n1:] >= 15000))
    assert 0 < rise[0] <= 3 * N * a.late_rate and rise[1] <= 5 * N * a.late_rate, rise
    assert np.median(dl[n1 + n2 - 300:n1 + n2]) >= 25000
    fall = int(np.argmax(dl[n1 + n2:] <= low + a.w))
    assert 0 < fall <= 5 * N, (fall, N)


def test_what_is_measured():
    """first packets, duplicates, restarts and arrivals while stalled leave the statistics as they are; placed and late
    packets are measured against the anchor in force"""
    p = jm.Params(16000, 160, C=1, D=15, W=16, max_out=16)
    a = Adapt(p, 0, 64000, 0.5)
    T = period(p)
    pk = jm.packets_of(p, 64, 2)
    st = a.fresh()[0]
    lat = []
    adaptive_run(a, pk, [([5], 10000, [9000])], st=st, lateness=lat)      # the first packet: the anchor, unmeasured
    assert stats(st, a)[1] == 0 and lat == [] and words(st)[A_T] == 9000
    adaptive_run(a, pk, [([7, 7], 40000, [9000 + 2 * T + 700, 39000])], st=st, lateness=lat)   # a duplicate
    assert stats(st, a)[1] == 1 and lat == [700]
    adaptive_run(a, pk, [([6, 4], 41000, [41000, 41000])], st=st, lateness=lat)   # 6 placed; then 4 is late
    assert lat[1:] == [41000 - (9000 + 2 * T + 700 - T), 41000 - (9000 + 2 * T + 700 - 3 * T)]
    assert words(st)[7] == 1 and stats(st, a)[1] == 3
    b, k, _ = stats(st, a)
    assert b[bin_of(lat[1], a)] > 0 and b[bin_of(lat[2], a)] > 0
    adaptive_run(a, pk, [([7 + 40], 42000, [42000])], st=st, lateness=lat)    # beyond the window: a restart
    assert words(st)[10] == 1 and stats(st, a)[1] == 3
    # stall: nothing arrives until the slot has expired S packets past the anchor
    t = 42000
    while words(st)[1] - 47 - 1 < stall(p):
        t += tm.TICK
        adaptive_run(a, pk, [([], t)], st=st)
    before = stats(st, a)
    adaptive_run(a, pk, [([46, 45], t + 1000, [t + 500, t + 900])], st=st, lateness=lat)   # late while stalled
    assert stats(st, a)[1] == before[1] and words(st)[7] == 3
    adaptive_run(a, pk, [([int(words(st)[1]) + 1], t + 2000)], st=st, lateness=lat)      # the restart out of a stall
    assert stats(st, a)[1] == before[1] and words(st)[10] == 2
    assert np.array_equal(stats(st, a)[0], before[0])


def test_cuts_give_the_same_statistics():
    """the same timestamped arrivals cut into other calls (each at a clock no earlier than its arrivals, deadlines never
    reached) give the same statistics, anchors and counters"""
    p = jm.Params(44100, 441, C=1, D=2, W=16, max_out=64)
    a = Adapt(p, 50000, 64000, 0.05)
    T = period(p)
    arrive = jittered(400, gamma_lat(2.0, 3000.0), T, seed=9, gone={40, 41, 200})
    items = sorted((t, s) for s, t in arrive.items() if t is not None)
    pk = [np.zeros((1, p.P), np.float32)]
    results = []
    for seed in range(3):
        cuts = jm.random_cuts(len(items), 100 + seed, 5)
        plan, i = [], 0
        for c in cuts:
            got = items[i:i + c]
            i += c
            if got:
                plan.append(([s for _, s in got], got[-1][0] + seed * 997, [t for t, _ in got]))
        _, _, st = adaptive_run(a, pk, plan)
        results.append(st)
    for st in results[1:]:
        assert np.array_equal(st[0, a.o_stats:].view(np.int32), results[0][0, a.o_stats:].view(np.int32))
        assert np.array_equal(words(st)[[1, 6, 7, 8, 10, A_S, A_T]], words(results[0])[[1, 6, 7, 8, 10, A_S, A_T]])
    assert stats(results[0], a)[1] > 300 and words(results[0])[EXPIRED] == 0


def test_arrivals_after_now_are_now():
    p = jm.Params(16000, 160, C=2, D=1, W=16, max_out=8)
    a = Adapt(p, 5000, 40000, 0.05)
    T = period(p)
    plan = timed_plan(jittered(200, gamma_lat(1.5, 4000.0), T, seed=3, gone={50, 51, 52}))
    pk = jm.packets_of(p, 16, 3)
    want, _, st0 = adaptive_run(a, pk, [(seq, now, [now] * len(seq)) for seq, now, _ in plan])
    later = [(seq, now, [now + 1 + 7 * j for j in range(len(seq))]) for seq, now, _ in plan]
    got, _, st1 = adaptive_run(a, pk, later)
    assert np.array_equal(cat(got).view(np.int32), cat(want).view(np.int32))
    assert np.array_equal(st1.view(np.int32), st0.view(np.int32))


@pytest.mark.parametrize("t0,first", [(2 ** 31 - 60000, 65520), (2 ** 32 - 60000, 65530), (-60000, 100)])
def test_sequence_and_clock_wraps(t0, first):
    p = jm.Params(44100, 441, C=2, D=1, W=16, max_out=8)
    a = Adapt(p, 5000, 60000, 0.05)
    T = period(p)
    pk = jm.packets_of(p, 40, 27)
    lat = gamma_lat(2.0, 4000.0)
    gone = {60, 61, 62, 100, 101, 102, 103, 104, 105, 106, 107, 108}
    want, _, st0 = adaptive_run(a, lambda s: pk[(s - 1000) % 40], timed_plan(jittered(300, lat, T, 1000, 8, gone)))
    got, _, st = adaptive_run(a, lambda s: pk[(s - first) % SEQ % 40], timed_plan(jittered(300, lat, T, first, 8, gone), t0))
    assert np.array_equal(cat(got).view(np.int32), cat(want).view(np.int32))
    assert np.array_equal(words(st)[6:13], words(st0)[6:13]) and words(st)[EXPIRED] == words(st0)[EXPIRED] > 0
    assert np.array_equal(st[0, a.o_stats:].view(np.int32), st0[0, a.o_stats:].view(np.int32))
    assert stats(st, a)[2] < 60000


# ---- interfaces ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from lookoncetohear_b200 import _cabi, build
    build.build()
    return _cabi.lib()


def test_entry_exported_and_documented(lib):
    hdr = header()
    for name in ("l2h_jitter_buffer_adaptive", "l2h_jitter_buffer_adaptive_layout"):
        assert hasattr(lib, name) and declaration(hdr, name)[0], name
    decl, args = declaration(hdr, "l2h_jitter_buffer_adaptive")
    doc = doc_before(hdr, hdr.index("int l2h_jitter_buffer_adaptive_layout("))
    for arg in ("now_dev", "arrivals_dev", "lo_us", "hi_us", "late_rate"):
        assert arg in args and arg in doc, arg
    for words_ in ("serial", "anchor", "lateness", "late packet", "first packet", "duplicate", "restarts the slot",
                   "stalled", "64", "max(1, ceil(hi_us / 64))", "clamp(floor(l / w), 0, 63)", "round(5e6 / period)",
                   "min(k + 1, N)", "floor(2^24 / m)", "round(late_rate 2^16)", "T_b 2^16 <= r T",
                   "clamp((b + 1) w, lo_us", "ceil(1 / late_rate)", "lo_us == hi_us", "bit", "66", "Errors", "1 = "):
        assert words_ in doc, words_


@pytest.mark.parametrize("rate,P,W", [(16000, 160, 16), (44100, 441, 8)])
def test_layout(lib, rate, P, W):
    rf, rfa = ctypes.c_int32(), ctypes.c_int32()
    assert lib.l2h_jitter_buffer_layout(2, rate, P, 1, W, 4, ctypes.byref(rf)) == 0
    assert lib.l2h_jitter_buffer_adaptive_layout(2, rate, P, 1, W, 4, ctypes.byref(rfa)) == 0
    assert rf.value == jm.Params(rate, P, W=W).rf and rfa.value == rf.value + STATS
    assert lib.l2h_jitter_buffer_adaptive_layout(2, rate, P, W, W, 4, ctypes.byref(rfa)) == 1
    assert lib.l2h_jitter_buffer_adaptive_layout(2, rate, P, 1, W, 4, None) == 1


def test_call_errors(lib):
    i32 = ctypes.c_void_p(0x20000)

    def call(now=i32, lo=5000, hi=40000, rate_=0.02, slots=i32, n=2, depth=1, arrivals=None):
        return lib.l2h_jitter_buffer_adaptive(FAKE_DEV, 320, 320, 2, i32, i32, ctypes.c_void_p(0x100000), 640, 640, i32,
                                              n, 1, slots, FAKE_DEV, 4, 16000, 160, depth, 16, 4, now, arrivals, lo, hi,
                                              rate_, None)

    assert call(now=None) == 1 and "l2h_jitter_buffer_adaptive" in lib.l2h_last_error().decode()
    for kw in (dict(lo=-1), dict(lo=5000, hi=4999), dict(hi=-1)):
        assert call(**kw) == 1 and "lo_us" in lib.l2h_last_error().decode(), kw
    for bad in (0.0, -0.1, 0.51, float("nan"), float("inf")):
        assert call(rate_=bad) == 1 and "late_rate" in lib.l2h_last_error().decode(), bad
    assert call(slots=None) == 1 and call(n=5) == 1 and call(depth=16) == 1
    assert "l2h_jitter_buffer_adaptive" in lib.l2h_last_error().decode()


def test_constructor_checks():
    for bad in ((1,), (1, 2, 3), (-1, 5), (5, 4), (0, 2 ** 31), (1.5, 3), (True, 3)):
        with pytest.raises(ValueError):
            JitterBuffer(4, 2, 44100, 441, deadline=bad, device="cpu")
    for bad in (0, 0.0, -0.1, 0.6, float("nan"), True, "0.1"):
        with pytest.raises(ValueError, match="late_rate"):
            JitterBuffer(4, 2, 44100, 441, deadline=(0, 40000), late_rate=bad, device="cpu")
    for deadline in (None, 20000):
        with pytest.raises(ValueError, match="late_rate"):
            JitterBuffer(4, 2, 44100, 441, deadline=deadline, late_rate=0.02, device="cpu")
    with pytest.raises(RuntimeError, match="CUDA"):
        JitterBuffer(4, 2, 44100, 441, deadline=(0, 40000), late_rate=0.5, device="cpu")


def stub(adaptive=True):
    jb = JitterBuffer.__new__(JitterBuffer)
    jb.state, jb.adaptive = torch.zeros(3, 1, 10), adaptive
    jb.deadline = (0, 40000) if adaptive else 20000
    return jb


def test_arrivals_checks():
    jb = stub()
    assert jb._arrivals(None, 2, 3) is None
    got = jb._arrivals([[5, 2 ** 31, -1], [2 ** 32 + 7, 3 * 2 ** 32 - 2, 0]], 2, 3)
    assert got.dtype == torch.int32 and got.tolist() == [[5, -2 ** 31, -1], [7, -2, 0]]
    assert jb._arrivals(np.arange(6, dtype=np.uint32).reshape(2, 3), 2, 3).tolist() == [[0, 1, 2], [3, 4, 5]]
    for bad in ([[1.0, 2, 3], [4, 5, 6]], [[1, 2], [3, 4]], [[True, False, True]] * 2, "abc", [[2 ** 70, 0, 0]] * 2):
        with pytest.raises(ValueError, match="arrivals"):
            jb._arrivals(bad, 2, 3)
    with pytest.raises(ValueError, match="adaptive"):
        stub(False)._arrivals([[1, 2, 3]] * 2, 2, 3)
    assert stub(False)._arrivals(None, 2, 3) is None


def test_deadline_us_view():
    jb = stub()
    jb.state[:, 0, -1] = torch.tensor([7, 8, 9], dtype=torch.int32).view(torch.float32)
    assert jb.deadline_us.tolist() == [7, 8, 9]
    with pytest.raises(ValueError, match="adaptive"):
        stub(False).deadline_us
