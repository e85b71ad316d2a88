"""The jitter buffer released on time (JitterBuffer(deadline=...), l2h_jitter_buffer_timed) without a GPU: an exact model
of its bookkeeping and a float64 model of its concealment over the kernel's own state layout, built on the untimed model
of tests/test_jitter_buffer_cpu.py (so the GPU tests can run one call of it from the kernel's state), checked against
the rules of include/lookonce_b200.h; and the argument errors, the Python checks, the header and the export."""
import ctypes

import numpy as np
import pytest
import torch

import test_jitter_buffer_cpu as jm
from lookoncetohear_b200 import JitterBuffer
from serving_util import FAKE_DEV, declaration, doc_before, header

HEAD, LOST, RECOVER, SEQ = jm.HEAD, jm.LOST, jm.RECOVER, jm.SEQ
A_S, A_T, EXPIRED = 13, 14, 15                       # channel 0's head words of the timed form
NEVER = 2 ** 31 - 1                                  # a deadline no call below reaches
TICK = 8000                                          # the server's tick, µs


def ser16(v):
    v &= SEQ - 1
    return v - SEQ if v >= SEQ // 2 else v


def ser32(v):
    v &= 0xFFFFFFFF
    return v - 2 ** 32 if v >= 2 ** 31 else v


def period(p):
    """round(1e6 packet / rate) µs, exactly"""
    return (2_000_000 * p.P + p.rate) // (2 * p.rate)


def stall(p):
    """S = ceil(gb / packet): the packets past the anchor after which deadline releases stop"""
    return -(-p.gb // p.P)


def timed_call(st, x, seqs, cnt, p, now, deadline, force=None, trace=None):
    """One timed call of one row at clock `now` (µs, any int, taken mod 2^32), as jm.model_call: st [C, rf] float32
    updated in place.  Returns (y [C, m P] float32, m)."""
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

    far = max([d for d in range(W) if held(d)], default=-1)
    cp = [-1] * cnt
    for j in range(cnt):
        s = int(seqs[j])
        if s < 0 or s >= SEQ:
            continue
        if not started:
            started, next_, a_s = True, s, s
        d = ser16(s - next_)
        recover = False
        if d < 0:
            add["late"] += 1
            continue
        if d < W and not stalled():
            if held(d):
                add["dup"] += 1
                continue
        else:
            for e in range(W):
                add["dropped"] += int(held(e))
                tg[slot(e)] = 0
            add["restarts"] += 1
            next_, d, far, recover, a_s = s, 0, -1, True, s
        if ser16(s - a_s) >= 0:
            a_s, a_t = s, now
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
    while started:                                   # the release rule once more at now, with the deadline
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


def timed_run(p, src, plan, deadline, st=None, check=None):
    """plan: (arrivals, now) per call, packet s being src(s) [C, P], or src[s % len] for a list.  Returns (the outputs
    per call, the out counts, the final state); check(st, m, k) runs after call k."""
    st = p.fresh()[0] if st is None else st
    packet = src if callable(src) else (lambda s: src[s % len(src)])
    ys, ms = [], []
    for k, (seq, now) in enumerate(plan):
        x = np.concatenate([packet(s) for s in seq], 1) if seq else np.zeros((p.C, 0), np.float32)
        y, m = timed_call(st, x, seq, len(seq), p, now, deadline)
        ys.append(y)
        ms.append(m)
        if check:
            check(st, m, k)
    return ys, ms, st


def ticked(arrive, t0=0, tick=TICK, extra=2):
    """a plan from arrival times: arrive[s] the µs at which packet s reaches the server (None: never).  Call k runs at
    t0 + k tick with the packets that arrived since the last tick, in arrival order; `extra` more ticks follow."""
    items = sorted((t, s) for s, t in arrive.items() if t is not None)
    last = max(t for t, _ in items)
    plan, k = [], 0
    while True:
        now = k * tick
        plan.append(([s for t, s in items if now - tick < t <= now], t0 + now))
        if now >= last + extra * tick:
            return plan
        k += 1


def stream(n, P=10000, lat=3000, gone=(), late=None, first=0):
    """the arrival times of packets first .. first + n - 1 sent every P µs from 1000 with a fixed latency; `gone` never
    arrive, `late` maps a packet to an extra delay"""
    late = late or {}
    return {(first + k) & (SEQ - 1): None if k in gone else 1000 + k * P + lat + late.get(k, 0) for k in range(n)}


def words(st):
    return st[0].view(np.int32)


def cat(ys):
    return np.concatenate(ys, 1)


# ---- the deadline never reached: the untimed buffer ------------------------------------------------------------------
@pytest.mark.parametrize("rate,P,W,D", [(16000, 160, 16, 1), (44100, 441, 8, 0), (48000, 480, 16, 3)])
def test_unreached_deadline_is_the_untimed_buffer(rate, P, W, D):
    p = jm.Params(rate, P, C=2, D=D, W=W, max_out=4)
    pk = jm.packets_of(p, 64, 4)
    for seed, arr in enumerate((jm.schedule(120, 5, loss=0.15, start=65500), jm.schedule(90, 8, loss=0.3, swap=0.2))):
        cuts = jm.random_cuts(len(arr), seed, 3) + [0] * 30
        st0, st1, a = p.fresh()[0], p.fresh()[0], 0
        for k, c in enumerate(cuts):
            seq = arr[a:a + c]
            x = np.concatenate([pk[s % 64] for s in seq], 1) if seq else np.zeros((p.C, 0), np.float32)
            want, m0 = jm.model_call(st0, x, seq, c, p)
            got, m1 = timed_call(st1, x, seq, c, p, 2 ** 31 - 5000 + k * TICK, NEVER)   # the clock wraps too
            assert m0 == m1 and np.array_equal(got.view(np.int32), want.view(np.int32)), k
            assert np.array_equal(words(st1)[:13], words(st0)[:13]), k
            assert np.array_equal(st1[:, HEAD:].view(np.int32), st0[:, HEAD:].view(np.int32))
            a += c
        assert words(st1)[EXPIRED] == 0


# ---- outages ---------------------------------------------------------------------------------------------------------
def test_an_outage_is_concealed_as_it_happens():
    """k < S packets never arrive: each call releases exactly the gap packets whose deadlines have passed by its now,
    gap packets that arrive after that are late, and no call writes more than the packets due by its clock"""
    p = jm.Params(44100, 441, C=2, D=3, W=16, max_out=8)      # depth 3 leaves the gap to the clock
    T, dl = period(p), 15000
    pk = jm.packets_of(p, 40, 21)
    gap = range(10, 14)
    arrive = stream(30, T, gone=set(gap) - {12}, late={12: 90000})     # 12 arrives 90 ms late
    plan = ticked(arrive)
    a_t = max(now for seq, now in plan if 9 in seq)  # the anchor while the gap lasts: packet 9 and its call
    sent = []

    def check(st, m, k):
        now = plan[k][1]
        due = [s for s in gap if now - (a_t + (s - 9) * T) >= dl]
        w = words(st)
        if k < [i for i, (seq, _) in enumerate(plan) if 14 in seq][0]:
            assert w[6] == w[EXPIRED] == len(due), (k, due)
        assert w[EXPIRED] <= w[6]
        sent.append(m)
        # the packets due by the clock: everything sent before now - latency - deadline, plus one in flight
        assert sum(sent) <= (now - 1000 - 3000) // T + 2, (k, sent)

    ys, ms, st = timed_run(p, pk, plan, dl, check=check)
    w = words(st)
    assert (w[6], w[EXPIRED], w[7], w[10]) == (4, 4, 1, 0) and max(ms) <= 2
    y = cat(ys)
    assert y.shape[1] == 30 * p.P
    assert np.array_equal(y[:, :10 * p.P], cat(pk[:10]))
    assert np.array_equal(y[:, 14 * p.P + p.lr:], cat(pk[14:30])[:, p.lr:])
    # the untimed buffer on the same calls writes nothing while the gap lasts
    st0, outs = p.fresh()[0], []
    for seq, _ in plan:
        x = np.concatenate([pk[s % 40] for s in seq], 1) if seq else np.zeros((p.C, 0), np.float32)
        outs.append(jm.model_call(st0, x, seq, len(seq), p)[1])
    i14 = [i for i, (seq, _) in enumerate(plan) if 14 in seq][0]
    assert sum(outs[:i14]) == 10 < sum(ms[:i14])


@pytest.mark.parametrize("rate,P", [(44100, 441), (16000, 160)])
def test_a_long_outage_stops_at_s_and_restarts(rate, P):
    p = jm.Params(rate, P, C=2, D=1, W=16, max_out=8)
    T, S, dl = period(p), stall(p), 20000
    assert S == 6
    pk = jm.packets_of(p, 64, 22)
    arrive = stream(40, T, gone=set(range(8, 28)), first=65530)         # a 200 ms outage across the wrap
    plan = ticked(arrive)
    ys, ms, st = timed_run(p, pk, plan, dl)
    w = words(st)
    assert (w[6], w[EXPIRED], w[10], w[7]) == (S, S, 1, 0)
    y = cat(ys)
    assert y.shape[1] == (8 + S + 12) * P           # no silent packets: the restart at 28 follows the S concealed ones
    seqs = [(65530 + k) & (SEQ - 1) for k in range(40)]
    assert np.array_equal(y[:, :8 * P], cat([pk[s % 64] for s in seqs[:8]]))
    conceal = y[:, 8 * P:(8 + S) * P]
    assert np.any(conceal[:, :p.ga] != 0)
    after = y[:, (8 + S) * P:]
    want = cat([pk[s % 64] for s in seqs[28:]])
    assert not np.array_equal(after[:, :p.lr], want[:, :p.lr])          # faded in
    assert np.array_equal(after[:, p.lr:], want[:, p.lr:])
    assert w[1] == (seqs[-1] + 1) & (SEQ - 1) and w[A_S] == seqs[-1]


def test_a_stalled_slot_keeps_late_packets_late():
    p = jm.Params(16000, 160, D=1, W=16, max_out=8)
    pk = jm.packets_of(p, 16, 23)
    st = p.fresh()[0]
    timed_run(p, pk, [([0, 1, 2], 0)] + [([], t * TICK) for t in range(1, 20)], 10000, st=st)
    w = words(st)
    assert (w[1], w[6], w[EXPIRED]) == (3 + stall(p), stall(p), stall(p))
    timed_run(p, pk, [([2, 1], 20 * TICK)], 10000, st=st)                 # behind next: late, no restart
    assert (words(st)[7], words(st)[10]) == (2, 0)
    timed_run(p, pk, [([3 + stall(p)], 21 * TICK)], 10000, st=st)        # at next: a restart
    assert (words(st)[10], words(st)[1]) == (1, 4 + stall(p))


# ---- reordering and the deadline against depth -----------------------------------------------------------------------
def test_reordering_inside_the_deadline_is_the_stream():
    p = jm.Params(44100, 441, C=2, D=1, W=16, max_out=8)
    T = period(p)
    pk = jm.packets_of(p, 40, 24)
    late = {5: 12000, 11: 18000, 20: 9000}         # swaps, up to two ticks late
    plan = ticked(stream(30, T, late=late))
    ys, _, st = timed_run(p, pk, plan, 25000)
    assert np.array_equal(cat(ys).view(np.int32), cat(pk[:30]).view(np.int32))
    assert words(st)[6:8].tolist() == [0, 0] and words(st)[EXPIRED] == 0
    # beyond the deadline: late, and concealed
    ys, _, st = timed_run(p, pk, plan, 8000)
    w = words(st)
    assert w[6] == w[EXPIRED] == w[7] >= 1
    assert cat(ys).shape[1] == 30 * p.P


@pytest.mark.parametrize("e", [1, 2, 4])
def test_a_deadline_of_e_periods_acts_as_depth(e):
    """every call at one now: the deadline fires from the anchor alone, at the arrival e past the gap"""
    p = jm.Params(16000, 160, D=15, W=16, max_out=16)
    T = period(p)
    pk = jm.packets_of(p, 16, 25)
    st = p.fresh()[0]
    timed_run(p, pk, [([0, 1, 2], 5000)], e * T, st=st)
    for k in range(1, e + 1):
        timed_run(p, pk, [([3 + k], 5000)], e * T, st=st)
        assert words(st)[6] == int(k == e), k
    assert words(st)[EXPIRED] == 1 and words(st)[1] == 4 + e


# ---- clocks, wraps and max_out ---------------------------------------------------------------------------------------
def outage_plan(t0, first):
    return ticked(stream(40, 10000, gone={6, 7, 8, 15, 16, 17, 18, 19, 20, 21, 22, 23, 30}, late={11: 25000},
                         first=first), t0=t0)


@pytest.mark.parametrize("t0,first", [(2 ** 31 - 60000, 65520), (2 ** 32 - 60000, 65530), (-60000, 100)])
def test_sequence_and_clock_wraps(t0, first):
    p = jm.Params(44100, 441, C=2, D=1, W=16, max_out=8)
    pk = jm.packets_of(p, 40, 27)
    want, _, st0 = timed_run(p, lambda s: pk[(s - 1000) % 40], outage_plan(0, 1000), 20000)
    got, _, st = timed_run(p, lambda s: pk[(s - first) % SEQ], outage_plan(t0, first), 20000)
    assert np.array_equal(cat(got).view(np.int32), cat(want).view(np.int32))
    assert np.array_equal(words(st)[6:13], words(st0)[6:13]) and words(st)[EXPIRED] == words(st0)[EXPIRED] > 0


def test_max_out_moves_only_the_cut():
    p0 = jm.Params(44100, 441, C=2, D=1, W=16, max_out=64)
    pk = jm.packets_of(p0, 64, 26)
    plan = outage_plan(0, 65500)
    plan += [([], plan[-1][1])] * 20                 # the backlog drains at the last clock

    def lost_ok(st, m, k):
        assert words(st)[EXPIRED] <= words(st)[6], k

    want, _, st0 = timed_run(p0, pk, plan, 15000, check=lost_ok)
    for mo in (2, 3, 5):
        p = jm.Params(44100, 441, C=2, D=1, W=16, max_out=mo)
        got, _, st = timed_run(p, pk, plan, 15000, check=lost_ok)
        assert np.array_equal(cat(got).view(np.int32), cat(want).view(np.int32)), mo
        assert np.array_equal(words(st)[6:11], words(st0)[6:11]) and words(st)[EXPIRED] == words(st0)[EXPIRED]


# ---- interfaces ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from lookoncetohear_b200 import _cabi, build
    build.build()
    return _cabi.lib()


def test_entry_exported_and_documented(lib):
    hdr = header()
    assert hasattr(lib, "l2h_jitter_buffer_timed")
    decl, args = declaration(hdr, "l2h_jitter_buffer_timed")
    assert decl
    doc = doc_before(hdr, decl.start())
    for a in ("now_dev", "deadline_us"):
        assert a in args and a in doc, a
    for words_ in ("serial arithmetic", "anchor", "expired", "stall", "restart", "round(1e6 P / rate)", "13", "15",
                   "lists every live slot", "bit for", "max_out", "Errors", "1 = "):
        assert words_ in doc, words_


def test_call_errors(lib):
    i32 = ctypes.c_void_p(0x20000)

    def call(now=i32, deadline=10000, slots=i32, n=2, depth=1):
        return lib.l2h_jitter_buffer_timed(FAKE_DEV, 320, 320, 2, i32, i32, ctypes.c_void_p(0x100000), 640, 640, i32, n,
                                           1, slots, FAKE_DEV, 4, 16000, 160, depth, 16, 4, now, deadline, None)

    assert call(now=None) == 1 and "l2h_jitter_buffer_timed" in lib.l2h_last_error().decode()
    assert call(deadline=-1) == 1 and "deadline" in lib.l2h_last_error().decode()
    assert call(slots=None) == 1 and call(n=5) == 1 and call(depth=16) == 1
    assert "l2h_jitter_buffer_timed" in lib.l2h_last_error().decode()


def test_constructor_and_call_checks():
    for bad in (-1, True, 1.5, 2 ** 31):
        with pytest.raises(ValueError):
            JitterBuffer(4, 2, 44100, 441, deadline=bad, device="cpu")
    with pytest.raises(RuntimeError, match="CUDA"):
        JitterBuffer(4, 2, 44100, 441, deadline=20000, device="cpu")
    jb = JitterBuffer.__new__(JitterBuffer)
    jb.state, jb.deadline = torch.zeros(1), None
    assert jb._now(None) is None
    with pytest.raises(ValueError, match="without a deadline"):
        jb._now(5)
    jb.deadline = 20000
    with pytest.raises(ValueError, match="needs now"):
        jb._now(None)
    for bad in (1.0, True, "5", torch.zeros(1, dtype=torch.int32)):
        with pytest.raises(ValueError):
            jb._now(bad)


def test_host_clock_is_taken_mod_2_32():
    jb = JitterBuffer.__new__(JitterBuffer)
    jb.state, jb.deadline = torch.zeros(1), 0
    for v, want in ((5, 5), (2 ** 31, -2 ** 31), (2 ** 32 + 7, 7), (-1, -1), (3 * 2 ** 32 - 2, -2)):
        assert jb._now(v).tolist() == [want]
