"""The jitter buffer with adaptive deadlines on the GPU (JitterBuffer(deadline=(lo, hi)), l2h_jitter_buffer_adaptive),
against the adaptive model of tests/test_jitter_adaptive_cpu.py, each call compared with one call of the model run from
the kernel's own state before it, with the bounds and the near-tie rule of tests/test_jitter_buffer_gpu.py.  Also: equal
bounds give the timed buffer bit for bit, graph replays with the lists, the clock and the arrival times rewritten in
place, rows that store nothing, and mixed links on one state through jb -> PacketResampler -> HopFifo at 44.1 kHz."""
import numpy as np
import pytest
import torch

import serving_util as su
import test_jitter_adaptive_cpu as am
import test_jitter_buffer_cpu as jm
import test_jitter_deadline_cpu as tm
from lookoncetohear_b200 import HopFifo, JitterBuffer, PacketResampler
from serving_util import dev  # noqa: F401
from test_jitter_buffer_gpu import BOUND_U, CASES, near_tie

pytestmark = pytest.mark.gpu


def model_row(before, after, x, seqs, count, a, now, times, stats):
    """one adaptive model call from the kernel's state `before` [C, rf] of a slot: (y, out count, the model's state
    after); run again at the kernel's lag (in `after`) where the two lie within the fp32 error of their scores"""
    st, trace = before.copy(), []
    want, m = am.adaptive_call(st, x, seqs, count, a, now, times, trace=trace)
    lag = int(after.view(np.int32)[0, 12])
    if trace and lag != st.view(np.int32)[0, 12]:
        assert len(trace) == 1 and near_tie(trace, lag), (trace[0][0], lag)
        st = before.copy()
        want, m = am.adaptive_call(st, x, seqs, count, a, now, times, force=[lag])
        stats["forced"] += 1
    stats["searches"] += len(trace)
    return want, m, st


def call_and_check(jb, a, x, seqs, counts, slots, now, times, stats):
    """one kernel call at `now` with arrival times `times` ([n, M] host ints, or None), checked against one model call
    per listed row from the kernel's state before it: out counts, every head, tag, ring and statistics word exactly"""
    p = a.p
    before = jb.state.cpu().numpy().copy()
    y, oc = jb(x, seqs, counts, slots, now=now, arrivals=times)
    after = jb.state.cpu().numpy()
    yk, ock = y.cpu().numpy(), oc.cpu().tolist()
    xs, sq = x.cpu().numpy(), seqs.cpu().numpy() if isinstance(seqs, torch.Tensor) else np.asarray(seqs)
    for i, s in enumerate(slots):
        row_times = None if times is None else times[i]
        want, m, st = model_row(before[s], after[s], xs[i], sq[i], counts[i], a, now, row_times, stats)
        kw, mw = after[s].view(np.int32), st.view(np.int32)
        assert ock[i] == m
        assert np.array_equal(kw[0, :p.o_ring], mw[0, :p.o_ring]), (i, kw[0, :16], mw[0, :16])
        assert np.array_equal(kw[:, p.o_ring:p.o_hist], mw[:, p.o_ring:p.o_hist])
        assert np.array_equal(kw[0, a.o_stats:], mw[0, a.o_stats:]), (i, kw[0, a.o_stats:], mw[0, a.o_stats:])
        peak = max(float(np.abs(before[s][:, p.o_hist:p.rf]).max()), float(np.abs(xs[i]).max(initial=0)), 1e-30)
        bound = BOUND_U * jm.U * peak
        assert float(np.abs(yk[i, :, :m * p.P].astype(np.float64) - want).max(initial=0)) <= bound
        assert np.abs(after[s][:, p.o_hist:p.rf].astype(np.float64) - st[:, p.o_hist:p.rf]).max() <= bound
    return y, oc


def traffic(n, seed, T, first=0):
    """arrival times of n packets with seeded gamma jitter, 3 % loss, an outage shorter than S and one longer"""
    g = np.random.default_rng(seed)
    out = {}
    for k in range(n):
        if g.random() < 0.03 or 40 <= k < 43 or 80 <= k < 95:
            continue
        out[(first + k) & 0xFFFF] = 1000 + k * T + 2000 + int(g.gamma(2.0, 3000.0 + 2000.0 * (seed % 3)))
    return out


@pytest.mark.parametrize("rate,P,C", CASES)
def test_matches_the_model(dev, rate, P, C):
    S, n, M = 6, 3, 4
    p = jm.Params(rate, P, C=C, D=1, W=16, max_out=4)
    a = am.Adapt(p, 2000, 40000, 0.1)
    jb = JitterBuffer(S, C, rate, P, depth=1, window=16, max_out=4, device=dev, deadline=(2000, 40000), late_rate=0.1)
    src = [jm.voiced(rate, 110.0 + 60 * i, 200 * P, i, C) for i in range(n)]
    T = tm.period(p)
    plans = [am.timed_plan(traffic(140, 31 + i, T, 65500 + 9 * i), t0=2 ** 31 - 300000) for i in range(n)]
    stats = {"forced": 0, "searches": 0}
    slots = [4, 1, 2]
    for t in range(min(len(pl) for pl in plans)):
        x = torch.zeros(n, C, M * P)
        seqs = torch.full((n, M), -1, dtype=torch.int32)
        times = [[0] * M for _ in range(n)]
        cnt = []
        for i in range(n):
            arr, at = plans[i][t][0][:M], plans[i][t][2][:M]
            cnt.append(len(arr))
            for j, s in enumerate(arr):
                seqs[i, j] = s
                times[i][j] = at[j] - (5000 if j == 1 and t % 5 == 0 else 0) + (9000 if j == 2 else 0)  # some after now
                x[i, :, j * P:(j + 1) * P] = torch.from_numpy(src[i][:, (s % 200) * P:(s % 200 + 1) * P])
        now = plans[0][t][1]
        call_and_check(jb, a, x.to(dev), seqs.to(dev), cnt, slots, now, None if t % 7 == 3 else times, stats)
    w = jb.state[:, 0].view(torch.int32).cpu()
    assert int(w[slots, tm.EXPIRED].min()) > 0 and int(w[slots, 10].min()) > 0     # deadline releases and restarts
    dl = jb.deadline_us.cpu()[slots]
    assert int(dl.max()) < 40000 and int(dl.min()) >= 2000 and stats["searches"] > 3
    print(stats, dl.tolist())


@pytest.mark.parametrize("rate,P,C", CASES)
def test_equal_bounds_are_the_timed_buffer(dev, rate, P, C):
    dl = 15000
    ad = JitterBuffer(3, C, rate, P, depth=1, window=16, max_out=3, device=dev, deadline=(dl, dl))
    timed = JitterBuffer(3, C, rate, P, depth=1, window=16, max_out=3, device=dev, deadline=dl)
    rf = timed.state.shape[2]
    assert ad.state.shape[2] == rf + am.STATS
    p = jm.Params(rate, P, C=C)
    plans = [tm.ticked(traffic(150, 50 + i, tm.period(p), 65500 + 3 * i), t0=2 ** 31 - 100000) for i in range(3)]
    g = torch.Generator().manual_seed(rate)
    for t in range(min(len(pl) for pl in plans)):
        arr = [plans[i][t][0][:3] for i in range(3)]
        cnt = [len(v) for v in arr]
        sq = su.i32([[*v, *[-1] * (3 - len(v))] for v in arr], dev)
        now = plans[0][t][1]
        x = torch.randn(3, C, 3 * P, generator=g).to(dev)
        times = None if t % 2 else [[now] * 3] * 3
        y1, o1 = ad(x, sq, cnt, [2, 0, 1], now=now, arrivals=times)
        y0, o0 = timed(x, sq, cnt, [2, 0, 1], now=now)
        assert torch.equal(o1, o0)
        for i in range(3):
            m = int(o0[i]) * P
            assert torch.equal(su.bits(y1[i, :, :m]), su.bits(y0[i, :, :m])), t
        assert torch.equal(su.bits(ad.state[:, :, :rf]), su.bits(timed.state)), t
    assert int(timed.expired.sum()) > 0 and int(timed.restarts.sum()) > 0
    assert (ad.deadline_us == dl).all()


def test_graph_replay_with_lists_clock_and_arrivals_rewritten(dev):
    C, P, S, n, M = 2, 441, 5, 3, 2
    kw = dict(device=dev, deadline=(3000, 40000), late_rate=0.1)
    live, twin = JitterBuffer(S, C, 44100, P, **kw), JitterBuffer(S, C, 44100, P, **kw)
    x = torch.zeros(n, C, M * P, device=dev)
    seqs = torch.full((n, M), -1, dtype=torch.int32, device=dev)
    counts, slots, now = su.i32([0] * n, dev), su.i32([0, 1, 2], dev), su.i32([0], dev)
    times = torch.zeros(n, M, dtype=torch.int32, device=dev)
    b = {"y": torch.empty(n, C, 4 * P, device=dev), "oc": torch.empty(n, dtype=torch.int32, device=dev)}
    graph = su.captured(lambda: live(x, seqs, counts, slots, out=b["y"], out_counts=b["oc"], now=now, arrivals=times))
    twin.state.copy_(live.state)
    g = torch.Generator().manual_seed(6)
    rng = np.random.default_rng(6)
    sched = [jm.schedule(200, 30 + i, loss=0.05, start=100 * i) for i in range(S)]
    for s in range(S):                               # outages, so that deadlines fire
        sched[s] = [v for v in sched[s] if not 60 <= (v - 100 * s) & 0xFFFF < 68 + s]
    pos = [0] * S
    clock = 2 ** 31 - 400000
    for t in range(200):
        clock += 8000
        sl = torch.randperm(S, generator=g)[:n].tolist()
        cnt = [min(int(v), len(sched[s]) - pos[s]) for v, s in zip(torch.randint(0, 3, (n,), generator=g), sl)]
        x.copy_(torch.randn(n, C, M * P, generator=g).to(dev))
        sq = [[*sched[s][pos[s]:pos[s] + c], *[-1] * (M - c)] for s, c in zip(sl, cnt)]
        for s, c in zip(sl, cnt):
            pos[s] += c
        at = [[clock - int(rng.integers(0, 30000)) for _ in range(M)] for _ in range(n)]
        seqs.copy_(su.i32(sq, dev))
        counts.copy_(su.i32(cnt, dev))
        slots.copy_(su.i32(sl, dev))
        now.fill_(tm.ser32(clock))
        times.copy_(su.i32([[tm.ser32(v) for v in r] for r in at], dev))
        su.refill(b)
        graph.replay()
        want = {"y": torch.full_like(b["y"], su.SENTINEL), "oc": torch.empty_like(b["oc"])}
        twin(x, su.i32(sq, dev), su.i32(cnt, dev), su.i32(sl, dev), out=want["y"], out_counts=want["oc"], now=clock,
             arrivals=at)
        su.assert_same(b, want, {"jb": live}, {"jb": twin}, t)
    measured = live.state[:, 0, -am.STATS + am.BINS].view(torch.int32)
    assert int(live.expired.sum()) > 0 and int(measured.min()) >= 10 and torch.equal(live.deadline_us, twin.deadline_us)


def test_rows_that_store_nothing(dev):
    C, P = 2, 160
    jb = JitterBuffer(4, C, 16000, P, device=dev, deadline=(2000, 10000), late_rate=0.5)
    x = torch.randn(3, C, 2 * P, device=dev)
    jb(x, [[0, 1], [0, 1], [0, 1]], [2, 2, 2], [0, 1, 2], now=0, arrivals=[[-500, -200]] * 3)
    before = jb.state.clone()
    y = torch.full((3, C, 4 * P), su.SENTINEL, device=dev)
    oc = torch.full((3,), 7, dtype=torch.int32, device=dev)
    # long past every deadline, but a slot outside the state, a count above M and a negative count: nothing happens
    jb(x, su.i32([[2, 3], [2, 3], [2, 3]], dev), su.i32([2, 3, -1], dev), su.i32([-1, 1, 2], dev), out=y,
       out_counts=oc, now=10 ** 6, arrivals=[[0, 0]] * 3)
    assert oc.tolist() == [0, 0, 0] and torch.isnan(y).all()
    assert torch.equal(su.bits(jb.state), su.bits(before))
    # a fresh slot listed with nothing to push starts nothing, and its statistics stay zero
    y, oc = jb(x[:1], [[-1, -1]], [0], [3], now=10 ** 6)
    assert int(oc[0]) == 0 and not torch.any(su.bits(jb.state[3])) and int(jb.deadline_us[3]) == 0
    # slot 0: one packet measured (-200 - (-500 + 10000)), k = 1 < 2, the deadline hi; listed alone, it expires S
    w = jb.state[0, 0, -am.STATS:].view(torch.int32).cpu()
    assert int(w[am.BINS]) == 1 and int(w[0]) == am.UNIT and int(w[am.BINS + 1]) == 10000
    y, oc = jb(x[:1], [[-1, -1]], [0], [0], now=10 ** 6)
    assert int(oc[0]) == 4 and int(jb.expired[0]) == tm.stall(jm.Params(16000, 160)) == int(jb.lost[0])


def mixed_plan(S, ticks, M, seed):
    """[ticks] lists per slot of (seq, arrival µs): packets every 10 ms; even slots 2 ms of uniform jitter, odd 30 ms"""
    rng = np.random.default_rng(seed)
    per_tick = [[[] for _ in range(S)] for _ in range(ticks)]
    for s in range(S):
        spread = 2000 if s % 2 == 0 else 30000
        for k in range(ticks * 8 // 10 + 4):
            t = 1000 + k * 10000 + 2000 + int(rng.integers(0, spread + 1))
            tick = -(-t // 8000)
            if tick < ticks:
                per_tick[tick][s].append(((k + 1000 * s) & 0xFFFF, t))
    for tick in per_tick:
        for lst in tick:
            lst.sort(key=lambda v: v[1])
            assert len(lst) <= M
    return per_tick


def test_mixed_links_on_one_state(dev):
    """half the slots on a 2 ms-jitter link, half on 30 ms, through jb -> PacketResampler -> HopFifo at 44.1 kHz: against
    a fixed 20 ms deadline the adaptive buffer drops fewer packets as late on the bad links, and keeps a lower deadline
    on the good ones (depth 8 on both, so the deadline rather than the reordering depth decides what is late)"""
    C, P, S, M, ticks = 2, 441, 8, 6, 900
    plan = mixed_plan(S, ticks, M, 12)
    sig = su.signals(S, C, 120 * P, 9951, dev)
    runs = {}
    for name, deadline in (("fixed", 20000), ("adaptive", (0, 60000))):
        jb = JitterBuffer(S, C, 44100, P, depth=8, window=16, max_out=6, device=dev, deadline=deadline)
        down = PacketResampler(44100, 16000, S, C, 6 * P, device=dev)
        fifo = HopFifo(S, C, 8, 4096, device=dev)
        dls = []
        for t in range(ticks):
            x = torch.zeros(S, C, M * P, device=dev)
            sq = [[-1] * M for _ in range(S)]
            at = [[0] * M for _ in range(S)]
            for s in range(S):
                for j, (q, a) in enumerate(plan[t][s]):
                    sq[s][j], at[s][j] = q, a
                    k = ((q - 1000 * s) & 0xFFFF) % 120
                    x[s, :, j * P:(j + 1) * P] = sig[s, :, k * P:(k + 1) * P]
            kw = {"arrivals": at} if name == "adaptive" else {}
            y, oc = jb(x, su.i32(sq, dev), [len(plan[t][s]) for s in range(S)], list(range(S)), now=8000 * t, **kw)
            y16, n16 = down(y, oc, list(range(S)), unit=P)
            fifo(y16, n16, list(range(S)))
            if name == "adaptive" and t >= ticks // 2:
                dls.append(jb.deadline_us.cpu())
        torch.cuda.synchronize()
        runs[name] = dict(late=jb.late.cpu(), expired=jb.expired.cpu(), lost=jb.lost.cpu(), dl=dls)
    good, bad = list(range(0, S, 2)), list(range(1, S, 2))
    fixed, ad = runs["fixed"], runs["adaptive"]
    dl = torch.stack(ad["dl"]).double()
    print({k: (v["late"].tolist(), v["expired"].tolist()) for k, v in runs.items()}, dl.mean(0).tolist())
    assert int(ad["late"][bad].sum()) < int(fixed["late"][bad].sum())
    assert float(dl[:, good].mean()) < 20000 and float(dl[:, good].mean()) < float(dl[:, bad].mean())
