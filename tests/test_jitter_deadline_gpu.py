"""The jitter buffer released on time on the GPU (JitterBuffer(deadline=...), l2h_jitter_buffer_timed), against the timed
model of tests/test_jitter_deadline_cpu.py, each call compared with one call of the model run from the kernel's own state
before it, with the bounds and the near-tie rule of tests/test_jitter_buffer_gpu.py.  Also: a deadline never reached
gives the untimed buffer bit for bit, graph replays with the lists and the clock rewritten in place, rows that store
nothing, and the 44.1 kHz chain jb -> PacketResampler -> HopFifo -> advance_slots through an outage."""
import numpy as np
import pytest
import torch

import serving_util as su
import test_jitter_buffer_cpu as jm
import test_jitter_deadline_cpu as tm
from lookoncetohear_b200 import HopFifo, JitterBuffer, PacketResampler
from serving_util import dev, model  # noqa: F401
from test_jitter_buffer_gpu import BOUND_U, CASES, near_tie

pytestmark = pytest.mark.gpu


def model_row(before, after, x, seqs, count, p, now, deadline, stats):
    """one timed model call from the kernel's state `before` [C, rf] of a slot: (y, out count, the model's state after);
    run again at the kernel's lag (in `after`) where the two lie within the fp32 error of their scores"""
    st, trace = before.copy(), []
    want, m = tm.timed_call(st, x, seqs, count, p, now, deadline, trace=trace)
    lag = int(after.view(np.int32)[0, 12])
    if trace and lag != st.view(np.int32)[0, 12]:
        assert len(trace) == 1 and near_tie(trace, lag), (trace[0][0], lag)
        st = before.copy()
        want, m = tm.timed_call(st, x, seqs, count, p, now, deadline, force=[lag])
        stats["forced"] += 1
    stats["searches"] += len(trace)
    return want, m, st


def call_and_check(jb, p, x, seqs, counts, slots, now, stats):
    """one kernel call at `now`, checked against one model call per listed row from the kernel's state before it"""
    before = jb.state.cpu().numpy().copy()
    y, oc = jb(x, seqs, counts, slots, now=now)
    after = jb.state.cpu().numpy()
    yk, ock = y.cpu().numpy(), oc.cpu().tolist()
    xs, sq = x.cpu().numpy(), seqs.cpu().numpy() if isinstance(seqs, torch.Tensor) else np.asarray(seqs)
    for i, s in enumerate(slots):
        want, m, st = model_row(before[s], after[s], xs[i], sq[i], counts[i], p, now, jb.deadline, stats)
        kw, mw = after[s].view(np.int32), st.view(np.int32)
        assert ock[i] == m
        assert np.array_equal(kw[0, :p.o_ring], mw[0, :p.o_ring]), (i, kw[0, :16], mw[0, :16])
        assert np.array_equal(after[s][:, p.o_ring:p.o_hist].view(np.int32), st[:, p.o_ring:p.o_hist].view(np.int32))
        peak = max(float(np.abs(before[s][:, p.o_hist:]).max()), float(np.abs(xs[i]).max(initial=0)), 1e-30)
        bound = BOUND_U * jm.U * peak
        assert float(np.abs(yk[i, :, :m * p.P].astype(np.float64) - want).max(initial=0)) <= bound
        assert np.abs(after[s][:, p.o_hist:].astype(np.float64) - st[:, p.o_hist:]).max() <= bound
    return y, oc


def traffic(n, seed, P=10000, first=0):
    """arrival times of n packets with seeded jitter, 5 % loss, an outage shorter than S and one longer"""
    g = np.random.default_rng(seed)
    out = {}
    for k in range(n):
        if g.random() < 0.05 or 20 <= k < 24 or 45 <= k < 60:
            continue
        out[(first + k) & 0xFFFF] = 1000 + k * P + 2000 + int(g.integers(0, 14000))
    return out


@pytest.mark.parametrize("rate,P,C", CASES)
def test_matches_the_model(dev, rate, P, C):
    S, n, dl = 6, 3, 15000
    p = jm.Params(rate, P, C=C, D=1, W=16, max_out=4)
    jb = JitterBuffer(S, C, rate, P, depth=1, window=16, max_out=4, device=dev, deadline=dl)
    src = [jm.voiced(rate, 110.0 + 60 * i, 200 * P, i, C) for i in range(n)]
    T = tm.period(p)
    plans = [tm.ticked(traffic(80, 31 + i, T, 65500 + 9 * i), t0=2 ** 31 - 300000) for i in range(n)]
    stats = {"forced": 0, "searches": 0}
    slots = [4, 1, 2]
    for t in range(min(len(pl) for pl in plans)):
        x = torch.zeros(n, C, 3 * P)
        seqs = torch.full((n, 3), -1, dtype=torch.int32)
        cnt = []
        for i in range(n):
            arr = plans[i][t][0][:3]
            cnt.append(len(arr))
            for j, s in enumerate(arr):
                seqs[i, j] = s
                x[i, :, j * P:(j + 1) * P] = torch.from_numpy(src[i][:, (s % 200) * P:(s % 200 + 1) * P])
        now = plans[0][t][1]                         # one clock for the call: the rows' plans share the tick
        call_and_check(jb, p, x.to(dev), seqs.to(dev), cnt, slots, now, stats)
    w = jb.state[:, 0].view(torch.int32).cpu()
    assert int(w[slots, tm.EXPIRED].min()) > 0 and int(w[slots, 10].min()) > 0     # deadline releases and restarts
    assert stats["searches"] > 3
    print(stats)


@pytest.mark.parametrize("rate,P,C", CASES)
def test_unreached_deadline_is_the_untimed_buffer(dev, rate, P, C):
    timed = JitterBuffer(3, C, rate, P, depth=1, window=16, max_out=3, device=dev, deadline=2 ** 31 - 1)
    plain = JitterBuffer(3, C, rate, P, depth=1, window=16, max_out=3, device=dev)
    g = torch.Generator().manual_seed(rate)
    sched = [jm.schedule(120, 50 + i, loss=0.15, swap=0.1, dup=0.05, start=65500 + 3 * i) for i in range(3)]
    pos = [0] * 3
    for t in range(90):
        cnt = [min(int(v), len(sched[i]) - pos[i]) for i, v in enumerate(torch.randint(0, 4, (3,), generator=g))]
        sq = [[*sched[i][pos[i]:pos[i] + cnt[i]], *[-1] * (3 - cnt[i])] for i in range(3)]
        for i in range(3):
            pos[i] += cnt[i]
        x = torch.randn(3, C, 3 * P, generator=g).to(dev)
        y1, o1 = timed(x, su.i32(sq, dev), cnt, [2, 0, 1], now=2 ** 31 - 100000 + 8000 * t)   # wraps past 2^31
        y0, o0 = plain(x, su.i32(sq, dev), cnt, [2, 0, 1])
        assert torch.equal(o1, o0)
        for i in range(3):
            m = int(o0[i]) * P
            assert torch.equal(su.bits(y1[i, :, :m]), su.bits(y0[i, :, :m])), t
        a, b = su.bits(timed.state), su.bits(plain.state)
        assert torch.equal(a[:, 0, :13], b[:, 0, :13]) and torch.equal(a[:, :, 16:], b[:, :, 16:]), t
    assert int(timed.expired.sum()) == 0 and int(timed.lost.sum()) > 0


def test_graph_replay_with_lists_and_clock_rewritten(dev):
    C, P, S, n = 2, 441, 5, 3
    live = JitterBuffer(S, C, 44100, P, device=dev, deadline=15000)
    twin = JitterBuffer(S, C, 44100, P, device=dev, deadline=15000)
    x = torch.zeros(n, C, 2 * P, device=dev)
    seqs = torch.full((n, 2), -1, dtype=torch.int32, device=dev)
    counts, slots, now = su.i32([0] * n, dev), su.i32([0, 1, 2], dev), su.i32([0], dev)
    b = {"y": torch.empty(n, C, 4 * P, device=dev), "oc": torch.empty(n, dtype=torch.int32, device=dev)}
    graph = su.captured(lambda: live(x, seqs, counts, slots, out=b["y"], out_counts=b["oc"], now=now))
    twin.state.copy_(live.state)
    g = torch.Generator().manual_seed(6)
    sched = [jm.schedule(80, 30 + i, loss=0.1, start=100 * i) for i in range(S)]
    for s in range(S):                               # outages, so that deadlines fire
        sched[s] = [v for v in sched[s] if not 30 <= (v - 100 * s) & 0xFFFF < 38 + s]
    pos = [0] * S
    for t in range(60):
        sl = torch.randperm(S, generator=g)[:n].tolist()
        cnt = [min(int(v), len(sched[s]) - pos[s]) for v, s in zip(torch.randint(0, 3, (n,), generator=g), sl)]
        x.copy_(torch.randn(n, C, 2 * P, generator=g).to(dev))
        sq = [[*sched[s][pos[s]:pos[s] + c], *[-1] * (2 - c)] for s, c in zip(sl, cnt)]
        for s, c in zip(sl, cnt):
            pos[s] += c
        seqs.copy_(su.i32(sq, dev))
        counts.copy_(su.i32(cnt, dev))
        slots.copy_(su.i32(sl, dev))
        now.fill_(-2 ** 31 + 40000 + 8000 * t if t % 7 else 2 ** 31 - 4000)   # the clock jumps and wraps
        su.refill(b)
        graph.replay()
        want = {"y": torch.full_like(b["y"], su.SENTINEL), "oc": torch.empty_like(b["oc"])}
        twin(x, su.i32(sq, dev), su.i32(cnt, dev), su.i32(sl, dev), out=want["y"], out_counts=want["oc"],
             now=int(now.item()))
        su.assert_same(b, want, {"jb": live}, {"jb": twin}, t)
    assert int(live.expired.sum()) > 0


def test_rows_that_store_nothing(dev):
    C, P = 2, 160
    jb = JitterBuffer(4, C, 16000, P, device=dev, deadline=10000)
    x = torch.randn(3, C, 2 * P, device=dev)
    jb(x, [[0, 1], [0, 1], [0, 1]], [2, 2, 2], [0, 1, 2], now=0)
    before = jb.state.clone()
    y = torch.full((3, C, 4 * P), su.SENTINEL, device=dev)
    oc = torch.full((3,), 7, dtype=torch.int32, device=dev)
    # long past every deadline, but a slot outside the state, a count above M and a negative count: nothing happens
    jb(x, su.i32([[2, 3], [2, 3], [2, 3]], dev), su.i32([2, 3, -1], dev), su.i32([-1, 1, 2], dev), out=y,
       out_counts=oc, now=10 ** 6)
    assert oc.tolist() == [0, 0, 0] and torch.isnan(y).all()
    assert torch.equal(su.bits(jb.state), su.bits(before))
    # a fresh slot listed with nothing to push starts nothing
    y, oc = jb(x[:1], [[-1, -1]], [0], [3], now=10 ** 6)
    assert int(oc[0]) == 0 and not torch.any(su.bits(jb.state[3]))
    # slot 0 listed alone with count 0: its deadlines fire, up to S packets
    y, oc = jb(x[:1], [[-1, -1]], [0], [0], now=10 ** 6)
    assert int(oc[0]) == 4 and int(jb.expired[0]) == tm.stall(jm.Params(16000, 160)) == int(jb.lost[0])


def test_chain_at_44k_through_an_outage(dev, model):
    """timed jb -> PacketResampler -> HopFifo -> advance_slots at 44.1 kHz, one 8 ms tick per call, through a 60 ms
    outage: the hop counts keep pace with the clock during the gap, and no tick after it catches up more than the hops
    of one tick's packets, where the untimed buffer on the same calls falls behind and then bursts"""
    net, _ = model
    C, P, S, n, T = 2, 441, 4, 3, 8
    e = su.emb(n, 9940, dev)
    runs = {}
    for name, deadline in (("timed", 15000), ("plain", None)):
        jb = JitterBuffer(S, C, 44100, P, depth=1, window=16, max_out=6, device=dev, deadline=deadline)
        down = PacketResampler(44100, 16000, S, C, 6 * P, device=dev)
        fifo, st = HopFifo(S, C, T, 4096, device=dev), net.init_buffers(S, dev)
        plans = [tm.ticked(tm.stream(60, 10000, gone=set(range(20, 26)), first=100 * i)) for i in range(n)]
        sig = su.signals(n, C, 60 * P, 9950, dev)
        hops = []
        for t in range(len(plans[0])):
            arr = [plans[i][t][0][:3] for i in range(n)]
            x = torch.zeros(n, C, 3 * P, device=dev)
            for i in range(n):
                for j, s in enumerate(arr[i]):
                    k = (s - 100 * i) & 0xFFFF
                    x[i, :, j * P:(j + 1) * P] = sig[i, :, k * P:(k + 1) * P]
            sq = su.i32([[*a, *[-1] * (3 - len(a))] for a in arr], dev)
            kw = {} if deadline is None else {"now": plans[0][t][1]}
            y, oc = jb(x, sq, [len(a) for a in arr], [0, 1, 2], **kw)
            y16, n16 = down(y, oc, [0, 1, 2], unit=P)
            chunk, h = fifo(y16, n16, [0, 1, 2])
            net.advance_slots(chunk, e, st, [0, 1, 2], hops=h)
            hops.append(h.cpu())
        runs[name] = torch.stack(hops)                # [ticks, n]
    torch.cuda.synchronize()
    # the gap: packets 20 .. 25 would have arrived from 204 ms to 254 ms; packet 20 expires at 225 ms (the tick at 232)
    gap = [t for t in range(len(runs["timed"])) if 232000 <= t * tm.TICK <= 256000]
    cum = runs["timed"].cumsum(0)
    for t in range(len(cum)):                        # 16 kHz hops due by the clock: 160 per 10 ms packet sent
        due = max(0, (t * tm.TICK - 4000) // 10000 + 1) * 160 // 128
        assert (cum[t] <= due + 1).all() and (cum[t] >= due - 5).all(), (t, cum[t].tolist(), due)
    assert (runs["timed"][gap].sum(0) >= len(gap) - 1).all() and (runs["plain"][gap].sum(0) <= 1).all()
    assert int(runs["timed"].max()) <= 3 < int(runs["plain"].max())
