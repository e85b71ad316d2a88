"""The jitter buffer on the GPU (JitterBuffer, l2h_jitter_buffer), against the model of tests/test_jitter_buffer_cpu.py.

Each call is compared with one call of the model run from the kernel's own state before it, so errors cannot compound:
the out counts, the head words, the ring tags and the ring exactly; the samples and the history to BOUND_U fp32 units of
the call's peak (a concealed sample is a gain or a fade weight times stored samples: a few roundings each).  Where the
model's best lag and the kernel's lie within the fp32 error of their scores, the model is run again at the kernel's lag.
Also: bit-for-bit results across cuts and max_out and on a perfect network, graph replays with lists rewritten in place,
rows that store nothing, non-finite input, and the 44.1 kHz chain jb -> PacketResampler -> HopFifo -> advance_slots."""
import numpy as np
import pytest
import torch

import serving_util as su
import test_jitter_buffer_cpu as jm
from lookoncetohear_b200 import HopFifo, JitterBuffer, PacketResampler
from serving_util import dev, model  # noqa: F401

pytestmark = pytest.mark.gpu

BOUND_U = 16                                          # fp32 units of the call's peak
CASES = [(16000, 160, 1), (44100, 441, 2), (48000, 480, 2)]


def near_tie(trace, lag):
    """every search of the trace picks a lag whose score lies within the fp32 error of `lag`'s"""
    return all(lag in sc and sc[lag] > 0 and sc[best] - sc[lag] <= bd[best] + bd[lag] for best, sc, bd in trace)


def model_row(before, after, x, seqs, count, p, stats):
    """one model call from the kernel's state `before` [C, rf] of a slot: (y, out count, the model's state after); run
    again at the kernel's lag (in `after`) where the two lie within the fp32 error of their scores"""
    st, trace = before.copy(), []
    want, m = jm.model_call(st, x, seqs, count, p, trace=trace)
    lag = int(after.view(np.int32)[0, 12])
    if trace and lag != st.view(np.int32)[0, 12]:
        assert len(trace) == 1 and near_tie(trace, lag), (trace[0][0], lag)
        st = before.copy()
        want, m = jm.model_call(st, x, seqs, count, p, force=[lag])
        stats["forced"] += 1
    stats["searches"] += len(trace)
    return want, m, st


def call_and_check(jb, p, x, seqs, counts, slots, stats):
    """one kernel call, checked against one model call per listed row from the kernel's state before it"""
    before = jb.state.cpu().numpy().copy()
    y, oc = jb(x, seqs, counts, slots)
    after = jb.state.cpu().numpy()
    yk, ock = y.cpu().numpy(), oc.cpu().tolist()
    xs, sq = x.cpu().numpy(), seqs.cpu().numpy() if isinstance(seqs, torch.Tensor) else np.asarray(seqs)
    for i, s in enumerate(slots):
        want, m, st = model_row(before[s], after[s], xs[i], sq[i], counts[i], p, stats)
        kw, mw = after[s].view(np.int32), st.view(np.int32)
        assert ock[i] == m
        assert np.array_equal(kw[0, :p.o_ring], mw[0, :p.o_ring]), (i, kw[0, :13], mw[0, :13])
        assert np.array_equal(after[s][:, p.o_ring:p.o_hist].view(np.int32), st[:, p.o_ring:p.o_hist].view(np.int32))
        peak = max(float(np.abs(before[s][:, p.o_hist:]).max()), float(np.abs(xs[i]).max(initial=0)), 1e-30)
        bound = BOUND_U * jm.U * peak
        err = float(np.abs(yk[i, :, :m * p.P].astype(np.float64) - want).max(initial=0))
        assert err <= bound
        assert np.abs(after[s][:, p.o_hist:].astype(np.float64) - st[:, p.o_hist:]).max() <= bound
        stats["worst"] = max(stats["worst"], err / bound)
    return y, oc


def arrivals(n, seed, loss, start):
    """a seeded schedule with losses, a burst longer than 60 ms, swaps within and beyond depth, duplicates and a restart"""
    seq = jm.schedule(n, seed, loss=loss, swap=0.08, dup=0.05, start=start)
    k = len(seq) // 3
    seq = seq[:k] + [s for s in seq[k:] if not 2 <= (s - seq[k]) & 0xFFFF <= 9]       # an 8-packet burst
    j = 2 * len(seq) // 3
    seq[j:j] = [seq[j - 6]]                                                               # late beyond depth
    seq += [(seq[-1] + 5000 + i) & 0xFFFF for i in range(6)]                              # a restart
    return seq


@pytest.mark.parametrize("rate,P,C", CASES)
@pytest.mark.parametrize("loss", [0.05, 0.2])
def test_matches_the_model(dev, rate, P, C, loss):
    S, n, D = 6, 3, 1
    p = jm.Params(rate, P, C=C, D=D, W=16, max_out=4)
    jb = JitterBuffer(S, C, rate, P, depth=D, window=16, max_out=4, device=dev)
    g = torch.Generator().manual_seed(int(rate + 100 * loss))
    sched = [arrivals(90, 10 * i + int(100 * loss), loss, 65480 + 7 * i) for i in range(n)]
    src = [jm.voiced(rate, 110.0 + 60 * i, 200 * P, i, C) for i in range(n)]
    pos, stats = [0] * n, {"forced": 0, "searches": 0, "worst": 0.0}
    slots = [4, 1, 2]
    for t in range(60):
        cnt = [int(v) for v in torch.randint(0, 3, (n,), generator=g)]
        x = torch.zeros(n, C, 2 * P)
        seqs = torch.full((n, 2), -1, dtype=torch.int32)
        for i in range(n):
            cnt[i] = min(cnt[i], len(sched[i]) - pos[i])
            for j in range(cnt[i]):
                s = sched[i][pos[i] + j]
                seqs[i, j] = s
                x[i, :, j * P:(j + 1) * P] = torch.from_numpy(src[i][:, (s % 200) * P:(s % 200 + 1) * P])
            pos[i] += cnt[i]
        call_and_check(jb, p, x.to(dev), seqs.to(dev), cnt, slots, stats)
    assert stats["searches"] > 3
    print(stats)


@pytest.mark.parametrize("rate,P,C", CASES)
def test_cuts_max_out_and_perfect_network_bit_for_bit(dev, rate, P, C):
    pk = [(0.3 * torch.randn(C, P, generator=torch.Generator().manual_seed(k))) for k in range(64)]
    sched = jm.schedule(100, 3, loss=0.1, swap=0.1, dup=0.05, start=65530)
    perfect = list(range(65500, 65536)) + list(range(0, 40))

    def run(arr, mo, cuts):
        jb = JitterBuffer(2, C, rate, P, depth=1, window=16, max_out=mo, device=dev)
        out, a = [], 0
        for c in cuts + [0] * 40:
            x = torch.zeros(1, C, 4 * P)
            for j, s in enumerate(arr[a:a + c]):
                x[0, :, j * P:(j + 1) * P] = pk[s % 64]
            seqs = su.i32([[*arr[a:a + c], *[-1] * (4 - c)]], dev)
            y, oc = jb(x.to(dev), seqs, su.i32([c], dev), su.i32([1], dev))
            out.append(y[0, :, :int(oc[0]) * P].cpu())
            a += c
        return torch.cat(out, 1), jb.state[1].cpu()

    for arr in (sched, perfect):
        want, st = run(arr, 4, [1] * len(arr))
        for seed, mo, hi in ((1, 2, 1), (2, 4, 3), (3, 5, 4)):
            got, st2 = run(arr, mo, jm.random_cuts(len(arr), seed, hi))
            assert torch.equal(su.bits(got), su.bits(want)), (seed, mo)
            w, w2 = su.bits(st)[0], su.bits(st2)[0]
            assert torch.equal(w[6:11], w2[6:11])
    got, _ = run(perfect, 4, jm.random_cuts(len(perfect), 9, 4))
    assert torch.equal(su.bits(got), su.bits(torch.cat([pk[s % 64] for s in perfect], 1)))


@pytest.mark.parametrize("max_out", [1, 2, 8])
def test_a_restart_keeps_the_decided_backlog(dev, max_out):
    """a restart while released packets wait unwritten (the schedule of tests/test_jitter_buffer_cpu.py): every
    max_out gives the model's output at max_out 16, bit for bit on the packets that are copied, within the bound on
    the restart's fade"""
    p, pk, want, st = jm.restart_behind_a_backlog(16, C=2)
    jb = JitterBuffer(1, 2, 16000, 160, depth=8, window=16, max_out=max_out, device=dev)
    out, a = [], 0
    for c in jm.RESTART_CUTS + [0] * 8:
        arr = jm.RESTART_ARRIVALS[a:a + c]
        x = torch.zeros(1, 2, 7 * 160)
        for j, s in enumerate(arr):
            x[0, :, j * 160:(j + 1) * 160] = torch.from_numpy(pk[s % 16])
        seqs = su.i32([[*arr, *[-1] * (7 - c)]], dev)
        y, oc = jb(x.to(dev), seqs, su.i32([c], dev), su.i32([0], dev))
        out.append(y[0, :, :int(oc[0]) * 160].cpu().numpy())
        a += c
    got = np.concatenate(out, 1)
    assert got.shape == want.shape
    assert np.array_equal(got[:, :7 * 160].view(np.int32), want[:, :7 * 160].view(np.int32))
    assert np.abs(got.astype(np.float64) - want).max() <= BOUND_U * jm.U * float(np.abs(want).max())
    w = jb.state[0, 0].view(torch.int32).cpu().numpy()
    assert np.array_equal(w[6:11], st.view(np.int32)[0, 6:11])


def test_graph_replay_with_lists_rewritten(dev):
    C, P, S, n = 2, 441, 5, 3
    live = JitterBuffer(S, C, 44100, P, device=dev)
    twin = JitterBuffer(S, C, 44100, P, device=dev)
    x = torch.zeros(n, C, 2 * P, device=dev)
    seqs = torch.full((n, 2), -1, dtype=torch.int32, device=dev)
    counts, slots = su.i32([0] * n, dev), su.i32([0, 1, 2], dev)
    b = {"y": torch.empty(n, C, 4 * P, device=dev), "oc": torch.empty(n, dtype=torch.int32, device=dev)}
    graph = su.captured(lambda: live(x, seqs, counts, slots, out=b["y"], out_counts=b["oc"]))
    twin.state.copy_(live.state)
    g = torch.Generator().manual_seed(5)
    sched = [jm.schedule(80, 20 + i, loss=0.1, start=100 * i) for i in range(S)]
    pos = [0] * S
    for t in range(40):
        sl = torch.randperm(S, generator=g)[:n].tolist()
        cnt = [min(int(v), len(sched[s]) - pos[s]) for v, s in zip(torch.randint(0, 3, (n,), generator=g), sl)]
        x.copy_(torch.randn(n, C, 2 * P, generator=g).to(dev))
        sq = [[*sched[s][pos[s]:pos[s] + c], *[-1] * (2 - c)] for s, c in zip(sl, cnt)]
        for s, c in zip(sl, cnt):
            pos[s] += c
        seqs.copy_(su.i32(sq, dev))
        counts.copy_(su.i32(cnt, dev))
        slots.copy_(su.i32(sl, dev))
        su.refill(b)
        graph.replay()
        want = {"y": torch.full_like(b["y"], su.SENTINEL), "oc": torch.empty_like(b["oc"])}
        twin(x, su.i32(sq, dev), su.i32(cnt, dev), su.i32(sl, dev), out=want["y"], out_counts=want["oc"])
        su.assert_same(b, want, {"jb": live}, {"jb": twin}, t)


def test_rows_that_store_nothing_and_bad_input(dev):
    C, P = 2, 160
    jb = JitterBuffer(4, C, 16000, P, device=dev)
    x = torch.randn(3, C, 2 * P, device=dev)
    x[0, 0, 5], x[0, 1, 7], x[0, 0, 200] = float("nan"), float("inf"), 2.0 ** 40
    jb(x, [[0, 1], [0, 1], [0, 1]], [2, 2, 2], [0, 1, 2])
    before = jb.state.clone()
    y = torch.full((3, C, 4 * P), su.SENTINEL, device=dev)
    oc = torch.full((3,), 7, dtype=torch.int32, device=dev)
    # a slot outside the state, a count above M and a negative count: nothing stored, out count 0
    jb(x, su.i32([[2, 3], [2, 3], [2, 3]], dev), su.i32([2, 3, -1], dev), su.i32([-1, 1, 2], dev), out=y, out_counts=oc)
    assert oc.tolist() == [0, 0, 0] and torch.isnan(y).all()
    assert torch.equal(su.bits(jb.state), su.bits(before))
    y, oc = jb(x[:1], su.i32([[5, 70000]], dev), [2], [0])   # 70000 is skipped; 5 declares 2 and 3 lost (depth 1)
    assert int(oc[0]) == 2 and int(jb.lost[0]) == 2
    # the non-finite and huge samples entered as 0
    jb2 = JitterBuffer(1, C, 16000, P, device=dev)
    y, oc = jb2(x[:1], [[0, 1]], [2], [0])
    ref = x[0].clone()
    ref[0, 5] = ref[1, 7] = ref[0, 200] = 0.0
    assert torch.equal(y[0, :, :2 * P], ref)


def test_chain_at_44k_with_loss(dev, model):
    """jb -> PacketResampler -> HopFifo -> advance_slots at 44.1 kHz with 5 % loss: the hop counts equal, and the chunks
    lie within the model's sample bound carried through the resampler (sum |taps| < 2), of the model's jb output sent
    through the same unchanged stages"""
    net, _ = model
    C, P, S, n, T = 2, 441, 4, 3, 2
    x16, _ = su.clips(n, 40, 9920, dev)
    x44 = su.resample(x16[..., :su.HOP * 40].reshape(n * C, -1), 16000, 44100).reshape(n, C, -1).contiguous().cpu()
    e = su.emb(n, 9930, dev)
    p = jm.Params(44100, P, C=C, W=16, max_out=4)
    stages = [(JitterBuffer(S, C, 44100, P, device=dev), PacketResampler(44100, 16000, S, C, 4 * P, device=dev),
               HopFifo(S, C, T, 4096, device=dev), net.init_buffers(S, dev)) for _ in range(2)]
    sched = [jm.schedule(32, 40 + i, loss=0.05, swap=0.05, dup=0.0) for i in range(n)]   # the 32 packets of x44
    g = torch.Generator().manual_seed(7)
    pos, slots, stats = [0] * n, [0, 1, 2], {"forced": 0, "searches": 0}
    for t in range(60):
        cnt = [min(int(v), len(sched[i]) - pos[i]) for i, v in enumerate(torch.randint(0, 3, (n,), generator=g))]
        x = torch.zeros(n, C, 2 * P)
        sq = [[*sched[i][pos[i]:pos[i] + cnt[i]], *[-1] * (2 - cnt[i])] for i in range(n)]
        for i in range(n):
            for j, s in enumerate(sq[i][:cnt[i]]):
                x[i, :, j * P:(j + 1) * P] = x44[i, :, s * P:(s + 1) * P]
            pos[i] += cnt[i]
        jb, down, fifo, st = stages[0]
        before = jb.state.cpu().numpy().copy()
        y, oc = jb(x.to(dev), su.i32(sq, dev), cnt, slots)
        after = jb.state.cpu().numpy()
        y16, n16 = down(y, oc, slots, unit=P)
        chunk, hops = fifo(y16, n16, slots)
        net.advance_slots(chunk, e, st, slots, hops=hops)
        ym = torch.zeros(n, C, 4 * P)
        ocm, peak = [], 1e-30
        for i in range(n):
            peak = max(peak, float(np.abs(before[i][:, p.o_hist:]).max()), float(x[i].abs().max()))
            yi, m, _ = model_row(before[i], after[i], x[i].numpy(), sq[i], cnt[i], p, stats)
            ym[i, :, :m * P] = torch.from_numpy(yi)
            ocm.append(m)
        _, down2, fifo2, st2 = stages[1]
        y16m, n16m = down2(ym.to(dev), su.i32(ocm, dev), slots, unit=P)
        chunk_m, hops_m = fifo2(y16m, n16m, slots)
        net.advance_slots(chunk_m, e, st2, slots, hops=hops_m)
        assert oc.tolist() == ocm and torch.equal(hops, hops_m)
        for i in range(n):
            h = int(hops[i])
            d = (chunk[i, :, :su.HOP * h + su.LA] - chunk_m[i, :, :su.HOP * h + su.LA]).abs().max()
            assert float(d) <= 2 * BOUND_U * 4 * jm.U * peak
    torch.cuda.synchronize()
