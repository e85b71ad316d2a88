"""Packet streams on the GPU (l2h_resample_packets / PacketResampler, l2h_hop_fifo / HopFifo): ragged pushes of any length
against `resample` of each stream's whole input delayed by D, bit for bit, and against the float64 restatement
oracle/resample.py; whole-period pushes against StreamResampler; the FIFO's chunks, hop counts, draining and overflow
against the host model of test_packet_stream_cpu.py, every state row bit for bit; 48 kHz packets through the FIFO against
StreamResampler(keep=64); graph replays with the lists rewritten in place; and a tick of 44.1 kHz listeners sending 10 ms
packets, down -> FIFO -> separator -> up, against the same chain built from whole-signal resampling and the same hop
schedule."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_packet_stream_cpu as ps
from lookoncetohear_b200 import HopFifo, PacketResampler, StreamResampler, synth
from oracle import resample as ors
from serving_util import SENTINEL as NAN, bits, delayed, dev, i32, model, signals  # noqa: F401
from serving_util import assert_same, captured, refill

pytestmark = pytest.mark.gpu

RATES = [44100, 22050, 11025, 48000, 32000, 24000, 8000]
PAIRS = [(r, 16000) for r in RATES] + [(16000, r) for r in RATES]


@pytest.mark.parametrize("orig,new", PAIRS)
def test_ragged_pushes_match_whole_signal_resample(dev, orig, new):
    S, C, n, ticks, max_in = 5, 2, 4, 10, 1000
    pr = PacketResampler(orig, new, S, C, max_in, device=dev)
    o = orig // np.gcd(orig, new)
    lengths = [0, 1, 2, 3, 7, 13, 97, 251, o - 1, o + 1, 2 * o + 5, max_in]
    lengths = [m for m in lengths if 0 <= m <= max_in]
    sig = signals(S, C, max_in * ticks, 7 * orig + new, dev)
    g = torch.Generator().manual_seed(orig + 3 * new)
    fed, outs = [0] * S, [[] for _ in range(S)]
    for t in range(ticks):
        sl = torch.randperm(S, generator=g)[:n].tolist()
        sl[t % n] = -1 if t % 2 else S + t                      # one row per tick outside the state
        pushes = [lengths[int(k)] for k in torch.randint(0, len(lengths), (n,), generator=g)]
        x = torch.full((n, C, max_in), NAN, device=dev)         # samples past a row's push are never read
        for i, (s, m) in enumerate(zip(sl, pushes)):
            if 0 <= s < S:
                x[i, :, :m] = sig[s, :, fed[s]:fed[s] + m]
        y = torch.full((n, C, pr.max_out), NAN, device=dev)
        oc = torch.full((n,), -5, dtype=torch.int32, device=dev)
        r = pr(x, i32(pushes, dev), i32(sl, dev), out=y, out_counts=oc)
        assert r[0] is y and r[1] is oc
        oc = oc.tolist()
        for i, (s, m) in enumerate(zip(sl, pushes)):
            if not 0 <= s < S:
                assert oc[i] == 0 and torch.isnan(y[i]).all()
                continue
            want = (fed[s] + m) * new // orig - fed[s] * new // orig
            assert oc[i] == want, (t, i, s, m)
            assert torch.isnan(y[i, :, want:]).all(), "samples past the row's out count were written"
            outs[s].append(y[i, :, :want])
            fed[s] += m
    for s in range(S):
        N = fed[s]
        got = torch.cat(outs[s], -1)
        assert got.shape == (C, N * new // orig)
        if N == 0:
            continue
        ref = delayed(sig[s:s + 1, :, :N], orig, new, pr.delay, N * new // orig)[0]
        assert torch.equal(bits(got), bits(ref)), (s, (got != ref).sum().item())
        if got.shape[-1] > pr.delay:                          # and the float64 restatement, within 1e-5
            want = ors.resample(sig[s, :, :N].cpu().double().numpy(), orig, new)[:, :got.shape[-1] - pr.delay]
            assert np.linalg.norm(got[:, pr.delay:].cpu().double().numpy() - want) <= 1e-5 * np.linalg.norm(want)


@pytest.mark.parametrize("orig,new,block", [(44100, 16000, 441), (16000, 44100, 160), (48000, 16000, 384),
                                            (16000, 48000, 128), (11025, 16000, 441)])
def test_whole_periods_match_the_block_stream(dev, orig, new, block):
    """pushes of h blocks (counts = hops, unit = block) give StreamResampler's keep=0 outputs, bit for bit"""
    S, C, n, T = 6, 2, 4, 3
    pr = PacketResampler(orig, new, S, C, block * T, device=dev)
    rs = StreamResampler(orig, new, S, C, block, device=dev)
    assert pr.delay == rs.delay and pr.max_out == T * rs.out_block
    g = torch.Generator().manual_seed(block)
    for t in range(8):
        sl = i32(torch.randperm(S, generator=g)[:n].tolist(), dev)
        hops = i32(torch.randint(0, T + 1, (n,), generator=g).tolist(), dev)
        x = signals(n, C, block * T, 90 + t, dev)
        y, oc = pr(x, hops, sl, unit=block)
        want = rs(x, sl, hops)
        for i, h in enumerate(hops.tolist()):
            assert oc[i].item() == h * rs.out_block
            assert torch.equal(bits(y[i, :, :h * rs.out_block]), bits(want[i, :, :h * rs.out_block])), (t, i)


def test_fifo_chunks_hops_drain_and_overflow(dev):
    S, C, n, T, cap, L = 6, 2, 4, 1, 300, 300                   # one hop a call: backlogs build, drain and overflow
    fifo = HopFifo(S, C, T, cap, device=dev)
    assert fifo.state.shape == (S, C, 3 + 64 + cap) and not fifo.state.any()
    g = torch.Generator().manual_seed(606)
    held, dropped = [0] * S, [0] * S
    drained = overflowed = 0
    for t in range(60):
        sl = torch.randperm(S, generator=g)[:n].tolist()
        if t % 3 == 0:
            sl[t % n] = -2 if t % 2 else S
        counts = [[0, 0, 1, 17, 128, 160, 200, 300][int(k)] for k in torch.randint(0, 8, (n,), generator=g)]
        x = signals(n, C, L, 700 + t, dev)
        before = fifo.state.clone()
        chunk = torch.full((n, C, 128 * T + 64), NAN, device=dev)
        hops = torch.full((n,), -7, dtype=torch.int32, device=dev)
        r = fifo(x, i32(counts, dev), i32(sl, dev), out=chunk, hops=hops)
        assert r[0] is chunk and r[1] is hops
        hops = hops.tolist()
        for i, (s, m) in enumerate(zip(sl, counts)):
            if not 0 <= s < S:
                assert hops[i] == 0 and torch.isnan(chunk[i]).all()
                continue
            for c in range(C):                                  # the host model from the row before the call
                row = before[s, c].cpu().numpy().copy()
                want, h, head, writes = ps.fifo_push(row[:3].view(np.int32).tolist(), row[3:], x[i, c, :m].cpu().numpy(),
                                                     cap, T)
                assert hops[i] == h, (t, i, s)
                got = chunk[i, c].cpu().numpy()
                assert np.array_equal(got[:128 * h + 64].view(np.int32), np.array(want, np.float32).view(np.int32)), (t, i, s)
                assert np.isnan(got[128 * h + 64:]).all()
                row[:3] = np.array(head, np.int32).view(np.float32)
                for k, v in writes.items():
                    row[3 + k] = v
                assert np.array_equal(fifo.state[s, c].cpu().numpy().view(np.int32), row.view(np.int32)), (t, i, s, c)
            held[s] = head[1]
            dropped[s] = head[2]
            overflowed += head[2] > int(before[s, 0, 2].view(torch.int32))
            drained += m == 0 and h > 0
        assert fifo.held.tolist() == held and fifo.dropped.tolist() == dropped, t
        listed = {s for s in sl if 0 <= s < S}
        for s in set(range(S)) - listed:
            assert torch.equal(bits(fifo.state[s]), bits(before[s])), (t, s)
    assert drained and overflowed and sum(dropped) > 0
    fifo.reset([1, 4])
    assert not fifo.state[[1, 4]].any() and fifo.dropped[1] == 0


def test_48k_packets_through_the_fifo_are_the_keep_64_stream(dev):
    """48 kHz in 384-sample packets: PacketResampler -> HopFifo (T = 1) gives StreamResampler(keep=64)'s chunks"""
    S, C = 3, 2
    pr = PacketResampler(48000, 16000, S, C, 384, device=dev)
    fifo = HopFifo(S, C, 1, 512, device=dev)
    rs = StreamResampler(48000, 16000, S, C, 384, keep=64, device=dev)
    sig = signals(2, C, 384 * 12, 48, dev)
    sl = i32([2, 0], dev)
    for k in range(12):
        x = sig[:, :, 384 * k:384 * (k + 1)]
        y, oc = pr(x, i32([384, 384], dev), sl)
        chunk, hops = fifo(y, oc, sl)
        assert hops.tolist() == [1, 1]
        assert torch.equal(bits(chunk), bits(rs(x, sl))), k


def test_graph_replay_with_lists_rewritten_in_place(dev):
    """down 44.1 -> 16 kHz, FIFO, up 16 -> 44.1 kHz (unit 128) in one graph, against direct calls: bits and states"""
    S, C, n, T = 8, 2, 5, 2

    def chain():
        return {"down": PacketResampler(44100, 16000, S, C, 882, device=dev),
                "fifo": HopFifo(S, C, T, 1024, device=dev),
                "up": PacketResampler(16000, 44100, S, C, 128 * T, device=dev)}

    def bufs():
        return {"y16": torch.full((n, C, 320), NAN, device=dev), "oc": torch.zeros(n, dtype=torch.int32, device=dev),
                "chunk": torch.full((n, C, 128 * T + 64), NAN, device=dev),
                "hops": torch.zeros(n, dtype=torch.int32, device=dev),
                "y44": torch.full((n, C, 353 * T), NAN, device=dev), "oc44": torch.zeros(n, dtype=torch.int32, device=dev)}

    def tick(o, b, x, counts, slots):
        o["down"](x, counts, slots, out=b["y16"], out_counts=b["oc"])
        o["fifo"](b["y16"], b["oc"], slots, out=b["chunk"], hops=b["hops"])
        o["up"](b["chunk"][..., 64:], b["hops"], slots, unit=128, out=b["y44"], out_counts=b["oc44"])

    live, twin = chain(), chain()
    assert live["up"].max_out == 353 * T
    x = torch.zeros(n, C, 882, device=dev)
    counts, slots = i32([0] * n, dev), i32(list(range(n)), dev)
    b = bufs()
    graph = captured(lambda: tick(live, b, x, counts, slots))     # pushes of nothing: the states stay fresh
    g = torch.Generator().manual_seed(51)
    for t in range(10):
        sl = torch.randperm(S, generator=g)[:n].tolist()
        sl[t % n] = -1 if t % 2 else S
        cn = [[0, 1, 441, 882, 300][int(k)] for k in torch.randint(0, 5, (n,), generator=g)]
        x.copy_(signals(n, C, 882, 60 + t, dev))
        slots.copy_(i32(sl, dev))
        counts.copy_(i32(cn, dev))
        refill(b)
        graph.replay()
        want = bufs()
        tick(twin, want, x, i32(cn, dev), i32(sl, dev))
        assert_same(b, want, live, twin, t)


def test_python_call_checks(dev):
    pr = PacketResampler(44100, 16000, 4, 2, 882, device=dev)
    fifo = HopFifo(4, 2, 3, 1024, device=dev)
    x = torch.zeros(2, 2, 882, device=dev)
    for bad in ([0, 0], [0, 4], [-1, 0], [0]):
        with pytest.raises(ValueError):
            pr(x, [441, 441], bad)
        with pytest.raises(ValueError):
            fifo(x, [441, 441], bad)
    for bad in ([0, 883], [-1, 1], [1], [0.5, 1]):
        with pytest.raises(ValueError):
            pr(x, bad, [0, 1])
        with pytest.raises(ValueError):
            fifo(x, bad, [0, 1])
    with pytest.raises(ValueError):
        pr(x, [3, 1], [0, 1], unit=441)                             # 3 packets of 441 are past max_in
    with pytest.raises(ValueError):
        pr(x, [1, 1], [0, 1], unit=0)
    with pytest.raises(ValueError):
        pr(x, [0, 1], torch.tensor([0, 1], dtype=torch.int64, device=dev))   # CUDA lists are int32
    for shape in ((2, 2, 881), (2, 3, 882), (2, 2, 0)):
        with pytest.raises(ValueError):
            pr(torch.zeros(shape, device=dev), [0, 0], [0, 1])
    with pytest.raises(ValueError):
        fifo(torch.zeros(2, 3, 160, device=dev), [0, 0], [0, 1])
    with pytest.raises(ValueError):
        pr(x, [0, 0], [0, 1], out=torch.zeros(2, 2, 319, device=dev))
    with pytest.raises(ValueError):
        pr(x, [0, 0], [0, 1], out_counts=torch.zeros(2, dtype=torch.int64, device=dev))
    with pytest.raises(ValueError):
        fifo(x, [0, 0], [0, 1], out=torch.zeros(2, 2, 447, device=dev))
    with pytest.raises(ValueError):
        fifo(x, [0, 0], [0, 1], hops=torch.zeros(3, dtype=torch.int32, device=dev))
    with pytest.raises(RuntimeError, match="CUDA"):
        pr(x.cpu(), [0, 0], [0, 1])
    with pytest.raises(ValueError):
        pr.reset([4])
    assert not pr.state.any() and not fifo.state.any()


def test_44k_packets_through_the_separator(model, dev):
    """Three listeners at 44.1 kHz sending 10 ms packets with jitter (0-2 per 8 ms tick) and one at 16 kHz in 160-sample
    packets, on scattered slots of a seven-slot state, ~4 s with T = 3, per tick: down -> FIFO -> advance_slots(hops = the
    FIFO's CUDA hops) -> up(unit = 128).  Equals the chain on whole-signal resampling with the same hop schedule."""
    net, _ = model
    S, slots, T, ticks, cap = 7, [5, 1, 3, 6], 3, 500, 1024
    n = len(slots)
    g = torch.Generator().manual_seed(4400)
    packets = torch.multinomial(torch.tensor([0.3, 0.6, 0.1]), n * ticks, True, generator=g).view(ticks, n)
    total = packets.sum(0).tolist()
    size = [441, 441, 441, 160]
    x44, _ = synth.mixture(3, 441 * max(total[:3]), seed0=4500)
    x16, _ = synth.mixture(1, 160 * total[3], seed0=4600)
    x44, x16 = x44.to(dev), x16.to(dev)
    e = synth.embedding(n, seed0=4700)[:, 0].to(dev)
    down = PacketResampler(44100, 16000, S, 2, 882, device=dev)
    up = PacketResampler(16000, 44100, S, 2, 128 * T, device=dev)
    fifo = HopFifo(S, 2, T, cap, device=dev)
    st = net.init_buffers(S, dev)
    sl_d, sl_f = i32(slots[:3], dev), i32(slots, dev)
    xd = torch.zeros(3, 2, 882, device=dev)
    xf = torch.zeros(n, 2, down.max_out, device=dev)
    cnt_d, cnt_f = torch.zeros(3, dtype=torch.int32, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)
    fed = [0] * n
    hops_t, got44, got16 = [], [[] for _ in range(3)], []
    with torch.no_grad():
        for t in range(ticks):
            k = packets[t].tolist()
            for i in range(3):
                xd[i, :, :441 * k[i]] = x44[i, :, fed[i]:fed[i] + 441 * k[i]]
            xf[3, :, :160 * k[3]] = x16[0, :, fed[3]:fed[3] + 160 * k[3]]
            fed = [f + s * c for f, s, c in zip(fed, size, k)]
            cnt_d.copy_(i32([441 * c for c in k[:3]], dev))
            cnt_f[3:].copy_(i32([160 * k[3]], dev))
            down(xd, cnt_d, sl_d, out=xf[:3], out_counts=cnt_f[:3])
            chunk, hops = fifo(xf, cnt_f, sl_f)
            y16 = net.advance_slots(chunk, e, st, sl_f, hops=hops)
            y44, oc = up(y16[:3], hops[:3], sl_d, unit=128)
            hops_t.append(hops.clone())
            for i in range(3):
                got44[i].append((y44[i].clone(), oc[i].clone()))
            got16.append(y16[3].clone())
        hops_t = torch.stack(hops_t).tolist()                   # the hop schedule, read back for the check only
        # the FIFOs' signals from whole-signal resampling, and the separator fed the same schedule
        sig = [F.pad(delayed(x44[i:i + 1, :, :fed[i]], 44100, 16000, down.delay, fed[i] * 160 // 441)[0], (64, 0))
               for i in range(3)] + [F.pad(x16[0, :, :fed[3]], (64, 0))]
        st_ref = net.init_buffers(S, dev)
        pos, y_ref = [0] * n, [[] for _ in range(n)]
        for t in range(ticks):
            ch = torch.zeros(n, 2, 128 * T + 64, device=dev)
            for i, h in enumerate(hops_t[t]):
                ch[i, :, :128 * h + 64] = sig[i][:, pos[i]:pos[i] + 128 * h + 64]
                pos[i] += 128 * h
            y = net.advance_slots(ch, e, st_ref, sl_f, hops=i32(hops_t[t], dev))
            for i, h in enumerate(hops_t[t]):
                y_ref[i].append(y[i, :, :128 * h])
    for i in range(n):                                          # every hop the FIFO held was popped (T never binds)
        assert sum(h[i] for h in hops_t) == (sig[i].shape[-1] - 64) // 128
        assert fifo.held[slots[i]].item() == (sig[i].shape[-1] - 64) % 128
    assert fifo.dropped.sum().item() == 0
    y16_ref = [torch.cat(y, -1) for y in y_ref]
    got = torch.cat([y[:, :128 * h[3]] for y, h in zip(got16, hops_t)], -1)
    assert got.abs().max() > 0 and torch.equal(bits(got), bits(y16_ref[3]))
    for i in range(3):
        M = y16_ref[i].shape[-1]
        want = delayed(y16_ref[i][None], 16000, 44100, up.delay, M * 441 // 160)[0]
        got = torch.cat([y[:, :c.item()] for y, c in got44[i]], -1)
        assert got.shape == want.shape and want[:, up.delay:].abs().max() > 0
        assert torch.equal(bits(got), bits(want)), i
