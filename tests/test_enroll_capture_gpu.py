"""Enrollment from a listener's own stream on the GPU (l2h_enroll_capture / EnrollCapture, l2h_embed_forward_slots /
EmbedTFGridNet.enroll): the capture's rings against what was pushed, bit for bit, across many wraps, 0-hop rows and rows on
outside slots; the same ticks replayed from a CUDA graph (FIFO -> capture) with the lists rewritten in place; enrollment
from the rings against EmbedTFGridNet.forward(x, lengths) of the same windows gathered by torch, bit for bit, and against
the oracle; and a listener re-enrolled mid-stream through FIFO -> capture -> advance_slots."""
import pytest
import torch

from lookoncetohear_b200 import EmbedTFGridNet, EnrollCapture, HopFifo, synth
from oracle import restate as rs
from serving_util import assert_same, bits, captured, dev, i32, model  # noqa: F401

pytestmark = pytest.mark.gpu

HEAD, HOP, CARRY = 2, 128, 64
NAN = float("nan")


def ring_last(cap, s, L):
    """[C, L] the last L samples slot s of an EnrollCapture holds, read through its head"""
    w = int(cap.state[s, 0, 0].view(torch.int32))
    idx = (w - L + torch.arange(L, device=cap.state.device)) % cap.capacity
    return cap.state[s][:, HEAD + idx]


@pytest.fixture(scope="module")
def embed(embed_params, dev):
    torch.manual_seed(0)
    net = EmbedTFGridNet(**embed_params).eval()
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    return net.to(dev), sd


def test_capture_is_exact(dev):
    """a few hundred ticks of per-row hops in [0, T], one row per tick on an outside slot, a ring that wraps many times"""
    S, C, n, T, capacity, ticks = 7, 2, 4, 3, 700, 300
    cap = EnrollCapture(S, C, capacity, device=dev)
    g = torch.Generator().manual_seed(700)
    pushed = [torch.zeros(C, 0, device=dev) for _ in range(S)]
    for t in range(ticks):
        sl = torch.randperm(S - 1, generator=g)[:n].tolist()      # slot S - 1 is never listed
        sl[t % n] = [-1, S, S + 5, -9][t % 4]
        hops = torch.randint(0, T + 1, (n,), generator=g).tolist()
        chunk = torch.full((n, C, HOP * T + CARRY), NAN, device=dev)     # samples a row does not capture are NaN
        for i, h in enumerate(hops):
            chunk[i, :, CARRY:CARRY + HOP * h] = torch.randn(C, HOP * h, generator=g).to(dev)
        cap(chunk, i32(sl, dev), i32(hops, dev))
        for i, (s, h) in enumerate(zip(sl, hops)):
            if 0 <= s < S:
                pushed[s] = torch.cat([pushed[s], chunk[i, :, CARRY:CARRY + HOP * h]], 1)
    got = cap.captured.tolist()
    for s in range(S - 1):
        P = pushed[s].shape[1]
        assert P > 3 * capacity and got[s] == capacity
        assert int(cap.state[s, 0, 0].view(torch.int32)) == P % capacity
        assert torch.equal(bits(ring_last(cap, s, capacity)), bits(pushed[s][:, P - capacity:])), s
    assert not cap.state[S - 1].any() and got[S - 1] == 0
    cap.reset([0, 2])
    assert cap.captured.tolist()[:3] == [0, got[1], 0] and not cap.state[0].any()


def test_graph_replay_fifo_then_capture(dev):
    """FIFO -> capture captured once in a CUDA graph and replayed with slots, counts and pieces rewritten in place, against
    direct calls; the capture holds the last `capacity` samples the FIFO popped"""
    S, C, n, T, max_in, capacity = 6, 2, 4, 3, 400, 900

    def pair():
        return {"fifo": HopFifo(S, C, T, 2048, device=dev), "cap": EnrollCapture(S, C, capacity, device=dev)}

    def tick(o, x, counts, slots, chunk, hops):
        o["fifo"](x, counts, slots, out=chunk, hops=hops)
        o["cap"](chunk, slots, hops)

    live, twin = pair(), pair()
    x = torch.zeros(n, C, max_in, device=dev)
    counts, slots = i32([0] * n, dev), i32(list(range(n)), dev)
    chunk = torch.zeros(n, C, HOP * T + CARRY, device=dev)
    hops = torch.zeros(n, dtype=torch.int32, device=dev)
    graph = captured(lambda: tick(live, x, counts, slots, chunk, hops))   # pushes of nothing: the states stay empty
    g = torch.Generator().manual_seed(90)
    fed = [torch.zeros(C, 0, device=dev) for _ in range(S)]
    for t in range(200):
        sl = torch.randperm(S, generator=g)[:n].tolist()
        sl[t % n] = -1 if t % 2 else S
        cn = torch.randint(0, max_in + 1, (n,), generator=g).tolist()
        x.copy_(torch.randn(n, C, max_in, generator=g).to(dev))
        slots.copy_(i32(sl, dev))
        counts.copy_(i32(cn, dev))
        graph.replay()
        c2, h2 = torch.zeros_like(chunk), torch.zeros_like(hops)
        tick(twin, x, i32(cn, dev), i32(sl, dev), c2, h2)
        for i, (s, m) in enumerate(zip(sl, cn)):
            if 0 <= s < S:
                fed[s] = torch.cat([fed[s], x[i, :, :m]], 1)
    torch.cuda.synchronize()
    fifo, cap = live["fifo"], live["cap"]
    assert fifo.dropped.sum().item() == 0
    assert_same({}, {}, live, twin, "after 200 ticks")
    for s in range(S):
        popped = fed[s].shape[1] - int(fifo.held[s])
        k = min(popped, capacity)
        assert popped > capacity and cap.captured[s].item() == k
        assert torch.equal(bits(ring_last(cap, s, k)), bits(fed[s][:, popped - k:popped])), s


def _filled_capture(dev, S, capacity, totals, T=4, seed=3000):
    """an EnrollCapture of S slots, slot s fed totals[s] samples (multiples of 128) of a seeded signal, in T-hop calls of
    every slot at once; and the signals [S, 2, max(totals)]"""
    sig = synth.enrollment(S, max(totals), seed0=seed).to(dev)
    cap = EnrollCapture(S, 2, capacity, device=dev)
    fed = [0] * S
    while any(f < t for f, t in zip(fed, totals)):
        hops = [min(T, (t - f) // HOP) for f, t in zip(fed, totals)]
        chunk = torch.full((S, 2, HOP * T + CARRY), NAN, device=dev)
        for s, h in enumerate(hops):
            chunk[s, :, CARRY:CARRY + HOP * h] = sig[s, :, fed[s]:fed[s] + HOP * h]
            fed[s] += HOP * h
        cap(chunk, list(range(S)), hops)
    return cap, sig


@pytest.mark.parametrize("n", [1, 5, 17])
def test_enroll_from_rings_equals_forward(embed, dev, n):
    """windows of 192 .. n_max samples, many wrapping the ring; a slot that captured fewer samples than asked (its whole
    capture is used) and one under 192 (not written); host and CUDA slot lists; a row-strided out"""
    net, sd = embed
    S, capacity = 24, 6000
    g = torch.Generator().manual_seed(40 + n)
    totals = [HOP * int(k) for k in torch.randint(capacity // HOP + 2, 3 * capacity // HOP, (S,), generator=g)]
    totals[22], totals[23] = 128, 1024                        # under 192; 1024 only
    cap, sig = _filled_capture(dev, S, capacity, totals)
    pick = torch.randperm(22, generator=g)[:n].tolist()
    lens = torch.randint(192, capacity + 1, (n,), generator=g).tolist()
    lens[0] = capacity if n == 1 else 192
    if n > 1:
        pick[1], lens[1], lens[-1] = 23, 5000, capacity
    if n > 5:
        pick[2] = 22
    used_want = []
    for s, L in zip(pick, lens):
        u = min(L, totals[s], capacity)
        used_want.append(u if u >= 192 else 0)
    N = max(lens)
    x = torch.zeros(n, 2, N, device=dev)
    for b, (s, u) in enumerate(zip(pick, used_want)):
        if u:
            x[b, :, :u] = sig[s, :, totals[s] - u:totals[s]]
        else:                                                 # a row enroll skips: any audio of the same batch
            x[b, :, :192] = sig[s, :, :192]
    with torch.no_grad():
        ref = net(x, [u or 192 for u in used_want])
    live = [b for b, u in enumerate(used_want) if u]
    for slots in (pick, i32(pick, dev)):
        staging = torch.randn(2 * n + 1, 256, device=dev)
        before = staging.clone()
        out = staging[1::2]
        used = torch.full((n,), -3, dtype=torch.int32, device=dev)
        with torch.no_grad():
            r = net.enroll(cap, slots, lens, out=out, used=used)
        assert r is out
        assert used.tolist() == used_want
        assert torch.equal(bits(staging[0::2]), bits(before[0::2]))
        for b in range(n):
            want = ref[b] if used_want[b] else before[1 + 2 * b]
            assert torch.equal(bits(out[b]), bits(want)), (b, pick[b], lens[b], used_want[b])
    with torch.no_grad():
        fresh = net.enroll(cap, pick, lens).cpu()
    for b in range(n):
        assert torch.isnan(fresh[b]).all() if not used_want[b] else torch.equal(bits(fresh[b]), bits(ref[b].cpu()))
    for b in live[:2]:
        r0 = rs.embed_forward(sd, x[b:b + 1, :, :used_want[b]].cpu())
        assert rs.rel_l2(fresh[b:b + 1], r0) <= 1e-3, (b, rs.rel_l2(fresh[b:b + 1], r0))


def test_enroll_cuda_slot_outside_capture(embed, dev):
    net, _ = embed
    cap, _ = _filled_capture(dev, 3, 1000, [1280, 1280, 1280])
    out = torch.zeros(3, 256, device=dev)
    used = torch.zeros(3, dtype=torch.int32, device=dev)
    with torch.no_grad():
        net.enroll(cap, i32([1, -1, 3], dev), [500, 500, 500], out=out, used=used)
    assert used.tolist() == [500, 0, 0]
    assert out[0].abs().sum() > 0 and not out[1:].any()


def test_reenroll_mid_stream(model, embed, dev):
    """Three listeners stream through FIFO -> capture -> advance_slots with embeddings A.  After hop h listener 1 is
    enrolled from its last 3 s of capture into its row of the staging buffer.  From hop h + 1 its output equals a run
    handed the torch-computed embedding of that window, and the other listeners' outputs equal a run without the
    enrollment, bit for bit."""
    sep, _ = model
    enet, _ = embed
    S, slots, T, win = 4, [2, 0, 3], 2, 48000
    n = len(slots)
    pre, post = win // (HOP * T) + 4, 6                       # ticks before the enrollment, and after it
    ticks = pre + post
    x, _ = synth.mixture(n, HOP * T * ticks, seed0=9100)
    x = x.to(dev)
    fifo, cap = HopFifo(S, 2, T, 4096, device=dev), EnrollCapture(S, 2, win, device=dev)
    st = sep.init_buffers(S, dev)
    E = synth.embedding(n, seed0=9200)[:, 0].to(dev)
    sl, cnt = i32(slots, dev), i32([HOP * T] * n, dev)

    def tick(objs, t, emb):
        fifo, cap, st = objs
        chunk, hops = fifo(x[:, :, HOP * T * t:HOP * T * (t + 1)], cnt, sl)
        cap(chunk, sl, hops)
        return sep.advance_slots(chunk, emb, st, sl, hops=hops), hops

    with torch.no_grad():
        for t in range(pre):
            tick((fifo, cap, st), t, E)
        popped = HOP * T * pre                                # every push of two hops is popped in its tick
        assert cap.captured[slots[1]].item() == win and popped >= win
        window = x[1:2, :, popped - win:popped]
        branches = {}
        for name in ("enrolled", "handed", "plain"):
            twin = sep.init_buffers(S, dev)
            twin.buf.copy_(st.buf)
            f2, c2 = HopFifo(S, 2, T, 4096, device=dev), EnrollCapture(S, 2, win, device=dev)
            f2.state.copy_(fifo.state)
            c2.state.copy_(cap.state)
            branches[name] = [(f2, c2, twin), E.clone(), []]
        e_objs, e_emb, _ = branches["enrolled"]
        used = torch.zeros(1, dtype=torch.int32, device=dev)
        enet.enroll(e_objs[1], [slots[1]], [win], out=e_emb[1:2], used=used)
        branches["handed"][1][1] = enet(window)[0]
        for t in range(pre, ticks):
            for name, (objs, emb, ys) in branches.items():
                y, hops = tick(objs, t, emb)
                assert hops.tolist() == [T] * n
                ys.append(y.clone())
    assert used.item() == win
    assert torch.equal(bits(branches["enrolled"][1][1]), bits(branches["handed"][1][1]))
    ye, yh, yp = (torch.cat(branches[k][2], -1) for k in ("enrolled", "handed", "plain"))
    assert rs.rel_l2(ye[1:2].cpu(), yh[1:2].cpu()) <= 1e-5
    assert not torch.equal(ye[1], yp[1])
    for i in (0, 2):
        assert torch.equal(bits(ye[i]), bits(yp[i])), i
