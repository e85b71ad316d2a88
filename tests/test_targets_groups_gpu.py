"""Several targets per mixture over a list of a state's groups (Net.advance_targets / l2h_sep_forward_targets_groups).

The oracle is the one of the slot-list tests, applied to whole groups: copy the listed groups' K records each into a
compact state of n*K records (copy_streams_from), run predict_targets there and copy them back.  A groups call chooses
every kernel form for its n*K target rows, as predict_targets of n mixtures does, so it must equal the oracle bit for bit
in every form of tests/test_targets_gpu.py, the fused one-hop form included.  Ragged hop counts are checked as in
tests/test_slot_list_hops_gpu.py."""
import time

import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import synth
from oracle import restate as rs
import serving_util as su
from serving_util import HOP, LA, L2H_FLAG_GRAPH, SENTINEL, dev, model  # noqa: F401

pytestmark = pytest.mark.gpu
# (listed groups, targets, hops per call, engine options): the forms of tests/test_targets_gpu.py
FORMS = [pytest.param((1, 2, 1, {}), id="fused-tail-1x2"),
         pytest.param((2, 3, 1, {}), id="fused-tail-2x3"),
         pytest.param((1, 2, 1, {"fused_tail": 0}), id="mid-kernel-1x2"),
         pytest.param((2, 3, 1, {"fused_tail": 0}), id="mid-kernel-2x3"),
         pytest.param((6, 2, 1, {"fused_tail": 0}), id="mid-split-6x2"),
         pytest.param((8, 3, 1, {}), id="tc-mid-8x3"),
         pytest.param((64, 3, 1, {}), id="tc-mid-64x3"),
         pytest.param((1, 2, 3, {}), id="T3-1x2"),
         pytest.param((1, 2, 3, {"back_many": 0}), id="T3-1x2-per-frame"),
         pytest.param((4, 2, 3, {}), id="T3-tc-lstm-rec-4x2"),
         pytest.param((16, 3, 2, {}), id="T2-tc-lstm-16x3"),
         pytest.param((16, 3, 2, {"fuse_ih": 1}), id="T2-tc-lstm-x-16x3")]
# multi-hop forms with at least two listed groups, for the ragged hop counts
RAGGED = [pytest.param((2, 2, 3, {}), id="T3-2x2"),
          pytest.param((2, 2, 3, {"back_many": 0}), id="T3-2x2-per-frame"),
          pytest.param((4, 2, 3, {}), id="T3-tc-lstm-rec-4x2"),
          pytest.param((16, 3, 2, {}), id="T2-tc-lstm-16x3"),
          pytest.param((16, 3, 2, {"fuse_ih": 1}), id="T2-tc-lstm-x-16x3")]


@pytest.fixture(params=FORMS)
def form(request, model):
    """(net, sd, n, K, T): the network switched to the kernel form under test for the test's duration."""
    n, K, T, opts = request.param
    net, sd = model
    with su.switched(net, opts):
        yield net, sd, n, K, T


@pytest.fixture(params=RAGGED)
def ragged(request, model):
    n, K, T, opts = request.param
    net, sd = model
    with su.switched(net, opts):
        yield net, sd, n, K, T


# ---- every form against copy / predict_targets / copy back ----------------------------------------------------------
def test_groups_equal_copy_run_copy_back(form, dev):
    """4 calls over changing random subsets of a warm state of G > n groups: y and every listed record equal the oracle
    bit for bit, unlisted records are untouched, and so are the conv tails and block 0 of the non-lead records."""
    net, _, n, K, T = form
    G = n + 3
    st, fed = su.warm_groups(net, G, n, K, T, 4100, dev)
    ref = su.copy(net, st)
    compact = net.init_buffers(n * K, dev)
    clips, _ = su.clips(G, 8 * T, 4100, dev)
    emb = su.embeds(G, K, 4101, dev)                      # the warm-up's embeddings: the gate memos stay valid
    foreign = su.foreign(st, K)
    with torch.no_grad():
        for c, sl in enumerate(su.subsets(G, n, 4, 4200)):
            x = torch.stack([su.chunk(clips[g], fed[g], T) for g in sl])
            before = su.bits(st._rec()).clone()
            y = net.advance_targets(x, emb[sl], st, sl)
            y_ref = su.oracle(net, ref, su.recs(sl, K), x, emb[sl], compact)
            for g in sl:
                fed[g] += T
            assert y.shape == (n, K, 2, HOP * T)
            assert torch.equal(su.bits(y), su.bits(y_ref)), f"call {c}: y"
            listed = su.recs(sl, K)
            unlisted = [r for r in range(G * K) if r not in listed]
            assert torch.equal(su.bits(st._rec())[unlisted], before[unlisted]), f"call {c}: an unlisted record changed"
            assert torch.equal(su.records(st), su.records(ref)), f"call {c}: records"
            assert torch.equal(su.bits(st._rec())[foreign], before[foreign]), f"call {c}: a non-lead conv tail or block 0"
    assert st.stream_pos() == ref.stream_pos() == [fed[r // K] for r in range(G * K)]


# ---- ragged hop counts -----------------------------------------------------------------------------------------------
def test_all_hops_T_equal_no_hop_list(ragged, dev):
    net, _, n, K, T = ragged
    G = n + 2
    st, _ = su.warm_groups(net, G, n, K, T, 4300, dev)
    twin = su.copy(net, st)
    clips, _ = su.clips(n, T, 4400, dev)
    e = su.embeds(n, K, 4500, dev).reshape(n * K, 256)
    groups = su.i32(su.subsets(G, n, 1, 4600)[0], dev)
    y = torch.full((n, K, 2, HOP * T), SENTINEL, device=dev)
    y_ref = torch.full_like(y, SENTINEL)
    net._launch("targets_groups", clips.contiguous(), e, st, y, T, slots=groups, hops=su.i32([T] * n, dev), K=K)
    net._launch("targets_groups", clips.contiguous(), e, twin, y_ref, T, slots=groups, K=K)
    torch.cuda.synchronize()
    assert torch.equal(su.bits(y), su.bits(y_ref))
    assert torch.equal(su.bits(st.buf), su.bits(twin.buf))


def test_zero_hops_and_outside_groups_store_nothing(ragged, dev):
    net, _, n, K, T = ragged
    G = n + 2
    st, _ = su.warm_groups(net, G, n, K, T, 4700, dev)
    before = su.bits(st._rec()).clone()
    clips, _ = su.clips(n, T, 4800, dev)
    e = su.embeds(n, K, 4900, dev).reshape(n * K, 256)
    sl = su.subsets(G, n, 1, 5000)[0]
    for groups, hops in ((sl, [0] * n), ([-1 - i if i % 2 else G + i for i in range(n)], [T] * n),
                         (sl, [T + 1 + i if i % 2 else -1 - i for i in range(n)])):      # counts outside [0, T] count as 0
        y = torch.full((n, K, 2, HOP * T), SENTINEL, device=dev)
        net._launch("targets_groups", clips.contiguous(), e, st, y, T, slots=su.i32(groups, dev), hops=su.i32(hops, dev), K=K)
        torch.cuda.synchronize()
        assert bool(torch.isnan(y).all()), (groups, hops, "a y row was written")
        assert torch.equal(su.bits(st._rec()), before), (groups, hops, "a record changed")


def test_mixed_hops_match_uniform_call_where_they_advance(ragged, dev):
    """x NaN past each group's 128 h_i + 64 samples: the y samples and ring rows of the frames each group advances equal a
    uniform T-hop call on a copy bit for bit; later y samples keep the sentinel; other ring rows and unlisted records are
    as before; every record of a group advances its clock by h_i (its calls by 1 if h_i > 0)."""
    net, _, n, K, T = ragged
    G = n + 2
    st, _ = su.warm_groups(net, G, n, K, T, 5100, dev)
    twin = su.copy(net, st)
    before = st._rec().clone()
    pos0, calls0 = st.stream_pos(), st._clocks()[1].cpu().tolist()
    clips, _ = su.clips(n, T, 5200, dev)
    x = clips.contiguous().clone()
    hops = su.hop_mix(n, T, 5300)
    for i, h in enumerate(hops):
        x[i, :, HOP * h + LA:] = float("nan")
    e = su.embeds(n, K, 5400, dev).reshape(n * K, 256)
    sl = su.subsets(G, n, 1, 5500)[0]
    y = torch.full((n, K, 2, HOP * T), SENTINEL, device=dev)
    y_ref = torch.full_like(y, SENTINEL)
    net._launch("targets_groups", x, e, st, y, T, slots=su.i32(sl, dev), hops=su.i32(hops, dev), K=K)
    net._launch("targets_groups", clips.contiguous(), e, twin, y_ref, T, slots=su.i32(sl, dev), K=K)
    torch.cuda.synchronize()
    ring_all = su.ring_mask(st, range(st.lay["ring"]))
    for i, (g, h) in enumerate(zip(sl, hops)):
        assert torch.equal(su.bits(y[i, ..., :HOP * h]), su.bits(y_ref[i, ..., :HOP * h])), (i, h)
        assert bool(torch.isnan(y[i, ..., HOP * h:]).all()), (i, h, "y written past the group's hops")
        for r in su.recs([g], K):
            new = su.ring_mask(st, range(pos0[r], pos0[r] + h))
            assert torch.equal(su.bits(st._rec()[r][new]), su.bits(twin._rec()[r][new])), (i, h, r, "ring rows of the new frames")
            other = ring_all & ~new
            assert torch.equal(su.bits(st._rec()[r][other]), su.bits(before[r][other])), (i, h, r, "another ring row changed")
            if h == 0:
                assert torch.equal(su.bits(st._rec()[r]), su.bits(before[r])), (i, r, "h = 0 stored something")
            if h == T:
                assert torch.equal(su.bits(st._rec()[r]), su.bits(twin._rec()[r])), (i, r, "h = T")
    unlisted = [r for r in range(G * K) if r not in su.recs(sl, K)]
    assert torch.equal(su.bits(st._rec()[unlisted]), su.bits(before[unlisted]))
    pos, calls = st.stream_pos(), st._clocks()[1].cpu().tolist()
    for g, h in zip(sl, hops):
        for r in su.recs([g], K):
            assert pos[r] == pos0[r] + h and calls[r] == calls0[r] + (1 if h > 0 else 0), (g, r, h)


# ---- K = 1 is the ragged slot-list call ------------------------------------------------------------------------------
@pytest.mark.parametrize("n, T", [pytest.param(3, 1, id="one-hop"), pytest.param(4, 3, id="T3")])
def test_one_target_is_slots_hops(model, dev, n, T):
    net, _ = model
    S = n + 3
    clips, _ = su.clips(n, 3 * T, 5600, dev)
    e = su.embeds(n, 1, 5700, dev).reshape(n, 256)
    a, b = net.init_buffers(S, dev), net.init_buffers(S, dev)
    ya, yb = torch.full((n, 1, 2, HOP * T), SENTINEL, device=dev), torch.full((n, 2, HOP * T), SENTINEL, device=dev)
    for c, sl in enumerate(su.subsets(S, n, 3, 5800)):
        x = clips[..., HOP * T * c:HOP * T * (c + 1) + LA].contiguous()
        groups, hops = su.i32(sl, dev), su.i32(su.hop_mix(n, T, 5900 + c), dev)
        net._launch("targets_groups", x, e, a, ya, T, slots=groups, hops=hops, K=1)
        net._launch("slots_hops", x, e, b, yb, T, slots=groups, hops=hops)
        torch.cuda.synchronize()
        assert torch.equal(su.bits(ya[:, 0]), su.bits(yb)), c
    assert torch.equal(su.bits(a.buf), su.bits(b.buf))


# ---- graph replay with the lists rewritten in place --------------------------------------------------------------------
@pytest.mark.parametrize("n, K, T", [pytest.param(2, 2, 1, id="one-hop"), pytest.param(8, 3, 1, id="tc-mid"),
                                     pytest.param(3, 2, 3, id="T3")])
def test_graph_replay_with_groups_and_hops_rewritten(model, dev, n, K, T):
    """With L2H_FLAG_GRAPH and fixed buffers, groups and hops rewritten in place between ticks (a different subset, a
    different mix of depths, one group outside the state): every replayed tick equals the same tick launched directly on a
    twin state, bit for bit.  Only the first tick captures: the graph cached for (n, K, T) reads the lists when it runs."""
    net, _ = model
    G, calls = n + 3, 5
    clips, _ = su.clips(G, calls * T, 6000, dev)
    emb = su.embeds(G, K, 6100, dev)
    xbuf, ebuf = torch.empty(n, 2, HOP * T + LA, device=dev), torch.empty(n * K, 256, device=dev)
    groups, hops = torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, dtype=torch.int32, device=dev)
    yg, yd = torch.empty(n, K, 2, HOP * T, device=dev), torch.empty(n, K, 2, HOP * T, device=dev)
    sg, sdir = net.init_buffers(G * K, dev), net.init_buffers(G * K, dev)
    fed = [0] * G
    host = []
    for c, sl in enumerate(su.subsets(G, n, calls, 6200)):
        hh = su.hop_mix(n, T, 6300 + c) if T > 1 else [1] * n
        listed = list(sl)
        listed[c % n] = G + c if c % 2 else -1 - c            # one group misses the tick
        xbuf.copy_(torch.stack([su.chunk(clips[g], fed[g], T) for g in sl]))
        ebuf.copy_(emb[sl].reshape(n * K, 256))
        groups.copy_(torch.tensor(listed, dtype=torch.int32))
        hops.copy_(torch.tensor(hh, dtype=torch.int32))
        yg.fill_(SENTINEL)
        yd.fill_(SENTINEL)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        net._launch("targets_groups", xbuf, ebuf, sg, yg, T, L2H_FLAG_GRAPH, slots=groups, hops=hops, K=K)
        host.append(time.perf_counter() - t0)
        net._launch("targets_groups", xbuf, ebuf, sdir, yd, T, slots=groups, hops=hops, K=K)
        for i, g in enumerate(listed):
            if 0 <= g < G:
                fed[g] += hh[i]
        torch.cuda.synchronize()
        assert torch.equal(su.bits(yg), su.bits(yd)), c
        assert bool(torch.isnan(yg[c % n]).all()), (c, "the missing group wrote y")
    assert torch.equal(su.bits(sg.buf), su.bits(sdir.buf))
    assert sg.stream_pos() == [fed[r // K] for r in range(G * K)]
    assert max(host[1:]) < 0.5 * host[0], ("a replay took as long as a capture: new graph per tick?", host)


# ---- end to end: streaming with missed hops, against the whole clip and the reference ---------------------------------
def test_streaming_with_missed_hops_equals_whole_clip(model, dev):
    """Two groups of K = 2 streamed by one-hop advance_targets ticks; a group whose chunk is late (seeded) misses ticks and
    catches its backlog up with hops= on the tick its chunks arrive.  Against forward_targets of the whole clips: relative
    L2 <= 1e-4; one target against the reference restatement: 1e-3 relative L2 and 0.1 dB SI-SDR."""
    net, sd = model
    G, K, total = 2, 2, 40
    x, tgt = synth.mixture(G, HOP * total, seed0=6400)
    emb = su.embeds(G, K, 6500, dev)
    xp = F.pad(x.to(dev), (0, LA + HOP * total))          # a call's x rows span its longest backlog
    st = net.init_buffers(G * K, dev)
    gen = torch.Generator().manual_seed(6600)
    arrived, fed = [0] * G, [0] * G
    outs = [[] for _ in range(G)]
    catch_ups = 0
    with torch.no_grad():
        y_full = net.forward_targets(x.to(dev), emb)
        tick = 0
        while min(fed) < total:
            for g in range(G):                              # this tick's chunk of each group arrives, or is late
                late = tick < total - 4 and float(torch.rand(1, generator=gen)) < 0.3
                if not late:
                    arrived[g] = min(tick + 1, total)
            h = [a - f for a, f in zip(arrived, fed)]
            tick += 1
            T = max(h)
            if T == 0:
                continue
            catch_ups += T > 1
            xs = torch.stack([su.chunk(xp[g], fed[g], T) for g in range(G)])
            y = net.advance_targets(xs, emb, st, list(range(G)), hops=h)
            for g in range(G):
                outs[g].append(y[g, ..., :HOP * h[g]])
                fed[g] += h[g]
        assert catch_ups > 0, "no hop was missed"
    ys = torch.stack([torch.cat(o, -1) for o in outs])
    assert ys.shape == y_full.shape == (G, K, 2, HOP * total)
    assert rs.rel_l2(ys.cpu(), y_full.cpu()) <= 1e-4
    assert st.stream_pos() == [total] * (G * K)
    y_ref = rs.sep_forward(sd, x[1:2], emb[1, 0].cpu()[None, None])
    got = ys[1, 0][None].cpu()
    assert rs.rel_l2(got, y_ref) <= 1e-3
    d = (rs.si_sdr(got, tgt[1:2]) - rs.si_sdr(y_ref, tgt[1:2])).abs().max()
    assert float(d) <= 0.1
