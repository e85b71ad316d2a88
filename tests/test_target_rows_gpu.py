"""Listeners with different numbers of targets in one call (Net.advance_target_rows / l2h_sep_forward_targets_rows).

Two oracles.  With uniform lists (offsets i*K, records g_i*K + k) the call is the groups call, bit for bit, y and state.  With
mixed lists (K_i in {1, 2, 3}, scattered records, spare rows) it is a slot-list call over the same R target rows with each
target row fed its listener's mixture: every form is chosen for the R rows in both, so y is bit-identical except in the
fused one-hop form, where block 1's input projection is a separate GEMM in a targets call (rounding only, see
include/lookonce_b200.h).  The forms are those of tests/test_targets_groups_gpu.py."""
import time

import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import synth
from oracle import restate as rs
import serving_util as su
from serving_util import HOP, LA, L2H_FLAG_GRAPH, SENTINEL, dev, model  # noqa: F401
from test_targets_groups_gpu import FORMS, RAGGED

pytestmark = pytest.mark.gpu


def _switched(request, model):
    n, K, T, opts = request.param
    net, sd = model
    with su.switched(net, opts):
        yield net, n, K, T, opts


@pytest.fixture(params=FORMS)
def form(request, model):
    """(net, n, K, T, opts): the network switched to the kernel form under test for the test's duration."""
    yield from _switched(request, model)


@pytest.fixture(params=RAGGED)
def ragged(request, model):
    yield from _switched(request, model)


def fused_one_hop(T, K_rows, opts):
    """whether a call of K_rows target rows and T hops takes the fused one-hop form (tail_kernel), where a targets call
    rounds block 1's input projection differently from a call that is not one"""
    return T == 1 and opts.get("fused_tail", 1) == 1 and K_rows * T * 97 <= 2048


def mix(R, seed):
    """the targets per listener of a call of R target rows: K_i in {1, 2, 3}, and R // 8 spare rows; all ones for R <= 3
    (as many listeners as rows: block 0's rows then do not fit beside it in the workspace, the fallback path)"""
    if R <= 3:
        return [1] * R
    g = torch.Generator().manual_seed(seed)
    live, ks = R - R // 8, []
    while sum(ks) < live:
        ks.append(min(int(torch.randint(1, 4, (1,), generator=g)), live - sum(ks)))
    return ks


def offsets_of(ks):
    o = [0]
    for k in ks:
        o.append(o[-1] + k)
    return o


def owners(ks, R):
    """the listener of every target row, -1 past the listed ones"""
    own = [i for i, k in enumerate(ks) for _ in range(k)]
    return own + [-1] * (R - len(own))


def outside_front(st):
    """bool [stride]: everything of a record but its conv tails and block 0 (a targets call's lead-only areas)"""
    L = st.lay
    m = torch.ones(st.stride, dtype=torch.bool, device=st.buf.device)
    m[L["st_conv"]:L["st_deconv"]] = False
    m[L["st_blk"]:L["st_blk"] + L["bk_stride"]] = False
    return m


# ---- uniform lists are the groups call ---------------------------------------------------------------------------------
def test_uniform_lists_equal_groups_call(form, dev):
    """offsets i*K and records g_i*K + k over a warm targets state: y and the whole state equal advance_targets with the
    same groups (and, for multi-hop forms, hops) on a copy, bit for bit, over 3 calls."""
    net, n, K, T, _ = form
    G = n + 3
    st, fed = su.warm_groups(net, G, n, K, T, 7100, dev)
    twin = su.copy(net, st)
    clips, _ = su.clips(G, 8 * T, 7100, dev)
    emb = su.embeds(G, K, 7101, dev)
    with torch.no_grad():
        for c, sl in enumerate(su.subsets(G, n, 3, 7200)):
            hops = su.hop_mix(n, T, 7300 + c) if T > 1 and n >= 2 else None
            x = torch.stack([su.chunk(clips[g], fed[g], T) for g in sl])
            y = net.advance_target_rows(x, emb[sl].reshape(n * K, 256), st, su.recs(sl, K), [i * K for i in range(n + 1)],
                                        hops=hops)
            y_ref = net.advance_targets(x, emb[sl], twin, sl, hops=hops)
            torch.cuda.synchronize()
            for i, g in enumerate(sl):
                fed[g] += hops[i] if hops else T
            assert y.shape == (n * K, 2, HOP * T)
            if hops is None:
                assert torch.equal(su.bits(y), su.bits(y_ref.reshape(n * K, 2, -1))), f"call {c}: y"
            else:
                for i, h in enumerate(hops):
                    got, ref = y[i * K:(i + 1) * K, :, :HOP * h], y_ref[i, :, :, :HOP * h]
                    assert torch.equal(su.bits(got), su.bits(ref)), (c, i, h)
            assert torch.equal(su.bits(st.buf), su.bits(twin.buf)), f"call {c}: state"


# ---- mixed lists against a slot-list call with repeated mixtures -------------------------------------------------------
def test_mixed_lists_equal_slot_call(form, dev):
    """K_i in {1, 2, 3}, scattered unordered records, spare rows past offsets[n]; 2 ticks on fresh states with their own
    hop counts.  Against slots_hops over the same R rows (spare rows at slot -1), each target row fed its listener's
    mixture: y equal bit for bit (1e-5 relative L2 in the fused one-hop form); every target record equal outside its conv
    tails and block 0, each lead record equal whole; non-lead block-0 areas and unlisted records untouched."""
    net, n0, K0, T, opts = form
    R = n0 * K0
    ks = mix(R, 7400 + R)
    n = len(ks)
    own = owners(ks, R)
    off = offsets_of(ks)
    S = R + 3
    g = torch.Generator().manual_seed(7500 + R)
    records = torch.randperm(S, generator=g)[:R].tolist()
    lead = [records[off[i]] for i in range(n)]
    live = [records[r] for r in range(R) if own[r] >= 0]
    nonlead = [rec for rec in live if rec not in lead]
    unlisted = [s for s in range(S) if s not in live]
    clips, _ = su.clips(n, 2 * T, 7600 + R, dev)
    e = su.emb(R, 7700 + R, dev)
    st, ref = net.init_buffers(S, dev), net.init_buffers(S, dev)
    fused = fused_one_hop(T, R, opts)
    outside = outside_front(st)
    blk0 = ~outside
    fed = [0] * n
    with torch.no_grad():
        for c in range(2):
            hops = su.hop_mix(n, T, 7800 + c) if n >= 2 else [T]
            x = torch.stack([su.chunk(clips[i], fed[i], T) for i in range(n)]).contiguous()
            x_rows = x[[max(i, 0) for i in own]].contiguous()
            slots = [records[r] if own[r] >= 0 else -1 for r in range(R)]
            row_hops = [hops[i] if i >= 0 else 0 for i in own]
            before = su.bits(st._rec()).clone()
            y = torch.full((R, 2, HOP * T), SENTINEL, device=dev)
            y_ref = torch.full_like(y, SENTINEL)
            net._launch("targets_rows", x, e, st, y, T, slots=su.i32(records, dev), offsets=su.i32(off, dev),
                        hops=su.i32(hops, dev))
            net._launch("slots_hops", x_rows, e, ref, y_ref, T, slots=su.i32(slots, dev), hops=su.i32(row_hops, dev))
            torch.cuda.synchronize()
            for i in range(n):
                fed[i] += hops[i]
            if fused:
                assert rs.rel_l2(torch.nan_to_num(y).cpu(), torch.nan_to_num(y_ref).cpu()) <= 1e-5, c
                assert torch.equal(torch.isnan(y), torch.isnan(y_ref)), c
            else:
                assert torch.equal(su.bits(y), su.bits(y_ref)), f"tick {c}: y"
            a, b = su.bits(st._rec()), su.bits(ref._rec())
            if not fused:
                for rec in live:
                    assert torch.equal(a[rec][outside], b[rec][outside]), (c, rec, "blocks 1.., tails, memo, clock")
            for rec in lead:
                assert torch.equal(a[rec][blk0], b[rec][blk0]), (c, rec, "a lead's conv tails and block 0")
            for rec in nonlead:
                assert torch.equal(a[rec][blk0], before[rec][blk0]), (c, rec, "a non-lead block 0 changed")
            assert torch.equal(a[unlisted], before[unlisted]), (c, "an unlisted record changed")
            pos = st.stream_pos()
            assert [pos[rec] for rec in live] == [ref.stream_pos()[rec] for rec in live]
            assert [pos[records[r]] for r in range(R) if own[r] >= 0] == [fed[i] for i in own if i >= 0]


# ---- rows that store nothing -------------------------------------------------------------------------------------------
def test_rows_that_store_nothing(ragged, dev):
    """Over a state one call has warmed: a listener with 0 hops, one whose lead record lies outside the state, one with no
    rows, a row whose own record lies outside the state, and rows past offsets[n] store nothing (records as they were,
    y rows at the sentinel); the one ordinary listener still advances."""
    net, _, _, T, _ = ragged
    ks = [2, 1, 0, 2, 2]                    # listeners: ordinary, 0 hops, no rows, lead outside, one row outside
    off = offsets_of(ks)
    R = off[-1] + 2                         # two spare rows
    S = R + 2
    records = torch.randperm(S, generator=torch.Generator().manual_seed(8000))[:R].tolist()
    clips, _ = su.clips(len(ks), 2 * T, 8100, dev)
    e = su.emb(R, 8200, dev)
    st = net.init_buffers(S, dev)
    rec_d, off_d = su.i32(records, dev), su.i32(off, dev)
    with torch.no_grad():
        net._launch("targets_rows", clips[..., :HOP * T + LA].contiguous(), e, st,
                    torch.empty(R, 2, HOP * T, device=dev), T, slots=rec_d, offsets=off_d)
        bad = list(records)
        bad[off[3]] = S + 5                 # listener 3's lead
        bad[off[4] + 1] = -1                # listener 4's second row
        before = su.bits(st._rec()).clone()
        y = torch.full((R, 2, HOP * T), SENTINEL, device=dev)
        net._launch("targets_rows", clips[..., HOP * T:2 * HOP * T + LA].contiguous(), e, st, y, T, slots=su.i32(bad, dev),
                    offsets=off_d, hops=su.i32([T, 0, T, T, T], dev))
        torch.cuda.synchronize()
    a = su.bits(st._rec())
    silent_rows = list(range(off[1], off[2])) + list(range(off[3], off[4])) + [off[4] + 1] + list(range(off[5], R))
    for r in silent_rows:
        assert bool(torch.isnan(y[r]).all()), (r, "a y row was written")
        if 0 <= bad[r] < S:
            assert torch.equal(a[bad[r]], before[bad[r]]), (r, "a record changed")
    for r in (off[0], off[0] + 1, off[4]):
        assert not bool(torch.isnan(y[r]).any()), (r, "an ordinary row stored nothing")
    assert st.stream_pos()[records[0]] == 2 * T and st.stream_pos()[records[off[1]]] == T


# ---- one graph across ticks --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n, R, T", [pytest.param(4, 8, 1, id="one-hop"), pytest.param(12, 30, 1, id="tc-mid"),
                                     pytest.param(3, 7, 3, id="T3")])
def test_graph_replay_with_lists_rewritten(model, dev, n, R, T):
    """With L2H_FLAG_GRAPH and fixed buffers, records, offsets and hops rewritten in place between ticks (another K mix,
    other records, spare rows): every replayed tick equals the same tick launched directly on a twin state, bit for bit,
    and only the first tick captures."""
    net, _ = model
    S, calls = R + 4, 5
    clips, _ = su.clips(n, calls * T, 8300, dev)
    e = su.emb(R, 8400, dev)
    xbuf = torch.empty(n, 2, HOP * T + LA, device=dev)
    rec_b, off_b = torch.empty(R, dtype=torch.int32, device=dev), torch.empty(n + 1, dtype=torch.int32, device=dev)
    hop_b = torch.empty(n, dtype=torch.int32, device=dev)
    yg, yd = torch.empty(R, 2, HOP * T, device=dev), torch.empty(R, 2, HOP * T, device=dev)
    sg, sdir = net.init_buffers(S, dev), net.init_buffers(S, dev)
    g = torch.Generator().manual_seed(8500)
    host = []
    for c in range(calls):
        ks = [int(v) for v in torch.randint(0, 4, (n,), generator=g)]
        while sum(ks) > R:
            ks[ks.index(max(ks))] -= 1
        ks[0] = max(ks[0], 1)
        ks[0] -= max(0, sum(ks) - R)
        xbuf.copy_(clips[..., HOP * T * c:HOP * T * (c + 1) + LA])
        rec_b.copy_(torch.randperm(S, generator=g)[:R].to(torch.int32))
        off_b.copy_(torch.tensor(offsets_of(ks), dtype=torch.int32))
        hop_b.copy_(torch.tensor(su.hop_mix(n, T, 8600 + c) if T > 1 else [1] * n, dtype=torch.int32))
        yg.fill_(SENTINEL)
        yd.fill_(SENTINEL)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        net._launch("targets_rows", xbuf, e, sg, yg, T, L2H_FLAG_GRAPH, slots=rec_b, offsets=off_b, hops=hop_b)
        host.append(time.perf_counter() - t0)
        net._launch("targets_rows", xbuf, e, sdir, yd, T, slots=rec_b, offsets=off_b, hops=hop_b)
        torch.cuda.synchronize()
        assert torch.equal(su.bits(yg), su.bits(yd)), c
        assert bool(torch.isnan(yg[sum(ks):]).all()), (c, "a spare row wrote y")
    assert torch.equal(su.bits(sg.buf), su.bits(sdir.buf))
    assert max(host[1:]) < 0.5 * host[0], ("a replay took as long as a capture: new graph per tick?", host)


# ---- end to end: streaming with mixed K and missed hops, against the whole clip -----------------------------------------
def test_streaming_with_missed_hops_equals_whole_clip(model, dev):
    """Three listeners with 1, 3 and 2 targets on scattered records of one state, streamed by one-hop advance_target_rows
    ticks with a spare row; a listener whose chunk is late misses ticks and catches up with hops= on the tick its chunks
    arrive.  Every target against forward of its clip with its embedding: relative L2 <= 1e-4."""
    net, _ = model
    ks, total = [1, 3, 2], 40
    n, R = len(ks), sum(ks) + 1
    off = offsets_of(ks)
    own = owners(ks, R)
    records = [9, 2, 7, 4, 0, 11, 5]
    x, _ = synth.mixture(n, HOP * total, seed0=8700)
    e = su.emb(R, 8800, dev)
    xp = F.pad(x.to(dev), (0, LA + HOP * total))
    st = net.init_buffers(12, dev)
    gen = torch.Generator().manual_seed(8900)
    arrived, fed = [0] * n, [0] * n
    outs = [[] for _ in range(R - 1)]
    catch_ups = 0
    with torch.no_grad():
        live = [r for r in range(R) if own[r] >= 0]
        y_full = net.forward(x.to(dev)[[own[r] for r in live]], e[live][:, None])
        tick = 0
        while min(fed) < total:
            for i in range(n):
                if not (tick < total - 4 and float(torch.rand(1, generator=gen)) < 0.3):
                    arrived[i] = min(tick + 1, total)
            h = [a - f for a, f in zip(arrived, fed)]
            tick += 1
            T = max(h)
            if T == 0:
                continue
            catch_ups += T > 1
            xs = torch.stack([su.chunk(xp[i], fed[i], T) for i in range(n)])
            y = net.advance_target_rows(xs, e, st, records, off, hops=h)
            for r in live:
                outs[r].append(y[r, :, :HOP * h[own[r]]])
            for i in range(n):
                fed[i] += h[i]
        assert catch_ups > 0, "no hop was missed"
    ys = torch.stack([torch.cat(o, -1) for o in outs])
    assert ys.shape == y_full.shape == (R - 1, 2, HOP * total)
    assert rs.rel_l2(ys.cpu(), y_full.cpu()) <= 1e-4
    pos = st.stream_pos()
    assert [pos[records[r]] for r in live] == [total] * len(live)
