"""Adding and dropping the targets of a running listener on the GPU (Net.target_history, advance_target_rows(history=),
Net.join_targets, SepState.move_lead), on seeded weights and inputs and fresh states.

Oracles: a rows tick without a history (the history is observational, bit for bit); a listener that listed the joining
record from the start (a join replaying the whole stream equals it within the streaming-vs-whole bound, 1e-4 relative L2,
since the replay is a multi-hop chain and the ticks are one-hop chains); a cold join plus live ticks (a partial replay);
and the same ticks on a twin state (drops and handovers, bit for bit).  Records are compared through
SepState.to_reference(), so the parity of their double-buffered tails does not matter.  R stays fixed within a test, so
the kernel forms of the compared calls match: a row whose record is -1 (a CUDA list, used in place) stores nothing."""
import pytest
import torch

from oracle import restate as rs
import serving_util as su
from serving_util import HOP, L2H_FLAG_GRAPH, SENTINEL, dev, model  # noqa: F401

pytestmark = pytest.mark.gpu

BOUND = 1e-4


def tick(net, st, clips, t, e, recs, off, hist=None, hops=None):
    """one advance_target_rows tick of the listeners' clips at hop t (T = 1, or T = max(hops) with hops)"""
    dev = clips.device
    T = max(hops) if hops else 1
    x = torch.stack([su.chunk(clips[i], t, T) for i in range(len(off) - 1)]).contiguous()
    return net.advance_target_rows(x, e, st, su.i32(recs, dev), su.i32(off, dev),
                                   hops=None if hops is None else su.i32(hops, dev), history=hist)


def record_ref(st, r):
    """record r as the reference's state (tails, K/V history, h / c of every block), one flat float64 vector"""
    ref = st.to_reference()
    parts = [ref["conv_buf"][r], ref["deconv_buf"][r], ref["istft_buf"][r]]
    for i in range(st.n_blocks):
        g = ref["gridnet_bufs"][f"buf{i}"]
        parts += [g["K_buf"][4 * r:4 * r + 4], g["V_buf"][4 * r:4 * r + 4], g["h0"][0, 97 * r:97 * r + 97],
                  g["c0"][0, 97 * r:97 * r + 97]]
    return torch.cat([p.flatten() for p in parts]).double().cpu()


def gate(st, r):
    """record r's gate memo: the embedding it was built from, the weight generation and the gate (not the clock)"""
    L, rec = st.lay, st._rec()[r]
    return su.bits(torch.cat([rec[L["st_emb"]:L["st_emb"] + 257], rec[L["st_gate"]:L["st_gate"] + 97 * 64]]))


# ---- 1. the history is observational ---------------------------------------------------------------------------------
@pytest.mark.parametrize("n, K, T", [pytest.param(2, 2, 1, id="fused-one-hop"), pytest.param(12, 2, 1, id="tensor-core"),
                                     pytest.param(3, 2, 3, id="ragged-T3")])
def test_history_is_observational(model, dev, n, K, T):
    """Rows ticks with and without a history: y and the state bit for bit equal; the ring of each lead holds exactly the
    frames it advanced (slots of later frames and every non-lead ring stay zero), and ragged listeners with h = 0 write
    nothing."""
    net, _ = model
    R, S, F = n * K, n * K + 2, 16
    clips, _ = su.clips(n, 4 * T, 9100 + R, dev)
    e = su.emb(R, 9200 + R, dev)
    recs = torch.randperm(S, generator=torch.Generator().manual_seed(9300))[:R].tolist()
    off = [i * K for i in range(n + 1)]
    st, twin = net.init_buffers(S, dev), net.init_buffers(S, dev)
    hist = net.target_history(st, F)
    fed = [0] * n
    with torch.no_grad():
        for c in range(3):
            hops = su.hop_mix(n, T, 9400 + c) if T > 1 else None
            x = torch.stack([su.chunk(clips[i], fed[i], T) for i in range(n)]).contiguous()
            args = (su.i32(recs, dev), su.i32(off, dev))
            hd = None if hops is None else su.i32(hops, dev)
            y = net.advance_target_rows(x, e, st, *args, hops=hd, history=hist)
            y_ref = net.advance_target_rows(x, e, twin, *args, hops=hd)
            torch.cuda.synchronize()
            for i in range(n):      # the samples listener i's rows receive
                w = HOP * (hops[i] if hops else T)
                assert torch.equal(su.bits(y[i * K:(i + 1) * K, :, :w]), su.bits(y_ref[i * K:(i + 1) * K, :, :w])), (c, i)
            assert torch.equal(su.bits(st.buf), su.bits(twin.buf)), f"tick {c}: state"
            for i in range(n):
                fed[i] += hops[i] if hops else T
    pos = st.stream_pos()
    leads = [recs[i * K] for i in range(n)]
    assert [pos[r] for r in leads] == fed
    for r in range(S):
        live = hist.buf[r].abs().sum(-1) > 0
        want = torch.zeros(F, dtype=torch.bool, device=dev)
        if r in leads:
            want[:fed[leads.index(r)]] = True
        assert torch.equal(live, want), (r, live.tolist())


# ---- 2. a join over the whole stream equals the listener that always had the target -----------------------------------
@pytest.mark.parametrize("n", [pytest.param(1, id="fused-one-hop"), pytest.param(12, id="tensor-core")])
def test_full_history_join_equals_always_on(model, dev, n):
    """Listeners {A_i} (their second row at record -1) with a 64-frame history for 40 hops, then B_i joins with W = 40,
    against listeners {A_i, B_i} from the start: B's record within 1e-4 relative L2 (gate memo and clock exact), the join's
    y against B's first 40 hops, and B's next 20 hops within 1e-4; A's outputs bit for bit unchanged on every hop."""
    net, _ = model
    R, S = 2 * n, 2 * n + 1
    A, B = list(range(0, R, 2)), list(range(1, R, 2))
    clips, _ = su.clips(n, 60, 9500 + n, dev)
    e = su.emb(R, 9600 + n, dev)
    off = [2 * i for i in range(n + 1)]
    st, ref = net.init_buffers(S, dev), net.init_buffers(S, dev)
    hist = net.target_history(st, 64)
    solo = [r if r in A else -1 for r in range(R)]
    outs, refs = [], []
    with torch.no_grad():
        for t in range(40):
            outs.append(tick(net, st, clips, t, e, solo, off, hist))
            refs.append(tick(net, ref, clips, t, e, list(range(R)), off))
        y_join, used = net.join_targets(st, B, A, e[B], history=hist, frames=40)
        torch.cuda.synchronize()
        assert used.tolist() == [40] * n
        assert st.stream_pos()[:R] == ref.stream_pos()[:R] == [40] * R
        for b in B:
            assert rs.rel_l2(record_ref(st, b), record_ref(ref, b)) <= BOUND, b
            assert torch.equal(gate(st, b), gate(ref, b)), (b, "gate memo")
        ref_b = torch.cat([y[B] for y in refs], -1)
        assert rs.rel_l2(y_join.cpu(), ref_b.cpu()) <= BOUND
        for t in range(40, 60):
            outs.append(tick(net, st, clips, t, e, list(range(R)), off, hist))
            refs.append(tick(net, ref, clips, t, e, list(range(R)), off))
        torch.cuda.synchronize()
    for t, (y, yr) in enumerate(zip(outs, refs)):
        assert torch.equal(su.bits(y[A]), su.bits(yr[A])), (t, "A changed")
    got = torch.cat([y[B] for y in outs[40:]], -1)
    want = torch.cat([y[B] for y in refs[40:]], -1)
    assert rs.rel_l2(got.cpu(), want.cpu()) <= BOUND


# ---- 3. a partial replay equals a cold join plus live hops -----------------------------------------------------------
def test_partial_history_equals_cold_join_plus_live(model, dev):
    """Listener {A} for 80 hops with a 64-frame history (the ring wraps), then B joins replaying W = 30; against B cold
    joined at hop 50 and advanced 30 live hops: B's record within 1e-4.  In the same call, C joins lead D, which has
    advanced only 10 hops (h = 0 before): it replays its 10 (used), not 30, and ends at D's clock."""
    net, _ = model
    A, B, D, C, S = 0, 1, 2, 3, 4
    clips, _ = su.clips(2, 80, 9700, dev)
    e = su.emb(4, 9800, dev)
    off = [0, 2, 4]
    st, ref = net.init_buffers(S, dev), net.init_buffers(S, dev)
    hist = net.target_history(st, 64)
    fed = [0, 0]
    with torch.no_grad():
        for t in range(80):
            hops = [1, 1 if t >= 70 else 0]
            x = torch.stack([su.chunk(clips[0], fed[0]), su.chunk(clips[1], fed[1])]).contiguous()
            net.advance_target_rows(x, e, st, su.i32([A, -1, D, -1], dev), su.i32(off, dev), hops=su.i32(hops, dev),
                                    history=hist)
            fed = [f + h for f, h in zip(fed, hops)]
        y, used = net.join_targets(st, [B, C], [A, D], e[[1, 3]], history=hist, frames=30)
        for t in range(50):
            tick(net, ref, clips[:1], t, e[:2], [A, -1], off[:2])
        net.join_targets(ref, [B], [A], e[[1]])                        # cold: no history
        torch.cuda.synchronize()
        assert ref.stream_pos()[B] == 50
        for t in range(50, 80):
            tick(net, ref, clips[:1], t, e[:2], [A, B], off[:2])
        torch.cuda.synchronize()
    assert used.tolist() == [30, 10]
    assert st.stream_pos()[:4] == [80, 80, 10, 10]
    assert rs.rel_l2(record_ref(st, B), record_ref(ref, B)) <= BOUND
    assert not bool(torch.isnan(y[0, :, :HOP * 30]).any()) and not bool(torch.isnan(y[1, :, :HOP * 10]).any())


# ---- 4. a cold join --------------------------------------------------------------------------------------------------
def test_cold_join(model, dev):
    """frames = 0 with a history: B's deep blocks and tails are zero, its clock is the lead's and its gate memo is built
    (equal to the one a tick builds); a row whose lead lies outside the state (a CUDA list) stores nothing; every other
    record, NaN-filled beforehand, is byte-identical."""
    net, _ = model
    A, B, X, S = 0, 1, 2, 5
    clips, _ = su.clips(1, 5, 9900, dev)
    e = su.emb(2, 9910, dev)
    st, ref = net.init_buffers(S, dev), net.init_buffers(S, dev)
    hist = net.target_history(st, 8)
    with torch.no_grad():
        for t in range(5):
            tick(net, st, clips, t, e, [A, -1], [0, 2], hist)
            tick(net, ref, clips, t, e, [A, B], [0, 2])
        others = [r for r in range(S) if r not in (A, B)]
        st._rec()[others] = SENTINEL
        before = su.bits(st._rec()).clone()
        y, used = net.join_targets(st, su.i32([B, X], dev), su.i32([A, S + 3], dev), e[[1, 1]], history=hist, frames=0)
        torch.cuda.synchronize()
    assert used.tolist() == [0, 0] and y.shape == (2, 2, 0)
    a = su.bits(st._rec())
    for r in [A] + others:
        assert torch.equal(a[r], before[r]), r
    L = st.lay
    assert st.stream_pos()[B] == 5
    assert int(st._clocks()[1][B]) == 0
    assert not bool(st._rec()[B, L["st_conv"]:].any()), "a cold join computed past the gate memo"
    assert torch.equal(gate(st, B), gate(ref, B))


# ---- 5. drops ----------------------------------------------------------------------------------------------------------
def test_dropping_a_non_lead_row(model, dev):
    """{A, B, C} for 6 hops, then C's row is left out (record -1): A's and B's outputs stay bit for bit those of the twin
    that keeps C."""
    net, _ = model
    clips, _ = su.clips(1, 10, 9950, dev)
    e = su.emb(3, 9960, dev)
    st = net.init_buffers(4, dev)
    with torch.no_grad():
        for t in range(6):
            tick(net, st, clips, t, e, [0, 1, 2], [0, 3])
        twin = su.copy(net, st)
        for t in range(6, 10):
            y = tick(net, st, clips, t, e, [0, 1, -1], [0, 3])
            y_ref = tick(net, twin, clips, t, e, [0, 1, 2], [0, 3])
            torch.cuda.synchronize()
            assert torch.equal(su.bits(y[:2]), su.bits(y_ref[:2])), t


def test_move_lead_then_drop_the_old_lead(model, dev):
    """{A} with a history, B joins warm (its tails' parity differs from A's), both advance 3 hops; then move_lead(A, B) and
    A's row dropped gives B outputs bit for bit those of the twin that keeps A as the lead, and the history's ring moves
    with it.  Clocks that differ are refused."""
    net, _ = model
    A, B, F = 0, 1, 16
    clips, _ = su.clips(1, 20, 9970, dev)
    e = su.emb(2, 9980, dev)
    st = net.init_buffers(3, dev)
    hist = net.target_history(st, F)
    with torch.no_grad():
        for t in range(10):
            tick(net, st, clips, t, e, [A, -1], [0, 2], hist)
        net.join_targets(st, [B], [A], e[[1]], history=hist)
        for t in range(10, 13):
            tick(net, st, clips, t, e, [A, B], [0, 2], hist)
        torch.cuda.synchronize()
        calls = st._clocks()[1].tolist()
        assert calls[A] % 2 != calls[B] % 2, calls
        with pytest.raises(ValueError, match="different clocks"):
            st.move_lead([A], [2])
        twin, twin_hist = su.copy(net, st), hist.buf.clone()
        st.move_lead([A], [B])
        hist.move([A], [B])
        assert torch.equal(hist.buf[B], twin_hist[A]), "the ring did not move with the lead"
        eb = e[[1, 0]].contiguous()
        for t in range(13, 20):
            y = tick(net, st, clips, t, eb, [B, -1], [0, 2], hist)
            y_ref = tick(net, twin, clips, t, e, [A, B], [0, 2])
            torch.cuda.synchronize()
            assert torch.equal(su.bits(y[0]), su.bits(y_ref[1])), t
    assert st.stream_pos()[B] == twin.stream_pos()[A] == 20


# ---- 6. graphs -------------------------------------------------------------------------------------------------------
def test_graphs_with_lists_rewritten(model, dev):
    """A rows tick with a history and a join, each with L2H_FLAG_GRAPH on fixed buffers whose lists are rewritten in place,
    equal the same calls launched directly on a twin state and history, bit for bit (y, used, state, history)."""
    net, _ = model
    n, R, S, F, T = 2, 4, 8, 8, 1
    clips, _ = su.clips(n, 12, 9990, dev)
    e = su.emb(R, 9995, dev)
    xbuf = torch.empty(n, 2, HOP * T + 64, device=dev)
    rec_b, off_b = torch.empty(R, dtype=torch.int32, device=dev), su.i32([0, 2, 4], dev)
    yg, yd = torch.empty(R, 2, HOP, device=dev), torch.empty(R, 2, HOP, device=dev)
    jr, jl = torch.empty(2, dtype=torch.int32, device=dev), torch.empty(2, dtype=torch.int32, device=dev)
    jy, jyd = torch.empty(2, 2, HOP * 4, device=dev), torch.empty(2, 2, HOP * 4, device=dev)
    ju, jud = torch.empty(2, dtype=torch.int32, device=dev), torch.empty(2, dtype=torch.int32, device=dev)
    sg, sd = net.init_buffers(S, dev), net.init_buffers(S, dev)
    hg, hd = net.target_history(sg, F), net.target_history(sd, F)
    layouts = [([0, -1, 1, -1], [2, 3]), ([2, 0, 1, -1], [4, 5])]      # ticks, then the records that join leads 0 and 1
    with torch.no_grad():
        for phase, (recs, joiners) in enumerate(layouts):
            rec_b.copy_(su.i32(recs, dev))
            for t in range(6 * phase, 6 * phase + 6):
                xbuf.copy_(torch.stack([su.chunk(clips[i], t) for i in range(n)]))
                yg.fill_(SENTINEL)
                yd.fill_(SENTINEL)
                net._launch("targets_rows", xbuf, e, sg, yg, T, L2H_FLAG_GRAPH, slots=rec_b, offsets=off_b, history=hg)
                net._launch("targets_rows", xbuf, e, sd, yd, T, slots=rec_b, offsets=off_b, history=hd)
                torch.cuda.synchronize()
                assert torch.equal(su.bits(yg), su.bits(yd)), t
            jr.copy_(su.i32(joiners, dev))
            jl.copy_(su.i32([recs[0] if recs[0] >= 0 else 0, recs[2]], dev))
            jy.fill_(SENTINEL)
            jyd.fill_(SENTINEL)
            net.join_targets(sg, jr, jl, e[:2], history=hg, frames=4, out=jy, used=ju, flags=L2H_FLAG_GRAPH)
            net.join_targets(sd, jr, jl, e[:2], history=hd, frames=4, out=jyd, used=jud)
            torch.cuda.synchronize()
            assert ju.tolist() == jud.tolist() == [4, 4]
            assert torch.equal(su.bits(jy), su.bits(jyd)), phase
            assert torch.equal(su.bits(sg.buf), su.bits(sd.buf)), phase
            assert torch.equal(su.bits(hg.buf), su.bits(hd.buf)), phase


# ---- a ring shorter than a tick, and one-frame joins ------------------------------------------------------------------
def test_ring_shorter_than_the_tick(model, dev):
    """Ragged T = 3 ticks (h in {0, 1, 3}) into a 2-frame history: each lead's ring holds exactly its last 2 frames, those a
    16-frame history of the same ticks holds; a 2-frame join from it equals the join from the 16-frame history, bit for bit
    (y, used, state)."""
    net, _ = model
    n, K, T, F = 3, 2, 3, 2
    R, S = n * K, n * K + n
    clips, _ = su.clips(n, 4 * T, 9150, dev)
    e = su.emb(S, 9160, dev)
    recs = list(range(R))
    off = [i * K for i in range(n + 1)]
    st, twin = net.init_buffers(S, dev), net.init_buffers(S, dev)
    short, long_ = net.target_history(st, F), net.target_history(twin, 16)
    fed = [0] * n
    with torch.no_grad():
        for c in range(3):
            hops = su.hop_mix(n, T, 9170 + c)
            x = torch.stack([su.chunk(clips[i], fed[i], T) for i in range(n)]).contiguous()
            for s, h in ((st, short), (twin, long_)):
                net.advance_target_rows(x, e[:R], s, su.i32(recs, dev), su.i32(off, dev), hops=su.i32(hops, dev), history=h)
            fed = [f + h for f, h in zip(fed, hops)]
        torch.cuda.synchronize()
        assert torch.equal(su.bits(st.buf), su.bits(twin.buf))
        for i in range(n):
            lead = recs[i * K]
            for fr in range(max(0, fed[i] - F), fed[i]):
                assert torch.equal(su.bits(short.buf[lead, fr % F]), su.bits(long_.buf[lead, fr])), (i, fr)
        joiners, leads = list(range(R, S)), [recs[i * K] for i in range(n)]
        ys, us = [], []
        for s, h in ((st, short), (twin, long_)):
            y = torch.full((n, 2, HOP * F), SENTINEL, device=dev)
            _, u = net.join_targets(s, joiners, leads, e[R:], history=h, frames=F, out=y)
            ys.append(y)
            us.append(u)
        torch.cuda.synchronize()
    assert us[0].tolist() == us[1].tolist() == [min(F, f) for f in fed]
    assert torch.equal(su.bits(ys[0]), su.bits(ys[1]))
    assert torch.equal(su.bits(st.buf), su.bits(twin.buf))


@pytest.mark.parametrize("n", [pytest.param(1, id="fused-one-hop"), pytest.param(22, id="tensor-core-mid")])
def test_one_frame_join(model, dev, n):
    """A join replaying one frame (the one-hop forms of the join chain) against a cold join one hop earlier plus one live
    tick: B's record and the join's y within 1e-4 relative L2; A's records bit for bit equal."""
    net, _ = model
    R, S = 2 * n, 2 * n + 1
    A, B = list(range(0, R, 2)), list(range(1, R, 2))
    clips, _ = su.clips(n, 5, 9180 + n, dev)
    e = su.emb(R, 9190 + n, dev)
    off = [2 * i for i in range(n + 1)]
    solo = [r if r in A else -1 for r in range(R)]
    st = net.init_buffers(S, dev)
    hist = net.target_history(st, 8)
    with torch.no_grad():
        for t in range(4):
            tick(net, st, clips, t, e, solo, off, hist)
        twin = su.copy(net, st)
        tick(net, st, clips, 4, e, solo, off, hist)
        y_join, used = net.join_targets(st, B, A, e[B], history=hist, frames=1)
        net.join_targets(twin, B, A, e[B])
        y_ref = tick(net, twin, clips, 4, e, list(range(R)), off)
        torch.cuda.synchronize()
    assert used.tolist() == [1] * n
    assert st.stream_pos()[:R] == twin.stream_pos()[:R] == [5] * R
    for a in A:
        assert torch.equal(su.bits(st._rec()[a]), su.bits(twin._rec()[a])), a
    for b in B:
        assert rs.rel_l2(record_ref(st, b), record_ref(twin, b)) <= BOUND, b
    assert rs.rel_l2(y_join.cpu(), y_ref[B].cpu()) <= BOUND
