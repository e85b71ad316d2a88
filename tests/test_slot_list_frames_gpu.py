"""Multi-hop calls over a list of a state's records (Net.advance_slots / l2h_sep_forward_slots_frames).  The oracle is the
one of tests/test_slot_list_gpu.py: copy the listed records into a dense state of n streams (copy_streams_from), run a
plain T-hop predict(pad=False) there and copy them back.  A slot-list call runs the kernel form of a dense call of n
streams and T hops, with the inter-LSTM's carried (h, c) gathered from the listed records and scattered back, so it must
equal that bit for bit in every form: CUDA-core rows (n = 2, T = 3 and n = 4, T = 5, with the multi-frame front / back
walkers and without), the tensor-core chain with the lstm_rec inter recurrence (n = 8, T = 3: 2328 rows) and with the
tensor-core recurrence tc_lstm (n = 48, T = 2: 4656 sequences), alone and with the input projection fused (fuse_ih)."""
import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import synth
from oracle import restate as rs
import serving_util as su
from serving_util import HOP, LA, L2H_FLAG_GRAPH, dev, model  # noqa: F401

pytestmark = pytest.mark.gpu
# (records in the state, listed rows per call, hops per call, engine options)
FORMS = [pytest.param((12, 2, 3, {"back_many": 1}), id="n2-T3"),
         pytest.param((12, 2, 3, {"back_many": 0}), id="n2-T3-per-frame"),
         pytest.param((12, 4, 5, {"back_many": 1}), id="n4-T5"),
         pytest.param((12, 4, 5, {"back_many": 0}), id="n4-T5-per-frame"),
         pytest.param((16, 8, 3, {}), id="n8-T3-tc"),
         pytest.param((56, 48, 2, {}), id="n48-T2-tc-lstm"),
         pytest.param((56, 48, 2, {"fuse_ih": 1}), id="n48-T2-tc-lstm-x")]


@pytest.fixture(params=FORMS)
def form(request, model):
    """(net, sd, S, n, T): the network switched to the kernel form under test for the test's duration."""
    S, n, T, opts = request.param
    net, sd = model
    with su.switched(net, opts):
        yield net, sd, S, n, T


def test_slots_frames_equal_copy_run_copy_back(form, dev):
    """6 calls of T hops, each over a different unsorted subset: y, every listed record (clock included) and the unlisted
    records (untouched) equal the copy / dense T-hop predict / copy back oracle bit for bit."""
    net, _, S, n, T = form
    calls = 6
    clips, _ = su.clips(S, calls * T, 4100, dev)
    e = su.emb(S, 4200, dev)
    got, ref = net.init_buffers(S, dev), net.init_buffers(S, dev)
    fed = [0] * S
    with torch.no_grad():
        for c, sl in enumerate(su.subsets(S, n, calls, 4300)):
            x = torch.stack([su.chunk(clips[s], fed[s], T) for s in sl])
            before = got._rec().clone()
            y = net.advance_slots(x, e[sl], got, sl)
            y_ref = su.oracle(net, ref, sl, x, e[sl])
            for s in sl:
                fed[s] += T
            assert y.shape == (n, 2, HOP * T)
            assert torch.equal(y, y_ref), f"call {c}: y"
            unlisted = [s for s in range(S) if s not in sl]
            assert torch.equal(su.bits(got._rec()[unlisted]), su.bits(before[unlisted])), f"call {c}: an unlisted record changed"
            assert torch.equal(su.records(got), su.records(ref)), f"call {c}: records"
    assert got.stream_pos() == fed and got.header() == (calls * T, calls)


@pytest.mark.parametrize("S, n, opts", [pytest.param(10, 4, {}, id="n4"), pytest.param(16, 8, {}, id="n8-tc"),
                                        pytest.param(10, 4, {"back_many": 0}, id="n4-per-frame")])
def test_mixed_clocks_and_hop_counts(model, dev, S, n, opts):
    """Records with different clocks, calls of 1, 2 and 5 hops interleaved with one-hop predict(slots=) calls on the same
    records, calls whose hops cross a multiple of the 56-slot K/V ring, and records reset mid-test: every call equals
    the oracle bit for bit."""
    net, _ = model
    with su.switched(net, opts):
        clips, _ = su.clips(S, 120, 4400, dev)
        e = su.emb(S, 4500, dev)
        got = net.init_buffers(S, dev)
        warm = 50 + torch.arange(S) % 5                    # clocks 50 .. 54: 2 to 6 hops below the ring's wrap
        fed = warm.tolist()
        with torch.no_grad():
            for s in range(S):                              # one dense multi-hop call per record, in a state of one
                one = net.init_buffers(1, dev)
                net.predict(su.chunk(clips[s], 0, fed[s])[None], e[s:s + 1], one, pad=False)
                got.copy_streams_from(one, [0], [s])
            ref = net.init_buffers(S, dev)
            ref.buf.copy_(got.buf)
            # (hops, how): "p" = predict(slots=), "a" = advance_slots
            plan = [(2, "a"), (5, "a"), (1, "p"), (5, "a"), (1, "a"), (2, "a"), ("reset", None), (5, "a"), (1, "p"),
                    (5, "a"), (2, "a"), (1, "p"), (5, "a")]
            lists = iter(su.subsets(S, n, len(plan), 4600))
            frames = calls = 0
            for step, (T, how) in enumerate(plan):
                sl = next(lists)
                if T == "reset":
                    got.reset_streams(sl[:2])
                    ref.reset_streams(sl[:2])
                    for s in sl[:2]:
                        fed[s] = 0
                    continue
                x = torch.stack([su.chunk(clips[s], fed[s], T) for s in sl])
                if how == "p":
                    y, _ = net.predict(x, e[sl], got, pad=False, slots=sl)
                else:
                    y = net.advance_slots(x, e[sl], got, sl)
                y_ref = su.oracle(net, ref, sl, x, e[sl])
                for s in sl:
                    fed[s] += T
                frames, calls = frames + T, calls + 1
                assert torch.equal(y, y_ref), f"step {step}: y"
                assert torch.equal(su.records(got), su.records(ref)), f"step {step}: records"
        assert got.stream_pos() == fed and max(fed) > 56
        assert got.header() == (frames, calls)          # copying records in leaves the header as it was


def test_entries_outside_the_state_store_nothing(form, dev):
    """Rows whose entry lies outside [0, S) are computed from record 0 but leave every record and their NaN-filled y rows
    untouched for all of their hops; the other rows equal the same call with those entries pointing at spare records of
    a copy of the state."""
    net, _, S, n, T = form
    clips, _ = su.clips(S, 4 * T, 4700, dev)
    e = su.emb(S, 4800, dev)
    st = net.init_buffers(S, dev)
    with torch.no_grad():
        for c, sl in enumerate(su.subsets(S, n, 3, 4900)):     # records with history and different clocks
            net.advance_slots(torch.stack([su.chunk(clips[s], c * T, T) for s in sl]), e[sl], st, sl)
    sl = su.subsets(S, n, 1, 5000)[0]
    bad = {0: -1, n - 1: S + 3} if n > 2 else {0: -1}
    spare = [s for s in range(S) if s not in sl][:len(bad)]
    with_bad = [bad.get(i, s) for i, s in enumerate(sl)]
    with_spare = list(with_bad)
    for i, sp in zip(bad, spare):
        with_spare[i] = sp
    x = torch.stack([su.chunk(clips[s], 3 * T, T) for s in sl])
    ee = e[sl].contiguous()
    net._sync_weights(dev)
    twin = net.init_buffers(S, dev)
    twin.buf.copy_(st.buf)
    before = st._rec().clone()
    y = torch.full((n, 2, HOP * T), float("nan"), device=dev)
    y_twin = torch.full_like(y, float("nan"))
    net._launch("slots_frames", x, ee, st, y, T, slots=torch.tensor(with_bad, dtype=torch.int32, device=dev))
    net._launch("slots_frames", x, ee, twin, y_twin, T, slots=torch.tensor(with_spare, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()
    stored = [s for s in with_bad if 0 <= s < S]
    for i in range(n):
        if i in bad:
            assert bool(torch.isnan(y[i]).all()), f"row {i} (entry {with_bad[i]}) wrote y"
        else:
            assert torch.equal(y[i], y_twin[i]), f"row {i}"
            assert not bool(torch.isnan(y[i]).any())
    others = [s for s in range(S) if s not in stored]
    assert torch.equal(su.bits(st._rec()[others]), su.bits(before[others])), "a record not listed (or listed out of range) changed"
    assert torch.equal(su.bits(st._rec()[stored]), su.bits(twin._rec()[stored]))
    assert [st.stream_pos()[s] for s in spare] == [twin.stream_pos()[s] - T for s in spare]


def test_graph_replay_with_list_rewritten_in_place(form, dev):
    """With L2H_FLAG_GRAPH the list, the inputs and the embeddings are rewritten in place every call and one cached graph
    is replayed: y and the whole state equal direct calls."""
    net, _, S, n, T = form
    calls = 4
    clips, _ = su.clips(S, calls * T, 5100, dev)
    e = su.emb(S, 5200, dev)
    net._sync_weights(dev)
    xbuf, ebuf = torch.empty(n, 2, HOP * T + LA, device=dev), torch.empty(n, 256, device=dev)
    slots = torch.empty(n, dtype=torch.int32, device=dev)
    yg, yd = torch.empty(n, 2, HOP * T, device=dev), torch.empty(n, 2, HOP * T, device=dev)
    sg, sdir = net.init_buffers(S, dev), net.init_buffers(S, dev)
    fed = [0] * S
    for c, sl in enumerate(su.subsets(S, n, calls, 5300)):
        xbuf.copy_(torch.stack([su.chunk(clips[s], fed[s], T) for s in sl]))
        ebuf.copy_(e[sl])
        slots.copy_(torch.tensor(sl, dtype=torch.int32))
        net._launch("slots_frames", xbuf, ebuf, sg, yg, T, L2H_FLAG_GRAPH, slots=slots)
        net._launch("slots_frames", xbuf, ebuf, sdir, yd, T, slots=slots)
        for s in sl:
            fed[s] += T
        assert torch.equal(yg, yd), c
    assert torch.equal(su.bits(sg.buf), su.bits(sdir.buf))


@pytest.mark.parametrize("S, n", [pytest.param(6, 2, id="n2"), pytest.param(16, 8, id="n8-tc")])
def test_listed_stream_vs_oracle(model, dev, S, n):
    """A stream advanced by multi-hop slot calls of 3, 2, 5, 1 and 4 hops, skipping some calls, among others, against the
    reference implementation fed the chunks it got: its output and its state (exported with to_reference() from a copy
    of its record) within the 1e-3 gate."""
    net, sd = model
    s = S - 1
    plan = [3, 2, 5, 2, 1, 4, 3, 2]
    skipped = {1, 5}
    n_fed = sum(T for c, T in enumerate(plan) if c not in skipped)
    x_cpu, tgt = synth.mixture(1, HOP * n_fed, seed0=5400)
    xc = F.pad(x_cpu, (0, LA)).to(dev)
    others, _ = su.clips(S, sum(plan), 5500, dev)
    e = su.emb(S, 5600, dev)
    st = net.init_buffers(S, dev)
    got, fed, t0 = [], 0, 0
    with torch.no_grad():
        for c, (T, sl) in enumerate(zip(plan, su.subsets(S - 1, n, len(plan), 5700))):
            if c not in skipped:
                sl[c % n] = s
            x = torch.stack([su.chunk(xc[0], fed, T) if b == s else su.chunk(others[b], t0, T) for b in sl])
            y = net.advance_slots(x, e[sl], st, sl)
            if c not in skipped:
                got.append(y[c % n])
                fed += T
            t0 += T
    y = torch.cat(got, -1).cpu()[None]
    y_ref, st_ref = rs.sep_predict(sd, x_cpu, e[s:s + 1].cpu(), rs.sep_init_state(sd, 1))
    assert rs.rel_l2(y, y_ref) <= 1e-3
    assert float((rs.si_sdr(y, tgt) - rs.si_sdr(y_ref, tgt)).abs().max()) <= 0.1
    one = net.init_buffers(1, dev)
    one.copy_streams_from(st, [s], [0])
    exported = one.to_reference()
    for k in ("conv_buf", "deconv_buf", "istft_buf"):
        assert rs.rel_l2(exported[k].cpu(), st_ref[k]) <= 1e-3, k
    for i in range(3):
        for k in ("K_buf", "V_buf", "h0", "c0"):
            a, b = exported["gridnet_bufs"][f"buf{i}"][k].cpu(), st_ref["gridnet_bufs"][f"buf{i}"][k]
            assert rs.rel_l2(a, b) <= 1e-3, (i, k)
