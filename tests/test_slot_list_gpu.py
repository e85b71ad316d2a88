"""One-hop calls over a list of a state's records (Net.predict(slots=) / l2h_sep_forward_slots).  The oracle is the API
that existed before: copy the listed records into a dense state of n streams (copy_streams_from), run a plain one-hop
predict there and copy them back.  A slot-list call runs the kernel form of a dense call of n streams, so it must equal
that bit for bit, in every form: n = 2 with the fused one-hop tail, n = 2 with fused_tail = 0 (separate kernels), n = 16
(the mid section split in three kernels) and n = 24 (the tensor-core chain, h gathered from the listed records)."""
import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import synth
from oracle import restate as rs
import serving_util as su
from serving_util import HOP, LA, L2H_FLAG_GRAPH, dev, model  # noqa: F401

pytestmark = pytest.mark.gpu
# (records in the state, listed rows per call, fused_tail)
FORMS = [pytest.param((40, 2, 1), id="n2-fused"), pytest.param((40, 2, 0), id="n2-separate"),
         pytest.param((40, 16, 1), id="n16-mid-split"), pytest.param((64, 24, 1), id="n24-tc")]


@pytest.fixture(params=FORMS)
def form(request, model):
    """(net, sd, S, n): the network switched to the kernel form under test for the test's duration."""
    S, n, fused = request.param
    net, sd = model
    with su.switched(net, {"fused_tail": fused}):
        yield net, sd, S, n


def test_slots_equal_copy_run_copy_back(form, dev):
    """12 hops, each over a different unsorted subset: y, every listed record (clock included) and the unlisted records
    (untouched) equal the copy / dense predict / copy back oracle bit for bit."""
    net, _, S, n = form
    T = 12
    clips, _ = su.clips(S, T, 2100, dev)
    e = su.emb(S, 2200, dev)
    got, ref = net.init_buffers(S, dev), net.init_buffers(S, dev)
    dense = net.init_buffers(n, dev)
    fed = [0] * S
    with torch.no_grad():
        for t, sl in enumerate(su.subsets(S, n, T, 2300)):
            x = torch.stack([su.chunk(clips[s], fed[s]) for s in sl])
            before = got._rec().clone()
            y, _ = net.predict(x, e[sl], got, pad=False, slots=sl)
            y_ref = su.oracle(net, ref, sl, x, e[sl], dense)
            for s in sl:
                fed[s] += 1
            assert torch.equal(y, y_ref), f"hop {t}: y"
            unlisted = [s for s in range(S) if s not in sl]
            assert torch.equal(su.bits(got._rec()[unlisted]), su.bits(before[unlisted])), f"hop {t}: an unlisted record changed"
            assert torch.equal(su.records(got), su.records(ref)), f"hop {t}: records"
    assert got.stream_pos() == fed and got.header() == (T, T)


def test_identity_list_equals_dense_predict(form, dev):
    """slots = 0 .. n-1 (as a CUDA int32 tensor, used in place) over a state of n records is a plain predict."""
    net, _, _, n = form
    clips, _ = su.clips(n, 3, 2400, dev)
    e = su.emb(n, 2500, dev)
    a, b = net.init_buffers(n, dev), net.init_buffers(n, dev)
    ident = torch.arange(n, dtype=torch.int32, device=dev)
    with torch.no_grad():
        for t in range(3):
            x = clips[..., HOP * t:HOP * t + HOP + LA]
            ya, _ = net.predict(x, e, a, pad=False, slots=ident)
            yb, _ = net.predict(x, e, b, pad=False)
            assert torch.equal(ya, yb), t
    assert torch.equal(su.bits(a.buf), su.bits(b.buf))


def test_entries_outside_the_state_store_nothing(form, dev):
    """Rows whose entry lies outside [0, S) are computed but leave every record and their NaN-filled y row untouched; the
    other rows equal the same call with those entries pointing at spare records of a copy of the state."""
    net, _, S, n = form
    clips, _ = su.clips(S, 4, 2600, dev)
    e = su.emb(S, 2700, dev)
    st = net.init_buffers(S, dev)
    warm = su.subsets(S, n, 3, 2800)
    with torch.no_grad():
        for t, sl in enumerate(warm):        # records with history and different clocks
            net.predict(torch.stack([su.chunk(clips[s], t) for s in sl]), e[sl], st, pad=False, slots=sl)
    sl = su.subsets(S, n, 1, 2900)[0]
    bad = {0: -1, n - 1: S + 3} if n > 2 else {0: -1}
    spare = [s for s in range(S) if s not in sl][:len(bad)]
    with_bad = [bad.get(i, s) for i, s in enumerate(sl)]
    with_spare = list(with_bad)
    for i, sp in zip(bad, spare):
        with_spare[i] = sp
    x = torch.stack([su.chunk(clips[s], 3) for s in sl])
    ee = e[sl].contiguous()
    net._sync_weights(dev)
    twin = net.init_buffers(S, dev)
    twin.buf.copy_(st.buf)
    before = st._rec().clone()
    y = torch.full((n, 2, HOP), float("nan"), device=dev)
    y_twin = torch.full_like(y, float("nan"))
    net._launch("slots", x, ee, st, y, 1, slots=torch.tensor(with_bad, dtype=torch.int32, device=dev))
    net._launch("slots", x, ee, twin, y_twin, 1, slots=torch.tensor(with_spare, dtype=torch.int32, device=dev))
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
    assert [st.stream_pos()[s] for s in spare] == [twin.stream_pos()[s] - 1 for s in spare]


def test_graph_replay_with_list_rewritten_in_place(form, dev):
    """With L2H_FLAG_GRAPH the list, the inputs and the embeddings are rewritten in place every hop and one cached graph
    is replayed: y and the whole state equal direct calls."""
    net, _, S, n = form
    T = 6
    clips, _ = su.clips(S, T, 3000, dev)
    e = su.emb(S, 3100, dev)
    net._sync_weights(dev)
    xbuf, ebuf = torch.empty(n, 2, HOP + LA, device=dev), torch.empty(n, 256, device=dev)
    slots = torch.empty(n, dtype=torch.int32, device=dev)
    yg, yd = torch.empty(n, 2, HOP, device=dev), torch.empty(n, 2, HOP, device=dev)
    sg, sdir = net.init_buffers(S, dev), net.init_buffers(S, dev)
    fed = [0] * S
    for t, sl in enumerate(su.subsets(S, n, T, 3200)):
        xbuf.copy_(torch.stack([su.chunk(clips[s], fed[s]) for s in sl]))
        ebuf.copy_(e[sl])
        slots.copy_(torch.tensor(sl, dtype=torch.int32))
        net._launch("slots", xbuf, ebuf, sg, yg, 1, L2H_FLAG_GRAPH, slots=slots)
        net._launch("slots", xbuf, ebuf, sdir, yd, 1, slots=slots)
        for s in sl:
            fed[s] += 1
        assert torch.equal(yg, yd), t
    assert torch.equal(su.bits(sg.buf), su.bits(sdir.buf))


def test_listed_stream_vs_oracle(form, dev):
    """A stream listed on 16 of 20 hops, among others, against the reference implementation fed the chunks it got: its
    output and its state (exported with to_reference() from a copy of its record) within the 1e-3 gate."""
    net, sd, S, n = form
    s, T = S - 1, 20
    skipped = {2, 9, 10, 15}
    n_fed = T - len(skipped)
    x_cpu, tgt = synth.mixture(1, HOP * n_fed, seed0=3300)
    xc = F.pad(x_cpu, (0, LA)).to(dev)
    others, _ = su.clips(S, T, 3400, dev)
    e = su.emb(S, 3500, dev)
    st = net.init_buffers(S, dev)
    got, fed = [], 0
    with torch.no_grad():
        for t, sl in enumerate(su.subsets(S - 1, n, T, 3600)):
            if t not in skipped:
                sl[t % n] = s
            x = torch.stack([su.chunk(xc[0], fed) if b == s else su.chunk(others[b], t) for b in sl])
            y, _ = net.predict(x, e[sl], st, pad=False, slots=sl)
            if t not in skipped:
                got.append(y[t % n])
                fed += 1
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
