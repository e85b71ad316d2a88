"""Several targets per mixture in one call (l2h_sep_forward_targets, Net.predict_targets / forward_targets).

The oracle is a dense call of batch*K streams with every mixture repeated K times (x.repeat_interleave(K, 0)) and the
embeddings flattened, on a fresh state of batch*K records.  A targets call chooses every kernel form for its batch*K
target rows and runs block 0 in those forms over the mixtures, so its outputs and the parts of the state it owns must
equal the oracle bit for bit in every form.  The one named exception is the fused one-hop form (tail_kernel), where block
1's input projection runs as a rows GEMM instead of in block 0's tail kernel: there the gate is 1e-5 relative L2, the
repo's gate between the fused and the separate kernels.  The parts a targets call owns are everything except the conv
tails and block 0 of the non-lead records (record i*K + k, k > 0), which it never reads or writes."""
import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import synth
from oracle import restate as rs
import serving_util as su
from serving_util import HOP, LA, L2H_FLAG_GRAPH, dev, model  # noqa: F401

pytestmark = pytest.mark.gpu
# (mixtures, targets, hops per call, engine options, exact)
FORMS = [pytest.param((1, 2, 1, {}, False), id="fused-tail-1x2"),
         pytest.param((2, 3, 1, {}, False), id="fused-tail-2x3"),
         pytest.param((1, 2, 1, {"fused_tail": 0}, True), id="mid-kernel-1x2"),
         pytest.param((2, 3, 1, {"fused_tail": 0}, True), id="mid-kernel-2x3"),
         pytest.param((6, 2, 1, {"fused_tail": 0}, True), id="mid-split-6x2"),
         pytest.param((8, 3, 1, {}, True), id="tc-mid-8x3"),
         pytest.param((64, 3, 1, {}, True), id="tc-mid-64x3"),        # BiLSTM: several sequences per CTA (lstm_rec4_kernel)
         pytest.param((1, 2, 3, {}, True), id="T3-1x2"),
         pytest.param((1, 2, 3, {"back_many": 0}, True), id="T3-1x2-per-frame"),
         pytest.param((4, 2, 3, {}, True), id="T3-tc-lstm-rec-4x2"),
         pytest.param((16, 3, 2, {}, True), id="T2-tc-lstm-16x3"),
         pytest.param((16, 3, 2, {"fuse_ih": 1}, True), id="T2-tc-lstm-x-16x3")]


@pytest.fixture(params=FORMS)
def form(request, model):
    """(net, sd, B, K, T, exact): the network switched to the kernel form under test for the test's duration."""
    B, K, T, opts, exact = request.param
    net, sd = model
    with su.switched(net, opts):
        yield net, sd, B, K, T, exact


def _owned(st, K):
    """every record as bits, the regions a targets call does not own cleared"""
    r = su.bits(st._rec()).clone()
    r[su.foreign(st, K)] = 0
    return r


def _owned_values(st, K):
    r = st._rec().clone()
    r[su.foreign(st, K)] = 0
    return r


def _same(a, b, exact):
    if exact:
        return torch.equal(a, b)
    return rs.rel_l2(a.float().cpu(), b.float().cpu()) <= 1e-5


def test_targets_equal_duplicated_dense_call(form, dev):
    """4 consecutive calls: y and the owned part of every record equal the duplicated dense call's."""
    net, _, B, K, T, exact = form
    calls = 4
    clips, _ = su.clips(B, calls * T, 7100, dev)
    emb = su.embeds(B, K, 7200, dev)
    got, ref = net.init_buffers(B * K, dev), net.init_buffers(B * K, dev)
    with torch.no_grad():
        for c in range(calls):
            x = su.chunk(clips, c * T, T)
            y, _ = net.predict_targets(x, emb, got, pad=False)
            y_ref, _ = net.predict(x.repeat_interleave(K, 0), emb.reshape(B * K, 256), ref, pad=False)
            assert y.shape == (B, K, 2, HOP * T)
            assert _same(y.reshape(B * K, 2, -1), y_ref, exact), f"call {c}: y"
            if exact:
                assert torch.equal(_owned(got, K), _owned(ref, K)), f"call {c}: records"
            else:
                assert rs.rel_l2(_owned_values(got, K).cpu(), _owned_values(ref, K).cpu()) <= 1e-5, f"call {c}: records"
    assert got.stream_pos() == ref.stream_pos() == [calls * T] * (B * K)
    assert got.header() == ref.header()


@pytest.mark.parametrize("B, K, T, opts", [pytest.param(1, 3, 1, {}, id="fused-tail"),
                                           pytest.param(8, 3, 1, {}, id="tc-mid"),
                                           pytest.param(2, 2, 3, {}, id="T3")])
def test_non_lead_regions_are_never_read(model, dev, B, K, T, opts):
    """NaN in the conv tails and block 0 of every non-lead record: the outputs stay finite and equal those of a state
    without the NaN, and those regions still hold NaN afterwards."""
    net, _ = model
    with su.switched(net, opts):
        clips, _ = su.clips(B, 3 * T, 7300, dev)
        emb = su.embeds(B, K, 7400, dev)
        clean, poisoned = net.init_buffers(B * K, dev), net.init_buffers(B * K, dev)
        foreign = su.foreign(poisoned, K)
        poisoned._rec()[foreign] = float("nan")
        with torch.no_grad():
            for c in range(3):
                x = su.chunk(clips, c * T, T)
                y, _ = net.predict_targets(x, emb, clean, pad=False)
                yp, _ = net.predict_targets(x, emb, poisoned, pad=False)
                assert bool(torch.isfinite(yp).all()), f"call {c}"
                assert torch.equal(yp, y), f"call {c}"
        assert bool(torch.isnan(poisoned._rec()[foreign]).all())
        assert torch.equal(_owned(poisoned, K), _owned(clean, K))


@pytest.mark.parametrize("T", [1, 3])
def test_one_target_is_forward(model, dev, T):
    """n_targets = 1 is l2h_sep_forward bit for bit: outputs and the whole state."""
    net, _ = model
    B = 3
    clips, _ = su.clips(B, 3 * T, 7500, dev)
    emb = su.embeds(B, 1, 7600, dev)
    got, ref = net.init_buffers(B, dev), net.init_buffers(B, dev)
    with torch.no_grad():
        for c in range(3):
            x = su.chunk(clips, c * T, T)
            y, _ = net.predict_targets(x, emb, got, pad=False)
            y_ref, _ = net.predict(x, emb[:, 0], ref, pad=False)
            assert torch.equal(y[:, 0], y_ref), f"call {c}"
    assert torch.equal(su.bits(got.buf), su.bits(ref.buf))


def test_streaming_equals_whole_clip(model, dev):
    """500 one-hop predict_targets calls equal forward_targets of the whole clip, at the streaming test's gate."""
    net, _ = model
    B, K, hops = 1, 2, 500
    x, _ = synth.mixture(B, HOP * hops, seed0=7700)
    x = x.to(dev)
    emb = su.embeds(B, K, 7800, dev)
    xp = F.pad(x, (0, LA))
    st = net.init_buffers(B * K, dev)
    with torch.no_grad():
        y = net.forward_targets(x, emb)
        ys = torch.cat([net.predict_targets(su.chunk(xp, t, 1), emb, st, pad=False)[0] for t in range(hops)], -1)
    assert y.shape == ys.shape == (B, K, 2, HOP * hops)
    assert rs.rel_l2(ys.cpu(), y.cpu()) < 1e-4


def test_embedding_change_touches_only_its_target(model, dev):
    """Changing one target's embedding mid-stream changes that target's output only: the other targets stay
    bit-identical to a run without the change."""
    net, _ = model
    B, K, calls = 2, 3, 8
    clips, _ = su.clips(B, calls, 7900, dev)
    emb = su.embeds(B, K, 8000, dev)
    emb2 = emb.clone()
    emb2[1, 2] = su.embeds(1, 1, 8100, dev)[0, 0]
    a, b = net.init_buffers(B * K, dev), net.init_buffers(B * K, dev)
    with torch.no_grad():
        for c in range(calls):
            x = su.chunk(clips, c, 1)
            ya, _ = net.predict_targets(x, emb, a, pad=False)
            yb, _ = net.predict_targets(x, emb if c < calls // 2 else emb2, b, pad=False)
            changed = torch.zeros(B, K, dtype=torch.bool)
            if c >= calls // 2:
                changed[1, 2] = True
                assert not torch.equal(ya[1, 2], yb[1, 2]), f"call {c}: the changed target"
            assert torch.equal(ya[~changed], yb[~changed]), f"call {c}: another target"


def test_group_reset_equals_fresh_group(model, dev):
    """reset_streams of a whole group and then continuing equals the group in a fresh state fed the same calls."""
    net, _ = model
    B, K = 2, 2
    clips, _ = su.clips(B, 10, 8200, dev)
    emb = su.embeds(B, K, 8300, dev)
    st = net.init_buffers(B * K, dev)
    fresh = net.init_buffers(B * K, dev)
    group = [K * 1 + k for k in range(K)]
    with torch.no_grad():
        for c in range(4):
            net.predict_targets(su.chunk(clips, c, 1), emb, st, pad=False)
        st.reset_streams(group)
        for c in range(4):
            x = su.chunk(clips, 4 + c, 1)
            x_fresh = x.clone()
            x_fresh[1] = su.chunk(clips, c, 1)[1]          # group 1 starts from the clip's beginning again
            y, _ = net.predict_targets(x_fresh, emb, st, pad=False)
            y_ref, _ = net.predict_targets(x_fresh, emb, fresh, pad=False)
            assert torch.equal(y[1], y_ref[1]), f"call {c}"
    assert torch.equal(_owned(st, K)[group], _owned(fresh, K)[group])


@pytest.mark.parametrize("B, K, T", [pytest.param(2, 2, 1, id="one-hop"), pytest.param(8, 3, 1, id="tc-mid"),
                                     pytest.param(2, 2, 3, id="T3")])
def test_graph_replay_equals_direct_launches(model, dev, B, K, T):
    """With L2H_FLAG_GRAPH and the input and embedding buffers rewritten in place every call, the replayed graph equals
    direct launches: outputs and the whole state."""
    net, _ = model
    calls = 4
    clips, _ = su.clips(B, calls * T, 8400, dev)
    net._sync_weights(dev)
    xbuf, ebuf = torch.empty(B, 2, HOP * T + LA, device=dev), torch.empty(B * K, 256, device=dev)
    yg, yd = torch.empty(B, K, 2, HOP * T, device=dev), torch.empty(B, K, 2, HOP * T, device=dev)
    sg, sdir = net.init_buffers(B * K, dev), net.init_buffers(B * K, dev)
    for c in range(calls):
        xbuf.copy_(su.chunk(clips, c * T, T))
        ebuf.copy_(su.embeds(B, K, 8500 + 10 * (c // 2), dev).reshape(B * K, 256))      # the embeddings change once
        net._launch("targets", xbuf, ebuf, sg, yg, T, L2H_FLAG_GRAPH, K=K)
        net._launch("targets", xbuf, ebuf, sdir, yd, T, K=K)
        assert torch.equal(yg, yd), c
    assert torch.equal(su.bits(sg.buf), su.bits(sdir.buf))


def test_offline_batch_split_equals_duplicated_forward(model, dev):
    """forward_targets of 4 s clips, 2 mixtures x 2 targets, split into one mixture per launch, equals the duplicated
    dense forward split the same way (the same target rows per launch)."""
    net, _ = model
    B, K = 2, 2
    x, _ = synth.mixture(B, 64000, seed0=8600)
    x = x.to(dev)
    emb = su.embeds(B, K, 8700, dev)
    keep = net.max_frames_per_launch
    net.max_frames_per_launch = 500 * K           # one mixture (K target rows of 500 frames) per launch
    try:
        with torch.no_grad():
            y = net.forward_targets(x, emb)
            y_ref = net(x.repeat_interleave(K, 0), emb.reshape(B * K, 1, 256))
    finally:
        net.max_frames_per_launch = keep
    assert y.shape == (B, K, 2, 64000)
    assert torch.equal(y.reshape(B * K, 2, -1), y_ref)


def test_targets_vs_oracle(model, dev):
    """Against the reference restatement run on each (mixture, target): within 1e-3 relative L2 and 0.1 dB SI-SDR."""
    net, sd = model
    B, K = 2, 2
    x, tgt = synth.mixture(B, HOP * 40, seed0=8800)
    emb = su.embeds(B, K, 8900, dev)
    with torch.no_grad():
        y = net.forward_targets(x.to(dev), emb).cpu()
    for i in range(B):
        for k in range(K):
            y_ref = rs.sep_forward(sd, x[i:i + 1], emb[i, k].cpu()[None, None])
            assert rs.rel_l2(y[i, k][None], y_ref) <= 1e-3, (i, k)
            d = (rs.si_sdr(y[i, k][None], tgt[i:i + 1]) - rs.si_sdr(y_ref, tgt[i:i + 1])).abs().max()
            assert float(d) <= 0.1, (i, k)
