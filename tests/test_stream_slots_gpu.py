"""Streams of one batched state on their own clocks: admitted into a running state (reset_streams), skipping hops
(predict(..., active=) / l2h_sep_forward_active) and moved between states (copy_streams_from).  The oracle of each
behaviour is bit-exact: the same stream run on its own in a state of the same batch size, where the kernel forms are the
same (B = 2: the fused one-hop tail; B = 2 with fused_tail = 0: the separate kernels; B = 32: the tensor-core chain)."""
import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import synth
from oracle import restate as rs
import serving_util as su
from serving_util import HOP, LA, dev, model  # noqa: F401

pytestmark = pytest.mark.gpu
FORMS = [pytest.param((2, 1), id="B2-fused"), pytest.param((2, 0), id="B2-separate"), pytest.param((32, 1), id="B32-tc")]


@pytest.fixture(params=FORMS)
def form(request, model):
    """(net, sd, B): the network switched to the kernel form under test for the test's duration."""
    B, fused = request.param
    net, sd = model
    with su.switched(net, {"fused_tail": fused}):
        yield net, sd, B


def _hop(net, st, x, e, active=None):
    with torch.no_grad():
        y, _ = net.predict(x, e, st, pad=False, active=active)
    return y


def _rec(st, b):
    return st._rec()[b].clone()


def test_admit_into_running_state(form, dev):
    """Stream X joins slot s at hop 40 and runs 70 hops (the 56-slot ring wraps; its window history is longer than the
    admission offset): it equals X run from hop 0 in slot s of a fresh state, and the other streams equal a run without
    the admission."""
    net, _, B = form
    s = B - 1
    other, _ = su.clips(B, 110, 100, dev)
    xc, _ = su.clips(1, 70, 200, dev)
    e_other, e_x = su.emb(B, 300, dev), su.emb(1, 400, dev)[0]

    def inputs(t, x_hop):            # slot s carries X's hop x_hop (None: its original stream's hop t)
        x = torch.stack([su.chunk(other[b], t) for b in range(B)])
        e = e_other.clone()
        if x_hop is not None:
            x[s], e[s] = su.chunk(xc[0], x_hop), e_x
        return x, e

    st_a, st_b = net.init_buffers(B, dev), net.init_buffers(B, dev)
    ya, yb = [], []
    for t in range(110):
        if t == 40:
            st_a.reset_streams([s])
        ya.append(_hop(net, st_a, *inputs(t, t - 40 if t >= 40 else None)))
        yb.append(_hop(net, st_b, *inputs(t, None)))
    st_c = net.init_buffers(B, dev)
    yc = [_hop(net, st_c, *inputs(40 + t, t)) for t in range(70)]
    torch.cuda.synchronize()
    for t in range(70):
        assert torch.equal(ya[40 + t][s], yc[t][s]), f"admitted stream, hop {t}"
    assert torch.equal(_rec(st_a, s), _rec(st_c, s))
    assert st_a.stream_pos()[s] == 70 and st_a.header() == (110, 110)
    for t in range(110):
        for b in range(B):
            if b != s or t < 40:
                assert torch.equal(ya[t][b], yb[t][b]), (t, b)
    for b in range(B):
        if b != s:
            assert torch.equal(_rec(st_a, b), _rec(st_b, b)), b


@pytest.mark.parametrize("graph", [False, True], ids=["direct", "graph"])
def test_skip_hops(form, dev, graph):
    """Stream X in slot s misses hops 3, 4, 17 and 60: across each its record does not change and its rows of y are not
    written; on the other hops its output equals X fed only the chunks it received, on its own fresh state.  With
    L2H_FLAG_GRAPH the mask is rewritten in place and the same cached graph (the same argument set) is replayed."""
    net, _, B = form
    s, skip, T = B // 2, {3, 4, 17, 60}, 70
    other, _ = su.clips(B, T, 500, dev)
    xc, _ = su.clips(1, T, 600, dev)
    e = su.emb(B, 700, dev)
    net._sync_weights(dev)
    xbuf = torch.empty(B, 2, HOP + LA, device=dev)
    ybuf = torch.empty(B, 2, HOP, device=dev)
    mask = torch.ones(B, dtype=torch.uint8, device=dev)
    flags = 2 if graph else 0
    st = net.init_buffers(B, dev)
    got, fed = [], 0
    for t in range(T):
        for b in range(B):
            xbuf[b] = su.chunk(xc[0], fed) if b == s else su.chunk(other[b], t)
        mask[s] = 0 if t in skip else 1
        ybuf.fill_(1234.5)
        before = _rec(st, s)
        net._launch("forward_active", xbuf, e, st, ybuf, 1, flags, mask=mask)
        if t in skip:
            assert torch.equal(_rec(st, s), before), f"record changed on skipped hop {t}"
            assert bool((ybuf[s] == 1234.5).all()), f"y written on skipped hop {t}"
        else:
            got.append(ybuf[s].clone())
            fed += 1
        assert not bool((ybuf[:s] == 1234.5).any()) and not bool((ybuf[s + 1:] == 1234.5).any())
    assert st.stream_pos()[s] == T - len(skip) and st.header() == (T, T)
    ref_st = net.init_buffers(B, dev)
    for j in range(fed):
        x = torch.stack([su.chunk(xc[0], j) if b == s else su.chunk(other[b], j) for b in range(B)])
        y = _hop(net, ref_st, x, e)
        assert torch.equal(got[j], y[s]), f"active hop {j}"
    assert torch.equal(_rec(st, s), _rec(ref_st, s))


def test_copy_between_states(form, dev):
    """A stream moved mid-run into a state whose header clock differs (built with load_reference) continues exactly as
    if never moved, also through a 5-frame call (the K/V history gather reads the stream's own clock), and that call
    agrees with five one-hop calls."""
    net, sd, B = form
    s = B - 1
    xo, _ = su.clips(B, 63, 800, dev)
    xp, _ = su.clips(B, 49, 900, dev)
    e1, e2 = su.emb(B, 1000, dev), su.emb(B, 1100, dev)
    s1 = net.init_buffers(B, dev)
    s2 = net.init_buffers(B, dev).load_reference(rs.sep_init_state(sd, B))
    for t in range(13):
        _hop(net, s1, xo[..., HOP * t:HOP * t + HOP + LA], e1)
    for t in range(4):
        _hop(net, s2, xp[..., HOP * t:HOP * t + HOP + LA], e2)
    s2.copy_streams_from(s1, [s], [s])
    e2[s] = e1[s]
    for t in range(13, 58):          # the moved stream crosses the ring wrap (frame 56) in its new state
        x2 = xp[..., HOP * (t - 9):HOP * (t - 9) + HOP + LA].clone()
        x2[s] = xo[s, :, HOP * t:HOP * t + HOP + LA]
        y1 = _hop(net, s1, xo[..., HOP * t:HOP * t + HOP + LA], e1)
        y2 = _hop(net, s2, x2, e2)
        assert torch.equal(y1[s], y2[s]), t
    assert s1.header() == (58, 58) and s2.header() == (98, 49) and s2.stream_pos()[s] == 58
    assert torch.equal(_rec(s1, s), _rec(s2, s))
    s3 = net.init_buffers(B, dev)
    s3.buf.copy_(s1.buf)
    x5 = xo[..., HOP * 58:HOP * 63 + LA]
    x5b = xp[..., :HOP * 5 + LA].clone()           # the other streams of s2 are not compared
    x5b[s] = x5[s]
    y1 = _hop(net, s1, x5, e1)
    y2 = _hop(net, s2, x5b, e2)
    assert torch.equal(y1[s], y2[s])
    assert torch.equal(_rec(s1, s), _rec(s2, s))
    y3 = torch.cat([_hop(net, s3, xo[..., HOP * t:HOP * t + HOP + LA], e1) for t in range(58, 63)], -1)
    assert rs.rel_l2(y1[s].cpu(), y3[s].cpu()) <= 1e-3


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_copy_between_devices(model):
    net, _ = model
    d0, d1 = torch.device("cuda", 0), torch.device("cuda", 1)
    xo, _ = su.clips(2, 20, 1200, d0)
    e = su.emb(2, 1300, d0)
    a = net.init_buffers(2, d0)
    for t in range(10):
        _hop(net, a, xo[..., HOP * t:HOP * t + HOP + LA], e)
    ref = net.init_buffers(2, d0)
    ref.buf.copy_(a.buf)
    net.to(d1)
    b = net.init_buffers(2, d1)
    b.copy_streams_from(a, [0, 1], [1, 0])
    y = _hop(net, b, xo[[1, 0], :, HOP * 10:HOP * 10 + HOP + LA].to(d1), e[[1, 0]].to(d1))
    net.to(d0)
    y_ref = _hop(net, ref, xo[..., HOP * 10:HOP * 10 + HOP + LA], e)
    assert torch.equal(y[[1, 0]].cpu(), y_ref.cpu())


def test_admitted_skipping_stream_vs_oracle(form, dev):
    """A stream admitted at hop 10 that then misses two hops, against the reference implementation fed the chunks it got."""
    net, sd, B = form
    s, T = 0, 40
    other, _ = su.clips(B, T, 1400, dev)
    n_fed = T - 10 - 2
    x_cpu, tgt = synth.mixture(1, HOP * n_fed, seed0=1500)
    xc = F.pad(x_cpu, (0, LA)).to(dev)
    e = su.emb(B, 1600, dev)
    st = net.init_buffers(B, dev)
    got, fed = [], 0
    for t in range(T):
        if t == 10:
            st.reset_streams([s])
        x = other[..., HOP * t:HOP * t + HOP + LA].clone()
        active = None
        if t >= 10:
            x[s] = su.chunk(xc[0], fed)
            active = torch.ones(B, dtype=torch.bool, device=dev)
            active[s] = t not in (13, 25)
        y = _hop(net, st, x, e, active)
        if t >= 10 and t not in (13, 25):
            got.append(y[s])
            fed += 1
    assert fed == n_fed
    y = torch.cat(got, -1).cpu()[None]
    y_ref, _ = rs.sep_predict(sd, x_cpu, e[s:s + 1].cpu(), rs.sep_init_state(sd, 1))
    assert rs.rel_l2(y, y_ref) <= 1e-3
    d = (rs.si_sdr(y, tgt) - rs.si_sdr(y_ref, tgt)).abs().max()
    assert float(d) <= 0.1
