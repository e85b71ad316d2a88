"""Ragged multi-hop calls over a list of a state's records (Net.advance_slots(hops=) / l2h_sep_forward_slots_hops): row i
advances its record by its own h_i of the call's T hops.  The model is causal in time, so the first h_i hops of a T-hop
call are those of an h_i-hop call; the call computes all T and stores only what h_i hops leave.  Kernel forms as in
tests/test_slot_list_frames_gpu.py: CUDA-core rows (n = 2, T = 3 and n = 4, T = 5, with the multi-frame front / back
walkers and without), the tensor-core chain (n = 8, T = 3) and the tensor-core recurrence (n = 48, T = 2), alone and with
the input projection fused (fuse_ih, which masks the padded steps inside the recurrence kernel)."""
import time

import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import synth
from oracle import restate as rs
from kernels import harness as kh
import serving_util as su
from serving_util import HOP, LA, L2H_FLAG_GRAPH, SENTINEL, dev, model  # noqa: F401

pytestmark = pytest.mark.gpu
FORMS = [pytest.param((12, 2, 3, {"back_many": 1}), id="n2-T3"),
         pytest.param((12, 2, 3, {"back_many": 0}), id="n2-T3-per-frame"),
         pytest.param((12, 4, 5, {"back_many": 1}), id="n4-T5"),
         pytest.param((12, 4, 5, {"back_many": 0}), id="n4-T5-per-frame"),
         pytest.param((16, 8, 3, {}), id="n8-T3-tc"),
         pytest.param((56, 48, 2, {}), id="n48-T2-tc-lstm"),
         pytest.param((56, 48, 2, {"fuse_ih": 1}), id="n48-T2-tc-lstm-x")]


@pytest.fixture(params=FORMS)
def form(request, model):
    S, n, T, opts = request.param
    net, sd = model
    with su.switched(net, opts):
        yield net, sd, S, n, T


# ---- all hops = T: the ragged call is l2h_sep_forward_slots_frames --------------------------------------------------
def test_all_hops_T_equal_slots_frames(form, dev):
    net, _, S, n, T = form
    st = su.warm_slots(net, S, n, T, 6100, dev)
    twin = su.copy(net, st)
    clips, _ = su.clips(n, T, 6200, dev)
    x = clips.contiguous()
    e = su.emb(n, 6300, dev)
    sl = torch.tensor(su.subsets(S, n, 1, 6400)[0], dtype=torch.int32, device=dev)
    y = torch.full((n, 2, HOP * T), SENTINEL, device=dev)
    y_ref = torch.full_like(y, SENTINEL)
    net._launch("slots_hops", x, e, st, y, T, slots=sl, hops=torch.full((n,), T, dtype=torch.int32, device=dev))
    net._launch("slots_frames", x, e, twin, y_ref, T, slots=sl)
    torch.cuda.synchronize()
    assert torch.equal(su.bits(y), su.bits(y_ref))
    assert torch.equal(su.bits(st.buf), su.bits(twin.buf))


# ---- all hops 0, and slots out of range: nothing stored --------------------------------------------------------------
def test_zero_hops_and_outside_slots_store_nothing(form, dev):
    net, _, S, n, T = form
    st = su.warm_slots(net, S, n, T, 6500, dev)
    before = su.bits(st._rec()).clone()
    clips, _ = su.clips(n, T, 6600, dev)
    e = su.emb(n, 6700, dev)
    sl = su.subsets(S, n, 1, 6800)[0]
    for slots, hops in ((sl, [0] * n), ([-1 - i if i % 2 else S + i for i in range(n)], [T] * n),
                        (sl, [T + 1 + i if i % 2 else -1 - i for i in range(n)])):      # counts outside [0, T] count as 0
        y = torch.full((n, 2, HOP * T), SENTINEL, device=dev)
        net._launch("slots_hops", clips.contiguous(), e, st, y, T, slots=torch.tensor(slots, dtype=torch.int32, device=dev),
                    hops=torch.tensor(hops, dtype=torch.int32, device=dev))
        torch.cuda.synchronize()
        assert bool(torch.isnan(y).all()), "a y row was written"
        assert torch.equal(su.bits(st._rec()), before), "a record changed"


# ---- mixed hops against a uniform T-hop call on a copy ---------------------------------------------------------------
def test_mixed_hops_match_uniform_call_where_they_advance(form, dev):
    """x NaN past each row's 128 h_i + 64 samples: y[i, :, :128 h_i] and the ring rows of the h_i new frames equal a
    uniform T-hop call on a copy bit for bit; later y samples keep the sentinel; other ring rows, and unlisted records,
    are as before; clocks advance by h_i (calls by 1 if h_i > 0)."""
    net, _, S, n, T = form
    st = su.warm_slots(net, S, n, T, 6900, dev)
    twin = su.copy(net, st)
    before = st._rec().clone()
    pos0 = st.stream_pos()
    calls0 = st._clocks()[1].cpu().tolist()
    clips, _ = su.clips(n, T, 7000, dev)
    x = clips.contiguous().clone()
    hops = su.hop_mix(n, T, 7100)
    for i, h in enumerate(hops):
        x[i, :, HOP * h + LA:] = float("nan")
    e = su.emb(n, 7200, dev)
    sl = su.subsets(S, n, 1, 7300)[0]
    slots = torch.tensor(sl, dtype=torch.int32, device=dev)
    y = torch.full((n, 2, HOP * T), SENTINEL, device=dev)
    y_ref = torch.full_like(y, SENTINEL)
    net._launch("slots_hops", x, e, st, y, T, slots=slots, hops=torch.tensor(hops, dtype=torch.int32, device=dev))
    net._launch("slots_frames", clips.contiguous(), e, twin, y_ref, T, slots=slots)
    torch.cuda.synchronize()
    for i, (s, h) in enumerate(zip(sl, hops)):
        assert torch.equal(su.bits(y[i, :, :HOP * h]), su.bits(y_ref[i, :, :HOP * h])), (i, h)
        assert bool(torch.isnan(y[i, :, HOP * h:]).all()), (i, h, "y written past the row's hops")
        new = su.ring_mask(st, range(pos0[s], pos0[s] + h))
        assert torch.equal(su.bits(st._rec()[s][new]), su.bits(twin._rec()[s][new])), (i, h, "ring rows of the new frames")
        other = su.ring_all(st) & ~new
        assert torch.equal(su.bits(st._rec()[s][other]), su.bits(before[s][other])), (i, h, "another ring row changed")
        if h == 0:
            assert torch.equal(su.bits(st._rec()[s]), su.bits(before[s])), (i, "h = 0 stored something")
        if h == T:
            assert torch.equal(su.bits(st._rec()[s]), su.bits(twin._rec()[s])), (i, "h = T")
    unlisted = [s for s in range(S) if s not in sl]
    assert torch.equal(su.bits(st._rec()[unlisted]), su.bits(before[unlisted]))
    pos, calls = st.stream_pos(), st._clocks()[1].cpu().tolist()
    for s, h in zip(sl, hops):
        assert pos[s] == pos0[s] + h and calls[s] == calls0[s] + (1 if h > 0 else 0), (s, h)


# ---- against today's recipe: one advance_slots per depth on copied-out records ----------------------------------------
def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _state_parts(st, s):
    """the parts of record s a call stores, as float tensors: rings, (h, c) of every block, the current tails"""
    L, r = st.lay, st._rec()[s]
    par = int(st._clocks()[1][s]) & 1
    parts = {"ring": r[su.ring_all(st)]}
    for blk in range(st.n_blocks):
        base = L["st_blk"] + blk * L["bk_stride"]
        parts[f"h{blk}"] = r[base + L["bk_h"]:base + L["bk_h"] + 97 * 64]
        parts[f"c{blk}"] = r[base + L["bk_c"]:base + L["bk_c"] + 97 * 64]
    conv, deconv, istft = 2 * 4 * 97, 2 * 97 * 64, 2 * 194
    parts["conv"] = r[L["st_conv"] + par * conv:L["st_conv"] + (par + 1) * conv]
    parts["deconv"] = r[L["st_deconv"] + par * deconv:L["st_deconv"] + (par + 1) * deconv]
    parts["istft"] = r[L["st_istft"] + par * istft:L["st_istft"] + (par + 1) * istft]
    return parts


def test_mixed_hops_match_per_depth_recipe(form, dev, record_property):
    """The listed records advanced by one ragged call, against copying them out and running one advance_slots per depth:
    clocks exact; rings / h / c / tails and y within 1e-5 relative L2 where the ragged call and every per-depth call run
    on the same side of the tensor-core threshold (2048 rows), 5e-5 where one runs the bf16x3 tensor-core chain and the
    other the fp32 CUDA-core one; then 10 one-hop predict(slots=) calls on both, with y within the same bound.  Which
    depths came out bit-identical is recorded as the test's `bit_identical_by_depth` property."""
    net, _, S, n, T = form
    st = su.warm_slots(net, S, n, T, 7400, dev)
    ref = su.copy(net, st)
    clips, _ = su.clips(S, T + 70, 7500, dev)
    e = su.emb(S, 7600, dev)
    sl = su.subsets(S, n, 1, 7700)[0]
    hops = su.hop_mix(n, T, 7800)
    pos0 = st.stream_pos()
    tc = lambda rows, hops_: rows * hops_ * 97 > 2048          # the engine's tensor-core threshold (TC_MIN_ROWS)
    bound = 1e-5 if all(tc(hops.count(h), h) == tc(n, T) for h in set(hops) - {0}) else 5e-5
    with torch.no_grad():
        x = torch.stack([su.chunk(clips[s], 0, T) for s in sl])
        y = net.advance_slots(x, e[sl], st, sl, hops=hops)
        for h in sorted(set(hops) - {0}):
            rows = [i for i in range(n) if hops[i] == h]
            ss = [sl[i] for i in rows]
            tmp = net.init_buffers(len(ss), dev)
            tmp.copy_streams_from(ref, ss, list(range(len(ss))))
            y_h = net.advance_slots(torch.stack([su.chunk(clips[s], 0, h) for s in ss]), e[ss], tmp, list(range(len(ss))))
            ref.copy_streams_from(tmp, list(range(len(ss))), ss)
            for j, i in enumerate(rows):
                assert _rel(y[i, :, :HOP * h], y_h[j]) <= bound, (i, h)
    assert st.stream_pos() == ref.stream_pos()
    assert [st.stream_pos()[s] - pos0[s] for s in sl] == hops
    exact, worst = {}, {}
    for s, h in zip(sl, hops):
        a, b = _state_parts(st, s), _state_parts(ref, s)
        for k in a:
            same = torch.equal(su.bits(a[k]), su.bits(b[k]))
            exact[f"h{h}"] = exact.get(f"h{h}", True) and same
            if not same:
                worst[k] = max(worst.get(k, 0.0), _rel(a[k], b[k]))
    record_property("bit_identical_by_depth", exact)
    record_property("max_rel_l2", worst)
    assert all(v <= bound for v in worst.values()), (bound, worst)
    fed = {s: h for s, h in zip(sl, hops)}
    with torch.no_grad():
        for k in range(10):                 # (records near the ring's wrap: test_recipe_calls_cross_the_ring)
            xs = torch.stack([su.chunk(clips[s], fed[s] + k, 1) for s in sl])
            ya, _ = net.predict(xs, e[sl], st, pad=False, slots=sl)
            yb, _ = net.predict(xs, e[sl], ref, pad=False, slots=sl)
            assert _rel(ya, yb) <= bound, k
    assert max(st.stream_pos()[s] for s in sl) >= 10


def test_recipe_calls_cross_the_ring(model, dev):
    """A ragged call whose records sit a few hops below the 56-slot ring's wrap, then 10 one-hop calls: against the
    per-depth recipe, y within 1e-5 on every call and the clocks exact."""
    net, _ = model
    S, n, T = 10, 4, 5
    clips, _ = su.clips(S, 120, 7900, dev)
    e = su.emb(S, 8000, dev)
    st = net.init_buffers(S, dev)
    fed = (50 + torch.arange(S) % 4).tolist()
    with torch.no_grad():
        for s in range(S):
            one = net.init_buffers(1, dev)
            net.predict(su.chunk(clips[s], 0, fed[s])[None], e[s:s + 1], one, pad=False)
            st.copy_streams_from(one, [0], [s])
        ref = su.copy(net, st)
        sl = [1, 4, 6, 9]
        hops = [0, 1, 5, 3]
        y = net.advance_slots(torch.stack([su.chunk(clips[s], fed[s], T) for s in sl]), e[sl], st, sl, hops=hops)
        for h in (1, 3, 5):
            ss = [s for s, hh in zip(sl, hops) if hh == h]
            yy = net.advance_slots(torch.stack([su.chunk(clips[s], fed[s], h) for s in ss]), e[ss], ref, ss)
            i = hops.index(h)
            assert _rel(y[i, :, :HOP * h], yy[0]) <= 1e-5, h
        for s, h in zip(sl, hops):
            fed[s] += h
        assert st.stream_pos() == ref.stream_pos() == fed
        for k in range(10):
            xs = torch.stack([su.chunk(clips[s], fed[s] + k, 1) for s in sl])
            ya, _ = net.predict(xs, e[sl], st, pad=False, slots=sl)
            yb, _ = net.predict(xs, e[sl], ref, pad=False, slots=sl)
            assert _rel(ya, yb) <= 1e-5, k
    assert max(st.stream_pos()) > 56


# ---- the premise: masked gates leave c where T_b steps leave it --------------------------------------------------------
RECURRENCES = [("rec3_pre", 3), ("rec3_ring", 3), ("rec4_2", 3), ("rec4_4", 3), ("tc", 1), ("tc", 2), ("tc", 3)]


@pytest.mark.parametrize("variant,passes", RECURRENCES, ids=[f"{v}_p{p}" for v, p in RECURRENCES])
def test_masked_inter_steps_carry_c(variant, passes, dev):
    """The inter layout (sequence (b, f), steps NF rows apart, carried (h, c)), gate pre-activations of steps >= T_b set to
    i = -inf, f = +inf, g = 0 as inter_gate_mask_kernel sets them: every output is finite, and the outputs of steps < T_b
    and the final c equal, bit for bit, a run of only T_b steps (sigma(+inf) = 1 exactly, sigma(-inf) = 0)."""
    NF = 97
    Tbs = [4, 1, 3, 0, 2]
    B, L = len(Tbs), 4
    g = torch.Generator().manual_seed(8100)
    gx = 0.8 * torch.randn(B, L, NF, 256, generator=g)
    for b, tb in enumerate(Tbs):
        gv = gx[b, tb:].view(-1, NF, 64, 4)
        gv[..., 0], gv[..., 1], gv[..., 2] = float("-inf"), float("inf"), 0.0
    whh = ((torch.rand(256, 64, generator=g) * 2 - 1) * 0.25).to(dev)
    h0 = 0.5 * torch.randn(B, NF, 64, generator=g)
    c0 = torch.randn(B, NF, 64, generator=g)

    def run(gx_, steps, rows):
        nb = gx_.shape[0]
        gd = gx_[:, :steps].contiguous().to(dev)
        out = torch.full((nb, max(steps, 1), NF, 64), float("nan"), device=dev)
        hs, cs = h0[rows].clone().to(dev), c0[rows].clone().to(dev)
        a = kh.Lstm()
        a.gx, a.gx_ld, a.out, a.out_ld, a.whh = gd.data_ptr(), 256, out.data_ptr(), 64, whh.data_ptr()
        a.h_state, a.c_state, a.hc_outer_stride = hs.data_ptr(), cs.data_ptr(), NF * 64
        a.nseq, a.L, a.inner_count, a.ndir = nb * NF, steps, NF, 1
        a.outer_stride, a.inner_stride, a.step_stride = steps * NF, 1, NF
        rc, why = kh.lstm(a, variant, passes)
        torch.cuda.synchronize()
        assert rc == 0, why
        return out.cpu(), hs.cpu(), cs.cpu()

    out, _, c = run(gx, L, slice(0, B))
    assert bool(torch.isfinite(out).all()) and bool(torch.isfinite(c).all())
    for b, tb in enumerate(Tbs):
        if tb == 0:
            assert torch.equal(su.bits(c[b]), su.bits(c0[b])), (b, "c moved through masked steps only")
            continue
        o1, _, c1 = run(gx[b:b + 1], tb, slice(b, b + 1))
        assert torch.equal(su.bits(out[b, :tb]), su.bits(o1[0, :tb])), (b, variant, passes)
        assert torch.equal(su.bits(c[b]), su.bits(c1[0])), (b, variant, passes, "final c")


# ---- one stream against the reference ---------------------------------------------------------------------------------
@pytest.mark.parametrize("S, n", [pytest.param(6, 3, id="n3"), pytest.param(16, 8, id="n8-tc")])
def test_ragged_stream_vs_oracle(model, dev, S, n):
    """A stream advanced by ragged calls of T = 3, 5, 2, 4 with its own hops 2, 0, 2, 4, 1, ... among rows with other
    counts, against the reference implementation fed the chunks it got: output and to_reference() state within 1e-3."""
    net, sd = model
    s = S - 1
    plan = [(3, 2), (5, 0), (2, 2), (4, 4), (5, 1), (3, 3), (4, 0), (2, 1)]
    n_fed = sum(h for _, h in plan)
    x_cpu, tgt = synth.mixture(1, HOP * n_fed, seed0=8200)
    xc = F.pad(F.pad(x_cpu, (0, LA)), (0, HOP * 5), value=float("nan")).to(dev)     # never read past its own hops
    others, _ = su.clips(S, 5 * len(plan), 8300, dev)
    e = su.emb(S, 8400, dev)
    st = net.init_buffers(S, dev)
    fed_o = [0] * S
    got, fed = [], 0
    with torch.no_grad():
        for c, ((T, h), sl) in enumerate(zip(plan, su.subsets(S - 1, n, len(plan), 8500))):
            sl[c % n] = s
            hops = su.hop_mix(n, T, 8600 + c)
            hops[c % n] = h
            x = torch.stack([su.chunk(xc[0], fed, T) if b == s else su.chunk(others[b], fed_o[b], T) for b in sl])
            y = net.advance_slots(x, e[sl], st, sl, hops=hops)
            got.append(y[c % n, :, :HOP * h])
            fed += h
            for b, hh in zip(sl, hops):
                if b != s:
                    fed_o[b] += hh
    y = torch.cat(got, -1).cpu()[None]
    y_ref, st_ref = rs.sep_predict(sd, x_cpu, e[s:s + 1].cpu(), rs.sep_init_state(sd, 1))
    assert rs.rel_l2(y, y_ref) <= 1e-3
    one = net.init_buffers(1, dev)
    one.copy_streams_from(st, [s], [0])
    exported = one.to_reference()
    for k in ("conv_buf", "deconv_buf", "istft_buf"):
        assert rs.rel_l2(exported[k].cpu(), st_ref[k]) <= 1e-3, k
    for i in range(3):
        for k in ("K_buf", "V_buf", "h0", "c0"):
            a, b = exported["gridnet_bufs"][f"buf{i}"][k].cpu(), st_ref["gridnet_bufs"][f"buf{i}"][k]
            assert rs.rel_l2(a, b) <= 1e-3, (i, k)


# ---- graph replay with slots and hops rewritten in place -------------------------------------------------------------
def test_graph_replay_with_slots_and_hops_rewritten(form, dev):
    """With L2H_FLAG_GRAPH, the inputs, slots and hops rewritten in place every tick and one graph replayed: y and the
    whole state equal direct calls bit for bit.  The hops' contents are not part of the graph key: only the first call
    captures (capture + instantiation costs milliseconds of host time, a replay tens of microseconds)."""
    net, _, S, n, T = form
    calls = 5
    clips, _ = su.clips(S, calls * T, 8700, dev)
    e = su.emb(S, 8800, dev)
    xbuf, ebuf = torch.empty(n, 2, HOP * T + LA, device=dev), torch.empty(n, 256, device=dev)
    slots = torch.empty(n, dtype=torch.int32, device=dev)
    hops = torch.empty(n, dtype=torch.int32, device=dev)
    yg, yd = torch.empty(n, 2, HOP * T, device=dev), torch.empty(n, 2, HOP * T, device=dev)
    sg, sdir = net.init_buffers(S, dev), net.init_buffers(S, dev)
    fed = [0] * S
    host = []
    for c, sl in enumerate(su.subsets(S, n, calls, 8900)):
        hh = su.hop_mix(n, T, 9000 + c)
        xbuf.copy_(torch.stack([su.chunk(clips[s], fed[s], T) for s in sl]))
        ebuf.copy_(e[sl])
        slots.copy_(torch.tensor(sl, dtype=torch.int32))
        hops.copy_(torch.tensor(hh, dtype=torch.int32))
        yg.fill_(SENTINEL)
        yd.fill_(SENTINEL)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        net._launch("slots_hops", xbuf, ebuf, sg, yg, T, L2H_FLAG_GRAPH, slots=slots, hops=hops)
        host.append(time.perf_counter() - t0)
        net._launch("slots_hops", xbuf, ebuf, sdir, yd, T, slots=slots, hops=hops)
        for s, h in zip(sl, hh):
            fed[s] += h
        torch.cuda.synchronize()
        assert torch.equal(su.bits(yg), su.bits(yd)), c
    assert torch.equal(su.bits(sg.buf), su.bits(sdir.buf))
    assert sg.stream_pos() == fed
    assert max(host[1:]) < 0.5 * host[0], ("a replay took as long as a capture: new graph per hop mix?", host)
