"""The target mixer on the GPU (TargetMixer, l2h_target_mix, l2h_target_mix_set), on seeded inputs and fresh mixers.

Oracles: y itself and its fp32 row-order sums (unity gains, bit for bit); the float64 numpy model of
tests/test_target_mix_cpu.py (ramps, to 1e-6 of each row's peak); the same hops cut into other ticks (bit for bit); eager
calls (graph replays, bit for bit); and, on the seeded separator, the engine's own y run through the model."""
import math

import numpy as np
import pytest
import torch

import serving_util as su
from lookoncetohear_b200 import HopFifo, PacketResampler, TargetMixer
from serving_util import HOP, LA, SENTINEL, dev, model  # noqa: F401
from test_target_mix_cpu import _schedule, clamped_starts, level, model_mix, model_set, model_state

pytestmark = pytest.mark.gpu

TOL = 1e-6


def randn(*shape, seed, dev):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(dev)


def to_model(m):
    """the mixer's state as the model's float64 words"""
    s = m.state.cpu()
    w = s.double().numpy().copy()
    w[..., 2:] = s[..., 2:].contiguous().view(torch.int32).numpy()
    return w


def close(got, want, what, tol=TOL):
    """got (CUDA) against the model's float64 rows, to `tol` of each row's peak, on the samples the model wrote"""
    got = got.double().cpu().numpy()
    for i in range(want.shape[0]):
        live = ~np.isnan(want[i])
        assert np.array_equal(live, ~np.isnan(got[i])), (what, i, "written samples")
        if live.any():
            peak = max(np.abs(want[i][live]).max(), 1e-30)
            err = np.abs(got[i][live] - want[i][live]).max()
            assert err <= tol * peak, (what, i, err / peak)


# ---- 1. unity gains and muted rows -----------------------------------------------------------------------------------
@pytest.mark.parametrize("strided", [False, True], ids=["float4", "scalar"])
def test_unity_sums_and_muted_rows(dev, strided):
    """one unity target is y; several are their fp32 sum in row order; a muted record's rows and a silent ambient's chunk
    are never read (NaN in them does not reach out)"""
    R, C, T = 6, 2, 2
    L = HOP * T
    base = randn(R, C, L + (1 if strided else 0), seed=1, dev=dev)
    y = base[..., :L]                                   # the odd stride takes the scalar kernel
    m = TargetMixer(8, 4, C, device=dev)
    records, offsets, slots = [3, 0, 5, 1, 2, 4], [0, 1, 4, 6], [1, 0, 3]
    m.set_gains([2], [0.0])                              # record 2 (row 4): muted at once
    y[4] = float("nan")
    chunk = torch.full((3, C, L + LA), float("nan"), device=dev)
    out = m(y, records, offsets, slots, chunk=chunk)
    torch.cuda.synchronize()
    assert torch.equal(su.bits(out[0]), su.bits(y[0]))
    assert torch.equal(su.bits(out[1]), su.bits((y[1] + y[2]) + y[3]))
    assert torch.equal(su.bits(out[2]), su.bits(y[5]))
    assert not m.fading.any()


# ---- 2. random ramps against the model -------------------------------------------------------------------------------
def test_random_ramps_match_the_model(dev):
    """ramps of F in {0, 1, 127, 128, 129, 1000} from and to gains in [0, 2], sets with and without a start between
    ticks, ambient on, ragged hops: the model to 1e-6 of each row's peak, and the level and fading views"""
    NR, S, C, T, n = 12, 6, 2, 3, 4
    records, offsets, slots = [7, 2, 9, 0, 4, 11, 5, 1], [0, 2, 3, 5, 8], [5, 0, 3, 2]
    g = np.random.default_rng(11)
    m = TargetMixer(NR, S, C, device=dev)
    st = model_state(NR, S, C)
    fades = [0, 1, 127, 128, 129, 1000]
    for t in range(10):
        if t % 3 == 0:
            rows = g.permutation(NR)[:5].tolist()
            amb = g.permutation(S)[:2].tolist()
            gains = g.uniform(0, 2, 7).astype(np.float32).astype(np.float64).tolist()
            starts = g.uniform(0, 2, 7).astype(np.float32).astype(np.float64).tolist()
            fd = [fades[k] for k in g.integers(0, len(fades), 7)]
            with_start = t != 3
            m.set_gains(rows, gains[:5], fd[:5], starts[:5] if with_start else None)
            m.set_ambient(amb, gains[5:], fd[5:], starts[5:] if with_start else None)
            model_set(st, NR, rows + [NR + s for s in amb], gains, fd, starts if with_start else None)
        hops = g.integers(0, T + 1, n).tolist()
        y = randn(len(records), C, HOP * T, seed=100 + t, dev=dev)
        chunk = randn(n, C, HOP * T + LA, seed=200 + t, dev=dev)
        out = torch.full((n, C, HOP * T), SENTINEL, device=dev)
        m(y, records, offsets, slots, hops=hops, chunk=chunk, out=out)
        want = model_mix(st, NR, y.double().cpu().numpy(), records, offsets, slots, hops, chunk.double().cpu().numpy())
        close(out, want, f"tick {t}")
    torch.cuda.synchronize()
    words = to_model(m)
    assert np.array_equal(words[..., 2:], st[..., 2:])                  # F + 1 and p exactly
    lvl = [level(st[r, 0], 1.0 if r < NR else 0.0) for r in range(NR + S)]
    assert m.level.cpu().tolist() == pytest.approx(lvl, abs=1e-5)
    assert m.fading.cpu().tolist() == [bool(w[2] > 0 and w[3] < w[2] - 1) for w in st[:, 0]]


# ---- 3. the cut into ticks never changes a bit -----------------------------------------------------------------------
def test_hop_cuts_do_not_change_a_bit(dev):
    """16 hops per listener cut into ticks of one hop or into mixes of 0-3 hops: the concatenated outputs and the final
    ramps bit for bit equal"""
    NR, S, C, T, total = 8, 4, 2, 3, 16
    records, offsets, slots = [6, 1, 3, 0, 7, 5], [0, 3, 4, 5, 6], [2, 0, 3, 1]
    n, R = len(slots), len(records)
    ys = randn(R, C, HOP * total, seed=31, dev=dev)
    ys[5] = -ys[5].abs()                      # listener 3: one term fading to 0 at sample 300, negative samples ...
    ys[5, :, 300:] = float("nan")             # ... and NaN from where its gain is 0: neither reaches out
    amb = randn(n, C, HOP * total, seed=32, dev=dev)
    owner = [0, 0, 0, 1, 2, 3]
    results = []
    for sched in ([[1] * total] * n, [_schedule(total, T, 40 + i) for i in range(n)]):
        m = TargetMixer(NR, S, C, device=dev)
        m.set_gains([6, 1, 3, 0, 7], [1.0, 0.0, 2.0, 0.5, 1.5], [127, 129, 1000, 0, 300], [0.0, 1.0, 0.25, 1.0, 0.0])
        m.set_ambient([2, 0, 3], [0.3, 1.0, 0.0], [300, 1, 128])
        m.set_gains([5], [0.0], [300], [1.0])
        pos, got = [0] * n, [[] for _ in range(n)]
        for t in range(max(len(s) for s in sched)):
            hops = [s[t] if t < len(s) else 0 for s in sched]
            y = torch.full((R, C, HOP * T), SENTINEL, device=dev)
            ck = torch.full((n, C, HOP * T + LA), SENTINEL, device=dev)
            for r in range(R):
                i = owner[r]
                y[r, :, :HOP * hops[i]] = ys[r, :, pos[i]:pos[i] + HOP * hops[i]]
            for i in range(n):
                ck[i, :, :HOP * hops[i]] = amb[i, :, pos[i]:pos[i] + HOP * hops[i]]
            out = m(y, su.i32(records, dev), su.i32(offsets, dev), su.i32(slots, dev), hops=su.i32(hops, dev), chunk=ck)
            for i in range(n):
                got[i].append(out[i, :, :HOP * hops[i]])
                pos[i] += HOP * hops[i]
        results.append(([torch.cat(x, -1) for x in got], m.state.clone()))
    (a, sa), (b, sb) = results
    for i in range(n):
        assert a[i].shape[-1] == HOP * total
        assert torch.equal(su.bits(a[i]), su.bits(b[i])), i
    assert torch.equal(su.bits(sa), su.bits(sb))
    tail = a[3][:, 300:]                      # no term enters these samples: -0 under every cut
    assert not bool(a[3].isnan().any()) and bool((tail == 0).all()) and bool(torch.signbit(tail).all())


# ---- 4. what is stored, read and advanced ----------------------------------------------------------------------------
def test_store_rules(dev):
    """samples past 128 h keep the sentinel; a slot outside the mixer or h = 0 stores nothing and freezes its ramps;
    rows past offsets[n] and records outside the mixer are not read; decreasing and out-of-range offsets are clamped
    like the separator's, with no read or write out of bounds"""
    NR, S, C, T = 10, 5, 2, 2
    L = HOP * T
    m = TargetMixer(NR, S, C, device=dev)
    m.set_gains(list(range(NR)), 0.5, 1000, 1.5)
    m.set_ambient(list(range(S)), 0.5, 1000, 0.0)
    R = 7
    guard = torch.full((R + 4, C, L), float("nan"), device=dev)        # NaN around y: an out-of-bounds read shows
    y = guard[2:2 + R]
    y.copy_(randn(R, C, L, seed=61, dev=dev))
    ck = randn(4, C, L + LA, seed=62, dev=dev)
    frame = torch.full((4 + 4, C, L), 7.0, device=dev)                  # 7.0 around out: an out-of-bounds write shows
    out = frame[2:6]
    cases = [   # records, offsets, slots, hops
        ([0, 1, 2, 3, 4, 5, 6], [0, 2, 3, 5, 6], [0, 1, 2, 3], [2, 1, 0, 2]),            # h = 0: listener 2 stores nothing
        ([0, 1, 2, 3, 4, 5, 6], [0, 2, 3, 5, 6], [0, 9, 2, -1], [2, 2, 1, 2]),           # slots outside the mixer
        ([0, -1, 2, 30, 4, 5, 6], [0, 2, 3, 5, 6], [0, 1, 2, 3], [1, 2, 2, 2]),          # records outside: skipped
        ([0, 1, 2, 3, 4, 5, 6], [0, 4, 2, 9, -3], [0, 1, 2, 3], [2, 2, 2, 2]),           # decreasing, out of range
        ([0, 1, 2, 3, 4, 5, 6], [-5, 1, 1, 1, 2], [4, 1, 2, 3], [2, 2, 2, 2]),
    ]
    for c, (rec, off, sl, hops) in enumerate(cases):
        yc = y.clone()
        end = clamped_starts(off, R)[-1]
        for r in range(R):
            if r >= end or not 0 <= rec[r] < NR:
                y[r] = float("nan")                                     # never read
        st = to_model(m)
        out.fill_(SENTINEL)
        m(y, su.i32(rec, dev), su.i32(off, dev), su.i32(sl, dev), hops=su.i32(hops, dev), chunk=ck, out=out)
        want = model_mix(st, NR, y.double().cpu().numpy(), rec, off, sl, hops, ck.double().cpu().numpy())
        close(out, want, f"case {c}")
        assert np.array_equal(to_model(m)[..., 2:], st[..., 2:]), f"case {c}: ramps"
        assert bool((frame[:2] == 7.0).all()) and bool((frame[6:] == 7.0).all()), f"case {c}: guard"
        assert bool(guard[:2].isnan().all()) and bool(guard[2 + R:].isnan().all())
        y.copy_(yc)
    frozen = to_model(m)
    m(y, list(range(R)), [0, 2, 3, 5, 6], [0, 1, 2, 3], hops=[0, 0, 0, 0], chunk=ck, out=out)
    assert np.array_equal(to_model(m), frozen)


def test_listener_of_many_terms(dev):
    """one listener of 150 target rows (three passes of the kernel's 64 staged terms), some muted with NaN in their rows,
    beside a listener of 2: at unity gains the fp32 sum of the live rows in row order, bit for bit; with ramps and the
    ambient term (added in the last pass), the model"""
    R, C, T, NR, S = 152, 2, 2, 160, 3
    L = HOP * T
    records = torch.randperm(NR, generator=torch.Generator().manual_seed(81))[:R].tolist()
    offsets, slots = [0, 150, 152], [2, 0]
    muted = list(range(3, 150, 7))
    m = TargetMixer(NR, S, C, device=dev)
    m.set_gains([records[r] for r in muted], 0.0)
    y = randn(R, C, L, seed=82, dev=dev)
    y[muted] = float("nan")
    out = m(y, records, offsets, slots)
    want = None
    for r in range(150):
        if r not in muted:
            want = y[r].clone() if want is None else want + y[r]
    assert torch.equal(su.bits(out[0]), su.bits(want))
    assert torch.equal(su.bits(out[1]), su.bits(y[150] + y[151]))
    g = np.random.default_rng(83)
    live = [r for r in range(R) if r not in muted]
    m.set_gains([records[r] for r in live], g.uniform(0, 2, len(live)).astype(np.float32).tolist(), 700,
                g.uniform(0, 2, len(live)).astype(np.float32).tolist())
    m.set_ambient([2, 0], [0.5, 0.25], 100, [0.0, 1.0])
    st = to_model(m)
    chunk = randn(2, C, L + LA, seed=84, dev=dev)
    for t in range(3):
        out = m(y, records, offsets, slots, chunk=chunk)
        want = model_mix(st, NR, y.double().cpu().numpy(), records, offsets, slots, None, chunk.double().cpu().numpy())
        close(out, want, f"tick {t}", tol=4 * TOL)        # an fp32 sum of 130 terms rounds up to 130 times


def test_set_rows_outside_the_mixer(dev):
    """CUDA entries outside the mixer's records (or slots) in a set store nothing: record entry n_records does not touch
    slot 0's ambient ramp, slot entry n_slots nothing past the state"""
    NR, S, C = 4, 3, 2
    m = TargetMixer(NR, S, C, device=dev)
    m.set_ambient([0, 1, 2], 0.5, 10, 0.25)
    before = m.state.clone()
    m.set_gains(su.i32([NR, -1, NR + S], dev), torch.full((3,), 16.0, device=dev), su.i32([0, 0, 0], dev))
    m.set_ambient(su.i32([S, -1], dev), torch.full((2,), 16.0, device=dev), su.i32([0, 0], dev))
    torch.cuda.synchronize()
    assert torch.equal(su.bits(m.state), su.bits(before))
    m.set_gains(su.i32([1], dev), torch.full((1,), 2.0, device=dev), su.i32([0], dev))
    assert m.level.cpu().tolist() == pytest.approx([1.0, 2.0, 1.0, 1.0, 0.25, 0.25, 0.25])   # the slots' starts


# ---- 5. one CUDA graph per tick --------------------------------------------------------------------------------------
def test_graph_replay_with_lists_and_sets_rewritten(dev):
    """44.1 kHz packets down, FIFO, mixer (a seeded y stands in for the separator), up to 44.1 kHz, and a gain set, all in
    one captured graph with every list and value rewritten in place, against eager calls: outputs and states bit for bit"""
    S, C, T, n, NR, R = 6, 2, 2, 4, 10, 7

    def chain():
        return {"down": PacketResampler(44100, 16000, S, C, 882, device=dev),
                "fifo": HopFifo(S, C, T, 1024, device=dev), "mix": TargetMixer(NR, S, C, device=dev),
                "up": PacketResampler(16000, 44100, S, C, HOP * T, device=dev)}

    def bufs():
        return {"y16": torch.full((n, C, 320), SENTINEL, device=dev), "oc": torch.zeros(n, dtype=torch.int32, device=dev),
                "chunk": torch.full((n, C, HOP * T + LA), SENTINEL, device=dev),
                "hops": torch.zeros(n, dtype=torch.int32, device=dev),
                "mix": torch.full((n, C, HOP * T), SENTINEL, device=dev),
                "y44": torch.full((n, C, 353 * T), SENTINEL, device=dev),
                "oc44": torch.zeros(n, dtype=torch.int32, device=dev)}

    def tick(o, b, x, counts, slots, y, rec, off, sets):
        o["mix"].set_gains(sets["rows"], sets["gains"], sets["fades"], sets["starts"])
        o["mix"].set_ambient(sets["slots"], sets["amb"], sets["fades"][:1].contiguous())
        o["down"](x, counts, slots, out=b["y16"], out_counts=b["oc"])
        o["fifo"](b["y16"], b["oc"], slots, out=b["chunk"], hops=b["hops"])
        o["mix"](y, rec, off, slots, hops=b["hops"], chunk=b["chunk"], out=b["mix"])
        o["up"](b["mix"], b["hops"], slots, unit=HOP, out=b["y44"], out_counts=b["oc44"])

    def lists(t):
        g = torch.Generator().manual_seed(70 + t)
        sl = torch.randperm(S, generator=g)[:n].tolist()
        if t % 4 == 3:
            sl[t % n] = -1
        cn = [[0, 1, 441, 882, 300][int(k)] for k in torch.randint(0, 5, (n,), generator=g)]
        rec = torch.randperm(NR, generator=g)[:R].tolist()
        off = [0, 1, 3, 3, 6] if t % 2 else [0, 2, 4, 5, 7]
        rows = [rec[0], rec[1]] if t % 3 else [-1, -1]                   # a set of nothing
        fades = [int(k) for k in torch.randint(0, 400, (2,), generator=g)]
        sets = {"rows": rows, "gains": [float(t % 3) * 0.5, 1.0], "fades": fades, "starts": [0.0, 0.5],
                "slots": [sl[0] if t % 5 else -1], "amb": [0.1 * (t % 4)]}
        return sl, cn, rec, off, sets

    live, twin = chain(), chain()
    x = torch.zeros(n, C, 882, device=dev)
    y = torch.zeros(R, C, HOP * T, device=dev)
    slots, counts = su.i32(list(range(n)), dev), su.i32([0] * n, dev)
    rec, off = su.i32(list(range(R)), dev), su.i32([0, 1, 3, 5, 7], dev)
    sets = {"rows": su.i32([-1, -1], dev), "gains": torch.zeros(2, device=dev), "fades": su.i32([0, 0], dev),
            "starts": torch.zeros(2, device=dev), "slots": su.i32([-1], dev), "amb": torch.zeros(1, device=dev)}
    b = bufs()
    graph = su.captured(lambda: tick(live, b, x, counts, slots, y, rec, off, sets))   # nothing pushed or set
    for t in range(12):
        sl, cn, rl, ol, st = lists(t)
        x.copy_(su.signals(n, C, 882, 80 + t, dev))
        y.copy_(randn(R, C, HOP * T, seed=90 + t, dev=dev))
        slots.copy_(su.i32(sl, dev)); counts.copy_(su.i32(cn, dev))
        rec.copy_(su.i32(rl, dev)); off.copy_(su.i32(ol, dev))
        sets["rows"].copy_(su.i32(st["rows"], dev)); sets["gains"].copy_(torch.tensor(st["gains"]))
        sets["fades"].copy_(su.i32(st["fades"], dev)); sets["starts"].copy_(torch.tensor(st["starts"]))
        sets["slots"].copy_(su.i32(st["slots"], dev)); sets["amb"].copy_(torch.tensor(st["amb"]))
        su.refill(b)
        graph.replay()
        want = bufs()
        eager = {k: (su.i32(st[k], dev) if k in ("rows", "fades", "slots") else torch.tensor(st[k], device=dev))
                 for k in st}
        tick(twin, want, x, su.i32(cn, dev), su.i32(sl, dev), y, su.i32(rl, dev), su.i32(ol, dev), eager)
        su.assert_same(b, want, live, twin, t)


# ---- 6. on the separator ---------------------------------------------------------------------------------------------
def test_on_the_separator(model, dev):
    """listeners of 1, 2 and 3 voices ticked with advance_target_rows: the mix is the model of the engine's own y; a voice
    joined with join_targets and faded in over 480 samples enters at G(0) = (1 - cos(pi / 480)) / 2; a faded-out voice,
    once settled at 0, gives the mix of the same y with its record -1, bit for bit (R stays fixed)"""
    net, _ = model
    ks = [1, 2, 3]
    n, R = len(ks), sum(ks)
    offsets = [0, 1, 3, 6]
    S = R + 2
    clips, _ = su.clips(n, 16, 9700, dev)
    e = su.emb(R, 9710, dev)
    recs = [4, 0, 7, 2, 6, 1]
    B = recs[2]                      # the second voice of listener 1 joins late
    st = net.init_buffers(S, dev)
    hist = net.target_history(st, 16)
    m = TargetMixer(S, n, 2, device=dev)
    m.set_ambient([0, 1, 2], [0.1, 0.0, 0.25], 200)
    ms = model_state(S, n, 2)
    model_set(ms, S, [S, S + 1, S + 2], [0.1, 0.0, 0.25], [200] * 3)
    listed = [r if r != B else -1 for r in recs]
    G0 = (1 - math.cos(math.pi / 480)) / 2
    with torch.no_grad():
        for t in range(12):
            if t == 4:
                net.join_targets(st, [B], [recs[1]], e[[2]], history=hist)
                m.set_gains([B], [1.0], fade=480, start=0.0)
                model_set(ms, S, [B], [1.0], [480], [0.0])
                listed = list(recs)
            if t == 7:
                m.set_gains([B], [0.0], fade=480)
                model_set(ms, S, [B], [0.0], [480])
            x = torch.stack([su.chunk(clips[i], t) for i in range(n)]).contiguous()
            y = net.advance_target_rows(x, e, st, su.i32(listed, dev), su.i32(offsets, dev), history=hist)
            twin = TargetMixer(S, n, 2, device=dev)
            twin.state.copy_(m.state)
            out = m(y, su.i32(listed, dev), offsets, [0, 1, 2], chunk=x)
            want = model_mix(ms, S, y.double().cpu().numpy(), listed, offsets, [0, 1, 2], None, x.double().cpu().numpy())
            close(out, want, f"tick {t}")
            if t == 4:                                  # B enters at G(0), not at full level
                yb = y[2].double()
                rest = out[1].double() - y[1].double()
                assert float((rest[:, 0] - G0 * yb[:, 0]).abs().max()) <= 1e-6 * float(yb[:, 0].abs().max()) + 1e-7
                assert float((rest[:, 0] - yb[:, 0]).abs().max()) > 0.5 * float(yb[:, 0].abs().max())
            if t >= 11:                                 # settled at 0: the same mix as record -1
                assert not bool(m.fading[B])
                dropped = [r if r != B else -1 for r in recs]
                alt = twin(y, su.i32(dropped, dev), offsets, [0, 1, 2], chunk=x)
                assert torch.equal(su.bits(out), su.bits(alt))


def test_advance_targets_view(model, dev):
    """the y of advance_targets viewed as [n K, S, 128 T] with offsets i K and records g_i K + k mixes exactly as the
    equivalent advance_target_rows call"""
    net, _ = model
    G, K, n = 4, 2, 3
    groups = [2, 0, 3]
    clips, _ = su.clips(n, 3, 9800, dev)
    e = su.embeds(n, K, 9810, dev)
    st_g, st_r = net.init_buffers(G * K, dev), net.init_buffers(G * K, dev)
    recs = su.recs(groups, K)
    off = [i * K for i in range(n + 1)]
    mg, mr = TargetMixer(G * K, n, 2, device=dev), TargetMixer(G * K, n, 2, device=dev)
    for m in (mg, mr):
        m.set_gains(recs, [1.0, 0.5, 0.0, 1.0, 2.0, 0.25], 300, 0.0)
        m.set_ambient([0, 1, 2], 0.2, 100)
    with torch.no_grad():
        for t in range(3):
            x = torch.stack([su.chunk(clips[i], t) for i in range(n)]).contiguous()
            yg = net.advance_targets(x, e, st_g, groups)
            yr = net.advance_target_rows(x, e.reshape(n * K, 256), st_r, recs, off)
            a = mg(yg.view(n * K, 2, -1), recs, off, [0, 1, 2], chunk=x)
            b = mr(yr, recs, off, [0, 1, 2], chunk=x)
            assert torch.equal(su.bits(a), su.bits(b)), t
    assert torch.equal(su.bits(mg.state), su.bits(mr.state))
