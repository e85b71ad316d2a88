"""The leveler on the GPU (Leveler, l2h_leveler), on seeded inputs and fresh levelers.

Oracles: the input itself (with a gain range of 0 dB, bit for bit); the float64 numpy model of tests/test_leveler_cpu.py
(telemetry to 0.01 dB, output to 2e-3 of each row's peak, on hops built to sit at least 1 dB from every gate edge); the
target loudness itself, measured on the output; the same hops cut into other ticks (bit for bit); eager calls (graph
replays, bit for bit); and, on the seeded separator, the eager 44.1 kHz chain and a leveler that heard a joined voice from
the start."""
import math

import numpy as np
import pytest
import torch
from scipy.signal import lfilter

import serving_util as su
from lookoncetohear_b200 import Leveler
from serving_util import HOP, SENTINEL, dev, model  # noqa: F401
from test_leveler_cpu import DEFAULTS, FILTERS, lufs, model_hop, model_state, voice

pytestmark = pytest.mark.gpu

C = 2


def params(lev):
    """the model's parameters of a Leveler"""
    return {"target": lev.target, "gate": lev.gate, "relative": lev.relative, "alpha": lev.alpha,
            "settle": lev.settle_hops, "min_gain": lev.min_gain, "max_gain": lev.max_gain, "rise": lev.rise_step,
            "fall": lev.fall_step}


def owners(offsets, n, R):
    """the listener of every row (-1: none), with the separator's clamp"""
    own = []
    for r in range(R):
        first = next((j for j in range(n + 1) if offsets[j] > r), n + 1)
        own.append(first - 1 if 0 <= first - 1 < n else -1)
    return own


def margin(st, x, p):
    """how far (dB) the hop x [C, 128] lies from the gate edges the row's state puts it against"""
    sb, sa, hb, ha = FILTERS
    u, _ = lfilter(sb, sa, x, axis=1, zi=st["shelf"])
    w, _ = lfilter(hb, ha, u, axis=1, zi=st["hp"])
    L = lufs(float((w ** 2).sum()) / HOP)
    m = abs(L - p["gate"])
    if st["n"]:
        m = min(m, abs(L - lufs(st["E"]) - p["relative"]))
    return m


def k_loudness(x):
    """the K-weighted loudness (LUFS) of x [C, N] float64 over all of it"""
    sb, sa, hb, ha = FILTERS
    w = lfilter(hb, ha, lfilter(sb, sa, x, axis=1), axis=1)
    return lufs((w ** 2).sum(0).mean())


# ---- 1. a gain range of 0 dB: the input bit for bit --------------------------------------------------------------------
def test_identity_at_zero_gain_range(dev):
    """min_gain = max_gain = 0: every finite sample of out is y's, -0 included, in place and not; non-finite samples stay
    non-finite; the telemetry moves"""
    R, T = 5, 6
    y = su.signals(R, C, HOP * T, 1, dev) * 3
    y[0, 0, 10:20] = -0.0
    y[1, 1, 300] = float("nan")
    y[2, 0, 500] = float("inf")
    y[3, :, 128:256] = 1e-40
    lev = Leveler(8, C, gate=-90.0, settle=0.008, min_gain=0.0, max_gain=0.0, device=dev)
    keep = y.clone()
    out = lev(y, [7, 0, 3, 5, 1], [0, 2, 5], hops=[T, T])
    lev(y, su.i32([6, 2, 4, 1, -1], dev), out=y)
    torch.cuda.synchronize()
    fin = torch.isfinite(keep)
    for got in (out, y):
        assert torch.equal(su.bits(got)[fin], su.bits(keep)[fin])
        assert not bool(torch.isfinite(got[~fin]).any())
    assert bool((lev.loudness[[7, 0, 3, 5, 1]] > -60).all()) and not lev.gain.any()


# ---- 2. the model -----------------------------------------------------------------------------------------------------
def test_random_rows_agree_with_the_model(dev):
    """records scattered over the state, listeners of 1 to 3 rows with ragged hops (0 included), rows of voices at
    levels from -40 to 0 dB in ticks: telemetry to 0.01 dB, output to 2e-3 of each row's peak"""
    R, n, S, T, ticks = 7, 4, 12, 3, 40
    offsets = [0, 1, 3, 6, 7]
    own = owners(offsets, n, R)
    g = torch.Generator().manual_seed(3)
    records = torch.randperm(S, generator=g)[:R].tolist()
    sched = [su.hop_mix(n, T, 100 + t) for t in range(ticks)]
    total = [sum(s[own[r]] for s in sched) for r in range(R)]
    levels = [-45.0, -3.0, 0.0, -10.0, 5.0, -8.0, -40.0]                 # clear of the -50 LUFS gate by 5 dB and more
    xs = [voice(C, total[r], 200 + r, db=levels[r]) for r in range(R)]
    lev = Leveler(S, C, settle=0.08, rise=20.0, fall=30.0, window=0.5, device=dev)
    p = params(lev)
    mst, pos, want, got = [model_state(C) for _ in range(R)], [0] * R, [[] for _ in range(R)], [[] for _ in range(R)]
    for t in range(ticks):
        y = torch.full((R, C, HOP * T), SENTINEL)
        for r in range(R):
            h = sched[t][own[r]]
            y[r, :, :HOP * h] = torch.from_numpy(xs[r][:, HOP * pos[r]:HOP * (pos[r] + h)]).float()
            for k in range(h):
                hop = xs[r][:, HOP * (pos[r] + k):HOP * (pos[r] + k + 1)]
                assert margin(mst[r], hop, p) >= 1.0, (t, r, k)          # fp32 and float64 take the same gate decision
                want[r].append(model_hop(mst[r], hop, p))
            pos[r] += h
        out = lev(y.to(dev), su.i32(records, dev), su.i32(offsets, dev), hops=su.i32(sched[t], dev))
        for r in range(R):
            got[r].append(out[r, :, :HOP * sched[t][own[r]]].cpu())
    torch.cuda.synchronize()
    for r in range(R):
        a, b = torch.cat(got[r], -1).double().numpy(), np.concatenate(want[r], 1)
        assert np.abs(a - b).max() <= 2e-3 * np.abs(b).max(), r
        assert abs(float(lev.gain[records[r]]) - mst[r]["g"]) <= 0.01, r
        if mst[r]["n"]:
            assert abs(float(lev.loudness[records[r]]) - lufs(mst[r]["E"])) <= 0.01, r
        else:
            assert float(lev.loudness[records[r]]) == -math.inf, r
        assert int(lev.state[records[r], 0, 1].view(torch.int32)) == mst[r]["n"], r
    assert any(abs(m["g"]) > 1 for m in mst)                          # the gains did move


def test_two_voices_reach_the_target(dev):
    """one listener's two rows, voices 20 dB apart: after settling both play within 0.5 dB of the target, and the two
    channels of each row always share one gain"""
    T, ticks = 4, 300
    x = np.stack([voice(C, T * ticks, 300, db=15.0), voice(C, T * ticks, 301, db=-5.0)])      # about -8 and -28 LUFS
    assert abs(k_loudness(x[0]) - k_loudness(x[1]) - 20) < 1.0
    xd = torch.from_numpy(x).float().to(dev)
    lev = Leveler(4, C, device=dev)
    outs = [lev(xd[:, :, HOP * T * t:HOP * T * (t + 1)], [3, 1], [0, 2]) for t in range(ticks)]
    out = torch.cat(outs, -1)
    torch.cuda.synchronize()
    tail = out[:, :, -HOP * 1000:].double().cpu().numpy()
    for r in range(2):
        assert abs(k_loudness(tail[r]) - lev.target) <= 0.5, (r, k_loudness(tail[r]))
        ratio = out[r].double() / xd[r].double()
        ok = (xd[r].abs() > 1e-6).all(0)
        assert float(((ratio[0] - ratio[1])[ok] / ratio[0][ok]).abs().max()) <= 2 ** -22, r


# ---- 3. cuts, and what is stored --------------------------------------------------------------------------------------
def test_cuts_do_not_change_a_bit(dev):
    """the same hops of every listener cut into two schedules of ticks (T = 4, hops of 0 included), with a row on a
    record outside the state and a spare row past offsets[n]: outputs and states bit for bit; those rows keep their out
    samples and the state rows nobody lists stay zero"""
    S, R, n, T = 8, 6, 3, 4
    offsets = [0, 2, 3, 5]                                           # row 5 is spare
    records = [6, -1, 2, 0, 4, 1]                                    # row 1 is outside the state
    own = owners(offsets, n, R)
    total = [40, 33, 27]
    xs = torch.from_numpy(np.stack([voice(C, 40, 400 + r, db=-6.0 * r) for r in range(R)])).float().to(dev)
    res = []
    for seed in (0, 1):
        g = np.random.default_rng(500 + seed)
        sched, left = [], list(total)
        while any(left):
            h = [int(min(g.integers(0, T + 1), l)) for l in left]
            sched.append(h)
            left = [l - k for l, k in zip(left, h)]
        lev = Leveler(S, C, gate=-70.0, settle=0.04, window=0.3, device=dev)
        pos, got = [0] * n, [[] for _ in range(R)]
        for h in sched:
            y = torch.full((R, C, HOP * T), SENTINEL, device=dev)
            for r in range(R):
                if own[r] >= 0:
                    i = own[r]
                    y[r, :, :HOP * h[i]] = xs[r, :, HOP * pos[i]:HOP * (pos[i] + h[i])]
            y[5] = 7.0
            out = torch.full_like(y, 5.0)
            lev(y, su.i32(records, dev), su.i32(offsets, dev), hops=su.i32(h, dev), out=out)
            torch.cuda.synchronize()
            assert bool((out[1] == 5.0).all()) and bool((out[5] == 5.0).all())
            for r in range(R):
                if own[r] >= 0:
                    got[r].append(out[r, :, :HOP * h[own[r]]])
                    assert bool((out[r, :, HOP * h[own[r]]:] == 5.0).all())
            pos = [p + k for p, k in zip(pos, h)]
        res.append(([torch.cat(v, -1) if v else None for v in got], lev.state.clone()))
    for r in (0, 2, 3, 4):
        assert torch.equal(su.bits(res[0][0][r]), su.bits(res[1][0][r])), r
    assert torch.equal(su.bits(res[0][1]), su.bits(res[1][1]))
    assert not res[0][1][[1, 3, 5, 7]].any() and bool(res[0][1][[6, 2, 0, 4]].any())


def test_non_finite_hops_leave_the_state_unchanged(dev):
    """hops with NaN, Inf or a sample of 2^32: the state bit for bit as before, finite; out is y times the held gain"""
    lev = Leveler(3, C, settle=0.04, device=dev)
    x = torch.from_numpy(voice(C, 60, 600, db=-2.0)).float().to(dev)
    for t in range(10):
        lev(x[None, :, HOP * 5 * t:HOP * 5 * (t + 1)], [1])
    torch.cuda.synchronize()
    g = float(lev.gain[1])
    assert g != 0
    for bad in (float("nan"), float("inf"), -2.0 ** 32):
        before = lev.state.clone()
        y = x[None, :, :HOP * 2].clone()
        y[0, 1, 77] = bad
        y[0, 0, HOP + 3] = bad
        out = lev(y, [1])
        torch.cuda.synchronize()
        assert torch.equal(su.bits(lev.state), su.bits(before)) and bool(torch.isfinite(lev.state).all())
        fin = torch.isfinite(y)
        want = y * torch.tensor(10 ** (g / 20), dtype=torch.float32)
        assert float(((out - want)[fin]).abs().max()) <= 1e-6 * float(y[fin].abs().max())


def test_reset_and_moved_rows(dev):
    """a row moved by copying continues bit for bit; a reset row is a fresh leveler's"""
    x = torch.from_numpy(voice(C, 80, 700, db=-4.0)).float().to(dev)
    a, b = Leveler(4, C, settle=0.04, device=dev), Leveler(4, C, settle=0.04, device=dev)
    for t in range(10):
        a(x[None, :, HOP * 4 * t:HOP * 4 * (t + 1)], [1])
        b(x[None, :, HOP * 4 * t:HOP * 4 * (t + 1)], [1])
    b.state[3].copy_(b.state[1])
    b.reset([1])
    ya = a(x[None, :, HOP * 40:], [1])
    yb = b(x[None, :, HOP * 40:], [3])
    fresh = Leveler(4, C, settle=0.04, device=dev)
    yr, yf = b(x[None, :, :HOP * 40], [1]), fresh(x[None, :, :HOP * 40], [2])
    torch.cuda.synchronize()
    assert torch.equal(su.bits(ya), su.bits(yb)) and torch.equal(su.bits(a.state[1]), su.bits(b.state[3]))
    assert torch.equal(su.bits(yr), su.bits(yf)) and torch.equal(su.bits(b.state[1]), su.bits(fresh.state[2]))


# ---- 4. one CUDA graph ------------------------------------------------------------------------------------------------
def test_graph_replay_with_lists_rewritten(dev):
    """a captured in-place call with y, records, offsets and hops rewritten every replay, against eager calls of a twin:
    outputs and states bit for bit"""
    S, R, n, T = 10, 6, 3, 3
    live, twin = Leveler(S, C, settle=0.04, device=dev), Leveler(S, C, settle=0.04, device=dev)
    y = torch.zeros(R, C, HOP * T, device=dev)
    rec, off, hops = su.i32(list(range(R)), dev), su.i32([0, 2, 4, 6], dev), su.i32([0] * n, dev)
    graph = su.captured(lambda: live(y, rec, off, hops=hops, out=y))
    src = torch.from_numpy(np.stack([voice(C, T * 16, 800 + r, db=-5.0 * r) for r in range(R)])).float().to(dev)
    for t in range(16):
        g = torch.Generator().manual_seed(900 + t)
        rl = torch.randperm(S, generator=g)[:R].tolist()
        if t % 4 == 3:
            rl[t % R] = -1
        ol = sorted(torch.randint(0, R + 1, (n - 1,), generator=g).tolist())
        ol = [0] + ol + [R - (t % 2)]
        hl = su.hop_mix(n, T, 950 + t)
        y.copy_(src[:, :, HOP * T * t:HOP * T * (t + 1)])
        rec.copy_(su.i32(rl, dev))
        off.copy_(su.i32(ol, dev))
        hops.copy_(su.i32(hl, dev))
        want = y.clone()
        graph.replay()
        twin(want, su.i32(rl, dev), su.i32(ol, dev), hops=su.i32(hl, dev), out=want)
        su.assert_same({"y": y}, {"y": want}, {"lev": live}, {"lev": twin}, t)


# ---- 5. on the separator ----------------------------------------------------------------------------------------------
def test_full_tick_on_the_separator(model, dev):
    """44.1 kHz packets down, FIFO, advance_target_rows, the leveler in place on the rows, the mixer, up to 44.1 kHz and
    the limiter, all in one captured graph replayed with counts rewritten in place: bit for bit the eager chain"""
    def build(o):
        o["lev"] = Leveler(su.TICK_S, C, gate=-90.0, settle=0.04, min_gain=-40.0, device=dev)

    def rows(o, b, y, slots, rec, off):
        o["lev"](y, rec, off, hops=b["hops"], out=y)

    live = su.separator_tick(model[0], dev, build, rows=rows)
    assert int((live["lev"].state[:, 0, 1].view(torch.int32) > 0).sum()) == len(su.TICK_RECS)   # every voice measured
    print(f"\nseparated voices (untrained weights): loudness {live['lev'].loudness.tolist()} LUFS, "
          f"gains {live['lev'].gain.tolist()} dB")


def test_advance_targets_view(model, dev):
    """the output of advance_targets served as y.view(n K, S, 128 T) with offsets i K and records g_i K + k: bit for bit
    the same rows leveled one listener per row with their group's hops"""
    net, _ = model
    G, K, n, T = 3, 2, 2, 2
    groups = [2, 0]
    clips, _ = su.clips(n, 3 * T, 9950, dev)
    e = su.embeds(n, K, 9960, dev)
    st = net.init_buffers(G * K, dev)
    a, b = Leveler(G * K, C, gate=-90.0, settle=0.008, device=dev), Leveler(G * K, C, gate=-90.0, settle=0.008, device=dev)
    recs = su.recs(groups, K)
    with torch.no_grad():
        for t in range(3):
            hops = [T, 1] if t != 1 else [0, T]
            x = torch.stack([su.chunk(clips[i], t * T, T) for i in range(n)]).contiguous()
            y = net.advance_targets(x, e, st, groups, hops=hops).view(n * K, C, HOP * T)
            ya = a(y, recs, [i * K for i in range(n + 1)], hops=hops)
            yb = b(y, recs, hops=[h for h in hops for _ in range(K)])
            torch.cuda.synchronize()
            for i in range(n):
                w = HOP * hops[i]
                assert torch.equal(su.bits(ya[i * K:(i + 1) * K, :, :w]), su.bits(yb[i * K:(i + 1) * K, :, :w])), (t, i)
    assert torch.equal(su.bits(a.state), su.bits(b.state)) and bool(a.state[recs].any())


def test_warm_join_is_leveled_from_the_start(model, dev):
    """listener A with a 64-frame history for 48 hops; B joins warm (replaying 48 frames) and is primed with
    lev(y_warm, [B], [0, 1], hops=used): 8 hops later its gain is within 0.5 dB of a leveler that heard B from the start,
    while a cold-joined B, leveled only from the join on, still sits at 0 dB"""
    net, _ = model
    A, B = 0, 1
    clips, _ = su.clips(1, 56, 9970, dev)
    e = su.emb(2, 9980, dev)
    st, ref, cold = (net.init_buffers(2, dev) for _ in range(3))
    hist = net.target_history(st, 64)
    kw = {"gate": -90.0, "settle": 0.256, "min_gain": -40.0, "max_gain": 40.0, "device": dev}   # untrained voices are loud
    lev, lev_ref, lev_cold = Leveler(2, C, **kw), Leveler(2, C, **kw), Leveler(2, C, **kw)
    off = su.i32([0, 2], dev)

    def tick(s, t, recs, h=None):
        x = su.chunk(clips[:1], t).contiguous()
        return net.advance_target_rows(x, e, s, su.i32(recs, dev), off, history=h)

    with torch.no_grad():
        for t in range(48):
            tick(st, t, [A, -1], hist)
            tick(cold, t, [A, -1])
            y = tick(ref, t, [A, B])
            lev_ref(y, [A, B], [0, 2], out=y)
        y_warm, used = net.join_targets(st, [B], [A], e[[B]], history=hist)
        net.join_targets(cold, [B], [A], e[[B]])
        scratch = torch.empty_like(y_warm)
        lev(y_warm, [B], [0, 1], hops=used, out=scratch)
        for t in range(48, 56):
            for s, lv in ((st, lev), (ref, lev_ref), (cold, lev_cold)):
                y = tick(s, t, [A, B])
                lv(y, [A, B], [0, 2], out=y)
        torch.cuda.synchronize()
    assert used.tolist() == [48]
    g, g_ref = float(lev.gain[B]), float(lev_ref.gain[B])
    print(f"\njoined voice: warm gain {g:+.2f} dB, from the start {g_ref:+.2f} dB, cold {float(lev_cold.gain[B]):+.2f} dB")
    assert abs(g - g_ref) <= 0.5 and -40.0 < g_ref < 40.0 and g_ref != 0.0
    assert float(lev_cold.gain[B]) == 0.0 and int(lev_cold.state[B, 0, 1].view(torch.int32)) <= 8
