"""The band compressor on the GPU (BandCompressor, l2h_band_compressor), on seeded inputs and fresh compressors.

Oracles: the input itself, delayed by D (a fresh state, and a profile of 0 dB gains at ratio 1, bit for bit); the float64
numpy model of tests/test_band_compressor_cpu.py (telemetry to 0.01 dB, output to 1e-3 of each row's peak); the ears'
level ratio of the input (bit for bit); the same hops cut into other ticks (bit for bit); guard regions around y and out; eager calls
(graph replays, bit for bit), on the seeded separator's full 44.1 kHz tick."""
import math

import numpy as np
import pytest
import torch

import serving_util as su
from lookoncetohear_b200 import BandCompressor, Leveler
from serving_util import HOP, SENTINEL, dev, model  # noqa: F401
from test_band_compressor_cpu import BANK, model_hop, model_state, set_profile, speech

pytestmark = pytest.mark.gpu

C, D = 2, 64


def delayed(x, D=D):
    """x [..., N] delayed by D samples, zeros first"""
    return torch.nn.functional.pad(x, (D, 0))[..., :x.shape[-1]]


def profile(g, n):
    """n seeded profiles: per-ear gains [n, C, 5] in [-10, 20] dB with the ears up to 8 dB apart, knees [n, 5] in
    [-60, -30] dBFS, ratios [n, 5] in [1, 4]"""
    gains = g.uniform(-10, 12, (n, 1, 5)) + g.uniform(0, 8, (n, C, 5))
    return gains, g.uniform(-60, -30, (n, 5)), g.uniform(1, 4, (n, 5))


# ---- 1. 0 dB everywhere: the delayed input bit for bit -----------------------------------------------------------------
@pytest.mark.parametrize("flat", [False, True])
def test_zero_db_is_the_delayed_input(dev, flat):
    """a fresh state, and a set profile of 0 dB gains at ratio 1 over a compressing one: every output sample is the
    input's D samples before, -0 and subnormals included, in place and not, across ticks of 1 to 3 hops"""
    S, n, T = 6, 3, 3
    x = su.signals(n, C, HOP * 12, 7, dev) * 4
    x[0, 0, 10:20] = -0.0
    x[1, 1, 300:340] = 1e-40
    a = BandCompressor(S, C, device=dev)
    b = BandCompressor(S, C, device=dev)
    if flat:
        for c in (a, b):
            c.set_profile([4, 1, 0], [6.0] * 5, knees=-50.0, ratios=3.0)
            c(x[:, :, :HOP * 3].clone(), [4, 1, 0])                 # the compressing profile runs for a while
            c.reset([4, 1, 0])
            c.set_profile([4, 1, 0], [0.0] * 5, knees=-50.0, ratios=1.0)
    outs_a, outs_b, pos = [], [], 0
    for T_t in (1, 3, 2, 3, 1, 2):
        y = x[:, :, HOP * pos:HOP * (pos + T_t)].clone()
        outs_a.append(a(y, su.i32([4, 1, 0], dev)))
        b(y, [4, 1, 0], out=y)
        outs_b.append(y)
        pos += T_t
    torch.cuda.synchronize()
    want = su.bits(delayed(x))
    assert torch.equal(su.bits(torch.cat(outs_a, -1)), want) and torch.equal(su.bits(torch.cat(outs_b, -1)), want)
    assert bool((a.level[[4, 1, 0]] > -80).all()) and not a.gain.any()   # measured, never a gain


# ---- 2. the model -----------------------------------------------------------------------------------------------------
def test_random_profiles_agree_with_the_model(dev):
    """slots scattered over the state, ragged hops (0 included), voices from -30 to 0 dB, random per-ear profiles set at
    the start and again between ticks: telemetry to 0.01 dB, output to 1e-3 of each row's peak"""
    S, n, T, ticks = 9, 4, 3, 30
    g = np.random.default_rng(11)
    slots = [7, 2, 5, 0]
    sched = [su.hop_mix(n, T, 1100 + t) for t in range(ticks)]
    total = [sum(s[i] for s in sched) for i in range(n)]
    xs = [speech(C, total[i], 1200 + i, db=[-30.0, -6.0, 0.0, -15.0][i]) for i in range(n)]
    cmp = BandCompressor(S, C, device=dev)
    mst = [model_state(C, 5, 129) for _ in range(n)]
    pos, want, got = [0] * n, [[] for _ in range(n)], [[] for _ in range(n)]
    for t in range(ticks):
        if t in (0, 12):
            gains, knees, ratios = profile(g, n)
            cmp.set_profile(slots, torch.from_numpy(gains), torch.from_numpy(knees), torch.from_numpy(ratios))
            for i in range(n):
                set_profile(mst[i], gains[i], knees[i], ratios[i])
        y = torch.full((n, C, HOP * T), SENTINEL)
        for i in range(n):
            h = sched[t][i]
            seg = xs[i][:, HOP * pos[i]:HOP * (pos[i] + h)]
            y[i, :, :HOP * h] = torch.from_numpy(seg).float()
            for k in range(h):
                want[i].append(model_hop(mst[i], seg[:, HOP * k:HOP * (k + 1)], BANK))
            pos[i] += h
        out = cmp(y.to(dev), su.i32(slots, dev), hops=su.i32(sched[t], dev))
        for i in range(n):
            got[i].append(out[i, :, :HOP * sched[t][i]].cpu())
    torch.cuda.synchronize()
    for i in range(n):
        a, b = torch.cat(got[i], -1).double().numpy(), np.concatenate(want[i], 1)
        assert np.abs(a - b).max() <= 1e-3 * np.abs(b).max(), i
        with np.errstate(divide="ignore"):
            lvl = 10 * np.log10(mst[i]["S"])
        assert np.abs(cmp.level[slots[i]].double().cpu().numpy() - lvl).max() <= 0.01, i
        assert np.abs(cmp.gain[slots[i]].double().cpu().numpy() - mst[i]["g"]).max() <= 0.01, i
    assert max(np.abs(m["g"] - m["prof"]).max() for m in mst) > 3          # the compression did act


def test_ild_is_kept(dev):
    """equal gains in both ears and compression active: a source 12 dB softer in the right ear (a quarter of the left's
    amplitude, which scales every product exactly) stays exactly that much softer at every sample"""
    x = torch.from_numpy(speech(1, 60, 1300, db=-3.0)).float().to(dev)
    y = torch.cat([x, x * 0.25])[None]
    cmp = BandCompressor(2, C, device=dev)
    cmp.set_profile([1], [4.0, 8.0, 14.0, 18.0, 10.0], knees=-55.0, ratios=[2, 3, 3, 4, 2])
    out = torch.cat([cmp(y[:, :, HOP * 4 * t:HOP * 4 * (t + 1)], [1]) for t in range(15)], -1)
    torch.cuda.synchronize()
    assert torch.equal(cmp.gain[1, 0], cmp.gain[1, 1]) and float((cmp.gain[1] - 8.0).abs().max()) > 1
    assert torch.equal(out[0, 1], out[0, 0] * 0.25) and float(out.abs().max()) > 0


# ---- 3. cuts, and what is stored --------------------------------------------------------------------------------------
def test_cuts_do_not_change_a_bit(dev):
    """the same hops of every slot through ticks of T = 1 and through ragged ticks of T = 3: outputs and states bit for
    bit"""
    S, n, hops = 6, 3, 24
    slots = [5, 0, 3]
    xs = torch.from_numpy(np.stack([speech(C, hops, 1400 + i, db=-8.0 * i) for i in range(n)])).float().to(dev)
    g = np.random.default_rng(14)
    gains, knees, ratios = profile(g, n)
    res = []
    for T in (1, 3):
        cmp = BandCompressor(S, C, device=dev)
        cmp.set_profile(slots, torch.from_numpy(gains), torch.from_numpy(knees), torch.from_numpy(ratios))
        rng = np.random.default_rng(1500 + T)
        pos, got = [0] * n, [[] for _ in range(n)]
        while min(pos) < hops:
            h = [int(min(rng.integers(0, T + 1), hops - p)) for p in pos] if T > 1 else [int(p < hops) for p in pos]
            y = torch.full((n, C, HOP * T), SENTINEL, device=dev)
            for i in range(n):
                y[i, :, :HOP * h[i]] = xs[i, :, HOP * pos[i]:HOP * (pos[i] + h[i])]
            out = cmp(y, su.i32(slots, dev), hops=su.i32(h, dev))
            for i in range(n):
                got[i].append(out[i, :, :HOP * h[i]])
            pos = [p + k for p, k in zip(pos, h)]
        torch.cuda.synchronize()
        res.append((torch.stack([torch.cat(v, -1) for v in got]), cmp.state.clone()))
    assert torch.equal(su.bits(res[0][0]), su.bits(res[1][0])) and torch.equal(su.bits(res[0][1]), su.bits(res[1][1]))
    assert bool(res[0][1][slots].any()) and not res[0][1][[1, 2, 4]].any()


def test_store_rules_with_guards(dev):
    """rows whose CUDA slot lies outside the state, or whose hop count lies outside [1, T], store nothing: their out
    rows, every out sample past 128 h and a guard region around y and out keep their values, and the state rows of the
    slots nobody advanced keep theirs"""
    S, n, T, G = 6, 6, 2, 1000
    slots = [4, -1, 2, 3, 0, 7]
    hops = [2, 2, 0, 1, 3, 1]
    flat_y = torch.full((G + n * C * HOP * T + G,), 9.0, device=dev)
    flat_o = torch.full((G + n * C * HOP * T + G,), 5.0, device=dev)
    y = flat_y[G:G + n * C * HOP * T].view(n, C, HOP * T)
    y.copy_(su.signals(n, C, HOP * T, 16, dev))
    keep = y.clone()
    out = flat_o[G:G + n * C * HOP * T].view(n, C, HOP * T)
    cmp = BandCompressor(S, C, device=dev)
    cmp.set_profile(list(range(S)), [3.0] * 5, knees=-60.0, ratios=2.0)
    before = cmp.state.clone()
    cmp(y, su.i32(slots, dev), hops=su.i32(hops, dev), out=out)
    torch.cuda.synchronize()
    assert bool((flat_o[:G] == 5.0).all()) and bool((flat_o[-G:] == 5.0).all())
    assert bool((flat_y[:G] == 9.0).all()) and bool((flat_y[-G:] == 9.0).all()) and torch.equal(y, keep)
    for i in (1, 2, 4, 5):
        assert bool((out[i] == 5.0).all()), i
    assert bool((out[3, :, HOP:] == 5.0).all()) and not bool((out[3, :, :HOP] == 5.0).any())
    assert not bool((out[0] == 5.0).any()) and bool(torch.isfinite(out).all())
    assert torch.equal(cmp.state[[0, 1, 2, 5]], before[[0, 1, 2, 5]])
    assert not torch.equal(cmp.state[4], before[4]) and not torch.equal(cmp.state[3], before[3])


# ---- 4. state rows ----------------------------------------------------------------------------------------------------
def test_reset_moved_rows_and_profiles_between_ticks(dev):
    """a slot moved by copying continues bit for bit; a reset slot is a fresh compressor's; a profile set between ticks
    takes effect from the next hop across one hop's ramp"""
    x = torch.from_numpy(speech(C, 80, 1700, db=-4.0)).float().to(dev)
    a, b = BandCompressor(4, C, device=dev), BandCompressor(4, C, device=dev)
    for c in (a, b):
        c.set_profile([1], [[[2.0, 5.0, 9.0, 12.0, 6.0], [0.0, 3.0, 12.0, 16.0, 8.0]]], knees=-45.0, ratios=2.5)
    for t in range(10):
        a(x[None, :, HOP * 4 * t:HOP * 4 * (t + 1)], [1])
        b(x[None, :, HOP * 4 * t:HOP * 4 * (t + 1)], [1])
    b.state[3].copy_(b.state[1])
    b.reset([1])
    ya = a(x[None, :, HOP * 40:], [1])
    yb = b(x[None, :, HOP * 40:], [3])
    fresh = BandCompressor(4, C, device=dev)
    yr, yf = b(x[None, :, :HOP * 40], [1]), fresh(x[None, :, :HOP * 40], [2])
    torch.cuda.synchronize()
    assert torch.equal(su.bits(ya), su.bits(yb)) and torch.equal(su.bits(a.state[1]), su.bits(b.state[3]))
    assert torch.equal(su.bits(yr), su.bits(yf)) and torch.equal(su.bits(b.state[1]), su.bits(fresh.state[2]))
    # a +6 dB flat profile set between ticks: the next hop ramps to it, the one after is twice the delayed input
    c = BandCompressor(2, C, device=dev)
    y0 = c(x[None, :, :HOP * 2], [0])
    c.set_profile([0], [20 * math.log10(2.0)] * 5)
    y1 = c(x[None, :, HOP * 2:HOP * 4], [0])
    torch.cuda.synchronize()
    assert torch.equal(su.bits(y0), su.bits(delayed(x[None, :, :HOP * 2])))
    want = delayed(x[None])[..., HOP * 3:HOP * 4] * 2
    assert float((y1[..., HOP:] - want).abs().max()) <= 1e-5 * float(x.abs().max())
    assert float((y1[..., 0] - delayed(x[None])[..., HOP * 2]).abs().max()) <= 0.01 * float(x.abs().max())


def test_non_finite_input_keeps_state_and_output_finite(dev):
    """NaN, Inf and 2^32 samples enter as 0: the hop is not measured (the detectors keep their bits), every output sample
    and state word stays finite"""
    cmp = BandCompressor(3, C, device=dev)
    cmp.set_profile([2], [6.0, 9.0, 12.0, 15.0, 9.0], knees=-50.0, ratios=3.0)
    x = torch.from_numpy(speech(C, 40, 1800, db=-2.0)).float().to(dev)
    cmp(x[None, :, :HOP * 20], [2])
    torch.cuda.synchronize()
    for bad in (float("nan"), float("inf"), -2.0 ** 32):
        S_before = cmp.state[2, 0, 10:15].clone()
        y = x[None, :, HOP * 20:HOP * 22].clone()
        y[0, 1, 77] = bad
        y[0, 0, HOP + 3] = bad
        out = cmp(y, [2])
        torch.cuda.synchronize()
        assert torch.equal(su.bits(cmp.state[2, 0, 10:15]), su.bits(S_before)), bad
        assert bool(torch.isfinite(cmp.state).all()) and bool(torch.isfinite(out).all()), bad
    assert float(cmp.gain[2].abs().max()) > 1


# ---- 5. the full tick, one CUDA graph ---------------------------------------------------------------------------------
def test_full_tick_on_the_separator(model, dev):
    """44.1 kHz packets down, FIFO, advance_target_rows, the leveler on the rows, the mixer, the compressor in place on the
    mixer's sum, up to 44.1 kHz and the limiter, all in one captured graph replayed with counts rewritten in place: bit
    for bit the eager chain"""
    def build(o):
        o["lev"] = Leveler(su.TICK_S, C, gate=-90.0, settle=0.04, min_gain=-40.0, device=dev)
        o["cmp"] = BandCompressor(su.TICK_S, C, device=dev)
        o["cmp"].set_profile([0, 1, 2], [[0.0, 4.0, 10.0, 15.0, 8.0]] * 3, knees=-40.0, ratios=[1.5, 2, 2, 2.5, 2])

    def rows(o, b, y, slots, rec, off):
        o["lev"](y, rec, off, hops=b["hops"], out=y)

    def mixed(o, b, y, slots, rec, off):
        o["cmp"](b["mix"], slots, hops=b["hops"], out=b["mix"])

    live = su.separator_tick(model[0], dev, build, rows=rows, mixed=mixed)
    assert bool(torch.isfinite(live["cmp"].level[:3]).all()) and float(live["cmp"].gain[:3].abs().max()) > 1
    print(f"\nmixed voices (untrained weights): band levels {live['cmp'].level[:3].tolist()} dBFS, "
          f"gains {live['cmp'].gain[:3, 0].tolist()} dB")
