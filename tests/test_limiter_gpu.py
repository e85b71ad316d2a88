"""The limiter on the GPU (Limiter, l2h_limiter), on seeded inputs and fresh limiters.

Oracles: the input delayed by La samples (below the ceiling, bit for bit); the ceiling itself (an exact fp32 comparison);
the float64 numpy model of tests/test_limiter_cpu.py (to 1e-5 of each row's peak, the telemetry too); the same streams
cut into other pushes (bit for bit); eager calls (graph replays, bit for bit); and, on the seeded separator, the eager
44.1 kHz chain."""
import math

import numpy as np
import pytest
import torch

import serving_util as su
from lookoncetohear_b200 import Limiter, PacketResampler
from serving_util import HOP, SENTINEL, dev, model  # noqa: F401
from test_limiter_cpu import CEILING, cuts, loud, model_push, model_state

pytestmark = pytest.mark.gpu

C, TOL = 2, 1e-5


def stream(lim, xs, pushes, slots, unit=1, L=None):
    """the signals xs [n, C, N] (CUDA) pushed through `slots` tick by tick, row i pushing pushes[i][t] * unit samples
    (CUDA lists, rows padded with NaN): the concatenated outputs of every row"""
    n = xs.shape[0]
    L = L or unit * max(max(p) for p in pushes)
    pos, got = [0] * n, [[] for _ in range(n)]
    for t in range(max(len(p) for p in pushes)):
        cnt = [p[t] if t < len(p) else 0 for p in pushes]
        x = torch.full((n, C, L), SENTINEL, device=xs.device)
        for i in range(n):
            x[i, :, :cnt[i] * unit] = xs[i, :, pos[i]:pos[i] + cnt[i] * unit]
        y = lim(x, su.i32(cnt, xs.device), su.i32(slots, xs.device), unit=unit)
        for i in range(n):
            got[i].append(y[i, :, :cnt[i] * unit])
            pos[i] += cnt[i] * unit
    return [torch.cat(g, -1) for g in got]


def model_stream(x, pushes, ceiling, La, step, st=None):
    """the model of one row: x [C, N] float64 in pushes; (y, state)"""
    st = st or model_state(x.shape[0], La)
    ys, pos = [], 0
    for m in pushes:
        if m:
            ys.append(model_push(st, x[:, pos:pos + m], ceiling, La, step))
        pos += m
    return np.concatenate(ys, 1), st


def delayed(x, La):
    return torch.nn.functional.pad(x, (La, 0))[..., :x.shape[-1]]


def loud_inputs(N, dev):
    """[4, C, N] float32: three voices at mixer gain 16 summed, impulses up to FLT_MAX, full-scale and 8x squares, and a
    loud signal with NaN and Inf in it"""
    g = torch.Generator().manual_seed(5)
    voices = 16 * (0.1 * torch.randn(3, C, N, generator=g)).sum(0)
    imp = torch.zeros(C, N)
    for k, v in zip(range(300, N, 1700), [1e3, -1e30, torch.finfo(torch.float32).max, -2.0, 1e-3, 50.0]):
        imp[0, k], imp[1, k + 3] = v, -v / 3
    t = torch.arange(N)
    sq = torch.stack([torch.where((t // 55) % 2 == 0, 1.0, -1.0), torch.where((t // 37) % 2 == 0, 8.0, -8.0)])
    bad = torch.from_numpy(loud(C, N, 6)).float()
    bad[0, 1000], bad[1, 2500], bad[0, 2501], bad[1, 4000:4010] = float("nan"), float("inf"), -float("inf"), float("nan")
    return torch.stack([voices, imp, sq, bad]).to(dev)


# ---- 1. below the ceiling the input, delayed, bit for bit -------------------------------------------------------------
def test_transparent_below_the_ceiling(dev):
    N = 6000
    x = su.signals(3, C, N, 1, dev) * 1.5                              # peaks near 0.7, under the -1 dBFS ceiling
    x[0, 0, 100:110] = -0.0
    x[1, 1, 200:210] = 1e-40                                           # subnormals and signed zeros pass as they are
    assert float(x.abs().max()) <= CEILING
    lim = Limiter(5, C, 44100, device=dev)
    ys = stream(lim, x, [cuts(N, 10 + i, 700) for i in range(3)], [4, 0, 2])
    for i in range(3):
        assert torch.equal(su.bits(ys[i]), su.bits(delayed(x[i], lim.lookahead))), i
    assert not lim.limited.any() and not lim.reduction.any()


# ---- 2. the ceiling, the linked gain and the model ------------------------------------------------------------------
@pytest.mark.parametrize("La_s,release", [(0.001, 80.0), (0.0, 80.0), (0.003, 2000.0)])
def test_loud_inputs_stay_under_the_ceiling(dev, La_s, release):
    """voices at gain 16, impulses up to FLT_MAX, squares, NaN/Inf, in random pushes: every sample finite and
    |y| <= ceiling exactly; one gain for both channels; the model to 1e-5 of each row's peak; `limited` exactly and `reduction` to 1e-3 dB"""
    N = 9000
    x = loud_inputs(N, dev)
    n = x.shape[0]
    lim = Limiter(6, C, 44100, lookahead=La_s, release=release, device=dev)
    pushes = [cuts(N, 20 + i, 900) for i in range(n)]
    slots = [5, 1, 3, 0]
    ys = stream(lim, x, pushes, slots)
    torch.cuda.synchronize()
    ceiling = torch.tensor(CEILING, dtype=torch.float32)
    for i in range(n):
        y = ys[i].cpu()
        assert bool(torch.isfinite(y).all()), i
        assert bool((y.abs() <= ceiling).all()), (i, float(y.abs().max()))
        xd = delayed(x[i], lim.lookahead).cpu()
        both = torch.isfinite(xd).all(0) & (xd != 0).all(0) & (y.abs() > 1e-30).all(0)   # normal products
        g = (y.double() / xd.double())[:, both]
        if g.shape[1]:
            assert float(((g[0] - g[1]).abs() / g.abs().max(0).values).max()) <= 2 ** -22, i   # fp32 rounding only
        want, st = model_stream(x[i].double().cpu().numpy(), pushes[i], CEILING, lim.lookahead, lim.release_step)
        err = np.abs(y.double().numpy() - want).max()
        assert err <= TOL * np.abs(want).max(), (i, err)
        assert int(lim.limited[slots[i]]) == st["limited"], i
        assert abs(float(lim.reduction[slots[i]]) - st["db"]) <= 1e-3, i
    assert float(ys[0].abs().max()) > 0.99 * CEILING                   # the loud voices reach the ceiling


# ---- 3. the cut into pushes never changes a bit --------------------------------------------------------------------
@pytest.mark.parametrize("unit", [1, 128])
def test_cuts_do_not_change_a_bit(dev, unit):
    """one stream per row pushed in two halves, and cut into random pushes (0 .. 3 hops at unit 128, 0 .. 1000 samples
    at unit 1): outputs and states bit for bit"""
    T = 3 if unit == 128 else 1000
    N = unit * 40 if unit == 128 else 5000
    x = loud_inputs(max(N, 4096), dev)[..., :N].contiguous()
    n = x.shape[0]
    outs, states = [], []
    for sched in ([[N // unit // 2] * 2] * n, [cuts(N // unit, 30 + i, T + 1) for i in range(n)]):
        lim = Limiter(n, C, 44100, device=dev)
        outs.append(stream(lim, x, sched, list(range(n)), unit=unit))
        states.append(lim.state.clone())
    for i in range(n):
        assert torch.equal(su.bits(outs[0][i]), su.bits(outs[1][i])), i
    assert torch.equal(su.bits(states[0]), su.bits(states[1]))


# ---- 4. what is stored --------------------------------------------------------------------------------------------
def test_rows_that_store_nothing(dev):
    """CUDA slots outside the limiter, counts whose count * unit lies outside [0, L], and counts of 0: their out rows keep
    the guard and their state rows do not change; the other rows' samples past their count are not written"""
    S, L, unit = 6, 256, 2
    lim = Limiter(S, C, 16000, device=dev)
    src = loud_inputs(4096, dev)
    lim(src[..., :L].contiguous(), [L // unit] * 4, [0, 1, 2, 3], unit=unit)
    x = src[[3, 2, 1, 0, 3, 2], :, L:2 * L].contiguous()
    frame = torch.full((8, C, L), 7.0, device=dev)                     # 7.0 around out: an out-of-bounds write shows
    out = frame[1:7]
    out.fill_(SENTINEL)
    before = lim.state.clone()
    slots, counts = [0, 6, -1, 2, 3, 1], [50, 10, 10, 129, -1, 0]
    lim(x, su.i32(counts, dev), su.i32(slots, dev), unit=unit, out=out)
    torch.cuda.synchronize()
    assert bool(out[1:].isnan().all()) and bool(out[0, :, 100:].isnan().all()) and not bool(out[0, :, :100].isnan().any())
    assert bool((frame[0] == 7.0).all()) and bool((frame[7] == 7.0).all())
    changed = [bool((su.bits(lim.state[s]) != su.bits(before[s])).any()) for s in range(S)]
    assert changed == [True, False, False, False, False, False]


# ---- 5. fresh, reset and moved rows -------------------------------------------------------------------------------
def test_reset_and_moved_rows(dev):
    """a listener moved by copying its rows continues bit for bit, and a reset row is a fresh limiter's"""
    N, S = 8000, 4
    x = loud_inputs(N, dev)[[0, 3]]
    p = cuts(N, 40, 600)
    half = len(p) // 2
    a, b = Limiter(S, C, 44100, device=dev), Limiter(S, C, 44100, device=dev)
    ya = stream(a, x[:1], [p[:half]], [1])[0]
    stream(b, x[:1], [p[:half]], [1])
    b.state[3].copy_(b.state[1])
    b.reset([1])
    ya2 = stream(a, x[:1, :, sum(p[:half]):], [p[half:]], [1])[0]
    yb2 = stream(b, x[:1, :, sum(p[:half]):], [p[half:]], [3])[0]
    assert torch.equal(su.bits(ya2), su.bits(yb2))
    assert torch.equal(su.bits(a.state[1]), su.bits(b.state[3]))
    assert not b.state[1].any()
    fresh = Limiter(S, C, 44100, device=dev)
    yr = stream(b, x[1:], [p], [1])[0]
    yf = stream(fresh, x[1:], [p], [2])[0]
    assert torch.equal(su.bits(yr), su.bits(yf)) and ya.shape[-1] == sum(p[:half])


# ---- 6. per-slot ceilings -----------------------------------------------------------------------------------------
def test_set_ceiling_applies_to_later_samples(dev):
    """a slot's own ceiling holds for every sample pushed after the set and leaves the other slots alone; 0 returns the
    slot to the limiter's ceiling; the model with the slot's ceiling word agrees"""
    N = 2048
    x = loud_inputs(2 * N, dev)[[0, 0]]
    lim = Limiter(3, C, 44100, device=dev)
    La = lim.lookahead
    st = [model_state(C, La), model_state(C, La)]
    xs = x.double().cpu().numpy()
    ys = [lim(x[:, :, :N], [N, N], [0, 2])]
    lim.set_ceiling([2], [0.25])
    ys.append(lim(x[:, :, N:], [N, N], [0, 2]))
    torch.cuda.synchronize()
    assert float(ys[1][1, :, La:].abs().max()) <= 0.25 < float(ys[1][0, :, La:].abs().max())
    for k, y in enumerate(ys):
        if k == 1:
            st[1]["ceil"] = float(np.float32(0.25))
        for i in range(2):
            want = model_push(st[i], xs[i, :, k * N:(k + 1) * N], CEILING, La, lim.release_step)
            assert np.abs(y[i].double().cpu().numpy() - want).max() <= TOL * np.abs(want).max(), (i, k)
    lim.set_ceiling([2], 0)
    assert float(lim.state[2, 0, 1]) == 0.0


# ---- 7. one CUDA graph ----------------------------------------------------------------------------------------------
def test_graph_replay_with_lists_rewritten(dev):
    """a captured call with its x, slots and counts rewritten in place every replay, against eager calls of a twin: the
    outputs and the states bit for bit"""
    S, n, L = 6, 4, 600
    live, twin = Limiter(S, C, 44100, device=dev), Limiter(S, C, 44100, device=dev)
    x = torch.zeros(n, C, L, device=dev)
    slots, counts = su.i32(list(range(n)), dev), su.i32([0] * n, dev)
    y = torch.full((n, C, L), SENTINEL, device=dev)
    graph = su.captured(lambda: live(x, counts, slots, out=y))
    src = loud_inputs(L * 12, dev)
    for t in range(12):
        g = torch.Generator().manual_seed(50 + t)
        sl = torch.randperm(S, generator=g)[:n].tolist()
        if t % 4 == 3:
            sl[t % n] = -1
        cn = [[0, 1, 441, 600, 700][int(k)] for k in torch.randint(0, 5, (n,), generator=g)]
        x.copy_(src[:, :, L * t:L * (t + 1)])
        slots.copy_(su.i32(sl, dev))
        counts.copy_(su.i32(cn, dev))
        y.fill_(SENTINEL)
        graph.replay()
        want = torch.full_like(y, SENTINEL)
        twin(x, su.i32(cn, dev), su.i32(sl, dev), out=want)
        su.assert_same({"y": y}, {"y": want}, {"lim": live}, {"lim": twin}, t)


# ---- 8. the 44.1 kHz tick on the separator --------------------------------------------------------------------------
def test_full_tick_on_the_separator(model, dev):
    """44.1 kHz packets down, FIFO, advance_target_rows, the mixer at gains up to 16, up to 44.1 kHz and the limiter, all
    in one captured graph replayed with counts rewritten in place: under the ceiling and bit for bit the eager chain.
    It also limits the mixer's 16 kHz output before `up` and reports how far upsampling takes that over the ceiling."""
    S, T = su.TICK_S, su.TICK_T
    peak = {"post": 0.0, "pre": 0.0, "played": 0}

    def build(o):
        o["mix"].set_gains(su.TICK_RECS, [16.0, 12.0, 16.0, 4.0])
        o["lim16"] = Limiter(S, C, 16000, device=dev)
        o["up16"] = PacketResampler(16000, 44100, S, C, HOP * T, device=dev)

    def after(o, b, y, slots, rec, off):                                    # limiting before `up` instead
        o["lim16"](b["mix"], b["hops"], slots, unit=HOP, out=b["m16"])
        o["up16"](b["m16"], b["hops"], slots, unit=HOP, out=b["pre"], out_counts=b["ocp"])

    def each(b, t):
        oc, ocp = b["oc44"].cpu().tolist(), b["ocp"].cpu().tolist()
        for i in range(su.TICK_N):
            if oc[i]:
                z = b["out"][i, :, :oc[i]]
                assert bool(torch.isfinite(z).all()) and float(z.abs().max()) <= CEILING, (t, i)
                peak["post"] = max(peak["post"], float(z.abs().max()))
                peak["played"] += oc[i]
            if ocp[i]:
                peak["pre"] = max(peak["pre"], float(b["pre"][i, :, :ocp[i]].abs().max()))

    live = su.separator_tick(model[0], dev, build, after=after, each=each,
                             bufs={"m16": HOP * T, "pre": 353 * T, "ocp": None})
    assert peak["played"] > 0 and int(live["lim"].limited.sum()) > 0     # the gains of 16 did call for limiting
    post, pre = (20 * math.log10(peak[k] / CEILING) for k in ("post", "pre"))
    print(f"\n44.1 kHz tick: limiter after up peaks at {post:+.2f} dB re the ceiling; "
          f"limiting at 16 kHz before up peaks at {pre:+.2f} dB")
