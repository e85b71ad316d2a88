"""The band compressor on its Linkwitz-Riley banks on the GPU (BandCompressor(bank="lr4" / "lr8"),
l2h_band_compressor_lr), for both orders and K = 1, 2, 5 and 16 bands, on seeded inputs and fresh compressors.

Oracles: the float64 numpy model of tests/test_band_compressor_lr_cpu.py (telemetry to 0.01 dB; output within a bound
made from the cascade's own roundoff, measured by running the same sections in float32, and never looser than 1e-3 of
each row's peak); the input itself (K = 1 at 0 dB, bit for bit); the same hops cut into other ticks, in place and not
(bit for bit); guard regions around y and out; eager calls (graph replays, bit for bit), also on the seeded separator's
44.1 kHz tick, where the compressed mixer's sum is checked against the model too."""
import numpy as np
import pytest
import torch
from scipy.signal import sosfilt

import serving_util as su
from lookoncetohear_b200 import BandCompressor
from serving_util import HOP, SENTINEL, dev, model  # noqa: F401
from test_band_compressor_cpu import EDGES, set_profile, speech
from test_band_compressor_lr_cpu import DELAY_AT, bank_resp, group_delay_ms, model_hop, model_state

pytestmark = pytest.mark.gpu

C = 2
BANDS = {1: (), 2: (1000.0,), 5: EDGES, 16: tuple(450.0 * (k + 1) for k in range(15))}
CASES = [(f"lr{N}", K) for N in (4, 8) for K in (1, 2, 5, 16)]


def profile(g, n, K):
    """n seeded per-ear profiles: gains [n, C, K] in [-10, 20] dB, knees [n, K] in [-60, -30] dBFS, ratios [n, K] in
    [1, 4]"""
    return g.uniform(-10, 12, (n, 1, K)) + g.uniform(0, 8, (n, C, K)), g.uniform(-60, -30, (n, K)), g.uniform(1, 4, (n, K))


def roundoff(bank, x):
    """the largest deviation of any band's cascade run in float32 from the same cascade in float64, over the channels of
    x [C, N]: the scale of the fp32 filter's error"""
    if bank.shape[1] == 0:
        return 0.0
    worst = 0.0
    for b in range(bank.shape[0]):
        sos = np.concatenate([bank[b][:, :3], np.ones((bank.shape[1], 1)), bank[b][:, 3:]], 1)
        for c in range(x.shape[0]):
            lo = sosfilt(sos.astype(np.float32), x[c].astype(np.float32)).astype(np.float64)
            worst = max(worst, float(np.abs(lo - sosfilt(sos, x[c])).max()))
    return worst


# ---- 1. the model ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bank,K", CASES)
def test_random_profiles_agree_with_the_model(dev, bank, K):
    """slots scattered over the state, ragged hops (0 included), voices from -30 to 0 dB, per-ear profiles that compress,
    set at the start and again between ticks"""
    S, n, T, ticks = 7, 3, 3, 14
    g = np.random.default_rng(31 + K)
    slots = [5, 0, 3]
    sched = [su.hop_mix(n, T, 3100 + t) for t in range(ticks)]
    total = [sum(s[i] for s in sched) for i in range(n)]
    xs = [speech(C, total[i], 3200 + i, db=[-30.0, -6.0, 0.0][i]) for i in range(n)]
    cmp = BandCompressor(S, C, edges=BANDS[K], bank=bank, device=dev)
    table = cmp.taps.double().cpu().numpy()
    mst = [model_state(C, K, table.shape[1]) for _ in range(n)]
    pos, want, got = [0] * n, [[] for _ in range(n)], [[] for _ in range(n)]
    for t in range(ticks):
        if t in (0, 6):
            gains, knees, ratios = profile(g, n, K)
            cmp.set_profile(slots, torch.from_numpy(gains), torch.from_numpy(knees), torch.from_numpy(ratios))
            for i in range(n):
                set_profile(mst[i], gains[i], knees[i], ratios[i])
        y = torch.full((n, C, HOP * T), SENTINEL)
        for i in range(n):
            h = sched[t][i]
            seg = xs[i][:, HOP * pos[i]:HOP * (pos[i] + h)]
            y[i, :, :HOP * h] = torch.from_numpy(seg).float()
            for k in range(h):
                want[i].append(model_hop(mst[i], seg[:, HOP * k:HOP * (k + 1)], table))
            pos[i] += h
        out = cmp(y.to(dev), su.i32(slots, dev), hops=su.i32(sched[t], dev))
        for i in range(n):
            got[i].append(out[i, :, :HOP * sched[t][i]].cpu())
    torch.cuda.synchronize()
    for i in range(n):
        a, b = torch.cat(got[i], -1).double().numpy(), np.concatenate(want[i], 1)
        peak = np.abs(b).max()
        lin = 10 ** (np.abs(mst[i]["prof"]).max() / 20)                  # the largest band gain reached
        bound = min(1e-3 * peak, 16 * K * lin * roundoff(table, xs[i]) + 1e-5 * peak)
        assert np.abs(a - b).max() <= bound, (i, np.abs(a - b).max(), bound, peak)
        with np.errstate(divide="ignore"):
            lvl = 10 * np.log10(mst[i]["S"])
        assert np.abs(cmp.level[slots[i]].double().cpu().numpy() - lvl).max() <= 0.01, i
        assert np.abs(cmp.gain[slots[i]].double().cpu().numpy() - mst[i]["g"]).max() <= 0.01, i
    assert max(np.abs(m["g"] - m["prof"]).max() for m in mst) > 1            # the compression did act


# ---- 2. bits ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bank", ["lr4", "lr8"])
def test_one_band_at_zero_db_is_the_input(dev, bank):
    x = su.signals(3, C, HOP * 6, 41, dev) * 4
    x[0, 0, 10:20] = -0.0
    x[1, 1, 300:340] = 1e-40
    cmp = BandCompressor(4, C, edges=(), bank=bank, device=dev)
    y = torch.cat([cmp(x[:, :, HOP * t:HOP * (t + 2)], [3, 0, 2]) for t in range(0, 6, 2)], -1)
    torch.cuda.synchronize()
    assert torch.equal(su.bits(y), su.bits(x)) and bool((cmp.level[[3, 0, 2]] > -80).all())


@pytest.mark.parametrize("bank,K", CASES)
def test_cuts_and_in_place_do_not_change_a_bit(dev, bank, K):
    """the same hops of every slot through ticks of 1 hop and ragged ticks of 1-3 hops, out of place and in place"""
    S, n, hops = 5, 3, 12
    slots = [4, 0, 2]
    xs = torch.from_numpy(np.stack([speech(C, hops, 4100 + i, db=-8.0 * i) for i in range(n)])).float().to(dev)
    gains, knees, ratios = profile(np.random.default_rng(42), n, K)
    res = []
    for T, in_place in ((1, False), (3, False), (3, True)):
        cmp = BandCompressor(S, C, edges=BANDS[K], bank=bank, device=dev)
        cmp.set_profile(slots, torch.from_numpy(gains), torch.from_numpy(knees), torch.from_numpy(ratios))
        rng = np.random.default_rng(4200 + T)
        pos, got = [0] * n, [[] for _ in range(n)]
        while min(pos) < hops:
            h = [int(min(rng.integers(0, T + 1), hops - p)) for p in pos] if T > 1 else [int(p < hops) for p in pos]
            y = torch.full((n, C, HOP * T), SENTINEL, device=dev)
            for i in range(n):
                y[i, :, :HOP * h[i]] = xs[i, :, HOP * pos[i]:HOP * (pos[i] + h[i])]
            out = cmp(y, su.i32(slots, dev), hops=su.i32(h, dev), out=y if in_place else None)
            for i in range(n):
                got[i].append(out[i, :, :HOP * h[i]])
            pos = [p + k for p, k in zip(pos, h)]
        torch.cuda.synchronize()
        res.append((torch.stack([torch.cat(v, -1) for v in got]), cmp.state.clone()))
    for r in res[1:]:
        assert torch.equal(su.bits(r[0]), su.bits(res[0][0])) and torch.equal(su.bits(r[1]), su.bits(res[0][1]))
    assert bool(res[0][1][slots].any()) and not res[0][1][[1, 3]].any()


@pytest.mark.parametrize("bank", ["lr4", "lr8"])
def test_store_rules_with_guards(dev, bank):
    """rows whose slot lies outside the state, or whose hop count lies outside [1, T], store nothing: their out rows, out
    samples past 128 h and guard regions around y and out keep their values, and unlisted slots' rows keep theirs"""
    S, n, T, G = 6, 6, 2, 1000
    slots, hops = [4, -1, 2, 3, 0, 7], [2, 2, 0, 1, 3, 1]
    flat_y = torch.full((G + n * C * HOP * T + G,), 9.0, device=dev)
    flat_o = torch.full((G + n * C * HOP * T + G,), 5.0, device=dev)
    y = flat_y[G:G + n * C * HOP * T].view(n, C, HOP * T)
    y.copy_(su.signals(n, C, HOP * T, 43, dev))
    keep = y.clone()
    out = flat_o[G:G + n * C * HOP * T].view(n, C, HOP * T)
    cmp = BandCompressor(S, C, bank=bank, device=dev)
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
    assert torch.equal(su.bits(cmp.state[[0, 1, 2, 5]]), su.bits(before[[0, 1, 2, 5]]))
    assert not torch.equal(cmp.state[4], before[4]) and not torch.equal(cmp.state[3], before[3])


@pytest.mark.parametrize("bank", ["lr4", "lr8"])
def test_non_finite_input_is_not_measured(dev, bank):
    cmp = BandCompressor(3, C, bank=bank, device=dev)
    cmp.set_profile([2], [6.0, 9.0, 12.0, 15.0, 9.0], knees=-50.0, ratios=3.0)
    x = torch.from_numpy(speech(C, 40, 4400, db=-2.0)).float().to(dev)
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


@pytest.mark.parametrize("bank", ["lr4", "lr8"])
def test_graph_replay_is_the_eager_call(dev, bank):
    """one call captured with its slot and hop lists, replayed with them rewritten in place: eager calls bit for bit"""
    S, n, T = 6, 3, 3
    live, twin = (BandCompressor(S, C, bank=bank, device=dev) for _ in range(2))
    for c in (live, twin):
        c.set_profile([0, 1, 2, 3, 4, 5], [2.0, 6.0, 10.0, 14.0, 8.0], knees=-50.0, ratios=2.5)
    y = torch.zeros(n, C, HOP * T, device=dev)
    out = torch.zeros_like(y)
    slots, hops = su.i32([0, 1, 2], dev), su.i32([1, 1, 1], dev)
    graph = su.captured(lambda: live(y, slots, hops=hops, out=out), warm=lambda: live(y, su.i32([-1] * n, dev), out=out))
    g = np.random.default_rng(45)
    for t in range(8):
        sl, hp = [int(v) for v in g.permutation(S)[:n]], [int(v) for v in g.integers(0, T + 1, n)]
        y.copy_(su.signals(n, C, HOP * T, 4500 + t, dev))
        slots.copy_(su.i32(sl, dev))
        hops.copy_(su.i32(hp, dev))
        out.fill_(SENTINEL)
        graph.replay()
        want = torch.full_like(out, SENTINEL)
        twin(y, sl, hops=hp, out=want)
        torch.cuda.synchronize()
        assert torch.equal(su.bits(out), su.bits(want)) and torch.equal(su.bits(live.state), su.bits(twin.state)), t


def test_impulse_peaks_within_the_group_delay(dev):
    """an impulse through a flat LR4 slot: the output peaks within the documented delay of the lowest band (1.83 ms at
    250 Hz, 29 samples), far before the FIR bank's 64 samples, and sums to the allpass cascade's impulse response"""
    cmp = BandCompressor(2, 1, bank="lr4", device=dev)
    x = torch.zeros(1, 1, HOP * 4, device=dev)
    x[0, 0, 0] = 1.0
    y = cmp(x, [1])[0, 0].double().cpu().numpy()
    table = cmp.taps.double().cpu().numpy()
    gd = group_delay_ms(lambda f: bank_resp(table, f).sum(0), DELAY_AT)
    assert int(np.argmax(np.abs(y))) <= gd[0] * 16 and int(np.argmax(np.abs(y))) < 32
    st = model_state(1, 5, table.shape[1])
    want = np.concatenate([model_hop(st, x[0, :, HOP * k:HOP * (k + 1)].double().cpu().numpy(), table) for k in range(4)], 1)
    assert np.abs(y - want[0]).max() <= 1e-5


# ---- 3. the full tick, one CUDA graph ---------------------------------------------------------------------------------
def test_full_tick_on_the_separator(model, dev):
    """the LR4 compressor in place on the mixer's sum of the seeded separator's 44.1 kHz tick, in the captured graph:
    bit for bit the eager chain, and every tick's compressed sum the model's from the sum before it"""
    T = su.TICK_T
    gains = [0.0, 4.0, 10.0, 15.0, 8.0]
    ratios = [1.5, 2, 2, 2.5, 2]
    mst = []

    def build(o):
        o["cmp"] = BandCompressor(su.TICK_S, C, bank="lr4", device=dev)
        o["cmp"].set_profile([0, 1, 2], [gains] * 3, knees=-40.0, ratios=ratios)
        if not mst:
            table = o["cmp"].taps.double().cpu().numpy()
            for _ in range(su.TICK_N):
                st = model_state(C, 5, table.shape[1])
                set_profile(st, gains, -40.0, ratios)
                mst.append((st, table))

    def mixed(o, b, y, slots, rec, off):
        b["pre"].copy_(b["mix"])
        o["cmp"](b["mix"], slots, hops=b["hops"], out=b["mix"])

    worst = [0.0]

    def each(b, t):
        hops = b["hops"].tolist()
        pre, post = b["pre"].double().cpu().numpy(), b["mix"].double().cpu().numpy()
        for i, h in enumerate(hops):
            if not 1 <= h <= T:
                continue
            st, table = mst[i]
            want = np.concatenate([model_hop(st, pre[i, :, HOP * k:HOP * (k + 1)], table) for k in range(h)], 1)
            peak = max(np.abs(want).max(), 1e-30)
            worst[0] = max(worst[0], np.abs(post[i, :, :HOP * h] - want).max() / peak)

    live = su.separator_tick(model[0], dev, build, mixed=mixed, bufs={"pre": HOP * T}, each=each)
    assert worst[0] <= 1e-4, worst[0]
    assert bool(torch.isfinite(live["cmp"].level[:3]).all()) and float(live["cmp"].gain[:3].abs().max()) > 1
