"""The per-slot gain stages of csrc/resample.cu called through the C ABI: band_compressor_kernel (l2h_band_compressor),
leveler_kernel (l2h_leveler) and limiter_kernel (l2h_limiter), every hop against the float64 models of
test_band_compressor_cpu.py, test_leveler_cpu.py and test_limiter_cpu.py, within the bounds derived there.

Each case runs one hop per call (one push for the limiter), reads the state back, and compares that hop's output and new
state with the model started from the kernel's own state at the hop's start, so errors cannot compound across hops.
The same hops sent again as ragged multi-hop calls (hop counts 0 to T, and counts outside [1, T] that store nothing)
must give the one-hop outputs and states bit for bit.  States are also written by hand before a hop: counters at and
near INT32_MAX or negative, the hop that reaches `settle`, a failing relative gate, gains at their clamps, detectors at
0, slopes of 0 and 0.999, r and history words past LM_MUTE or negative, slot ceilings that are not positive normal
floats, and reductions that mute.  Each mutant of the models (their MUTANTS) must miss its bound by SENSITIVITY in every
case that exercises it.

Compressor (K, L, C): all four band_compressor_kernel<KP> instantiations, histories H = L - 1 below, at and above one
thread's 128 samples, C up to 12 and the staging closest to shared memory, each with the designed bank and a seeded
asymmetric one (only an asymmetric bank shows the order of the taps).  Leveler: C = 1, 2, 3, 8, 128, 129 and 257, with
and without offsets, non-monotonic and out-of-range offsets, records outside the state, strided rows in and out of
place.  Limiter: C = 1, 2, 3 and 8 with La = 0, 16 and 48; pushes of 1, under 256, over 256 and at the staging limit of
(C + 2)(La + max_in) floats, unit 1 and 3, counts outside [0, max_in].

Every input, output, list and state buffer is a Guarded one: the guards and every state row no call lists must keep the
sentinel bit for bit, as must the output rows of calls that store nothing.
Measured on one NVIDIA H100 80GB HBM3 (700 W power limit): worst error / bound 0.673 (compressor), 0.534 (leveler),
0.890 (limiter); smallest mutant margin 145 (compressor), 294 (leveler), and every limiter mutant changes an exact word
(margin inf).  The file runs in about 140 s, most of it in the float64 models.
"""
import math

import numpy as np
import pytest
import torch

import test_band_compressor_cpu as bc
import test_leveler_cpu as lv
import test_limiter_cpu as lm
from kernels.scaffold import Guarded, Ledger, bits, dev, is_sentinel  # noqa: F401
from lookoncetohear_b200 import BandCompressor, _cabi

pytestmark = pytest.mark.gpu
HOP = 128
LEDGER = Ledger()
F32 = lambda v: float(np.float32(v))   # noqa: E731


def lib():
    return _cabi.lib()


def ints(values, dev):
    """a Guarded int32 list"""
    g = Guarded((len(values),), dev)
    g.t.view(torch.int32).copy_(torch.tensor(values, dtype=torch.int32))
    return g


def ptr(g):
    return None if g is None else g.t.data_ptr()


def f32(a):
    return np.asarray(a, np.float32)


def fold(errs, into):
    for k, v in errs.items():
        into[k] = max(into.get(k, 0.0), v)


def check(key, errs, mutants, bufs):
    for g in bufs:
        assert g is None or g.ok(), "a guard lost its sentinel"
    LEDGER.check(key, errs, mutants)


# ---- band compressor -------------------------------------------------------------------------------------------------
BC_CONFIGS = [(1, 33, 1), (4, 127, 2), (5, 129, 1), (5, 129, 2), (5, 129, 12), (8, 131, 4), (9, 255, 2), (12, 201, 3),
              (13, 255, 3), (16, 255, 3)]
BC_ATTACK, BC_RELEASE = F32(bc.ATTACK), F32(bc.RELEASE)


def bc_bank(K, L, kind):
    if kind == "random":
        return bc.random_bank(K, L, K * 1000 + L)
    edges = tuple(float(e) for e in np.geomspace(150.0, 7000.0, K - 1)) if K > 1 else ()
    return BandCompressor.design(edges, L).double().numpy()


def bc_presets(K, C, g):
    """name -> a function(st) that writes a hand-set state over the kernel's own (keeping its history)"""
    def prof(st):
        bc.set_profile(st, g.uniform(-10, 12, (C, K)), knees=g.uniform(-50, -30, K), ratios=g.uniform(1, 4, K))

    def zero_detectors(st):
        prof(st)
        st["S"][:] = 0

    def slopes(st):
        prof(st)
        st["slope"] = np.where(np.arange(K) % 2, 0.0, F32(0.999))
        st["knee"][:] = -60

    def clamp(st):
        st["g"] = np.where(np.arange(K) % 2, 40.0, -40.0)[None].repeat(C, 0)
        st["prof"] = np.where(np.arange(K) % 2, 40.0, -40.0)[None].repeat(C, 0)
        st["slope"][:] = 0

    def unprofiled(st):
        st["prof"][:], st["slope"][:] = 0, 0
        st["g"] = g.uniform(-6, 6, (C, K))

    def flat(st):
        for k in ("prof", "g", "slope"):
            st[k][:] = 0
    return {"flat": flat, "profile": prof, "zero_detectors": zero_detectors, "slopes": slopes, "clamp": clamp,
            "unprofiled": unprofiled, "back_to_flat": flat}


def bc_call(y, out, y_strides, o_strides, slots, hops, taps, K, L, state, C, T, n_slots=3):
    return lib().l2h_band_compressor(ptr(y), *y_strides, ptr(out), *o_strides, 2, C, T, ptr(slots), ptr(hops), ptr(taps),
                                     K, L, ptr(state), n_slots, BC_ATTACK, BC_RELEASE, None)


@pytest.mark.parametrize("kind", ["designed", "random"])
@pytest.mark.parametrize("K,L,C", BC_CONFIGS, ids=lambda v: str(v))
def test_band_compressor(K, L, C, kind, dev):
    bank = bc_bank(K, L, kind)
    taps = Guarded(bank.shape, dev, torch.from_numpy(f32(bank)))
    rf = 5 * K + L - 1
    state = Guarded((3, C, rf), dev)
    slots = ints([2, 0], dev)
    listed = (2, 0)
    for s in listed:
        state.t[s] = 0
    g = np.random.default_rng(K * 100 + L + C)
    presets = bc_presets(K, C, g)
    errs = {}
    live = [m for m in bc.MUTANTS if not ((m in ("unlinked", "undivided") and C == 1) or (m == "reversed" and kind != "random")
                                          or (m == "history" and L - 1 <= HOP))]
    shown = {m: 0.0 for m in live}
    for seg, (name, preset) in enumerate(presets.items()):
        for s in listed:                                  # the hand-set state, over the kernel's own
            st = bc.from_row(state.t[s].cpu().numpy(), K)
            preset(st)
            state.t[s] = torch.from_numpy(bc.to_row(st))
        start = state.t.clone()
        x = {s: bc.speech(C, 3, 100 * seg + s + K, db=float(g.uniform(-30, 0))) for s in listed}
        if name == "profile":                             # not measured, staged as 0
            x[2][0, 5] = np.nan
            x[0][C - 1, HOP + 9] = -np.inf
            x[2][C - 1, 2 * HOP + 3] = 2.0 ** 32
        ys = {s: [] for s in listed}
        for h in range(3):
            y = Guarded((2, C, HOP), dev, torch.from_numpy(f32(np.stack([x[s][:, h * HOP:(h + 1) * HOP] for s in listed]))))
            out = Guarded((2, C, HOP), dev)
            before = {s: bc.from_row(state.t[s].cpu().numpy(), K) for s in listed}
            rc = bc_call(y, out, (C * HOP, HOP), (C * HOP, HOP), slots, None, taps, K, L, state, C, 1)
            assert rc == 0, lib().l2h_last_error().decode()
            torch.cuda.synchronize(dev)
            for i, s in enumerate(listed):
                after = bc.from_row(state.t[s].cpu().numpy(), K)
                got = {"y": out.t[i].cpu().numpy(), "S": after["S"], "g": after["g"], "hist": after["hist"]}
                xh = x[s][:, h * HOP:(h + 1) * HOP]
                fold(bc.hop_errors(before[s], xh, bank, got, None, BC_ATTACK, BC_RELEASE), errs)
                for m in live:
                    shown[m] = max(shown[m], max(bc.hop_errors(before[s], xh, bank, got, m, BC_ATTACK, BC_RELEASE).values()))
                ys[s].append(got["y"])
                if name in ("flat", "back_to_flat") and h > 0:
                    delayed = np.concatenate([before[s]["hist"], np.where(np.abs(xh) < 2.0 ** 32, xh, 0)], 1)
                    assert np.array_equal(got["y"], f32(delayed[:, (L - 1) - (L - 1) // 2:][:, :HOP])), "0 dB: the delayed input"
            assert out.ok() and y.ok()
        end = state.t.clone()
        # the same hops, ragged, in place: row 0 takes 2, none (-1), 1; row 1 none, 3 (T = 3), none (4 > T)
        state.t.copy_(start)
        pos = {s: 0 for s in listed}
        got_y = {s: [] for s in listed}
        for counts in ([2, 0], [-1, 3], [1, 4]):
            buf = np.zeros((2, C, 3 * HOP), np.float32)
            for i, s in enumerate(listed):
                if 1 <= counts[i] <= 3:
                    buf[i, :, :counts[i] * HOP] = x[s][:, pos[s] * HOP:(pos[s] + counts[i]) * HOP]
            y = Guarded((2, C, 3 * HOP), dev, torch.from_numpy(buf))
            hops = ints(counts, dev)
            rc = bc_call(y, y, (C * 3 * HOP, 3 * HOP), (C * 3 * HOP, 3 * HOP), slots, hops, taps, K, L, state, C, 3)
            assert rc == 0, lib().l2h_last_error().decode()
            torch.cuda.synchronize(dev)
            res = y.t.cpu().numpy()
            for i, s in enumerate(listed):
                if 1 <= counts[i] <= 3:
                    got_y[s].append(res[i, :, :counts[i] * HOP])
                    pos[s] += counts[i]
                else:
                    assert np.array_equal(res[i].view(np.int32), buf[i].view(np.int32)), "a row that stores nothing"
            assert y.ok()
        for s in listed:
            assert np.array_equal(np.concatenate(got_y[s], 1).view(np.int32), f32(np.concatenate(ys[s], 1)).view(np.int32))
        assert torch.equal(bits(state.t), bits(end)), "ragged calls: the same state bit for bit"
    assert is_sentinel(state.t[1]), "an unlisted slot"
    check("compressor", errs, shown, [taps, state, slots])


@pytest.mark.parametrize("K,C", [(16, 4), (5, 13)])
def test_band_compressor_refuses_staging_past_shared_memory(K, C, dev):
    L = 255 if K == 16 else 129
    state = Guarded((3, C, 5 * K + L - 1), dev)
    y, out = Guarded((2, C, HOP), dev), Guarded((2, C, HOP), dev)
    taps, slots = Guarded((K, L), dev, torch.zeros(K, L)), ints([2, 0], dev)
    assert bc_call(y, out, (C * HOP, HOP), (C * HOP, HOP), slots, None, taps, K, L, state, C, 1) == 2
    assert b"shared memory" in lib().l2h_last_error()
    torch.cuda.synchronize(dev)
    assert is_sentinel(state.t) and is_sentinel(out.t) and state.ok() and out.ok()


# ---- leveler ---------------------------------------------------------------------------------------------------------
LV_P = dict(target=-20.0, gate=-50.0, relative=-20.0, alpha=F32(0.05), settle=4, min_gain=-12.0, max_gain=12.0, rise=0.5,
            fall=1.0)
# (offsets or None, the listener of rows 0, 1, 2 under it): rows 0 .. 2 map to state rows 3, 0 and 5 (outside the state)
LV_OFFSETS = [(None, [0, 1, None]), ([0, 1, 3], [0, 1, 1]), ([0, 2, 1], [0, 0, None]), ([1, 1, 3], [None, 1, 1])]
LV_RECORDS = [3, 0, 5]


def lv_call(y, ys, out, os_, offsets, hops, state, C, T, p):
    return lib().l2h_leveler(ptr(y), *ys, ptr(out), *os_, 2, 3, C, T, ptr(ints(LV_RECORDS, y.t.device)),
                             ptr(offsets), ptr(hops), ptr(state), 4, p["target"], p["gate"], p["relative"], p["alpha"],
                             p["settle"], p["min_gain"], p["max_gain"], p["rise"], p["fall"], None)


def lv_presets(g):
    M = lv.INT32_MAX
    return [("fresh", {}), ("near_max", {"n": M - 1}), ("max", {"n": M}), ("negative", {"n": -5}),
            ("settle", {"n": LV_P["settle"] - 1}), ("relative", {"n": 9, "E": 1e3}), ("min_gain", {"n": 9, "g": -12.0}),
            ("max_gain", {"n": 9, "g": 12.0}), ("quiet", {"n": 9}), ("no_steps", {"n": 9, "g": 3.0})]


def strided(dev, C, T, pad_row, pad_ch, values=None):
    """a Guarded [3][C][128 T] tensor with pad_ch floats between channels and pad_row between rows: (buffer, view,
    strides)"""
    ch = HOP * T + pad_ch
    row = C * ch + pad_row
    buf = Guarded((3 * row,), dev)
    v = buf.t.as_strided((3, C, HOP * T), (row, ch, 1))
    if values is not None:
        v.copy_(torch.from_numpy(f32(values)))
    return buf, v, (row, ch)


@pytest.mark.parametrize("C", [1, 2, 3, 8, 128, 129, 257])
def test_leveler(C, dev):
    g = np.random.default_rng(C)
    state = Guarded((4, C, lv.FLOATS), dev)
    state.t[3], state.t[0] = 0, 0
    errs, shown = {}, {m: -math.inf for m in lv.MUTANTS}
    for seg, (name, kw) in enumerate(lv_presets(g)):
        offsets, owner = LV_OFFSETS[seg % len(LV_OFFSETS)]
        p = dict(LV_P, rise=0.0, fall=0.0) if name == "no_steps" else LV_P
        for r in (3, 0):
            st = lv.from_row(state.t[r].cpu().numpy())
            st.update(kw)
            state.t[r] = torch.from_numpy(lv.to_row(st))
        start = state.t.clone()
        db = -75.0 if name == "quiet" else float(g.uniform(-30, 0))
        x = np.stack([lv.voice(C, 3, 50 * seg + r + C, db=db) for r in range(3)])
        if name == "negative":
            x[1, C - 1, HOP + 7] = np.nan                     # hop 1 of row 1 is not measured
        outs = []
        for h in range(3):
            hop = x[:, :, h * HOP:(h + 1) * HOP]
            gy, vy, ys = strided(dev, C, 1, 3, 5, hop)
            in_place = h == 1
            go, vo, os_ = (gy, vy, ys) if in_place else strided(dev, C, 1, 7, 2)
            before = {r: lv.from_row(state.t[r].cpu().numpy()) for r in (3, 0)}
            hops = ints([1, 1], dev)
            offs = None if offsets is None else ints(offsets, dev)
            assert lv_call(gy, ys, go, os_, offs, hops, state, C, 1, p) == 0, lib().l2h_last_error().decode()
            torch.cuda.synchronize(dev)
            res = vo.cpu().numpy()
            outs.append(res)
            for row in range(3):
                rec = LV_RECORDS[row]
                if owner[row] is None or rec >= 4:
                    want = hop[row] if in_place else None
                    assert (is_sentinel(vo[row]) if want is None else np.array_equal(res[row], f32(want))), "stores nothing"
                    continue
                after = lv.from_row(state.t[rec].cpu().numpy())
                got = dict(after, y=res[row])
                fold(lv.hop_errors(before[rec], hop[row], p, got), errs)
                model = lv.kernel_like(before[rec], hop[row], p)
                for m in shown:
                    if max(lv.hop_errors(before[rec], hop[row], p, model, m).values()) > 1e-6:    # the hop exercises m
                        shown[m] = max(shown[m], max(lv.hop_errors(before[rec], hop[row], p, got, m).values()))
            assert gy.ok() and go.ok()
        end = state.t.clone()
        # ragged: rows take 2 hops then 1 (listener 0) or none then 3 (listener 1), in place
        state.t.copy_(start)
        pos = [0, 0]
        ragged = [[] for _ in range(3)]
        for counts in ([2, 0], [1, 3]):
            buf = np.zeros((3, C, 3 * HOP))
            for row in range(3):
                i = owner[row]
                if i is not None and counts[i]:
                    buf[row, :, :counts[i] * HOP] = x[row, :, pos[i] * HOP:(pos[i] + counts[i]) * HOP]
            gy, vy, ys = strided(dev, C, 3, 1, 4, buf)
            offs = None if offsets is None else ints(offsets, dev)
            assert lv_call(gy, ys, gy, ys, offs, ints(counts, dev), state, C, 3, p) == 0
            torch.cuda.synchronize(dev)
            res = vy.cpu().numpy()
            for row in range(3):
                i = owner[row]
                if i is not None and counts[i] and LV_RECORDS[row] < 4:
                    ragged[row].append(res[row, :, :counts[i] * HOP])
            for i in range(2):
                pos[i] += counts[i]
        for row in range(3):
            if ragged[row]:
                one = np.concatenate([o[row] for o in outs], 1)
                assert np.array_equal(np.concatenate(ragged[row], 1).view(np.int32), one.view(np.int32)), row
        assert torch.equal(bits(state.t), bits(end)), "ragged calls: the same state bit for bit"
    assert is_sentinel(state.t[1]) and is_sentinel(state.t[2]), "unlisted rows"
    check("leveler", errs, {m: v for m, v in shown.items() if v > -math.inf}, [state])


# ---- limiter ---------------------------------------------------------------------------------------------------------
LM_STEP = 20


def lm_presets(C):
    M, Q = lm.MUTE, lm.Q
    return [("fresh", {}, LM_STEP), ("r_mute", {"r": M}, 4000), ("r_negative", {"r": -9}, LM_STEP),
            ("history_words", {"qh": [M + 5, -3], "rh": [M + 7, -1]}, 5000),
            ("subnormal_ceiling", {"ceil": 1e-40, "r": 2 * Q}, 600), ("inf_ceiling", {"ceil": math.inf}, LM_STEP),
            ("nan_ceiling", {"ceil": math.nan}, LM_STEP), ("negative_ceiling", {"ceil": -0.5}, LM_STEP),
            ("own_ceiling", {"ceil": 0.3}, LM_STEP), ("limited_near_max", {"limited": lm.INT32_MAX - 3}, LM_STEP),
            ("mutes", {"r": M - 1, "rh": [M - 1]}, 1)]


def lm_call(x, max_in, counts, unit, y, slots, state, C, La, step):
    return lib().l2h_limiter(ptr(x), C * max_in, max_in, max_in, ptr(counts), unit, ptr(y), C * max_in, max_in, 2, C,
                             ptr(slots), ptr(state), 3, lm.CEILING, La, step, None)


@pytest.mark.parametrize("La", [0, 16, 48])
@pytest.mark.parametrize("C", [1, 2, 3, 8])
def test_limiter(C, La, dev):
    max_in = 12288 // (C + 2) - La                       # the staging at its limit
    rf = lm.HEAD + 3 * La
    state = Guarded((3, C, rf), dev)
    slots, listed = ints([2, 0], dev), (2, 0)
    for s in listed:
        state.t[s] = 0
    g = np.random.default_rng(C * 100 + La)
    errs = {}
    shown = {m: -math.inf for m in lm.MUTANTS}
    lengths = [1, 100, 700, max_in, 37]
    for seg, (name, kw, step) in enumerate(lm_presets(C)):
        for s in listed:
            st = lm.from_row(state.t[s].cpu().numpy(), La)
            for k, v in kw.items():
                st[k] = np.resize(np.asarray(v, np.int64), La) if k in ("qh", "rh") else v
            state.t[s] = torch.from_numpy(lm.to_row(st, C))
        start = state.t.clone()
        n = [lengths[(seg + i) % len(lengths)] for i in range(2)]
        unit = 3 if seg % 3 == 1 else 1
        n = [max(unit, v // unit * unit) for v in n]
        x = {s: lm.loud(C, 2 * n[i], 30 * seg + s, peak=float(g.uniform(0.5, 12))) for i, s in enumerate(listed)}
        if name == "r_negative":
            x[0][C - 1, 0] = np.nan
        ys = {s: [] for s in listed}
        for push in range(2):
            buf = np.zeros((2, C, max_in), np.float32)
            for i, s in enumerate(listed):
                buf[i, :, :n[i]] = x[s][:, push * n[i]:(push + 1) * n[i]]
            gx = Guarded((2, C, max_in), dev, torch.from_numpy(buf))
            gy = Guarded((2, C, max_in), dev)
            counts = [n[0] // unit, n[1] // unit]
            if push == 1 and seg % 4 == 3:
                counts[1] = -1                            # stores nothing
            before = {s: lm.from_row(state.t[s].cpu().numpy(), La) for s in listed}
            snap = state.t.clone()
            assert lm_call(gx, max_in, ints(counts, dev), unit, gy, slots, state, C, La, step) == 0, \
                lib().l2h_last_error().decode()
            torch.cuda.synchronize(dev)
            res = gy.t.cpu().numpy()
            for i, s in enumerate(listed):
                if counts[i] < 0:
                    assert is_sentinel(gy.t[i]) and torch.equal(bits(state.t[s]), bits(snap[s])), "stores nothing"
                    continue
                m = n[i]
                after = lm.from_row(state.t[s].cpu().numpy(), La)
                got = dict(after, y=res[i, :, :m])
                xp = x[s][:, push * m:(push + 1) * m]
                fold(lm.push_errors(before[s], xp, lm.CEILING, La, step, got), errs)
                model = lm.kernel_like(before[s], xp, La, step)
                for mu in shown:
                    if max(lm.push_errors(before[s], xp, lm.CEILING, La, step, model, mu).values()) > 0:   # exercised
                        shown[mu] = max(shown[mu], max(lm.push_errors(before[s], xp, lm.CEILING, La, step, got, mu).values()))
                ys[s].append(res[i, :, :m])
                assert is_sentinel(gy.t[i, :, m:]), "past the push"
            assert gx.ok() and gy.ok()
        end = state.t.clone()
        # the same samples cut differently: row 0 in one push where it fits, row 1 split unevenly (unit 1)
        state.t.copy_(start)
        total = [sum(a.shape[1] for a in ys[s]) for s in listed]
        cuts = [[total[0]] if total[0] <= max_in else [total[0] - max_in, max_in],
                [1, total[1] - 1] if 1 < total[1] <= max_in else ([total[1] - max_in, max_in] if total[1] > 1 else [1])]
        got = {s: [] for s in listed}
        done = [0, 0]
        for j in range(2):
            buf = np.zeros((2, C, max_in), np.float32)
            counts = []
            for i, s in enumerate(listed):
                c = cuts[i][j] if j < len(cuts[i]) else 0
                buf[i, :, :c] = x[s][:, done[i]:done[i] + c]
                counts.append(c)
            gx, gy = Guarded((2, C, max_in), dev, torch.from_numpy(buf)), Guarded((2, C, max_in), dev)
            assert lm_call(gx, max_in, ints(counts, dev), 1, gy, slots, state, C, La, step) == 0
            torch.cuda.synchronize(dev)
            for i, s in enumerate(listed):
                got[s].append(gy.t[i, :, :counts[i]].cpu().numpy())
                done[i] += counts[i]
        for s in listed:
            assert np.array_equal(np.concatenate(got[s], 1).view(np.int32), np.concatenate(ys[s], 1).view(np.int32)), s
        assert torch.equal(bits(state.t), bits(end)), "recut pushes: the same state bit for bit"
    assert is_sentinel(state.t[1]), "an unlisted slot"
    check("limiter", errs, {m: v for m, v in shown.items() if v > -math.inf}, [state, slots])


def test_summary():
    LEDGER.summary()
