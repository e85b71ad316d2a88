"""The resamplers, the hop FIFO, the enrollment capture and the target mixer of csrc/resample.cu called through the C ABI:
resample_kernel (l2h_resample), resample_stream_kernel (l2h_resample_stream) and resample_packets_kernel
(l2h_resample_packets) against the float64 models of test_resample_cpu.py; hop_fifo_kernel (l2h_hop_fifo) and
enroll_capture_kernel (l2h_enroll_capture) against the exact host models of test_packet_stream_cpu.py; target_mix_kernel<1>,
<4> (l2h_target_mix) and target_mix_set_kernel (l2h_target_mix_set) against the float64 model of test_target_mix_cpu.py;
each within the bound derived there.

Each call is compared with the model started from the kernel's own state at the call's start, so errors cannot compound.
Resamplers: every serving rate to and from 16 kHz, 45:1 (and 46:1 refused), 231:200 (a tap at |u| = 6 exactly) and
16001 <-> 16000; lengths 0, 1, below, on and across the 256-output tiles, capacities under 32, launch splits at
RS_MAX_RATES, RS_MAX_RUNS and RS_MAX_ROWS.  The streamers push once per call: hop counts 0 .. T and outside [1, T], pushes
of 0, 1, o - 1, o, o + 1 and max_in and counts outside [0, max_in], unit 1 and 3, keep 0, below and above one push,
stagings at the 12288-float limit, count words 0, D - 1, D, above D, negative, NaN and 3e38 (the whole-period stream's
count word is also its first history word: outputs stay finite), phase words o - 1, past o, negative and fractional.
FIFO and capture: chunks, hop counts, every head word and every ring word written match bit for bit, and nothing else is
written.  Their head words are also written by hand: positions at and past the ring's end, held and captured counts at
and past the capacity, dropped counts at and near INT32_MAX and negative; pushes fill, overflow, drain and wrap the ring
inside one call, T caps the hops, capture hops outrun the capacity, and slots lie outside the state.  One FIFO of
capacity 2^30 + 64 (a 4.3 GB state) pushes where its ring indices pass INT32_MAX.

Mixer: every case runs in the float4 form and, with strides that are not a multiple of 4, the scalar form, which must give
the same bits.  Listeners of 1, 63, 64, 65, 128 and 129 live terms (across the TM_TERMS passes), a listener with no term
(every sample -0), muted terms whose rows hold the sentinel, a term whose gain reaches 0 with NaN at exactly those samples,
ramp words written by hand on live terms (F + 1 = 0 and < 0, p > F, p < 0, F + 1 = INT32_MAX), gain sets of fades 0,
INT32_MAX - 1 and INT32_MAX, rows outside the state and sets without starts, no chunk, offsets non-monotonic and out of
range, C up to 8.  A case exercises a mutant where the mutant's model misses the true model by 2 SENSITIVITY bounds; there
the kernel must miss the mutant by SENSITIVITY.

Every input, output, list and state buffer is a Guarded one: the guards, every state row no call lists and the outputs of
rows that store nothing must keep the sentinel bit for bit.
Measured on one NVIDIA H100 80GB HBM3 (700 W power limit): FIFO and capture exact; worst error / bound 0.449 (resample),
0.351 (stream), 0.377 (packets), 0.973 (mix: the per-fmaf rounding bound is nearly met by a sum just above a power of 2)
and 0.154 (set); smallest mutant margin 23.3 (resample, "taps"), 3.4e5 (stream, packets), 8.2e4 (mix) and 1.0e4 (set).
The file runs in about 50 s.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import test_packet_stream_cpu as ps
import test_resample_cpu as rs
import test_target_mix_cpu as tm
from kernels.scaffold import SENSITIVITY, SENTINEL, Guarded, Ledger, bits, dev, is_sentinel, ratio  # noqa: F401
from lookoncetohear_b200 import _cabi
from oracle import resample as ors

pytestmark = pytest.mark.gpu
HOP, CARRY = 128, 64
INT32_MAX = 2 ** 31 - 1
LEDGER = Ledger()


def lib():
    return _cabi.lib()


def ints(values, dev):
    """a Guarded int32 list"""
    g = Guarded((len(values),), dev)
    g.t.view(torch.int32).copy_(torch.tensor(values, dtype=torch.int32))
    return g


def ptr(g):
    return None if g is None else g.t.data_ptr()


def i32bits(a):
    return np.asarray(a, np.float32).view(np.int32)


def words(values):
    """int32 head words as the floats that hold their bits"""
    return np.asarray(values, np.int64).astype(np.int32).view(np.float32)


def check(key, errs, mutants, bufs):
    for g in bufs:
        assert g is None or g.ok(), "a guard lost its sentinel"
    LEDGER.check(key, errs, mutants)


# ---- the resamplers --------------------------------------------------------------------------------------------------
SERVING = (48000, 44100, 32000, 24000, 22050, 11025, 8000)
RS_PAIRS = ([(r, 16000) for r in SERVING] + [(16000, r) for r in SERVING]
            + [(720000, 16000), (46200, 40000), (16001, 16000), (16000, 16001)])


def rs_call(x, n_in, rates, new, y, cap, dev):
    arr = (ctypes.c_int32 * len(rates))(*rates)
    return lib().l2h_resample(ptr(x), max(n_in, 1), n_in, len(rates), arr, new, ptr(y), max(cap, 1), cap, None)


def exercise(shown, m, got, mutant, want, bound):
    """a case exercises a mutant where the models themselves differ by 2 SENSITIVITY bounds; there the kernel must miss
    the mutant by SENSITIVITY"""
    if ratio(mutant, want, bound) >= 2 * SENSITIVITY:
        shown[m] = max(shown.get(m, -math.inf), ratio(got, mutant, bound))


def rs_check(key, got, x, rates, new, cap, rows, errs, shown):
    """rows `rows` of a resample_kernel output against the model, and each mutant"""
    for i in rows:
        want, b = rs.whole(x[i], rates[i], new, cap)
        errs["y"] = max(errs.get("y", 0.0), ratio(got[i], want, b))
        if rates[i] == new:
            assert np.array_equal(i32bits(got[i]), i32bits(want)), "equal rates: a copy"
            continue
        for m in rs.RS_MUTANTS:
            ym, _ = rs.whole(x[i], rates[i], new, cap, m)
            exercise(shown, m, got[i], ym, want, b)


@pytest.mark.parametrize("orig,new", RS_PAIRS)
def test_resample(orig, new, dev):
    o, q, w, base = rs.rs_filter(orig, new)
    g = np.random.default_rng(orig + new)
    errs, shown = {}, {}
    n_for = lambda k: -(-k * o // q)                    # noqa: E731  the fewest inputs that give k outputs
    lengths = [0, 1, 37, n_for(255), n_for(256), n_for(257), n_for(600)]
    for n_in in lengths:
        n_out = ors.output_length(n_in, orig, new)
        for cap in sorted({n_out, n_out + 3, max(n_out, 20)}):
            rates = [orig, orig, new, orig]             # a row of equal rates is copied
            cap = max(cap, n_in)
            x = np.float32(g.standard_normal((4, max(n_in, 1)))).astype(np.float64)
            gx = Guarded((4, max(n_in, 1)), dev, torch.from_numpy(np.float32(x)))
            gy = Guarded((4, max(cap, 1)), dev)
            assert rs_call(gx, n_in, rates, new, gy, cap, dev) == 0, lib().l2h_last_error().decode()
            torch.cuda.synchronize(dev)
            got = gy.t.cpu().numpy()
            if cap == 0:
                assert is_sentinel(gy.t)
            else:
                rs_check("resample", got[:, :cap], x[:, :n_in], rates, new, cap, range(4), errs, shown)
            assert gx.ok() and gy.ok()
    live = {m: v for m, v in shown.items()}
    if (orig, new) == (720000, 16000):                  # 45:1 stages 12023 floats; 46:1 (12290) is refused
        gx, gy = Guarded((1, 4600), dev), Guarded((1, 100), dev)
        assert rs_call(gx, 4600, [736000], 16000, gy, 100, dev) == 2 and is_sentinel(gy.t)
    check("resample", errs, live, [])


@pytest.mark.parametrize("split", ["rates", "runs", "rows"])
def test_resample_launch_splits(split, dev):
    """rows on both sides of a launch split at RS_MAX_RATES (16), RS_MAX_RUNS (768) and RS_MAX_ROWS (65535)"""
    new = 16000
    if split == "rates":
        rates = [8000 + 1000 * k for k in range(17) if 8000 + 1000 * k != new] + [48000]
        edge = 16
    elif split == "runs":
        rates = [48000 if k % 2 else 44100 for k in range(770)]
        edge = 768
    else:
        rates = [48000] * 65537
        edge = 65535
    n_in = 30
    g = np.random.default_rng(len(rates))
    x = np.float32(g.standard_normal((len(rates), n_in))).astype(np.float64)
    cap = max(ors.output_length(n_in, r, new) for r in rates)
    gx = Guarded(x.shape, dev, torch.from_numpy(np.float32(x)))
    gy = Guarded((len(rates), cap), dev)
    assert rs_call(gx, n_in, rates, new, gy, cap, dev) == 0, lib().l2h_last_error().decode()
    torch.cuda.synchronize(dev)
    got = gy.t.cpu().numpy()
    rows = sorted({0, edge - 2, edge - 1, edge, edge + 1, len(rates) - 1} & set(range(len(rates))))
    errs, shown = {}, {}
    rs_check("split", got, x, rates, new, cap, rows, errs, shown)
    assert gx.ok() and gy.ok()
    check("resample", errs, {}, [])


# (orig, new, block for the whole-period stream)
ST_PAIRS = [(48000, 16000, 384), (16000, 48000, 128), (44100, 16000, 441), (16000, 44100, 160), (8000, 16000, 160)]
PK_PAIRS = ST_PAIRS + [(16001, 16000, None), (16000, 16001, None)]
COUNT_WORDS = lambda D: [None, 0.0, float(D - 1), float(D), float(D + 5), -3.0, math.nan, 3e38]   # noqa: E731


@pytest.mark.parametrize("orig,new,block", ST_PAIRS)
def test_resample_stream(orig, new, block, dev):
    o, q, w, base = rs.rs_filter(orig, new)
    D = w * q // o
    out_block = block // o * q
    g = np.random.default_rng(block + orig)
    errs, shown = {}, {}
    for keep in (0, 5, out_block + 7):
        hist = -(-D * o // q) + w
        T = max(1, min(3, (12288 - hist - keep) // (block + out_block)))
        if keep == 5:                                   # the staging at (or nearest) the 12288-float limit
            T = (12288 - hist - keep) // (block + out_block)
        if T < 1:
            continue
        S, C, n = 3, 2, 2
        rf = hist + keep
        state = Guarded((S, C, rf), dev)
        for s in (0, 2):
            state.t[s] = torch.from_numpy(np.float32(g.standard_normal((C, rf))))
            state.t[s, :, 0] = 0
        for step, cw in enumerate(COUNT_WORDS(D)):
            if cw is not None:
                state.t[2, :, 0] = cw                   # the count word, also the history's first word
            hops = [[1, T, 0, 2, T + 1, -1, 1, 1][step], 1]
            hops[1] = min(T, step % (T + 1))
            sl = [2, [0, 4, -1][step % 3]]
            L = T * block
            x = np.float32(g.standard_normal((n, C, L)))
            gx = Guarded((n, C, L), dev, torch.from_numpy(x))
            Ly = keep + T * out_block
            gy = Guarded((n, C, Ly), dev)
            gs, gh = ints(sl, dev), ints(hops, dev)
            before = state.t.cpu().numpy()
            rc = lib().l2h_resample_stream(ptr(gx), C * L, L, ptr(gy), C * Ly, Ly, n, C, T, ptr(gs), ptr(gh), ptr(state),
                                           S, orig, new, block, keep, None)
            assert rc == 0, lib().l2h_last_error().decode()
            torch.cuda.synchronize(dev)
            got, after = gy.t.cpu().numpy(), state.t.cpu().numpy()
            want_state = before.copy()
            for i in range(n):
                h = hops[i]
                if not (0 <= sl[i] < S and 1 <= h <= T):
                    assert is_sentinel(gy.t[i]), "a row that stores nothing"
                    continue
                for c in range(C):
                    xs = x[i, c, :h * block].astype(np.float64)
                    y, b, st = rs.stream_push(before[sl[i], c], xs, orig, new, block, keep)
                    m = len(y)
                    assert np.isfinite(got[i, c, :m]).all() and is_sentinel(gy.t[i, c, m:])
                    errs["y"] = max(errs.get("y", 0.0), ratio(got[i, c, :m], y, b))
                    st[len(st) - keep:] = got[i, c, m - keep:m]     # the keep tail: the kernel's own outputs
                    want_state[sl[i], c] = np.float32(st)
                    for mu in rs.STREAM_MUTANTS:
                        ym, _, _ = rs.stream_push(before[sl[i], c], xs, orig, new, block, keep, mu)
                        exercise(shown, mu, got[i, c, :m], ym, y, b)
            # the state: the count word and the keep tail exactly, the history copied bit for bit
            assert np.array_equal(i32bits(after), i32bits(want_state)), (keep, step)
            for gb in (gx, gy, gs, gh, state):
                assert gb.ok()
        assert is_sentinel(state.t[1])
    check("stream", errs, shown, [])


PHASE_WORDS = lambda o: [None, float(o - 1), float(o + 3), -2.0, 0.5, 2.7, math.nan]   # noqa: E731


@pytest.mark.parametrize("orig,new,block", PK_PAIRS)
@pytest.mark.parametrize("unit", [1, 3])
def test_resample_packets(orig, new, block, unit, dev):
    o, q, w, base = rs.rs_filter(orig, new)
    D = w * q // o
    g = np.random.default_rng(orig + new + unit)
    errs, shown = {}, {}
    H = -(-(D + 1) * o // q) + w + 1
    for max_in in (882, 12288 - H):                     # the second: history and push at the 12288-float limit
        max_out = -(-max_in * q // o)
        S, C, n = 3, 2, 2
        rf = 2 + H
        state = Guarded((S, C, rf), dev)
        for s in (0, 2):
            state.t[s] = torch.from_numpy(np.float32(g.standard_normal((C, rf))))
            state.t[s, :, :2] = 0
        lens = [0, 1, o - 1, o, o + 1, max_in, 37, 5 * o + 2]
        words = list(zip(COUNT_WORDS(D), PHASE_WORDS(o) + [None]))
        for step, (cw, pw) in enumerate(words):
            for s in (0, 2):
                if cw is not None:
                    state.t[s, :, 0] = cw
                if pw is not None:
                    state.t[s, :, 1] = pw
            k = [lens[step % len(lens)], lens[(step + 3) % len(lens)]]
            counts = [v // unit for v in k]
            if step == 3:
                counts[1] = -1                          # outside [0, max_in]
            if step == 5:
                counts[1] = max_in // unit + 1
            sl = [2, [0, 4, -1][step % 3]]
            pushed = [c * unit if 0 <= c * unit <= max_in else 0 for c in counts]
            x = np.float32(g.standard_normal((n, C, max_in)))
            gx = Guarded((n, C, max_in), dev, torch.from_numpy(x))
            gy = Guarded((n, C, max_out), dev)
            gc, gs, goc = ints(counts, dev), ints(sl, dev), ints([-9] * n, dev)
            before = state.t.cpu().numpy()
            rc = lib().l2h_resample_packets(ptr(gx), C * max_in, max_in, ptr(gy), C * max_out, max_out, n, C, max_in,
                                            ptr(gc), unit, ptr(goc), ptr(gs), ptr(state), S, orig, new, None)
            assert rc == 0, lib().l2h_last_error().decode()
            torch.cuda.synchronize(dev)
            got, after, oc = gy.t.cpu().numpy(), state.t.cpu().numpy(), goc.t.view(torch.int32).tolist()
            want_state = before.copy()
            for i in range(n):
                if not (0 <= sl[i] < S) or pushed[i] == 0:
                    assert oc[i] == 0 and is_sentinel(gy.t[i]), "a row that stores nothing"
                    continue
                for c in range(C):
                    xs = x[i, c, :pushed[i]].astype(np.float64)
                    y, b, st = rs.packet_push(before[sl[i], c], xs, orig, new)
                    m = len(y)
                    assert oc[i] == m and np.isfinite(got[i, c, :m]).all() and is_sentinel(gy.t[i, c, m:])
                    errs["y"] = max(errs.get("y", 0.0), ratio(got[i, c, :m], y, b))
                    want_state[sl[i], c] = np.float32(st)
                    for mu in rs.PACKET_MUTANTS:
                        ym, _, sm = rs.packet_push(before[sl[i], c], xs, orig, new, mu)
                        if len(ym) != m:                # another output count: the exact out_counts word differs
                            shown[mu] = max(shown.get(mu, -math.inf), math.inf)
                        else:
                            exercise(shown, mu, got[i, c, :m], ym, y, b)
                        if not np.array_equal(sm, st):  # the state's exact words: inf where they differ
                            shown[mu] = max(shown.get(mu, -math.inf),
                                            math.inf if not np.array_equal(after[sl[i], c], np.float32(sm)) else 0.0)
            assert np.array_equal(i32bits(after), i32bits(want_state)), (max_in, step)
            for gb in (gx, gy, gc, gs, goc, state):
                assert gb.ok()
        assert is_sentinel(state.t[1])
    check("packets", errs, shown, [])


# ---- the hop FIFO ----------------------------------------------------------------------------------------------------
# (name, head words (pos, held, dropped) written into both listed slots before the call, or None: the kernel's own)
def fifo_presets(cap):
    R = CARRY + cap
    M = INT32_MAX
    return [("fresh", None), ("fill", None), ("overflow", None), ("drain", None), ("drain", None),
            ("pos_last", (R - 1, cap - 300, 0)), ("pos_past", (R + 7, cap - 200, 5)), ("pos_far", (M, 10, 0)),
            ("held_full", (17, cap, 0)), ("held_past", (R - 40, cap + 9, M - 100)), ("held_far", (3, M, 1)),
            ("dropped_max", (5, cap - 50, M)), ("dropped_near", (5, cap - 50, M - 2)), ("negative", (-3, -8, -100)),
            ("wrap", (R - 70, 10, 7)), ("after", None)]


@pytest.mark.parametrize("cap,C,unit", [(200, 1, 1), (300, 2, 3), (1000, 3, 1)])
def test_hop_fifo(cap, C, unit, dev):
    S, n, T, max_in = 4, 3, 3, 600
    R = CARRY + cap
    rf = 3 + R
    state = Guarded((S, C, rf), dev)
    listed = (2, 0)
    g = np.random.default_rng(cap + C)
    for s in listed:                                    # an empty FIFO over a ring of noise, which a chunk may read
        state.t[s] = torch.from_numpy(np.concatenate([np.zeros((C, 3), np.float32),
                                                      np.float32(g.standard_normal((C, R)))], 1))
    pushes = {"fresh": 0, "fill": min(cap, max_in), "overflow": max_in, "drain": 0, "wrap": max_in, "after": 7}
    for seg, (name, head) in enumerate(fifo_presets(cap)):
        if head is not None:
            for s in listed:
                state.t[s, :, :3] = torch.from_numpy(np.tile(words(head), (C, 1)))
        sl = [2, 0, [-1, S, S + 9][seg % 3]]            # the third row's slot lies outside the state
        m = [pushes.get(name, int(g.integers(0, max_in // unit + 1)) * unit) for _ in range(2)]
        counts = [v // unit for v in m] + [5]
        if name == "drain":
            counts[1] = [-1, max_in // unit + 1][seg % 2]   # outside [0, max_in]: a push of nothing
        m = [c * unit if 0 <= c * unit <= max_in else 0 for c in counts]
        x = Guarded((n, C, max_in), dev)
        for i in range(n):                              # samples past a row's push keep the sentinel: never read
            x.t[i, :, :m[i]] = torch.from_numpy(np.float32(g.standard_normal((C, m[i]))))
        chunk = Guarded((n, C, HOP * T + CARRY), dev)
        hops = ints([-7] * n, dev)
        before = state.t.cpu().numpy()
        want = before.copy()
        gcounts, gslots = ints(counts, dev), ints(sl, dev)    # held until the kernel has run: no reuse of their memory
        rc = lib().l2h_hop_fifo(ptr(x), C * max_in, max_in, max_in, ptr(gcounts), unit, ptr(chunk), C * (HOP * T + CARRY),
                                HOP * T + CARRY, ptr(hops), n, C, T, ptr(gslots), ptr(state), S, cap, None)
        assert rc == 0, lib().l2h_last_error().decode()
        torch.cuda.synchronize(dev)
        got_chunk, got_hops = chunk.t.cpu().numpy(), hops.t.view(torch.int32).tolist()
        xs = x.t.cpu().numpy()
        for i, s in enumerate(sl):
            if not 0 <= s < S:
                assert got_hops[i] == 0 and is_sentinel(chunk.t[i]), "a slot outside the state stores nothing"
                continue
            for c in range(C):
                row = before[s, c]
                ck, h, head2, writes = ps.fifo_push(row[:3].view(np.int32).tolist(), row[3:], xs[i, c, :m[i]], cap, T)
                assert got_hops[i] == h, (name, i)
                assert np.array_equal(i32bits(got_chunk[i, c, :HOP * h + CARRY]), i32bits(ck)), (name, i, c)
                assert is_sentinel(chunk.t[i, c, HOP * h + CARRY:]), "past the chunk"
                want[s, c, :3] = words(head2)
                for k, v in writes.items():
                    want[s, c, 3 + k] = v
        assert np.array_equal(i32bits(state.t.cpu().numpy()), i32bits(want)), name
        for gb in (x, chunk, hops, state, gcounts, gslots):
            assert gb.ok()
    assert is_sentinel(state.t[1]) and is_sentinel(state.t[3]), "unlisted slots"
    check("fifo", 0.0, {}, [state])


@pytest.mark.parametrize("cap,C", [(192, 1), (700, 2), (4096, 3)])
def test_enroll_capture(cap, C, dev):
    S, n, T = 4, 3, 3
    rf = 2 + cap
    state = Guarded((S, C, rf), dev)
    listed = (2, 0)
    for s in listed:
        state.t[s] = 0
    g = np.random.default_rng(cap + 7 * C)
    M = INT32_MAX
    presets = [None, None, (cap - 1, cap), (cap, cap + 1), (M, M), (-5, -5), (cap + 3, -1), (7, M - 1), None,
               (cap - 2, 3), None]
    for seg, head in enumerate(presets):
        if head is not None:
            for s in listed:
                state.t[s, :, :2] = torch.from_numpy(np.tile(words(head), (C, 1)))
        sl = [2, 0, [-1, S, 1 + S][seg % 3]]
        hops = [T if seg % 4 == 1 else int(g.integers(1, T + 1)), int(g.integers(0, T + 2)), 2]
        if seg % 5 == 2:
            hops[1] = -1
        chunk = Guarded((n, C, HOP * T + CARRY), dev, torch.from_numpy(np.float32(g.standard_normal((n, C, HOP * T + CARRY)))))
        before = state.t.cpu().numpy()
        want = before.copy()
        gslots, ghops = ints(sl, dev), ints(hops, dev)
        rc = lib().l2h_enroll_capture(ptr(chunk), C * (HOP * T + CARRY), HOP * T + CARRY, n, C, T, ptr(gslots), ptr(ghops),
                                      ptr(state), S, cap, None)
        assert rc == 0, lib().l2h_last_error().decode()
        torch.cuda.synchronize(dev)
        ck = chunk.t.cpu().numpy()
        for i, s in enumerate(sl):
            if not (0 <= s < S and 1 <= hops[i] <= T):
                continue
            for c in range(C):
                head2, writes = ps.capture_push(before[s, c, :2].view(np.int32).tolist(),
                                                ck[i, c, CARRY:CARRY + HOP * hops[i]], cap)
                want[s, c, :2] = words(head2)
                for k, v in writes.items():
                    want[s, c, 2 + k] = v
        assert np.array_equal(i32bits(state.t.cpu().numpy()), i32bits(want)), (seg, head, hops)
        assert chunk.ok() and state.ok() and gslots.ok() and ghops.ok()
    assert is_sentinel(state.t[1]) and is_sentinel(state.t[3]), "unlisted slots"
    check("capture", 0.0, {}, [state])


def test_hop_fifo_past_int32_indices(dev):
    """capacity 2^30 + 64: pos = R - 1 and held = capacity - 100, a push of 300 samples.  The append's ring index pos +
    held + i and the chunk read's pos + R - 64 + i both pass INT32_MAX; they must wrap in the ring, in int64."""
    cap = 2 ** 30 + 64
    R = CARRY + cap
    free = torch.cuda.mem_get_info(dev)[0]
    if free < 8 * 2 ** 30:
        pytest.skip(f"a 4.3 GB FIFO state needs 8 GB of free device memory, {free / 2 ** 30:.1f} GB free")
    T = 3
    head = (R - 1, cap - 100, INT32_MAX - 150)
    state = Guarded((1, 1, 3 + R), dev)
    st = state.t[0, 0]
    g = np.random.default_rng(30)
    # the ring words the chunk reads: the carry ring[R - 65 .. R - 1], then ring[0 .. 383]
    carry = np.float32(g.standard_normal(CARRY + 1))
    front = np.float32(g.standard_normal(HOP * T))
    st[:3] = torch.from_numpy(words(head))
    st[3 + R - CARRY - 1:3 + R] = torch.from_numpy(carry)
    st[3:3 + HOP * T] = torch.from_numpy(front)
    ring = {R - CARRY - 1 + i: v for i, v in enumerate(carry)} | {i: v for i, v in enumerate(front)}
    x = Guarded((1, 1, 300), dev, torch.from_numpy(np.float32(g.standard_normal(300))))
    chunk = Guarded((1, 1, HOP * T + CARRY), dev)
    hops = ints([-7], dev)
    counts, slots = ints([300], dev), ints([0], dev)
    rc = lib().l2h_hop_fifo(ptr(x), 300, 300, 300, ptr(counts), 1, ptr(chunk), HOP * T + CARRY, HOP * T + CARRY,
                            ptr(hops), 1, 1, T, ptr(slots), ptr(state), 1, cap, None)
    assert rc == 0, lib().l2h_last_error().decode()
    torch.cuda.synchronize(dev)
    want, h, head2, writes = ps.fifo_push(list(head), ring, x.t[0, 0].cpu().numpy(), cap, T)
    assert (R - 1) + (cap - 100) > INT32_MAX and min(writes) == cap - 101 and h == T
    assert hops.t.view(torch.int32).tolist() == [h]
    assert np.array_equal(i32bits(chunk.t[0, 0].cpu().numpy()), i32bits(want))
    assert st[:3].view(torch.int32).tolist() == list(head2) and head2[2] == INT32_MAX
    idx = torch.tensor(sorted(writes), dtype=torch.int64, device=dev) + 3
    assert np.array_equal(i32bits(st[idx].cpu().numpy()), i32bits([writes[k] for k in sorted(writes)]))
    # nothing else written: the words that differ from the sentinel are the head, the hand-set ones and the appended ones
    changed = torch.nonzero(bits(state.t).view(-1) != SENTINEL).view(-1).cpu()
    expect = sorted({0, 1, 2} | {3 + k for k in ring} | {3 + k for k in writes})
    assert changed.tolist() == expect
    assert state.ok() and chunk.ok() and x.ok()
    check("fifo", 0.0, {}, [state])


# ---- the target mixer ------------------------------------------------------------------------------------------------
def decode(st):
    """a device mixer state [rows, C, 4] as the model's float64 words"""
    a = np.asarray(st, np.float32)
    out = a.astype(np.float64)
    out[..., 2:] = a[..., 2:].view(np.int32)
    return out


def encode(model):
    a = model[..., :2].astype(np.float32)
    return np.concatenate([a, np.asarray(model[..., 2:], np.int64).astype(np.int32).view(np.float32)], -1)


def set_call(state, NR, S, C, rows, gains, fades, starts, dev):
    """l2h_target_mix_set, run to its end: its lists are held until then, so no list's memory is reused under it"""
    n = len(rows)
    lists = [ints(rows, dev), Guarded((n,), dev, torch.tensor(gains, dtype=torch.float32)),
             None if starts is None else Guarded((n,), dev, torch.tensor(starts, dtype=torch.float32)), ints(fades, dev)]
    rc = lib().l2h_target_mix_set(ptr(state), NR, S, C, ptr(lists[0]), n, ptr(lists[1]), ptr(lists[2]), ptr(lists[3]),
                                  None)
    torch.cuda.synchronize(dev)
    assert all(g is None or g.ok() for g in lists)
    return rc


def test_target_mix_set(dev):
    NR, S, C = 5, 3, 4
    state = Guarded((NR + S, C, 4), dev)
    state.t[:NR + S - 1] = 0                            # the last row is never listed
    g = np.random.default_rng(8)
    errs, shown = {}, {"set_start": -math.inf}
    sets = [([0, 1, 2, NR, NR + 1], [1.5, 0.0, 0.5, 0.75, 1.0], [300, 0, 1000, 97, 2 ** 31 - 2], [0.2, 1.0, 0.0, 0.0, 0.5]),
            ([1, 2, -1, NR + S, NR + 1], [0.25, 2.0, 1.0, 1.0, 0.0], [INT32_MAX - 1, 4096, 5, 5, INT32_MAX], None),
            ([0, 3, 4, NR], [0.0, 1.0, 0.5, 0.3], [-1, 0, 200, 50], None)]
    for k, (rows, gains, fades, starts) in enumerate(sets):
        gains = np.float32(gains).tolist()              # the fp32 values the device stores
        starts = None if starts is None else np.float32(starts).tolist()
        # mid-ramp positions written by hand, so a set without starts continues from them
        st = decode(state.t.cpu().numpy())
        for r in (0, 1, 2, NR):
            st[r, :, 3] = g.integers(0, 500, C)
        state.t.copy_(torch.from_numpy(encode(st)))
        before = state.t.cpu().numpy()
        model = decode(before)
        bound = tm.model_set(model, NR, rows, gains, fades, starts, with_bound=True)
        mut = decode(before)
        tm.model_set(mut, NR, rows, gains, fades, starts, mutant="set_start")
        assert set_call(state, NR, S, C, rows, gains, fades, starts, dev) == 0, lib().l2h_last_error().decode()
        torch.cuda.synchronize(dev)
        got = state.t.cpu().numpy()
        assert np.array_equal(got[..., 1:].view(np.int32), encode(model)[..., 1:].view(np.int32)), k
        assert np.array_equal(got[-1].view(np.int32), before[-1].view(np.int32)), "a row no set lists"
        k = slice(0, NR + S - 1)                        # the sentinel row is checked bit for bit above
        errs["start"] = max(errs.get("start", 0.0), ratio(got[k, :, 0], model[k, :, 0], bound[k]))
        if not np.array_equal(mut[k, :, 0], model[k, :, 0]):
            shown["set_start"] = max(shown["set_start"], ratio(got[k, :, 0], mut[k, :, 0], bound[k]))
    assert is_sentinel(state.t[-1])
    assert shown["set_start"] > -math.inf, "a set without starts continues a running ramp"
    check("mix_set", errs, shown, [state])


# (live terms of the three listeners, C, offsets form): "plain" offsets, or "ragged": non-monotonic and out of range
MIX_CASES = [((1, 63, 64), 1, "plain"), ((65, 128, 129), 2, "plain"), ((3, 1, 2), 8, "ragged"), ((64, 2, 65), 3, "ragged")]


def mix_layout(terms, form):
    """records (two outside the state after listener 1's) and offsets"""
    records, offsets = [], [0]
    for i, k in enumerate(terms):
        rows = list(range(len(records), len(records) + k))
        records += rows
        if i == 1:
            records += [-1, 10 ** 6]                    # records outside the state: not terms
        offsets.append(len(records))
    if form == "ragged":                                # the separator's clamp: running max of offsets clamped to [0, R]
        R = len(records)
        offsets = [-4, offsets[1], offsets[1] - 1, R + 5]
    return records, offsets


def mix_call(y, ys, ck, cs, out, os_, n, R, C, T, records, offsets, hops, slots, state, NR, S):
    return lib().l2h_target_mix(ptr(y), *ys, ptr(ck), *cs, ptr(out), *os_, n, R, C, T, ptr(records), ptr(offsets),
                                ptr(hops), ptr(slots), ptr(state), NR, S, None)


def strided(dev, R, C, L, pad, values=None):
    """a Guarded [R][C][L] tensor with `pad` floats after each channel row: (buffer, view, (row, ch) strides)"""
    ch = L + pad
    buf = Guarded((R * C * ch,), dev)
    v = buf.t.as_strided((R, C, L), (C * ch, ch, 1))
    if values is not None:
        v.copy_(torch.from_numpy(np.asarray(values, np.float32)))
    return buf, v, (C * ch, ch)


# ramp words (g0, g1, F + 1, p) written by hand: F + 1 = 0 and < 0, p > F, p < 0, F + 1 = INT32_MAX from two positions
RAMP_PRESETS = [(0.5, 1.0, 0, 3), (0.25, 1.5, 101, 150), (0.0, 1.0, INT32_MAX, 5),
                (0.5, 1.0, -7, 3), (0.25, 1.5, 101, -20), (1.0, 0.0, INT32_MAX, 2 ** 30)]


def hand_ramps(model, live, S, step):
    """three of RAMP_PRESETS (the first three at step 1, the others at step 3) over records of live terms, and the
    ambient ramp of one slot; returns {record: preset}"""
    C, NR = model.shape[1], model.shape[0] - S
    picks = [r for r in live if r not in (1, 2)][:3]     # not the muted term or the ramp to 0
    assert len(picks) == 3, "every preset reaches a live term"
    placed = dict(zip(picks, RAMP_PRESETS[:3] if step == 1 else RAMP_PRESETS[3:]))
    for r, w in placed.items():
        model[r] = np.tile(np.array(w, np.float64), (C, 1))
    model[NR + (step % S)] = np.tile(np.array((0.0, 0.4, 400, 100 * step), np.float64), (C, 1))
    return placed


@pytest.mark.parametrize("terms,C,form", MIX_CASES, ids=lambda v: str(v))
def test_target_mix(terms, C, form, dev):
    g = np.random.default_rng(sum(terms) * 10 + C)
    T, n, S = 3, 3, 5
    L = HOP * T
    records, offsets = mix_layout(terms, form)
    R = len(records)
    NR = sum(terms) + 2
    slots_v = [3, 0, 1]
    state = Guarded((NR + S, C, 4), dev)
    state.t[:NR + S - 1] = 0                            # the last slot is never listed
    # ramps through the set kernel: fades, gains to 0 (a muted term), and one ramp to 0 that the NaN case below uses
    rows = list(range(NR)) + [NR + s for s in range(S - 1)]
    fades = [int(v) for v in g.choice([0, 1, 97, 128, 300, 1000, 5000], len(rows))]
    gns = [float(v) for v in np.float32(g.uniform(0.1, 2.0, len(rows)))]
    starts = [float(v) for v in np.float32(g.uniform(0.0, 2.0, len(rows)))]
    muted, to_zero = 1 % NR, 2 % NR
    gns[muted], fades[muted], gns[to_zero], fades[to_zero], starts[to_zero] = 0.0, 0, 0.0, 200, 0.8
    assert set_call(state, NR, S, C, rows, gns, fades, starts, dev) == 0
    # the sum order shows only where rounding is exact (test_target_mix_sum_order), the set's start in test_target_mix_set
    errs, shown = {}, {m: -math.inf for m in tm.MIX_MUTANTS if m not in ("reversed", "set_start")}
    neg_zero, placed = 0, {}
    start_of = tm.clamped_starts(offsets, R)
    for step in range(4):
        # at step 1 every listener mixes and none has a chunk: a ragged case's listener 1, with no rows, is all -0
        hops = [[T, 1, T], [2, 1, 3], [1, T + 1, -1], None][step]
        sl = list(slots_v)
        if step == 2:
            sl[0] = S + 2                               # outside the state
        model0 = decode(state.t.cpu().numpy())
        if step in (1, 3):
            live = [records[r] for i in range(n) if 1 <= (T if hops is None else hops[i]) <= T
                    for r in range(start_of[i], start_of[i + 1]) if 0 <= records[r] < NR]
            placed = hand_ramps(model0, live, S, step)
            state.t.copy_(torch.from_numpy(encode(model0)))
            model0 = decode(state.t.cpu().numpy())
        y = np.float32(g.standard_normal((R, C, L)))
        chunk = np.float32(g.standard_normal((n, C, L + CARRY))) if step != 1 else None
        # the muted term's row is the sentinel, and the ramp to 0 is NaN where its gain is exactly 0
        y[muted] = np.float32(np.nan)
        y[muted].view(np.int32)[:] = SENTINEL
        w = model0[to_zero]
        for c in range(C):
            g0, g1, F, p = tm.ramp(w[c], 1.0)
            G, _ = tm.ramp_gains(g0, g1, F, p + np.arange(L) + 1)
            y[to_zero, c, G == 0] = np.nan
        hv = None if hops is None else ints(hops, dev)
        lists = dict(records=ints(records, dev), offsets=ints(offsets, dev), hops=hv, slots=ints(sl, dev))
        model = model0.copy()
        want, bound = tm.model_mix(model, NR, y.astype(np.float64), records, offsets, sl, hops,
                                   None if chunk is None else chunk.astype(np.float64), with_bound=True)
        results = []
        start = state.t.clone()
        for pad in (0, 1):                              # the float4 form, then the scalar one
            state.t.copy_(start)
            gy, vy, ys = strided(dev, R, C, L, pad, y)
            if chunk is None:
                gc, cs = None, (0, 0)
            else:
                gc, _, cs = strided(dev, n, C, L + CARRY, 4 * pad + 3 * pad, chunk)
            go, vo, os_ = strided(dev, n, C, L, 0 if pad == 0 else 5)
            rc = mix_call(gy, ys, gc, cs, go, os_, n, R, C, T, lists["records"], lists["offsets"], hv, lists["slots"],
                          state, NR, S)
            assert rc == 0, lib().l2h_last_error().decode()
            torch.cuda.synchronize(dev)
            results.append((vo.cpu().numpy(), state.t.cpu().numpy()))
            for gb in (gy, gc, go, state, *lists.values()):
                assert gb is None or gb.ok()
        (out, st), (out1, st1) = results
        assert np.array_equal(out.view(np.int32), out1.view(np.int32)), "the scalar and float4 forms differ"
        assert np.array_equal(st.view(np.int32), st1.view(np.int32))
        assert np.array_equal(st.view(np.int32), encode(model).view(np.int32)), step
        assert is_sentinel(state.t[-1]), "an unlisted slot"
        e = 0.0
        for i in range(n):
            h = T if hops is None else hops[i]
            if not (0 <= sl[i] < S and 1 <= h <= T):
                assert np.isnan(out[i]).all() and (out[i].view(np.int32) == SENTINEL).all(), "stores nothing"
                continue
            m = HOP * h
            assert np.isfinite(out[i, :, :m]).all(), "no NaN reaches out"
            assert (out[i, :, m:].view(np.int32) == SENTINEL).all(), "past the row's hops"
            e = max(e, ratio(out[i, :, :m], want[i, :, :m], bound[i, :, :m]))
            zero = (want[i, :, :m] == 0) & (bound[i, :, :m] == 0)
            neg_zero += int(np.signbit(want[i, :, :m][zero]).sum())
            assert np.array_equal(np.signbit(out[i, :, :m][zero]), np.signbit(want[i, :, :m][zero])), "-0 where no term enters"
        errs["out"] = max(errs.get("out", 0.0), e)
        for r, w in placed.items():                     # p > F stays as written: only a running ramp advances
            if step in (1, 3) and w[3] > w[2] - 1 >= 0:
                assert (st[r, :, 3].view(np.int32) == w[3]).all()
        for mu in shown:
            mm = model0.copy()
            mo = tm.model_mix(mm, NR, y.astype(np.float64), records, offsets, sl, hops,
                              None if chunk is None else chunk.astype(np.float64), mutant=mu)
            live = ~np.isnan(want)
            mo = np.where(live & np.isnan(mo), np.inf, mo)  # a mutant that lets a NaN through misses everywhere
            if mu == "p_frozen":                        # p is an exact word: the margin is inf where it differs
                if not np.array_equal(mm, model):
                    shown[mu] = math.inf if not np.array_equal(st.view(np.int32), encode(mm).view(np.int32)) else 0.0
                continue
            if np.array_equal(mo[live], want[live]):
                continue
            shown[mu] = max(shown[mu], max(ratio(out[i, :, :HOP * (T if hops is None else hops[i])],
                                                 mo[i, :, :HOP * (T if hops is None else hops[i])],
                                                 bound[i, :, :HOP * (T if hops is None else hops[i])])
                                           for i in range(n) if live[i].any()))
    if form == "ragged":
        assert neg_zero > 0, "a sample no term enters"
    check("mix", errs, {m: v for m, v in shown.items() if v > -math.inf}, [state])


def test_target_mix_sum_order(dev):
    """rows 2^25, -2^25, b at a gain of 1: the row order's sum is b exactly, the reverse order's is not"""
    st, y = tm._cancelling_case()
    y32 = np.float32(y)
    state = Guarded((4, 1, 4), dev, torch.zeros(4, 1, 4))
    gy = Guarded((3, 1, HOP), dev, torch.from_numpy(y32))
    go = Guarded((1, 1, HOP), dev)
    lists = [ints(v, dev) for v in ([0, 1, 2], [0, 3], [1], [0])]
    rc = mix_call(gy, (HOP, HOP), None, (0, 0), go, (HOP, HOP), 1, 3, 1, 1, *lists, state, 3, 1)
    assert rc == 0, lib().l2h_last_error().decode()
    torch.cuda.synchronize(dev)
    want, bound = tm.model_mix(st.copy(), 3, y, [0, 1, 2], [0, 3], [0], with_bound=True)
    rev = tm.model_mix(st.copy(), 3, y, [0, 1, 2], [0, 3], [0], mutant="reversed")
    got = go.t.cpu().numpy()
    check("mix", ratio(got, want, bound), {"reversed": ratio(got, rev, bound)}, [state, gy, go])


def test_summary():
    LEDGER.summary()
