"""Host-side checks of the target mixer, no device: a float64 numpy model of the mix (l2h_target_mix) and of its gain
ramps (the reference of tests/test_target_mix_gpu.py and test_stream_stage_kernels_gpu.py), the bound on the device's
error from it and its mutants, with their own checks; the layout; the argument errors of both C
entries, returned before anything is enqueued; the Python checks of TargetMixer; the header; the exports."""
import ctypes
import math

import numpy as np
import pytest
import torch

from lookoncetohear_b200 import TargetMixer
from serving_util import declaration, doc_before, header

HOP, CARRY, WORDS = 128, 64, 4
ENTRIES = ("l2h_target_mix_layout", "l2h_target_mix", "l2h_target_mix_set")


# ---- the model -------------------------------------------------------------------------------------------------------
# A state is float64 [records + slots, C, 4]: g0, g1, F + 1 (0: never set) and p, as the device's words.
def gain(g0, g1, F, q):
    """G(q): the gain of the sample at ramp position q"""
    if q + 1 >= F:
        return g1
    return g0 + (g1 - g0) * (1 - math.cos(math.pi * (q + 1) / F)) / 2


def ramp(w, rest):
    """(g0, g1, F, p) of a state word, a fresh one settled at `rest`"""
    if w[2] <= 0:
        return rest, rest, 0, 0
    F = int(w[2]) - 1
    return w[0], w[1], F, min(max(int(w[3]), 0), F)


def level(w, rest):
    """the gain of the last sample the row mixed (the start of a set without one)"""
    g0, g1, F, p = ramp(w, rest)
    return g1 if p >= F else g0 + (g1 - g0) * (1 - math.cos(math.pi * p / F)) / 2


def model_state(records, slots, C):
    return np.zeros((records + slots, C, WORDS))


def model_set(state, n_records, rows, gains, fades, starts=None, with_bound=False, mutant=None):
    """l2h_target_mix_set over state rows (records b, slots n_records + s).  With with_bound, returns [rows, C]: a bound
    on the device's error in each row's start word, which is 0 where `starts` gives it or the set stores nothing.
    `mutant` "set_start" starts a set without starts one sample late."""
    bound = np.zeros(state.shape[:2])
    for e, r in enumerate(rows):
        if not (0 <= r < state.shape[0]) or not (0 <= fades[e] < 2 ** 31 - 1):
            continue
        for c in range(state.shape[1]):
            if starts is None:
                g0, g1, F, p = ramp(state[r, c], 1.0 if r < n_records else 0.0)
                G, E = ramp_gains(g0, g1, F, [p + (mutant == "set_start")])
                g, bound[r, c] = G[0], E[0]
            else:
                g = starts[e]
            state[r, c] = (g, gains[e], fades[e] + 1, 0)
    return bound if with_bound else None


def clamped_starts(offsets, R):
    """the offsets as the separator clamps them: the running maximum of each clamped into [0, R]"""
    return np.maximum.accumulate(np.clip(np.asarray(offsets), 0, R)).tolist()


# The device's error.  The build has no --use_fast_math, so (float)q / (float)F is an IEEE division (0.5 ulp) and cospif
# is the CUDA Math API's (1 ulp, its documented maximum); every other operation rounds once, to fp32.
U = 2.0 ** -24                                              # the unit roundoff of fp32
MIX_MUTANTS = ("q", "linear", "ambient_64", "reversed", "p_frozen", "set_start")


def ramp_gains(g0, g1, F, k, mutant=None):
    """(G, E): the ramp's levels after k samples (an array; the sample at ramp position q is mixed at k = q + 1) and a
    bound on the error of the device's fp32 ramp_level at each.  At or past the ramp's end the device takes g1 itself:
    E = 0."""
    k = np.asarray(k, np.float64)
    D = g1 - g0
    flat = k >= F
    Fs = max(F, 1)
    t = k / Fs
    c = np.cos(np.pi * t)
    d = 1 - c
    G = np.where(flat, g1, g0 + D * (t if mutant == "linear" else d / 2))
    # (float)k and (float)F round past 2^24, then the quotient: t's error, then cospif's 1 ulp plus the slope times it
    et = t * (np.where(k >= 2 ** 24, U, 0) + (U if F >= 2 ** 24 else 0) + U) * (1 + 4 * U)
    ec = 2 * U * np.abs(c) + np.pi * et + 2.0 ** -149
    ed = ec + U * (d + ec)                                  # 1 - cospif
    ep = abs(D) * ed + d * U * abs(D) + U * abs(D) * (d + ed)   # (g1 - g0) * (1 - cospif), then * 0.5 exactly
    E = (ep / 2 + U * (np.abs(G) + ep / 2)) * (1 + 8 * U)   # g0 + ..., rounded
    return G, np.where(flat, 0.0, E)


def _exact_sum(a, b):
    """a + b in float64 and whether that sum is exact (two-sum)"""
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb) == 0


def model_mix(state, n_records, y, records, offsets, slots, hops=None, chunk=None, out=None, with_bound=False,
              mutant=None):
    """l2h_target_mix on numpy: y [R, C, 128 T], chunk [n, C, 128 T + 64] or None.  Returns out [n, C, 128 T] (NaN where
    nothing is written, unless `out` is given) and advances the state's ramps.  With with_bound, returns (out, bound):
    per sample, a bound on |device - out| for the sequential fmaf sum from -0 in row order, then the ambient term.  Each
    term adds its fp32 gain's error times |x|, and each fmaf one rounding of its result, which is 0 where the gain is
    exact, the sum so far has no error and the new sum is an fp32 number.  A sample no term enters is -0.  `mutant`
    (MIX_MUTANTS) computes a subtly wrong mix instead ("reversed": the fp32 sum in reverse order)."""
    R, C, L = y.shape
    T, n, n_slots = L // HOP, len(slots), state.shape[0] - n_records
    out = np.full((n, C, L), np.nan) if out is None else out
    bound = np.zeros((n, C, L))
    start = clamped_starts(offsets, R)
    for i in range(n):
        h = T if hops is None else hops[i]
        if not (0 <= slots[i] < n_slots and 1 <= h <= T):
            continue
        m = HOP * h
        terms = [(y[r], state[records[r]], 1.0) for r in range(start[i], start[i + 1]) if 0 <= records[r] < n_records]
        if chunk is not None:
            terms.append((chunk[i, :, 64:] if mutant == "ambient_64" else chunk[i], state[n_records + slots[i]], 0.0))
        for c in range(C):
            acc, err = np.full(m, -0.0), np.zeros(m)
            acc32 = np.full(m, -0.0, np.float32)
            for x, w, rest in (terms[::-1] if mutant == "reversed" else terms):
                g0, g1, F, p = ramp(w[c], rest)
                G, E = ramp_gains(g0, g1, F, p + np.arange(m) + (0 if mutant == "q" else 1), mutant)
                live = G != 0                               # a term enters only the samples where its gain is not 0
                xs = np.where(live, x[c, :m], 0.0)
                new, exact = _exact_sum(acc, G * xs)
                ex = exact & (err == 0) & (E == 0) & (np.float32(new) == new)
                ea = E * np.abs(xs)
                err = np.where(live, err + ea + np.where(ex, 0.0, U * (np.abs(new) + err + ea)), err)
                acc = np.where(live, new, acc)
                acc32 = np.where(live, np.float32(acc32 + np.float32(G * xs)), acc32)
            out[i, c, :m] = acc32 if mutant == "reversed" else acc
            bound[i, c, :m] = err
        if mutant == "p_frozen":
            continue
        for _, w, rest in terms + ([] if chunk is not None else [(None, state[n_records + slots[i]], 0.0)]):
            for c in range(C):
                g0, g1, F, p = ramp(w[c], rest)
                if w[c, 2] > 0 and p < F:                   # only a running ramp advances, from its clamped p
                    w[c, 3] = min(F, p + m)
    return (out, bound) if with_bound else out


# ---- the model's own checks ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F", [1, 2, 127, 128, 129, 480, 1000])
def test_ramp_ends_at_target(F):
    g = [gain(0.25, 1.5, F, q) for q in range(F + 3)]
    assert g[F - 1] == 1.5 and g[F] == 1.5 and g[F + 2] == 1.5
    assert all(a <= b for a, b in zip(g, g[1:]))                  # a raised cosine: monotone
    assert g[0] == pytest.approx(0.25 + 1.25 * (1 - math.cos(math.pi / F)) / 2, abs=1e-15)
    assert gain(0.25, 1.5, 0, 0) == 1.5                            # F = 0: an immediate change


def _schedule(total, T, seed):
    """hop counts in [0, T] (zeros included) that add up to `total`"""
    g = np.random.default_rng(seed)
    hops = []
    while sum(hops) < total:
        hops.append(int(min(g.integers(0, T + 1), total - sum(hops))))
    return hops


def _ticks(state, n_records, ys, chunk_sig, records, offsets, slots, schedules, T):
    """mix each listener's whole signals in ticks of the given hop schedules (one per listener, padded with zeros)"""
    n = len(slots)
    ticks = max(len(s) for s in schedules)
    pos, got = [0] * n, [[] for _ in range(n)]
    R, C, _ = ys.shape
    owner = [next(i for i in range(n) if offsets[i] <= r < offsets[i + 1]) for r in range(R)]
    for t in range(ticks):
        hops = [s[t] if t < len(s) else 0 for s in schedules]
        y = np.full((R, C, HOP * T), np.nan)
        ck = np.full((n, C, HOP * T + CARRY), np.nan)
        for r in range(R):
            i = owner[r]
            y[r, :, :HOP * hops[i]] = ys[r, :, pos[i]:pos[i] + HOP * hops[i]]
        for i in range(n):
            ck[i, :, :HOP * hops[i]] = chunk_sig[i, :, pos[i]:pos[i] + HOP * hops[i]]
        out = model_mix(state, n_records, y, records, offsets, slots, hops, ck)
        for i in range(n):
            got[i].append(out[i, :, :HOP * hops[i]])
            pos[i] += HOP * hops[i]
    return [np.concatenate(g, 1) for g in got]


def test_model_chunking_invariance():
    """16 hops of ramps cut into ticks of one hop or into mixes of 0-3 hops: the same output and the same ramps"""
    C, n_rec, n_slots, total = 2, 6, 3, 16
    g = np.random.default_rng(5)
    ys = g.standard_normal((4, C, HOP * total))
    amb = g.standard_normal((2, C, HOP * total))
    records, offsets, slots = [4, 0, 2, 5], [0, 3, 4], [2, 0]
    outs = []
    for sched in ([[1] * total] * 2, [_schedule(total, 3, 6), _schedule(total, 3, 7)]):
        st = model_state(n_rec, n_slots, C)
        model_set(st, n_rec, [4, 0, 2, 5, n_rec + 2, n_rec], [1.0, 0.0, 2.0, 0.5, 0.3, 1.0], [127, 129, 1000, 0, 300, 1],
                  [0.0, 1.0, 0.5, 1.0, 0.0, 0.0])
        outs.append((_ticks(st, n_rec, ys, amb, records, offsets, slots, sched, 3), st))
    (a, sa), (b, sb) = outs
    assert all(np.array_equal(x, z) for x, z in zip(a, b))
    assert np.array_equal(sa, sb)


def test_model_set_without_start_continues():
    """a set halfway through a ramp starts where the ramp got to: the new ramp's first gain is next to the old one's last"""
    C, st = 1, model_state(2, 1, 1)
    model_set(st, 2, [0], [0.0], [1000], [1.0])
    y = np.ones((1, C, HOP))
    out = model_mix(st, 2, y, [0], [0, 1], [0])
    last = out[0, 0, -1]
    assert last == pytest.approx(gain(1.0, 0.0, 1000, HOP - 1)) and level(st[0, 0], 1.0) == pytest.approx(last)
    model_set(st, 2, [0], [1.0], [480])
    out = model_mix(st, 2, y, [0], [0, 1], [0])
    assert out[0, 0, 0] == pytest.approx(last + (1 - last) * (1 - math.cos(math.pi / 480)) / 2)
    assert abs(out[0, 0, 0] - last) < 1e-4


def test_model_fresh_rows_and_store_rules():
    st = model_state(3, 2, 2)
    y = np.arange(3 * 2 * HOP * 2, dtype=np.float64).reshape(3, 2, 2 * HOP)
    out = model_mix(st, 3, y, [0, 1, 2], [0, 2, 3], [0, 1], hops=[2, 1])
    assert np.array_equal(out[0], y[0] + y[1]) and np.array_equal(out[1, :, :HOP], y[2, :, :HOP])
    assert np.isnan(out[1, :, HOP:]).all() and not st.any()
    out = model_mix(st, 3, y, [0, 1, 2], [0, 2, 3], [0, 5], hops=[0, 1])            # h = 0, slot outside: nothing
    assert np.isnan(out).all()
    assert clamped_starts([2, 1, 9, 0], 3) == [2, 2, 3, 3]


def _ramped_case(seed, C=2, T=2):
    """one listener of three running ramps and an ambient ramp, one hop count T"""
    g = np.random.default_rng(seed)
    st = model_state(4, 2, C)
    model_set(st, 4, [0, 1, 3, 4 + 1], [0.25, 1.5, 0.0, 0.75], [700, 97, 2 ** 31 - 2, 300], [1.0, 0.0, 0.5, 0.0])
    st[1, :, 3] = 40
    y = np.float32(g.standard_normal((3, C, HOP * T))).astype(np.float64)
    ck = np.float32(g.standard_normal((1, C, HOP * T + CARRY))).astype(np.float64)
    return st, y, ck


def _fp32_mix(state, y, chunk, records):
    """an fp32 emulation of one listener's mix (numpy's float32 cos for cospif), for the bound's own check"""
    f = np.float32
    C, m = y.shape[1], y.shape[2]
    out = np.full((C, m), f(-0.0))
    for x, w, rest in [(y[r], state[records[r]], 1.0) for r in range(len(records))] + [(chunk, state[-1], 0.0)]:
        for c in range(C):
            g0, g1, F, p = ramp(w[c], rest)
            k = p + np.arange(m) + 1
            lv = f(g0) + (f(g1) - f(g0)) * (f(1) - np.cos(f(np.pi) * (k.astype(f) / f(F)))) * f(0.5)
            gk = np.where(k >= F, f(g1), lv.astype(f))
            live = gk != 0
            out[c] = np.where(live, (out[c].astype(np.float64) + gk.astype(np.float64) * x[c, :m]).astype(f), out[c])
    return out


def test_mix_bound_covers_fp32_and_is_zero_where_exact():
    st, y, ck = _ramped_case(1)
    model_set(st, 4, [5], [0.75], [300], [0.0])          # the ambient ramp of slot 1, used by listener 0 below
    emu = _fp32_mix(st.copy(), y, ck[0], [0, 1, 3])
    st2 = st.copy()
    st2[4] = st[5]                                       # the listener's slot is 0
    out, bound = model_mix(st2, 4, y, [0, 1, 3], [0, 3], [0], chunk=ck, with_bound=True)
    assert (bound[0] > 0).all() and np.all(np.abs(emu - out[0]) <= bound[0])
    assert bound.max() < 1e-5
    # rest gains of 1 and integer samples: every fmaf exact, the bound 0, a sample no term enters -0
    st = model_state(3, 1, 1)
    yi = np.arange(3 * HOP, dtype=np.float64).reshape(3, 1, HOP) - 100
    yi[2, 0, 5] = 0
    out, bound = model_mix(st, 3, yi, [0, 1, 2], [0, 3], [0], with_bound=True)
    assert not bound.any() and np.array_equal(out[0], yi.sum(0))
    model_set(st, 3, [0, 1, 2], [0.0, 0.0, 0.0], [0, 0, 0], [0.0, 0.0, 0.0])
    out, bound = model_mix(st, 3, yi, [0, 1, 2], [0, 3], [0], with_bound=True)
    assert not bound.any() and np.signbit(out).all() and not out.any()


def _cancelling_case():
    """rest gains of 1: rows 2^25, -2^25, b (the row order's fp32 sum is b exactly; the reverse order loses b)"""
    st = model_state(3, 1, 1)
    b = np.float32(np.random.default_rng(3).standard_normal(HOP)).astype(np.float64)
    y = np.stack([np.full(HOP, 2.0 ** 25), np.full(HOP, -2.0 ** 25), b])[:, None]
    return st, y


@pytest.mark.parametrize("mutant", MIX_MUTANTS)
def test_mix_mutants_miss_their_bound(mutant):
    from kernels.scaffold import SENSITIVITY, ratio
    if mutant == "reversed":
        st, y = _cancelling_case()
        want, bound = model_mix(st.copy(), 3, y, [0, 1, 2], [0, 3], [0], with_bound=True)
        assert not bound.any()
        got = model_mix(st.copy(), 3, y, [0, 1, 2], [0, 3], [0], mutant=mutant)
        assert ratio(got, want, bound) >= SENSITIVITY
        return
    st, y, ck = _ramped_case(2)
    if mutant == "set_start":
        a, b = st.copy(), st.copy()
        bound = model_set(a, 4, [1, 0], [0.5, 0.5], [10, 10], with_bound=True)
        model_set(b, 4, [1, 0], [0.5, 0.5], [10, 10], mutant=mutant)
        assert ratio(b[:2, :, 0], a[:2, :, 0], bound[:2]) >= SENSITIVITY
        return
    a, b = st.copy(), st.copy()
    want, bound = model_mix(a, 4, y, [0, 1, 3], [0, 3], [1], chunk=ck, with_bound=True)
    got = model_mix(b, 4, y, [0, 1, 3], [0, 3], [1], chunk=ck, mutant=mutant)
    if mutant == "p_frozen":
        assert not np.array_equal(a, b) and np.array_equal(want, got)
    else:
        assert ratio(got, want, bound) >= SENSITIVITY


# ---- the library -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from lookoncetohear_b200 import build, _cabi
    build.build()
    return _cabi.lib()


def test_entries_exported_and_declared(lib):
    from lookoncetohear_b200 import _cabi
    hdr = header()
    for name in ENTRIES:
        assert hasattr(lib, name), name
        assert name in _cabi.declared_symbols(), name
        assert declaration(hdr, name)[0] is not None, name
    import lookoncetohear_b200 as pkg
    assert "TargetMixer" in pkg.__all__


def test_layout(lib):
    row = ctypes.c_int32(-1)
    assert lib.l2h_target_mix_layout(ctypes.byref(row)) == 0 and row.value == WORDS
    assert lib.l2h_target_mix_layout(None) == 1


def test_header_documents_the_mix():
    hdr = header()
    decl, args = declaration(hdr, "l2h_target_mix")
    assert args == ["y_dev", "y_row_stride", "y_ch_stride", "chunk_dev", "chunk_row_stride", "chunk_ch_stride", "out_dev",
                    "out_row_stride", "out_ch_stride", "n", "R", "channels", "frames", "records_dev", "offsets_dev",
                    "hops_dev", "slots_dev", "state_dev", "n_records", "n_slots", "stream"]
    _, set_args = declaration(hdr, "l2h_target_mix_set")
    assert set_args == ["state_dev", "n_records", "n_slots", "channels", "rows_dev", "n", "gains_dev", "starts_dev",
                        "fades_dev", "stream"]
    doc = doc_before(hdr, hdr.index("int l2h_target_mix_layout("))
    for phrase in ("raised cosine", "look-ahead", "bit for bit", "before anything is enqueued", "CUDA graph",
                   "All zeros is a fresh row", "stores nothing", "row order", "between them", "chunk_dev may be NULL"):
        assert phrase in doc, phrase


# argument errors: fake device addresses far apart, so only the argument under test is wrong
Y, CK, OUT, LIST, ST = (ctypes.c_void_p(a) for a in (0x1000000, 0x2000000, 0x3000000, 0x4000000, 0x5000000))


def _mix(lib, n=2, R=3, C=2, T=3, S=4, NR=8, y=Y, ck=CK, out=OUT, rec=LIST, off=LIST, hops=LIST, slots=LIST, st=ST,
         y_row=None, y_ch=None, c_row=None, c_ch=None, o_row=None, o_ch=None):
    L = HOP * T
    y_ch = L if y_ch is None else y_ch
    c_ch = L + CARRY if c_ch is None else c_ch
    o_ch = L if o_ch is None else o_ch
    y_row = C * y_ch if y_row is None else y_row
    c_row = C * c_ch if c_row is None else c_row
    o_row = C * o_ch if o_row is None else o_row
    return lib.l2h_target_mix(y, y_row, y_ch, ck, c_row, c_ch, out, o_row, o_ch, n, R, C, T, rec, off, hops, slots, st,
                              NR, S, None)


def test_mix_argument_errors(lib):
    for kw in ({"y": None}, {"out": None}, {"rec": None}, {"off": None}, {"slots": None}, {"st": None}):
        assert _mix(lib, **kw) == 1, kw
        assert b"null" in lib.l2h_last_error()
    for kw in ({"n": 0}, {"R": 0}, {"C": 0}, {"T": 0}, {"NR": 0}, {"S": 0}, {"n": -1}, {"T": -3}):
        assert _mix(lib, **kw) == 1, kw
        assert b"positive" in lib.l2h_last_error(), kw
    assert _mix(lib, n=4, R=3) == 1 and b"n <= R" in lib.l2h_last_error()
    assert _mix(lib, n=3, R=5, S=2) == 1 and b"n_slots" in lib.l2h_last_error()
    assert _mix(lib, T=2 ** 24) == 1 and b"frames" in lib.l2h_last_error()
    L = HOP * 3
    for kw in ({"y_ch": L - 1}, {"y_row": 2 * L - 1}, {"o_ch": L - 4}, {"o_row": L}, {"c_ch": L + CARRY - 1},
               {"c_row": 2 * (L + CARRY) - 1}):
        assert _mix(lib, **kw) == 1, kw
        assert b"stride" in lib.l2h_last_error(), kw
    for kw in ({"out": Y}, {"out": ctypes.c_void_p(0x1000000 + 4 * (3 * 2 * L - 1))}, {"out": CK},
               {"out": ctypes.c_void_p(0x2000000 - 4)}):
        assert _mix(lib, **kw) == 1, kw
        assert b"overlap" in lib.l2h_last_error(), kw


def _set(lib, st=ST, NR=8, S=4, C=2, rows=LIST, n=3, gains=LIST, starts=LIST, fades=LIST):
    return lib.l2h_target_mix_set(st, NR, S, C, rows, n, gains, starts, fades, None)


def test_set_argument_errors(lib):
    for kw in ({"st": None}, {"rows": None}, {"gains": None}, {"fades": None}):
        assert _set(lib, **kw) == 1, kw
        assert b"null" in lib.l2h_last_error()
    for kw in ({"NR": 0}, {"S": 0}, {"C": 0}, {"n": 0}, {"n": -2}):
        assert _set(lib, **kw) == 1, kw
        assert b"positive" in lib.l2h_last_error()
    assert _set(lib, NR=2 ** 31 - 2, S=2) == 1 and b"too large" in lib.l2h_last_error()


# ---- the Python checks -----------------------------------------------------------------------------------------------
def test_constructor_checks():
    for bad in ({"records": 0}, {"slots": 0}, {"channels": 0}, {"records": 1.5}, {"slots": True},
                {"records": 2 ** 30, "slots": 2 ** 30}):
        kw = {"records": 8, "slots": 4, "channels": 2, "device": "cuda"}
        kw.update(bad)
        with pytest.raises(ValueError):
            TargetMixer(**kw)
    with pytest.raises(RuntimeError, match="CUDA"):
        TargetMixer(8, 4, 2, device="cpu")


def _host_mixer(NR=8, S=4, C=2):
    """a TargetMixer whose state lives in host memory: the Python checks run, no engine call is reached"""
    m = TargetMixer.__new__(TargetMixer)
    m.n_records, m.n_slots, m.channels = NR, S, C
    m.state = torch.zeros(NR + S, C, WORDS)
    return m


def test_set_checks():
    m = _host_mixer()
    for gains in (float("nan"), float("inf"), -0.1, 16.5, True, "1", [1.0, 1.0]):
        with pytest.raises(ValueError):
            m.set_gains([0, 1, 2], gains)
    for fade in (-1, 1.5, 2 ** 31 - 1, True, [1, 2]):
        with pytest.raises(ValueError):
            m.set_gains([0, 1, 2], 1.0, fade=fade)
    for start in (float("nan"), -1.0, 17.0):
        with pytest.raises(ValueError):
            m.set_gains([0], 1.0, start=start)
    for records in ([8], [-1], [1, 1], [], [0.5]):
        with pytest.raises(ValueError):
            m.set_gains(records, 1.0)
    for slots in ([4], [-1], [2, 2]):
        with pytest.raises(ValueError):
            m.set_ambient(slots, 0.1)
    with pytest.raises(ValueError, match="a record lies outside"):
        m.reset(records=[8])
    with pytest.raises(ValueError, match="a slot lies outside"):
        m.reset(slots=[4])
    with pytest.raises(ValueError, match="integer record indices"):
        m.reset(records=[0.5])


def test_reset_one_list():
    """reset with only records, only slots, both or neither: the listed rows fresh, every other row kept"""
    m = _host_mixer(4, 3, 2)
    m.state.uniform_(0.5, 1.0)
    before = m.state.clone()
    m.reset(slots=[1])
    assert not m.state[4 + 1].any()
    m.reset(records=[2, 0])
    assert not m.state[[0, 2]].any()
    m.reset(records=torch.tensor([3]), slots=(2,))
    m.reset()
    kept = [1, 4]                                   # record 1 and slot 0
    assert torch.equal(m.state[kept], before[kept])
    assert not m.state[[0, 2, 3, 5, 6]].any()


def test_mix_needs_cuda():
    m = _host_mixer()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(3, 2, HOP), [0, 1, 2], [0, 2, 3], [0, 1])


def test_level_and_fading_follow_the_model():
    """the device views computed from hand-written words (here in host memory) against the model's level"""
    NR, S = 3, 2
    m = _host_mixer(NR, S, 1)
    words = [(0.0, 0.0, 0, 0), (0.5, 1.5, 101, 40), (2.0, 0.0, 11, 10), (0.0, 0.2, 481, 500), (0.7, 0.3, 1, 9)]
    for r, (g0, g1, f1, p) in enumerate(words):
        m.state[r, 0, 0], m.state[r, 0, 1] = g0, g1
        m.state[r, 0, 2:].view(torch.int32)[:] = torch.tensor([f1, p], dtype=torch.int32)
    want = [level(np.array(w, dtype=np.float64), 1.0 if r < NR else 0.0) for r, w in enumerate(words)]
    assert m.level.tolist() == pytest.approx(want, abs=1e-6)
    assert m.level[0] == 1.0 and m.level[3] == pytest.approx(0.2) and m.level[4] == pytest.approx(0.3)
    assert m.fading.tolist() == [False, True, False, False, False]
    m.state[0, 0, 2:].view(torch.int32)[:] = torch.tensor([0, 0], dtype=torch.int32)
    m.reset(records=[1], slots=[0])
    assert m.level.tolist()[:4] == pytest.approx([1.0, 1.0, want[2], 0.0]) and not m.fading.any()
