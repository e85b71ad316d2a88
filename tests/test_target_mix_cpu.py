"""Host-side checks of the target mixer, no device: a float64 numpy model of the mix (l2h_target_mix) and of its gain
ramps (the reference of tests/test_target_mix_gpu.py) with its own checks; the layout; the argument errors of both C
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


def model_set(state, n_records, rows, gains, fades, starts=None):
    """l2h_target_mix_set over state rows (records b, slots n_records + s)"""
    for e, r in enumerate(rows):
        if not (0 <= r < state.shape[0]) or not (0 <= fades[e] < 2 ** 31 - 1):
            continue
        for c in range(state.shape[1]):
            g = level(state[r, c], 1.0 if r < n_records else 0.0) if starts is None else starts[e]
            state[r, c] = (g, gains[e], fades[e] + 1, 0)


def clamped_starts(offsets, R):
    """the offsets as the separator clamps them: the running maximum of each clamped into [0, R]"""
    return np.maximum.accumulate(np.clip(np.asarray(offsets), 0, R)).tolist()


def model_mix(state, n_records, y, records, offsets, slots, hops=None, chunk=None, out=None):
    """l2h_target_mix on numpy: y [R, C, 128 T], chunk [n, C, 128 T + 64] or None.  Returns out [n, C, 128 T] (NaN where
    nothing is written, unless `out` is given) and advances the state's ramps."""
    R, C, L = y.shape
    T, n, n_slots = L // HOP, len(slots), state.shape[0] - n_records
    out = np.full((n, C, L), np.nan) if out is None else out
    start = clamped_starts(offsets, R)
    for i in range(n):
        h = T if hops is None else hops[i]
        if not (0 <= slots[i] < n_slots and 1 <= h <= T):
            continue
        m = HOP * h
        terms = [(y[r], state[records[r]], 1.0) for r in range(start[i], start[i + 1]) if 0 <= records[r] < n_records]
        if chunk is not None:
            terms.append((chunk[i], state[n_records + slots[i]], 0.0))
        acc = np.zeros((C, m))
        for x, w, rest in terms:
            for c in range(C):
                g0, g1, F, p = ramp(w[c], rest)
                g = np.array([gain(g0, g1, F, p + s) for s in range(m)])
                live = g != 0                                   # a term enters only the samples where its gain is not 0
                acc[c, live] += g[live] * x[c, :m][live]
        out[i, :, :m] = acc
        for _, w, rest in terms + ([] if chunk is not None else [(None, state[n_records + slots[i]], 0.0)]):
            for c in range(C):
                if w[c, 2] > 0:
                    w[c, 3] = min(int(w[c, 2]) - 1, int(w[c, 3]) + m)
    return out


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
