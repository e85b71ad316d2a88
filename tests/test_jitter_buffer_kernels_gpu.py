"""jitter_buffer_kernel called directly (l2h_jitter_buffer on raw device buffers): states set by hand, the ring full and
wrapping inside one call, every row starting a loss run, lags at tau_min and tau_max, the sentinel outside everything a
call writes, and mutants of the concealment.  The oracle is the model of tests/test_jitter_buffer_cpu.py run from the
same state: integer words, tags and ring exactly, samples and history within BOUND_U fp32 units of the call's peak."""
import ctypes

import numpy as np
import pytest
import torch

import test_jitter_buffer_cpu as jm
from kernels.scaffold import Guarded, Ledger, bits, dev, is_sentinel, ratio  # noqa: F401
from lookoncetohear_b200 import _cabi

pytestmark = pytest.mark.gpu

BOUND_U = 16
LEDGER = Ledger()


@pytest.fixture(scope="module")
def lib():
    return _cabi.lib()


def voiced_state(p, S, seed, period=None):
    """S slot states whose history holds a voiced signal (an exact period of `period` samples if given), started at
    sequence number 100 + s with nothing pending"""
    st = p.fresh(S)
    for s in range(S):
        if period is None:
            sig = jm.voiced(p.rate, 95.0 + 40 * s, p.H, seed + s, p.C)
        else:
            t = np.arange(p.H)
            sig = np.stack([0.4 * np.sin(2 * np.pi * t / period + c) + 0.1 * np.sin(6 * np.pi * t / period)
                            for c in range(p.C)]).astype(np.float32)
        st[s, :, p.o_hist:p.o_per] = sig
        w = st[s].view(np.int32)
        w[0, 0], w[0, 1] = 1, 100 + s
    return st


def run(lib, dev, p, st, x, seqs, counts, slots, extra_out=0):
    """one kernel call on guarded buffers: (y, out counts, state after) with the guards and every sample past each
    row's output checked against the sentinel"""
    n, M = len(counts), seqs.shape[1]
    S = st.shape[0]
    gs = Guarded(st.shape, dev, torch.from_numpy(st))
    gx = Guarded((n, p.C, M * p.P), dev, torch.from_numpy(x))
    gy = Guarded((n, p.C, p.max_out * p.P), dev)
    q = torch.tensor(seqs, dtype=torch.int32, device=dev)
    c = torch.tensor(counts, dtype=torch.int32, device=dev)
    sl = torch.tensor(slots, dtype=torch.int32, device=dev)
    oc = torch.full((n,), -7, dtype=torch.int32, device=dev)
    rc = lib.l2h_jitter_buffer(gx.t.data_ptr(), p.C * M * p.P, M * p.P, M, q.data_ptr(), c.data_ptr(), gy.t.data_ptr(),
                               p.C * p.max_out * p.P, p.max_out * p.P, oc.data_ptr(), n, p.C, sl.data_ptr(),
                               gs.t.data_ptr(), S, p.rate, p.P, p.D, p.W, p.max_out, None)
    assert rc == 0, lib.l2h_last_error()
    torch.cuda.synchronize()
    assert gs.ok() and gx.ok() and gy.ok()
    ocl = oc.tolist()
    for i in range(n):
        assert is_sentinel(gy.t[i, :, ocl[i] * p.P:])
    return gy.t.cpu().numpy(), ocl, gs.t.cpu().numpy()


def check(key, p, before, after, y, oc, x, seqs, counts, slots, mutants=None):
    """every listed row against the model from `before`; mutants: {name: (Params, force)} of the model"""
    errs, worst_m = {}, {}
    for i, s in enumerate(slots):
        if not 0 <= s < before.shape[0]:
            assert oc[i] == 0
            continue
        stm, trace = before[s].copy(), []
        want, m = jm.model_call(stm, x[i], seqs[i], counts[i], p, trace=trace)
        lag = int(after[s].view(np.int32)[0, 12])
        force = None
        if trace and lag != stm.view(np.int32)[0, 12]:
            assert len(trace) == 1 and abs(trace[0][1][trace[0][0]] - trace[0][1][lag]) <= \
                trace[0][2][trace[0][0]] + trace[0][2][lag]
            force = [lag]
            stm = before[s].copy()
            want, m = jm.model_call(stm, x[i], seqs[i], counts[i], p, force=force)
        assert oc[i] == m
        assert np.array_equal(after[s][0, :p.o_ring].view(np.int32), stm[0, :p.o_ring].view(np.int32)), \
            (after[s][0, :13].view(np.int32), stm[0, :13].view(np.int32))
        assert np.array_equal(bits(torch.from_numpy(after[s][:, p.o_ring:p.o_hist].copy())),
                              bits(torch.from_numpy(stm[:, p.o_ring:p.o_hist].copy())))
        peak = max(float(np.abs(before[s][:, p.o_hist:]).max()), float(np.abs(x[i]).max(initial=0)), 1e-30)
        bound = BOUND_U * jm.U * peak
        errs[f"row {i}"] = max(ratio(y[i, :, :m * p.P], want, bound),
                               ratio(after[s][:, p.o_hist:], stm[:, p.o_hist:], bound))
        for name, (pm, fm) in (mutants or {}).items():
            sm = before[s].copy()
            wm, mm = jm.model_call(sm, x[i], seqs[i], counts[i], pm, force=fm(trace, force) if fm else force)
            if mm == m and wm.size:
                worst_m[name] = min(worst_m.get(name, np.inf), ratio(y[i, :, :m * p.P], wm, bound))
    LEDGER.check(key, errs, worst_m)


def params(rate, P, C, **kw):
    return jm.Params(rate, P, C=C, **kw)


def mutated(p, **kw):
    q = jm.Params(p.rate, p.P, C=p.C, D=p.D, W=p.W, max_out=p.max_out)
    for k, v in kw.items():
        setattr(q, k, v)
    return q


@pytest.mark.parametrize("rate,P,C", [(16000, 160, 2), (44100, 441, 1), (48000, 480, 2)])
def test_every_row_starts_a_run(lib, dev, rate, P, C):
    """eight rows, each declaring three packets lost and recovering in one call: eight pitch searches"""
    p = params(rate, P, C, D=1, W=8, max_out=5 if P == 160 else 3)
    S, n = 9, 8
    st = voiced_state(p, S, 10)
    slots = list(range(1, 9))
    seqs = np.array([[100 + s + 4, 100 + s + 3] for s in slots], dtype=np.int32)
    x = (0.3 * np.random.default_rng(1).standard_normal((n, C, 2 * P))).astype(np.float32)
    y, oc, after = run(lib, dev, p, st, x, seqs, [2] * n, slots)
    lag1 = lambda tr, f: [(f or [tr[0][0]])[0] + 1]
    mutants = {"lag + 1": (p, lag1), "gain held 20 ms": (mutated(p, ga=jm.rnd(0.02 * rate)), None),
               "no fade": (mutated(p, lr=0), None), "fade 2x": (mutated(p, lr=2 * p.lr), None)}
    if p.max_out < 5:                                  # the fade lies past this call's writes
        mutants = {k: v for k, v in mutants.items() if "fade" not in k}
    check(f"runs {rate}", p, st, after, y, oc, x, seqs, [2] * n, slots, mutants)


@pytest.mark.parametrize("where", ["tmin", "tmax"])
def test_lags_at_the_ends(lib, dev, where):
    p = params(16000, 160, 2, D=0, W=8, max_out=2)
    st = voiced_state(p, 2, 3, period=p.tmin) if where == "tmin" else p.fresh(2)
    if where == "tmax":                                # a zero history: no numerator is positive
        st[:, 0].view(np.int32)[:, :2] = [[1, 100], [1, 101]]
    seqs = np.array([[101, 0], [103, 0]], dtype=np.int32)
    x = (0.2 * np.random.default_rng(2).standard_normal((2, 2, 320))).astype(np.float32)
    y, oc, after = run(lib, dev, p, st, x, seqs, [1, 1], [0, 1])
    assert [int(after[s].view(np.int32)[0, 12]) for s in (0, 1)] == [getattr(p, where)] * 2
    check(f"lag {where}", p, st, after, y, oc, x, seqs, [1, 1], [0, 1])


def test_state_words_set_by_hand(lib, dev):
    p = params(44100, 441, 2, D=1, W=8, max_out=4)
    st = voiced_state(p, 4, 20)
    w = [st[s].view(np.int32) for s in range(4)]
    w[0][0, 1] = 65535                                 # next at the wrap: 0 and 1 follow it
    w[1][0, jm.HEAD:jm.HEAD + p.R] = [12345678, -5, 70000, 102, 0, 1 << 17, 7, 103 | (1 << 17)] * 2   # corrupt tags
    w[1][0, 2], w[1][0, 3] = 5, 2                      # two decided packets: a malformed tag (concealed), then packet 6
    w[2][0, 6:11] = [-3, -1, -2 ** 31, -7, -1]         # negative counters count as 0
    w[3][0, 6:11] = [2 ** 31 - 2] * 5                  # counters near INT32_MAX saturate
    w[3][0, 4], w[3][0, 5] = 99999, 5                  # a run count past its cap and a lag outside the range
    seqs = np.array([[0, 1, 65534, 2], [102, 103, 105, 104], [103, 102, 102, 109], [104, 103, 103, 20000]],
                    dtype=np.int32)
    x = (0.3 * np.random.default_rng(3).standard_normal((4, 2, 4 * 441))).astype(np.float32)
    y, oc, after = run(lib, dev, p, st, x, seqs, [4, 4, 4, 4], [0, 1, 2, 3])
    check("words by hand", p, st, after, y, oc, x, seqs, [4, 4, 4, 4], [0, 1, 2, 3])
    aw = after[3].view(np.int32)[0]
    assert (aw[7], aw[10]) == (2 ** 31 - 1, 2 ** 31 - 1)    # a late 103 and the restart at 20000 saturate


def test_ring_full_and_wrapping_in_one_call(lib, dev):
    """the backlog at the ring's end, a window filled out of order and a full backlog dropping its oldest"""
    p = params(16000, 160, 1, D=2, W=4, max_out=6)
    st = voiced_state(p, 3, 30)
    w = st[0].view(np.int32)
    w[0, 2] = p.R - 2                                  # the oldest unwritten packet two slots from the ring's end
    seqs = np.array([[103, 102, 101, 100, 104, 106, 105, 107],
                     [100, 101, 102, 103, 104, 105, 106, 107],
                     [110, 109, 108, 107, 106, 105, 104, 103]], dtype=np.int32)
    x = (0.3 * np.random.default_rng(4).standard_normal((3, 1, 8 * 160))).astype(np.float32)
    y, oc, after = run(lib, dev, p, st, x, seqs, [8, 8, 8], [0, 1, 2])
    check("ring", p, st, after, y, oc, x, seqs, [8, 8, 8], [0, 1, 2])
    assert int(after[1].view(np.int32)[0, 9]) == 3     # 101 .. 107 released into a backlog of 4: the 3 oldest go


def test_rows_that_store_nothing_keep_everything(lib, dev):
    p = params(16000, 160, 2)
    st = voiced_state(p, 3, 40)
    x = np.ones((3, 2, 320), np.float32)
    seqs = np.array([[101, 102], [101, 102], [101, 102]], dtype=np.int32)
    y, oc, after = run(lib, dev, p, st, x, seqs, [2, 3, -1], [-1, 0, 1])
    assert oc == [0, 0, 0]
    assert np.array_equal(after.view(np.int32), st.view(np.int32))


def test_ledger_summary():
    LEDGER.summary()
