"""Host-side checks of enrollment from a listener's own stream, no device: the two entry points are built, exported and
declared; the capture's layout and its refusal of capacities under the shortest enrollment; a numpy model of the capture
(l2h_enroll_capture) whose "last L samples of slot s" is what was pushed to s; and the argument errors of the C entries
(returned before anything is enqueued) and of EnrollCapture and EmbedTFGridNet.enroll."""
import ctypes

import numpy as np
import pytest
import torch

from lookoncetohear_b200 import EmbedTFGridNet, EnrollCapture
from serving_util import FAKE_DEV, declaration, header

HEAD, HOP, CARRY = 2, 128, 64
ENTRIES = ("l2h_enroll_capture_layout", "l2h_enroll_capture", "l2h_embed_forward_slots")


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


@pytest.mark.parametrize("capacity", [192, 193, 1000, 48000, 16000 * 10])
def test_layout(lib, capacity):
    row = ctypes.c_int32()
    assert lib.l2h_enroll_capture_layout(capacity, ctypes.byref(row)) == 0
    assert row.value == HEAD + capacity


@pytest.mark.parametrize("capacity", [191, 128, 0, -1])
def test_layout_refuses_short_capacity(lib, capacity):
    row = ctypes.c_int32(-7)
    assert lib.l2h_enroll_capture_layout(capacity, ctypes.byref(row)) == 1
    assert b"192" in lib.l2h_last_error() and row.value == -7
    assert lib.l2h_enroll_capture_layout(192, None) == 1


# ---- a numpy model of the capture ------------------------------------------------------------------------------------
def model_capture(state, chunk, slots, hops, T):
    """l2h_enroll_capture on numpy: state [S, C, 2 + cap] float32 (head words as int32 bits), chunk [n, C, 128 T + 64]"""
    S, C, row = state.shape
    cap = row - HEAD
    head = state[..., :HEAD].view(np.int32)
    for i, (s, h) in enumerate(zip(slots, hops)):
        if not (0 <= s < S and 1 <= h <= T):
            continue
        new = chunk[i, :, CARRY:CARRY + HOP * h]
        for c in range(C):
            w, k = int(head[s, c, 0]), int(head[s, c, 1])
            for j in range(max(0, new.shape[1] - cap), new.shape[1]):
                state[s, c, HEAD + (w + j) % cap] = new[c, j]
            head[s, c, 0] = (w + new.shape[1]) % cap
            head[s, c, 1] = min(k + new.shape[1], cap)


def model_last(state, s, L):
    """[C, L] the last L samples slot s captured (L <= captured)"""
    cap = state.shape[2] - HEAD
    w, k = state[s, 0, :HEAD].view(np.int32)
    assert L <= k
    return state[s][:, HEAD + (w - L + np.arange(L)) % cap]


@pytest.mark.parametrize("cap", [192, 500, 1000])
def test_model_last_samples_are_what_was_pushed(cap):
    """random hop schedules with 0 hops, slots outside the state and rings that wrap many times"""
    S, C, T, n, ticks = 5, 2, 3, 4, 120
    g = np.random.default_rng(cap)
    state = np.zeros((S, C, HEAD + cap), np.float32)
    pushed = [np.zeros((C, 0), np.float32) for _ in range(S)]
    for t in range(ticks):
        slots = g.permutation(S)[:n].tolist()
        slots[t % n] = [-1, S, S + 3, -100][t % 4]
        hops = g.integers(0, T + 1, n).tolist()
        chunk = g.standard_normal((n, C, HOP * T + CARRY)).astype(np.float32)
        model_capture(state, chunk, slots, hops, T)
        for i, (s, h) in enumerate(zip(slots, hops)):
            if 0 <= s < S:
                pushed[s] = np.concatenate([pushed[s], chunk[i, :, CARRY:CARRY + HOP * h]], 1)
    for s in range(S):
        k = state[s, 0, 1].view(np.int32)
        assert k == min(pushed[s].shape[1], cap)
        assert pushed[s].shape[1] > 2 * cap              # wrapped
        for L in (192, k // 2, k):
            assert np.array_equal(model_last(state, s, L), pushed[s][:, pushed[s].shape[1] - L:])


# ---- argument errors -------------------------------------------------------------------------------------------------
def _cap_call(lib, n=2, C=2, T=3, slots=FAKE_DEV, hops=FAKE_DEV, state=FAKE_DEV, S=4, cap=1000, row=None, ch=None):
    L = HOP * T + CARRY
    ch = L if ch is None else ch
    row = C * ch if row is None else row
    return lib.l2h_enroll_capture(FAKE_DEV, row, ch, n, C, T, slots, hops, state, S, cap, None)


def test_capture_argument_errors(lib):
    assert _cap_call(lib, slots=None) == 1
    assert _cap_call(lib, hops=None) == 1
    assert _cap_call(lib, state=None) == 1
    for kw in ({"n": 0}, {"C": 0}, {"T": 0}, {"S": 0}, {"n": 5}, {"cap": 191}, {"ch": HOP * 3 + CARRY - 1},
               {"row": 2 * (HOP * 3 + CARRY) - 1}):
        assert _cap_call(lib, **kw) == 1, kw


@pytest.fixture(scope="module")
def handle(lib, embed_params):
    net = EmbedTFGridNet(**embed_params)            # weights never committed
    h = net._engine()
    yield h
    del net


def _slots_call(lib, h, lens, slots=(0, 1), on_dev=False, S=4, cap=1000, n_max=None, stride=256, used=FAKE_DEV,
                ws_bytes=None, both=False, neither=False):
    B = len(lens)
    n_max = max(lens, default=1000) if n_max is None else n_max
    if ws_bytes is None:
        w = ctypes.c_size_t()
        assert lib.l2h_embed_workspace_bytes(h, max(B, 1), max(n_max, 192), ctypes.byref(w)) == 0
        ws_bytes = w.value
    sh = (ctypes.c_int32 * len(slots))(*slots)
    s_host = None if (on_dev or neither) else sh
    s_dev = FAKE_DEV if (on_dev or both) and not neither else None
    ln = (ctypes.c_int32 * max(B, 1))(*lens)
    return lib.l2h_embed_forward_slots(h, FAKE_DEV, S, cap, s_host, s_dev, ln, B, n_max, FAKE_DEV, stride, used, FAKE_DEV,
                                       ws_bytes, None)


def test_forward_slots_argument_errors(lib, handle):
    # all good but the weights: error 4 once every argument passed
    assert _slots_call(lib, handle, [1000, 192]) == 4
    assert _slots_call(lib, handle, [1000, 192], on_dev=True) == 4
    assert _slots_call(lib, None, [1000, 192], ws_bytes=1 << 40) == 1
    assert _slots_call(lib, handle, [1000, 192], used=None) == 1
    assert _slots_call(lib, handle, [1000, 192], both=True) == 1
    assert _slots_call(lib, handle, [1000, 192], neither=True) == 1
    assert _slots_call(lib, handle, [1000, 192], slots=(0, 4)) == 1
    assert b"outside" in lib.l2h_last_error()
    assert _slots_call(lib, handle, [1000, 192], slots=(-1, 0)) == 1
    assert _slots_call(lib, handle, [1000, 192], slots=(2, 2)) == 1
    assert b"twice" in lib.l2h_last_error()
    assert _slots_call(lib, handle, [1000, 191]) == 1
    assert _slots_call(lib, handle, [1000, 192], n_max=999) == 1
    assert _slots_call(lib, handle, [1000, 192], cap=999) == 1                    # n_max > capacity
    assert b"capacity" in lib.l2h_last_error()
    assert _slots_call(lib, handle, [1000, 192], cap=191, n_max=191) == 1
    assert _slots_call(lib, handle, [1000, 192], stride=255) == 1
    assert _slots_call(lib, handle, [1000, 192], S=0) == 1
    assert _slots_call(lib, handle, [1000] * 5, slots=(0, 1, 2, 3, 4), S=4) == 1    # batch > n_slots
    assert _slots_call(lib, handle, [], slots=()) == 1
    assert _slots_call(lib, handle, [1000, 192], ws_bytes=1024) == 1


def test_enroll_capture_python_checks():
    for bad in ({"slots": 0}, {"channels": 0}, {"capacity": 191}, {"capacity": 1.5}, {"slots": True}):
        kw = {"slots": 4, "channels": 2, "capacity": 1000, "device": "cuda"}
        kw.update(bad)
        with pytest.raises(ValueError):
            EnrollCapture(**kw)
    with pytest.raises(RuntimeError, match="CUDA"):
        EnrollCapture(4, 2, 1000, device="cpu")


def _host_capture(S=4, C=2, cap=1000):
    """an EnrollCapture whose state lives in host memory, for the Python argument checks (no engine call is reached)"""
    c = EnrollCapture.__new__(EnrollCapture)
    c.n_slots, c.channels, c.capacity = S, C, cap
    c.state = torch.zeros(S, C, HEAD + cap)
    return c


def test_enroll_python_checks(embed_params):
    net = EmbedTFGridNet(**embed_params)
    cap = _host_capture()
    with pytest.raises(TypeError):
        net.enroll(object(), [0], [500])
    with pytest.raises(ValueError, match="channels"):
        net.enroll(_host_capture(C=1), [0], [500])
    for slots in ([0, 0], [0, 4], [-1, 1], [0.5, 1], [[0, 1]], []):
        with pytest.raises(ValueError):
            net.enroll(cap, slots, [500] * max(len(slots), 1))
    for lens in ([500], [500, 191], [500, 1001], [500, 2.5]):
        with pytest.raises(ValueError):
            net.enroll(cap, [0, 1], lens)
    with pytest.raises(ValueError, match="out"):
        net.enroll(cap, [0, 1], [500, 500], out=torch.zeros(2, 255))
    with pytest.raises(ValueError, match="out"):
        net.enroll(cap, [0, 1], [500, 500], out=torch.zeros(2, 256, dtype=torch.float64))
    with pytest.raises(ValueError, match="out"):
        net.enroll(cap, [0, 1], [500, 500], out=torch.zeros(256, 2).t())
    with pytest.raises(ValueError, match="used"):
        net.enroll(cap, [0, 1], [500, 500], used=torch.zeros(2, dtype=torch.int64))
    with pytest.raises(ValueError, match="used"):
        net.enroll(cap, [0, 1], [500, 500], used=torch.zeros(3, dtype=torch.int32))
