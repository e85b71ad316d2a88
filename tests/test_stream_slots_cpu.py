"""Host-side checks of the per-stream clock entry points: the record offsets they rely on, and the argument errors the
calls return before they touch the device (no GPU needed; the handles below never commit weights)."""
import ctypes

import pytest
import torch

import serving_util as su
from serving_util import FAKE_DEV, eng  # noqa: F401


def _slots(*s):
    return (ctypes.c_int32 * len(s))(*s)


def test_offsets_query_keeps_the_first_16_and_adds_the_clock(eng):
    net, h, L = eng
    old = (ctypes.c_int64 * 16)()
    assert L.l2h_sep_state_offsets(h, old, 16) == 0
    new = (ctypes.c_int64 * 18)()
    assert L.l2h_sep_state_offsets(h, new, 18) == 0
    assert list(new)[:16] == list(old)
    st_emb, st_gate, st_pos, st_calls = new[5], new[6], new[16], new[17]
    # the clock lives in the spare words between the embedding copy and the gate: the record size does not change
    assert st_emb + 256 < st_calls < st_pos < st_pos + 2 <= st_gate
    assert st_pos % 2 == 0
    assert L.l2h_sep_state_offsets(h, old, 15) == 1
    big = (ctypes.c_int64 * 20)(*([-7] * 20))
    assert L.l2h_sep_state_offsets(h, big, 20) == 0 and list(big)[18:] == [-7, -7]


def test_sepstate_layout_names_the_clock(eng):
    net, _, _ = eng
    st = su.host_state(net, 3)
    pos, calls = st._clocks()
    pos.copy_(torch.tensor([5, 0, 1 << 40]))
    calls.copy_(torch.tensor([3, 0, 8], dtype=torch.int32))
    assert st.stream_pos() == [5, 0, 1 << 40]
    assert st.header() == (0, 0)


def test_reset_streams_argument_errors(eng):
    _, h, L = eng
    st = None
    assert L.l2h_sep_state_reset_streams(h, None, 4, _slots(0), 1, st) == 1            # null state
    assert L.l2h_sep_state_reset_streams(h, FAKE_DEV, 4, None, 1, st) == 1             # null slot list
    assert L.l2h_sep_state_reset_streams(None, FAKE_DEV, 4, _slots(0), 1, st) == 1     # null handle
    assert L.l2h_sep_state_reset_streams(h, FAKE_DEV, 0, _slots(0), 1, st) == 1        # batch 0
    assert L.l2h_sep_state_reset_streams(h, FAKE_DEV, 4, _slots(0), 0, st) == 1        # no slots
    assert L.l2h_sep_state_reset_streams(h, FAKE_DEV, 4, _slots(4), 1, st) == 1        # out of range
    assert b"outside" in L.l2h_last_error()
    assert L.l2h_sep_state_reset_streams(h, FAKE_DEV, 4, _slots(-1), 1, st) == 1
    assert L.l2h_sep_state_reset_streams(h, FAKE_DEV, 4, _slots(1, 2, 1), 3, st) == 1  # duplicate
    assert b"twice" in L.l2h_last_error()


def test_copy_streams_argument_errors(eng):
    _, h, L = eng
    a, b = FAKE_DEV, ctypes.c_void_p(0x20000)
    assert L.l2h_sep_state_copy_streams(h, None, 4, _slots(0), b, 4, _slots(0), 1, None) == 1
    assert L.l2h_sep_state_copy_streams(h, a, 4, _slots(0), None, 4, _slots(0), 1, None) == 1
    assert L.l2h_sep_state_copy_streams(h, a, 4, _slots(4), b, 4, _slots(0), 1, None) == 1       # destination range
    assert L.l2h_sep_state_copy_streams(h, a, 4, _slots(0), b, 2, _slots(2), 1, None) == 1       # source range
    assert L.l2h_sep_state_copy_streams(h, a, 4, _slots(1, 1), b, 4, _slots(0, 2), 2, None) == 1  # destination twice
    assert L.l2h_sep_state_copy_streams(h, a, 4, _slots(1, 2), a, 4, _slots(2, 3), 2, None) == 1  # read and overwritten
    assert b"both a source and a destination" in L.l2h_last_error()


def test_forward_active_argument_errors(eng):
    _, h, L = eng
    p = FAKE_DEV
    mask = ctypes.c_void_p(0x30000)
    # a mask with a multi-frame call
    assert L.l2h_sep_forward_active(h, p, 384, 192, 192, p, p, p, 256, 128, 128, 1, 5, p, 1 << 20, 0, None, mask) == 1
    assert b"one-hop" in L.l2h_last_error()
    # a mask with the taps
    assert L.l2h_sep_forward_active(h, p, 384, 192, 192, p, p, p, 256, 128, 128, 1, 1, p, 1 << 20, 1, None, mask) == 1


def test_python_arguments_raise_value_error(eng):
    net, _, _ = eng
    st = su.host_state(net, 2)
    with pytest.raises(ValueError):
        st.reset_streams([0])                   # no engine behind a hand-made state
    st._net = net
    for bad in ([], [2], [0, 0]):
        with pytest.raises(ValueError):
            st.reset_streams(bad)
    with pytest.raises(ValueError):
        st.copy_streams_from(st, [0], [0, 1])
    with pytest.raises(ValueError):
        st.copy_streams_from(st, [0], [0])      # the same record read and overwritten
    with pytest.raises(ValueError):
        net._active_mask(torch.ones(2, dtype=torch.float32), torch.device("cpu"), 2)
    with pytest.raises(ValueError):
        net._active_mask(torch.ones(3, dtype=torch.bool), torch.device("cpu"), 2)
    assert net._active_mask(torch.ones(2, dtype=torch.bool), torch.device("cpu"), 2).dtype == torch.uint8
