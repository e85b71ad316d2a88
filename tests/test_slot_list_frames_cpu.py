"""Host-side checks of multi-hop calls over a list of a state's records (l2h_sep_forward_slots_frames,
Net.advance_slots): the argument errors the C call returns before it touches the device, the Python ValueErrors, and the
header's description (no GPU needed; the handle below never commits weights)."""
import ctypes

import pytest
import torch

import serving_util as su
from serving_util import FAKE_DEV, L2H_FLAG_TAPS, eng  # noqa: F401


def _call(L, h, state_batch, slots, n, frames, flags=0, p=FAKE_DEV):
    return L.l2h_sep_forward_slots_frames(h, p, 1024, 512, 128 * frames + 64, p, p, state_batch, slots, n, frames, p, 1024,
                                          512, 128 * frames, p, 1 << 20, flags, None)


def test_forward_slots_frames_argument_errors(eng):
    _, h, L = eng
    sl = ctypes.c_void_p(0x30000)
    assert _call(L, h, 4, None, 2, 3) == 1                   # no slot list
    assert b"null" in L.l2h_last_error()
    assert _call(L, None, 4, sl, 2, 3) == 1                  # no handle
    assert _call(L, h, 4, sl, 2, 3, p=None) == 1             # null buffers
    assert _call(L, h, 4, sl, 0, 3) == 1                     # no rows
    assert _call(L, h, 4, sl, -3, 3) == 1
    assert _call(L, h, 4, sl, 5, 3) == 1                     # more rows than records
    assert b"n <= state_batch" in L.l2h_last_error()
    assert _call(L, h, 0, sl, 1, 3) == 1                     # an empty state
    assert _call(L, h, -2, sl, 1, 3) == 1
    for frames in (0, -1, -128):                             # no hops
        assert _call(L, h, 4, sl, 2, frames) == 1
        assert b"frames > 0" in L.l2h_last_error()
    assert _call(L, h, 4, sl, 2, 3, flags=L2H_FLAG_TAPS) == 1   # the taps belong to the dense chain
    assert b"L2H_FLAG_TAPS" in L.l2h_last_error()


def test_forward_slots_is_the_one_hop_form(eng):
    """l2h_sep_forward_slots passes its arguments on with frames = 1: the same errors, for the same reasons."""
    _, h, L = eng
    sl = ctypes.c_void_p(0x30000)
    p = FAKE_DEV
    assert L.l2h_sep_forward_slots(h, p, 384, 192, 192, p, p, 4, sl, 5, p, 256, 128, 128, p, 1 << 20, 0, None) == 1
    assert b"n <= state_batch" in L.l2h_last_error()


def test_python_advance_slots_raises_value_error(eng):
    net, _, _ = eng
    st = su.host_state(net, 4)
    emb = torch.zeros(2, 256)
    for n in (128 * 3, 128 * 3 + 63, 128 * 3 + 65, 64, 0, 191):          # not 128*T + 64 with T >= 1
        with pytest.raises(ValueError):
            net.advance_slots(torch.zeros(2, 2, n), emb, st, [0, 1])
    with pytest.raises(ValueError):                                      # not [n, M, samples]
        net.advance_slots(torch.zeros(2, 128 * 3 + 64), emb, st, [0, 1])
    with pytest.raises(TypeError):
        net.advance_slots(torch.zeros(2, 2, 128 * 3 + 64), emb, object(), [0, 1])


def test_header_documents_forward_slots_frames():
    hdr = su.header()
    decl, args = su.declaration(hdr, "l2h_sep_forward_slots_frames")
    assert decl, "l2h_sep_forward_slots_frames is not declared"
    assert args == ["handle", "x_dev", "x_batch_stride", "x_ch_stride", "x_len", "emb_dev", "state_dev", "state_batch",
                    "slots_dev", "n", "frames", "y_dev", "y_batch_stride", "y_ch_stride", "y_len", "workspace_dev",
                    "workspace_bytes", "flags", "stream"]
    doc = su.doc_before(hdr, decl.start())
    for phrase in ("128*frames + 64", "128*frames samples", "l2h_sep_workspace_bytes(handle, n, frames, flags)",
                   "outside [0, state_batch)", "for all of its frames", "L2H_FLAG_GRAPH", "frames <= 0", "n > state_batch",
                   "L2H_FLAG_TAPS", "neither read nor written", "frames == 1"):
        assert phrase in doc, phrase
    assert "#define L2H_ABI_VERSION 1" in hdr
