"""Host-side checks of ragged multi-hop calls over a list of a state's records (l2h_sep_forward_slots_hops,
Net.advance_slots(hops=)): the argument errors the C call returns before it touches the device, the header's description,
and the Python ValueErrors for `hops` (no GPU needed; the handle below never commits weights)."""
import ctypes
import re

import pytest
import torch

import serving_util as su
from serving_util import FAKE_DEV, L2H_FLAG_TAPS, eng  # noqa: F401


def _call(L, h, state_batch, slots, hops, n, frames, flags=0, p=FAKE_DEV):
    return L.l2h_sep_forward_slots_hops(h, p, 1024, 512, 128 * frames + 64, p, p, state_batch, slots, hops, n, frames, p,
                                        1024, 512, 128 * frames, p, 1 << 20, flags, None)


@pytest.mark.parametrize("hops", [None, ctypes.c_void_p(0x40000)], ids=["no-hops", "hops"])
def test_forward_slots_hops_argument_errors(eng, hops):
    """the errors of l2h_sep_forward_slots_frames, with or without a hop list (NULL hops: every row all frames)"""
    _, h, L = eng
    sl = ctypes.c_void_p(0x30000)
    assert _call(L, h, 4, None, hops, 2, 3) == 1                   # no slot list
    assert b"null" in L.l2h_last_error()
    assert _call(L, None, 4, sl, hops, 2, 3) == 1                  # no handle
    assert _call(L, h, 4, sl, hops, 2, 3, p=None) == 1             # null buffers
    for n in (0, -3):                                              # no rows
        assert _call(L, h, 4, sl, hops, n, 3) == 1
    assert _call(L, h, 4, sl, hops, 5, 3) == 1                     # more rows than records
    assert b"n <= state_batch" in L.l2h_last_error()
    assert _call(L, h, 0, sl, hops, 1, 3) == 1                     # an empty state
    for frames in (0, -1, -128):
        assert _call(L, h, 4, sl, hops, 2, frames) == 1
        assert b"frames > 0" in L.l2h_last_error()
    assert _call(L, h, 4, sl, hops, 2, 3, flags=L2H_FLAG_TAPS) == 1
    assert b"L2H_FLAG_TAPS" in L.l2h_last_error()


def test_header_documents_forward_slots_hops():
    hdr = su.header()
    decl, args = su.declaration(hdr, "l2h_sep_forward_slots_hops")
    assert decl, "l2h_sep_forward_slots_hops is not declared"
    assert args == ["handle", "x_dev", "x_batch_stride", "x_ch_stride", "x_len", "emb_dev", "state_dev", "state_batch",
                    "slots_dev", "hops_dev", "n", "frames", "y_dev", "y_batch_stride", "y_ch_stride", "y_len",
                    "workspace_dev", "workspace_bytes", "flags", "stream"]
    prev = re.search(r"int l2h_sep_forward_slots_frames\(", hdr)
    assert prev and prev.start() < decl.start(), "declared after l2h_sep_forward_slots_frames"
    doc = su.doc_before(hdr, decl.start())
    for phrase in ("hops_dev", "[0, frames]", "128*h + 64", "L2H_FLAG_GRAPH", "NULL", "128*h - 1", "h = 0 stores nothing",
                   "l2h_sep_forward_slots_frames"):
        assert phrase in doc, phrase
    # the multi-hop call's description points at the ragged call for listeners with different backlogs
    frames_doc = su.doc_before(hdr, prev.start())
    assert "l2h_sep_forward_slots_hops" in frames_doc
    assert "#define L2H_ABI_VERSION 1" in hdr


def test_python_hops_raise_value_error(eng):
    net, _, _ = eng
    st = su.host_state(net, 4)
    emb = torch.zeros(2, 256)
    x = torch.zeros(2, 2, 128 * 3 + 64)                               # T = 3
    for bad in ([1], [1, 2, 3], [], [[1, 2]], [0, 4], [-1, 2], [3, 7], [1.0, 2.0], [True, False],
                torch.tensor([1, 2], dtype=torch.float32), torch.tensor([[1, 2]]), torch.tensor([0, 4])):
        with pytest.raises(ValueError):
            net.advance_slots(x, emb, st, [0, 1], hops=bad)
    for ok in ([0, 3], (1, 2), torch.tensor([3, 0]), torch.tensor([2, 2], dtype=torch.int64)):
        with pytest.raises(RuntimeError):                              # checked, then refused: no CPU fallback
            net.advance_slots(x, emb, st, [0, 1], hops=ok)
