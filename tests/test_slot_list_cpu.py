"""Host-side checks of one-hop calls over a list of a state's records (l2h_sep_forward_slots, Net.predict(slots=)): the
argument errors the C call returns before it touches the device, the Python ValueErrors, and the header's description
(no GPU needed; the handle below never commits weights)."""
import ctypes

import pytest
import torch

import serving_util as su
from serving_util import FAKE_DEV, L2H_FLAG_TAPS, eng  # noqa: F401


def _call(L, h, state_batch, slots, n, flags=0, p=FAKE_DEV):
    return L.l2h_sep_forward_slots(h, p, 384, 192, 192, p, p, state_batch, slots, n, p, 256, 128, 128, p, 1 << 20, flags,
                                   None)


def test_forward_slots_argument_errors(eng):
    _, h, L = eng
    sl = ctypes.c_void_p(0x30000)
    assert _call(L, h, 4, None, 2) == 1                      # no slot list
    assert b"null" in L.l2h_last_error()
    assert _call(L, None, 4, sl, 2) == 1                     # no handle
    assert _call(L, h, 4, sl, 2, p=None) == 1                # null buffers
    assert _call(L, h, 4, sl, 0) == 1                        # no rows
    assert _call(L, h, 4, sl, -3) == 1
    assert _call(L, h, 4, sl, 5) == 1                        # more rows than records
    assert b"n <= state_batch" in L.l2h_last_error()
    assert _call(L, h, 0, sl, 1) == 1                        # an empty state
    assert _call(L, h, -2, sl, 1) == 1
    assert _call(L, h, 4, sl, 2, flags=L2H_FLAG_TAPS) == 1   # the taps belong to the dense chain
    assert b"L2H_FLAG_TAPS" in L.l2h_last_error()


def test_python_slot_lists_raise_value_error(eng):
    net, _, _ = eng
    cpu = torch.device("cpu")
    for bad in ([0, 0, 1], [0, 1, 4], [-1, 0, 1], [0, 1], [0, 1, 2, 3], [[0, 1, 2]], [0.0, 1.0, 2.0],
                torch.tensor([True, False, True])):
        with pytest.raises(ValueError):
            net._slot_list(bad, cpu, 3, 4)
    got = net._slot_list(torch.tensor([3, 0, 2]), cpu, 3, 4)
    assert got.dtype == torch.int32 and got.tolist() == [3, 0, 2]
    assert net._slot_list((1, 2, 0), cpu, 3, 4).tolist() == [1, 2, 0]
    st = su.host_state(net, 4)
    one_hop, two_hops = torch.zeros(2, 2, 192), torch.zeros(2, 2, 320)
    emb = torch.zeros(2, 256)
    with pytest.raises(ValueError):          # a list needs a one-hop call
        net.predict(two_hops, emb, st, pad=False, slots=[0, 1])
    with pytest.raises(ValueError):          # a list and a mask
        net.predict(one_hop, emb, st, pad=False, slots=[0, 1], active=torch.ones(2, dtype=torch.bool))


def test_header_documents_forward_slots():
    hdr = su.header()
    decl, args = su.declaration(hdr, "l2h_sep_forward_slots")
    assert decl, "l2h_sep_forward_slots is not declared"
    assert args == ["handle", "x_dev", "x_batch_stride", "x_ch_stride", "x_len", "emb_dev", "state_dev", "state_batch",
                    "slots_dev", "n", "y_dev", "y_batch_stride", "y_ch_stride", "y_len", "workspace_dev", "workspace_bytes",
                    "flags", "stream"]
    doc = su.doc_before(hdr, decl.start())
    for phrase in ("slots_dev[i]", "l2h_sep_workspace_bytes(handle, n, 1, flags)", "outside [0, state_batch)",
                   "L2H_FLAG_GRAPH", "n > state_batch", "L2H_FLAG_TAPS", "neither read nor written"):
        assert phrase in doc, phrase
    assert "#define L2H_ABI_VERSION 1" in hdr
