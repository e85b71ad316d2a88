"""Host-side checks of calls that extract several targets per mixture (l2h_sep_forward_targets, Net.predict_targets /
forward_targets): the argument errors the C call returns before it touches the device, the Python ValueErrors, and the
header's description (no GPU needed; the handle below never commits weights)."""

import pytest
import torch

import serving_util as su
from serving_util import FAKE_DEV, L2H_FLAG_TAPS, eng  # noqa: F401


def _call(L, h, batch, n_targets, frames, flags=0, p=FAKE_DEV, emb=FAKE_DEV, y=FAKE_DEV):
    return L.l2h_sep_forward_targets(h, p, 384, 192, 192, emb, p, y, 256, 128, 128, batch, n_targets, frames, p, 1 << 20,
                                     flags, None)


def test_forward_targets_argument_errors(eng):
    _, h, L = eng
    assert _call(L, None, 2, 2, 1) == 1                      # no handle
    assert b"null" in L.l2h_last_error()
    assert _call(L, h, 2, 2, 1, p=None) == 1                 # null x / state / workspace
    assert b"null" in L.l2h_last_error()
    assert _call(L, h, 2, 2, 1, emb=None) == 1               # no embeddings
    assert _call(L, h, 2, 2, 1, y=None) == 1                 # no output
    for batch, k, frames in ((0, 2, 1), (-1, 2, 1), (2, 0, 1), (2, -3, 1), (2, 2, 0), (2, 2, -5)):
        assert _call(L, h, batch, k, frames) == 1, (batch, k, frames)
        assert b"n_targets" in L.l2h_last_error()
    assert _call(L, h, 1 << 12, 1 << 10, 1 << 10) == 1       # batch * n_targets * frames * 97 rows past the limit
    assert b"too large" in L.l2h_last_error()
    assert _call(L, h, 1024, 64, 500) == 1                   # (a product that also fits in 32 bits)
    assert b"too large" in L.l2h_last_error()
    assert _call(L, h, 2, 2, 1, flags=L2H_FLAG_TAPS) == 1    # the taps belong to the dense chain
    assert b"L2H_FLAG_TAPS" in L.l2h_last_error()


def test_python_targets_raise_value_error(eng):
    net, _, _ = eng
    st6 = su.host_state(net, 6)
    x = torch.zeros(2, 2, 192)
    for bad in (torch.zeros(2, 256), torch.zeros(2, 3, 128), torch.zeros(3, 3, 256), torch.zeros(2, 0, 256),
                torch.zeros(2, 3, 256, 1), [[0.0] * 256] * 2):
        with pytest.raises(ValueError):
            net.predict_targets(x, bad, st6, pad=False)
        with pytest.raises(ValueError):
            net.forward_targets(x, bad)
    with pytest.raises(ValueError):                         # a state of 6 records for 2 mixtures x 2 targets
        net.predict_targets(x, torch.zeros(2, 2, 256), st6, pad=False)
    with pytest.raises(ValueError):                         # ... and for 3 mixtures x 3 targets
        net.predict_targets(torch.zeros(3, 2, 192), torch.zeros(3, 3, 256), st6, pad=False)
    with pytest.raises(ValueError):                         # pad=False with a length that is not 128*T + 64
        net.predict_targets(torch.zeros(2, 2, 200), torch.zeros(2, 3, 256), st6, pad=False)
    with pytest.raises(RuntimeError):                       # right shapes: the call then needs a CUDA device
        net.predict_targets(x, torch.zeros(2, 3, 256), st6, pad=False)


def test_header_documents_forward_targets():
    hdr = su.header()
    decl, args = su.declaration(hdr, "l2h_sep_forward_targets")
    assert decl, "l2h_sep_forward_targets is not declared"
    assert args == ["handle", "x_dev", "x_batch_stride", "x_ch_stride", "x_len", "emb_dev", "state_dev", "y_dev",
                    "y_batch_stride", "y_ch_stride", "y_len", "batch", "n_targets", "frames", "workspace_dev",
                    "workspace_bytes", "flags", "stream"]
    doc = su.doc_before(hdr, decl.start())
    for phrase in ("i*K + k", "l2h_sep_state_bytes(handle, batch*K)", "l2h_sep_workspace_bytes(handle, batch*K, frames, flags)",
                   "lead record", "not a standalone stream", "n_targets == 1 is l2h_sep_forward", "L2H_FLAG_GRAPH",
                   "L2H_FLAG_TAPS", "slot lists", "l2h_sep_stream_host", "no compact record"):
        assert phrase in doc, phrase
