"""Host-side checks of adding and dropping the targets of a running listener (l2h_sep_forward_targets_rows_history,
l2h_sep_join_targets, l2h_sep_state_move_lead; Net.target_history, Net.join_targets, SepState.move_lead): the argument
errors the C calls return before they touch the device, the Python checks, the header and the exported symbols (no GPU
needed; the handle below never commits weights)."""
import ctypes

import pytest
import torch

import serving_util as su
from serving_util import FAKE_DEV, L2H_FLAG_TAPS, eng  # noqa: F401

from lookoncetohear_b200 import TargetHistory

LISTS = ctypes.c_void_p(0x30000)
HIST = ctypes.c_void_p(0x50000)


def _rows(L, h, hist=HIST, hist_frames=64, n=2, rows=4, frames=1, records=LISTS, p=FAKE_DEV):
    return L.l2h_sep_forward_targets_rows_history(h, p, 1024, 512, 128 * frames + 64, p, p, 8, records, LISTS, None, n, rows,
                                                  frames, p, 1024, 512, 128 * frames, p, 1 << 20, 0, None, hist, hist_frames)


def _join(L, h, J=2, batch=8, hist=HIST, hist_frames=64, frames=16, records=LISTS, leads=LISTS, emb=FAKE_DEV, state=FAKE_DEV,
          y=FAKE_DEV, ws=FAKE_DEV, flags=0):
    return L.l2h_sep_join_targets(h, records, leads, emb, J, state, batch, hist, hist_frames, frames, y, 1024, 512, None, ws,
                                  1 << 20, flags, None)


def _slots(v):
    return (ctypes.c_int32 * len(v))(*v)


def _move(L, h, old, new, batch=8, n=None, state=FAKE_DEV):
    return L.l2h_sep_state_move_lead(h, state, batch, _slots(old), _slots(new), len(old) if n is None else n, None)


def test_rows_history_argument_errors(eng):
    _, h, L = eng
    assert _rows(L, None) == 1 and b"null" in L.l2h_last_error()
    for kw in ({"hist": None}, {"records": None}, {"p": None}):
        assert _rows(L, h, **kw) == 1, kw
        assert b"null" in L.l2h_last_error()
    for hf in (0, -3):
        assert _rows(L, h, hist_frames=hf) == 1
        assert b"hist_frames >= 1" in L.l2h_last_error()
    for n, rows in ((0, 4), (-1, 4), (2, 0)):                 # the checks of l2h_sep_forward_targets_rows come back too
        assert _rows(L, h, n=n, rows=rows) == 1
        assert b"n_rows and frames > 0" in L.l2h_last_error()


def test_join_argument_errors(eng):
    _, h, L = eng
    assert _join(L, None) == 1 and b"null" in L.l2h_last_error()
    for kw in ({"records": None}, {"leads": None}, {"emb": None}, {"state": None}, {"ws": None}):
        assert _join(L, h, **kw) == 1, kw
        assert b"null" in L.l2h_last_error()
    assert _join(L, h, y=None) == 1 and b"y_dev" in L.l2h_last_error()       # frames are replayed: y is needed
    for J in (0, -2, 9):
        assert _join(L, h, J=J) == 1, J
        assert b"0 < J <= state_batch" in L.l2h_last_error()
    assert _join(L, h, frames=-1) == 1 and b"frames >= 0" in L.l2h_last_error()
    for hf in (0, -1):
        assert _join(L, h, hist_frames=hf) == 1
        assert b"hist_frames >= 1" in L.l2h_last_error()
    assert _join(L, h, J=1 << 16, batch=1 << 20, frames=1 << 12, hist_frames=1 << 12) == 1
    assert b"too large" in L.l2h_last_error()
    assert _join(L, h, flags=L2H_FLAG_TAPS) == 1 and b"L2H_FLAG_TAPS" in L.l2h_last_error()


def test_move_lead_argument_errors(eng):
    _, h, L = eng
    assert _move(L, None, [0], [1]) == 1 and b"null" in L.l2h_last_error()
    assert _move(L, h, [0], [1], state=None) == 1 and b"null" in L.l2h_last_error()
    assert L.l2h_sep_state_move_lead(h, FAKE_DEV, 8, None, _slots([1]), 1, None) == 1
    for batch, n in ((0, 1), (8, 0), (8, -1)):
        assert _move(L, h, [0], [1], batch=batch, n=n) == 1, (batch, n)
        assert b"must be positive" in L.l2h_last_error()
    assert _move(L, h, [0, 8], [1, 2]) == 1 and b"outside [0, 8)" in L.l2h_last_error()
    assert _move(L, h, [0, 3], [1, -1]) == 1 and b"outside [0, 8)" in L.l2h_last_error()
    assert _move(L, h, [0, 0], [1, 2]) == 1 and b"listed twice" in L.l2h_last_error()
    assert _move(L, h, [0, 1], [1, 2]) == 1 and b"both an old and a new lead" in L.l2h_last_error()


def test_python_join_and_history_checks(eng):
    net, _, _ = eng
    st = su.host_state(net, 8)
    other = su.host_state(net, 8)
    hist = TargetHistory(st, 4)
    assert tuple(hist.buf.shape) == (8, 4, 97 * 64) and hist.frames == 4
    for frames in (0, -1, 2.0, True):
        with pytest.raises(ValueError):
            net.target_history(st, frames)
    with pytest.raises(TypeError):
        net.target_history(hist, 4)
    e = torch.zeros(2, 256)
    for records, leads in (([3, 0], [0, 5]),                  # a joining record is a listed lead
                           ([3, 3], [0, 0]),                  # a record listed twice
                           ([3, 8], [0, 0]),                  # a record outside the state
                           ([3, -1], [0, 0]),
                           ([3, 4], [0, 8]),                  # a lead outside the state
                           ([3], [0, 0]), ([3, 4], [0])):     # wrong counts
        with pytest.raises(ValueError):
            net.join_targets(st, records, leads, e, history=hist)
    with pytest.raises(ValueError):                           # a history of another state
        net.join_targets(st, [3, 4], [0, 0], e, history=TargetHistory(other, 4))
    bent = TargetHistory(st, 4)
    bent.buf = torch.zeros(8, 5, 97 * 64)                     # a history of the wrong shape
    with pytest.raises(ValueError):
        net.join_targets(st, [3, 4], [0, 0], e, history=bent)
    with pytest.raises(TypeError):
        net.join_targets(st, [3, 4], [0, 0], e, history=torch.zeros(8, 4, 97 * 64))
    for bad in (torch.zeros(2, 128), torch.zeros(9, 256), torch.zeros(2, 1, 256)):
        with pytest.raises(ValueError):
            net.join_targets(st, [3, 4], [0, 0], bad, history=hist)
    for frames in (-1, 1.5):
        with pytest.raises(ValueError):
            net.join_targets(st, [3, 4], [0, 0], e, history=hist, frames=frames)
    for out in (torch.zeros(2, 2, 128 * 4, dtype=torch.float64), torch.zeros(2, 2, 100), torch.zeros(3, 2, 128 * 4)):
        with pytest.raises(ValueError):                       # out: dtype, too short, wrong rows
            net.join_targets(st, [3, 4], [0, 0], e, history=hist, out=out)
    with pytest.raises(RuntimeError):                         # checked, then refused: no CPU fallback
        net.join_targets(st, [3, 4], [0, 0], e, history=hist)
    x = torch.zeros(2, 2, 128 + 64)
    with pytest.raises(ValueError):                           # advance_target_rows with another state's history
        net.advance_target_rows(x, torch.zeros(3, 256), st, [4, 1, 6], [0, 2, 3], history=TargetHistory(other, 4))
    with pytest.raises(TypeError):
        net.advance_target_rows(x, torch.zeros(3, 256), st, [4, 1, 6], [0, 2, 3], history=hist.buf)


def test_history_reset_and_move_on_host(eng):
    net, _, _ = eng
    st = su.host_state(net, 4)
    hist = TargetHistory(st, 3)
    hist.buf.copy_(torch.arange(hist.buf.numel(), dtype=torch.float32).view_as(hist.buf))
    ref = hist.buf.clone()
    hist.move([1, 2], [3, 0])
    assert torch.equal(hist.buf[3], ref[1]) and torch.equal(hist.buf[0], ref[2]) and torch.equal(hist.buf[1], ref[1])
    hist.reset([1])
    assert not hist.buf[1].any() and torch.equal(hist.buf[2], ref[2])
    with pytest.raises(ValueError):
        hist.move([1], [2, 3])


def test_header_documents_the_calls():
    hdr = su.header()
    for name, args in (
            ("l2h_sep_forward_targets_rows_history",
             ["handle", "x_dev", "x_batch_stride", "x_ch_stride", "x_len", "emb_dev", "state_dev", "state_batch", "records_dev",
              "offsets_dev", "hops_dev", "n", "n_rows", "frames", "y_dev", "y_batch_stride", "y_ch_stride", "y_len",
              "workspace_dev", "workspace_bytes", "flags", "stream", "hist_dev", "hist_frames"]),
            ("l2h_sep_join_targets",
             ["handle", "records_dev", "leads_dev", "emb_dev", "J", "state_dev", "state_batch", "hist_dev", "hist_frames",
              "frames", "y_dev", "y_batch_stride", "y_ch_stride", "used_dev", "workspace_dev", "workspace_bytes", "flags",
              "stream"]),
            ("l2h_sep_state_move_lead", ["handle", "state_dev", "batch", "old_host", "new_host", "n", "stream"])):
        decl, got = su.declaration(hdr, name)
        assert decl, f"{name} is not declared"
        assert got == args, name
        assert name in hdr[:hdr.index('extern "C"')], f"{name} missing from the header's call map"
    doc = su.doc_before(hdr, su.declaration(hdr, "l2h_sep_join_targets")[0].start())
    for phrase in ("min(frames, hist_frames, p)", "cold join", "128*W_j - 1", "used_dev", "outside [0, state_batch)",
                   "l2h_sep_workspace_bytes(handle, J, max(1, min(frames, hist_frames)), flags)", "L2H_FLAG_GRAPH"):
        assert phrase in doc, phrase
    assert "adding a record to a running listener is not supported" not in hdr


def test_symbols_are_exported(eng):
    _, _, L = eng
    for name, n in (("l2h_sep_forward_targets_rows_history", 24), ("l2h_sep_join_targets", 18), ("l2h_sep_state_move_lead", 7)):
        fn = getattr(L, name)
        assert fn.restype is ctypes.c_int and len(fn.argtypes) == n, name
