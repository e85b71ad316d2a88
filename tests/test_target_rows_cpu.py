"""Host-side checks of calls over per-listener lists of target rows (l2h_sep_forward_targets_rows,
Net.advance_target_rows): the argument errors the C call returns before it touches the device, the Python ValueErrors, the
header's description and the exported symbol (no GPU needed; the handle below never commits weights)."""
import ctypes

import pytest
import torch

import serving_util as su
from serving_util import FAKE_DEV, L2H_FLAG_TAPS, eng  # noqa: F401

LISTS = ctypes.c_void_p(0x30000)


def _call(L, h, state_batch, n, rows, frames, records=LISTS, offsets=LISTS, hops=None, flags=0, p=FAKE_DEV, emb=FAKE_DEV,
          y=FAKE_DEV):
    return L.l2h_sep_forward_targets_rows(h, p, 1024, 512, 128 * max(frames, 1) + 64, emb, p, state_batch, records, offsets,
                                          hops, n, rows, frames, y, 1024, 512, 128 * max(frames, 1), p, 1 << 20, flags, None)


@pytest.mark.parametrize("hops", [None, ctypes.c_void_p(0x40000)], ids=["no-hops", "hops"])
def test_forward_targets_rows_argument_errors(eng, hops):
    _, h, L = eng
    assert _call(L, None, 8, 2, 4, 1, hops=hops) == 1                          # no handle
    assert b"null" in L.l2h_last_error()
    for kw in ({"records": None}, {"offsets": None}, {"p": None}, {"emb": None}, {"y": None}):
        assert _call(L, h, 8, 2, 4, 1, hops=hops, **kw) == 1, kw
        assert b"null" in L.l2h_last_error()
    for n, rows, frames in ((0, 4, 1), (-1, 4, 1), (2, 0, 1), (2, -3, 1), (2, 4, 0), (2, 4, -5)):
        assert _call(L, h, 8, n, rows, frames, hops=hops) == 1, (n, rows, frames)
        assert b"n_rows and frames > 0" in L.l2h_last_error()
    assert _call(L, h, 8, 2, 9, 1, hops=hops) == 1                             # 9 target rows, the state holds 8
    assert b"n_rows <= state_batch" in L.l2h_last_error()
    assert _call(L, h, 8, 5, 4, 1, hops=hops) == 1                             # more listeners than target rows
    assert b"n <= n_rows" in L.l2h_last_error()
    assert _call(L, h, 1 << 24, 1, 1 << 22, 1 << 3, hops=hops) == 1           # n_rows * frames * 97 rows past the limit
    assert b"too large" in L.l2h_last_error()
    assert _call(L, h, 1 << 16, 64, 1 << 15, 500, hops=hops) == 1             # (a product that also fits in 32 bits)
    assert b"too large" in L.l2h_last_error()
    assert _call(L, h, 8, 2, 4, 1, hops=hops, flags=L2H_FLAG_TAPS) == 1        # the taps belong to the dense chain
    assert b"L2H_FLAG_TAPS" in L.l2h_last_error()


def test_python_advance_target_rows_raise_value_error(eng):
    net, _, _ = eng
    st = su.host_state(net, 8)
    x = torch.zeros(2, 2, 128 * 3 + 64)                                           # n = 2 listeners, T = 3
    emb = torch.zeros(3, 256)                                                     # R = 3 target rows
    good = ([4, 1, 6], [0, 2, 3])
    for bad in (torch.zeros(3, 128), torch.zeros(3, 1, 256), torch.zeros(1, 256), torch.zeros(9, 256),
                [[0.0] * 256] * 3):                                               # embeds not [R, 256] with n <= R <= 8
        with pytest.raises(ValueError):
            net.advance_target_rows(x, bad, st, *good)
    for n_samples in (200, 128 * 3, 64):                                          # not 128*T + 64 samples
        with pytest.raises(ValueError):
            net.advance_target_rows(torch.zeros(2, 2, n_samples), emb, st, *good)
    with pytest.raises(ValueError):                                               # x not [n, M, N]
        net.advance_target_rows(torch.zeros(2, 128 * 3 + 64), emb, st, *good)
    for bad in ([4, 1], [4, 1, 6, 7], [4, 4, 6], [4, 1, 8], [-1, 1, 6], [4.0, 1.0, 6.0], [True, False, True],
                [[4, 1, 6]], torch.tensor([4, 1, 6], dtype=torch.float32)):
        with pytest.raises(ValueError):                                           # records: count, duplicate, range, type
            net.advance_target_rows(x, emb, st, bad, good[1])
    for bad in ([0, 2], [0, 2, 3, 3], [1, 2, 3], [0, 2, 1], [0, 2, 4], [0, -1, 3], [0.0, 2.0, 3.0], [[0, 2, 3]],
                torch.tensor([0, 3, 2])):
        with pytest.raises(ValueError):                                           # offsets: count, start, order, range, type
            net.advance_target_rows(x, emb, st, good[0], bad)
    for bad in ([1], [1, 2, 3], [0, 4], [-1, 2], [1.0, 2.0], torch.tensor([0, 4])):
        with pytest.raises(ValueError):                                           # hops outside [0, T] or the wrong count
            net.advance_target_rows(x, emb, st, *good, hops=bad)
    for records, offsets, hops in ((good[0], good[1], None), ([7, 0, 3], [0, 0, 3], [0, 3]),
                                   (torch.tensor([2, 5, 1]), torch.tensor([0, 1, 1]), torch.tensor([2, 2]))):
        with pytest.raises(RuntimeError):                                         # checked, then refused: no CPU fallback
            net.advance_target_rows(x, emb, st, records, offsets, hops=hops)


def test_header_documents_forward_targets_rows():
    hdr = su.header()
    decl, args = su.declaration(hdr, "l2h_sep_forward_targets_rows")
    assert decl, "l2h_sep_forward_targets_rows is not declared"
    assert args == ["handle", "x_dev", "x_batch_stride", "x_ch_stride", "x_len", "emb_dev", "state_dev", "state_batch",
                    "records_dev", "offsets_dev", "hops_dev", "n", "n_rows", "frames", "y_dev", "y_batch_stride",
                    "y_ch_stride", "y_len", "workspace_dev", "workspace_bytes", "flags", "stream"]
    prev, _ = su.declaration(hdr, "l2h_sep_forward_targets_groups")
    assert prev and prev.start() < decl.start(), "declared after l2h_sep_forward_targets_groups"
    doc = su.doc_before(hdr, decl.start())
    for phrase in ("records_dev", "offsets_dev", "hops_dev", "lead record", "records_dev[offsets_dev[i]]",
                   "outside [0, state_batch)", "store nothing", "clamped on the device", "non-decreasing and <= R",
                   "NULL", "128*h + 63", "128*h - 1", "h = 0 stores nothing", "l2h_sep_state_reset_streams",
                   "l2h_sep_workspace_bytes(handle, n_rows, frames, flags)", "(n, R, T)", "L2H_FLAG_GRAPH", "L2H_FLAG_TAPS",
                   "n > n_rows", "n_rows > state_batch"):
        assert phrase in doc, phrase
    assert "l2h_sep_forward_targets_rows" in hdr[:hdr.index('extern "C"')], "missing from the header's call map"
    assert "#define L2H_ABI_VERSION 1" in hdr


def test_forward_targets_rows_is_exported(eng):
    _, _, L = eng
    assert hasattr(L, "l2h_sep_forward_targets_rows")
    fn = L.l2h_sep_forward_targets_rows
    assert fn.restype is ctypes.c_int and len(fn.argtypes) == 22
