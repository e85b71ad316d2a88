"""Host-side checks of calls over a list of a targets state's groups (l2h_sep_forward_targets_groups,
Net.advance_targets): the argument errors the C call returns before it touches the device, the Python ValueErrors and the
header's description (no GPU needed; the handle below never commits weights)."""
import ctypes
import re

import pytest
import torch

import serving_util as su
from serving_util import FAKE_DEV, L2H_FLAG_TAPS, eng  # noqa: F401


def _call(L, h, state_batch, n, k, frames, groups=ctypes.c_void_p(0x30000), hops=None, flags=0, p=FAKE_DEV, emb=FAKE_DEV,
          y=FAKE_DEV):
    return L.l2h_sep_forward_targets_groups(h, p, 1024, 512, 128 * max(frames, 1) + 64, emb, p, state_batch, groups, hops, n,
                                            k, frames, y, 1024, 512, 128 * max(frames, 1), p, 1 << 20, flags, None)


@pytest.mark.parametrize("hops", [None, ctypes.c_void_p(0x40000)], ids=["no-hops", "hops"])
def test_forward_targets_groups_argument_errors(eng, hops):
    _, h, L = eng
    assert _call(L, None, 8, 2, 2, 1, hops=hops) == 1                      # no handle
    assert b"null" in L.l2h_last_error()
    for kw in ({"groups": None}, {"p": None}, {"emb": None}, {"y": None}):  # no group list / x, state, workspace / emb / y
        assert _call(L, h, 8, 2, 2, 1, hops=hops, **kw) == 1, kw
        assert b"null" in L.l2h_last_error()
    for n, k, frames in ((0, 2, 1), (-1, 2, 1), (2, 0, 1), (2, -3, 1), (2, 2, 0), (2, 2, -5)):
        assert _call(L, h, 8, n, k, frames, hops=hops) == 1, (n, k, frames)
        assert b"n_targets" in L.l2h_last_error()
    for state_batch, k in ((0, 2), (-4, 2), (7, 2), (8, 3), (5, 4)):         # not a positive multiple of K
        assert _call(L, h, state_batch, 1, k, 1, hops=hops) == 1, (state_batch, k)
        assert b"groups of n_targets" in L.l2h_last_error()
    assert _call(L, h, 8, 5, 2, 1, hops=hops) == 1                         # 5 groups listed, the state holds 4
    assert b"n <= state_batch / n_targets" in L.l2h_last_error()
    assert _call(L, h, 1 << 22, 1 << 12, 1 << 10, 1 << 10, hops=hops) == 1  # n * K * frames * 97 rows past the limit
    assert b"too large" in L.l2h_last_error()
    assert _call(L, h, 1 << 16, 1024, 64, 500, hops=hops) == 1             # (a product that also fits in 32 bits)
    assert b"too large" in L.l2h_last_error()
    assert _call(L, h, 8, 2, 2, 1, hops=hops, flags=L2H_FLAG_TAPS) == 1     # the taps belong to the dense chain
    assert b"L2H_FLAG_TAPS" in L.l2h_last_error()


def test_python_advance_targets_raise_value_error(eng):
    net, _, _ = eng
    st = su.host_state(net, 8)                                                    # G = 4 groups of K = 2
    x = torch.zeros(2, 2, 128 * 3 + 64)                                           # n = 2, T = 3
    emb = torch.zeros(2, 2, 256)
    for bad in (torch.zeros(2, 256), torch.zeros(2, 2, 128), torch.zeros(3, 2, 256), torch.zeros(2, 0, 256),
                torch.zeros(2, 2, 256, 1), [[[0.0] * 256] * 2] * 2):              # embeds not [n, K, 256]
        with pytest.raises(ValueError):
            net.advance_targets(x, bad, st, [0, 1])
    with pytest.raises(ValueError):                                               # 8 records are no groups of 3
        net.advance_targets(x, torch.zeros(2, 3, 256), st, [0, 1])
    for n_samples in (200, 128 * 3, 64):                                          # not 128*T + 64 samples
        with pytest.raises(ValueError):
            net.advance_targets(torch.zeros(2, 2, n_samples), emb, st, [0, 1])
    with pytest.raises(ValueError):                                               # x not [n, M, N]
        net.advance_targets(torch.zeros(2, 128 * 3 + 64), emb, st, [0, 1])
    for bad in ([0], [0, 1, 2], [], [1, 1], [0, 4], [-1, 2], [0.0, 1.0], [True, False], [[0, 1]],
                torch.tensor([0, 1], dtype=torch.float32), torch.tensor([3, 3])):
        with pytest.raises(ValueError):                                           # a wrong count, a duplicate, out of range
            net.advance_targets(x, emb, st, bad)
    for bad in ([1], [1, 2, 3], [0, 4], [-1, 2], [1.0, 2.0], torch.tensor([0, 4])):
        with pytest.raises(ValueError):                                           # hops outside [0, T] or the wrong count
            net.advance_targets(x, emb, st, [0, 1], hops=bad)
    for groups, hops in (([0, 3], None), ((2, 1), [0, 3]), (torch.tensor([3, 0]), torch.tensor([2, 2]))):
        with pytest.raises(RuntimeError):                                         # checked, then refused: no CPU fallback
            net.advance_targets(x, emb, st, groups, hops=hops)


def test_header_documents_forward_targets_groups():
    hdr = su.header()
    decl, args = su.declaration(hdr, "l2h_sep_forward_targets_groups")
    assert decl, "l2h_sep_forward_targets_groups is not declared"
    assert args == ["handle", "x_dev", "x_batch_stride", "x_ch_stride", "x_len", "emb_dev", "state_dev", "state_batch",
                    "groups_dev", "hops_dev", "n", "n_targets", "frames", "y_dev", "y_batch_stride", "y_ch_stride", "y_len",
                    "workspace_dev", "workspace_bytes", "flags", "stream"]
    prev = re.search(r"int l2h_sep_forward_targets\(", hdr)
    assert prev and prev.start() < decl.start(), "declared after l2h_sep_forward_targets"
    doc = su.doc_before(hdr, decl.start())
    for phrase in ("g*K + k", "lead record", "groups_dev", "outside [0, G)", "hops_dev", "NULL", "128*h + 63", "128*h - 1",
                   "h = 0 stores nothing", "outside [0, frames] counts as 0", "l2h_sep_workspace_bytes(handle, n*K, frames, flags)",
                   "(n, K, T)", "L2H_FLAG_GRAPH", "L2H_FLAG_TAPS", "n_targets == 1 is l2h_sep_forward_slots_hops"):
        assert phrase in doc, phrase
    # the targets call's description points at this one for slot lists and hop counts
    targets_doc = su.doc_before(hdr, prev.start())
    assert "l2h_sep_forward_targets_groups" in targets_doc
    assert "#define L2H_ABI_VERSION 1" in hdr
