"""The scaffold of the kernel-level GPU tests (kernels/scaffold.py), on the CPU: guarded buffers see a write into either
guard, ratio's exact and empty cases, the ledger's two failures, and where the views of a state's records land."""
import math

import pytest
import torch

from kernels import harness as kh
from kernels.scaffold import GUARD, SENSITIVITY, Guarded, Ledger, Records, bits, is_sentinel, ratio

CPU = torch.device("cpu")


def test_guarded_buffer_reports_a_write_into_either_guard():
    assert GUARD % 128 == 0
    for i in (GUARD - 1, 0, -GUARD, -1):                          # the front guard's ends, the back guard's ends
        g = Guarded((3, 5), CPU)
        assert g.ok() and is_sentinel(g.t) and g.whole.numel() == 15 + 2 * GUARD
        g.t.fill_(1.0)                                            # the buffer itself is free to write
        assert g.ok()
        g.whole[i] = 0.0
        assert not g.ok(), i


def test_guarded_buffer_initial_values():
    init = torch.arange(6.0).view(2, 3)
    g = Guarded((2, 3), CPU, init)
    assert torch.equal(g.t, init) and g.ok()
    assert torch.equal(Guarded((6,), CPU, init.numpy()).t, init.view(6))


def test_ratio_exact_and_empty():
    z = torch.zeros(3)
    assert ratio(z, z.double(), torch.zeros(3)) == 0.0                       # 0 / 0: exact
    assert ratio(torch.tensor([1.0, 0.0]), torch.zeros(2), torch.zeros(2)) == math.inf
    assert ratio(torch.zeros(0), torch.zeros(0), torch.zeros(0)) == 0.0
    assert ratio(torch.tensor([1.5, 3.0]), torch.tensor([1.0, 2.0]), torch.tensor([1.0, 4.0])) == 0.5
    assert math.isnan(ratio(torch.tensor([float("nan")]), torch.zeros(1), torch.ones(1)))


def test_ledger_checks_errors_and_mutants():
    led = Ledger()
    led.check("k", 0.5, {"m": SENSITIVITY})
    led.check("k", {"X": 0.25, "h": 0.75}, {"m": 2 * SENSITIVITY})
    assert led.worst == {"k": 0.75} and led.margin == {"k": SENSITIVITY}
    with pytest.raises(AssertionError):
        led.check("k", {"X": 0.25, "h": 1.01}, {})
    with pytest.raises(AssertionError):
        led.check("k", 0.5, {"m": 0.99 * SENSITIVITY})
    with pytest.raises(AssertionError):
        led.check("k", math.nan, {})


# a small hand-written layout: a header of 8 floats; a record of the clock (floats 2, 3), calls, the weight generation,
# the embedding, gate and tails back to back, then one block of (h, c) and the K and V rings at the kernels' own sizes
# (kh.Ring checks them)
RING_K, RING_V = kh.NHEAD * kh.RING * kh.QK_LD, kh.NHEAD * kh.RING * kh.V_DIM
LAY = dict(HEADER_BYTES=32, ST_POS=2, ST_CALLS=4, ST_GEN=5, ST_EMB=6, ST_GATE=6 + kh.SPK, ST_CONV=6 + kh.SPK + kh.FC,
           ST_DECONV=8100, ST_ISTFT=8100 + 4 * kh.FC, ST_BLK=40000, BK_H=0, BK_C=kh.FC, BK_K=2 * kh.FC,
           BK_V=2 * kh.FC + RING_K, BK_STRIDE=2 * kh.FC + RING_K + RING_V, RING=kh.RING, ATT=kh.ATT, QK_LD=kh.QK_LD,
           V_DIM=kh.V_DIM)
LAY["STREAM_STRIDE"] = LAY["ST_BLK"] + LAY["BK_STRIDE"]


def test_records_views_land_at_the_layout_offsets():
    st = Records(LAY, 3, CPU, gap=6)
    assert st.hdr == 8 and st.ss == LAY["STREAM_STRIDE"] + 6 and st.t.numel() == 8 + 3 * st.ss
    assert is_sentinel(st.t) and st.buf.ok()
    st.t.copy_(torch.arange(st.t.numel(), dtype=torch.float32))   # every float holds its own offset (< 2^24: exact)
    b, rec = 2, 8 + 2 * st.ss
    at = lambda v: int(v.reshape(-1)[0])
    assert at(st.rec(b)) == rec and st.rec(b).numel() == st.ss
    assert at(st.gate(b)) == rec + LAY["ST_GATE"] and st.gate(b).shape == (kh.NF, kh.CH)
    assert at(st.emb(b)) == rec + LAY["ST_EMB"] and st.emb(b).shape == (kh.SPK,)
    assert at(st.conv(b)) == rec + LAY["ST_CONV"] and st.conv(b).shape == (2, 2, 4, kh.NF)
    assert at(st.deconv(b)) == rec + LAY["ST_DECONV"] and st.deconv(b).shape == (2, 2, kh.NF, kh.CH)
    assert at(st.istft(b)) == rec + LAY["ST_ISTFT"] and st.istft(b).shape == (2, 2, kh.NROW)
    assert at(st.field(b, 77, (2,))) == rec + 77
    assert at(st.hc(b, 0, "h")) == rec + 40000 and at(st.hc(b, 0, "c")) == rec + 40000 + kh.FC
    k, v = st.ring(b, 0, "k"), st.ring(b, 0, "v")
    assert k.shape == (kh.NHEAD, kh.RING, kh.QK_LD) and v.shape == (kh.NHEAD, kh.RING, kh.V_DIM)
    ring = kh.Ring(LAY)
    for h, n in ((0, 0), (3, -1), (2, 123)):
        assert at(k[h, ring.slot(n)]) == rec + ring.row(0, "k", h, n)
        assert at(v[h, ring.slot(n)]) == rec + ring.row(0, "v", h, n)
    # index() gives the flat offsets of any view, strided ones too
    for view in (st.gate(b), k[:, 5], v[1:3, 7, 100:200], st.conv(b)[1]):
        assert torch.equal(st.index(view), view.reshape(-1).long())
    # the int views: the clock (int64 over floats 2, 3), calls and the weight generation
    st.pos(1).fill_(2 ** 40 + 3)
    st.calls(1).fill_(-7)
    st.gen(1).fill_(5)
    r1 = bits(st.rec(1))
    assert int(r1[2]) == 3 and int(r1[3]) == 2 ** 8 and int(r1[4]) == -7 and int(r1[5]) == 5
    assert int(st.pos(1)) == 2 ** 40 + 3 and int(st.calls(1)) == -7 and int(st.gen(1)) == 5


def test_records_same_outside():
    st = Records(LAY, 2, CPU)
    before = st.snapshot()
    assert st.same_outside(st.index(), before)
    st.gate(1)[3, 4] = 1.0
    assert not st.same_outside(st.index(), before)
    assert st.same_outside(st.index(st.gate(1)), before)
    assert not st.same_outside(st.index(st.gate(0)), before)
    exp = before.clone()
    st.gate(1, exp)[3, 4] = 1.0                                   # a view of a snapshot
    assert st.same_outside(st.index(), exp)
    st.buf.whole[0] = 0.0                                         # a write before the state
    assert not st.same_outside(st.index(st.gate(1)), before)
