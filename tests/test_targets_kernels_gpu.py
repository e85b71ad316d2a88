"""The several-target kernels (csrc/targets_kernels.cuh) and the slot-list helpers (csrc/sep_kernels.cuh) launched
directly through their engine launchers, every output against an exact or float64 reference.

target_lists_kernel (one 1024-thread CTA: a running-maximum scan of the offsets in 1024-entry passes with a carry, and a
binary search for each row's owner) runs on the problems of kernels/harness.py::target_lists_cases: n = 1, 31, 1023,
1024, 1025 and 2500 listeners over up to 4096 rows, offsets monotone, decreasing (also across the 1024-entry pass
boundaries), negative, above `rows` and with spare rows past offsets[n]; empty listeners; records -1, batch and
+-(2^31 - 1), one of them a listener's lead; groups outside [0, batch / K); hops absent or outside [0, T].  Every int of
the 5 rows + 1 list buffer must equal target_lists_ref exactly, and what the kernel must not write (rec_hops without
hops, start in groups mode, the lead and start entries past n, the guard) keeps the sentinel.
spk_gate_kernel (dense map, and the Records map with and without hops): a row whose memo key matches (same embedding,
same weight generation) writes nothing, neither its gate nor its spk_pre row; a changed generation, one changed
embedding element, a NaN key (a fresh record) or one NaN key element rebuilds it; a row that is out of range or
advances no frame writes nothing, and record 0, which such rows read, stays untouched.  The gate is compared with
harness.gate64 within its element-wise bound, spk_pre with W e + b within u sqrt(16) sum |terms|.
gate_fanout_kernel (dense owner r / K; a listed owner list with -1; apply_gate 0 and 1; T = 1 and 3) is compared bit for
bit with an fp32 multiply on the CPU.  gather_h_kernel and scatter_hc_kernel (1-3 blocks from b0 = 0 or 1, records
GAP floats apart, rows out of range or advancing no frame) are exact copies; inter_gate_mask_kernel and
inter_h_last_kernel are exact for T_b in {-1, 0, 1, T - 1, T, T + 1}, T in {1, 2, 5}.  The fused-projection tensor-core
recurrence with per-sequence step counts (LstmXArgs::steps, passes 1-3) must give, for a sequence of T_b steps, the
outputs of its first T_b steps and its final c bit-identical to a run of T_b steps, and c0 for T_b outside [1, L].

Every buffer is followed by guard floats holding the sentinel 0x7FC0DEAD, every float a kernel must not write holds it
too and must keep it bit for bit, and each state is compared whole with the one the launch must leave.  Mutants: the
scan without the carry between passes, the offsets unclamped, the owner search off by one (start < r), an unvalidated
lead (target_lists); the owner r % K and a gated row without owner (gate_fanout); the gate in (c, f) order and with
unbiased variance (spk_gate).  Each must miss the kernel: the list and fan-out mutants differ on the cases that name
them, the gate mutants by >= 10x the bound.
Measured on one NVIDIA H100 80GB HBM3 (700 W power limit): worst error / bound 0.21 (the gate) and 0.18 (spk_pre);
the smallest gate mutant error / bound is 14 (unbiased variance); every list and fan-out mutant differs from the
kernel on each case that names it, and every other output is bit-exact.  The file runs in about 4 s.
"""
import math

import pytest
import torch

from kernels import harness as kh
from lookoncetohear_b200.configs import TSH_PARAMS

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC0DEAD
SENSITIVITY = 10.0
GUARD = 1024
N_BLOCKS = 3
GAP = 132                   # floats between two records (a multiple of 4: the kernels read float4s)
GEN = 5
NF, CH, FC, SPK = kh.NF, kh.CH, kh.FC, kh.SPK
INT_MAX = kh.INT_MAX
WORST, MARGIN = {}, {}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    kh.lib()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def lay(dev):
    return kh.sep_layout(N_BLOCKS)


def sentinel(n, dev):
    return torch.full((n,), SENTINEL, dtype=torch.int32, device=dev).view(torch.float32)


def bits(t):
    return t.contiguous().view(torch.int32)


def guarded(shape, dev):
    """a sentinel buffer of `shape` followed by GUARD sentinel floats; returns (view, whole)"""
    n = math.prod(shape)
    whole = sentinel(n + GUARD, dev)
    return whole[:n].view(shape), whole


def guard_ok(whole):
    return bool((bits(whole[-GUARD:]) == SENTINEL).all())


def i32(v, dev):
    return torch.tensor(v, dtype=torch.int32, device=dev)


def ratio(got, ref, bound):
    d = (got.double().cpu() - ref).abs()
    return float((d / bound.clamp_min(1e-300)).max())


class State:
    """`batch` records of lay's layout, ss = STREAM_STRIDE + GAP floats apart, every float the sentinel"""

    def __init__(self, lay, batch, dev):
        self.lay, self.batch = lay, batch
        self.hdr, self.ss = lay["HEADER_BYTES"] // 4, lay["STREAM_STRIDE"] + GAP
        self.t = sentinel(self.hdr + batch * self.ss + GUARD, dev)

    def rec(self, k, t=None):
        t = self.t if t is None else t
        return t[self.hdr + k * self.ss:self.hdr + (k + 1) * self.ss]

    def field(self, k, off, n, t=None):
        return self.rec(k, t)[off:off + n]

    def gate(self, k, t=None):
        return self.field(k, self.lay["ST_GATE"], FC, t).view(NF, CH)

    def emb(self, k, t=None):
        return self.field(k, self.lay["ST_EMB"], SPK, t)

    def gen(self, k, t=None):
        return self.rec(k, t).view(torch.int32)[self.lay["ST_GEN"]:self.lay["ST_GEN"] + 1]

    def hc(self, k, blk, which, t=None):
        """block blk's carried h or c of record k, [97][64]"""
        o = self.lay["ST_BLK"] + blk * self.lay["BK_STRIDE"] + self.lay["BK_H" if which == "h" else "BK_C"]
        return self.field(k, o, FC, t).view(NF, CH)


def records(st, slots, hops, T, dev):
    """(Records map, the device lists it points to: keep them alive)"""
    s = i32(slots, dev)
    h = None if hops is None else i32(hops, dev)
    return kh.records_map(st.ss, s, st.batch, h, T), (s, h)


def stores(slots, hops, b, batch, T):
    """row b stores: its slot inside the state and a frame to advance (sep_kernels.cuh row_record)"""
    return 0 <= slots[b] < batch and kh.row_frames(hops, b, T) > 0


# ---- target_lists_kernel ---------------------------------------------------------------------------------------------
LIST_CASES = kh.target_lists_cases()


def lists_expected(ref, n, rows):
    """the 5 rows + 1 + GUARD ints the launch must leave: rec, rec_hops (or the sentinel), owner, lead [n], start [n + 1]
    (or the sentinel)"""
    out = [SENTINEL] * (5 * rows + 1 + GUARD)
    out[0:rows] = ref["rec"]
    if ref["rec_hops"] is not None:
        out[rows:2 * rows] = ref["rec_hops"]
    out[2 * rows:3 * rows] = ref["owner"]
    out[3 * rows:3 * rows + n] = ref["lead"]
    if ref["start"] is not None:
        out[4 * rows:4 * rows + n + 1] = ref["start"]
    return out


@pytest.mark.parametrize("case", LIST_CASES, ids=[c["name"] for c in LIST_CASES])
def test_target_lists(case, dev):
    c = case
    n, K, rows, batch = c["n"], c["K"], c["rows"], c["batch"]
    args = [None if c[k] is None else i32(c[k], dev) for k in ("records", "offsets", "groups", "hops")]
    lists = torch.full((5 * rows + 1 + GUARD,), SENTINEL, dtype=torch.int32, device=dev)
    assert kh.target_lists(*args, n, K, rows, batch, lists) == 0
    torch.cuda.synchronize()
    got = lists.cpu().tolist()
    ref = kh.target_lists_ref(c["records"], c["offsets"], c["groups"], c["hops"], n, K, rows, batch)
    exp = lists_expected(ref, n, rows)
    if got != exp:
        j = next(j for j in range(len(exp)) if got[j] != exp[j])
        names = ("rec", "rec_hops", "owner", "lead", "start")
        pytest.fail(f"{c['name']}: {names[min(j // rows, 4)]}[{j % rows}] = {got[j]}, expected {exp[j]}")
    for m in c["catches"]:
        mref = kh.target_lists_ref(c["records"], c["offsets"], c["groups"], c["hops"], n, K, rows, batch, mutant=m)
        assert got != lists_expected(mref, n, rows), (c["name"], m)
    print(f"[{c['name']}] exact; mutants missed: {sorted(c['catches'])}; rows that store {sum(r >= 0 for r in ref['rec'])}"
          f" / {rows}")


# ---- spk_gate_kernel -------------------------------------------------------------------------------------------------
class GateWeights:
    """the speaker projection of a seeded Net and a random gate LayerNorm, as test_front_back_kernels_gpu.py builds them"""

    def __init__(self, dev):
        from lookoncetohear_b200 import Net
        torch.manual_seed(0)
        sd = Net(**TSH_PARAMS).state_dict()
        g = torch.Generator().manual_seed(1)
        s = lambda k: sd["tfgridnet." + k].detach().float()
        self.We, self.be = s("embed_to_feats_proj.0.weight"), s("embed_to_feats_proj.0.bias")
        self.lg, self.lb = 1 + 0.3 * torch.randn(FC, generator=g), 0.3 * torch.randn(FC, generator=g)
        self.d = {k: getattr(self, k).contiguous().to(dev) for k in ("We", "be", "lg", "lb")}
        self.c = kh.SepFrontBack()
        self.c.we, self.c.be = self.d["We"].data_ptr(), self.d["be"].data_ptr()
        self.c.lne_g, self.c.lne_b = self.d["lg"].data_ptr(), self.d["lb"].data_ptr()
        self.c.gen = GEN

    def gate(self, e, **mut):
        return kh.gate64(e, self.We, self.be, self.lg, self.lb, **mut)

    def pre(self, e):
        p = self.We.double() @ e.double() + self.be.double()
        return p, kh.U32 * 4 * (self.We.double().abs() @ e.double().abs() + self.be.double().abs())


@pytest.fixture(scope="module")
def gw(dev):
    return GateWeights(dev)


# record k's memo key, relative to the embedding of the row that lists it: "match" (same embedding and generation: no
# rebuild), "gen" (built with the previous weight generation), "elem" (one embedding element changed), "nan" (a fresh
# record), "nan_elem" (one key element NaN)
MEMO = ["nan", "match", "gen", "elem", "nan_elem", "match", "gen", "elem", "nan", "match"]
# the Records map: rows -> slots (out of range: -1, batch, 2^31 - 1) and hops (0 and outside [0, T]: no frame)
GATE_SLOTS = [3, 1, -1, 2, 10, 4, 5, 6, 7, INT_MAX, 9, 8]
GATE_HOPS = [1, 1, 1, 0, 1, 4, 3, -1, 2, 1, 1, 1]
GATE_T = 3


@pytest.mark.parametrize("form", ["dense", "records", "records_hops"])
def test_spk_gate(form, gw, lay, dev):
    batch = len(MEMO)
    st = State(lay, batch, dev)
    g = torch.Generator().manual_seed(21)
    if form == "dense":
        slots, hops = list(range(batch)), None
    else:
        slots, hops = GATE_SLOTS, (GATE_HOPS if form == "records_hops" else None)
    rows = len(slots)
    emb = torch.randn(rows, SPK, generator=g)
    row_of = {s: b for b, s in enumerate(slots) if 0 <= s < batch}
    for k in range(batch):                                        # the memo keys
        e = emb[row_of[k]].clone() if k in row_of else torch.randn(SPK, generator=g)
        kind = MEMO[k]
        if kind == "nan":
            e[:] = float("nan")
        elif kind == "elem":
            e[77] += 0.5
        elif kind == "nan_elem":
            e[5] = float("nan")
        st.emb(k).copy_(e.to(dev))
        st.gen(k).fill_(GEN - 1 if kind == "gen" else GEN)
        st.gate(k).copy_((1 + 0.5 * torch.randn(NF, CH, generator=g)).to(dev))      # an old gate
    before = st.t.clone()
    pre, pre_w = guarded((rows, FC), dev)
    demb = emb.to(dev)
    recs, keep = (None, None) if form == "dense" else records(st, slots, hops, GATE_T, dev)
    assert kh.spk_gate(gw.c, demb, pre, st.t, st.ss, recs, rows) == 0
    torch.cuda.synchronize()
    assert guard_ok(pre_w)
    exp = before.clone()
    err, perr, muts, rebuilt = 0.0, 0.0, {}, []
    for b in range(rows):
        writes = stores(slots, hops, b, batch, GATE_T) and MEMO[slots[b]] != "match"
        if not writes:
            assert bool((bits(pre[b]) == SENTINEL).all()), (form, b, "spk_pre row written")
            continue
        k = slots[b]
        rebuilt.append(k)
        ref, bound = gw.gate(emb[b])
        got = st.gate(k)
        err = max(err, ratio(got, ref, bound))
        for m, kw in (("cf_order", dict(cf_order=True)), ("unbiased", dict(unbiased=True))):
            muts[m] = min(muts.get(m, math.inf), ratio(got, gw.gate(emb[b], **kw)[0], bound))
        p, pb = gw.pre(emb[b])
        perr = max(perr, ratio(pre[b], p, pb))
        st.gate(k, exp).copy_(got)
        st.emb(k, exp).copy_(demb[b])
        st.gen(k, exp).fill_(GEN)
    assert torch.equal(bits(st.t), bits(exp)), (form, "state written outside the rebuilt memos")
    expect_rebuilt = {"dense": [0, 2, 3, 4, 6, 7, 8], "records": [3, 2, 4, 6, 7, 8],
                      "records_hops": [3, 7, 8]}[form]
    assert sorted(rebuilt) == sorted(expect_rebuilt), (form, rebuilt)
    if form != "dense":
        assert torch.equal(bits(st.rec(0)), bits(st.rec(0, before))), "record 0 written"
    WORST["gate"] = max(WORST.get("gate", 0.0), err)
    WORST["spk_pre"] = max(WORST.get("spk_pre", 0.0), perr)
    MARGIN["gate"] = min([MARGIN.get("gate", math.inf)] + list(muts.values()))
    print(f"[spk_gate {form}] rebuilt records {sorted(rebuilt)}; gate err {err:.3f} x bound, spk_pre {perr:.3f}; "
          "mutants / bound: " + ", ".join(f"{m} {e:.1f}" for m, e in muts.items()))
    assert err <= 1.0 and perr <= 1.0
    for m, e in muts.items():
        assert e >= SENSITIVITY, (m, e)


# ---- gate_fanout_kernel ----------------------------------------------------------------------------------------------
FAN_BATCH = 10
FAN_SLOTS = [4, 2, -1, 9, 7, 10, 1, 3]
FAN_OWNER = [0, 1, -1, 2, -1, 1, 0, 2]


@pytest.mark.parametrize("T", [1, 3])
@pytest.mark.parametrize("apply_gate", [0, 1])
@pytest.mark.parametrize("form", ["dense", "listed"])
def test_gate_fanout(form, apply_gate, T, lay, dev):
    st = State(lay, FAN_BATCH, dev)
    g = torch.Generator().manual_seed(31 + T)
    for k in range(FAN_BATCH):
        st.gate(k).copy_((1 + 0.5 * torch.randn(NF, CH, generator=g)).to(dev))
    before = st.t.clone()
    K = 3
    if form == "dense":
        M, rows, owner, slots = 3, 9, None, list(range(9))
    else:
        M, rows, owner, slots = 3, len(FAN_SLOTS), FAN_OWNER, FAN_SLOTS
    X0 = torch.randn(M, T, NF, CH, generator=g)
    X, Xw = guarded((rows, T, NF, CH), dev)
    gates = torch.stack([st.gate(s if 0 <= s < FAN_BATCH else 0).cpu() for s in slots])
    if form == "dense":
        rc = kh.gate_fanout(X0.to(dev), X, st.t, st.ss, None, None, K, T, apply_gate, rows)
    else:
        recs, keep = records(st, slots, None, T, dev)
        rc = kh.gate_fanout(X0.to(dev), X, st.t, st.ss, recs, i32(owner, dev), K, T, apply_gate, rows)
    assert rc == 0
    torch.cuda.synchronize()
    assert guard_ok(Xw) and torch.equal(bits(st.t), bits(before))
    got = bits(X.cpu())
    assert torch.equal(got, bits(kh.gate_fanout_ref(X0, gates, owner, K, apply_gate))), (form, apply_gate, T)
    caught = []
    for m in kh.FANOUT_MUTANTS:
        if (m == "owner_mod" and form == "dense") or (m == "gate_unowned" and form == "listed" and apply_gate):
            assert not torch.equal(got, bits(kh.gate_fanout_ref(X0, gates, owner, K, apply_gate, mutant=m))), m
            caught.append(m)
    print(f"[gate_fanout {form} gate={apply_gate} T={T}] bit-exact; mutants missed: {caught}")


# ---- gather_h_kernel / scatter_hc_kernel -----------------------------------------------------------------------------
HC_BATCH = 6
HC_SLOTS = [4, -1, 1, 5, 6, 0, 2]          # 6 = batch: out of range; record 3 is listed by no row
HC_HOPS = [2, 1, 0, 3, 1, 4, -1]           # frames T = 3: rows 2, 5, 6 advance none
HC_T = 3
HC_FORMS = [(0, 1), (0, 2), (0, 3), (1, 1), (1, 2)]


def hc_state(lay, dev, seed):
    st = State(lay, HC_BATCH, dev)
    g = torch.Generator().manual_seed(seed)
    for k in range(HC_BATCH):
        for blk in range(N_BLOCKS):
            for w in "hc":
                st.hc(k, blk, w).copy_(torch.randn(NF, CH, generator=g).to(dev))
    return st


@pytest.mark.parametrize("hops", [None, "ragged"])
@pytest.mark.parametrize("b0,nb", HC_FORMS, ids=[f"b0{b}_blocks{n}" for b, n in HC_FORMS])
@pytest.mark.parametrize("with_c", [False, True])
def test_gather_h(b0, nb, hops, with_c, lay, dev):
    st = hc_state(lay, dev, 41)
    hp = HC_HOPS if hops else None
    B = len(HC_SLOTS)
    recs, keep = records(st, HC_SLOTS, hp, HC_T, dev)
    before = st.t.clone()
    Hg, Hw = guarded((N_BLOCKS, B, NF, CH), dev)
    Cg, Cw = guarded((N_BLOCKS, B, NF, CH), dev)
    assert kh.gather_h(st.t, recs, b0, nb, B, Hg, Cg if with_c else None) == 0
    torch.cuda.synchronize()
    assert guard_ok(Hw) and guard_ok(Cw) and torch.equal(bits(st.t), bits(before))
    for which, buf in (("h", Hg), ("c", Cg)):
        for blk in range(N_BLOCKS):
            for b in range(B):
                s = HC_SLOTS[b]
                got = bits(buf[blk, b])
                if b0 <= blk < b0 + nb and (which == "h" or with_c):
                    # an out-of-range row reads record 0 (a copy nothing stores back)
                    assert torch.equal(got, bits(st.hc(s if 0 <= s < HC_BATCH else 0, blk, which))), (which, blk, b)
                else:
                    assert bool((got == SENTINEL).all()), (which, blk, b, "written outside the call's blocks")


@pytest.mark.parametrize("hops", [None, "ragged"])
@pytest.mark.parametrize("b0,nb", HC_FORMS, ids=[f"b0{b}_blocks{n}" for b, n in HC_FORMS])
def test_scatter_hc(b0, nb, hops, lay, dev):
    st = hc_state(lay, dev, 43)
    hp = HC_HOPS if hops else None
    B = len(HC_SLOTS)
    recs, keep = records(st, HC_SLOTS, hp, HC_T, dev)
    before = st.t.clone()
    g = torch.Generator().manual_seed(44)
    Hg = torch.randn(N_BLOCKS, B, NF, CH, generator=g).to(dev)
    Cg = torch.randn(N_BLOCKS, B, NF, CH, generator=g).to(dev)
    assert kh.scatter_hc(st.t, recs, b0, nb, B, Hg, Cg) == 0
    torch.cuda.synchronize()
    exp = before.clone()
    n_stored = 0
    for b in range(B):
        if not stores(HC_SLOTS, hp, b, HC_BATCH, HC_T):
            continue
        n_stored += 1
        for blk in range(b0, b0 + nb):
            st.hc(HC_SLOTS[b], blk, "h", exp).copy_(Hg[blk, b])
            st.hc(HC_SLOTS[b], blk, "c", exp).copy_(Cg[blk, b])
    assert n_stored == (2 if hops else 5)
    assert torch.equal(bits(st.t), bits(exp)), "state written outside the storing rows' blocks b0 .. b0 + nb - 1"


# ---- inter_gate_mask_kernel / inter_h_last_kernel --------------------------------------------------------------------
@pytest.mark.parametrize("ragged", [True, False])
@pytest.mark.parametrize("T", [1, 2, 5])
def test_inter_gate_mask_and_h_last(T, ragged, lay, dev):
    hops = [-1, 0, 1, T - 1, T, T + 1] if ragged else None
    B = 6
    st = State(lay, B, dev)
    recs, keep = records(st, list(range(B)), hops, T, dev)
    g = torch.Generator().manual_seed(51 + T)
    gx0 = torch.randn(B, T, NF, 256, generator=g)
    gx, gxw = guarded((B, T, NF, 256), dev)
    gx.copy_(gx0.to(dev))
    assert kh.inter_gate_mask(gx, recs, B) == 0
    Y = torch.randn(B, T, NF, CH, generator=g)
    Hg, Hw = guarded((B, NF, CH), dev)
    assert kh.inter_h_last(Y.to(dev), Hg, recs, B) == 0
    torch.cuda.synchronize()
    assert guard_ok(gxw) and guard_ok(Hw)
    exp = gx0.clone()
    for b in range(B):
        Tb = kh.row_frames(hops, b, T)
        exp[b, Tb:, :, 0::4] = -math.inf
        exp[b, Tb:, :, 1::4] = math.inf
        exp[b, Tb:, :, 2::4] = 0.0
        got = bits(Hg[b].cpu())
        if 0 < Tb < T:
            assert torch.equal(got, bits(Y[b, Tb - 1])), (b, Tb)
        else:
            assert bool((got == SENTINEL).all()), (b, Tb, "h of a row that ends with the recurrence written")
    assert torch.equal(bits(gx.cpu()), bits(exp))


# ---- the fused-projection tensor-core recurrence with per-sequence step counts (tc_lstm.cuh) --------------------------
class Ragged:
    """the separator's inter layout: B streams x 97 bins, L steps (row b*L*97 + t*97 + f), carried (h, c) at a stride with
    gaps, step counts per stream"""
    B, L, X_LD, OUT_LD = 7, 5, 68, 68
    STEPS = [-1, 0, 1, 4, 5, 6, 2]
    HC_STRIDE = NF * 64 + 16

    def __init__(self, dev):
        g = torch.Generator().manual_seed(61)
        self.dev = dev
        rows = self.B * self.L * NF
        self.x = torch.randn(rows, self.X_LD, generator=g).to(dev)
        self.ln_g, self.ln_b = (1 + 0.2 * torch.randn(64, generator=g)).to(dev), (0.2 * torch.randn(64, generator=g)).to(dev)
        wih = (torch.rand(256, 64, generator=g) * 2 - 1) * 0.25
        self.bias = (0.3 * torch.randn(256, generator=g)).to(dev)
        self.whh = ((torch.rand(1, 256, 64, generator=g) * 2 - 1) * 0.25).to(dev)
        hi, lo = kh.split_bf16(wih)
        self.hi, self.lo = hi.to(dev), lo.to(dev)
        self.h0 = torch.randn(self.B * self.HC_STRIDE, generator=g).to(dev)
        self.c0 = torch.randn(self.B * self.HC_STRIDE, generator=g).to(dev)
        self.steps = i32(self.STEPS, dev)

    def run(self, L, passes, steps):
        out = sentinel(self.B * self.L * NF * self.OUT_LD, self.dev)
        h, c = self.h0.clone(), self.c0.clone()
        a = kh.Lstm()
        a.out, a.out_ld, a.whh = out.data_ptr(), self.OUT_LD, self.whh.data_ptr()
        a.h_state, a.c_state, a.hc_outer_stride = h.data_ptr(), c.data_ptr(), self.HC_STRIDE
        a.nseq, a.L, a.inner_count, a.ndir = self.B * NF, L, NF, 1
        a.outer_stride, a.inner_stride, a.step_stride = self.L * NF, 1, NF
        a.x, a.x_ld, a.wih_hi, a.wih_lo = self.x.data_ptr(), self.X_LD, self.hi.data_ptr(), self.lo.data_ptr()
        a.bias, a.ln_g, a.ln_b = self.bias.data_ptr(), self.ln_g.data_ptr(), self.ln_b.data_ptr()
        a.steps = self.steps.data_ptr() if steps else None
        rc, why = kh.lstm(a, "tc_x", passes)
        torch.cuda.synchronize()
        assert rc == 0, why
        return out.view(self.B, self.L, NF, self.OUT_LD)[..., :64].cpu(), h.view(self.B, -1)[:, :NF * 64].cpu(), \
            c.view(self.B, -1)[:, :NF * 64].cpu(), c.view(self.B, -1)[:, NF * 64:].cpu()


@pytest.mark.parametrize("passes", [1, 2, 3])
def test_tc_lstm_x_steps(passes, dev):
    p = Ragged(dev)
    out, _, c, gap = p.run(p.L, passes, True)
    assert bool((bits(gap) == bits(p.c0.view(p.B, -1)[:, NF * 64:].cpu())).all()), "state gap written"
    c0 = p.c0.view(p.B, -1)[:, :NF * 64].cpu()
    for Tb in sorted(set(p.STEPS)):
        streams = [b for b, s in enumerate(p.STEPS) if s == Tb]
        if not 0 < Tb <= p.L:                                         # no step: c passes through every step unchanged
            for b in streams:
                assert torch.equal(bits(c[b]), bits(c0[b])), (passes, Tb)
            continue
        out_r, _, c_r, _ = p.run(Tb, passes, False)
        for b in streams:
            assert torch.equal(bits(out[b, :Tb]), bits(out_r[b, :Tb])), (passes, Tb, "outputs of the steps below T_b")
            assert torch.equal(bits(c[b]), bits(c_r[b])), (passes, Tb, "final c")
    assert bool(torch.isfinite(out).all())
    print(f"[tc_lstm_x steps, passes {passes}] steps {p.STEPS}: bit-identical to runs of T_b steps")


def test_tc_lstm_steps_refused_elsewhere(dev):
    """steps apply to the fused-projection kernel only: every other variant refuses them and launches nothing"""
    p = Ragged(dev)
    a = kh.Lstm()
    a.steps = p.steps.data_ptr()
    n0 = kh.lib().kh_launch_count()
    for v in ("auto", "tc"):
        rc, _ = kh.lstm(a, v)
        assert rc != 0, v
    assert kh.lib().kh_launch_count() == n0


def test_summary():
    for k, v in sorted(WORST.items()):
        print(f"worst {k:>8s}: {v:.3f} x bound; smallest mutant margin {MARGIN.get(k, math.nan):.1f}")
    assert all(v <= 1.0 for v in WORST.values()) and all(v >= SENSITIVITY for v in MARGIN.values())
