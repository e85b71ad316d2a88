"""The separator's one-hop middle section (csrc/mid_kernel.cuh) and the tensor-core chain's cell kernel
(csrc/sep_kernels.cuh: lstm_cell_rows_kernel) launched directly, against float64.

mid_kernel runs the section of a one-hop call of at most 10 streams; mid_a -> mid_b -> mid_c run it for 11-21 streams
and, over a batch of hops (n_hops, hop_stride), in the pipelined graph, where mid_b carries h in shared memory and c in
registers from hop to hop.  lstm_cell_rows is the inter-LSTM cell of the many-stream one-hop tensor-core chain.  Every
launch goes through the engine's launchers (sep_launch.cuh), with the engine's grids for 132 SMs: at B = 11 mid_kernel's
CTAs walk more than one (stream, row tile) item, at B = 41 those of mid_a, mid_b and mid_c do too.

Each state holds B in {1, 5, 11, 41} streams and two blocks, at a record stride with a gap; the kernels run on block 1,
and one stream (of B > 1) is inactive: it computes X, QKV, H' and Hout as usual and leaves its h and c alone, bit for bit.
The references (kernels/harness.py: mid64, mid_a64, mid_b64, mid_c64, lstm_cell64) work on the unpacked weights:
X1 = X + Y W_l1 + b; the inter-LSTM step from LN(X1) and the carried (h, c), gates in columns j*4 + q; X2 = X1 + h' W_l2 +
b; P = PReLU(X2 W_qkv + b) with the Q / K / V slope of each column's group.  Each value has its own bound (u = 2^-24,
u sqrt(n) sum |terms| per n-term sum, input bounds carried through the LayerNorm by |g| / sigma and through the
activations by their derivatives); fast_sigmoid / fast_tanh (and lstm_cell_rows's ex2.approx.ftz form) add __expf's
documented 2 + 1.16 |x| ulp, the rounding of 1 + e and __fdividef's 2 ulp.  Two rows of each stream (7 and 96, the last
tile's one live row) have an X1 of spread 0.01, where eps inside or outside the sqrt differs.

Every float a kernel must not write holds the NaN sentinel 0x7FC0DEAD and must survive: the rows past each stream's 97,
the guard floats around every buffer, every other part of each record and the other block, the hop slots outside a
launch.  Bit identities the code implies are asserted without a tolerance: mid_kernel == mid_a; mid_b; mid_c (the same
mid_mm products, the operand order (h W_hh) + ((x W_ih) + b), X1 exact through global memory), and one launch over
n_hops hops == n_hops launches of one hop, for mid_a, mid_b and mid_c.

Mutants (each must miss the bound by >= 10x on the kernel's outputs): the LayerNorm's variance unbiased, eps outside the
sqrt, gates i and f swapped, the c carry dropped, h W_hh taken from the new h, the PReLU slope groups shifted by 4
columns, a residual or a bias dropped; over hops, h not advanced between hops and the state stored after the first hop.
Measured on one NVIDIA H100 80GB HBM3 (700 W power limit): worst error / bound 0.19 (mid_kernel), 0.19 (mid_a/b/c, one
hop), 0.18 (over 2 and 4 hops), 0.37 (lstm_cell_rows); the smallest mutant error / bound is 122 (eps outside the sqrt,
mid_kernel), then 279 (unbiased variance), 2092 (slope groups), 44364 (hop mutants), 3.0e6 (lstm_cell_rows).
"""
import pytest
import torch

from kernels import harness as kh
from kernels.scaffold import Guarded, Ledger, Records, bits, dev, lay, ratio  # noqa: F401

pytestmark = pytest.mark.gpu

N_BLOCKS, BLK = 2, 1
NF, NQKV = kh.NF, kh.NQKV
LOW_SPREAD_ROWS = (7, 96)
LEDGER = Ledger()


class Weights:
    def __init__(self, dev, seed=0):
        g = torch.Generator().manual_seed(seed)
        r = lambda *s, scale=1.0: scale * torch.randn(*s, generator=g)
        self.p = dict(wl1_t=r(128, 64, scale=128 ** -0.5), bl1=r(64, scale=0.3), ln2_g=1 + r(64, scale=0.2),
                      ln2_b=r(64, scale=0.2), wih2_t=r(64, 256, scale=0.25), whh2_t=r(64, 256, scale=0.25),
                      b2=r(256, scale=0.3), wl2_t=r(64, 64, scale=0.125), bl2=r(64, scale=0.3),
                      wqkv_t=r(64, NQKV, scale=0.125), bqkv=r(NQKV, scale=0.3),
                      slopes=torch.tensor([0.25, -0.3, 0.6, 0.1]))
        packed = kh.mid_pack(*(self.p[k] for k in ("wl1_t", "wih2_t", "whh2_t", "wl2_t", "wqkv_t")))
        self.d = {k: v.to(dev) for k, v in self.p.items()}
        self.d["mid_pack"] = packed.to(dev)
        self.c = kh.MidWeights(**{k: self.d[k].data_ptr() for k in
                                  ("mid_pack", "bl1", "ln2_g", "ln2_b", "b2", "bl2", "bqkv", "slopes")})


@pytest.fixture(scope="module")
def W(dev):
    return Weights(dev)


class State(Records):
    """B streams, N_BLOCKS blocks, records a gap apart; every float the sentinel except block BLK's (h, c)"""

    def __init__(self, lay, B, dev, seed):
        g = torch.Generator().manual_seed(seed)
        super().__init__(lay, B, dev, gap=36)
        assert self.hc(0, BLK, "h").data_ptr() % 16 == 0 and self.hc(0, BLK, "c").data_ptr() % 16 == 0
        self.h0 = 0.5 * torch.randn(B * NF, 64, generator=g)
        self.c0 = torch.randn(B * NF, 64, generator=g)
        for b in range(B):
            self.hc(b, BLK, "h").copy_(self.h0[b * NF:(b + 1) * NF])
            self.hc(b, BLK, "c").copy_(self.c0[b * NF:(b + 1) * NF])
        self.before = self.snapshot()

    def h(self):
        return torch.cat([self.hc(b, BLK, "h") for b in range(self.batch)])

    def c(self):
        return torch.cat([self.hc(b, BLK, "c") for b in range(self.batch)])

    def only_hc_of(self, live):
        """the state equals its initial image outside the (h, c) of the streams live ([B] bool)"""
        written = [self.hc(b, BLK, w) for b in range(self.batch) if live[b] for w in "hc"]
        return self.same_outside(self.index(*written), self.before)


def inputs(B, p, seed):
    """Y [B*97][128], X [B*97][64]; rows LOW_SPREAD_ROWS of each stream have an X1 of spread 0.01"""
    g = torch.Generator().manual_seed(seed)
    Y = torch.randn(B * NF, 128, generator=g)
    X = torch.randn(B * NF, 64, generator=g)
    for b in range(B):
        for f in LOW_SPREAD_ROWS:
            Y[b * NF + f] = 0
            X[b * NF + f] = 0.4 - p["bl1"] + 0.01 * torch.randn(64, generator=g)
    return Y, X


def active_mask(B, dev):
    """one inactive stream (B // 2) when B > 1; returns (device mask, per-stream bool, per-row bool)"""
    a = torch.ones(B, dtype=torch.uint8)
    if B > 1:
        a[B // 2] = 0
    return a.to(dev), a.bool(), a.bool().repeat_interleave(NF)


MID_MUTANTS = {"unbiased": True, "eps_outside": True, "swap_if": True, "drop_c": True, "whh_new_h": True,
               "drop_residual": True, "drop_bias": True, "slope_groups": (20, 48)}


def mutant(r, mr):
    """a mutated reference's values with the reference's bounds"""
    return {k: (r[k] if k.endswith("_b") else v) for k, v in mr.items()}


def mid_outputs_ratio(r, X2, P, h, c, live):
    """error / bound over the outputs of the section: X2, P and the stored (h, c) of the active rows"""
    return {"X": ratio(X2, r["X2"], r["X2_b"]), "QKV": ratio(P, r["P"], r["P_b"]),
            "h": ratio(h[live], r["h"][live], r["h_b"][live]), "c": ratio(c[live], r["c"][live], r["c_b"][live])}


def run_mid(W, st, Y, X, B, act, dev):
    dY, dX, dQ = Guarded((B * NF, 128), dev, Y), Guarded((B * NF, 64), dev, X), Guarded((B * NF, NQKV), dev)
    y0 = dY.whole.clone()
    assert kh.mid(W.c, dY.t, dX.t, dQ.t, st.t, st.ss, BLK, B, act) == 0
    torch.cuda.synchronize()
    assert torch.equal(bits(dY.whole), bits(y0)) and dX.ok() and dQ.ok()
    assert bool(torch.isfinite(dX.t).all()) and bool(torch.isfinite(dQ.t).all())
    return dX.t.clone(), dQ.t.clone()


def run_split(W, st, Y, X, B, act, dev):
    """mid_a -> mid_b -> mid_c, one hop (hop_stride 0): returns X1 (after mid_a), GI, Hn, X2, QKV"""
    dY, dX = Guarded((B * NF, 128), dev, Y), Guarded((B * NF, 64), dev, X)
    dGI, dHn, dQ = Guarded((B * NF, 256), dev), Guarded((B * NF, 64), dev), Guarded((B * NF, NQKV), dev)
    y0 = dY.whole.clone()
    assert kh.mid_a(W.c, dY.t, dX.t, dGI.t, B) == 0
    torch.cuda.synchronize()
    X1 = dX.t.clone()
    assert kh.mid_b(W.c, dGI.t, dHn.t, st.t, st.ss, BLK, B, active=act) == 0
    assert kh.mid_c(W.c, dHn.t, dX.t, dQ.t, B) == 0
    torch.cuda.synchronize()
    assert torch.equal(bits(dY.whole), bits(y0))
    for w in (dX, dGI, dHn, dQ):
        assert w.ok()
    for t in (X1, dGI.t, dHn.t, dX.t, dQ.t):
        assert bool(torch.isfinite(t).all())
    return X1, dGI.t.clone(), dHn.t.clone(), dX.t.clone(), dQ.t.clone()


@pytest.mark.parametrize("B", [1, 5, 11, 41])
def test_mid_kernel_and_split_form(B, W, lay, dev):
    """mid_kernel and mid_a;mid_b;mid_c against mid64, and against each other bit for bit"""
    Y, X = inputs(B, W.p, seed=B)
    act, streams, live = active_mask(B, dev)
    st = State(lay, B, dev, seed=100 + B)
    r = kh.mid64(Y, X, st.h0, st.c0, W.p)
    X2, P = run_mid(W, st, Y, X, B, act, dev)
    h, c = st.h(), st.c()
    assert st.only_hc_of(streams), "mid_kernel wrote outside the active streams' (h, c)"
    errs = mid_outputs_ratio(r, X2, P, h, c, live)
    mutated = {m: mutant(r, kh.mid64(Y, X, st.h0, st.c0, W.p, **{m: v})) for m, v in MID_MUTANTS.items()}
    muts = {m: max(mid_outputs_ratio(mr, X2, P, h, c, live).values()) for m, mr in mutated.items()}
    LEDGER.check("mid_kernel", errs, muts)

    st2 = State(lay, B, dev, seed=100 + B)
    X1s, GI, Hn, X2s, Ps = run_split(W, st2, Y, X, B, act, dev)
    assert st2.only_hc_of(streams), "mid_b wrote outside the active streams' (h, c)"
    errs = {"X1": ratio(X1s, r["X1"], r["X1_b"]), "GI": ratio(GI, r["GI"], r["GI_b"]), "Hn": ratio(Hn, r["h"], r["h_b"])}
    errs.update(mid_outputs_ratio(r, X2s, Ps, st2.h(), st2.c(), live))
    muts = {m: max(ratio(GI, mr["GI"], r["GI_b"]), ratio(Hn, mr["h"], r["h_b"]),
                   *mid_outputs_ratio(mr, X2s, Ps, st2.h(), st2.c(), live).values())
            for m, mr in mutated.items()}
    LEDGER.check("mid_a/b/c", errs, muts)
    # the same arithmetic in one kernel and in three
    assert torch.equal(bits(X2s), bits(X2)) and torch.equal(bits(Ps), bits(P))
    assert torch.equal(bits(st2.t), bits(st.t))


class HopSlab:
    """n_hops + 2 hop slots of `slot` floats (a multiple of 512); the launch covers slots 1 .. n_hops.  Slot layout:
    X [rows][64] | Y [rows][128] | GI [rows][256] directly followed by Hn [rows][64] (as in the engine's GX slot) | QKV
    [rows][112], 32 sentinel floats between regions"""

    def __init__(self, B, n_hops, dev):
        self.rows, self.n_hops = B * NF, n_hops
        o, self.off = 0, {}
        for name, cols in (("X", 64), ("Y", 128), ("GI", 256), ("QKV", NQKV)):
            self.off[name] = o
            o += self.rows * (cols + (64 if name == "GI" else 0)) + 32
        self.off["Hn"] = self.off["GI"] + self.rows * 256
        self.slot = -(-o // 512) * 512
        self.buf = Guarded(((n_hops + 2) * self.slot,), dev)
        self.t = self.buf.t

    def view(self, name, hop, cols):
        o = (hop + 1) * self.slot + self.off[name]
        return self.t[o:o + self.rows * cols].view(self.rows, cols)

    def ptr(self, name, hop=0):
        return self.t[(hop + 1) * self.slot + self.off[name]:]


def run_hops(W, st, Ys, Xs, B, n_hops, act, dev, singles=False):
    slab = HopSlab(B, n_hops, dev)
    for j in range(n_hops):
        slab.view("Y", j, 128)[:] = Ys[j].to(dev)
        slab.view("X", j, 64)[:] = Xs[j].to(dev)
    before = slab.buf.whole.clone()
    S = slab.slot
    if singles:
        for j in range(n_hops):
            assert kh.mid_a(W.c, slab.ptr("Y", j), slab.ptr("X", j), slab.ptr("GI", j), B) == 0
        for j in range(n_hops):
            assert kh.mid_b(W.c, slab.ptr("GI", j), slab.ptr("Hn", j), st.t, st.ss, BLK, B, active=act) == 0
        for j in range(n_hops):
            assert kh.mid_c(W.c, slab.ptr("Hn", j), slab.ptr("X", j), slab.ptr("QKV", j), B) == 0
    else:
        assert kh.mid_a(W.c, slab.ptr("Y"), slab.ptr("X"), slab.ptr("GI"), B, S, n_hops) == 0
        torch.cuda.synchronize()
        X1 = torch.stack([slab.view("X", j, 64).clone() for j in range(n_hops)])
        assert kh.mid_b(W.c, slab.ptr("GI"), slab.ptr("Hn"), st.t, st.ss, BLK, B, S, n_hops, act) == 0
        assert kh.mid_c(W.c, slab.ptr("Hn"), slab.ptr("X"), slab.ptr("QKV"), B, S, n_hops) == 0
    torch.cuda.synchronize()
    out = {k: torch.stack([slab.view(k, j, c).clone() for j in range(n_hops)])
           for k, c in (("GI", 256), ("Hn", 64), ("X", 64), ("QKV", NQKV))}
    if not singles:
        out["X1"] = X1
    # nothing outside the written regions of the launched hops changed (inputs included, Y read-only)
    exp = before.clone()
    for j in range(n_hops):
        for k, c in (("GI", 256), ("Hn", 64), ("X", 64), ("QKV", NQKV)):
            v = slab.view(k, j, c)
            o = v.data_ptr() - slab.buf.whole.data_ptr()
            exp[o // 4:o // 4 + v.numel()] = v.reshape(-1)
    assert torch.equal(bits(slab.buf.whole), bits(exp)), "a hop-batch kernel wrote outside its hops' regions"
    for v in out.values():
        assert bool(torch.isfinite(v).all())
    return out


@pytest.mark.parametrize("n_hops", [2, 4])
@pytest.mark.parametrize("B", [5, 41])
def test_mid_split_over_hops(B, n_hops, W, lay, dev):
    """mid_a, mid_b, mid_c over n_hops hops at the engine's hop stride (one slot) against the references hop by hop;
    one launch over the batch == n_hops launches of one hop, bit for bit (all streams active: a stream that does not
    store carries h and c only inside a batch)"""
    g = torch.Generator().manual_seed(B * 7 + n_hops)
    Ys, Xs = zip(*(inputs(B, W.p, seed=1000 * B + 10 * n_hops + j) for j in range(n_hops)))
    act, streams, live = active_mask(B, dev)
    st = State(lay, B, dev, seed=int(torch.randint(1 << 30, (1,), generator=g)))
    out = run_hops(W, st, Ys, Xs, B, n_hops, act, dev)
    a = [kh.mid_a64(Ys[j], Xs[j], W.p) for j in range(n_hops)]
    GIs = torch.stack([x[2] for x in a])
    GIe = torch.stack([x[3] for x in a])
    H, He, (hs, hb, cs, cb) = kh.mid_b64(GIs, st.h0, st.c0, W.p, GIe)
    cc = [kh.mid_c64(a[j][0], a[j][1], H[j], He[j], W.p) for j in range(n_hops)]
    assert st.only_hc_of(streams)
    h, c = st.h(), st.c()
    errs = {"X1": max(ratio(out["X1"][j], a[j][0], a[j][1]) for j in range(n_hops)),
            "GI": ratio(out["GI"], GIs, GIe), "Hn": ratio(out["Hn"], H, He),
            "X2": max(ratio(out["X"][j], cc[j][0], cc[j][1]) for j in range(n_hops)),
            "QKV": max(ratio(out["QKV"][j], cc[j][2], cc[j][3]) for j in range(n_hops)),
            "h": ratio(h[live], hs[live], hb[live]), "c": ratio(c[live], cs[live], cb[live])}
    muts = {}
    for m in ("no_advance", "store_first"):
        Hm, _, (hm, _, cm, _) = kh.mid_b64(GIs, st.h0, st.c0, W.p, GIe, **{m: True})
        muts[m] = max(ratio(out["Hn"], Hm, He), ratio(h[live], hm[live], hb[live]), ratio(c[live], cm[live], cb[live]))
    LEDGER.check(f"mid_b over {n_hops} hops", errs, muts)

    runs = []
    for singles in (False, True):
        s = State(lay, B, dev, seed=5)
        o = run_hops(W, s, Ys, Xs, B, n_hops, None, dev, singles)
        runs.append((o, s.t.clone()))
    (o1, t1), (o2, t2) = runs
    for k in ("GI", "Hn", "X", "QKV"):
        assert torch.equal(bits(o1[k]), bits(o2[k])), k
    assert torch.equal(bits(t1), bits(t2)), "state"


@pytest.mark.parametrize("B", [3, 41])
def test_lstm_cell_rows(B, lay, dev):
    """rows = 97 B with B odd: the last CTA of 256 (row, unit) threads is partial"""
    g = torch.Generator().manual_seed(B)
    rows = B * NF
    assert (rows * 64) % 256 != 0
    gates = 2 * torch.randn(rows, 256, generator=g)
    act, streams, live = active_mask(B, dev)
    st = State(lay, B, dev, seed=B + 77)
    dG, dH = Guarded((rows, 256), dev, gates), Guarded((rows, 64), dev)
    g0 = dG.whole.clone()
    assert kh.lstm_cell_rows(dG.t, st.t, st.ss, BLK, dH.t, rows, act) == 0
    torch.cuda.synchronize()
    assert torch.equal(bits(dG.whole), bits(g0)) and dH.ok()
    dH = dH.t
    assert st.only_hc_of(streams)
    h_ref, hb, c_ref, cb = kh.lstm_cell64(gates, st.c0)
    h, c = st.h(), st.c()
    errs = {"Hout": ratio(dH, h_ref, hb), "h": ratio(h[live], h_ref[live], hb[live]),
            "c": ratio(c[live], c_ref[live], cb[live])}
    muts = {}
    for m in ("swap_if", "drop_c"):
        hm, _, cm, _ = kh.lstm_cell64(gates, st.c0, **{m: True})
        muts[m] = max(ratio(dH, hm, hb), ratio(c[live], cm[live], cb[live]))
    LEDGER.check("lstm_cell_rows", errs, muts)


def test_summary(dev):
    LEDGER.summary()
