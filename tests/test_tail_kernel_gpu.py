"""The fused one-hop tail of a block (csrc/hop_kernels.cuh: tail_kernel) launched directly, against float64.

tail_kernel is one 16-CTA cluster per stream and runs everything of a block after the intra BiLSTM for one frame: the
middle section (phase M), the Q/K/V LayerNorms combined from 13 row tiles' (mean, M2) (phase Q), the 50-frame attention
over the K/V ring split over 4 CTAs per head (phase A), the merge of the heads' partials, Linear + PReLU, the
LayerNorm(6208) combined from the tiles, the residual and the speaker gate (phase O), and the next block's input
projection (phase G).  Both record maps run through the engine's launcher (sep_launch.cuh: launch_tail): the dense map
of one-hop calls and tail_kernel_t<Records> of slot-list, targets-groups and targets-rows calls.  frame_k is 0 as the
engine passes it.

The reference (kernels/harness.py: tail64, tail_chain64) is mid64, the Q/K/V LayerNorms per (Q/K/V, head) from the
tiles' statistics (chan_ln64), the window of frames pos - 49 .. pos in which frames before the stream start are zero rows
that take part in the softmax, softmax(q.k / sqrt(582)) V, channel h*16 + c, attn_out64's projection and LayerNorm, the
gate on the block output and ih64 of that output.  Each state holds streams with their own clocks from {0, 1, 48, 49,
50, 55, 56, 57, 111, 2^31 + 7} and two blocks at a record stride with a gap; the kernel runs on block 1.  Every float
the kernel must neither write nor read holds the NaN sentinel 0x7FC0DEAD: the 6 spare ring slots and the slot this hop
writes (a kernel that reads the newest row before it is written, or a spare slot, turns NaN), block 0, the other fields
of each record, the gains' padding and guard floats around every buffer.  Scores are ~1 ("unit") or spread over +-80
("wide", where each part of a head's window has its own max); the "edge" weights give one K head and the
LayerNorm(6208)'s input a mean >> spread, and two rows of each stream (7 and 96, the last tile's only row) an X1 of
spread 0.01, where eps inside or outside the sqrt differs.

Bounds.  (h, c): mid64's element-wise bounds (u = 2^-24, u sqrt(n) sum |terms| per n-term sum, input bounds carried
through the LayerNorm by |g| / sigma and through the activations by their derivatives).  K/V rows, per (Q/K/V, head)
group: 5e-5 |g|max for the projection and its rows of low X1 spread, plus 32 u |mean| / sigma |g|max for the tiles'
statistics and 4 u |P|max / sigma |g|max for P's own rounding.  X: 2e-4 for the attention and the projection, twice the
largest group bound (a K/V or q error moves a score, and so Z, by about as much), twice the window rows' bound in a
chain, and 24 u |mean| / sigma |g|max of the LayerNorm(6208), times max(1, |gate|).  GX: ih64's element-wise bound of the
kernel's own X output (as in test_front1_kernel).

Bit identities, without a tolerance: the (h, c) tail_kernel stores equal mid_kernel's from the same inputs (the same
mid_tile and mid_mm products; tail_kernel only computes h W_hh before the dependency wait); the K pad columns 582 and 583
of the written row are 0.0; nothing outside slot pos % 56 and (h, c) of the storing records changes; the Records form
equals the dense form row for row (X, GX, ring rows, h, c), and its rows with an out-of-range slot or hops = 0 store
nothing.

Mutants (each must miss its bound by >= 10x on at least one output of each test it applies to): the window shifted by
one frame, the newest row stale (|score| ~ 1 only: with wide scores it carries no weight), the head partials merged
without max rescaling, the Q/K/V statistics with equal tile weights or without the between-tile term, the
LayerNorm(6208) per tile, heads transposed, the gate before the residual or dropped, phase G applied to X2, and mid64's
eps outside the sqrt, gates i and f swapped and the c carry dropped.

Measured on one NVIDIA H100 80GB HBM3 (700 W power limit), which holds 7 tail_kernel clusters at once: worst error /
bound 0.166 (GX, "unit"), 0.150 (c, "wide edge") and 0.020 (the chain); the smallest mutant error / bound is 329 (eps
outside the sqrt, on (h, c)), then 1119 (the Q/K/V statistics without the between-tile term) and 3827 (the chain's
shifted window).  The file runs in about 10 s.
"""
import math

import pytest
import torch

from kernels import harness as kh
from kernels.scaffold import SENTINEL, Guarded, Ledger, Records, bits, dev, is_sentinel, lay, ratio  # noqa: F401

pytestmark = pytest.mark.gpu

N_BLOCKS, BLK = 2, 1
BIG = 2 ** 31 + 7
CLOCKS = (0, 1, 48, 49, 50, 55, 56, 57, 111, BIG)
NF, CH, NH, ATT, RING = kh.NF, kh.CH, kh.NHEAD, kh.ATT, kh.RING
QK_DIM, QK_LD, V_DIM, FC, NQKV = kh.QK_DIM, kh.QK_LD, kh.V_DIM, kh.FC, kh.NQKV
LOW_SPREAD_ROWS = (7, 96)
LEDGER = Ledger()


@pytest.fixture(scope="module")
def ncl(dev):
    n = kh.tail_clusters()
    assert n > 0, "tail_kernel's 16-CTA cluster cannot be scheduled: one-hop calls lose their 8-launch path"
    return n


class Weights:
    """block weights in the engine's layouts; edge: K head 2 (columns 36..41) and the LayerNorm(6208)'s input have a mean
    >> spread.  The Q/K LayerNorm vectors are 584 floats with sentinel padding (never read)."""

    def __init__(self, dev, edge, seed=0):
        g = torch.Generator().manual_seed(seed)
        r = lambda *s, scale=1.0: scale * torch.randn(*s, generator=g)
        p = dict(wl1_t=r(128, 64, scale=128 ** -0.5), bl1=r(64, scale=0.3), ln2_g=1 + r(64, scale=0.2),
                 ln2_b=r(64, scale=0.2), wih2_t=r(64, 256, scale=0.25), whh2_t=r(64, 256, scale=0.25),
                 b2=r(256, scale=0.3), wl2_t=r(64, 64, scale=0.125), bl2=r(64, scale=0.3),
                 wqkv_t=r(64, NQKV, scale=0.125), bqkv=r(NQKV, scale=0.3), slopes=torch.tensor([0.25, -0.3, 0.6, 0.1]),
                 wp_t=r(64, 64, scale=0.25), bp=r(64, scale=0.1), lnp_g=1 + r(FC, scale=0.2), lnp_b=r(FC, scale=0.2))
        pad = torch.tensor([SENTINEL, SENTINEL], dtype=torch.int32).view(torch.float32)
        for name, n in (("lnq", QK_DIM), ("lnk", QK_DIM), ("lnv", V_DIM)):
            gg, bb = 1 + r(n, scale=0.2), r(n, scale=0.2)
            p[name + "_g"], p[name + "_b"] = (torch.cat([gg, pad]), torch.cat([bb, pad])) if n == QK_DIM else (gg, bb)
        if edge:
            p["bqkv"][36:42] = 5.0                          # K head 2: mean 5, spread ~0.1
            p["wqkv_t"][:, 36:42] *= 0.1
            p["bp"] = 3.0 + 0.01 * r(64)                    # LayerNorm(6208) input: mean 3, spread ~0.03
            p["wp_t"] = p["wp_t"] * 0.1
        self.p = p
        self.nxt = (1 + r(64, scale=0.2), r(64, scale=0.2), r(64, 512, scale=0.125), r(512, scale=0.3))
        self.d = {k: v.to(dev) for k, v in p.items()}
        self.d["mid_pack"] = kh.mid_pack(*(p[k] for k in ("wl1_t", "wih2_t", "whh2_t", "wl2_t", "wqkv_t"))).to(dev)
        for k, v in zip(("nx_ln_g", "nx_ln_b", "nx_wih_t", "nx_bias"), self.nxt):
            self.d[k] = v.to(dev)
        names = [f[0] for f in kh.TailWeights._fields_]
        self.c_next = kh.TailWeights(**{k: self.d[k].data_ptr() for k in names})
        self.c_last = kh.TailWeights(**{k: (None if k.startswith("nx_") else self.d[k].data_ptr()) for k in names})
        self.c_mid = kh.MidWeights(**{k: self.d[k].data_ptr() for k in
                                      ("mid_pack", "bl1", "ln2_g", "ln2_b", "b2", "bl2", "bqkv", "slopes")})


@pytest.fixture(scope="module")
def weights(dev):
    return {edge: Weights(dev, edge) for edge in (False, True)}


class Stream:
    """one stream's inputs: Y, X (rows LOW_SPREAD_ROWS of X1 spread 0.01), (h, c), the gate (both signs), the K/V rows of
    frames pos - 50 .. pos - 1 (zero before the start) and the slot's old rows (the stale mutant).  unit: K ~ N(0, 1);
    wide: the score of frame n is t_n + ~0.05 with t_n uniform in [-80, 80], and 85 for frame pos - 50 (so a window
    shifted by one frame takes a new max)."""

    def __init__(self, W, pos, regime, seed):
        g = torch.Generator().manual_seed(seed)
        r = lambda *s, scale=1.0: scale * torch.randn(*s, generator=g)
        self.pos = pos
        self.Y, self.X = r(NF, 128), r(NF, 64)
        for f in LOW_SPREAD_ROWS:
            self.Y[f] = 0
            self.X[f] = 0.4 - W.p["bl1"] + 0.01 * r(64)
        self.h, self.c = r(NF, 64, scale=0.5), r(NF, 64)
        self.gate = (1 + 0.5 * r(NF, 64)) * torch.where(torch.rand(NF, 64, generator=g) < 0.2, -1.0, 1.0)
        k = torch.zeros(ATT, NH, QK_LD)
        if regime == "unit":
            k[..., :QK_DIM] = r(ATT, NH, QK_DIM)
        else:
            q = kh.tail64(self.Y, self.X, self.h, self.c, W.p, k, torch.zeros(ATT, NH, V_DIM))["Q"]     # Q needs no history
            t = 160 * torch.rand(ATT, NH, 1, generator=g, dtype=torch.float64) - 80
            t[0] = 85
            k[..., :QK_DIM] = (t * math.sqrt(QK_DIM) * q / (q * q).sum(-1, keepdim=True) + 0.05 * r(ATT, NH, QK_DIM)).float()
        v = r(ATT, NH, V_DIM)
        live = (torch.arange(ATT) + pos - ATT >= 0)[:, None, None]
        self.hk, self.hv = torch.where(live, k, 0.0), torch.where(live, v, 0.0)
        self.stale = (r(NH, QK_LD), r(NH, V_DIM))
        self.stale[0][:, QK_DIM:] = 0


class State(Records):
    """len(streams) records a gap apart, N_BLOCKS blocks, every float the sentinel except each record's clock, gate, block
    BLK's (h, c) and the ring rows of frames pos - 49 .. pos - 1 of block BLK"""

    def __init__(self, lay, streams, dev):
        super().__init__(lay, len(streams), dev, gap=36)
        self.B = len(streams)
        for b, s in enumerate(streams):
            self.put(b, s)
        self.before = self.snapshot()

    def put(self, b, s):
        self.pos(b).fill_(s.pos)
        self.gate(b).copy_(s.gate)
        self.hc(b, BLK, "h").copy_(s.h)
        self.hc(b, BLK, "c").copy_(s.c)
        for j in range(1, ATT):
            n = s.pos - ATT + j
            for hh in range(NH):
                self.row(b, "k", hh, n)[:] = s.hk[j, hh].to(self.t.device)
                self.row(b, "v", hh, n)[:] = s.hv[j, hh].to(self.t.device)

    def row(self, b, which, hh, n):
        return self.ring(b, BLK, which)[hh, kh.Ring.slot(n)]

    def written(self, b, pos):
        """what a storing launch at clock pos writes in record b: (h, c) and slot pos % 56 of K and V"""
        return [self.hc(b, BLK, "h"), self.hc(b, BLK, "c")] + [self.ring(b, BLK, w)[:, kh.Ring.slot(pos)] for w in "kv"]

    def only_written(self, stores):
        """the state equals its initial image outside what the launch at the current clocks writes for the records in
        `stores` ({record: pos})"""
        return self.same_outside(self.index(*(v for b, pos in stores.items() for v in self.written(b, pos))), self.before)


def launch(W, st, streams, B, apply_gate, has_next, dev, active=None):
    """kh.tail over the streams' rows; returns X [B][97][64], GX [B][97][512] (None without next block)"""
    dY = Guarded((B * NF, 128), dev, torch.stack([s.Y for s in streams]))
    dX, dG = Guarded((B * NF, 64), dev, torch.stack([s.X for s in streams])), Guarded((B * NF, 512), dev)
    y0 = dY.whole.clone()
    rc = kh.tail(W.c_next if has_next else W.c_last, dY.t, dX.t, dG.t, st.t, st.ss, BLK, B, apply_gate, 0, active)
    torch.cuda.synchronize()
    assert rc == 0
    assert torch.equal(bits(dY.whole), bits(y0)) and dX.ok() and dG.ok()
    if not has_next:
        assert is_sentinel(dG.t), "GX written without a next block"
    return dX.t.view(B, NF, 64).clone(), (dG.t.view(B, NF, 512).clone() if has_next else None)


def mutants_for(regime, apply_gate, has_next):
    names = [m for m in kh.TAIL_MUTANTS if not (m in ("gate_first", "drop_gate") and not apply_gate)
             and not (m == "ih_from_x2" and not has_next)]
    return names + (["stale"] if regime == "unit" else [])


def outputs_ratio(r, got, keys, GXb=None):
    """error / bound of the kernel's outputs `got` ({key: tensor}) against the reference r (GX against GXb)"""
    out = {}
    for k in keys:
        out[k] = ratio(got[k], r[k], GXb if k == "GX" else r[k + "_b"])
    return out


def stream_outputs(st, b, pos, X, GX):
    k = torch.stack([st.row(b, "k", hh, pos) for hh in range(NH)])
    v = torch.stack([st.row(b, "v", hh, pos) for hh in range(NH)])
    assert bool((bits(k[:, QK_DIM:]) == 0).all()), "K pad columns 582, 583"
    got = dict(X=X[b], K=k[:, :QK_DIM], V=v, h=st.hc(b, BLK, "h"), c=st.hc(b, BLK, "c"))
    if GX is not None:
        got["GX"] = GX[b]
    return got


CASES = [(1, "unit", 0, True, False), (3, "wide", 1, True, True), (3, "unit", 1, False, True),
         ("ncl", "unit", 1, True, False), ("ncl", "wide", 0, False, True), ("ncl", "unit", 0, True, True)]


@pytest.mark.parametrize("B,regime,apply_gate,has_next,edge", CASES,
                         ids=[f"B{b}-{r}-gate{g}-{'next' if n else 'last'}-{'edge' if e else 'plain'}" for b, r, g, n, e in CASES])
def test_tail_kernel(B, regime, apply_gate, has_next, edge, weights, lay, ncl, dev):
    """the dense form against tail64 per stream; one inactive stream (B > 1) leaves its record bit for bit; (h, c) equal
    mid_kernel's bit for bit"""
    B = ncl if B == "ncl" else B
    W = weights[edge]
    off = 5 if B == 1 else 3 * B
    streams = [Stream(W, CLOCKS[(off + b) % len(CLOCKS)], regime, seed=1000 * B + 10 * b + edge) for b in range(B)]
    act = torch.ones(B, dtype=torch.uint8)
    if B > 1:
        act[B // 2] = 0
    st = State(lay, streams, dev)
    X, GX = launch(W, st, streams, B, apply_gate, has_next, dev, act.to(dev))
    live = [b for b in range(B) if act[b]]
    assert st.only_written({b: streams[b].pos for b in live}), "tail_kernel wrote outside slot pos % 56 and (h, c)"
    errs, muts = {}, {}
    names = mutants_for(regime, apply_gate, has_next)
    for b in live:
        s = streams[b]
        gate = s.gate if apply_gate else None
        nxt = W.nxt if has_next else None
        r = kh.tail64(s.Y, s.X, s.h, s.c, W.p, s.hk, s.hv, gate, nxt)
        got = stream_outputs(st, b, s.pos, X, GX)
        keys = list(got)
        GXb = None
        if has_next:
            gx, GXb = kh.ih64(X[b].cpu(), *W.nxt)
            r = dict(r, GX=gx)
        for k, v in outputs_ratio(r, got, keys, GXb).items():
            errs[k] = max(errs.get(k, 0.0), v)
        for m in names:
            kw = dict(stale=s.stale) if m == "stale" else kh.TAIL_MUTANTS[m]
            mr = kh.tail64(s.Y, s.X, s.h, s.c, W.p, s.hk, s.hv, gate, nxt, **kw)
            ref_b = {k + "_b": r[k + "_b"] for k in keys if k != "GX"}
            muts[m] = max(muts.get(m, 0.0), max(outputs_ratio(dict(mr, **ref_b), got, keys, GXb).values()))
    LEDGER.check(f"tail {regime}{' edge' if edge else ''}", errs, muts)
    # the same mid_tile as mid_kernel: (h, c) bit for bit
    st2 = State(lay, streams, dev)
    dY = Guarded((B * NF, 128), dev, torch.stack([s.Y for s in streams]))
    dX = Guarded((B * NF, 64), dev, torch.stack([s.X for s in streams]))
    dQ = Guarded((B * NF, NQKV), dev)
    assert kh.mid(W.c_mid, dY.t, dX.t, dQ.t, st2.t, st2.ss, BLK, B, act.to(dev)) == 0
    torch.cuda.synchronize()
    for b in live:
        for w in ("h", "c"):
            assert torch.equal(bits(st.hc(b, BLK, w)), bits(st2.hc(b, BLK, w))), (b, w)


@pytest.mark.parametrize("hops", ["none", "list"])
def test_tail_kernel_records(hops, weights, lay, dev):
    """tail_kernel_t<Records> over a permuted, non-adjacent slot list of a state of 9 records, with one entry out of range
    and (hops = list) one row of hops = 0: those rows store nothing; every other row equals the dense form on the same
    records bit for bit (X, GX, ring rows, h, c)"""
    W = weights[True]
    batch = 9
    slots = [6, 2, 11, 4, 8]
    hop = [1, 1, 1, 0, 1] if hops == "list" else None
    stores = [b for b, sl in enumerate(slots) if 0 <= sl < batch and (hop is None or hop[b] > 0)]
    n = len(slots)
    recs = [Stream(W, CLOCKS[(3 * i) % len(CLOCKS)], "unit", seed=5000 + i) for i in range(batch)]
    calls = [Stream(W, 0, "unit", seed=6000 + b) for b in range(n)]          # the rows' Y and X
    st = State(lay, recs, dev)
    dY = Guarded((n * NF, 128), dev, torch.stack([s.Y for s in calls]))
    dX, dG = Guarded((n * NF, 64), dev, torch.stack([s.X for s in calls])), Guarded((n * NF, 512), dev)
    dslots = torch.tensor(slots, dtype=torch.int32, device=dev)
    dhops = None if hop is None else torch.tensor(hop, dtype=torch.int32, device=dev)
    assert kh.tail_slots(W.c_next, dY.t, dX.t, dG.t, st.t, st.ss, dslots, batch, dhops, BLK, n, 1) == 0
    torch.cuda.synchronize()
    assert dX.ok() and dG.ok()
    dX, dG = dX.t, dG.t
    assert st.only_written({slots[b]: recs[slots[b]].pos for b in stores}), "a row that stores nothing wrote its record"
    # the dense form over the same records, in call-row order (row b = record slots[b], record 0 for the out-of-range row)
    dense = [recs[sl] if 0 <= sl < batch else recs[0] for sl in slots]
    sd = State(lay, dense, dev)
    act = torch.zeros(n, dtype=torch.uint8)
    act[stores] = 1
    for b in range(n):
        dense[b].Y, dense[b].X = calls[b].Y, calls[b].X
    X, GX = launch(W, sd, dense, n, 1, True, dev, act.to(dev))
    for b in stores:
        assert torch.equal(bits(dX.view(n, NF, 64)[b]), bits(X[b])), b
        assert torch.equal(bits(dG.view(n, NF, 512)[b]), bits(GX[b])), b
        for a, d in zip(st.written(slots[b], recs[slots[b]].pos), sd.written(b, dense[b].pos)):
            assert torch.equal(bits(a), bits(d)), b


def test_tail_kernel_chain(weights, lay, dev):
    """6 consecutive launches over the ring wrap (clocks 53, 108 and 2^31 + 4 + 6 hops: slot 55 -> 0), ST_POS advanced
    on the host between them, against tail_chain64: the row written at slot pos % 56 is the one the next hops read"""
    W = weights[False]
    clocks, n_hops = [53, 108, BIG - 3], 6
    B = len(clocks)
    streams = [Stream(W, c, "unit", seed=7000 + b) for b, c in enumerate(clocks)]
    st = State(lay, streams, dev)
    g = torch.Generator().manual_seed(71)
    Ys = [[torch.randn(NF, 128, generator=g) for _ in range(n_hops)] for _ in range(B)]
    Xs = [[torch.randn(NF, 64, generator=g) for _ in range(n_hops)] for _ in range(B)]
    outs = []
    for j in range(n_hops):
        hop_streams = []
        for b, s in enumerate(streams):
            s.Y, s.X = Ys[b][j], Xs[b][j]
            st.pos(b).fill_(clocks[b] + j)
            hop_streams.append(s)
        X, _ = launch(W, st, hop_streams, B, 1, False, dev)
        outs.append(X)
    errs, muts = {}, {}
    for b, s in enumerate(streams):
        gates = [s.gate] * n_hops
        ref = kh.tail_chain64(Ys[b], Xs[b], s.h, s.c, W.p, s.hk, s.hv, gates)
        shifted = kh.tail_chain64(Ys[b], Xs[b], s.h, s.c, W.p, s.hk, s.hv, gates, shift=True)
        for j in range(n_hops):
            k = torch.stack([st.row(b, "k", hh, clocks[b] + j)[:QK_DIM] for hh in range(NH)])
            v = torch.stack([st.row(b, "v", hh, clocks[b] + j) for hh in range(NH)])
            errs["X"] = max(errs.get("X", 0.0), ratio(outs[j][b], ref[j]["X"], ref[j]["X_b"]))
            errs["K"] = max(errs.get("K", 0.0), ratio(k, ref[j]["K"], ref[j]["K_b"]))
            errs["V"] = max(errs.get("V", 0.0), ratio(v, ref[j]["V"], ref[j]["V_b"]))
            muts["shift"] = max(muts.get("shift", 0.0), ratio(outs[j][b], shifted[j]["X"], ref[j]["X_b"]))
        last = ref[-1]
        errs["h"] = max(errs.get("h", 0.0), ratio(st.hc(b, BLK, "h"), last["h"], last["h_b"]))
        errs["c"] = max(errs.get("c", 0.0), ratio(st.hc(b, BLK, "c"), last["c"], last["c_b"]))
    LEDGER.check("tail chain", errs, muts)


def test_summary(dev, ncl):
    print(f"tail_kernel: {ncl} clusters of 16 CTAs resident at once")
    LEDGER.summary()
