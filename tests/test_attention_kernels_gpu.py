"""The separator's attention section (csrc/sep_kernels.cuh) launched directly, every kernel against float64.

qkv_kernel (projection inside, or projections given), qkv_many_kernel, kv_gather_kernel, the three attention forms
(attn_kernel = one CTA per query, attn_tile_kernel = 8 queries per CTA, attn_cluster_kernel = the window split over an
8-CTA cluster), attn_out_kernel and ln_frame_res_kernel run through tests/kernels/kernel_harness.cu with the engine's
launch geometry, each form forced, whatever the engine's occupancy-based choice would be.  The references
(kernels/harness.py) restate the model (tfgridnet_causal.py:540-588): PReLU slopes per Q/K/V group, LayerNorm per
(Q/K/V, head) over element f*d + e with biased variance, the 50-frame window ending at the query's frame in which frames
before the stream start are zero rows that take part in the softmax, softmax(q.k / sqrt(582)) V, channel h*16 + c.

Every launch puts 3-6 streams with their OWN clocks (ST_POS) in one state of two blocks and runs on block 1.  Clocks
come from {0, 1, 48, 49, 50, 55, 56, 57, 111, 2^31 + 7}: no history (< 49), the ring wrap (50, 55, 56, 57, 111) and
slot arithmetic above 2^31.  Every float a kernel must not write holds a NaN sentinel that must survive: block 0, the
other fields of each record, the scratch rows a kernel does not own, the gains' padding, and the 6 spare ring slots of
each window (the rows later hops of the pipelined graph have already overwritten: a kernel that reads one turns NaN).

Bounds (absolute, u = 2^-24, rounding errors of n terms growing like sqrt(n) u).  qkv: a 64-term fp32 dot product
(~8 u |x||w|, ~1e-6 here) divided by the projections' spread (~1) and scaled by the gains (<= 2), plus the LayerNorm's
own rounding and rsqrtf (a few u |y|, |y| < 6): 1e-5.  Attention, |score| ~ 1: a score is a 582-term sum whose error
(~24 u * 24) is ~1.5e-6 after the 1/sqrt(582) scale; it moves each probability by that much relatively, __expf and the
reciprocal add 2 ulp, and 50 fmas of values |v| < 5 add ~7 u |v|: 5e-6.  Attention, |score| up to ~80: partial sums
reach ~1700 before the scale, so a score carries ~2e-5, which moves each probability by as much relatively: 6e-5.
attn_out / ln_frame_res: the 64-term projection, a LayerNorm over 6208 values (|y| < 6), the residual add and the gate
(|gate| < 3): 2e-5 / 1e-5.  Hop chain: the qkv error (1e-5 on K and V) carried into the |score| ~ 1 attention: 1e-5.
Each test also compares the kernel's output with the mutated references that apply to it (a window shifted by one
frame, 49- or 51-row windows, history masked instead of zero-included, 1/sqrt(584), unbiased variance, heads
transposed, Q/K slopes swapped, the gate before the residual, a LayerNorm per bin): each must miss by >= 10x the bound.
In the wide-score regime the softmax cancels a uniform change of scale, so 1/sqrt(584) is checked at |score| ~ 1 only.
Measured on one NVIDIA H100 80GB HBM3 (700 W power limit): worst error / bound 0.38 (qkv_kernel), 0.14 (qkv_many),
0.15 / 0.26 (attention, |score| ~ 1 / wide), 0.18 (attn_out), 0.14 (ln_frame_res), 0.32 (hop chain); the smallest
mutant error / bound is 28 (attn_out against the unbiased variance).
"""
import math

import pytest
import torch

from kernels import harness as kh
from kernels.scaffold import SENTINEL, Guarded, Ledger, Records, bits, dev, is_sentinel, lay, ratio  # noqa: F401

pytestmark = pytest.mark.gpu

N_BLOCKS, BLK = 2, 1
BIG = 2 ** 31 + 7
CLOCKS = ([0, 50, 56, BIG, 111], [1, 48, 49, 55, 57, BIG])      # each set: < 49, the 50 / 56 boundaries, > 2^31
TOL = {"qkv": 1e-5, "unit": 5e-6, "wide": 6e-5, "attn_out": 2e-5, "ln_frame_res": 1e-5, "chain": 1e-5}
NF, CH, NH, ATT, RING = kh.NF, kh.CH, kh.NHEAD, kh.ATT, kh.RING
QK_DIM, QK_LD, V_DIM, FC = kh.QK_DIM, kh.QK_LD, kh.V_DIM, kh.FC
LEDGER = Ledger()                                                # keys (kernel, regime); bounds absolute: TOL


class State(Records):
    """One state of len(clocks) streams and N_BLOCKS blocks, every float the sentinel except the streams' clocks."""

    def __init__(self, lay, clocks, dev):
        super().__init__(lay, len(clocks), dev)
        self.clocks, self.B = list(clocks), len(clocks)
        for b, c in enumerate(self.clocks):
            self.pos(b).fill_(c)

    def rings(self, b, t=None):
        """views K [4][56][584], V [4][56][1552] of stream b's rings in block BLK"""
        return self.ring(b, BLK, "k", t), self.ring(b, BLK, "v", t)


# ---- weights ---------------------------------------------------------------------------------------------------------
class Weights:
    """the block weights the section reads, with distinct Q / K / V / projection PReLU slopes; the Q/K gains and biases
    are 584 floats with NaN padding (never used)"""

    def __init__(self, dev, seed):
        g = torch.Generator().manual_seed(seed)
        self.wqkv_t = (torch.rand(64, kh.NQKV, generator=g) * 2 - 1) * 0.25
        self.bqkv = 0.1 * torch.randn(kh.NQKV, generator=g)
        self.slopes = torch.tensor([0.25, -0.1, 0.05, 0.2])
        pad = torch.tensor([SENTINEL, SENTINEL], dtype=torch.int32).view(torch.float32)

        def ln(n, padded):
            gg, bb = 1 + 0.2 * torch.randn(n, generator=g), 0.2 * torch.randn(n, generator=g)
            return (torch.cat([gg, pad]), torch.cat([bb, pad])) if padded else (gg, bb)
        self.lnq, self.lnk, self.lnv = ln(QK_DIM, True), ln(QK_DIM, True), ln(V_DIM, False)
        self.wp_t = (torch.rand(64, 64, generator=g) * 2 - 1) * 0.25
        self.bp = 0.1 * torch.randn(64, generator=g)
        self.lnp = (1 + 0.2 * torch.randn(FC, generator=g), 0.2 * torch.randn(FC, generator=g))
        self.d = {}
        for name in ("wqkv_t", "bqkv", "slopes", "wp_t", "bp"):
            self.d[name] = getattr(self, name).to(dev)
        for name, (gg, bb) in (("lnq", self.lnq), ("lnk", self.lnk), ("lnv", self.lnv), ("lnp", self.lnp)):
            self.d[name + "_g"], self.d[name + "_b"] = gg.to(dev), bb.to(dev)
        self.c = kh.SepWeights()
        for name, t in self.d.items():
            setattr(self.c, name, t.data_ptr())

    def qkv_ref(self, X=None, pre=None, **mut):
        """Q, K [N, 4, 582], V [N, 4, 1552] of frames X [N, 97, 64] (projection inside) or projections pre [N, 97, 112]"""
        swap = mut.pop("swap_qk_slopes", False)
        P = kh.qkv_proj64(X, self.wqkv_t, self.bqkv, self.slopes, swap_qk_slopes=swap) if pre is None else pre.double()
        return kh.qkv_ln64(P, self.lnq, self.lnk, self.lnv, **mut)


# ---- qkv_kernel / qkv_many_kernel ------------------------------------------------------------------------------------
def qkv_outputs(st, Q, K, V, T, frame_k, active):
    """what a qkv launch produced, gathered per frame: Q, K, V [B*T, 4, n] from the Q buffer and (T > 1) the scratch, the
    ring rows [(b, t, K [4, 584], V [4, 1552])] it must have written, and the set {(b, slot)} of those rows"""
    B = st.B
    q = Q.view(B, NH, T, QK_LD).permute(0, 2, 1, 3).reshape(B * T, NH, QK_LD)
    ring, written = [], set()
    for b in range(B):
        if active is not None and not active[b]:
            continue
        k, v = st.rings(b)
        for t in range(max(0, T - ATT), T):
            slot = (st.clocks[b] + frame_k + t) % RING
            ring.append((b, t, k[:, slot], v[:, slot]))
            written.add((b, slot))
    return q, ring, written


def qkv_buffers(B, T, dev):
    """Q [B][4][T][584] and the K, V scratch [B][4][49 + T][584 / 1552] of a T-frame call"""
    return (Guarded((B, NH, T, QK_LD), dev), Guarded((B, NH, ATT - 1 + T, QK_LD), dev),
            Guarded((B, NH, ATT - 1 + T, V_DIM), dev))


def check_qkv(st, before, Q, K, V, T, frame_k, active, refs, tol, key):
    """assert everything a qkv launch must (and must not) have written, and its error against each reference"""
    B = st.B
    q, ring, written = qkv_outputs(st, Q.t, K.t, V.t, T, frame_k, active)
    assert Q.ok() and K.ok() and V.ok()
    K, V = K.t, V.t
    assert bool((bits(q[..., QK_DIM:]) == 0).all()), "Q pad columns"
    assert len(written) == len(ring), "a ring slot written twice"
    rows = st.index(*(r[:, slot] for b, slot in written for r in st.rings(b)))
    assert st.same_outside(rows, before), "state written outside the expected ring rows"
    got = {"q": q[..., :QK_DIM]}
    if T > 1:
        ks = K.view(B, NH, ATT - 1 + T, QK_LD)
        vs = V.view(B, NH, ATT - 1 + T, V_DIM)
        assert is_sentinel(ks[:, :, :ATT - 1]) and is_sentinel(vs[:, :, :ATT - 1]), "history rows of the scratch written"
        assert bool((bits(ks[:, :, ATT - 1:, QK_DIM:]) == 0).all()), "scratch pad columns"
        got["k"] = ks[:, :, ATT - 1:, :QK_DIM].permute(0, 2, 1, 3).reshape(B * T, NH, QK_DIM)
        got["v"] = vs[:, :, ATT - 1:].permute(0, 2, 1, 3).reshape(B * T, NH, V_DIM)
    else:
        assert is_sentinel(K) and is_sentinel(V), "scratch written by a one-frame call"
    for _, _, kr, _ in ring:
        assert bool((bits(kr[:, QK_DIM:]) == 0).all()), "ring pad columns"
    idx = [b * T + t for b, t, _, _ in ring]
    errs = {}
    for name, (rq, rk, rv) in refs.items():
        e = ratio(got["q"], rq, tol)
        if T > 1:
            e = max(e, ratio(got["k"], rk, tol), ratio(got["v"], rv, tol))
        if ring:
            e = max(e, ratio(torch.stack([r[2][:, :QK_DIM] for r in ring]), rk[idx], tol),
                    ratio(torch.stack([r[3] for r in ring]), rv[idx], tol))
        errs[name] = e
    err = errs.pop("ref")
    LEDGER.check(key, err, errs)


QKV_T = [(1, 0), (1, 5), (2, 0), (49, 0), (50, 0), (51, 0), (70, 0)]


@pytest.mark.parametrize("masked", [False, True], ids=["all_active", "masked"])
@pytest.mark.parametrize("T,frame_k", QKV_T, ids=[f"T{t}_k{k}" for t, k in QKV_T])
@pytest.mark.parametrize("mode", ["proj", "pre"])
def test_qkv_kernel(mode, T, frame_k, masked, dev, lay):
    clocks = CLOCKS[(T + frame_k) % 2]
    B = len(clocks)
    w = Weights(dev, seed=11)
    g = torch.Generator().manual_seed(100 + T)
    X = torch.randn(B * T, NF, CH, generator=g)
    pre = kh.qkv_proj64(X, w.wqkv_t, w.bqkv, w.slopes).float()
    active = torch.tensor([1, 0, 1, 1, 0, 1][:B], dtype=torch.uint8) if masked else None
    st = State(lay, clocks, dev)
    before = st.snapshot()
    Q, K, V = qkv_buffers(B, T, dev)
    dX, dpre = X.to(dev), pre.to(dev)
    rc = kh.qkv(w.c, dX, dpre if mode == "pre" else None, Q.t, K.t, V.t, st.t, st.ss, BLK, B, T, frame_k,
                None if active is None else active.to(dev))
    torch.cuda.synchronize()
    assert rc == 0
    src = {"pre": pre} if mode == "pre" else {"X": X}
    refs = {"ref": w.qkv_ref(**src), "unbiased": w.qkv_ref(**src, unbiased=True),
            "heads_transposed": w.qkv_ref(**src, heads_transposed=True)}
    if mode == "proj":
        refs["swap_qk_slopes"] = w.qkv_ref(**src, swap_qk_slopes=True)
    check_qkv(st, before, Q, K, V, T, frame_k, active, refs, TOL["qkv"], ("qkv_" + mode, "-"))


MANY = [(3, 13), (4, 60)]


@pytest.mark.parametrize("grid", [1, 2, 3, 7, 0], ids=["g1", "g2", "g3", "g7", "g_frames"])
@pytest.mark.parametrize("B,T", MANY, ids=[f"B{b}_T{t}" for b, t in MANY])
def test_qkv_many_kernel(B, T, grid, dev, lay):
    """each CTA walks frames fi, fi + grid, ... through two TMA buffers (grid 1: 39 / 240 frames, both parities many
    times); within the float64 bound, and bit-identical to qkv_kernel on the same projections (same LayerNorm source)"""
    clocks = (CLOCKS[0] + CLOCKS[1])[:B] if B != 3 else [48, 56, BIG]
    n_frames = B * T
    grid = grid or n_frames
    w = Weights(dev, seed=12)
    g = torch.Generator().manual_seed(200 + T)
    pre = kh.qkv_proj64(torch.randn(n_frames, NF, CH, generator=g), w.wqkv_t, w.bqkv, w.slopes).float()
    active = torch.tensor([1, 1, 0, 1][:B], dtype=torch.uint8) if grid == 7 else None
    dact = None if active is None else active.to(dev)
    out = []
    for kernel in ("many", "one"):
        st = State(lay, clocks, dev)
        before = st.snapshot()
        Q, K, V = qkv_buffers(B, T, dev)
        if kernel == "many":
            rc = kh.qkv_many(w.c, pre.to(dev), Q.t, K.t, V.t, st.t, st.ss, BLK, T, grid, n_frames, dact)
        else:
            rc = kh.qkv(w.c, None, pre.to(dev), Q.t, K.t, V.t, st.t, st.ss, BLK, B, T, 0, dact)
        torch.cuda.synchronize()
        assert rc == 0
        out.append((st.t, Q.whole, K.whole, V.whole))
        if kernel == "many":
            refs = {"ref": w.qkv_ref(pre=pre), "unbiased": w.qkv_ref(pre=pre, unbiased=True),
                    "heads_transposed": w.qkv_ref(pre=pre, heads_transposed=True)}
            check_qkv(st, before, Q, K, V, T, 0, active, refs, TOL["qkv"], ("qkv_many", "-"))
    for a, b in zip(*out):
        assert torch.equal(bits(a), bits(b)), "qkv_many_kernel and qkv_kernel differ"


# ---- K/V history: a per-stream model of Q / K / V rows by frame -----------------------------------------------------
REGIMES = {"unit": (1.0, 0.0, 1.0), "wide": (5.0, 0.34, 0.1)}     # (gain, alpha, beta)


class History:
    """Q / K / V rows of stream b for frames clocks[b] - 60 .. clocks[b] + n_after - 1 (fp32; K and V rows of frames
    before the stream start are zero).  Q, K = gain * (alpha s u_h + beta noise) with s = +1 on frames m with
    (m + 4h) mod 16 >= 8 and -1 otherwise, u_h a fixed direction per head h of norm sqrt(582).  unit: scores ~ N(0, 1).
    wide: scores s * ~70 +- ~1, so an 8-CTA split meets partials whose maxima differ by ~140 (and the zero rows of the
    history, at 0, between them), while ~25 high rows share each window's weight and every frame is a high row of some
    head; frames 0..7 are low rows of head 0, where the zero rows carry the weight of a young stream's window."""

    BACK = 60

    def __init__(self, clocks, n_after, regime, seed):
        gain, alpha, beta = REGIMES[regime]
        g = torch.Generator().manual_seed(seed)
        u = torch.randn(NH, QK_DIM, generator=g)
        u = u / u.norm(dim=1, keepdim=True) * math.sqrt(QK_DIM)
        self.clocks, self.n = list(clocks), self.BACK + n_after
        self.q, self.k, self.v = [], [], []
        for c in self.clocks:
            frames = torch.arange(self.n, dtype=torch.int64) + (c - self.BACK)
            s = torch.where((frames[:, None] + 4 * torch.arange(NH)) % 16 >= 8, 1.0, -1.0)[:, :, None]
            q = torch.zeros(self.n, NH, QK_LD)
            k = torch.zeros(self.n, NH, QK_LD)
            q[..., :QK_DIM] = gain * (alpha * u + beta * torch.randn(self.n, NH, QK_DIM, generator=g))
            k[..., :QK_DIM] = gain * (alpha * s * u + beta * torch.randn(self.n, NH, QK_DIM, generator=g))
            v = torch.randn(self.n, NH, V_DIM, generator=g)
            live = (frames >= 0)[:, None, None]
            self.q.append(q)
            self.k.append(torch.where(live, k, 0.0))        # +0.0, as the kernels write it
            self.v.append(torch.where(live, v, 0.0))

    def row(self, b, n):
        return n - (self.clocks[b] - self.BACK)

    def queries(self, frames_of):
        """Q buffer [B][4][T][584] with query t of stream b at frame frames_of(b)[t]"""
        return torch.stack([self.q[b][[self.row(b, n) for n in frames_of(b)]].permute(1, 0, 2) for b in range(len(self.clocks))])

    def scratch(self, T):
        """K, V scratch [B][4][49+T][...] of a T-frame call: row r = frame clock - 49 + r"""
        K = torch.stack([self.k[b][self.row(b, c - ATT + 1):self.row(b, c + T)].permute(1, 0, 2) for b, c in enumerate(self.clocks)])
        V = torch.stack([self.v[b][self.row(b, c - ATT + 1):self.row(b, c + T)].permute(1, 0, 2) for b, c in enumerate(self.clocks)])
        return K, V

    def fill_ring(self, st, frames_of, zero_history=True):
        """stream b's ring slots of frames frames_of(b) from the model; every other slot keeps the sentinel.
        zero_history=False: slots of frames before the start keep the sentinel too."""
        ring = kh.Ring(st.lay)
        for b in range(st.B):
            k, v = st.rings(b)
            for n in frames_of(b):
                if n < 0 and not zero_history:
                    continue
                k[:, ring.slot(n)] = self.k[b][self.row(b, n)].to(k.device)
                v[:, ring.slot(n)] = self.v[b][self.row(b, n)].to(v.device)

    def reference(self, frames_of, lo=-(ATT - 1), hi=0, scale=1.0 / math.sqrt(QK_DIM), mask_history=False,
                  heads_transposed=False):
        """Z [B, T, 97, 64] of queries at frames frames_of(b): each attends to frames n+lo .. n+hi (the model: -49 .. 0)"""
        out = []
        for b, c in enumerate(self.clocks):
            qn = frames_of(b)
            kf = [c - self.BACK + j for j in range(self.n)]
            q = self.q[b][[self.row(b, n) for n in qn]]                     # [T, 4, 584]
            win = kh.window_mask(qn, kf, lo, hi, mask_before_start=mask_history)
            o = kh.attention64(q, self.k[b], self.v[b], win, scale=scale)   # [T, 4, 1552]
            out.append(kh.merge_heads64(o, transposed=heads_transposed))
        return torch.stack(out)

    def mutants(self, frames_of, regime):
        m = {"shift": self.reference(frames_of, lo=-ATT, hi=-1), "rows49": self.reference(frames_of, lo=-(ATT - 2)),
             "rows51": self.reference(frames_of, lo=-ATT), "masked_history": self.reference(frames_of, mask_history=True),
             "heads_transposed": self.reference(frames_of, heads_transposed=True)}
        if regime == "unit":
            m["scale_584"] = self.reference(frames_of, scale=1.0 / math.sqrt(QK_LD))
        return m


def run_attention(form, hist, st, T, frame_k, dev, scratch=True):
    """Z [B, T, 97, 64] of one launch: the ring (T == 1, st's rings filled by the caller) or the scratch"""
    B = len(hist.clocks)
    Q = hist.queries(lambda b: [hist.clocks[b] + frame_k + t for t in range(T)]).to(dev).contiguous()
    K = V = None
    if T > 1:
        k, v = hist.scratch(T)
        K, V = k.to(dev).contiguous(), v.to(dev).contiguous()
    Z = Guarded((B, T, NF, CH), dev)
    rc = kh.attention(form, Q, K, V, st.t, st.ss, BLK, Z.t, B, T, frame_k)
    torch.cuda.synchronize()
    assert rc == 0, (form, T, frame_k)
    assert Z.ok()
    return Z.t


@pytest.mark.parametrize("regime", ["unit", "wide"])
@pytest.mark.parametrize("frame_k", [0, 1, 6])
@pytest.mark.parametrize("clocks", [0, 1], ids=["clocksA", "clocksB"])
@pytest.mark.parametrize("form", ["query", "cluster"])
def test_attention_ring(form, clocks, frame_k, regime, dev, lay):
    """T = 1: the window of frame clock + frame_k read from the ring (crossing the wrap at 50 + 6, 55, 56, 57, ...).
    The history slots of frames before the start are zero, as a fresh stream's are; the spare slots hold NaN.  The
    scratch form of the same kernel on the same window (query frame_k of a (frame_k + 2)-frame call) is bit-identical."""
    cl = CLOCKS[clocks]
    hist = History(cl, 10, regime, seed=300 + frame_k)
    st = State(lay, cl, dev)
    hist.fill_ring(st, lambda b: kh.Ring.window(cl[b] + frame_k))
    before = st.snapshot()
    Z = run_attention(form, hist, st, 1, frame_k, dev)
    assert st.same_outside(st.index(), before), "state written"
    frames = lambda b: [cl[b] + frame_k]
    ref = hist.reference(frames)
    mut = {m: ratio(Z, r, TOL[regime]) for m, r in hist.mutants(frames, regime).items()}
    LEDGER.check((form + "_ring", regime), ratio(Z, ref, TOL[regime]), mut)
    Zs = run_attention(form, hist, st, frame_k + 2, 0, dev)
    assert torch.equal(bits(Zs[:, frame_k]), bits(Z[:, 0])), "ring and scratch forms of one window differ"


SCRATCH = [("query", T) for T in (2, 9, 50, 70)] + [("cluster", T) for T in (2, 9, 50, 70)] + \
          [("tile", T) for T in (2, 7, 8, 9, 16, 57, 70)]


@pytest.mark.parametrize("regime", ["unit", "wide"])
@pytest.mark.parametrize("form,T", SCRATCH, ids=[f"{f}_T{t}" for f, t in SCRATCH])
def test_attention_scratch(form, T, regime, dev, lay):
    """T > 1: query t's window is scratch rows t .. t+49 (rows 0..48 = the 49 frames before the call); the tile form's
    last tile is ragged for T = 2, 7, 9, 57, 70"""
    cl = CLOCKS[T % 2]
    hist = History(cl, T + 2, regime, seed=400 + T)
    st = State(lay, cl, dev)
    Z = run_attention(form, hist, st, T, 0, dev)
    frames = lambda b: [cl[b] + t for t in range(T)]
    mut = {m: ratio(Z, r, TOL[regime]) for m, r in hist.mutants(frames, regime).items()}
    LEDGER.check((form + "_scratch", regime), ratio(Z, hist.reference(frames), TOL[regime]), mut)


@pytest.mark.parametrize("T", [2, 70])
@pytest.mark.parametrize("clocks", [0, 1], ids=["clocksA", "clocksB"])
def test_kv_gather(clocks, T, dev, lay):
    """scratch rows 0..48 = ring slots of frames clock-49 .. clock-1, bit for bit; zeros for frames before the start
    although their slots hold NaN; the spare slots (NaN) never read; rows 49.. and the state untouched"""
    cl = CLOCKS[clocks]
    B = len(cl)
    hist = History(cl, T + 2, "unit", seed=500 + T)
    st = State(lay, cl, dev)
    hist.fill_ring(st, lambda b: range(cl[b] - ATT + 1, cl[b]), zero_history=False)
    before = st.snapshot()
    _, K, V = qkv_buffers(B, T, dev)
    assert kh.kv_gather(st.t, st.ss, BLK, K.t, V.t, B, T) == 0
    torch.cuda.synchronize()
    assert st.same_outside(st.index(), before) and K.ok() and V.ok()
    K, V = K.t, V.t
    rk, rv = hist.scratch(T)
    assert torch.equal(bits(K[:, :, :ATT - 1].cpu()), bits(rk[:, :, :ATT - 1]))
    assert torch.equal(bits(V[:, :, :ATT - 1].cpu()), bits(rv[:, :, :ATT - 1]))
    assert is_sentinel(K[:, :, ATT - 1:]) and is_sentinel(V[:, :, ATT - 1:])


# ---- attn_out_kernel / ln_frame_res_kernel ---------------------------------------------------------------------------
@pytest.mark.parametrize("apply_gate", [0, 1])
@pytest.mark.parametrize("T", [1, 3])
@pytest.mark.parametrize("kernel", ["attn_out", "ln_frame_res"])
def test_attention_output(kernel, T, apply_gate, dev, lay):
    """X [B, T, 97, 64] += LayerNorm(6208)(P), times each stream's own gate (ST_GATE) after block 0; P = PReLU(Z W + b)
    inside attn_out_kernel, given to ln_frame_res_kernel.  Without the gate, the gate fields hold NaN and stay unread."""
    cl = CLOCKS[T % 2][:4]
    B = len(cl)
    w = Weights(dev, seed=13)
    g = torch.Generator().manual_seed(600 + T)
    Z = torch.randn(B, T, NF, CH, generator=g)
    X = torch.randn(B, T, NF, CH, generator=g)
    P = kh.prelu64(Z.double() @ w.wp_t.double() + w.bp.double(), float(w.slopes[3])).float()
    gate = 1 + 0.5 * torch.randn(B, FC, generator=g)
    st = State(lay, cl, dev)
    if apply_gate:
        for b in range(B):
            st.gate(b).copy_(gate[b].view(NF, CH))
    before = st.snapshot()
    dX = Guarded((B, T, NF, CH), dev, X)
    src = (Z if kernel == "attn_out" else P).to(dev)
    src0 = src.clone()
    fn = kh.attn_out if kernel == "attn_out" else kh.ln_frame_res
    assert fn(w.c, src, dX.t, st.t, st.ss, B, T, apply_gate) == 0
    torch.cuda.synchronize()
    assert st.same_outside(st.index(), before) and torch.equal(bits(src), bits(src0)) and dX.ok()
    dX = dX.t
    gt = gate[:, None].expand(B, T, FC).reshape(B * T, NF, CH) if apply_gate else None
    g64, b64 = w.lnp

    def ref(**mut):
        if kernel == "attn_out":
            r = kh.attn_out64(Z.view(-1, NF, CH), X.view(-1, NF, CH), w.wp_t, w.bp, w.slopes[3], g64, b64, gt, **mut)
        else:
            r = kh.ln_frame_res64(P.view(-1, NF, CH), X.view(-1, NF, CH), g64, b64, gt, **mut)
        return r.view(B, T, NF, CH)
    mutants = {"per_bin": ref(per_bin=True), "unbiased": ref(unbiased=True)}
    if apply_gate:
        mutants["gate_first"] = ref(gate_first=True)
    LEDGER.check((kernel, f"gate{apply_gate}"), ratio(dX, ref(), TOL[kernel]),
                 {m: ratio(dX, r, TOL[kernel]) for m, r in mutants.items()})


# ---- a kernel-level hop chain ----------------------------------------------------------------------------------------
def test_hop_chain_equals_one_call(dev, lay):
    """60 one-hop steps as the pipelined graph runs them (qkv with frame_k = k, then the ring attention of both forms,
    the clock held) against one 60-frame call (kv_gather, qkv, scratch attention of every form).  Q / K / V, the 50
    window slots of the last frame and each form's outputs are bit-identical; both match float64."""
    cl = [0, 50, BIG, 49]
    B, T = len(cl), 60
    w = Weights(dev, seed=14)
    hist = History(cl, T, "unit", seed=700)
    g = torch.Generator().manual_seed(701)
    X = torch.randn(B, T, NF, CH, generator=g)
    dX = X.to(dev)
    hop, one = State(lay, cl, dev), State(lay, cl, dev)
    for st in (hop, one):
        hist.fill_ring(st, lambda b: range(cl[b] - ATT + 1, cl[b]))      # the slots of frames clock .. clock+6: NaN
    forms = ("query", "cluster")
    Qh = torch.empty(B, NH, T, QK_LD, device=dev)
    Zh = {f: torch.empty(B, T, NF, CH, device=dev) for f in forms}
    for k in range(T):
        Xk = dX[:, k].contiguous()
        Qk = Guarded((B, NH, 1, QK_LD), dev).t
        assert kh.qkv(w.c, Xk, None, Qk, None, None, hop.t, hop.ss, BLK, B, 1, k) == 0
        for f in forms:
            Zk = Guarded((B, 1, NF, CH), dev).t
            assert kh.attention(f, Qk, None, None, hop.t, hop.ss, BLK, Zk, B, 1, k) == 0
            Zh[f][:, k] = Zk[:, 0]
        Qh[:, :, k] = Qk[:, :, 0]
    Q, K, V = (b.t for b in qkv_buffers(B, T, dev))
    assert kh.kv_gather(one.t, one.ss, BLK, K, V, B, T) == 0
    assert kh.qkv(w.c, dX, None, Q, K, V, one.t, one.ss, BLK, B, T, 0) == 0
    Z1 = {}
    for f in forms + ("tile",):
        Z1[f] = Guarded((B, T, NF, CH), dev).t
        assert kh.attention(f, Q, K, V, one.t, one.ss, BLK, Z1[f], B, T, 0) == 0
    torch.cuda.synchronize()
    assert torch.equal(bits(Qh), bits(Q))
    for b, c in enumerate(cl):
        slots = [(c + t) % RING for t in range(T - ATT, T)]
        for a, o in zip(hop.rings(b), one.rings(b)):
            assert torch.equal(bits(a[:, slots]), bits(o[:, slots])), b
        ko, vo = one.rings(b)
        assert torch.equal(bits(ko[:, slots]), bits(K[b, :, ATT - 1 + T - ATT:])) and torch.equal(bits(vo[:, slots]), bits(V[b, :, ATT - 1 + T - ATT:]))
    for f in forms:
        assert torch.equal(bits(Zh[f]), bits(Z1[f])), f
    # float64: the new frames' Q / K / V from the model's weights, the history from the ring
    rq, rk, rv = w.qkv_ref(X=X.view(B * T, NF, CH))
    for b in range(B):
        r0 = hist.row(b, cl[b])
        hist.q[b][r0:r0 + T, :, :QK_DIM] = rq.view(B, T, NH, QK_DIM)[b].float()
        hist.k[b][r0:r0 + T, :, :QK_DIM] = rk.view(B, T, NH, QK_DIM)[b].float()
        hist.v[b][r0:r0 + T] = rv.view(B, T, NH, V_DIM)[b].float()
    frames = lambda b: [cl[b] + t for t in range(T)]
    ref = hist.reference(frames)
    for f in forms + ("tile",):
        LEDGER.check((f + "_chain", "unit"), ratio(Z1[f], ref, TOL["chain"]),
                     {"shift": ratio(Z1[f], hist.reference(frames, lo=-ATT, hi=-1), TOL["chain"])})


def test_summary(dev):
    """prints the worst error / bound per kernel and regime over the tests above (run in the same session), and how many
    attn_cluster_kernel CTAs the device holds at once: the engine picks the cluster form while B * T * 4 * 8 fit"""
    LEDGER.summary()
    resident = kh.lib().kh_attn_cluster_resident()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    print(f"attn_cluster_kernel: {resident} resident CTAs on {sms} SMs; the cluster form up to B * T = {resident // 32}")
    assert resident >= sms and resident % sms == 0
