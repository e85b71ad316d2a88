"""The separator's front and back (csrc/sep_kernels.cuh, csrc/hop_kernels.cuh) launched directly, every kernel against
float64.

front_kernel (an ordinary call, and one hop of the pipelined graph's group form), front_many_kernel (the engine's
geometry, and forced chunk / worker counts so that one CTA walks several (stream, chunk) items and the last chunk is
ragged), front1_kernel (the one-hop latency path), back_kernel (ordinary and group form) and back_many_kernel (the
engine's geometry and forced chunk / cluster counts) run through tests/kernels/kernel_harness.cu with the engine's launch
geometry.  The references (kernels/harness.py: front64, gate64, ih64, back64) restate the model
(tfgridnet_causal.py:229-273): frames of 192 samples every 128 with zeros outside [0, x_len), channels [Re m0, Re m1,
Im m0, Im m1], the causal 3x3 conv over [conv tail | frames] zero-padded in F, the gate LN_6208(W e + b) stored [f][c],
the transposed conv, channel o = 2 ear + ri, the synthesis over [iSTFT tail | frames] and the overlap-add of the previous
frame's last 64 samples; every reference takes the tails as input and returns the new ones.

Every launch puts 5 streams (140 for the engine geometry of many streams) in one state of two blocks.  The streams have
their own clocks (a fresh stream with zero tails, and ST_CALLS of both parities, ST_POS up to ~1.1 x 10^6, never
the header's pos), the two parity copies of every tail hold different data, and the speaker-gate memo keys differ per
stream (NaN key, matching key, an older weight generation, one changed embedding element).  Every float a kernel must
not write holds a NaN sentinel that must survive bit for bit: the rest of each record, the tail copy being read, the
buffers' guard floats, X rows past the call, y samples past y_len or of inactive streams.  Every float a kernel must not read is
NaN too: x past x_len and the two pad columns of the transposed analysis filters.

Bounds (element-wise, computed by the references next to each value; u = 2^-24, a sum of n terms bounded by
u sqrt(n) sum |terms|, input bounds carried through with |weights|).  front: the 192-tap STFT (u sqrt(192) per spectrum
value), then the 36-term conv plus bias (u sqrt(37)).  back: the 576-term transposed conv (u sqrt(576)), the synthesis
of 194 filter rows over 4 CTAs whose partial windows meet in a fixed order, plus the overlap-add (u sqrt(202)).  gate:
the 256-term GEMV (8 products per lane and a 5-level warp tree: u sqrt(16)) carried through the LayerNorm (|g| / sigma),
plus the LayerNorm's own rounding (<= 24 u relative).  front1's block-0 projection: LN_64(X) W_ih^T + b of the kernel's
own X, a 65-term sum plus the LayerNorm rounding.  The deconv tail is a copy and must be bit-exact.  Each test also
compares the kernel's output with the mutated references that apply to it (frames one hop late, Re/Im interleaved per
mic, the conv flipped in time, edges clamped, the other parity's tails, the x offset from the stream clock, a plain conv
for the transposed one, ear/ri swapped, the overlap-add tail dropped or from the wrong half, the iSTFT tail not carried,
the gate in (c, f) order, the gate's LayerNorm with unbiased variance): each must miss by >= 10x the bound.
Measured on one NVIDIA H100 80GB HBM3 (700 W power limit): worst error / bound 0.38 (front_kernel), 0.24 (front_kernel,
group form), 0.34 (front_many_kernel), 0.10 (front1_kernel X) and 0.17 (its GX), 0.27 (the gate), 0.055 (back_kernel),
0.029 (back_kernel, group form), 0.048 (back_many_kernel).  The smallest mutant error / bound is 14 (the gate against the
unbiased variance, which moves a value by only |LN| / 12416); every other mutant misses by more than 3500x.
"""
import math
import subprocess

import pytest
import torch

from kernels import harness as kh
from lookoncetohear_b200.configs import TSH_PARAMS

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC0DEAD
SENSITIVITY = 10.0
N_BLOCKS = 2
GUARD = 4096
NF, CH, FC, HOP, NROW, SPK = kh.NF, kh.CH, kh.FC, kh.HOP, kh.NROW, kh.SPK
GEN = 5
# per stream: frames consumed, calls (bit 0 = parity of the tails it reads), speaker-gate memo key
STREAMS = [dict(pos=0, calls=0, memo="nan"),              # a fresh stream: zero tails
           dict(pos=7, calls=3, memo="match"),
           dict(pos=12, calls=4, memo="gen"),              # gate built with an older weight generation
           dict(pos=1000003, calls=1001, memo="elem"),     # one embedding element changed
           dict(pos=58, calls=10, memo="nan")]
MASK = [1, 1, 0, 1, 0]
HDR_POS, HDR_CALLS = 40, 9
CLIPS = {"abs": (0, 0), "rel0": (1, 0), "rel37": (1, 37)}          # (pos_rel, header pos - clip_base)
WORST = {}                                                          # kernel -> worst error / bound, for the summary
MARGIN = {}                                                         # kernel -> smallest mutant error / bound


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    kh.lib()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def lay(dev):
    return kh.sep_layout(N_BLOCKS)


@pytest.fixture(scope="module")
def w(dev):
    return Weights(dev)


def sentinel(n, dev):
    return torch.full((n,), SENTINEL, dtype=torch.int32, device=dev).view(torch.float32)


def bits(t):
    return t.contiguous().view(torch.int32)


def buf(shape, dev):
    """a sentinel buffer of `shape` followed by GUARD sentinel floats; returns (view, whole)"""
    n = math.prod(shape)
    whole = sentinel(n + GUARD, dev)
    return whole[:n].view(shape), whole


def guard_ok(whole):
    return bool((bits(whole[-GUARD:]) == SENTINEL).all())


def is_sentinel(t):
    return bool((bits(t) == SENTINEL).all())


def ratio(got, ref, bound):
    """max |got - ref| / bound (an exact value has bound 0: any difference is infinitely far outside)"""
    d = (got.double().cpu() - ref).abs()
    return float((d / bound.clamp_min(1e-300)).max())


def check(key, err, mutants):
    """err (error / bound) <= 1; every mutant's error / bound >= SENSITIVITY.  Records the worst ratios."""
    WORST[key] = max(WORST.get(key, 0.0), err)
    if mutants:
        MARGIN[key] = min([MARGIN.get(key, math.inf)] + list(mutants.values()))
    print(f"[{key}] err {err:.3f} x bound; mutants / bound: " + ", ".join(f"{m} {e:.0f}" for m, e in mutants.items()))
    assert err <= 1.0, (key, err)
    for m, e in mutants.items():
        assert e >= SENSITIVITY, (key, m, e)


# ---- weights ---------------------------------------------------------------------------------------------------------
class Weights:
    """the front / back weights of a seeded Net (its STFT filters, default-initialised conv, deconv and speaker
    projection), a random gate LayerNorm, and a random block-0 input projection for front1_kernel"""

    def __init__(self, dev):
        from lookoncetohear_b200 import Net
        torch.manual_seed(0)
        sd = Net(**TSH_PARAMS).state_dict()
        g = torch.Generator().manual_seed(1)
        sd["tfgridnet.embed_to_feats_proj.1.weight"] = 1 + 0.3 * torch.randn(FC, generator=g)
        sd["tfgridnet.embed_to_feats_proj.1.bias"] = 0.3 * torch.randn(FC, generator=g)
        self.p = kh.pack_front_back(sd)                          # NaN in the 2 pad columns of wat
        s = lambda k: sd["tfgridnet." + k].float()
        self.Wa, self.Ws = s("enc.filterbank._filters")[:, 0], s("dec.filterbank._filters")[:, 0]
        self.Wc, self.bc, self.Wd, self.bd = s("conv.0.weight"), s("conv.0.bias"), s("deconv.weight"), s("deconv.bias")
        self.We, self.be = s("embed_to_feats_proj.0.weight"), s("embed_to_feats_proj.0.bias")
        self.lg, self.lb = s("embed_to_feats_proj.1.weight"), s("embed_to_feats_proj.1.bias")
        self.ln1_g, self.ln1_b = 1 + 0.2 * torch.randn(64, generator=g), 0.2 * torch.randn(64, generator=g)
        self.wih1_t = (torch.rand(64, 512, generator=g) * 2 - 1) * 0.125
        self.b1 = 0.1 * torch.randn(512, generator=g)
        self.d = {k: v.contiguous().to(dev) for k, v in self.p.items()}
        for k in ("ln1_g", "ln1_b", "wih1_t", "b1"):
            self.d[k] = getattr(self, k).to(dev)
        self.c = kh.SepFrontBack()
        for k, t in self.d.items():
            setattr(self.c, k, t.data_ptr())
        self.c.gen = GEN

    def front(self, x, x_len, s0, T, tail, **mut):
        return kh.front64(x, x_len, s0, T, tail, self.Wa, self.Wc, self.bc, **mut)

    def back(self, X, dtail, itail, **mut):
        return kh.back64(X, dtail, itail, self.Wd, self.bd, self.Ws, **mut)

    def gate(self, e, **mut):
        return kh.gate64(e, self.We, self.be, self.lg, self.lb, **mut)


# ---- state -----------------------------------------------------------------------------------------------------------
class State:
    """One state of B streams (STREAMS cycled, positions spread) and N_BLOCKS blocks, every float the sentinel except
    the header, the streams' clocks, tails (both parity copies, different data; zero for a fresh stream) and gate memo
    keys.  rel = header pos - clip_base."""

    def __init__(self, lay, B, dev, rel, emb, seed):
        self.lay, self.B, self.dev = lay, B, dev
        self.hdr, self.ss = lay["HEADER_BYTES"] // 4, lay["STREAM_STRIDE"]
        self.t = sentinel(self.hdr + B * self.ss, dev)
        i64, i32 = self.t.view(torch.int64), self.t.view(torch.int32)
        i64[0], i64[1], i64[2] = HDR_POS, HDR_CALLS, HDR_POS - rel
        i32[6] = 0                                                  # done: the last-CTA counter
        g = torch.Generator().manual_seed(seed)
        self.streams = []
        for b in range(B):
            s = dict(STREAMS[b % len(STREAMS)])
            if s["pos"] and b >= len(STREAMS):
                s["pos"] += 1000 * b                                # never the header's pos
            self.streams.append(s)
            o = self.hdr + b * self.ss
            i64[(o + lay["ST_POS"]) // 2] = s["pos"]
            i32[o + lay["ST_CALLS"]] = s["calls"]
            fresh = s["calls"] == 0
            for view, scale in ((self.conv(b), 1.5), (self.deconv(b), 0.7), (self.istft(b), 1.5)):
                v = torch.zeros(view.shape) if fresh else scale * torch.randn(view.shape, generator=g)
                view.copy_(v)
            e = emb[b].clone()
            if s["memo"] != "nan":
                if s["memo"] == "elem":
                    e[77] += 0.5
                self.rec(b)[lay["ST_EMB"]:lay["ST_EMB"] + SPK] = e.to(dev)
                i32[o + lay["ST_GEN"]] = GEN - 1 if s["memo"] == "gen" else GEN

    def rec(self, b, t=None):
        t = self.t if t is None else t
        return t[self.hdr + b * self.ss:self.hdr + (b + 1) * self.ss]

    def _f(self, b, name, shape, t=None):
        o = self.lay[name]
        return self.rec(b, t)[o:o + math.prod(shape)].view(shape)

    def conv(self, b, t=None):
        return self._f(b, "ST_CONV", (2, 2, 4, NF), t)

    def deconv(self, b, t=None):
        return self._f(b, "ST_DECONV", (2, 2, NF, CH), t)

    def istft(self, b, t=None):
        return self._f(b, "ST_ISTFT", (2, 2, NROW), t)

    def gate(self, b, t=None):
        return self._f(b, "ST_GATE", (NF, CH), t)

    def emb(self, b, t=None):
        return self._f(b, "ST_EMB", (SPK,), t)

    def par(self, b):
        return self.streams[b]["calls"] & 1

    def header(self, t=None):
        t = self.t if t is None else t
        i64 = t[:self.hdr].view(torch.int64)
        return int(i64[0]), int(i64[1]), int(i64[2]), int(t[:self.hdr].view(torch.int32)[6])

    def clock(self, b, t=None):
        r = self.rec(b, t)
        return int(r[self.lay["ST_POS"]:self.lay["ST_POS"] + 2].view(torch.int64)[0]), int(r.view(torch.int32)[self.lay["ST_CALLS"]])

    def advance(self, t, T, active):
        """t with the header and every active stream's clock advanced by one call of T frames (finish_call)"""
        t = t.clone()
        i64, i32 = t.view(torch.int64), t.view(torch.int32)
        i64[0] += T
        i64[1] += 1
        for b in range(self.B):
            if active is None or active[b]:
                o = self.hdr + b * self.ss
                i64[(o + self.lay["ST_POS"]) // 2] += T
                i32[o + self.lay["ST_CALLS"]] += 1
        return t


class Inputs:
    """x [B][2][cap] (samples past x_len NaN), the embeddings, X [B][T][97][64] for the back, and the activity mask"""

    def __init__(self, B, T, clip, xcut, dev, seed, masked):
        self.pos_rel, self.rel = CLIPS[clip]
        self.s0 = HOP * self.rel if self.pos_rel else 0
        self.x_len = self.s0 + HOP * T + xcut
        cap = self.s0 + HOP * T + 1024
        g = torch.Generator().manual_seed(seed)
        x = torch.randn(B, 2, cap, generator=g)
        x[..., self.x_len:] = torch.tensor([SENTINEL], dtype=torch.int32).view(torch.float32)
        self.x, self.dx = x, x.to(dev)
        self.emb = torch.randn(B, SPK, generator=g)
        self.demb = self.emb.to(dev)
        self.X = 0.7 * torch.randn(B, T, NF, CH, generator=g)
        self.active = [MASK[b % len(MASK)] for b in range(B)] if masked else None
        self.dact = None if self.active is None else torch.tensor(self.active, dtype=torch.uint8, device=dev)

    def live(self, b):
        return self.active is None or bool(self.active[b])


# ---- checks ----------------------------------------------------------------------------------------------------------
def check_front(key, w, st, before, inp, T, X, Xw, prew, frame_rows=None):
    """X (rows frame_rows of a group, or the whole call) against front64 and its mutants for every stream, active or not;
    the new conv tail of each active stream; the gate memo; and nothing else of the state written.  Returns the state the
    launch must have left (bits), for equality checks."""
    assert guard_ok(Xw) and guard_ok(prew)
    exp = before.clone()
    err, muts = 0.0, {}

    def mut(name, r):
        muts[name] = min(muts.get(name, math.inf), r)
    for b in range(st.B):
        par, s = st.par(b), st.streams[b]
        tail = st.conv(b, before)[par].cpu()
        ref = w.front(inp.x[b], inp.x_len, inp.s0, T, tail)
        Xb = X[b].cpu()
        err = max(err, ratio(Xb, ref["X"], ref["X_bound"]))
        rb = lambda r: ratio(Xb, r["X"], ref["X_bound"])
        if b % 5 == 1 or b == 3:                                      # mutants on two streams with history
            mut("shift", rb(w.front(inp.x[b], inp.x_len, inp.s0, T, tail, shift=1)))
            mut("reim_interleaved", rb(w.front(inp.x[b], inp.x_len, inp.s0, T, tail, reim_interleaved=True)))
            mut("conv_flip_time", rb(w.front(inp.x[b], inp.x_len, inp.s0, T, tail, conv_flip_time=True)))
            mut("edge_clamp", rb(w.front(inp.x[b], inp.x_len, inp.s0, T, tail, edge_clamp=True)))
            mut("other_parity", rb(w.front(inp.x[b], inp.x_len, inp.s0, T, st.conv(b, before)[par ^ 1].cpu())))
            if inp.pos_rel:
                s_clock = HOP * (s["pos"] - (HDR_POS - inp.rel))
                mut("x_offset_from_clock", rb(w.front(inp.x[b], inp.x_len, s_clock, T, tail)))
        if inp.live(b):
            got = st.conv(b)[par ^ 1]
            err = max(err, ratio(got, ref["tail"], ref["tail_bound"]))
            st.conv(b, exp)[par ^ 1] = got
            if s["memo"] != "match":
                g, gb = w.gate(inp.emb[b])
                got = st.gate(b)
                e = ratio(got, g, gb)
                gm = {"cf_order": ratio(got, w.gate(inp.emb[b], cf_order=True)[0], gb),
                      "unbiased": ratio(got, w.gate(inp.emb[b], unbiased=True)[0], gb)}
                check("gate", e, gm)
                st.gate(b, exp).copy_(got)
                st.emb(b, exp).copy_(inp.demb[b])
                st.rec(b, exp).view(torch.int32)[st.lay["ST_GEN"]] = GEN
    check(key, err, muts)
    assert torch.equal(bits(st.t), bits(exp)), "state written outside the new conv tails and the rebuilt gates"
    return exp


def check_back(key, w, st, before, inp, T, y, yw, y_len, advanced=True):
    """y against back64 and its mutants (active streams: the call's samples below y_len; everything else sentinel), the
    new deconv tail (bit-exact) and iSTFT tail of each active stream, the clocks advanced once, and nothing else written"""
    assert guard_ok(yw)
    exp = st.advance(before, T, inp.active) if advanced else before.clone()
    err, muts = 0.0, {}
    y = y.cpu()
    for b in range(st.B):
        if not inp.live(b):
            assert is_sentinel(y[b]), ("y of an inactive stream written", b)
            continue
        par = st.par(b)
        dt, it = st.deconv(b, before)[par].cpu(), st.istft(b, before)[par].cpu()
        ref = w.back(inp.X[b], dt, it)
        lo, hi = inp.s0, min(inp.s0 + HOP * T, y_len)
        assert is_sentinel(y[b, :, :lo]) and is_sentinel(y[b, :, hi:]), ("y written outside the call or past y_len", b)
        n = hi - lo
        if n <= 0:
            continue
        bound = ref["y_bound"][:, :n]
        got = y[b, :, lo:hi]
        err = max(err, ratio(got, ref["y"][:, :n], bound))
        if st.streams[b]["calls"]:                               # mutants on streams with history (a fresh one's is 0)
            for name, m in (("plain_conv", dict(plain_conv=True)), ("swap_ear_ri", dict(swap_ear_ri=True)),
                            ("ola_dropped", dict(ola="dropped")), ("ola_wrong_half", dict(ola="wrong_half")),
                            ("istft_not_carried", dict(carry_istft=False))):
                muts[name] = min(muts.get(name, math.inf), ratio(got, w.back(inp.X[b], dt, it, **m)["y"][:, :n], bound))
            o = w.back(inp.X[b], st.deconv(b, before)[par ^ 1].cpu(), st.istft(b, before)[par ^ 1].cpu())
            muts["other_parity"] = min(muts.get("other_parity", math.inf), ratio(got, o["y"][:, :n], bound))
        assert torch.equal(bits(st.deconv(b)[par ^ 1].cpu()), bits(ref["deconv_tail"].float())), ("deconv tail", b)
        got_i = st.istft(b)[par ^ 1]
        err = max(err, ratio(got_i, ref["istft_tail"], ref["istft_bound"]))
        st.deconv(b, exp)[par ^ 1] = st.deconv(b)[par ^ 1]
        st.istft(b, exp)[par ^ 1] = got_i
    check(key, err, muts)
    assert torch.equal(bits(st.t), bits(exp)), "state written outside the new tails and the clocks"


def setup(lay, dev, B, T, clip, masked, seed, xcut=64):
    inp = Inputs(B, T, clip, xcut, dev, seed, masked)
    st = State(lay, B, dev, inp.rel, inp.emb, seed + 1)
    return inp, st


def run_front(kind, w, st, inp, T, dev, **kw):
    X, Xw = buf((st.B, T, NF, CH), dev)
    pre, prew = buf((st.B, FC), dev)
    if kind == "front":
        rc = kh.front(w.c, inp.dx, inp.x_len, X, st.t, st.ss, st.B, T, inp.pos_rel, inp.demb, pre, active=inp.dact)
    else:
        rc = kh.front_many(w.c, inp.dx, inp.x_len, X, st.t, st.ss, st.B, T, inp.pos_rel, inp.demb, pre, kw["chunk"],
                           kw["workers"], active=inp.dact)
    torch.cuda.synchronize()
    assert rc == 0, (kind, rc)
    return X, Xw, pre, prew


def run_back(kind, w, st, inp, T, y_len, dev, **kw):
    y, yw = buf((st.B, 2, inp.s0 + HOP * T + 256), dev)
    dX = inp.X.to(dev)
    if kind == "back":
        rc = kh.back(w.c, dX, y, y_len, st.t, st.ss, st.B, T, inp.pos_rel, active=inp.dact)
    else:
        rc = kh.back_many(w.c, dX, y, y_len, st.t, st.ss, st.B, T, inp.pos_rel, kw["chunk"], kw["n_cl"], active=inp.dact)
    torch.cuda.synchronize()
    assert rc == 0, (kind, rc)
    return y, yw


TS = [1, 2, 3, 5, 37]
XCUT = {1: 37, 2: 64, 3: 0, 5: -50, 37: 1}          # x_len - (s0 + 128 T): inside the look-ahead, at its end, ...
YCUT = {1: 127, 2: 63, 3: 64, 5: 1, 37: 0}          # samples of the last frame below y_len


# ---- front_kernel ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masked", [False, True], ids=["all_active", "masked"])
@pytest.mark.parametrize("clip", list(CLIPS))
@pytest.mark.parametrize("T", TS)
def test_front_kernel(T, clip, masked, dev, lay, w):
    """an ordinary call of T frames: X of every stream (inactive ones too) against front64, the new conv tails of the
    active streams in the other parity copy, the gate rebuilt exactly for the active streams whose memo key differs"""
    inp, st = setup(lay, dev, 5, T, clip, masked, seed=10 * T, xcut=XCUT[T])
    before = st.t.clone()
    X, Xw, _, prew = run_front("front", w, st, inp, T, dev)
    check_front("front_kernel", w, st, before, inp, T, X, Xw, prew)
    assert st.header(before) == st.header()


# ---- front_many_kernel -----------------------------------------------------------------------------------------------
GEOM = ["engine", (1, 1), (1, 3), (3, 1), (3, 3), ("T", 3), ("T+4", 1)]


def _size(v, T):
    return {"T": T, "T+4": T + 4}.get(v, v)


@pytest.mark.parametrize("geom", GEOM, ids=["engine", "c1_w1", "c1_w3", "c3_w1", "c3_w3", "cT_w3", "cT4_w1"])
@pytest.mark.parametrize("T", [7, 37])
def test_front_many_kernel(T, geom, dev, lay, w):
    """one CTA walks several (stream, chunk) items (1 or 3 workers over up to 185 items, chunks of 1, 3 and >= T, the
    last one ragged): within the float64 bounds, and bit-identical to front_kernel (X, the whole state, the gate scratch)"""
    B = 5
    chunk, workers = kh.front_many_geometry(B, T) if geom == "engine" else (_size(geom[0], T), geom[1])
    out = []
    for kind in ("many", "front"):
        inp, st = setup(lay, dev, B, T, "rel37", True, seed=20 + T)
        before = st.t.clone()
        X, Xw, pre, prew = run_front(kind, w, st, inp, T, dev, chunk=chunk, workers=workers)
        if kind == "many":
            check_front("front_many_kernel", w, st, before, inp, T, X, Xw, prew)
        out.append((X, st.t, pre))
    for a, b in zip(*out):
        assert torch.equal(bits(a), bits(b)), "front_many_kernel and front_kernel differ"


# ---- front1_kernel ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masked", [False, True], ids=["all_active", "masked"])
@pytest.mark.parametrize("clip", ["abs", "rel37"])
def test_front1_kernel(clip, masked, dev, lay, w):
    """one frame over 13 bin tiles: X and the new conv tails within front64's bounds (and within them of front_kernel's
    X), block 0's input projection GX within ih64 of the kernel's own X, the gate as front_kernel builds it"""
    inp, st = setup(lay, dev, 5, 1, clip, masked, seed=30, xcut=37)
    before = st.t.clone()
    X, Xw = buf((st.B, 1, NF, CH), dev)
    GX, GXw = buf((st.B, NF, 512), dev)
    pre, prew = buf((st.B, FC), dev)
    rc = kh.front1(w.c, inp.dx, inp.x_len, X, GX, st.t, st.ss, st.B, inp.pos_rel, inp.demb, pre, active=inp.dact)
    torch.cuda.synchronize()
    assert rc == 0
    assert guard_ok(GXw)
    check_front("front1_kernel", w, st, before, inp, 1, X, Xw, prew)
    err = 0.0
    for b in range(st.B):
        ref, bound = kh.ih64(X[b, 0].cpu(), w.ln1_g, w.ln1_b, w.wih1_t, w.b1)
        err = max(err, ratio(GX[b], ref, bound))
    check("front1_kernel GX", err, {})
    st0 = State(lay, st.B, dev, inp.rel, inp.emb, 31)
    X0, _, _, _ = run_front("front", w, st0, inp, 1, dev)
    for b in range(st.B):
        ref = w.front(inp.x[b], inp.x_len, inp.s0, 1, st.conv(b, before)[st.par(b)].cpu())
        assert ratio(X[b], X0[b].double().cpu(), 2 * ref["X_bound"]) <= 1.0, b


# ---- back_kernel -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masked", [False, True], ids=["all_active", "masked"])
@pytest.mark.parametrize("clip", list(CLIPS))
@pytest.mark.parametrize("T", TS)
def test_back_kernel(T, clip, masked, dev, lay, w):
    """an ordinary call of T frames, y_len inside the last frame: y of the active streams against back64 below y_len and
    sentinel elsewhere, the new tails in the other parity copy, the clocks advanced exactly once"""
    inp, st = setup(lay, dev, 5, T, clip, masked, seed=40 + T)
    y_len = inp.s0 + HOP * (T - 1) + YCUT[T]
    before = st.t.clone()
    y, yw = run_back("back", w, st, inp, T, y_len, dev)
    check_back("back_kernel", w, st, before, inp, T, y, yw, y_len)
    pos, ncalls, _, done = st.header()
    assert (pos, ncalls, done) == (HDR_POS + T, HDR_CALLS + 1, 0)


@pytest.mark.parametrize("cut", [0, 1, 63, 64, 127, 128])
def test_back_kernel_y_len(cut, dev, lay, w):
    """y_len cuts the last of 3 frames after 0, 1, 63, 64, 127 and 128 samples (the overlap-add region is the first 64)"""
    T = 3
    inp, st = setup(lay, dev, 5, T, "rel37", False, seed=50 + cut)
    y_len = inp.s0 + HOP * (T - 1) + cut
    before = st.t.clone()
    y, yw = run_back("back", w, st, inp, T, y_len, dev)
    check_back("back_kernel", w, st, before, inp, T, y, yw, y_len)


# ---- back_many_kernel ------------------------------------------------------------------------------------------------
BGEOM = ["engine", (1, 1), (1, 2), (3, 1), (3, 2), ("T", 2)]


@pytest.mark.parametrize("geom", BGEOM, ids=["engine", "c1_n1", "c1_n2", "c3_n1", "c3_n2", "cT_n2"])
@pytest.mark.parametrize("T", [7, 37])
def test_back_many_kernel(T, geom, dev, lay, w):
    """one cluster walks several (stream, chunk) items (ragged last chunks): within the float64 bounds, the clocks
    advanced once, and bit-identical to back_kernel (y and the whole state)"""
    B = 5
    chunk, n_cl = kh.back_many_geometry(B, T) if geom == "engine" else (_size(geom[0], T), geom[1])
    out = []
    for kind in ("many", "back"):
        inp, st = setup(lay, dev, B, T, "rel37", True, seed=60 + T)
        y_len = inp.s0 + HOP * T - 5
        before = st.t.clone()
        y, yw = run_back(kind, w, st, inp, T, y_len, dev, chunk=chunk, n_cl=n_cl)
        if kind == "many":
            check_back("back_many_kernel", w, st, before, inp, T, y, yw, y_len)
        out.append((y, st.t))
    for a, b in zip(*out):
        assert torch.equal(bits(a), bits(b)), "back_many_kernel and back_kernel differ"


# ---- many streams: the engine's geometry at configs[2] / configs[4]-like stream counts --------------------------------
@pytest.mark.parametrize("T", [1, 2])
def test_many_streams_engine_geometry(T, dev, lay, w):
    """140 streams: with the engine's own geometry some front_many CTAs and back_many clusters walk two streams; both
    within the float64 bounds and bit-identical to front_kernel / back_kernel"""
    B = 140
    fc, fw = kh.front_many_geometry(B, T)
    bc, bn = kh.back_many_geometry(B, T)
    assert fw < B and bn < B
    res = {}
    for kind in ("many", "one"):
        inp, st = setup(lay, dev, B, T, "rel0", True, seed=70 + T)
        before = st.t.clone()
        X, Xw, pre, prew = run_front("front" if kind == "one" else "many", w, st, inp, T, dev, chunk=fc, workers=fw)
        if kind == "many":
            check_front("front_many_kernel", w, st, before, inp, T, X, Xw, prew)
        mid = st.t.clone()
        y_len = inp.s0 + HOP * T
        y, yw = run_back("back" if kind == "one" else "many", w, st, inp, T, y_len, dev, chunk=bc, n_cl=bn)
        if kind == "many":
            check_back("back_many_kernel", w, st, mid, inp, T, y, yw, y_len)
        res[kind] = (X, pre, y, st.t)
    for a, b in zip(res["many"], res["one"]):
        assert torch.equal(bits(a), bits(b))


# ---- the group form of the pipelined graph ---------------------------------------------------------------------------
@pytest.mark.parametrize("K", [2, 5, 8])
def test_group_form_equals_one_call(K, dev, lay, w):
    """K one-frame hops (front_kernel and back_kernel with frame_k = k of frames_total = K, samples at k * 128, each hop's
    X in its own workspace slot hist_stride floats apart) against one K-frame ordinary call: X, y and every tail
    bit-identical; the hops advance no clock (the graph's advance_header_kernel does), the ordinary call once"""
    B = 5
    slot = B * FC + 1000                                       # sentinel floats between the hops' slots
    res = {}
    for form in ("group", "call"):
        inp, st = setup(lay, dev, B, K, "rel37", False, seed=80 + K)
        before = st.t.clone()
        y_len = inp.s0 + HOP * K - 3
        y, yw = buf((B, 2, inp.s0 + HOP * K + 256), dev)
        pre, prew = buf((B, FC), dev)
        if form == "group":
            ws, wsw = buf((K * slot,), dev)
            Xk = [ws[k * slot:k * slot + B * FC].view(B, 1, NF, CH) for k in range(K)]
            for k in range(K):
                assert kh.front(w.c, inp.dx, inp.x_len, Xk[k], st.t, st.ss, B, 1, inp.pos_rel, inp.demb, pre, frame_k=k,
                                frames_total=K) == 0
            torch.cuda.synchronize()
            X = torch.cat(Xk, dim=1)
            assert guard_ok(wsw) and all(is_sentinel(ws[k * slot + B * FC:(k + 1) * slot]) for k in range(K))
            check_front("front_kernel group", w, st, before, inp, K, X, sentinel(GUARD, dev), prew)
            for k in range(K):
                Xk[k].copy_(inp.X[:, k:k + 1].to(dev))             # the back's input rows, in the same slots
            mid = st.t.clone()
            for k in range(K):
                assert kh.back(w.c, Xk[k], y, y_len, st.t, st.ss, B, 1, inp.pos_rel, frame_k=k, frames_total=K,
                               hist_stride=slot) == 0
            torch.cuda.synchronize()
            check_back("back_kernel group", w, st, mid, inp, K, y, yw, y_len, advanced=False)
            state = st.advance(st.t, K, None)
        else:
            X, _, pre, prew = run_front("front", w, st, inp, K, dev)
            y, yw = run_back("back", w, st, inp, K, y_len, dev)
            state = st.t
        res[form] = (X, y, pre, state)
    for name, a, b in zip(("X", "y", "gate scratch", "state"), res["group"], res["call"]):
        assert torch.equal(bits(a), bits(b)), name


def test_summary(dev):
    """prints the worst error / bound per kernel and the smallest mutant error / bound over the tests above (run in the
    same session) with the device's name and power limit"""
    p = torch.cuda.get_device_properties(dev)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(dev.index)],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    print(f"device: {p.name}, power limit {pl}")
    for k, v in sorted(WORST.items()):
        print(f"worst {k:>22s}: {v:.3f} x bound; smallest mutant margin {MARGIN.get(k, math.nan):.1f}")
    assert all(v <= 1.0 for v in WORST.values()) and all(v >= SENSITIVITY for v in MARGIN.values())
