"""Scaffolding shared by the serving tests (slot lists, multi-hop and ragged slot lists, per-stream clocks, several targets
per mixture and their groups) and the per-slot stages: fixtures, seeded inputs, state comparisons, the copy / run / copy
back oracle, graph replays against eager twins, the 44.1 kHz tick on the separator, and the header parsing of the
host-side tests.  Not a test module: each test file imports what it uses, the fixtures by name, so `model` is built
once per test file.  Fixed-buffer launches go through Net._launch, which names the C entry point."""
import contextlib
import ctypes
import os
import re

import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import HopFifo, Limiter, Net, PacketResampler, SepState, TargetMixer, resample, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOP, LA = 128, 64
L2H_FLAG_TAPS, L2H_FLAG_GRAPH = 1, 2
SENTINEL = float("nan")
FAKE_DEV = ctypes.c_void_p(0x10000)          # never dereferenced: every host-side call fails its argument checks first
# the engine's defaults of the options the tests' kernel forms switch (include/lookonce_b200.h, l2h_sep_set_option)
DEFAULTS = {"fused_tail": 1, "back_many": 1, "fuse_ih": 0}


# ---- fixtures --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def model(tsh_params, dev):
    """(net on dev with its weights committed, the seeded state dict the reference restatement runs)"""
    torch.manual_seed(0)
    net = Net(**tsh_params).eval()
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    net = net.to(dev)
    net._sync_weights(dev)
    return net, sd


@pytest.fixture(scope="module")
def eng(tsh_params):
    """(net, engine handle, library) for the host-side tests: the handle never commits weights"""
    from lookoncetohear_b200 import build, _cabi
    build.build()
    net = Net(**tsh_params)
    return net, net._engine(), _cabi.lib()


@contextlib.contextmanager
def switched(net, opts):
    """the engine options `opts` set for the block's duration, then back to their DEFAULTS"""
    for k, v in opts.items():
        net.set_option(k, v)
    try:
        yield
    finally:
        for k in opts:
            net.set_option(k, DEFAULTS[k])


# ---- inputs ----------------------------------------------------------------------------------------------------------
def clips(n, hops, seed, dev):
    """n seeded mixtures of `hops` hops, padded with the 64 look-ahead samples, on dev; and their targets"""
    x, tgt = synth.mixture(n, HOP * hops, seed0=seed)
    return F.pad(x, (0, LA)).to(dev), tgt


def embeds(G, K, seed, dev):
    """[G, K, 256] seeded embeddings on dev"""
    return synth.embedding(G * K, seed0=seed)[:, 0].view(G, K, 256).to(dev)


def emb(n, seed, dev):
    """[n, 256] seeded embeddings on dev"""
    return embeds(n, 1, seed, dev)[:, 0]


def chunk(clip, t, T=1):
    """hops t .. t+T-1 of padded clips [..., N]: their 128*T samples + the 64 look-ahead samples"""
    return clip[..., HOP * t:HOP * (t + T) + LA]


def subsets(S, n, calls, seed):
    """a different unsorted list of n distinct slots (or groups) of S for every call"""
    g = torch.Generator().manual_seed(seed)
    return [torch.randperm(S, generator=g)[:n].tolist() for _ in range(calls)]


def hop_mix(n, T, seed):
    """n hop counts in [0, T] that include 0, 1 and T (n >= 3), else 1 and T"""
    g = torch.Generator().manual_seed(seed)
    h = torch.randint(0, T + 1, (n,), generator=g)
    fixed = [0, 1, T] if n >= 3 else [1, T]
    h[torch.randperm(n, generator=g)[:len(fixed)]] = torch.tensor(fixed)
    return h.tolist()


def i32(v, dev):
    return torch.tensor(v, dtype=torch.int32, device=dev)


def signals(S, C, n, seed, dev):
    """[S, C, n] seeded signals on dev"""
    return (0.1 * torch.randn(S, C, n, generator=torch.Generator().manual_seed(seed))).to(dev)


def delayed(whole, orig, new, D, n=None):
    """resample of the whole signals [S, C, N], delayed by D samples (zeros first): its first n samples, or as many as
    the resampled signals hold"""
    z = resample(whole, orig, new)
    return F.pad(z, (D, 0))[..., :z.shape[-1] if n is None else n]


# ---- states ----------------------------------------------------------------------------------------------------------
def bits(t):
    """a float tensor as its bit patterns: records hold NaN (the embedding of a fresh stream), which torch.equal rejects"""
    return t.contiguous().view(torch.int32)


def records(st):
    """every record of the state as bits, the gate memo's weight generation word cleared: copy_streams_from invalidates
    the memo of the records it writes (by design), so the oracle's records carry generation 0 where a listed call
    keeps it."""
    r = bits(st._rec()).clone()
    r[:, st.lay["st_emb"] + 256] = 0
    return r


def recs(groups, K):
    """the records g*K + k of the listed groups of a targets state"""
    return [g * K + k for g in groups for k in range(K)]


def foreign(st, K):
    """[records, stride] bool: the conv tails and block 0 of the non-lead records, which a targets call does not own"""
    L = st.lay
    m = torch.zeros(st.batch, st.stride, dtype=torch.bool, device=st.buf.device)
    nonlead = [r for r in range(st.batch) if r % K]
    m[nonlead, L["st_conv"]:L["st_deconv"]] = True
    m[nonlead, L["st_blk"]:L["st_blk"] + L["bk_stride"]] = True
    return m


def copy(net, st):
    """a new state holding the same bytes as st"""
    twin = net.init_buffers(st.batch, st.buf.device)
    twin.buf.copy_(st.buf)
    return twin


def host_state(net, batch):
    """a zero-filled SepState in host memory, for the Python argument checks (it has no engine behind it)"""
    hb, stride, offs = net._state_layout()
    return SepState(torch.zeros(hb // 4 + batch * stride), batch, net.n_blocks, hb, stride, offs)


def ring_mask(st, frames):
    """bool [stride]: the ring rows of a record holding the given frames (every block, head, K and V)"""
    L = st.lay
    m = torch.zeros(st.stride, dtype=torch.bool, device=st.buf.device)
    for blk in range(st.n_blocks):
        base = L["st_blk"] + blk * L["bk_stride"]
        for h in range(4):
            for f in frames:
                slot = f % L["ring"]
                k0 = base + L["bk_k"] + (h * L["ring"] + slot) * L["k_ld"]
                v0 = base + L["bk_v"] + (h * L["ring"] + slot) * L["v_dim"]
                m[k0:k0 + L["k_ld"]] = True
                m[v0:v0 + L["v_dim"]] = True
    return m


def ring_all(st):
    return ring_mask(st, range(st.lay["ring"]))


def oracle(net, st, listed, x, e, compact=None):
    """y of a call over the records `listed` of st, the way the API did it before slot lists: copy them into a compact
    state (`compact`, else a fresh one), run the dense call there -- predict for e [n, 256], predict_targets for e
    [n, K, 256] (listed: recs(groups, K)) -- and copy them back"""
    idx = list(range(len(listed)))
    if compact is None:
        compact = net.init_buffers(len(listed), x.device)
    compact.copy_streams_from(st, listed, idx)
    y, _ = (net.predict if e.dim() == 2 else net.predict_targets)(x, e, compact, pad=False)
    st.copy_streams_from(compact, idx, listed)
    return y


def warm_slots(net, S, n, T, seed, dev):
    """a state of S records with history and different clocks: 3 T-hop advance_slots calls over n of them"""
    x, _ = clips(S, 3 * T, seed, dev)
    e = emb(S, seed + 1, dev)
    st = net.init_buffers(S, dev)
    with torch.no_grad():
        for c, sl in enumerate(subsets(S, n, 3, seed + 2)):
            net.advance_slots(torch.stack([chunk(x[s], c * T, T) for s in sl]), e[sl], st, sl)
    return st


def warm_groups(net, G, n, K, T, seed, dev):
    """a targets state of G groups of K with history and different clocks, advanced by 2 T-hop oracle calls over n of
    them; and the hops each group has been fed"""
    x, _ = clips(G, 2 * T, seed, dev)
    e = embeds(G, K, seed + 1, dev)
    st = net.init_buffers(G * K, dev)
    compact = net.init_buffers(n * K, dev)
    fed = [0] * G
    with torch.no_grad():
        for sl in subsets(G, n, 2, seed + 2):
            oracle(net, st, recs(sl, K), torch.stack([chunk(x[g], fed[g], T) for g in sl]), e[sl], compact)
            for g in sl:
                fed[g] += T
    return st, fed


# ---- one CUDA graph against an eager twin ----------------------------------------------------------------------------
def captured(fn, warm=None):
    """a CUDA graph of fn(), captured after one run of warm() (default: fn) on a side stream"""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        (warm or fn)()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return graph


def refill(bufs):
    """the float buffers of the dict to SENTINEL and the int buffers to -1, so a sample a replay does not write shows"""
    for v in bufs.values():
        v.fill_(SENTINEL) if v.is_floating_point() else v.fill_(-1)


def assert_same(got, want, live, twin, where):
    """the buffers got[k] and want[k] (floats as bits) and the states of the stages live[k] and twin[k] equal"""
    for k in got:
        a, b = got[k], want[k]
        assert torch.equal(bits(a), bits(b)) if a.is_floating_point() else torch.equal(a, b), (where, k)
    for k in live:
        assert torch.equal(bits(live[k].state), bits(twin[k].state)), (where, k)


# ---- the 44.1 kHz tick on the separator ------------------------------------------------------------------------------
TICK_S, TICK_T, TICK_N = 4, 2, 3                         # slots, hops per tick, listeners (on slots 0 .. TICK_N - 1)
TICK_RECS, TICK_OFFSETS = [0, 1, 2, 3], [0, 1, 3, 4]     # listener 1 hears two voices


def separator_tick(net, dev, build=None, rows=None, mixed=None, after=None, bufs=None, each=None):
    """24 ticks of 44.1 kHz packets of 0, 441 or 882 samples (seeds 60 + t) from three listeners: down, FIFO,
    advance_target_rows, the mixer, up to 44.1 kHz and the limiter, captured in one CUDA graph after a warm-up that
    pushes nothing (every state stays as it was) and replayed with x and the counts rewritten in place.  After every
    replay the buffers and every stage's state are bit for bit those of the same chain run eagerly from the same states.

    A test adds its own stages: build(o) adds them to a fresh chain o and sets it up; rows, mixed and after, called as
    f(o, b, y, slots, rec, off), run them on the separator's rows y, on the mixer's sum b["mix"] and at the end of the
    tick.  `bufs` gives its extra buffers by name and width (None: an int32 count per listener), and each(b, t) sees
    the live buffers after every tick's comparison.  Returns the live stages."""
    S, T, n, C = TICK_S, TICK_T, TICK_N, 2
    x16, _ = clips(n, 40, 9900, dev)
    x44 = resample(x16[..., :HOP * 40].reshape(n * C, -1), 16000, 44100).reshape(n, C, -1).contiguous()
    e = emb(len(TICK_RECS), 9910, dev)
    widths = {"y16": 320, "oc": None, "chunk": HOP * T + LA, "hops": None, "mix": HOP * T, "y44": 353 * T,
              "oc44": None, "out": 353 * T, **(bufs or {})}

    def fresh():
        """[n, C, w] of SENTINEL for a width w, [n] int32 zeros for a width None"""
        return {k: torch.zeros(n, dtype=torch.int32, device=dev) if w is None else
                torch.full((n, C, w), SENTINEL, device=dev) for k, w in widths.items()}

    def chain():
        o = {"down": PacketResampler(44100, 16000, S, C, 882, device=dev), "fifo": HopFifo(S, C, T, 2048, device=dev),
             "mix": TargetMixer(S, S, C, device=dev), "up": PacketResampler(16000, 44100, S, C, HOP * T, device=dev),
             "lim": Limiter(S, C, 44100, device=dev)}
        if build:
            build(o)
        return o

    def tick(o, b, st, x, counts, slots, rec, off):
        o["down"](x, counts, slots, out=b["y16"], out_counts=b["oc"])
        o["fifo"](b["y16"], b["oc"], slots, out=b["chunk"], hops=b["hops"])
        y = net.advance_target_rows(b["chunk"], e, st, rec, off, hops=b["hops"])
        if rows:
            rows(o, b, y, slots, rec, off)
        o["mix"](y, rec, off, slots, hops=b["hops"], chunk=b["chunk"], out=b["mix"])
        if mixed:
            mixed(o, b, y, slots, rec, off)
        o["up"](b["mix"], b["hops"], slots, unit=HOP, out=b["y44"], out_counts=b["oc44"])
        o["lim"](b["y44"], b["oc44"], slots, out=b["out"])
        if after:
            after(o, b, y, slots, rec, off)

    def lists():
        return i32(list(range(n)), dev), i32(TICK_RECS, dev), i32(TICK_OFFSETS, dev)

    live, b = chain(), fresh()
    st = net.init_buffers(S, dev)
    x = torch.zeros(n, C, 882, device=dev)
    counts = i32([0] * n, dev)
    ls = lists()
    with torch.no_grad():
        graph = captured(lambda: tick(live, b, st, x, counts, *ls))
        torch.cuda.synchronize()
        twin, st_twin = chain(), copy(net, st)
        for k in live:
            twin[k].state.copy_(live[k].state)
        pos = [0] * n
        for t in range(24):
            g = torch.Generator().manual_seed(60 + t)
            cn = [[0, 441, 882][int(k)] for k in torch.randint(0, 3, (n,), generator=g)]
            cn = [min(c, x44.shape[-1] - pos[i]) for i, c in enumerate(cn)]
            x.fill_(0.0)
            for i in range(n):
                x[i, :, :cn[i]] = x44[i, :, pos[i]:pos[i] + cn[i]]
                pos[i] += cn[i]
            counts.copy_(i32(cn, dev))
            refill(b)
            graph.replay()
            want = fresh()
            tick(twin, want, st_twin, x, i32(cn, dev), *lists())
            assert_same(b, want, live, twin, t)
            if each:
                each(b, t)
    torch.cuda.synchronize()
    return live


# ---- the header ------------------------------------------------------------------------------------------------------
def header():
    with open(os.path.join(ROOT, "include", "lookonce_b200.h")) as f:
        return f.read()


def declaration(hdr, name):
    """(the match of `int name(...);` in hdr or None, its argument names)"""
    decl = re.search(rf"int {name}\((.*?)\);", hdr, flags=re.S)
    args = decl and [a.split()[-1].lstrip("*") for a in " ".join(decl.group(1).split()).split(",")]
    return decl, args


def doc_before(hdr, pos):
    """the comment block that ends before hdr[pos], as one line of words"""
    return " ".join(re.sub(r"\n\s*\*", " ", hdr[:pos].rsplit("/*", 1)[1]).split())
