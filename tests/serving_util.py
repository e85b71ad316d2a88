"""Scaffolding shared by the serving tests (slot lists, multi-hop and ragged slot lists, per-stream clocks, several targets
per mixture and their groups): fixtures, seeded inputs, state comparisons, the copy / run / copy back oracle, and the
header parsing of the host-side tests.  Not a test module: each test file imports what it uses, the fixtures by name, so
`model` is built once per test file.  Fixed-buffer launches go through Net._launch, which names the C entry point."""
import contextlib
import ctypes
import os
import re

import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import Net, SepState, resample, synth

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
