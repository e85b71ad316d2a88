"""Streaming resampler on the GPU (l2h_resample_stream, lookoncetohear_b200.StreamResampler): every pushed sample against
`resample` of the stream's whole input delayed by D, bit for bit, and against the float64 restatement oracle/resample.py;
rows that store nothing, keep windows, reset and move, graph replays with the lists rewritten in place, and the chain
48 kHz device -> separator slot list -> 48 kHz device against the same chain built from whole-signal resampling."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import StreamResampler, resample, synth
from oracle import resample as ors
from serving_util import SENTINEL as NAN, bits, delayed, dev, hop_mix, i32, model, signals  # noqa: F401
from serving_util import assert_same, captured

pytestmark = pytest.mark.gpu

PAIRS = [(48000, 16000), (32000, 16000), (24000, 16000), (8000, 16000),
         (16000, 48000), (16000, 32000), (16000, 24000), (16000, 8000)]


def run_ticks(rs, sig, ticks, n, T, seed):
    """Push ragged seeded hop counts from sig [S, C, *] into the slots of rs over `ticks` calls of n rows (a fresh unsorted
    list of n of the S slots per call).  Checks every call's untouched samples (NaN sentinels), returns per slot the
    concatenated new samples and the keep windows seen, each with the number of outputs the slot had made before."""
    S, C, _ = sig.shape
    d = sig.device
    g = torch.Generator().manual_seed(seed)
    fed = [0] * S
    made = [0] * S
    outs = [[] for _ in range(S)]
    keeps = []
    for t in range(ticks):
        sl = torch.randperm(S, generator=g)[:n].tolist()
        hops = hop_mix(n, T, seed + t)
        x = torch.full((n, C, rs.block * T), NAN, device=d)        # samples past a row's pushes are never read
        for i, (s, h) in enumerate(zip(sl, hops)):
            x[i, :, :h * rs.block] = sig[s, :, fed[s]:fed[s] + h * rs.block]
        y = torch.full((n, C, rs.keep + T * rs.out_block), NAN, device=d)
        assert rs(x, i32(sl, d), i32(hops, d), out=y) is y
        for i, (s, h) in enumerate(zip(sl, hops)):
            w = rs.keep + h * rs.out_block
            assert torch.isnan(y[i, :, w:]).all(), "samples past the row's pushes were written"
            if h == 0:
                continue
            keeps.append((s, made[s], y[i, :, :rs.keep]))
            outs[s].append(y[i, :, rs.keep:w])
            fed[s] += h * rs.block
            made[s] += h * rs.out_block
    return [torch.cat(o, -1) if o else sig.new_zeros(C, 0) for o in outs], keeps, fed


@pytest.mark.parametrize("T", [1, 3, 8])
@pytest.mark.parametrize("orig,new", PAIRS)
def test_pushes_match_whole_signal_resample(dev, orig, new, T):
    S, C, n, ticks = 5, 2, 4, 7
    block = orig * 8 // 1000
    rs = StreamResampler(orig, new, S, C, block, keep=48, device=dev)
    sig = signals(S, C, block * T * ticks, 10 * orig + new + T, dev)
    outs, keeps, fed = run_ticks(rs, sig, ticks, n, T, seed=orig + T)
    for s in range(S):
        ref = delayed(sig[s:s + 1, :, :fed[s]], orig, new, rs.delay)[0] if fed[s] else sig.new_zeros(C, 0)
        assert outs[s].shape == ref.shape == (C, fed[s] * new // orig)
        assert torch.equal(bits(outs[s]), bits(ref)), (s, (outs[s] != ref).sum().item())
        if fed[s]:                                           # and the float64 restatement, within 1e-5
            want = ors.resample(sig[s, :, :fed[s]].cpu().double().numpy(), orig, new)[:, :ref.shape[-1] - rs.delay]
            got = outs[s][:, rs.delay:].cpu().double().numpy()
            assert np.linalg.norm(got - want) <= 1e-5 * np.linalg.norm(want)
    for s, m, kw in keeps:                                   # every keep window: the outputs m - keep .. m - 1
        full = F.pad(torch.cat([outs[s]], -1), (rs.keep, 0))
        assert torch.equal(bits(kw), bits(full[:, m:m + rs.keep])), (s, m)


def test_keep_window_is_the_one_hop_separator_chunk(dev):
    """48 kHz pushes of one hop with keep=64: each [C, 192] row is the pad=False chunk of the delayed 16 kHz signal"""
    rs = StreamResampler(48000, 16000, 3, 2, 384, keep=64, device=dev)
    assert (rs.hist, rs.delay, rs.out_block) == (37, 6, 128)
    assert rs.state.shape == (3, 2, 37 + 64) and rs.state.dtype == torch.float32 and not rs.state.any()
    sig = signals(1, 2, 384 * 6, 77, dev)
    z = F.pad(delayed(sig, 48000, 16000, 6)[0], (64, 0))       # 64 zeros, then the delayed signal
    for k in range(6):
        y = rs(sig[:, :, 384 * k:384 * (k + 1)], [1])
        assert y.shape == (1, 2, 192)
        assert torch.equal(bits(y[0]), bits(z[:, 128 * k:128 * k + 192])), k


def test_rows_that_store_nothing(dev):
    S, C, T = 6, 2, 2
    rs = StreamResampler(48000, 16000, S, C, 384, keep=16, device=dev)
    warm = signals(S, C, 384 * 3, 5, dev)
    rs(warm, list(range(S)), [3, 1, 2, 3, 0, 2])                # states with history and different clocks
    before = rs.state.clone()
    x = signals(4, C, 384 * T, 6, dev)
    y = torch.full((4, C, 16 + T * 128), NAN, device=dev)
    rs(x, i32([2, -1, 5, S + 3], dev), i32([0, 2, 1, 2], dev), out=y)
    assert torch.isnan(y[[0, 1, 3]]).all()                     # h = 0, and slots outside the state
    assert not torch.isnan(y[2, :, :16 + 128]).any() and torch.isnan(y[2, :, 16 + 128:]).all()
    changed = [s for s in range(S) if not torch.equal(bits(rs.state[s]), bits(before[s]))]
    assert changed == [5]


def test_reset_and_move(dev):
    S, C = 4, 2
    a = StreamResampler(16000, 48000, S, C, 128, keep=8, device=dev)
    b = StreamResampler(16000, 48000, S, C, 128, keep=8, device=dev)
    sig = signals(2, C, 128 * 10, 9, dev)
    a(sig[:, :, :128 * 4].contiguous(), [3, 1])                # slot 3 and 1 with history
    a.reset([3])
    assert not a.state[3].any() and a.state[1].any()
    y_a = a(sig[:1, :, 128 * 4:128 * 6].contiguous(), [3])
    y_b = b(sig[:1, :, 128 * 4:128 * 6].contiguous(), [0])     # a fresh stream
    assert torch.equal(bits(y_a), bits(y_b))
    b.state[2] = a.state[1]                                      # move slot 1 of a to slot 2 of b
    y_a = a(sig[1:, :, 128 * 4:128 * 7].contiguous(), [1])
    y_b = b(sig[1:, :, 128 * 4:128 * 7].contiguous(), [2])
    assert torch.equal(bits(y_a), bits(y_b)) and torch.equal(bits(a.state[1]), bits(b.state[2]))


def test_graph_replay_with_lists_rewritten_in_place(dev):
    S, C, n, T = 8, 2, 5, 3
    live = StreamResampler(48000, 16000, S, C, 384, keep=64, device=dev)
    twin = StreamResampler(48000, 16000, S, C, 384, keep=64, device=dev)
    x = torch.zeros(n, C, 384 * T, device=dev)
    y = torch.zeros(n, C, 64 + 128 * T, device=dev)
    slots, hops = i32(list(range(n)), dev), i32([T] * n, dev)
    graph = captured(lambda: live(x, slots, hops, out=y),              # warm-up pushes of zeros into slots 0 .. n-1
                     warm=lambda: (live(x, slots, hops, out=y), twin(x, slots, hops)))
    g = torch.Generator().manual_seed(31)
    for t in range(6):
        sl = torch.randperm(S, generator=g)[:n].tolist()
        sl[t % n] = -1 if t % 2 else S                              # one row per tick outside the state
        hp = hop_mix(n, T, 40 + t)
        x.copy_(signals(n, C, 384 * T, 50 + t, dev))
        slots.copy_(i32(sl, dev))
        hops.copy_(i32(hp, dev))
        y.fill_(NAN)
        graph.replay()
        want = torch.full_like(y, NAN)
        twin(x, i32(sl, dev), i32(hp, dev), out=want)
        assert_same({"y": y}, {"y": want}, {"rs": live}, {"rs": twin}, t)


def test_python_call_checks(dev):
    rs = StreamResampler(48000, 16000, 4, 2, 384, device=dev)
    x = torch.zeros(2, 2, 768, device=dev)
    for bad in ([0, 0], [0, 4], [-1, 0], [0], [0, 1, 2]):
        with pytest.raises(ValueError):
            rs(x, bad)
    for bad in ([0, 3], [-1, 1], [1]):
        with pytest.raises(ValueError):
            rs(x, [0, 1], bad)
    with pytest.raises(ValueError):
        rs(x, torch.tensor([0, 1], dtype=torch.int64, device=dev))     # CUDA lists are int32
    for shape in ((2, 2, 700), (2, 3, 768), (2, 2, 0)):
        with pytest.raises(ValueError):
            rs(torch.zeros(shape, device=dev), [0, 1])
    with pytest.raises(ValueError):
        rs(torch.zeros(5, 2, 384, device=dev), i32([0, 1, 2, 3, -1], dev))  # more rows than slots
    with pytest.raises(ValueError):
        rs(x, [0, 1], out=torch.zeros(2, 2, 255, device=dev))
    with pytest.raises(ValueError):
        rs(torch.zeros(2, 2, 384 * 24, device=dev), [0, 1])               # a window past shared memory
    with pytest.raises(RuntimeError, match="CUDA"):
        rs(x.cpu(), [0, 1])
    with pytest.raises(ValueError):
        rs.reset([4])
    assert not rs.state.any()


def test_device_rate_chain_through_the_separator(model, dev):
    """A 4 s binaural 48 kHz mixture per listener, three listeners on slots of a five-record state, per 8 ms tick: down
    (keep=64) -> predict(pad=False, slots=) -> up.  Equals the same chain on whole-signal resampling, bit for bit."""
    net, _ = model
    S, slots = 5, [4, 0, 2]
    n, ticks = len(slots), 500
    x48, _ = synth.mixture(n, 384 * ticks, seed0=4100)
    x48 = x48.to(dev)
    e = synth.embedding(n, seed0=4200)[:, 0].to(dev)
    sl = i32(slots, dev)
    down = StreamResampler(48000, 16000, S, 2, 384, keep=64, device=dev)
    up = StreamResampler(16000, 48000, S, 2, 128, device=dev)
    st = net.init_buffers(S, dev)
    got = []
    with torch.no_grad():
        for k in range(ticks):
            chunk = down(x48[:, :, 384 * k:384 * (k + 1)], sl)
            y16, _ = net.predict(chunk, e, st, pad=False, slots=sl)
            got.append(up(y16, sl))
        got = torch.cat(got, -1)
        p = F.pad(resample(x48, 48000, 16000), (down.delay + 64, 0))
        st_ref = net.init_buffers(S, dev)
        y16 = torch.cat([net.predict(p[..., 128 * k:128 * k + 192], e, st_ref, pad=False, slots=sl)[0]
                         for k in range(ticks)], -1)
        want = delayed(y16, 16000, 48000, up.delay)
    assert got.shape == want.shape == (n, 2, 384 * ticks)
    assert want[..., up.delay:].abs().max() > 0
    assert torch.equal(bits(got), bits(want))
