"""Packet streams without a GPU: the layout queries (l2h_resample_packets_layout, l2h_hop_fifo_layout) against the sizes of
their definitions for every rate pair, the argument errors of l2h_resample_packets and l2h_hop_fifo, returned before anything
touches the device, and the checks of lookoncetohear_b200.PacketResampler and HopFifo that run before any CUDA call.  Also
the exact host models of one push through the hop FIFO and the enrollment capture (fifo_push, capture_push), with their
own checks."""
import collections
import ctypes
import math

import numpy as np
import pytest
import torch

import serving_util as su
from serving_util import FAKE_DEV

RATES = [44100, 22050, 11025, 48000, 32000, 24000, 8000]
PAIRS = [(r, 16000) for r in RATES] + [(16000, r) for r in RATES]
# orig, new, w, D: the 44.1 kHz family, which the block streams refuse
TABLE = [(44100, 16000, 17, 6), (16000, 44100, 7, 19), (22050, 16000, 9, 6), (11025, 16000, 7, 10)]


@pytest.fixture(scope="module")
def lib():
    from lookoncetohear_b200 import _cabi, build
    build.build()
    return _cabi.lib()


def rate(orig, new):
    """(o, q, w) of the filter: the rates reduced by their gcd, w = ceil(6 o / (0.99 min(o, q))) taps per side"""
    g = math.gcd(orig, new)
    o, q = orig // g, new // g
    return o, q, math.ceil(6 * o / (0.99 * min(o, q)))


def sizes(orig, new, max_in):
    """(row_floats, D, max_out) from the definition: 2 counter words, then H = ceil((D + 1) o / q) + w + 1 samples"""
    o, q, w = rate(orig, new)
    D = w * q // o
    return 2 + -(-(D + 1) * o // q) + w + 1, D, -(-max_in * q // o)


def layout(lib, orig, new, max_in):
    r, d, m = ctypes.c_int32(-1), ctypes.c_int32(-1), ctypes.c_int32(-1)
    rc = lib.l2h_resample_packets_layout(orig, new, max_in, ctypes.byref(r), ctypes.byref(d), ctypes.byref(m))
    return rc, (r.value, d.value, m.value)


@pytest.mark.parametrize("orig,new", PAIRS)
def test_layout_matches_the_definition(lib, orig, new):
    for max_in in (1, 441, 2 * orig // 100, 1000):
        rc, got = layout(lib, orig, new, max_in)
        assert rc == 0, lib.l2h_last_error()
        assert got == sizes(orig, new, max_in), max_in


@pytest.mark.parametrize("orig,new", PAIRS)
def test_history_covers_every_phase(orig, new):
    """The window a push stages is H history samples and its n new ones.  For every phase p (input count mod o) and push,
    the lowest tap of the first output and the highest tap of the last one lie inside it: the delay D makes every tap of
    an output the stream returns arrive before it is returned."""
    o, q, w = rate(orig, new)
    D = w * q // o
    H = sizes(orig, new, 1)[0] - 2
    for p in range(o):
        j0 = p * q // o
        assert H - p + (j0 - D) * o // q - w >= 0, p
        for n in range(1, 2 * o + 2):
            j1 = (p + n) * q // o
            if j1 > j0:
                assert H - p + (j1 - 1 - D) * o // q + w <= H + n - 1, (p, n)


@pytest.mark.parametrize("orig,new,w,delay", TABLE)
def test_the_44k_family(lib, orig, new, w, delay):
    assert rate(orig, new)[2] == w
    assert layout(lib, orig, new, 882)[1][1] == delay


# ---- host models of the hop FIFO and the enrollment capture ----------------------------------------------------------
# One row of one channel, from a given state row: the head words as Python ints (the int32 words of the state) and a ring
# that is any indexable of floats.  Each returns what the kernel writes: its chunk and hop count, the new head, and the
# ring words written as {ring index: value}.  Python ints cannot overflow, so the models hold at any capacity.
INT32_MAX = 2 ** 31 - 1
FF_HEAD, EC_HEAD, HOP, CARRY = 3, 2, 128, 64


def clamp(w, hi):
    """an int32 head word clamped into [0, hi]"""
    return min(max(w, 0), hi)


def fifo_push(head, ring, x, capacity, T):
    """hop_fifo_kernel for one (row, channel) of a live slot: head (pos, held, dropped), the pushed samples x (empty for
    a count outside [0, max_in]).  Returns (chunk [128 h + 64], h, new head, writes)."""
    R = CARRY + capacity
    pos, held = clamp(head[0], R - 1), clamp(head[1], capacity)
    n = len(x)
    kept = min(n, capacity - held)
    writes = {(pos + held + i) % R: x[i] for i in range(kept)}
    h = min(T, (held + kept) // HOP)
    chunk = [writes.get(k, ring[k]) for k in ((pos + R - CARRY + i) % R for i in range(HOP * h + CARRY))]
    dropped = min(max(head[2], 0) + n - kept, INT32_MAX)
    return chunk, h, ((pos + HOP * h) % R, held + kept - HOP * h, dropped), writes


def capture_push(head, new, capacity):
    """enroll_capture_kernel for one (row, channel) of a live slot with h in [1, T]: head (wpos, captured), the hops'
    new samples `new` (chunk samples 64 .. 64 + 128 h - 1).  Returns (new head, writes): only the last `capacity` samples
    are written."""
    wpos, captured = clamp(head[0], capacity - 1), clamp(head[1], capacity)
    n = len(new)
    writes = {(wpos + i) % capacity: new[i] for i in range(max(0, n - capacity), n)}
    return ((wpos + n) % capacity, min(captured + n, capacity)), writes


def test_fifo_model_is_the_stream_it_was_pushed():
    """pushes that fill, overflow and drain: each chunk is the kept samples after 64 zeros, read at the popped position,
    and the dropped count is everything not kept"""
    rng = np.random.default_rng(11)
    capacity, T = 300, 2
    ring, head = [0.0] * (CARRY + capacity), (0, 0, 0)
    kept_all, pos, dropped = [], 0, 0
    for n in [0, 1, 127, 300, 300, 17, 0, 0, 0, 256, 5, 400]:
        x = rng.standard_normal(n).tolist()
        chunk, h, new_head, writes = fifo_push(head, ring, x, capacity, T)
        kept = min(n, capacity - head[1])
        kept_all += x[:kept]
        dropped += n - kept
        stream = [0.0] * CARRY + kept_all
        assert chunk == stream[pos:pos + HOP * h + CARRY]
        assert h == min(T, (head[1] + kept) // HOP) and new_head[1:] == (head[1] + kept - HOP * h, dropped)
        pos += HOP * h
        for k, v in writes.items():
            ring[k] = v
        head = new_head
    assert dropped > 0 and head[1] < capacity


def test_fifo_model_clamps_and_saturates():
    ring = list(range(CARRY + 200))
    _, h, head, w = fifo_push((10 ** 6, 10 ** 6, INT32_MAX - 3), ring, [1.0] * 9, 200, 5)   # pos, held past their clamps
    assert h == 1 and head == ((CARRY + 199 + HOP) % (CARRY + 200), 200 - HOP, INT32_MAX) and not w
    _, h, head, w = fifo_push((-4, -1, -9), ring, [1.0] * 9, 200, 5)                       # negative words count as 0
    assert h == 0 and head == (0, 9, 0) and sorted(w) == list(range(9))
    cap = 2 ** 30 + 64                                      # the int32 overflow: indices past INT32_MAX, kept in the ring
    R = CARRY + cap
    chunk, h, head, w = fifo_push((R - 1, cap - 100, 0), collections.defaultdict(float), [2.0] * 300, cap, 3)
    assert h == 3 and head == (HOP * 3 - 1, cap - 384, 200) and min(w) == cap - 101 and max(w) == cap - 2
    assert (R - 1) + (cap - 100) > INT32_MAX and 2 * R - 65 > INT32_MAX


def test_capture_model_keeps_the_last_capacity_samples():
    cap = 200
    ring, head = [None] * cap, (0, 0)
    pushed = []
    rng = np.random.default_rng(12)
    for n in (128, 256, 128 * 3, 128):
        new = rng.standard_normal(n).tolist()
        head, w = capture_push(head, new, cap)
        pushed += new
        assert len(w) == min(n, cap)
        for k, v in w.items():
            ring[k] = v
        assert head == (len(pushed) % cap, min(len(pushed), cap))
        k = min(len(pushed), cap)
        assert [ring[(head[0] - k + i) % cap] for i in range(k)] == pushed[-k:]
    assert capture_push((-3, -3), [1.0] * 128, cap)[0] == (128, 128)
    assert capture_push((cap + 5, INT32_MAX), [1.0] * 128, cap)[0] == ((cap - 1 + 128) % cap, cap)


def test_fifo_layout(lib):
    r = ctypes.c_int32(-1)
    for cap in (128, 1000, 4096):
        assert lib.l2h_hop_fifo_layout(cap, ctypes.byref(r)) == 0 and r.value == 3 + 64 + cap
    for cap in (127, 0, -5):
        assert lib.l2h_hop_fifo_layout(cap, ctypes.byref(r)) == 1
        assert b"cannot hold one hop" in lib.l2h_last_error()
    assert lib.l2h_hop_fifo_layout(256, ctypes.POINTER(ctypes.c_int32)()) == 1


def test_layout_refusals(lib):
    def refused(code, words, *args):
        assert layout(lib, *args)[0] == code, args
        assert words.encode() in lib.l2h_last_error(), lib.l2h_last_error()

    refused(1, "needs no resampling", 16000, 16000, 160)
    refused(1, "needs no resampling", 44100, 44100, 441)
    refused(1, "rates must be positive", 0, 16000, 441)
    refused(1, "rates must be positive", 44100, -16000, 441)
    refused(1, "max_in 0 is not positive", 44100, 16000, 0)
    refused(1, "max_in -1 is not positive", 44100, 16000, -1)
    refused(2, "exceed shared memory", 44100, 16000, 12288)              # history + push past 48 KB
    refused(2, "exceed shared memory", 17600000, 16000, 441)             # taps reaching too far back
    assert layout(lib, 44100, 16000, 12288 - 38)[0] == 0                 # the largest push still fits
    null = ctypes.POINTER(ctypes.c_int32)()
    x = ctypes.c_int32()
    assert lib.l2h_resample_packets_layout(44100, 16000, 441, null, ctypes.byref(x), ctypes.byref(x)) == 1
    assert lib.l2h_resample_packets_layout(44100, 16000, 441, ctypes.byref(x), ctypes.byref(x), null) == 1


def _packets(lib, n=4, C=2, max_in=882, counts=FAKE_DEV, unit=1, out_counts=FAKE_DEV, slots=FAKE_DEV, state=FAKE_DEV,
             n_slots=8, orig=44100, new=16000, x=FAKE_DEV, y=FAKE_DEV, x_strides=None, y_strides=None):
    """l2h_resample_packets with placeholder device addresses: only for argument sets that must be refused before any
    launch.  Strides default to contiguous [n][C][*] rows."""
    yl = max(1, -(-max_in * new // orig))
    xs = x_strides or (C * max_in, max_in)
    ys = y_strides or (C * yl, yl)
    return lib.l2h_resample_packets(x, xs[0], xs[1], y, ys[0], ys[1], n, C, max_in, counts, unit, out_counts, slots, state,
                                    n_slots, orig, new, None)


def test_packets_call_refusals(lib):
    def refused(code, words, **kw):
        assert _packets(lib, **kw) == code, kw
        assert words.encode() in lib.l2h_last_error(), lib.l2h_last_error()

    for k in ("x", "y", "counts", "out_counts", "slots", "state"):
        refused(1, "null pointer", **{k: None})
    for kw in ({"n": 0}, {"n": -1}, {"C": 0}, {"unit": 0}, {"unit": -128}, {"n_slots": 0}):
        refused(1, "must be positive", **kw)
    refused(1, "n <= n_slots", n=9)
    refused(1, "needs no resampling", orig=16000)
    refused(1, "max_in 0 is not positive", max_in=0)
    refused(1, "bad stride", x_strides=(2 * 882, 881))                   # channels would overlap
    refused(1, "bad stride", x_strides=(882, 882))                       # rows would overlap
    refused(1, "bad stride", y_strides=(2 * 320, 319))                   # max_out of 882 samples is 320
    refused(1, "bad stride", y_strides=(2 * 319, 320))
    refused(2, "exceed shared memory", max_in=12288)


def _fifo(lib, n=4, C=2, max_in=320, counts=FAKE_DEV, unit=1, hops=FAKE_DEV, T=3, slots=FAKE_DEV, state=FAKE_DEV,
          n_slots=8, capacity=1024, x=FAKE_DEV, chunk=FAKE_DEV, x_strides=None, c_strides=None):
    """l2h_hop_fifo with placeholder device addresses, as _packets"""
    cl = 128 * T + 64
    xs = x_strides or (C * max_in, max_in)
    cs = c_strides or (C * cl, cl)
    return lib.l2h_hop_fifo(x, xs[0], xs[1], max_in, counts, unit, chunk, cs[0], cs[1], hops, n, C, T, slots, state,
                            n_slots, capacity, None)


def test_fifo_call_refusals(lib):
    def refused(code, words, **kw):
        assert _fifo(lib, **kw) == code, kw
        assert words.encode() in lib.l2h_last_error(), lib.l2h_last_error()

    for k in ("x", "counts", "chunk", "hops", "slots", "state"):
        refused(1, "null pointer", **{k: None})
    for kw in ({"n": 0}, {"C": 0}, {"max_in": 0}, {"unit": 0}, {"T": 0}, {"n_slots": -2}):
        refused(1, "must be positive", **kw)
    refused(1, "n <= n_slots", n=9)
    refused(1, "cannot hold one hop", capacity=100)
    refused(1, "bad stride", x_strides=(2 * 320, 319))
    refused(1, "bad stride", x_strides=(320, 320))
    refused(1, "bad stride", c_strides=(2 * 448, 447))                   # a chunk of 3 hops is 448 samples
    refused(1, "bad stride", T=4, c_strides=(2 * 448, 448))


def test_python_constructor_checks():
    from lookoncetohear_b200 import HopFifo, PacketResampler
    for args in ((44100.5, 16000, 4, 2, 441), (44100, "16k", 4, 2, 441), (44100, 16000, 0, 2, 441),
                 (44100, 16000, 4, 0, 441), (44100, 16000, 4, 2, 0), (44100, 16000, 4, 2, True)):
        with pytest.raises(ValueError):
            PacketResampler(*args)
    with pytest.raises(ValueError, match="needs no resampling"):
        PacketResampler(16000, 16000, 4, 2, 160)
    with pytest.raises(ValueError, match="shared memory"):
        PacketResampler(44100, 16000, 4, 2, 20000)
    with pytest.raises(RuntimeError, match="CUDA"):
        PacketResampler(44100, 16000, 4, 2, 882, device="cpu")
    for args in ((0, 2, 3, 1024), (4, 0, 3, 1024), (4, 2, 0, 1024), (4, 2, 3, 2.5), (4, 2, 3, 127)):
        with pytest.raises(ValueError):
            HopFifo(*args)
    with pytest.raises(RuntimeError, match="CUDA"):
        HopFifo(4, 2, 3, 1024, device="cpu")


def test_python_calls_refuse_cpu_tensors():
    from lookoncetohear_b200 import HopFifo, PacketResampler
    pr = PacketResampler.__new__(PacketResampler)       # a state in host memory: the calls refuse before using it
    pr.n_slots, pr.channels, pr.max_in, pr.max_out, pr.orig_freq, pr.new_freq = 4, 2, 882, 320, 44100, 16000
    pr.state = torch.zeros(4, 2, 40)
    fifo = HopFifo.__new__(HopFifo)
    fifo.n_slots, fifo.channels, fifo.frames, fifo.capacity = 4, 2, 3, 1024
    fifo.state = torch.zeros(4, 2, 3 + 64 + 1024)
    with pytest.raises(RuntimeError, match="CUDA"):
        pr(torch.zeros(2, 2, 882), [441, 0], [0, 1])
    with pytest.raises(RuntimeError, match="CUDA"):
        fifo(torch.zeros(2, 2, 320), [160, 0], [0, 1])
    with pytest.raises(RuntimeError, match="CUDA"):
        pr("not a tensor", [441, 0], [0, 1])


def test_header_documents_the_packet_calls():
    hdr = su.header()
    decl, args = su.declaration(hdr, "l2h_resample_packets")
    assert decl, "l2h_resample_packets is not declared"
    assert args == ["x_dev", "x_row_stride", "x_ch_stride", "y_dev", "y_row_stride", "y_ch_stride", "n", "channels",
                    "max_in", "counts_dev", "unit", "out_counts_dev", "slots_dev", "state_dev", "n_slots", "orig_freq",
                    "new_freq", "stream"]
    decl_l, args_l = su.declaration(hdr, "l2h_resample_packets_layout")
    assert args_l == ["orig_freq", "new_freq", "max_in", "row_floats", "delay", "max_out"]
    doc = su.doc_before(hdr, decl_l.start())
    for phrase in ("floor(N q / o)", "bit for bit", "44.1", "10 ms", "All zeros is a fresh stream", "outside [0, n_slots)",
                   "ceil((D + 1) o / q) + w + 1", "CUDA graph"):
        assert phrase in doc, phrase
    decl_f, args_f = su.declaration(hdr, "l2h_hop_fifo")
    assert args_f == ["x_dev", "x_row_stride", "x_ch_stride", "max_in", "counts_dev", "unit", "chunk_dev",
                      "chunk_row_stride", "chunk_ch_stride", "hops_dev", "n", "channels", "frames", "slots_dev",
                      "state_dev", "n_slots", "capacity", "stream"]
    assert su.declaration(hdr, "l2h_hop_fifo_layout")[1] == ["capacity", "row_floats"]
    doc = su.doc_before(hdr, su.declaration(hdr, "l2h_hop_fifo_layout")[0].start())
    for phrase in ("min(frames, floor(held / 128))", "64 zeros", "dropped", "All zeros is an empty FIFO",
                   "l2h_sep_forward_slots_hops", "row_floats = 3 + 64 + capacity"):
        assert phrase in doc, phrase


def test_library_exports_the_packet_calls(lib):
    from lookoncetohear_b200 import _cabi
    for name in ("l2h_resample_packets_layout", "l2h_resample_packets", "l2h_hop_fifo_layout", "l2h_hop_fifo"):
        assert name in _cabi.declared_symbols()
        assert getattr(lib, name) is not None
