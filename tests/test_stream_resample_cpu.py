"""Streaming resampling without a GPU: the layout query (l2h_resample_stream_layout) against the formulas of the stream's
definition, the argument errors of l2h_resample_stream, returned before anything touches the device, and the checks of
lookoncetohear_b200.StreamResampler that run before any CUDA call."""
import ctypes
import math

import pytest

import serving_util as su
from serving_util import FAKE_DEV

# orig, new, the delay D in samples at the output rate (one 8 ms block per push)
TABLE = [(48000, 16000, 6), (32000, 16000, 6), (24000, 16000, 6), (8000, 16000, 14),
         (16000, 48000, 21), (16000, 32000, 14), (16000, 24000, 10), (16000, 8000, 6)]


@pytest.fixture(scope="module")
def lib():
    from lookoncetohear_b200 import _cabi, build
    build.build()
    return _cabi.lib()


def formulas(orig, new, block):
    """(H, D, out_block) from the definition: o, q the reduced rates, w = ceil(6 o / (0.99 min(o, q))) taps per side"""
    g = math.gcd(orig, new)
    o, q = orig // g, new // g
    w = math.ceil(6 * o / (0.99 * min(o, q)))
    D = w * q // o
    return -(-D * o // q) + w, D, block * q // o


def layout(lib, orig, new, block, keep=0):
    h, d, ob = ctypes.c_int32(-1), ctypes.c_int32(-1), ctypes.c_int32(-1)
    rc = lib.l2h_resample_stream_layout(orig, new, block, keep, ctypes.byref(h), ctypes.byref(d), ctypes.byref(ob))
    return rc, (h.value, d.value, ob.value)


@pytest.mark.parametrize("orig,new,delay", TABLE)
def test_layout_matches_the_definition(lib, orig, new, delay):
    block = orig * 8 // 1000                                     # one 8 ms push
    rc, got = layout(lib, orig, new, block, keep=64)
    assert rc == 0, lib.l2h_last_error()
    assert got == formulas(orig, new, block)
    assert got[1] == delay
    assert got[2] == new * 8 // 1000
    assert layout(lib, orig, new, 4 * block)[1] == (got[0], got[1], 4 * got[2])   # H and D do not depend on the block


def test_layout_of_the_two_directions_a_48k_device_uses(lib):
    assert layout(lib, 48000, 16000, 384, 64)[1] == (37, 6, 128)
    assert layout(lib, 16000, 48000, 128)[1] == (14, 21, 384)
    assert layout(lib, 48000, 16000, 3)[1] == (37, 6, 1)           # the smallest block: one period


def test_layout_refusals(lib):
    def refused(code, words, *args):
        assert layout(lib, *args)[0] == code, args
        assert words.encode() in lib.l2h_last_error(), lib.l2h_last_error()

    refused(1, "not a positive multiple of 441", 44100, 16000, 352)       # 8 ms at 44.1 kHz is 352.8 samples
    refused(1, "not a positive multiple of 441", 44100, 16000, 353)
    refused(1, "not a positive multiple of 160", 16000, 44100, 128)
    refused(1, "not a positive multiple of 441", 22050, 16000, 176)
    refused(1, "not a positive multiple of 3", 48000, 16000, 385)
    refused(1, "not a positive multiple of 3", 48000, 16000, 0)
    refused(1, "not a positive multiple", 48000, 16000, -384)
    refused(1, "needs no resampling", 16000, 16000, 128)
    refused(1, "rates must be positive", 0, 16000, 128)
    refused(1, "rates must be positive", 48000, -16000, 384)
    refused(1, "keep -1 is negative", 48000, 16000, 384, -1)
    refused(2, "exceed shared memory", 48000, 16000, 384, 12000)         # a keep window too large to stage
    refused(2, "exceed shared memory", 48000, 16000, 384 * 40)           # a block too large to stage
    refused(2, "exceed shared memory", 17600000, 16000, 1100)            # taps reaching too far back
    assert layout(lib, 48000, 16000, 384, 11000)[0] == 0                 # the largest keeps still fit
    null = ctypes.POINTER(ctypes.c_int32)()
    x = ctypes.c_int32()
    assert lib.l2h_resample_stream_layout(48000, 16000, 384, 0, null, ctypes.byref(x), ctypes.byref(x)) == 1
    assert lib.l2h_resample_stream_layout(48000, 16000, 384, 0, ctypes.byref(x), ctypes.byref(x), null) == 1


def _call(lib, n=4, C=2, T=1, slots=FAKE_DEV, state=FAKE_DEV, n_slots=8, orig=48000, new=16000, block=384, keep=64,
          x=FAKE_DEV, y=FAKE_DEV, x_strides=None, y_strides=None):
    """l2h_resample_stream with placeholder device addresses: only for argument sets that must be refused before any
    launch.  Strides default to contiguous [n][C][*] rows."""
    xl, yl = block * T, keep + T * block * new // orig
    xs = x_strides or (C * xl, xl)
    ys = y_strides or (C * yl, yl)
    return lib.l2h_resample_stream(x, xs[0], xs[1], y, ys[0], ys[1], n, C, T, slots, None, state, n_slots, orig, new,
                                   block, keep, None)


def test_stream_call_refusals(lib):
    def refused(code, words, **kw):
        assert _call(lib, **kw) == code, kw
        assert words.encode() in lib.l2h_last_error(), lib.l2h_last_error()

    refused(1, "null pointer", x=None)
    refused(1, "null pointer", y=None)
    refused(1, "null pointer", slots=None)
    refused(1, "null pointer", state=None)
    for kw in ({"n": 0}, {"n": -1}, {"C": 0}, {"T": 0}, {"n_slots": 0}):
        refused(1, "must be positive", **kw)
    refused(1, "n <= n_slots", n=9)
    refused(1, "not a positive multiple of 441", orig=44100, block=352)
    refused(1, "needs no resampling", orig=16000, block=128)
    refused(1, "keep -2 is negative", keep=-2)
    refused(1, "bad stride", x_strides=(2 * 384, 383))                   # channels would overlap
    refused(1, "bad stride", x_strides=(384, 384))                       # rows would overlap
    refused(1, "bad stride", y_strides=(2 * 192, 191))
    refused(1, "bad stride", y_strides=(2 * 191, 192))
    refused(1, "bad stride", T=2, x_strides=(2 * 384, 384))              # x rows hold one block, the call pushes two
    refused(2, "exceed shared memory", T=24)                             # 37 + 24 * 384 + 64 + 24 * 128 floats > 48 KB
    assert b"24 blocks per row" in lib.l2h_last_error()


def test_python_constructor_checks():
    from lookoncetohear_b200 import StreamResampler
    for args in ((48000.5, 16000, 4, 2, 384), (48000, "16k", 4, 2, 384), (48000, 16000, 0, 2, 384),
                 (48000, 16000, 4, 0, 384), (48000, 16000, 4, 2, 0), (48000, 16000, 4, 2, True)):
        with pytest.raises(ValueError):
            StreamResampler(*args)
    with pytest.raises(ValueError, match="keep"):
        StreamResampler(48000, 16000, 4, 2, 384, keep=-1)
    with pytest.raises(ValueError, match="not a positive multiple of 441"):
        StreamResampler(44100, 16000, 4, 2, 352)
    with pytest.raises(ValueError, match="not a positive multiple of 3"):
        StreamResampler(48000, 16000, 4, 2, 128)
    with pytest.raises(ValueError, match="needs no resampling"):
        StreamResampler(16000, 16000, 4, 2, 128)
    with pytest.raises(ValueError, match="shared memory"):
        StreamResampler(48000, 16000, 4, 2, 384, keep=20000)
    with pytest.raises(RuntimeError, match="CUDA"):
        StreamResampler(48000, 16000, 4, 2, 384, keep=64, device="cpu")


def test_header_documents_the_stream_calls():
    hdr = su.header()
    decl, args = su.declaration(hdr, "l2h_resample_stream")
    assert decl, "l2h_resample_stream is not declared"
    assert args == ["x_dev", "x_row_stride", "x_ch_stride", "y_dev", "y_row_stride", "y_ch_stride", "n", "channels", "blocks",
                    "slots_dev", "hops_dev", "state_dev", "n_slots", "orig_freq", "new_freq", "block", "keep", "stream"]
    decl_l, args_l = su.declaration(hdr, "l2h_resample_stream_layout")
    assert args_l == ["orig_freq", "new_freq", "block", "keep", "hist", "delay", "out_block"]
    doc = su.doc_before(hdr, decl_l.start())
    for phrase in ("D = floor(w q / o)", "bit for bit", "outside [0, n_slots)", "h = 0", "All zeros is a fresh stream",
                   "[n_slots][channels][hist + keep]", "44.1 kHz", "CUDA graph"):
        assert phrase in doc, phrase
    assert "#define L2H_ABI_VERSION 1" in hdr
