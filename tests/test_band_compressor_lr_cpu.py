"""Host-side checks of the band compressor's Linkwitz-Riley bank, no device: the bank's design against an independent
float64 construction from scipy's Butterworth poles; the delays and separations INTEGRATION.md states; the layout; the
argument errors of the three C entries; the header; the Python checks of BandCompressor(bank=...); and a float64 numpy
model of l2h_band_compressor_lr (the reference of tests/test_band_compressor_lr_gpu.py) with its own checks."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch
from scipy.signal import butter, sosfilt

from lookoncetohear_b200 import BandCompressor
from serving_util import declaration, doc_before, header
from test_band_compressor_cpu import EDGES, cuts, detect, end_gains, ramp, set_profile, speech

HOP = 128
BIG = 2.0 ** 32
FS = 16000
ENTRIES = ("l2h_band_compressor_lr_design", "l2h_band_compressor_lr_layout", "l2h_band_compressor_lr")
GRID = np.linspace(1.0, 7999.0, 4000)
MIDS = (250.0, 700.0, 1400.0, 2800.0, 6000.0)           # the band mid frequencies of the FIR bank's separation check
DELAY_AT = (250.0, 1000.0, 2800.0, 6000.0)


# ---- the independent construction ------------------------------------------------------------------------------------
def zpk_resp(z, p, k, f):
    """the response of a digital zpk filter at f Hz"""
    w = np.exp(2j * np.pi * np.asarray(f) / FS)
    return k * np.prod(w[:, None] - np.asarray(z)[None], 1) / np.prod(w[:, None] - np.asarray(p)[None], 1)


def crossover(edge, order):
    """(LP, HP, AP) responses on the grid function of one edge: Butterworth of order / 2 squared, and the allpass on the
    same poles (zeros at the reflected poles 1 / conj(p), gain prod |p| so that it is 1 at DC)"""
    n = order // 2
    lp, hp = butter(n, edge, fs=FS, output="zpk"), butter(n, edge, btype="high", fs=FS, output="zpk")
    p = lp[1]
    ap = (1.0 / np.conj(p), p, float(np.prod(np.abs(p))))
    return (lambda f: zpk_resp(*lp, f) ** 2), (lambda f: zpk_resp(*hp, f) ** 2), (lambda f: zpk_resp(*ap, f))


def tree(edges, order, f):
    """each band's response [K, len(f)] from the independent construction, and the allpass cascade's"""
    xo = [crossover(e, order) for e in edges]
    K = len(edges) + 1
    out = np.ones((K, len(f)), complex)
    for j in range(K):
        for e in range(j):
            out[j] *= xo[e][1](f)
        if j < K - 1:
            out[j] *= xo[j][0](f)
        for e in range(j + 1, K - 1):
            out[j] *= xo[e][2](f)
    ap = np.ones(len(f), complex)
    for e in range(K - 1):
        ap *= xo[e][2](f)
    return out, ap


def sos_resp(sos, f):
    """the response of sections [S, 5] (b0, b1, b2, a1, a2) at f Hz, in float64"""
    sos = np.asarray(sos, np.float64)
    w = np.exp(-2j * np.pi * np.asarray(f) / FS)
    h = np.ones(len(f), complex)
    for b0, b1, b2, a1, a2 in sos:
        h *= (b0 + b1 * w + b2 * w * w) / (1 + a1 * w + a2 * w * w)
    return h


def bank_resp(bank, f):
    return np.stack([sos_resp(bank[b], f) for b in range(len(bank))])


def group_delay_ms(h_of, f, df=0.5):
    ph = np.unwrap(np.angle(np.stack([h_of(np.asarray(f) - df), h_of(np.asarray(f) + df)])), axis=0)
    return -(ph[1] - ph[0]) / (2 * np.pi * 2 * df) * 1000.0


def separation_db(bank):
    """the worst level of a band at another band's mid frequency, relative to its level at its own, as a positive dB"""
    r = 20 * np.log10(np.abs(bank_resp(bank, MIDS)))
    return -max(r[b, o] - r[b, b] for b in range(len(bank)) for o in range(len(bank)) if o != b)


def lr_bank(edges=EDGES, order=4):
    return BandCompressor.design_lr(edges, order).double().numpy()


# ---- the model -------------------------------------------------------------------------------------------------------
def model_state(C, K, S):
    """a fresh slot: the FIR model's head words, then each (channel, band)'s section states [C, K, S, 2]"""
    return {"prof": np.zeros((C, K)), "g": np.zeros((C, K)), "S": np.zeros(K), "knee": np.zeros(K),
            "slope": np.zeros(K), "z": np.zeros((C, K, S, 2))}


def lr_bands(st, x, bank):
    """the band signals [C, K, 128] of a hop, advancing st's section states, and whether every sample is measured"""
    with np.errstate(invalid="ignore"):
        ok = np.abs(x) < BIG
    w = np.where(ok, x, 0.0)
    C, K = st["prof"].shape
    band = np.empty((C, K, HOP))
    for c in range(C):
        for b in range(K):
            if bank.shape[1] == 0:
                band[c, b] = w[c]
                continue
            sos = np.concatenate([bank[b][:, :3], np.ones((bank.shape[1], 1)), bank[b][:, 3:]], 1)
            band[c, b], st["z"][c, b] = sosfilt(sos, w[c], zi=st["z"][c, b])
    return band, bool(ok.all())


def lr_hop_out(band, g0, g1):
    gk = ramp(g0, g1)
    return (np.where(gk == 0, 1.0, 10 ** (gk / 20)) * band).sum(1)


def model_hop(st, x, bank, **kw):
    """l2h_band_compressor_lr on one hop of one slot: x [C, 128] float64 (float32 values), bank [K, S, 5]; returns the
    hop's output and advances st"""
    band, ok = lr_bands(st, x, bank)
    if ok:
        st["S"] = detect(st["S"], band, **kw)[1]
    g0, g1 = st["g"], end_gains(st, st["S"])
    st["g"] = g1
    return lr_hop_out(band, g0, g1)


def model_run(x, ticks, bank, st=None, **kw):
    """x [C, 128 N] through one slot in ticks of the given hop counts: (y, state)"""
    st = st or model_state(x.shape[0], bank.shape[0], bank.shape[1])
    ys, h = [], 0
    for m in ticks:
        for _ in range(m):
            ys.append(model_hop(st, x[:, HOP * h:HOP * (h + 1)], bank, **kw))
            h += 1
    return np.concatenate(ys, 1), st


def allpass_sos(edges, order):
    """the allpass cascade AP_1 .. AP_{K-1} as float64 sections from scipy's poles"""
    out = []
    for e in edges:
        z, p, k = butter(order // 2, e, fs=FS, output="zpk")
        for i in range(0, len(p), 2):
            q = p[i] if p[i].imag > 0 else np.conj(p[i])
            a = [1.0, -2 * q.real, abs(q) ** 2]
            out.append([a[2], a[1], a[0]] + a)
    return np.array(out).reshape(-1, 6)


# ---- the design -------------------------------------------------------------------------------------------------------
DESIGNS = [(EDGES, 4), (EDGES, 8), ((1000.0,), 4), ((1000.0,), 8), ((300.0, 3000.0), 8),
           (tuple(450.0 * (k + 1) for k in range(15)), 4), (tuple(450.0 * (k + 1) for k in range(15)), 8)]


@pytest.mark.parametrize("edges,order", DESIGNS)
def test_design_is_the_linkwitz_riley_tree(edges, order):
    bank = lr_bank(edges, order)
    K = len(edges) + 1
    assert bank.shape == (K, order // 2 * (K - 1), 5)
    want, ap = tree(edges, order, GRID)
    got = bank_resp(bank, GRID)
    assert np.abs(got - want).max() < 1e-5, np.abs(got - want).max()     # fp32 coefficients: 2e-6 to 5e-6
    assert np.abs(np.abs(got.sum(0)) - 1).max() < 1e-5
    assert np.abs(got.sum(0) - ap).max() < 1e-5


def test_design_of_one_band_has_no_sections():
    assert BandCompressor.design_lr((), 4).shape == (1, 0, 5) and BandCompressor.design_lr((), 8).shape == (1, 0, 5)


def integration_row(name):
    """the numbers of INTEGRATION.md's bank table row `name`"""
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "INTEGRATION.md")
    for line in open(path):
        cells = [c.strip() for c in line.strip().strip("|").split("|")]
        if cells and cells[0] == name:
            return [float(re.sub(r"[^0-9.]", "", c)) for c in cells[1:6]]
    raise AssertionError(f"no row {name!r} in INTEGRATION.md")


@pytest.mark.parametrize("order", [4, 8])
def test_documented_delays_and_separation(order):
    """INTEGRATION.md's delays (ms) at 250 Hz, 1 kHz, 2.8 kHz and 6 kHz and worst separation (dB), from the fp32 design"""
    bank = lr_bank(EDGES, order)
    gd = group_delay_ms(lambda f: bank_resp(bank, f).sum(0), DELAY_AT)
    doc = integration_row(f"LR{order}")
    assert np.abs(gd - doc[:4]).max() <= 0.05, (gd, doc)
    assert abs(separation_db(bank) - doc[4]) <= 0.1, (separation_db(bank), doc)


def test_documented_fir_row():
    from test_band_compressor_cpu import BANK
    doc = integration_row("FIR 129 taps")
    assert doc[:4] == [4.0] * 4
    sep = -max(20 * np.log10(abs(np.sum(BANK[b] * np.exp(-2j * np.pi * MIDS[o] / FS * np.arange(129)))))
               - 20 * np.log10(abs(np.sum(BANK[b] * np.exp(-2j * np.pi * MIDS[b] / FS * np.arange(129)))))
               for b in range(5) for o in range(5) if o != b)
    assert abs(sep - doc[4]) <= 0.1, sep


# ---- the model's own checks ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [4, 8])
def test_flat_model_is_the_allpass_cascade(order):
    x = speech(2, 30, 21)
    bank = lr_bank(EDGES, order)
    y, _ = model_run(x, [30], bank)
    want = np.stack([sosfilt(allpass_sos(EDGES, order), x[c]) for c in range(2)])
    assert np.abs(y - want).max() <= 1e-5 * np.abs(x).max()
    one, _ = model_run(x, [30], lr_bank((), order))
    assert np.array_equal(one, x)


def test_model_cut_into_ticks_changes_nothing():
    x = speech(2, 40, 22, db=-6.0)
    bank = lr_bank(EDGES, 4)
    st0 = model_state(2, 5, bank.shape[1])
    set_profile(st0, np.array([[0, 4, 8, 12, 6], [2, 6, 14, 20, 10]]), knees=-45.0, ratios=[1.5, 2, 2, 3, 2])
    runs = [model_run(x, t, bank, st={k: v.copy() for k, v in st0.items()}) for t in ([40], cuts(40, 23), cuts(40, 24))]
    for y, st in runs[1:]:
        assert np.array_equal(y, runs[0][0]) and all(np.array_equal(st[k], runs[0][1][k]) for k in st)
    assert np.abs(runs[0][1]["g"] - runs[0][1]["prof"]).max() > 1              # the compression acted


# ---- the library -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from lookoncetohear_b200 import build, _cabi
    build.build()
    return _cabi.lib()


def test_entries_exported_and_declared(lib):
    from lookoncetohear_b200 import _cabi
    hdr = header()
    for name in ENTRIES:
        assert hasattr(lib, name), name
        assert name in _cabi.declared_symbols(), name
        assert declaration(hdr, name)[0] is not None, name


def test_layout(lib):
    row = ctypes.c_int32(-1)
    for C, K, N in ((1, 1, 4), (2, 5, 4), (2, 5, 8), (2, 16, 8), (8, 5, 4)):
        assert lib.l2h_band_compressor_lr_layout(C, K, N, ctypes.byref(row)) == 0
        assert row.value == 5 * K + 2 * K * (N // 2) * (K - 1), (C, K, N)
    assert lib.l2h_band_compressor_lr_layout(2, 5, 4, None) == 1 and b"null" in lib.l2h_last_error()
    assert lib.l2h_band_compressor_lr_layout(0, 5, 4, ctypes.byref(row)) == 1 and b"channels" in lib.l2h_last_error()
    for K in (0, 17, -1):
        assert lib.l2h_band_compressor_lr_layout(2, K, 4, ctypes.byref(row)) == 1 and b"bands" in lib.l2h_last_error()
    for N in (0, 2, 6, 16, -4):
        assert lib.l2h_band_compressor_lr_layout(2, 5, N, ctypes.byref(row)) == 1 and b"order" in lib.l2h_last_error()
    # 5 K S + 128 C + 130 C K words against 12288
    assert lib.l2h_band_compressor_lr_layout(3, 16, 8, ctypes.byref(row)) == 0
    assert lib.l2h_band_compressor_lr_layout(4, 16, 8, ctypes.byref(row)) == 2 and b"shared memory" in lib.l2h_last_error()
    assert lib.l2h_band_compressor_lr_layout(40, 5, 4, ctypes.byref(row)) == 2


def test_design_argument_errors(lib):
    out = np.zeros(5 * 16 * 5, dtype=np.float32)
    e = (ctypes.c_float * 4)(*EDGES)
    assert lib.l2h_band_compressor_lr_design(5, e, 4, None) == 1 and b"null" in lib.l2h_last_error()
    assert lib.l2h_band_compressor_lr_design(5, None, 4, out.ctypes.data) == 1 and b"null" in lib.l2h_last_error()
    assert lib.l2h_band_compressor_lr_design(1, None, 4, out.ctypes.data) == 0
    for K in (0, 17):
        assert lib.l2h_band_compressor_lr_design(K, e, 4, out.ctypes.data) == 1 and b"bands" in lib.l2h_last_error()
    for N in (2, 6, 0):
        assert lib.l2h_band_compressor_lr_design(5, e, N, out.ctypes.data) == 1 and b"order" in lib.l2h_last_error()
    for bad in ((500.0, 500.0, 2000.0, 4000.0), (1000.0, 500.0, 2000.0, 4000.0), (0.0, 1000.0, 2000.0, 4000.0),
                (500.0, 1000.0, 2000.0, 8000.0), (500.0, float("nan"), 2000.0, 4000.0)):
        eb = (ctypes.c_float * 4)(*bad)
        assert lib.l2h_band_compressor_lr_design(5, eb, 4, out.ctypes.data) == 1 and b"edges" in lib.l2h_last_error()


Y, OUT, SLOTS, SOS, ST = (ctypes.c_void_p(a) for a in (0x1000000, 0x2000000, 0x4000000, 0x5000000, 0x6000000))


def _call(lib, y=Y, y_row=None, y_ch=None, out=OUT, o_row=None, o_ch=None, n=2, C=2, T=3, slots=SLOTS, hops=None,
          sos=SOS, K=5, N=4, st=ST, S=4, attack=0.8, release=0.1):
    y_ch = HOP * T if y_ch is None else y_ch
    o_ch = HOP * T if o_ch is None else o_ch
    y_row = C * y_ch if y_row is None else y_row
    o_row = C * o_ch if o_row is None else o_row
    return lib.l2h_band_compressor_lr(y, y_row, y_ch, out, o_row, o_ch, n, C, T, slots, hops, sos, K, N, st, S,
                                      attack, release, None)


def test_call_argument_errors(lib):
    for kw in ({"y": None}, {"out": None}, {"slots": None}, {"sos": None}, {"st": None}):
        assert _call(lib, **kw) == 1 and b"null" in lib.l2h_last_error(), kw
    for kw in ({"n": 0}, {"C": 0}, {"T": 0}, {"S": 0}, {"n": -1}):
        assert _call(lib, **kw) == 1 and b"positive" in lib.l2h_last_error(), kw
    assert _call(lib, n=5, S=4) == 1 and b"n <= n_slots" in lib.l2h_last_error()
    assert _call(lib, T=2 ** 24, y_ch=2 ** 31, o_ch=2 ** 31) == 1 and b"frames" in lib.l2h_last_error()
    for kw in ({"attack": 0.0}, {"attack": 1.5}, {"release": float("nan")}):
        assert _call(lib, **kw) == 1 and b"attack" in lib.l2h_last_error(), kw
    for K in (0, 17):
        assert _call(lib, K=K) == 1 and b"bands" in lib.l2h_last_error(), K
    for N in (2, 129):
        assert _call(lib, N=N) == 1 and b"order" in lib.l2h_last_error(), N
    for kw in ({"y_ch": 383}, {"o_row": 384}):
        assert _call(lib, **kw) == 1 and b"stride" in lib.l2h_last_error(), kw
    for kw in ({"out": ctypes.c_void_p(0x1000000 + 4)}, {"out": Y, "o_row": 4 * 384}):
        assert _call(lib, **kw) == 1 and b"overlap" in lib.l2h_last_error(), kw
    assert _call(lib, C=4, K=16, N=8, n=1, S=1) == 2 and b"shared memory" in lib.l2h_last_error()


def test_header_documents_the_lr_bank():
    hdr = header()
    _, args = declaration(hdr, "l2h_band_compressor_lr")
    assert args == ["y_dev", "y_row_stride", "y_ch_stride", "out_dev", "out_row_stride", "out_ch_stride", "n", "channels",
                    "frames", "slots_dev", "hops_dev", "sos_dev", "bands", "order", "state_dev", "n_slots", "attack",
                    "release", "stream"]
    assert declaration(hdr, "l2h_band_compressor_lr_layout")[1] == ["channels", "bands", "order", "row_floats"]
    assert declaration(hdr, "l2h_band_compressor_lr_design")[1] == ["bands", "edges_hz", "order", "out"]
    doc = doc_before(hdr, hdr.index("int l2h_band_compressor_lr_design("))
    for phrase in ("Linkwitz-Riley", "scipy.signal.butter", "LP_e + HP_e = AP_e", "allpass", "float64",
                   "transposed direct form II", "identity sections", "There is no bypass", "bit for bit", "not measured",
                   "before anything is enqueued", "CUDA graph", "All zeros is a fresh slot", "stores nothing", "y itself",
                   "5 bands + 2 bands S", "Uploads nothing", "shared memory", "[bands][S][5]"):
        assert phrase in doc, phrase
    assert "l2h_band_compressor_lr" in hdr[:hdr.index("#ifndef")]


# ---- the Python checks -----------------------------------------------------------------------------------------------
def test_constructor_checks():
    for bad in ({"bank": "lr6"}, {"bank": "LR4"}, {"bank": None}, {"bank": "lr4", "taps": 97},
                {"bank": "lr8", "taps": 129.5}, {"bank": "lr4", "edges": (1000, 500)}, {"bank": "lr4", "attack": 0.0}):
        kw = {"slots": 4, "channels": 2, "device": "cuda"}
        kw.update(bad)
        with pytest.raises(ValueError):
            BandCompressor(**kw)
    with pytest.raises(ValueError, match="shared memory"):
        BandCompressor(4, 4, edges=tuple(450.0 * (k + 1) for k in range(15)), bank="lr8", device="cpu")
    for bad in (3, 0, "4", True, 2 ** 40):                     # refused before anything is allocated
        with pytest.raises(ValueError):
            BandCompressor.design_lr(EDGES, bad)


def test_per_hop_quantities(monkeypatch):
    got = {}
    monkeypatch.setattr(BandCompressor, "_allocate",
                        lambda self, row, device: (got.update(row=row), setattr(self, "state", torch.zeros(1))))
    for bank, N in (("lr4", 4), ("lr8", 8)):
        cmp = BandCompressor(4, 2, bank=bank)
        S = N // 2 * 4
        assert got["row"] == 5 * 5 + 2 * 5 * S and cmp.delay == 0 and cmp.bands == 5 and cmp.order == N
        assert cmp.taps.shape == (5, S, 5) and cmp.bank == bank and cmp.edges == EDGES
    one = BandCompressor(4, 1, edges=(), bank="lr4")
    assert (one.bands, one.delay, got["row"]) == (1, 0, 5)
    fir = BandCompressor(4, 2)
    assert fir.bank == "fir" and fir.order is None and fir.delay == 64
