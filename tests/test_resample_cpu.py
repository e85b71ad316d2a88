"""Resampling without a GPU: the float64 restatement (oracle/resample.py) against torchaudio.functional.resample and its
fixture, and the argument checks of l2h_resample / lookoncetohear_b200.resample, which run before any CUDA call."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import resample as ors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAIRS = [(44100, 16000), (48000, 16000), (16000, 8000), (8000, 16000), (22050, 16000)]
LENGTHS = [1, 7, 200, 2000, 80000]


def rel(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


@pytest.mark.parametrize("n", LENGTHS)
@pytest.mark.parametrize("orig,new", PAIRS)
def test_restatement_matches_torchaudio(orig, new, n):
    AF = pytest.importorskip("torchaudio.functional")
    x = np.random.default_rng(orig + n).standard_normal(n)
    y_ta = AF.resample(torch.from_numpy(x), orig, new).numpy()    # float64: torchaudio's filter is built in x's dtype
    y = ors.resample(x, orig, new)
    assert y.shape == y_ta.shape == (ors.output_length(n, orig, new),)
    assert rel(y, y_ta) <= 1e-6


def test_restatement_reproduces_fixture():
    g = np.load(os.path.join(ROOT, "tests", "golden", "resample_golden.npz"))
    xl = np.random.default_rng(int(g["long_seed"])).standard_normal(80000)
    np.testing.assert_allclose([xl.sum(), (xl ** 2).sum()], g["long_checksum"], rtol=1e-12)
    for orig, new in PAIRS:
        for n in LENGTHS[:-1]:
            ref = g[f"y_{orig}_{new}_{n}"]
            y = ors.resample(g[f"x_{n}"], orig, new)
            assert y.shape == ref.shape and rel(y, ref) <= 1e-6, (orig, new, n)
        y = ors.resample(xl, orig, new)
        key = f"y_{orig}_{new}_80000"
        assert y.size == int(g[key + "_len"])
        assert abs(np.linalg.norm(y) / float(g[key + "_norm"]) - 1) <= 1e-6
        assert rel(y[g[key + "_idx"]], g[key + "_val"]) <= 1e-6


def test_restatement_identity_and_lengths():
    x = np.random.default_rng(0).standard_normal((3, 101))
    assert np.array_equal(ors.resample(x, 16000, 16000), x)
    assert ors.resample(x, 44100, 16000).shape == (3, 37)                     # ceil(16000 * 101 / 44100)
    assert ors.output_length(80000, 16000, 8000) == 40000
    assert ors.output_length(1, 8000, 16000) == 2


@pytest.fixture(scope="module")
def lib():
    from lookoncetohear_b200 import _cabi, build
    build.build()
    return _cabi.lib()


def _call(lib, rates, new, n_in=200, cap=None, x_stride=None, y_stride=None, x=16, y=4096):
    """l2h_resample with placeholder device addresses: only for argument sets that must be refused before any launch."""
    arr = (ctypes.c_int32 * len(rates))(*rates)
    cap = 1000 if cap is None else cap
    return lib.l2h_resample(ctypes.c_void_p(x), n_in if x_stride is None else x_stride, n_in, len(rates), arr, new,
                            ctypes.c_void_p(y), cap if y_stride is None else y_stride, cap, None)


def test_abi_refuses_bad_rates(lib):
    assert _call(lib, [0], 16000) == 1 and b"orig_freq 0 is not positive" in lib.l2h_last_error()
    assert _call(lib, [44100, 44100, -16000], 16000) == 1 and b"row 2" in lib.l2h_last_error()
    assert _call(lib, [44100], 0) == 1 and b"new_freq 0" in lib.l2h_last_error()
    assert _call(lib, [44100], -8000) == 1
    # 50x downsampling: the input window of a 256-output tile no longer fits the kernel's shared memory
    assert _call(lib, [44100, 800000], 16000, cap=100000) == 2
    assert b"ratio 50/1 (800000 -> 16000 Hz) is too large" in lib.l2h_last_error()


def test_abi_refuses_small_capacity(lib):
    # 200 samples: 44100 -> 16000 gives ceil(16000 * 200 / 44100) = 73, 8000 -> 16000 gives 400
    assert _call(lib, [44100], 16000, cap=72) == 1 and b"73 output samples, capacity 72" in lib.l2h_last_error()
    assert _call(lib, [44100, 8000], 16000, cap=399) == 1 and b"row 1" in lib.l2h_last_error()
    assert _call(lib, [16000], 16000, cap=199) == 1                          # equal rates need n_in samples too


def test_abi_refuses_bad_sizes(lib):
    assert _call(lib, [44100], 16000, x=0) == 1 and b"bad argument" in lib.l2h_last_error()
    assert _call(lib, [44100], 16000, y=0) == 1
    assert _call(lib, [], 16000) == 1                                          # no rows
    assert _call(lib, [44100], 16000, x_stride=199) == 1                       # rows would overlap
    assert _call(lib, [44100], 16000, y_stride=999) == 1
    assert lib.l2h_resample(ctypes.c_void_p(16), 200, 200, 1, None, 16000, ctypes.c_void_p(4096), 100, 100, None) == 1


def test_python_refuses_other_methods_and_cpu_tensors():
    from lookoncetohear_b200 import resample
    x = torch.zeros(2, 100)
    for kw in ({"resampling_method": "sinc_interp_kaiser"}, {"lowpass_filter_width": 16}, {"rolloff": 0.95}, {"beta": 14.0}):
        with pytest.raises(ValueError, match="only torchaudio's default"):
            resample(x, 44100, 16000, **kw)
    with pytest.raises(ValueError):
        resample(x, 44100, 0)
    with pytest.raises(RuntimeError, match="CUDA"):
        resample(x, 44100, 16000)
