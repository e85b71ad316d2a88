"""Band-limited resampling restated from the definition of windowed-sinc interpolation, in float64 numpy.

The checker of `lookoncetohear_b200.resample` / `l2h_resample`.  It states the arithmetic of
`torchaudio.functional.resample(x, orig, new)` at that function's defaults (Hann-windowed sinc, 6 zero crossings on each
side, roll-off 0.99), which is the only form the reference calls (src/datasets/multi_ch_simulator.py:49,
MixLibriSpeechNoisyEnrollNorm.py:69-75).  Pinned to torchaudio by tests/test_resample_cpu.py and
tests/golden/resample_golden.npz.

With the rates reduced by their gcd to o (input samples) and q (output samples) per common period, input sample n sits
at time n / o and output sample m at time m / q (in periods).  The anti-aliasing low-pass has its cutoff at
base = min(o, q) * rolloff cycles per period, so

    y[m] = sum_n x[n] * (base / o) * sinc(u) * cos^2(pi u / (2 * width)),   u = base * (m / q - n / o),

with sinc(u) = sin(pi u) / (pi u), the window zero for |u| >= width, and x zero outside 0 .. len(x) - 1.  The factor
base / o keeps the pass-band gain at one.  The window spans |m o / q - n| < width * o / base input samples.
The output has ceil(q * len(x) / o) samples; equal rates return the input unchanged.
"""
import math

import numpy as np

LOWPASS_FILTER_WIDTH = 6
ROLLOFF = 0.99


def output_length(n, orig, new):
    """Samples out of `n` samples in: ceil(new * n / orig)."""
    return -(-new * n // orig)


def resample(x, orig, new):
    """x [..., n] (anything numpy takes) resampled from rate `orig` to rate `new` along the last axis, float64."""
    x = np.asarray(x, np.float64)
    if orig <= 0 or new <= 0 or int(orig) != orig or int(new) != new:
        raise ValueError(f"rates must be positive integers, got {orig}, {new}")
    if orig == new:
        return x.copy()
    g = math.gcd(int(orig), int(new))
    o, q = int(orig) // g, int(new) // g
    base = min(o, q) * ROLLOFF
    half = math.ceil(LOWPASS_FILTER_WIDTH * o / base)        # input samples on each side of the output's position
    n = x.shape[-1]
    m = np.arange(output_length(n, o, q), dtype=np.int64)
    idx = (m * o // q)[:, None] + np.arange(-half, half + 1, dtype=np.int64)[None, :]
    u = base * (m[:, None] * o - idx * q).astype(np.float64) / (o * q)
    h = np.where(np.abs(u) < LOWPASS_FILTER_WIDTH,
                 np.sinc(u) * np.cos(np.pi * u / (2 * LOWPASS_FILTER_WIDTH)) ** 2, 0.0) * (base / o)
    inside = (idx >= 0) & (idx < n)
    taps = np.where(inside, x[..., np.clip(idx, 0, max(n - 1, 0))], 0.0) if n > 0 else np.zeros(x.shape[:-1] + idx.shape)
    return (taps * h).sum(-1)
