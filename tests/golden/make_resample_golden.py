"""Generate tests/golden/resample_golden.npz from torchaudio itself, for machines where torchaudio does not import:

    python tests/golden/make_resample_golden.py

`torchaudio.functional.resample(x, orig, new)` at its defaults (the reference's only form) on seeded white noise, in
float64 (torchaudio builds its filter in the input's dtype; in float32 that filter alone is ~1e-5 off for 44100 Hz).
Lengths up to 2 000 are stored whole; the 80 000-sample input is re-created from its seed (checksum stored to detect RNG
drift) and its outputs stored as a fixed seeded sample of 512 values plus the L2 norm and the length.
"""
import os

import numpy as np
import torch
import torchaudio.functional as AF

HERE = os.path.dirname(os.path.abspath(__file__))
PAIRS = [(44100, 16000), (48000, 16000), (16000, 8000), (8000, 16000), (22050, 16000)]
SHORT = [1, 7, 200, 2000]
LONG, LONG_SEED, SAMPLES = 80000, 80000, 512


def long_input():
    return np.random.default_rng(LONG_SEED).standard_normal(LONG)


def main():
    out = {"long_seed": np.int64(LONG_SEED)}
    xl = long_input()
    out["long_checksum"] = np.array([xl.sum(), (xl ** 2).sum()])
    for n in SHORT:
        out[f"x_{n}"] = np.random.default_rng(n).standard_normal(n)
    for o, q in PAIRS:
        for n in SHORT:
            out[f"y_{o}_{q}_{n}"] = AF.resample(torch.from_numpy(out[f"x_{n}"]), o, q).numpy()
        y = AF.resample(torch.from_numpy(xl), o, q).numpy()
        idx = np.sort(np.random.default_rng(o + q).choice(y.size, SAMPLES, replace=False))
        out[f"y_{o}_{q}_{LONG}_idx"] = idx.astype(np.int32)
        out[f"y_{o}_{q}_{LONG}_val"] = y[idx]
        out[f"y_{o}_{q}_{LONG}_norm"] = np.float64(np.linalg.norm(y))
        out[f"y_{o}_{q}_{LONG}_len"] = np.int64(y.size)
    np.savez_compressed(os.path.join(HERE, "resample_golden.npz"), **out)


if __name__ == "__main__":
    main()
