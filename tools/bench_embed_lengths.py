"""Enrollment utterances of different lengths: utterances/s on one GPU for
  (a) one call per utterance,  (b) one forward(x, lengths),  (c) the same count at the full 5 s, equal lengths.
256 utterances by default, lengths seeded uniform in 1.5 .. 5 s (16 kHz).  CUDA events, every shape warmed up, median of 5.

    python tools/bench_embed_lengths.py [--n 256] [--reps 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from lookoncetohear_b200 import EmbedTFGridNet, synth  # noqa: E402
from lookoncetohear_b200.configs import EMBED_PARAMS  # noqa: E402
from lookoncetohear_b200.embed import group_by_length  # noqa: E402

SR, HOP = 16000, 64


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def timed(fn, reps):
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    name, q = card()
    print(json.dumps({"device": name, "power_limit_and_max_sm_clock": q}), flush=True)
    torch.manual_seed(0)
    net = EmbedTFGridNet(**EMBED_PARAMS).eval().to(dev)
    g = torch.Generator().manual_seed(5)
    lens = torch.randint(int(1.5 * SR), 5 * SR + 1, (args.n,), generator=g).tolist()
    n_max = 5 * SR
    x = synth.enrollment(args.n, n_max, seed0=9000).to(dev)
    views = [x[i:i + 1, :, :n] for i, n in enumerate(lens)]

    def per_utt():
        for v in views:
            net(v)

    cases = {"a_one_call_per_utterance": per_utt,
             "b_forward_lengths": lambda: net(x, lengths=lens),
             "c_equal_5s": lambda: net(x)}
    frames = [1 + n // HOP for n in lens]
    chunks = group_by_length(lens, net.max_batch) if args.n > net.max_batch(n_max) else [(list(range(args.n)), n_max)]
    padded = sum(len(idx) * (1 + m // HOP) for idx, m in chunks)
    with torch.no_grad():
        for fn in cases.values():             # warm-up: every shape once
            fn()
        torch.cuda.synchronize()
        res = {}
        for k, fn in cases.items():
            ms = timed(fn, args.reps)
            res[k] = ms
            print(json.dumps({"case": k, "utterances": args.n, "ms": round(ms, 1),
                              "utt_per_s": round(args.n / (ms * 1e-3), 1)}), flush=True)
    print(json.dumps({"audio_s": round(sum(lens) / SR, 1), "calls_b": len(chunks),
                      "chunk_sizes_b": [len(i) for i, _ in chunks],
                      "padding_overhead_b": round(padded / sum(frames), 4),
                      "speedup_b_over_a": round(res["a_one_call_per_utterance"] / res["b_forward_lengths"], 2)}), flush=True)


if __name__ == "__main__":
    main()
