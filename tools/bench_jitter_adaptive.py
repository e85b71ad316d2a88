"""Cost of adaptive deadlines: the adaptive jitter buffer (JitterBuffer(deadline=(lo, hi)), l2h_jitter_buffer_adaptive,
with arrival times) against the timed one at a fixed 20 ms (l2h_jitter_buffer_timed) on the same 44.1 kHz traffic,
alternating in one run.

    python tools/bench_jitter_adaptive.py [--reps 20] [--out FILE]

For n = 16, 64, 256 listeners, a state of n slots, every slot listed in every tick (in a seeded order): each device
sends a 441-sample packet every 10 ms, and 8 ms ticks take the packets that arrived since the last one, each with its
arrival time.  Workloads:
    mixed    even slots on a good link (2-4 ms after sending), odd slots on a bad one (2-32 ms, uniform); 1 % loss
    outage   2 % loss and 2-8 ms of latency, and every fourth slot loses 8 packets out of every 12 (an 80 ms outage
             every 120 ms), at staggered phases, as tools/bench_jitter_deadline.py runs it
Each tick is one graph replay: it gathers the tick's slot list, counts, sequence numbers, clock and arrival times from a
device table of precomputed ticks, steps a device tick counter, and runs the jitter buffer (depth 1, window 16, max_out
6; the adaptive one with lo 0, hi 60 ms, late_rate 0.02).  Both buffers replay the same ticks from their own states.
    adaptive_ms, timed_ms   the median of 5 windows of `--reps` ticks (CUDA events), the two graphs timed in turn
    added_ms                adaptive_ms - timed_ms
    per link class (good / bad slots; all slots for outage), for each buffer after the run: late, expired, and for the
    adaptive one the mean deadline_us over the slots
Printed as one JSON object with the GPU's name and power limit, which belong with the numbers.
"""
import argparse
import json
import sys

import numpy as np
import torch

from bench_common import LISTENERS, alternate, emit, gpu_info, graphed
from lookoncetohear_b200 import JitterBuffer

PACKET, RATE, M, MAX_OUT, TICK_US, PERIOD_US = 441, 44100, 6, 6, 8000, 10000
DEADLINE_US, LO_US, HI_US, LATE_RATE = 20000, 0, 60000, 0.02
T0 = 2 ** 31 - 400000                                   # the clock wraps during the run


def plan(n, ticks, workload, seed):
    """[ticks, n] slot lists (every slot once) and counts, [ticks, n, M] sequence numbers (-1 padded) and arrival times,
    [ticks] clock"""
    rng = np.random.default_rng(seed)
    g = torch.Generator().manual_seed(seed)
    lists = [torch.randperm(n, generator=g) for _ in range(ticks)]
    per_tick = [[[] for _ in range(n)] for _ in range(ticks)]
    for s in range(n):
        for k in range(ticks * TICK_US // PERIOD_US + 4):
            if workload == "mixed":
                if rng.random() < 0.01:
                    continue
                lat = int(rng.integers(2000, 4001)) if s % 2 == 0 else int(rng.integers(2000, 32001))
            else:
                if rng.random() < 0.02 or (s % 4 == 0 and (k + s) % 12 < 8):
                    continue
                lat = int(rng.integers(2000, 8001))
            t = k * PERIOD_US + lat
            tick = -(-t // TICK_US)                                          # the tick that takes it
            if tick < ticks:
                per_tick[tick][s].append((t, k & 0xFFFF))
    counts = torch.zeros(ticks, n, dtype=torch.int32)
    seqs = torch.full((ticks, n, M), -1, dtype=torch.int32)
    arrivals = torch.zeros(ticks, n, M, dtype=torch.int64)
    for t in range(ticks):
        for i, s in enumerate(lists[t].tolist()):
            arr = sorted(per_tick[t][s])[:M]
            counts[t, i] = len(arr)
            seqs[t, i, :len(arr)] = torch.tensor([q for _, q in arr], dtype=torch.int32)
            arrivals[t, i, :len(arr)] = torch.tensor([T0 + a for a, _ in arr], dtype=torch.int64)
    wrap = lambda v: (v + 2 ** 31) % 2 ** 32 - 2 ** 31                       # noqa: E731
    clock = wrap(torch.tensor([T0 + t * TICK_US for t in range(ticks)], dtype=torch.int64)).to(torch.int32)
    return torch.stack(lists).to(torch.int32), counts, seqs, wrap(arrivals).to(torch.int32), clock


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="ticks per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_jitter_adaptive: needs a CUDA device")
    dev = torch.device("cuda", 0)
    R = args.reps
    ticks = 12 * R                                       # warm-up and every timed window replay fresh ticks
    res = dict(gpu_info(), reps_per_window=R, deadline_us=DEADLINE_US, lo_us=LO_US, hi_us=HI_US, late_rate=LATE_RATE,
               cases={})
    for n in LISTENERS:
        for workload in ("mixed", "outage"):
            lists, counts, seqs, arrivals, clock = plan(n, ticks, workload, 5500 + n + (workload == "outage"))
            table = torch.cat([lists, counts, seqs.view(ticks, n * M), clock[:, None], arrivals.view(ticks, n * M)],
                              1).to(dev).contiguous()
            x44 = (0.1 * torch.randn(n, 2, M * PACKET, generator=torch.Generator().manual_seed(n))).to(dev)
            bufs = {k: torch.zeros(1, table.shape[1], dtype=torch.int32, device=dev) for k in ("adaptive", "timed")}
            step = {k: torch.zeros(1, dtype=torch.int64, device=dev) for k in bufs}
            kw = dict(depth=1, window=16, max_out=MAX_OUT, device=dev)
            jbs = {"adaptive": JitterBuffer(n, 2, RATE, PACKET, deadline=(LO_US, HI_US), late_rate=LATE_RATE, **kw),
                   "timed": JitterBuffer(n, 2, RATE, PACKET, deadline=DEADLINE_US, **kw)}
            outs = {k: (torch.empty(n, 2, MAX_OUT * PACKET, device=dev), torch.empty(n, dtype=torch.int32, device=dev))
                    for k in bufs}

            def tick(k):
                torch.index_select(table, 0, step[k], out=bufs[k])
                step[k].add_(1)
                step[k].remainder_(ticks)
                v = bufs[k][0]
                o = 2 * n + n * M
                slots, cnt, sq, now = v[:n], v[n:2 * n], v[2 * n:o].view(n, M), v[o:o + 1]
                extra = {"arrivals": v[o + 1:].view(n, M)} if k == "adaptive" else {}
                jbs[k](x44, sq, cnt, slots, out=outs[k][0], out_counts=outs[k][1], now=now, **extra)

            reps = {k: graphed(lambda k=k: tick(k)) for k in bufs}
            fns = {f"{k}_ms": (lambda _, r=r: r()) for k, r in reps.items()}
            for fn in fns.values():                      # warm-up: the graphs' first replays
                for i in range(2 * R):
                    fn(i)
            torch.cuda.synchronize()
            r = alternate(fns, R)
            r["added_ms"] = r["adaptive_ms"] - r["timed_ms"]
            classes = {"good": list(range(0, n, 2)), "bad": list(range(1, n, 2))} if workload == "mixed" else \
                {"all": list(range(n))}
            for c, idx in classes.items():
                for k, jb in jbs.items():
                    r[f"{c}_{k}_late"] = int(jb.late[idx].sum())
                    r[f"{c}_{k}_expired"] = int(jb.expired[idx].sum())
                r[f"{c}_adaptive_mean_deadline_us"] = float(jbs["adaptive"].deadline_us[idx].double().mean())
            res["cases"][f"n{n}_{workload}"] = r
            print(json.dumps({f"n{n}_{workload}": r}), file=sys.stderr)
    emit(res, args.out)


if __name__ == "__main__":
    main()
