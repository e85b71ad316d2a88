"""Cost of releasing on time: the timed jitter buffer (JitterBuffer(deadline=...), l2h_jitter_buffer_timed) against the
untimed one (l2h_jitter_buffer) on the same 44.1 kHz traffic, alternating in one run.

    python tools/bench_jitter_deadline.py [--reps 20] [--out FILE]

For n = 16, 64, 256 listeners, a state of n slots, every slot listed in every tick (in a seeded order, as a service
running deadlines lists them): each device sends a 441-sample packet every 10 ms, and it reaches the server 2-8 ms
later (seeded), so 8 ms ticks take 0, 1 or 2 packets per slot.  Workloads:
    loss{0,2,10}   seeded loss of 0, 2 or 10 % of the packets
    outage         2 % loss, and every fourth slot loses 8 packets out of every 12 (an 80 ms outage every 120 ms), at
                   staggered phases: in every tick some slots expire packets, start a concealment run (a pitch search)
                   or stall, and restart when their packets return
Each tick is one graph replay: it gathers the tick's slot list, counts, sequence numbers and clock from a device table
of precomputed ticks (the clock rewritten in place), steps a device tick counter, and runs the jitter buffer (depth 1,
window 16, max_out 4; deadline 20 ms for the timed one).  Both buffers replay the same ticks from their own states.
    timed_ms, untimed_ms   the median of 5 windows of `--reps` ticks (CUDA events), the two graphs timed in turn
    added_ms               timed_ms - untimed_ms
    lost, expired, late, restarts   the timed buffer's counters after the run; untimed_lost the untimed one's
Printed as one JSON object with the GPU's name and power limit, which belong with the numbers.
"""
import argparse
import json
import sys

import numpy as np
import torch

from bench_common import LISTENERS, alternate, emit, gpu_info, graphed
from lookoncetohear_b200 import JitterBuffer

PACKET, RATE, M, MAX_OUT, TICK_US, PERIOD_US, DEADLINE_US = 441, 44100, 2, 4, 8000, 10000, 20000


def plan(n, ticks, loss, outage, seed):
    """[ticks, n] slot lists (every slot once) and counts, [ticks, n, M] sequence numbers (-1 padded), [ticks] clock"""
    rng = np.random.default_rng(seed)
    g = torch.Generator().manual_seed(seed)
    lists = [torch.randperm(n, generator=g) for _ in range(ticks)]
    per_tick = [[[] for _ in range(n)] for _ in range(ticks)]
    for s in range(n):
        for k in range(ticks * TICK_US // PERIOD_US + 2):
            if rng.random() < loss or (outage and s % 4 == 0 and (k + s) % 12 < 8):
                continue
            t = -(-(k * PERIOD_US + int(rng.integers(2000, 8001))) // TICK_US)    # the tick that takes it
            if t < ticks:
                per_tick[t][s].append(k & 0xFFFF)
    counts = torch.zeros(ticks, n, dtype=torch.int32)
    seqs = torch.full((ticks, n, M), -1, dtype=torch.int32)
    for t in range(ticks):
        for i, s in enumerate(lists[t].tolist()):
            arr = per_tick[t][s][:M]
            counts[t, i] = len(arr)
            seqs[t, i, :len(arr)] = torch.tensor(arr, dtype=torch.int32)
    clock = torch.tensor([(2 ** 31 - 400000 + t * TICK_US + 2 ** 31) % 2 ** 32 - 2 ** 31 for t in range(ticks)],
                         dtype=torch.int32)                                     # the clock wraps during the run
    return torch.stack(lists).to(torch.int32), counts, seqs, clock


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="ticks per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_jitter_deadline: needs a CUDA device")
    dev = torch.device("cuda", 0)
    R = args.reps
    ticks = 12 * R                                       # warm-up and every timed window replay fresh ticks
    res = dict(gpu_info(), reps_per_window=R, deadline_us=DEADLINE_US, cases={})
    for n in LISTENERS:
        for name, loss, outage in (("loss0", 0.0, False), ("loss2", 0.02, False), ("loss10", 0.10, False),
                                   ("outage", 0.02, True)):
            lists, counts, seqs, clock = plan(n, ticks, loss, outage, 4400 + n + int(1000 * loss) + outage)
            table = torch.cat([lists, counts, seqs.view(ticks, n * M), clock[:, None]], 1).to(dev).contiguous()
            x44 = (0.1 * torch.randn(n, 2, M * PACKET, generator=torch.Generator().manual_seed(n))).to(dev)
            bufs = {k: torch.zeros(1, table.shape[1], dtype=torch.int32, device=dev) for k in ("timed", "untimed")}
            step = {k: torch.zeros(1, dtype=torch.int64, device=dev) for k in bufs}
            jbs = {"timed": JitterBuffer(n, 2, RATE, PACKET, depth=1, window=16, max_out=MAX_OUT, device=dev,
                                         deadline=DEADLINE_US),
                   "untimed": JitterBuffer(n, 2, RATE, PACKET, depth=1, window=16, max_out=MAX_OUT, device=dev)}
            outs = {k: (torch.empty(n, 2, MAX_OUT * PACKET, device=dev), torch.empty(n, dtype=torch.int32, device=dev))
                    for k in bufs}

            def tick(k):
                torch.index_select(table, 0, step[k], out=bufs[k])
                step[k].add_(1)
                step[k].remainder_(ticks)
                v = bufs[k][0]
                slots, cnt, sq = v[:n], v[n:2 * n], v[2 * n:2 * n + n * M].view(n, M)
                now = {"now": v[2 * n + n * M:]} if k == "timed" else {}
                jbs[k](x44, sq, cnt, slots, out=outs[k][0], out_counts=outs[k][1], **now)

            reps = {k: graphed(lambda k=k: tick(k)) for k in bufs}
            fns = {f"{k}_ms": (lambda _, r=r: r()) for k, r in reps.items()}
            for fn in fns.values():                      # warm-up: the graphs' first replays
                for i in range(2 * R):
                    fn(i)
            torch.cuda.synchronize()
            r = alternate(fns, R)
            r["added_ms"] = r["timed_ms"] - r["untimed_ms"]
            jb = jbs["timed"]
            for c in ("lost", "expired", "late", "restarts"):
                r[c] = int(getattr(jb, c).sum())
            r["untimed_lost"] = int(jbs["untimed"].lost.sum())
            res["cases"][f"n{n}_{name}"] = r
            print(json.dumps({f"n{n}_{name}": r}), file=sys.stderr)
    emit(res, args.out)


if __name__ == "__main__":
    main()
