"""Cost of catching up listeners with different backlogs in one ragged call (l2h_sep_forward_slots_hops) against one call
per backlog depth (what a service ran before).

    python tools/bench_ragged_backlog.py [--slots 256] [--reps 20] [--out FILE]

Calls run as a service runs them: fixed staging buffers, every call a replay of a cached graph (L2H_FLAG_GRAPH), the slot
list, the hop counts and the rows' embeddings rewritten in place on the device before every tick (a fresh random list
and a fresh seeded backlog mix over 0 .. T every tick), over a `--slots`-record state.  For n = 4, 16, 64 listed
listeners and the largest backlog T = 2, 4, 8:
    ragged_ms    one T-hop l2h_sep_forward_slots_hops call per tick
    per_depth_ms one l2h_sep_forward_slots_frames call per depth d >= 2 over the rows of that depth, and one
                 l2h_sep_forward_slots call for the rows of depth 1 (rows of depth 0 sit the tick out), each a replay
                 of the graph cached for its (rows, depth): a mix of many depths can need more graphs than the engine
                 keeps (32), and then captures again
    per_depth_direct_ms  the same calls launched directly, without graphs
    per_depth_over_ragged  the faster of the two recipes over ragged_ms
and, with every row T hops behind:
    equal_ragged_ms  the ragged call
    equal_frames_ms  the same call without a hop list (l2h_sep_forward_slots_frames): the cost of reading the hops
The per-depth grouping is precomputed on the host, so per_depth_ms counts only its device work and launches.  Every figure
is the median over 5 windows of `--reps` ticks timed with CUDA events.  Printed as one JSON object with the GPU's name and
power limit, which belong with the numbers.
"""
import argparse
import ctypes
import json
import sys

import torch

from bench_common import HOP, LA, L2H_FLAG_GRAPH, emit, gpu_info, median_ms, setup_net
from lookoncetohear_b200 import synth, _cabi


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=256, help="records in the serving state")
    ap.add_argument("--reps", type=int, default=20, help="ticks per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_ragged_backlog")
    S, R = args.slots, args.reps
    cases = [(n, T) for n in (4, 16, 64) for T in (2, 4, 8) if n <= S]
    L, h = _cabi.lib(), net._engine()

    def ws_bytes(n, T):
        b = ctypes.c_size_t()
        _cabi.check(L.l2h_sep_workspace_bytes(h, n, T, 0, ctypes.byref(b)))
        return b.value

    ws = torch.empty(max(ws_bytes(n, T) for n, T in cases), dtype=torch.uint8, device=dev)
    g = torch.Generator().manual_seed(7300)
    e = synth.embedding(8, seed0=8300)[:, 0].repeat((S + 7) // 8, 1)[:S].contiguous().to(dev)
    big = net.init_buffers(S, dev)
    res = dict(gpu_info(), slots=S, reps_per_window=R, cases={})

    for n, T in cases:
        x = {d: (0.1 * torch.randn(n, 2, HOP * d + LA, generator=g)).to(dev) for d in range(1, T + 1)}
        y = torch.empty(n, 2, HOP * T, device=dev)
        # per tick: the list, the mix, and for the per-depth recipe the rows of every depth
        lists = torch.stack([torch.randperm(S, generator=g)[:n] for _ in range(R)]).to(dev, torch.int32)
        mixes = torch.randint(0, T + 1, (R, n), generator=g, dtype=torch.int32)
        embs = e[lists.long()]
        groups = []
        for i in range(R):
            gi = {}
            for d in range(1, T + 1):
                rows = (mixes[i] == d).nonzero().flatten()
                if len(rows):
                    gi[d] = (lists[i][rows.to(dev)].contiguous(), embs[i][rows.to(dev)].contiguous())
            groups.append(gi)
        mixes = mixes.to(dev)
        slots, hops, ebuf = lists[0].clone(), mixes[0].clone(), embs[0].clone()
        full = torch.full((n,), T, dtype=torch.int32, device=dev)
        dslots = {d: torch.empty(n, dtype=torch.int32, device=dev) for d in range(1, T + 1)}
        debuf = {d: torch.empty(n, 256, device=dev) for d in range(1, T + 1)}

        def call(entry, sl, eb, m, d, flags=L2H_FLAG_GRAPH, hp=None):
            net._launch(entry, x[d][:m], eb, big, y[:m, :, :HOP * d], d, flags, slots=sl, hops=hp, ws=ws)

        def run_ragged(i):
            slots.copy_(lists[i % R])
            hops.copy_(mixes[i % R])
            ebuf.copy_(embs[i % R])
            call("slots_hops", slots, ebuf, n, T, hp=hops)

        def run_per_depth(i, flags=L2H_FLAG_GRAPH):
            for d, (sl, eb) in groups[i % R].items():
                m = sl.shape[0]
                dslots[d][:m].copy_(sl)
                debuf[d][:m].copy_(eb)
                call("slots" if d == 1 else "slots_frames", dslots[d], debuf[d], m, d, flags)

        def run_equal_ragged(i):
            slots.copy_(lists[i % R])
            ebuf.copy_(embs[i % R])
            call("slots_hops", slots, ebuf, n, T, hp=full)

        def run_equal_frames(i):
            slots.copy_(lists[i % R])
            ebuf.copy_(embs[i % R])
            call("slots_frames", slots, ebuf, n, T)

        fns = {"ragged_ms": run_ragged, "per_depth_ms": run_per_depth,
               "per_depth_direct_ms": lambda i: run_per_depth(i, 0), "equal_ragged_ms": run_equal_ragged,
               "equal_frames_ms": run_equal_frames}
        for fn in fns.values():                          # warm: graph captures, every listed slot's gate built
            for i in range(R):
                fn(i)
        torch.cuda.synchronize()
        r = {k: median_ms(fn, R) for k, fn in fns.items()}
        r["per_depth_over_ragged"] = min(r["per_depth_ms"], r["per_depth_direct_ms"]) / r["ragged_ms"]
        r["hops_overhead"] = r["equal_ragged_ms"] / r["equal_frames_ms"] - 1
        r["mean_calls_per_depth_tick"] = sum(len(gi) for gi in groups) / R
        res["cases"][f"n{n}_T{T}"] = r
        print(json.dumps({f"n{n}_T{T}": r}), file=sys.stderr)
    emit(res, args.out)


if __name__ == "__main__":
    main()
