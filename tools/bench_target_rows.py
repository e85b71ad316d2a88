"""Cost of a tick over listeners with different numbers of targets (l2h_sep_forward_targets_rows) against the ways to serve
the same population without it.

    python tools/bench_target_rows.py [--hops 20] [--out FILE]

A population of listeners, each with K = 1, 2 or 3 enrolled speakers (64 listeners: 32 x K=1, 24 x K=2, 8 x K=3; and a
quarter of that, 16 listeners: 8 / 6 / 2), advances one hop per tick.  Each tick rewrites fixed staging buffers in place
(x, embeddings and the lists) and replays one cached graph (L2H_FLAG_GRAPH) per call.  Ms per tick of:
  (a) rows     one l2h_sep_forward_targets_rows call over every listener, records scattered over one state
  (b) per-K    one call per K, each on its own state: l2h_sep_forward_slots for the K = 1 listeners,
               l2h_sep_forward_targets_groups for the K = 2 and for the K = 3 listeners
  (c) padded   one l2h_sep_forward_targets_groups call with every listener padded to K = 3 (the extra targets are computed
               for nobody)
The cases are timed alternately in one process, every shape warmed up first, median of 5 windows of `--hops` ticks.  (a)
and (b) start from fresh states fed the same ticks; their outputs are compared during the warm-up (max relative L2 over
target rows: the two choose their kernel forms for different row counts, so they agree up to rounding).  Printed as one JSON
object with the GPU's name, power limit and max SM clock, which belong with the numbers.
"""
import argparse

import torch

from bench_common import HOP, LA, L2H_FLAG_GRAPH, alternate, emit, gpu_info, rel_l2, setup_net
from lookoncetohear_b200 import synth

POPULATIONS = {"n64": {1: 32, 2: 24, 3: 8}, "n16": {1: 8, 2: 6, 3: 2}}     # listeners per K
TICKS = 8                                      # distinct precomputed ticks, cycled


def i32(v, dev):
    return torch.as_tensor(v, dtype=torch.int32).to(dev)


def case(net, dev, pop, reps):
    ks = [k for k in (1, 2, 3) for _ in range(pop[k])]
    n, R = len(ks), sum(ks)
    g = torch.Generator().manual_seed(9700 + n)
    ks = [ks[i] for i in torch.randperm(n, generator=g).tolist()]           # listeners of every K interleaved
    offsets = [0]
    for k in ks:
        offsets.append(offsets[-1] + k)
    S = R + R // 4
    records = torch.randperm(S, generator=g)[:R]
    x_all, _ = synth.mixture(n, HOP * TICKS, seed0=9800)
    x_all = torch.nn.functional.pad(x_all, (0, LA)).to(dev)
    xs = [x_all[..., HOP * t:HOP * (t + 1) + LA].contiguous() for t in range(TICKS)]
    e = synth.embedding(R, seed0=9900)[:, 0].to(dev)
    own = [i for i, k in enumerate(ks) for _ in range(k)]
    by_k = {k: [i for i in range(n) if ks[i] == k] for k in (1, 2, 3)}
    rows_k = {k: [r for r in range(R) if ks[own[r]] == k] for k in (1, 2, 3)}

    # (a) fixed staging buffers, rewritten in place every tick
    xa, ea = torch.empty_like(xs[0]), torch.empty_like(e)
    rec_a, off_a = i32(records, dev), i32(offsets, dev)
    rec_src, off_src = rec_a.clone(), off_a.clone()
    ya = torch.empty(R, 2, HOP, device=dev)
    st_a = net.init_buffers(S, dev)
    ws_a, _ = net._workspace(dev, R, 1)

    def run_rows(i):
        xa.copy_(xs[i % TICKS]); ea.copy_(e); rec_a.copy_(rec_src); off_a.copy_(off_src)
        net._launch("targets_rows", xa, ea, st_a, ya, 1, L2H_FLAG_GRAPH, slots=rec_a, offsets=off_a, ws=ws_a)

    # (b) one state and one call per K
    per_k = {}
    for k in (1, 2, 3):
        m = len(by_k[k])
        xk = [v[by_k[k]].contiguous() for v in xs]
        ek = e[rows_k[k]].contiguous()
        st = net.init_buffers(m * k, dev)
        lst = i32(list(range(m)), dev)
        y = torch.empty(m * k, 2, HOP, device=dev) if k == 1 else torch.empty(m, k, 2, HOP, device=dev)
        per_k[k] = (xk, ek, torch.empty_like(xk[0]), torch.empty_like(ek), st, lst, lst.clone(), y,
                    net._workspace(dev, m * k, 1)[0])

    def run_per_k(i):
        for k, (xk, ek, xb, eb, st, lst, lsrc, y, ws) in per_k.items():
            xb.copy_(xk[i % TICKS]); eb.copy_(ek); lst.copy_(lsrc)
            if k == 1:
                net._launch("slots", xb, eb, st, y, 1, L2H_FLAG_GRAPH, slots=lst, ws=ws)
            else:
                net._launch("targets_groups", xb, eb, st, y, 1, L2H_FLAG_GRAPH, slots=lst, K=k, ws=ws)

    # (c) everyone padded to K = 3: a listener's unused targets reuse its first embedding
    ec = torch.stack([e[offsets[i] + min(j, ks[i] - 1)] for i in range(n) for j in range(3)])
    xc, ecb = torch.empty_like(xs[0]), torch.empty_like(ec)
    gc = i32(list(range(n)), dev)
    gsrc = gc.clone()
    yc = torch.empty(n, 3, 2, HOP, device=dev)
    st_c = net.init_buffers(3 * n, dev)
    ws_c, _ = net._workspace(dev, 3 * n, 1)

    def run_padded(i):
        xc.copy_(xs[i % TICKS]); ecb.copy_(ec); gc.copy_(gsrc)
        net._launch("targets_groups", xc, ecb, st_c, yc, 1, L2H_FLAG_GRAPH, slots=gc, K=3, ws=ws_c)

    err = 0.0
    for i in range(reps):                      # warm-up (graph capture, gate memos), (a) and (b) in step
        run_rows(i)
        run_per_k(i)
        run_padded(i)
        torch.cuda.synchronize()
        for k in (1, 2, 3):
            yk = per_k[k][7].reshape(len(rows_k[k]), 2, HOP)
            err = max(err, rel_l2(ya[rows_k[k]], yk))
    t = alternate({"rows": run_rows, "per_k": run_per_k, "padded": run_padded}, reps)
    out = {"listeners": n, "target_rows": R, "listeners_per_K": {str(k): v for k, v in pop.items()}}
    out.update({f"{k}_ms": v for k, v in t.items()})
    out.update(rows_over_per_k=t["rows"] / t["per_k"], rows_over_padded=t["rows"] / t["padded"],
               max_rel_l2_rows_vs_per_k=err)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hops", type=int, default=20, help="ticks per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_target_rows")
    res = dict(gpu_info(), ticks_per_window=args.hops)
    with torch.no_grad():
        for name, pop in POPULATIONS.items():
            res[name] = case(net, dev, pop, args.hops)
    emit(res, args.out)


if __name__ == "__main__":
    main()
