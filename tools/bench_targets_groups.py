"""Cost of a tick over a list of a targets state's groups (l2h_sep_forward_targets_groups) against the alternatives.

    python tools/bench_targets_groups.py [--hops 20] [--out FILE]

A service keeps one state of G groups of K records (256 records for K = 2, 255 for K = 3) and every tick advances the n
live groups.  Each tick rewrites fixed staging buffers in place (x, embeddings, and the group / slot / hop lists) with a
different seeded subset of groups, and replays one cached graph (L2H_FLAG_GRAPH).  Per case, ms per tick of:
  (a) groups   l2h_sep_forward_targets_groups over the full state
  (b) dense    l2h_sep_forward_targets over a dense state of the n groups (no list: the lower bound of a targets call;
               the same n groups every tick, so their embeddings do not change)
  (c) slots    l2h_sep_forward_slots over the n*K records with each mixture repeated K times (the slot-list way to get
               K targets per listener before the groups call)
for n in 8, 32, 64, 128 (K = 2) and 8, 32, 64 (K = 3), one hop per tick; and one ragged case, T = 4 with a seeded mix of
backlogs, (a) with hops against (c) as l2h_sep_forward_slots_hops.  The cases are timed alternately in one process, every
shape warmed up first, median of 5 windows of `--hops` ticks.  (a) and (c) start from fresh states fed the same ticks;
their outputs are compared during the warm-up (max relative L2 over target rows).  Printed as one JSON object with the
GPU's name, power limit and max SM clock, which belong with the numbers.
"""
import argparse

import torch

from bench_common import HOP, LA, L2H_FLAG_GRAPH, alternate, emit, gpu_info, rel_l2, setup_net
from lookoncetohear_b200 import synth

STATES = {2: 256, 3: 255}                      # records per state: 128 groups of 2, 85 groups of 3
CASES = [(8, 2), (32, 2), (64, 2), (128, 2), (8, 3), (32, 3), (64, 3)]
RAGGED = (32, 2, 4)                            # (n, K, T)
TICKS = 8                                      # distinct precomputed ticks, cycled


def case(net, dev, n, K, T, reps, ragged):
    S = STATES[K]
    G = S // K
    g = torch.Generator().manual_seed(9400 + 10 * n + K)
    subsets = [torch.randperm(G, generator=g)[:n] for _ in range(TICKS)]
    hop_mix = [torch.randint(1 if not ragged else 0, T + 1, (n,), generator=g) for _ in range(TICKS)]
    x_all, _ = synth.mixture(G, HOP * T * 2, seed0=9500)
    x_all = torch.nn.functional.pad(x_all, (0, LA)).to(dev)
    emb_all = synth.embedding(S, seed0=9600)[:, 0].view(G, K, 256).to(dev)
    # per tick: the listed groups' x rows (a, b), the same rows repeated K times (c), their embeddings, the lists
    xa = [x_all[s.to(dev), :, HOP * T * (i % 2):HOP * T * (i % 2 + 1) + LA].contiguous() for i, s in enumerate(subsets)]
    xc = [v.repeat_interleave(K, 0) for v in xa]
    ea = [emb_all[s.to(dev)].reshape(n * K, 256).contiguous() for s in subsets]
    groups = [s.to(torch.int32).to(dev) for s in subsets]
    slots = [(s[:, None] * K + torch.arange(K)[None, :]).flatten().to(torch.int32).to(dev) for s in subsets]
    hops_a = [v.to(torch.int32).to(dev) for v in hop_mix]
    hops_c = [v.repeat_interleave(K).to(torch.int32).to(dev) for v in hop_mix]
    # fixed staging buffers, rewritten in place every tick
    xb, xcb, eb = torch.empty_like(xa[0]), torch.empty_like(xc[0]), torch.empty_like(ea[0])
    gb, slb = torch.empty_like(groups[0]), torch.empty_like(slots[0])
    hab, hcb = torch.empty_like(hops_a[0]), torch.empty_like(hops_c[0])
    ya = torch.empty(n, K, 2, HOP * T, device=dev)
    yb = torch.empty_like(ya)
    yc = torch.empty(n * K, 2, HOP * T, device=dev)
    ws, _ = net._workspace(dev, n * K, T)
    st_a, st_c, st_b = net.init_buffers(S, dev), net.init_buffers(S, dev), net.init_buffers(n * K, dev)

    def run_groups(i):
        j = i % TICKS
        xb.copy_(xa[j]); eb.copy_(ea[j]); gb.copy_(groups[j]); hab.copy_(hops_a[j])
        net._launch("targets_groups", xb, eb, st_a, ya, T, L2H_FLAG_GRAPH, slots=gb, hops=hab if ragged else None, K=K,
                    ws=ws)

    def run_dense(i):          # the dense state's rows are the same n groups every tick: their embeddings stay put
        j = i % TICKS
        xb.copy_(xa[j]); eb.copy_(ea[0])
        net._launch("targets", xb, eb, st_b, yb, T, L2H_FLAG_GRAPH, K=K, ws=ws)

    def run_slots(i):
        j = i % TICKS
        xcb.copy_(xc[j]); eb.copy_(ea[j]); slb.copy_(slots[j]); hcb.copy_(hops_c[j])
        net._launch("slots_hops", xcb, eb, st_c, yc, T, L2H_FLAG_GRAPH, slots=slb, hops=hcb if ragged else None, ws=ws)

    err = 0.0
    for i in range(reps):                      # warm-up (graph capture, gate memos), (a) and (c) in step
        ya.zero_()                             # (samples past a ragged row's hops are not written)
        yc.zero_()
        run_groups(i)
        run_slots(i)
        if not ragged:
            run_dense(i)
        torch.cuda.synchronize()
        err = max(err, rel_l2(ya.reshape(n * K, 2, -1), yc))
    fns = {"groups": run_groups, "slots": run_slots}
    if not ragged:
        fns["dense"] = run_dense
    t = alternate(fns, reps)
    out = {f"{k}_ms": v for k, v in t.items()}
    out.update(groups_over_slots=t["groups"] / t["slots"], max_rel_l2_groups_vs_slots=err)
    if not ragged:
        out["groups_over_dense"] = t["groups"] / t["dense"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hops", type=int, default=20, help="ticks per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_targets_groups")
    res = dict(gpu_info(), ticks_per_window=args.hops)
    with torch.no_grad():
        for n, K in CASES:
            res[f"hop_n{n}_K{K}"] = case(net, dev, n, K, 1, args.hops, False)
        n, K, T = RAGGED
        res[f"ragged_n{n}_K{K}_T{T}"] = case(net, dev, n, K, T, args.hops, True)
    emit(res, args.out)


if __name__ == "__main__":
    main()
