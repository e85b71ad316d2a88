"""Cost of a one-hop step over a list of a state's records, against its capacity and its occupancy.

    python tools/bench_slot_list.py [--slots 256] [--hops 20] [--out FILE]

For n = 16, 32, 64, 128 and 256 live listeners, one-hop steps as a service runs them: fixed staging buffers, every hop
a replay of one cached graph (L2H_FLAG_GRAPH), the per-hop list or mask rewritten in place on the device (a slot-list
step also rewrites the rows' embeddings: each listener keeps its own).  Per n:
  * slots_ms  l2h_sep_forward_slots over n records of a `--slots`-record state, a fresh random list every hop
  * dense_ms  l2h_sep_forward over a state of exactly n streams (what the n listeners cost on their own)
  * mask_ms   l2h_sep_forward_active over the whole `--slots`-record state, n slots active (a fresh random mask every hop)
Each figure is the median over 5 windows of `--hops` hops timed with CUDA events, per hop.  Printed as one JSON object
with the GPU's name and power limit, which belong with the numbers.
"""
import argparse

import torch

from bench_common import HOP, LA, L2H_FLAG_GRAPH, emit, gpu_info, median_ms, setup_net
from lookoncetohear_b200 import synth


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=256, help="records in the serving state")
    ap.add_argument("--hops", type=int, default=20, help="hops per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_slot_list")
    S, K = args.slots, args.hops
    g = torch.Generator().manual_seed(7000)
    x = (0.1 * torch.randn(S, 2, HOP + LA, generator=g)).to(dev)
    e = synth.embedding(8, seed0=8000)[:, 0].repeat((S + 7) // 8, 1)[:S].contiguous().to(dev)
    y = torch.empty(S, 2, HOP, device=dev)
    big = net.init_buffers(S, dev)
    res = dict(gpu_info(), slots=S, hops_per_window=K)

    for n in (m for m in (16, 32, 64, 128, 256) if m <= S):
        ws, _ = net._workspace(dev, S, 1)           # large enough for every n below
        lists = torch.stack([torch.randperm(S, generator=g)[:n] for _ in range(K)]).to(dev, torch.int32)
        masks = torch.zeros(K, S, dtype=torch.uint8)
        for i in range(K):
            masks[i, lists[i].cpu().long()] = 1
        masks = masks.to(dev)
        slots, mask = lists[0].clone(), masks[0].clone()
        # every listener keeps its embedding: the rows of a slot-list call carry those of the hop's listed slots
        embs = e[lists.long()]
        ebuf = embs[0].clone()
        dense = net.init_buffers(n, dev)

        def run_slots(i):
            slots.copy_(lists[i % K])
            ebuf.copy_(embs[i % K])
            net._launch("slots", x[:n], ebuf, big, y[:n], 1, L2H_FLAG_GRAPH, slots=slots, ws=ws)

        def run_dense(i):
            net._launch("forward", x[:n], e, dense, y[:n], 1, L2H_FLAG_GRAPH, ws=ws)

        def run_mask(i):
            mask.copy_(masks[i % K])
            net._launch("forward_active", x, e, big, y, 1, L2H_FLAG_GRAPH, mask=mask, ws=ws)

        for fn in (run_slots, run_dense, run_mask):      # warm: graph capture, every listed slot's gate built
            for i in range(K):
                fn(i)
        torch.cuda.synchronize()
        res[f"n{n}"] = {"slots_ms": median_ms(run_slots, K), "dense_ms": median_ms(run_dense, K),
                        "mask_ms": median_ms(run_mask, K)}
        r = res[f"n{n}"]
        r["slots_over_dense"] = r["slots_ms"] / r["dense_ms"]
        del dense
    emit(res, args.out)


if __name__ == "__main__":
    main()
