"""Cost of extracting K targets per mixture in one call (l2h_sep_forward_targets) against the duplicated dense call.

    python tools/bench_targets.py [--hops 20] [--out FILE]

Every case is compared with the dense call of the same target rows, each mixture repeated K times (what a caller had to
do before), the two timed alternately in the same process:
  * one hop   (mixtures, K) in {(1, 2), (1, 3), (16, 2), (64, 2), (64, 3), (128, 2)}: one-hop calls as a service runs
              them, fixed staging buffers and every hop a replay of one cached graph (L2H_FLAG_GRAPH); ms per hop,
              median over 5 windows of `--hops` hops
  * offline   32 clips of 4 s, K = 3: Net.forward_targets against Net.forward of the repeated batch; ms per batch,
              median of 5
Every shape is warmed up first (graph capture, gate memos).  The outputs of the two calls are compared on every timed
shape (max relative L2 over the target rows).  Printed as one JSON object with the GPU's name, power limit and max SM
clock, which belong with the numbers.
"""
import argparse

import torch

from bench_common import HOP, LA, L2H_FLAG_GRAPH, alternate, emit, gpu_info, rel_l2, setup_net
from lookoncetohear_b200 import synth

HOP_CASES = [(1, 2), (1, 3), (16, 2), (64, 2), (64, 3), (128, 2)]


def one_hop(net, dev, M, K, reps):
    n = M * K
    x, _ = synth.mixture(M, HOP * (reps + 1), seed0=9000)
    x = torch.nn.functional.pad(x, (0, LA)).to(dev)
    xd = x.repeat_interleave(K, 0)
    e = synth.embedding(n, seed0=9100)[:, 0].contiguous().to(dev)
    xb, xbd = torch.empty(M, 2, HOP + LA, device=dev), torch.empty(n, 2, HOP + LA, device=dev)
    yt, yd = torch.empty(M, K, 2, HOP, device=dev), torch.empty(n, 2, HOP, device=dev)
    ws, _ = net._workspace(dev, n, 1)
    st_t, st_d = net.init_buffers(n, dev), net.init_buffers(n, dev)

    def run_targets(i):
        xb.copy_(x[..., HOP * (i % reps):HOP * (i % reps) + HOP + LA])
        net._launch("targets", xb, e, st_t, yt, 1, L2H_FLAG_GRAPH, K=K, ws=ws)

    def run_dense(i):
        xbd.copy_(xd[..., HOP * (i % reps):HOP * (i % reps) + HOP + LA])
        net._launch("forward", xbd, e, st_d, yd, 1, L2H_FLAG_GRAPH, ws=ws)

    err = 0.0
    for i in range(reps):                      # warm-up from fresh states, in step: the outputs must agree
        run_targets(i)
        run_dense(i)
        err = max(err, rel_l2(yt.reshape(n, 2, HOP), yd))
    torch.cuda.synchronize()
    t_ms, d_ms = alternate({"t": run_targets, "d": run_dense}, reps).values()
    return {"targets_ms": t_ms, "dense_ms": d_ms, "targets_over_dense": t_ms / d_ms, "max_rel_l2": err}


def offline(net, dev, M, K, seconds):
    x, _ = synth.mixture(M, 16000 * seconds, seed0=9200)
    x = x.to(dev)
    emb = synth.embedding(M * K, seed0=9300)[:, 0].view(M, K, 256).to(dev)
    xd, ed = x.repeat_interleave(K, 0), emb.reshape(M * K, 1, 256)
    out = {}

    def run_targets(_):
        out["t"] = net.forward_targets(x, emb)

    def run_dense(_):
        out["d"] = net(xd, ed)

    with torch.no_grad():
        run_targets(0)
        run_dense(0)
        torch.cuda.synchronize()
        err = rel_l2(out["t"].reshape(M * K, 2, -1), out["d"])
        t_ms, d_ms = alternate({"t": run_targets, "d": run_dense}, 1).values()
    return {"targets_ms": t_ms, "dense_ms": d_ms, "targets_over_dense": t_ms / d_ms, "max_rel_l2": err}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hops", type=int, default=20, help="hops per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_targets")
    res = dict(gpu_info(), hops_per_window=args.hops)
    with torch.no_grad():
        for M, K in HOP_CASES:
            res[f"hop_{M}x{K}"] = one_hop(net, dev, M, K, args.hops)
    res["offline_32x3_4s"] = offline(net, dev, 32, 3, 4)
    emit(res, args.out)


if __name__ == "__main__":
    main()
