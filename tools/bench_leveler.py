"""Cost of the per-row loudness leveler (Leveler, l2h_leveler) in the 16 kHz side of the multi-voice tick: the rows tick
(l2h_sep_forward_targets_rows), then the leveler on the target rows in place, then the target mixer.

    python tools/bench_leveler.py [--hops 20] [--out FILE]

Listeners with K = 2 speakers each, at 16, 64 and 256 listeners, records scattered over one state of max(256, 1.25 R)
records, T = 1 and 3 hops per tick, every listener advancing T hops.  The leveler's gate is -120 LUFS and its settle one
hop, so every row is measured and moves its gain on every hop, the path a row takes while a voice is heard.  Each tick
rewrites fixed staging buffers in place and replays graphs; ms per tick of:
  tick          the rows tick (one cached engine graph), then the mixer (one graph)
  tick_leveled  the same with the leveler before the mixer in the second graph
  lev_alone     a graph of the leveler alone
The cases are timed alternately in one process, every graph warmed up first, median of 5 windows of `--hops` ticks.
Printed as one JSON object with the GPU's name, power limit and max SM clock, which belong with the numbers.
"""
import argparse

import torch

from bench_common import HOP, LA, L2H_FLAG_GRAPH, alternate, emit, gpu_info, graphed, setup_net
from lookoncetohear_b200 import Leveler, TargetMixer, synth

LISTENERS = (16, 64, 256)
K = 2
TICKS = 8                                      # distinct precomputed ticks, cycled


def i32(v, dev):
    return torch.as_tensor(v, dtype=torch.int32).to(dev)


def case(net, dev, n, T, reps):
    R = K * n
    g = torch.Generator().manual_seed(9700 + n)
    offsets = [K * i for i in range(n + 1)]
    S = max(256, R + R // 4)
    records = torch.randperm(S, generator=g)[:R]
    x_all, _ = synth.mixture(n, HOP * T * TICKS, seed0=9800)
    x_all = torch.nn.functional.pad(x_all, (0, LA)).to(dev)
    xs = [x_all[..., HOP * T * t:HOP * T * (t + 1) + LA].contiguous() for t in range(TICKS)]
    e = synth.embedding(R, seed0=9900)[:, 0].to(dev)

    x, ea = torch.empty_like(xs[0]), torch.empty_like(e)
    rec, off = i32(records, dev), i32(offsets, dev)
    slots = i32(torch.randperm(n, generator=g), dev)
    hops = i32([T] * n, dev)
    y = torch.empty(R, 2, HOP * T, device=dev)
    st = net.init_buffers(S, dev)
    ws, _ = net._workspace(dev, R, T)

    def rows(i):
        x.copy_(xs[i % TICKS]); ea.copy_(e)
        net._launch("targets_rows", x, ea, st, y, T, L2H_FLAG_GRAPH, slots=rec, offsets=off, ws=ws)

    mixer = TargetMixer(S, n, 2, device=dev)
    lev = Leveler(S, 2, gate=-120.0, relative=-120.0, settle=0.001, device=dev)
    mix = torch.empty(n, 2, HOP * T, device=dev)

    def back():
        mixer(y, rec, off, slots, hops=hops, chunk=x, out=mix)

    def back_leveled():
        lev(y, rec, off, hops=hops, out=y)
        back()

    plain, leveled = graphed(back), graphed(back_leveled)
    lev_alone = graphed(lambda: lev(y, rec, off, hops=hops, out=y))
    fns = {"tick": lambda i: (rows(i), plain()),
           "tick_leveled": lambda i: (rows(i), leveled()),
           "lev_alone": lambda i: lev_alone()}
    for i in range(reps):                      # warm-up: engine graphs, gate memos, every captured graph
        for f in fns.values():
            f(i)
    torch.cuda.synchronize()
    assert int(lev.state[records.to(dev), 0, 1].view(torch.int32).min()) > 0, "every row is measured"
    t = alternate(fns, reps)
    res = {"listeners": n, "target_rows": R, "T": T, "state_records": S}
    res.update({f"{k}_ms": v for k, v in t.items()})
    res.update(leveler_share_of_tick=(t["tick_leveled"] - t["tick"]) / t["tick"])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hops", type=int, default=20, help="ticks per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_leveler")
    res = dict(gpu_info(), ticks_per_window=args.hops, cases=[])
    with torch.no_grad():
        for T in (1, 3):
            for n in LISTENERS:
                res["cases"].append(case(net, dev, n, T, args.hops))
    emit(res, args.out)


if __name__ == "__main__":
    main()
