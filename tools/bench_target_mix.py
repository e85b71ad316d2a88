"""Cost of mixing each listener's target voices into one row (TargetMixer, l2h_target_mix) on top of a rows tick
(l2h_sep_forward_targets_rows), against the cheapest torch composition of the same sum.

    python tools/bench_target_mix.py [--hops 20] [--out FILE]

Listeners as in tools/bench_target_rows.py: half with K = 1 speaker, three eighths with K = 2, one eighth with K = 3, at
16, 64 and 256 listeners, records scattered over one state of max(256, 1.25 R) records (R target rows), T = 1 and 3 hops
per tick.  Every gain and ambient gain is mid-ramp for the whole run (fades of 10^9 samples), so the mixer computes a
raised cosine per sample and term.  Each tick rewrites fixed staging buffers in place and replays graphs; ms per tick of:
  rows          the rows tick alone (one cached engine graph)
  mix           rows + the mixer, no ambient (one more graph)
  mix_ambient   rows + the mixer with the ambient term
  torch         rows + zero_, index_add_ of the gain-scaled target rows and the gain-scaled ambient add (one graph)
  mix_alone     the mixer's graph alone, with ambient
The cases are timed alternately in one process, every graph warmed up first, median of 5 windows of `--hops` ticks.
Printed as one JSON object with the GPU's name, power limit and max SM clock, which belong with the numbers.
"""
import argparse

import torch

from bench_common import HOP, LA, L2H_FLAG_GRAPH, alternate, emit, gpu_info, graphed, setup_net
from lookoncetohear_b200 import TargetMixer, synth

LISTENERS = (16, 64, 256)
TICKS = 8                                      # distinct precomputed ticks, cycled


def i32(v, dev):
    return torch.as_tensor(v, dtype=torch.int32).to(dev)


def case(net, dev, n, T, reps):
    pop = {1: n // 2, 2: 3 * n // 8, 3: n // 8}
    ks = [k for k in (1, 2, 3) for _ in range(pop[k])]
    R = sum(ks)
    g = torch.Generator().manual_seed(9700 + n)
    ks = [ks[i] for i in torch.randperm(n, generator=g).tolist()]
    offsets = [0]
    for k in ks:
        offsets.append(offsets[-1] + k)
    S = max(256, R + R // 4)
    records = torch.randperm(S, generator=g)[:R]
    x_all, _ = synth.mixture(n, HOP * T * TICKS, seed0=9800)
    x_all = torch.nn.functional.pad(x_all, (0, LA)).to(dev)
    xs = [x_all[..., HOP * T * t:HOP * T * (t + 1) + LA].contiguous() for t in range(TICKS)]
    e = synth.embedding(R, seed0=9900)[:, 0].to(dev)
    owner = i32([i for i, k in enumerate(ks) for _ in range(k)], dev).long()

    x, ea = torch.empty_like(xs[0]), torch.empty_like(e)
    rec, off = i32(records, dev), i32(offsets, dev)
    slots = i32(torch.randperm(n, generator=g), dev)
    y = torch.empty(R, 2, HOP * T, device=dev)
    st = net.init_buffers(S, dev)
    ws, _ = net._workspace(dev, R, T)

    def rows(i):
        x.copy_(xs[i % TICKS]); ea.copy_(e)
        net._launch("targets_rows", x, ea, st, y, T, L2H_FLAG_GRAPH, slots=rec, offsets=off, ws=ws)

    mixer = TargetMixer(S, n, 2, device=dev)
    mixer.set_gains(records.tolist(), 1.0, fade=10 ** 9, start=0.5)
    mixer.set_ambient(list(range(n)), 0.1, fade=10 ** 9, start=0.0)
    out = torch.empty(n, 2, HOP * T, device=dev)
    mix = graphed(lambda: mixer(y, rec, off, slots, chunk=None, out=out))
    mix_amb = graphed(lambda: mixer(y, rec, off, slots, chunk=x, out=out))

    gains = torch.rand(R, generator=g).to(dev)
    amb = torch.full((n, 1, 1), 0.1, device=dev)
    out_t = torch.empty(n, 2, HOP * T, device=dev)

    def compose():
        out_t.zero_()
        out_t.index_add_(0, owner, y * gains[:, None, None])
        out_t.add_(amb * x[..., :HOP * T])
    torch_mix = graphed(compose)

    fns = {"rows": rows,
           "mix": lambda i: (rows(i), mix()),
           "mix_ambient": lambda i: (rows(i), mix_amb()),
           "torch": lambda i: (rows(i), torch_mix()),
           "mix_alone": lambda i: mix_amb()}
    for i in range(reps):                      # warm-up: engine graphs, gate memos, every captured graph
        for f in fns.values():
            f(i)
    torch.cuda.synchronize()
    t = alternate(fns, reps)
    res = {"listeners": n, "target_rows": R, "T": T, "state_records": S}
    res.update({f"{k}_ms": v for k, v in t.items()})
    res.update(mix_share_of_tick=(t["mix_ambient"] - t["rows"]) / t["rows"],
               torch_share_of_tick=(t["torch"] - t["rows"]) / t["rows"])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hops", type=int, default=20, help="ticks per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_target_mix")
    res = dict(gpu_info(), ticks_per_window=args.hops, cases=[])
    with torch.no_grad():
        for T in (1, 3):
            for n in LISTENERS:
                res["cases"].append(case(net, dev, n, T, args.hops))
    emit(res, args.out)


if __name__ == "__main__":
    main()
