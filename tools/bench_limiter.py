"""Cost of the per-listener look-ahead limiter (Limiter, l2h_limiter) in the output side of the 44.1 kHz tick: the rows
tick (l2h_sep_forward_targets_rows), the target mixer, the up-resampler to 44.1 kHz, then the limiter on what it returns.

    python tools/bench_limiter.py [--hops 20] [--out FILE]

Listeners as in tools/bench_target_mix.py: half with K = 1 speaker, three eighths with K = 2, one eighth with K = 3, at 16,
64 and 256 listeners, records scattered over one state of max(256, 1.25 R) records, T = 1 and 3 hops per tick, every
listener advancing T hops.  The limiter's ceiling is 0.001 (-60 dBFS), so every slot limits every sample and the gain
path is always taken.  Each tick rewrites fixed staging buffers in place and replays graphs; ms per tick of:
  tick          the rows tick (one cached engine graph), then the mixer and the up-resampler (one graph)
  tick_limited  the same with the limiter in the second graph
  lim_alone     a graph of the limiter alone
The cases are timed alternately in one process, every graph warmed up first, median of 5 windows of `--hops` ticks.
Printed as one JSON object with the GPU's name, power limit and max SM clock, which belong with the numbers.
"""
import argparse

import torch

from bench_common import HOP, LA, L2H_FLAG_GRAPH, alternate, emit, gpu_info, graphed, setup_net
from lookoncetohear_b200 import Limiter, PacketResampler, TargetMixer, synth

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
    up = PacketResampler(16000, 44100, n, 2, HOP * T, device=dev)
    lim = Limiter(n, 2, 44100, ceiling=1e-3, device=dev)
    mix = torch.empty(n, 2, HOP * T, device=dev)
    y44 = torch.empty(n, 2, up.max_out, device=dev)
    oc44 = torch.empty(n, dtype=torch.int32, device=dev)
    out = torch.empty(n, 2, up.max_out, device=dev)

    def back():
        mixer(y, rec, off, slots, hops=hops, chunk=x, out=mix)
        up(mix, hops, slots, unit=HOP, out=y44, out_counts=oc44)

    def back_limited():
        back()
        lim(y44, oc44, slots, out=out)

    plain, limited = graphed(back), graphed(back_limited)
    lim_alone = graphed(lambda: lim(y44, oc44, slots, out=out))
    fns = {"tick": lambda i: (rows(i), plain()),
           "tick_limited": lambda i: (rows(i), limited()),
           "lim_alone": lambda i: lim_alone()}
    for i in range(reps):                      # warm-up: engine graphs, gate memos, every captured graph
        for f in fns.values():
            f(i)
    torch.cuda.synchronize()
    assert int(lim.limited.min()) > 0, "every slot limits"
    t = alternate(fns, reps)
    res = {"listeners": n, "target_rows": R, "T": T, "state_records": S, "samples_per_row": int(oc44[0])}
    res.update({f"{k}_ms": v for k, v in t.items()})
    res.update(limiter_share_of_tick=(t["tick_limited"] - t["tick"]) / t["tick"])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hops", type=int, default=20, help="ticks per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_limiter")
    res = dict(gpu_info(), ticks_per_window=args.hops, cases=[])
    with torch.no_grad():
        for T in (1, 3):
            for n in LISTENERS:
                res["cases"].append(case(net, dev, n, T, args.hops))
    emit(res, args.out)


if __name__ == "__main__":
    main()
