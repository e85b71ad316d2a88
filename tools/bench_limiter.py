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
import torch

from bench_common import HOP, Tick, alternate, graphed, main, population, warm_up
from lookoncetohear_b200 import Limiter, PacketResampler, TargetMixer

def case(net, dev, n, T, reps):
    tk = Tick(net, dev, *population(n), T)
    slots, hops = tk.slots, tk.hops
    mixer = TargetMixer(tk.S, n, 2, device=dev)
    up = PacketResampler(16000, 44100, n, 2, HOP * T, device=dev)
    lim = Limiter(n, 2, 44100, ceiling=1e-3, device=dev)
    mix = torch.empty(n, 2, HOP * T, device=dev)
    y44 = torch.empty(n, 2, up.max_out, device=dev)
    oc44 = torch.empty(n, dtype=torch.int32, device=dev)
    out = torch.empty(n, 2, up.max_out, device=dev)

    def back():
        mixer(tk.y, tk.rec, tk.off, slots, hops=hops, chunk=tk.x, out=mix)
        up(mix, hops, slots, unit=HOP, out=y44, out_counts=oc44)

    def back_limited():
        back()
        lim(y44, oc44, slots, out=out)

    plain, limited = graphed(back), graphed(back_limited)
    lim_alone = graphed(lambda: lim(y44, oc44, slots, out=out))
    fns = {"tick": lambda i: (tk.rows(i), plain()),
           "tick_limited": lambda i: (tk.rows(i), limited()),
           "lim_alone": lambda i: lim_alone()}
    warm_up(fns, reps)
    assert int(lim.limited.min()) > 0, "every slot limits"
    t = alternate(fns, reps)
    res = tk.result(samples_per_row=int(oc44[0]))
    res.update({f"{k}_ms": v for k, v in t.items()})
    res.update(limiter_share_of_tick=(t["tick_limited"] - t["tick"]) / t["tick"])
    return res


if __name__ == "__main__":
    main("bench_limiter", case)
