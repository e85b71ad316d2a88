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
import torch

from bench_common import HOP, Tick, alternate, graphed, main, population, warm_up
from lookoncetohear_b200 import Leveler, TargetMixer

K = 2


def case(net, dev, n, T, reps):
    tk = Tick(net, dev, *population(n, K), T)
    y, rec, off, hops = tk.y, tk.rec, tk.off, tk.hops
    mixer = TargetMixer(tk.S, n, 2, device=dev)
    lev = Leveler(tk.S, 2, gate=-120.0, relative=-120.0, settle=0.001, device=dev)
    mix = torch.empty(n, 2, HOP * T, device=dev)

    def back():
        mixer(y, rec, off, tk.slots, hops=hops, chunk=tk.x, out=mix)

    def back_leveled():
        lev(y, rec, off, hops=hops, out=y)
        back()

    plain, leveled = graphed(back), graphed(back_leveled)
    lev_alone = graphed(lambda: lev(y, rec, off, hops=hops, out=y))
    fns = {"tick": lambda i: (tk.rows(i), plain()),
           "tick_leveled": lambda i: (tk.rows(i), leveled()),
           "lev_alone": lambda i: lev_alone()}
    warm_up(fns, reps)
    assert int(lev.state[tk.records.to(dev), 0, 1].view(torch.int32).min()) > 0, "every row is measured"
    t = alternate(fns, reps)
    res = tk.result()
    res.update({f"{k}_ms": v for k, v in t.items()})
    res.update(leveler_share_of_tick=(t["tick_leveled"] - t["tick"]) / t["tick"])
    return res


if __name__ == "__main__":
    main("bench_leveler", case)
