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
import torch

from bench_common import HOP, Tick, alternate, graphed, i32, main, population, warm_up
from lookoncetohear_b200 import TargetMixer

def case(net, dev, n, T, reps):
    tk = Tick(net, dev, *population(n), T)
    y, x, rec, off, slots = tk.y, tk.x, tk.rec, tk.off, tk.slots
    owner = i32([i for i, k in enumerate(tk.ks) for _ in range(k)], dev).long()
    mixer = TargetMixer(tk.S, n, 2, device=dev)
    mixer.set_gains(tk.records.tolist(), 1.0, fade=10 ** 9, start=0.5)
    mixer.set_ambient(list(range(n)), 0.1, fade=10 ** 9, start=0.0)
    out = torch.empty(n, 2, HOP * T, device=dev)
    mix = graphed(lambda: mixer(y, rec, off, slots, chunk=None, out=out))
    mix_amb = graphed(lambda: mixer(y, rec, off, slots, chunk=x, out=out))

    gains = torch.rand(tk.R, generator=tk.g).to(dev)
    amb = torch.full((n, 1, 1), 0.1, device=dev)
    out_t = torch.empty(n, 2, HOP * T, device=dev)

    def compose():
        out_t.zero_()
        out_t.index_add_(0, owner, y * gains[:, None, None])
        out_t.add_(amb * x[..., :HOP * T])
    torch_mix = graphed(compose)

    fns = {"rows": tk.rows,
           "mix": lambda i: (tk.rows(i), mix()),
           "mix_ambient": lambda i: (tk.rows(i), mix_amb()),
           "torch": lambda i: (tk.rows(i), torch_mix()),
           "mix_alone": lambda i: mix_amb()}
    warm_up(fns, reps)
    t = alternate(fns, reps)
    res = tk.result()
    res.update({f"{k}_ms": v for k, v in t.items()})
    res.update(mix_share_of_tick=(t["mix_ambient"] - t["rows"]) / t["rows"],
               torch_share_of_tick=(t["torch"] - t["rows"]) / t["rows"])
    return res


if __name__ == "__main__":
    main("bench_target_mix", case)
