"""Cost of the per-slot multiband compressor (BandCompressor, l2h_band_compressor) in the 16 kHz side of the multi-voice
tick: the rows tick (l2h_sep_forward_targets_rows), the target mixer, then the compressor in place on the mixer's sum.

    python tools/bench_band_compressor.py [--hops 20] [--out FILE]

Listeners with K = 2 speakers each, at 16, 64 and 256 listeners, records scattered over one state of max(256, 1.25 R)
records, T = 1 and 3 hops per tick, every listener advancing T hops.  The compressor runs at its defaults (five bands,
129 taps), with every slot fitted to a profile of 0 to 15 dB gains and ratio 2 above a -60 dBFS knee, so every hop takes
the filtered path, not the 0 dB bypass.  Each tick rewrites fixed staging buffers in place and replays graphs; ms per
tick of:
  tick             the rows tick (one cached engine graph), then the mixer (one graph)
  tick_compressed  the same with the compressor after the mixer in the second graph
  cmp_alone        a graph of the compressor alone
The cases are timed alternately in one process, every graph warmed up first, median of 5 windows of `--hops` ticks.
Printed as one JSON object with the GPU's name, power limit and max SM clock, which belong with the numbers.
"""
import torch

from bench_common import HOP, Tick, alternate, graphed, main, population, warm_up
from lookoncetohear_b200 import BandCompressor, TargetMixer

K = 2


def case(net, dev, n, T, reps):
    tk = Tick(net, dev, *population(n, K), T)
    slots, hops = tk.slots, tk.hops
    mixer = TargetMixer(tk.S, n, 2, device=dev)
    cmp = BandCompressor(n, 2, device=dev)
    cmp.set_profile(list(range(n)), [0.0, 4.0, 8.0, 15.0, 10.0], knees=-60.0, ratios=2.0)
    mix = torch.empty(n, 2, HOP * T, device=dev)

    def back():
        mixer(tk.y, tk.rec, tk.off, slots, hops=hops, chunk=tk.x, out=mix)

    def back_compressed():
        back()
        cmp(mix, slots, hops=hops, out=mix)

    plain, compressed = graphed(back), graphed(back_compressed)
    cmp_alone = graphed(lambda: cmp(mix, slots, hops=hops, out=mix))
    fns = {"tick": lambda i: (tk.rows(i), plain()),
           "tick_compressed": lambda i: (tk.rows(i), compressed()),
           "cmp_alone": lambda i: cmp_alone()}
    warm_up(fns, reps)
    assert bool((cmp.gain.abs().amax(dim=(1, 2)) > 0).all()), "every slot takes the filtered path"
    t = alternate(fns, reps)
    res = tk.result(bands=cmp.bands, taps=cmp.n_taps)
    res.update({f"{k}_ms": v for k, v in t.items()})
    res.update(compressor_share_of_tick=(t["tick_compressed"] - t["tick"]) / t["tick"])
    return res


if __name__ == "__main__":
    main("bench_band_compressor", case)
