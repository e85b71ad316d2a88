"""Cost of the per-slot multiband compressor (BandCompressor, l2h_band_compressor) in the 16 kHz side of the multi-voice
tick: the rows tick (l2h_sep_forward_targets_rows), the target mixer, then the compressor in place on the mixer's sum.

    python tools/bench_band_compressor.py [--hops 20] [--out FILE]

Listeners with K = 2 speakers each, at 16, 64 and 256 listeners, records scattered over one state of max(256, 1.25 R)
records, T = 1 and 3 hops per tick, every listener advancing T hops.  The compressor runs at its default edges (five
bands) on each of its banks: the FIR bank (129 taps, the default), and the Linkwitz-Riley banks of order 4 and 8, with
every slot fitted to a profile of 0 to 15 dB gains and ratio 2 above a -60 dBFS knee, so every FIR hop takes the
filtered path, not the 0 dB bypass.  Each tick rewrites fixed staging buffers in place and replays graphs; ms per tick
of:
  tick                    the rows tick (one cached engine graph), then the mixer (one graph)
  tick_compressed         the same with the FIR compressor after the mixer in the second graph
  cmp_alone               a graph of the FIR compressor alone
  tick_compressed_<bank>  and cmp_alone_<bank>: the same for each bank, fir, lr4 and lr8
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
    cmps = {}
    for bank in ("fir", "lr4", "lr8"):
        cmps[bank] = BandCompressor(n, 2, device=dev, bank=bank)
        cmps[bank].set_profile(list(range(n)), [0.0, 4.0, 8.0, 15.0, 10.0], knees=-60.0, ratios=2.0)
    mix = torch.empty(n, 2, HOP * T, device=dev)

    def back():
        mixer(tk.y, tk.rec, tk.off, slots, hops=hops, chunk=tk.x, out=mix)

    def compressed(cmp):
        def fn():
            back()
            cmp(mix, slots, hops=hops, out=mix)
        return fn

    plain = graphed(back)
    fns = {"tick": lambda i: (tk.rows(i), plain())}
    for bank, cmp in cmps.items():
        full, alone = graphed(compressed(cmp)), graphed(lambda cmp=cmp: cmp(mix, slots, hops=hops, out=mix))
        fns[f"tick_compressed_{bank}"] = lambda i, full=full: (tk.rows(i), full())
        fns[f"cmp_alone_{bank}"] = lambda i, alone=alone: alone()
    warm_up(fns, reps)
    assert all(bool((c.gain.abs().amax(dim=(1, 2)) > 0).all()) for c in cmps.values()), "every slot's gains move"
    t = alternate(fns, reps)
    t["tick_compressed"], t["cmp_alone"] = t["tick_compressed_fir"], t["cmp_alone_fir"]
    res = tk.result(bands=cmps["fir"].bands, taps=cmps["fir"].n_taps)
    res.update({f"{k}_ms": v for k, v in t.items()})
    res.update(compressor_share_of_tick=(t["tick_compressed"] - t["tick"]) / t["tick"])
    for bank in cmps:
        res[f"added_ms_{bank}"] = t[f"tick_compressed_{bank}"] - t["tick"]
    return res


if __name__ == "__main__":
    main("bench_band_compressor", case)
