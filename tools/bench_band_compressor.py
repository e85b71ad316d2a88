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
import argparse

import torch

from bench_common import HOP, LA, L2H_FLAG_GRAPH, alternate, emit, gpu_info, graphed, setup_net
from lookoncetohear_b200 import BandCompressor, TargetMixer, synth

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
    cmp = BandCompressor(n, 2, device=dev)
    cmp.set_profile(list(range(n)), [0.0, 4.0, 8.0, 15.0, 10.0], knees=-60.0, ratios=2.0)
    mix = torch.empty(n, 2, HOP * T, device=dev)

    def back():
        mixer(y, rec, off, slots, hops=hops, chunk=x, out=mix)

    def back_compressed():
        back()
        cmp(mix, slots, hops=hops, out=mix)

    plain, compressed = graphed(back), graphed(back_compressed)
    cmp_alone = graphed(lambda: cmp(mix, slots, hops=hops, out=mix))
    fns = {"tick": lambda i: (rows(i), plain()),
           "tick_compressed": lambda i: (rows(i), compressed()),
           "cmp_alone": lambda i: cmp_alone()}
    for i in range(reps):                      # warm-up: engine graphs, gate memos, every captured graph
        for f in fns.values():
            f(i)
    torch.cuda.synchronize()
    assert bool((cmp.gain.abs().amax(dim=(1, 2)) > 0).all()), "every slot takes the filtered path"
    t = alternate(fns, reps)
    res = {"listeners": n, "target_rows": R, "T": T, "state_records": S, "bands": cmp.bands, "taps": cmp.n_taps}
    res.update({f"{k}_ms": v for k, v in t.items()})
    res.update(compressor_share_of_tick=(t["tick_compressed"] - t["tick"]) / t["tick"])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hops", type=int, default=20, help="ticks per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_band_compressor")
    res = dict(gpu_info(), ticks_per_window=args.hops, cases=[])
    with torch.no_grad():
        for T in (1, 3):
            for n in LISTENERS:
                res["cases"].append(case(net, dev, n, T, args.hops))
    emit(res, args.out)


if __name__ == "__main__":
    main()
