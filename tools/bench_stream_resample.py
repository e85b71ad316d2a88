"""Cost of resampling a tick of listeners whose devices run at 48 kHz: the streaming resampler (l2h_resample_stream,
StreamResampler) against the same tick composed from the whole-signal `resample`, and beside the separator's tick.

    python tools/bench_stream_resample.py [--slots 256] [--reps 20] [--out FILE]

For n = 16, 64, 256 listed listeners of a `--slots`-slot state and T = 1, 4 pushes of 8 ms per row, one tick is: down
48 -> 16 kHz with keep = 64 (the [n, 2, 64 + 128 T] separator input), then up 16 -> 48 kHz of [n, 2, 128 T].
    stream_ms   the two StreamResampler calls
    recipe_ms   the same tick with the whole-signal call, per direction: gather the listed slots' input history, cat the
                new samples, `resample`, slice the final outputs, cat the keep window, scatter history and keep back
    sep_ms      the separator's slot-list call of the same n and T (l2h_sep_forward_slots / _slots_frames), for the
                resampler's share of a tick: stream_share = stream_ms / (stream_ms + sep_ms)
Every tick rewrites the slot list in place (a fresh random list of n), and each figure is one CUDA-graph replay per tick,
timed alternately with the others, every shape warmed up first, the median of 5 windows of `--reps` ticks (CUDA events).
recipe_agrees: the two resamplers, run from fresh states over the same three ticks, give the same bits on the third.
Printed as one JSON object with the GPU's name and power limit, which belong with the numbers.
"""
import argparse
import json
import math
import sys

import torch

from bench_common import HOP, L2H_FLAG_GRAPH, LA, alternate, emit, gpu_info, graphed, setup_net
from lookoncetohear_b200 import StreamResampler, resample, synth


class Recipe:
    """One direction of the tick composed from whole-signal `resample`: per slot the last Hc input samples (Hc >= H, a
    whole number of periods, so the window keeps the stream's phase) and the last `keep` outputs."""

    def __init__(self, rs, S, dev):
        self.rs = rs
        o = rs.orig_freq // math.gcd(rs.orig_freq, rs.new_freq)
        self.hc = -(-rs.hist // o) * o
        self.skip = self.hc * rs.new_freq // rs.orig_freq - rs.delay       # the first final output of the window
        self.hist = torch.zeros(S, rs.channels, self.hc, device=dev)
        self.tail = torch.zeros(S, rs.channels, rs.keep, device=dev)

    def __call__(self, x, idx, out):
        rs = self.rs
        xin = torch.cat([self.hist.index_select(0, idx), x], -1)
        new = resample(xin, rs.orig_freq, rs.new_freq)[..., self.skip:self.skip + x.shape[-1] * rs.new_freq // rs.orig_freq]
        if rs.keep:
            torch.cat([self.tail.index_select(0, idx), new], -1, out=out)
            self.tail.index_copy_(0, idx, out[..., -rs.keep:])
        else:
            out.copy_(new)
        self.hist.index_copy_(0, idx, xin[..., -self.hc:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=256, help="slots in the serving state")
    ap.add_argument("--reps", type=int, default=20, help="ticks per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_stream_resample")
    S, R = args.slots, args.reps
    g = torch.Generator().manual_seed(7700)
    e = synth.embedding(8, seed0=8700)[:, 0].repeat((S + 7) // 8, 1)[:S].contiguous().to(dev)
    big = net.init_buffers(S, dev)
    ws, _ = net._workspace(dev, S, 4)
    res = dict(gpu_info(), slots=S, reps_per_window=R, cases={})

    for n in (m for m in (16, 64, 256) if m <= S):
        for T in (1, 4):
            down = StreamResampler(48000, 16000, S, 2, 384, keep=64, device=dev)
            up = StreamResampler(16000, 48000, S, 2, 128, device=dev)
            rdown, rup = Recipe(down, S, dev), Recipe(up, S, dev)
            x48 = (0.1 * torch.randn(n, 2, 384 * T, generator=g)).to(dev)
            x16 = (0.1 * torch.randn(n, 2, 128 * T, generator=g)).to(dev)
            y16 = {k: torch.empty(n, 2, 64 + 128 * T, device=dev) for k in ("stream", "recipe")}
            y48 = {k: torch.empty(n, 2, 384 * T, device=dev) for k in ("stream", "recipe")}
            lists = torch.stack([torch.randperm(S, generator=g)[:n] for _ in range(R)]).to(dev, torch.int32)
            slots, idx = lists[0].clone(), lists[0].long()
            xs = (0.1 * torch.randn(n, 2, HOP * T + LA, generator=g)).to(dev)
            ys = torch.empty(n, 2, HOP * T, device=dev)
            embs = e[lists.long()]
            ebuf = embs[0].clone()

            def stream():
                down(x48, slots, out=y16["stream"])
                up(x16, slots, out=y48["stream"])

            def recipe():
                rdown(x48, idx, y16["recipe"])
                rup(x16, idx, y48["recipe"])

            # agreement: fresh states, three ticks of one list; the third tick's outputs lie past every stream's start
            for _ in range(3):
                stream()
                recipe()
            agree = all(torch.equal(a["stream"], a["recipe"]) for a in (y16, y48))

            replay_stream, replay_recipe = graphed(stream), graphed(recipe)

            def run_stream(i):
                slots.copy_(lists[i % R])
                replay_stream()

            def run_recipe(i):
                idx.copy_(lists[i % R])
                replay_recipe()

            def run_sep(i):
                slots.copy_(lists[i % R])
                ebuf.copy_(embs[i % R])
                net._launch("slots" if T == 1 else "slots_frames", xs, ebuf, big, ys, T, L2H_FLAG_GRAPH, slots=slots,
                            ws=ws)

            fns = {"stream_ms": run_stream, "recipe_ms": run_recipe, "sep_ms": run_sep}
            for fn in fns.values():                          # warm: every listed slot's gate built, graphs captured
                for i in range(R):
                    fn(i)
            torch.cuda.synchronize()
            r = alternate(fns, R)
            r["recipe_over_stream"] = r["recipe_ms"] / r["stream_ms"]
            r["stream_share"] = r["stream_ms"] / (r["stream_ms"] + r["sep_ms"])
            r["recipe_agrees"] = agree
            res["cases"][f"n{n}_T{T}"] = r
            print(json.dumps({f"n{n}_T{T}": r}), file=sys.stderr)
    emit(res, args.out)


if __name__ == "__main__":
    main()
