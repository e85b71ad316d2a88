"""Cost of the jitter buffer (JitterBuffer, l2h_jitter_buffer) at the head of a tick of listeners at 44.1 kHz that send
10 ms packets over a lossy network: the graph jb -> down -> FIFO against the same graph without the jitter buffer, beside
the separator's tick.

    python tools/bench_jitter_buffer.py [--slots 256] [--reps 20] [--out FILE]

The tick set-up of tools/bench_packet_ticks.py: for n = 16, 64, 256 listed listeners of a `--slots`-slot state, every
tick each listener sends 0, 1 or 2 packets of 441 samples (seeded jitter, probabilities 0.3, 0.6, 0.1), and the FIFO
pops up to T = 3 hops.  Each slot's packets carry sequence numbers with seeded loss (0, 2 or 10 %) and one packet in 20
swapped with its neighbour; every tick rewrites the slot list, the counts and the sequence numbers in place.
    with_ms     one graph replay: jb (depth 1, window 16, max_out 4) -> down 44.1 -> 16 kHz -> l2h_hop_fifo
    without_ms  the same graph without the jitter buffer (the packets go straight to down)
    added_ms    with_ms - without_ms
    worst_ms    a graph of the jitter buffer alone where every listed slot starts a loss run in every call (depth 0,
                each row sends next + 1: one concealed packet, one pitch search and one recovery fade per row); every
                slot is started before timing, so every listed row conceals
    lists_ms    a graph of the list gather alone; worst_jb_ms = worst_ms - lists_ms
    sep_ms      the separator's slot-list call over the same lists (l2h_sep_forward_slots_hops), for the shares
                added_share = added_ms / sep_ms and worst_share = worst_jb_ms / sep_ms
Each graph starts by gathering its tick's slot list, counts and sequence numbers from a device table of precomputed
ticks (one gather and a step of a device tick counter, the same three small kernels in every graph), so a timed tick is
one graph replay with no eager work around it, and no tick repeats.  The graphs are timed alternately, the median of 5
windows of `--reps` ticks (CUDA events), every graph warmed up first.  lost, late and worst_lost are the counters after
the run (worst_lost counts one per listed row and tick).
Printed as one JSON object with the GPU's name and power limit, which belong with the numbers.
"""
import argparse
import json
import sys

import numpy as np
import torch

from bench_common import L2H_FLAG_GRAPH, alternate, emit, gpu_info, graphed, setup_net
from lookoncetohear_b200 import HopFifo, JitterBuffer, PacketResampler, synth

T, CAP, PACKET, M, MAX_OUT = 3, 1024, 441, 2, 4


def arrivals(n, loss, g):
    """the arrival order of a slot's first n packets: seeded losses, one in 20 swapped with its neighbour"""
    seq = [k for k in range(n) if g.random() >= loss]
    for k in range(0, len(seq) - 1):
        if g.random() < 0.05:
            seq[k], seq[k + 1] = seq[k + 1], seq[k]
    return seq


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=256, help="slots in the serving state")
    ap.add_argument("--reps", type=int, default=20, help="ticks per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_jitter_buffer")
    S, R = args.slots, args.reps
    ticks = 8 * R                                        # every tick of the warm-up and the timed windows is fresh
    e = synth.embedding(8, seed0=8800)[:, 0].repeat((S + 7) // 8, 1)[:S].contiguous().to(dev)
    big = net.init_buffers(S, dev)
    ws, _ = net._workspace(dev, S, T)
    res = dict(gpu_info(), slots=S, reps_per_window=R, frames=T, cases={})

    for n in (m for m in (16, 64, 256) if m <= S):
        for loss in (0.0, 0.02, 0.10):
            g = torch.Generator().manual_seed(4410 + n)
            rng = np.random.default_rng(int(1000 * loss) + n)
            lists = [torch.randperm(S, generator=g)[:n] for _ in range(ticks)]
            packets = torch.multinomial(torch.tensor([0.3, 0.6, 0.1]), ticks * n, True, generator=g).view(ticks, n)
            order = [arrivals(3 * ticks, loss, rng) for _ in range(S)]
            at, seqs = [0] * S, torch.full((ticks, n, M), -1, dtype=torch.int32)
            for t in range(ticks):
                for i, s in enumerate(lists[t].tolist()):
                    c = int(packets[t, i])
                    seqs[t, i, :c] = torch.tensor(order[s][at[s]:at[s] + c], dtype=torch.int32)
                    at[s] += c
            # Every graph starts by gathering its tick's lists from a device table into one packed buffer, then steps
            # its tick counter: three small kernels, the same in every graph, and no eager work around the replays.
            wseq = torch.zeros(ticks, n, dtype=torch.int32)  # the worst case: listing k of a slot sends 2 k
            listed = [0] * S
            for t in range(ticks):
                for i, s in enumerate(lists[t].tolist()):
                    listed[s] += 1
                    wseq[t, i] = 2 * listed[s]
            lists_t = torch.stack(lists).to(torch.int32)
            tables = {"with_ms": torch.cat([lists_t, packets.to(torch.int32), seqs.view(ticks, n * M)], 1),
                      "without_ms": torch.cat([lists_t, (PACKET * packets).to(torch.int32)], 1),
                      "worst_ms": torch.cat([lists_t, wseq], 1), "lists_ms": lists_t}
            tables = {k: v.to(dev).contiguous() for k, v in tables.items()}
            bufs = {k: torch.zeros(1, v.shape[1], dtype=torch.int32, device=dev) for k, v in tables.items()}
            step = {k: torch.zeros(1, dtype=torch.int64, device=dev) for k in tables}

            def next_tick(k):
                torch.index_select(tables[k], 0, step[k], out=bufs[k])
                step[k].add_(1)
                step[k].remainder_(ticks)
                return bufs[k][0]

            x44 = (0.1 * torch.randn(n, 2, M * PACKET, generator=g)).to(dev)
            b = {"y": torch.empty(n, 2, MAX_OUT * PACKET, device=dev), "oc": torch.empty(n, dtype=torch.int32, device=dev),
                 "y16": torch.empty(n, 2, 640, device=dev), "y16o": torch.empty(n, 2, 320, device=dev),
                 "n16": torch.empty(n, dtype=torch.int32, device=dev),
                 "chunk": torch.empty(n, 2, 128 * T + 64, device=dev),
                 "hops": torch.zeros(n, dtype=torch.int32, device=dev)}
            jb = JitterBuffer(S, 2, 44100, PACKET, depth=1, window=16, max_out=MAX_OUT, device=dev)
            down_w = PacketResampler(44100, 16000, S, 2, MAX_OUT * PACKET, device=dev)
            fifo_w = HopFifo(S, 2, T, CAP, device=dev)
            down_o = PacketResampler(44100, 16000, S, 2, M * PACKET, device=dev)
            fifo_o = HopFifo(S, 2, T, CAP, device=dev)
            worst = JitterBuffer(S, 2, 44100, PACKET, depth=0, window=16, max_out=MAX_OUT, device=dev)
            worst(torch.zeros(S, 2, PACKET, device=dev), torch.zeros(S, 1, dtype=torch.int32), [1] * S, list(range(S)))
            wy, woc = torch.empty(n, 2, MAX_OUT * PACKET, device=dev), torch.empty(n, dtype=torch.int32, device=dev)

            def with_jb():
                v = next_tick("with_ms")
                slots, counts, sq = v[:n], v[n:2 * n], v[2 * n:].view(n, M)
                jb(x44, sq, counts, slots, out=b["y"], out_counts=b["oc"])
                down_w(b["y"], b["oc"], slots, unit=PACKET, out=b["y16"], out_counts=b["n16"])
                fifo_w(b["y16"], b["n16"], slots, out=b["chunk"], hops=b["hops"])

            def without_jb():
                v = next_tick("without_ms")
                slots, samples = v[:n], v[n:]
                down_o(x44, samples, slots, out=b["y16o"], out_counts=b["n16"])
                fifo_o(b["y16o"], b["n16"], slots, out=b["chunk"], hops=b["hops"])

            def worst_jb():
                v = next_tick("worst_ms")
                worst(x44[..., :PACKET], v[n:].view(n, 1), one, v[:n], out=wy, out_counts=woc)

            one = torch.ones(n, dtype=torch.int32, device=dev)
            rep_with, rep_without, rep_worst = graphed(with_jb), graphed(without_jb), graphed(worst_jb)
            rep_lists = graphed(lambda: next_tick("lists_ms"))
            xs, ys = b["chunk"], torch.empty(n, 2, 128 * T, device=dev)
            ebuf, hops_sep, slots_sep = e[:n].clone(), torch.ones(n, dtype=torch.int32, device=dev), lists_t[0].to(dev)
            lists_dev = lists_t.to(dev)
            embs = e[lists_dev.long()]
            sep_tick = [0]

            def run_sep(_):
                i = sep_tick[0] % ticks
                sep_tick[0] += 1
                slots_sep.copy_(lists_dev[i])
                ebuf.copy_(embs[i])
                net._launch("slots_hops", xs, ebuf, big, ys, T, L2H_FLAG_GRAPH, slots=slots_sep, hops=hops_sep, ws=ws)

            run_with, run_without, run_worst = (lambda _: rep_with()), (lambda _: rep_without()), (lambda _: rep_worst())
            fns = {"with_ms": run_with, "without_ms": run_without, "worst_ms": run_worst, "lists_ms": lambda _: rep_lists(),
                   "sep_ms": run_sep}
            for fn in fns.values():
                for i in range(R):
                    fn(i)
            torch.cuda.synchronize()
            r = alternate(fns, R)
            r["added_ms"] = r["with_ms"] - r["without_ms"]
            r["added_share"] = r["added_ms"] / r["sep_ms"]
            r["worst_jb_ms"] = r["worst_ms"] - r["lists_ms"]
            r["worst_share"] = r["worst_jb_ms"] / r["sep_ms"]
            r["lost"] = int(jb.lost.sum())
            r["late"] = int(jb.late.sum())
            r["worst_lost"] = int(worst.lost.sum())
            res["cases"][f"n{n}_loss{int(100 * loss)}"] = r
            print(json.dumps({f"n{n}_loss{int(100 * loss)}": r}), file=sys.stderr)
    emit(res, args.out)


if __name__ == "__main__":
    main()
