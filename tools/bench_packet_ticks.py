"""Cost of a tick of listeners at 44.1 kHz that send 10 ms packets: resampling down, the per-slot hop FIFO and resampling
up on the device in one graph (PacketResampler, HopFifo), against the same tick with the FIFO kept by the host, and beside
the separator's tick.

    python tools/bench_packet_ticks.py [--slots 256] [--reps 20] [--out FILE]

For n = 16, 64, 256 listed listeners of a `--slots`-slot state, every tick each listener sends 0, 1 or 2 packets of 441
samples (seeded jitter, probabilities 0.3, 0.6, 0.1: 0.8 packets per 8 ms tick on average, the real-time rate), and the
FIFO pops up to T = 3 hops.  One tick is:
    device_ms  one graph replay: down 44.1 -> 16 kHz (l2h_resample_packets), l2h_hop_fifo, up 16 -> 44.1 kHz of the
               separator's [n, 2, 128 T] output with the FIFO's hop counts (unit 128)
    host_ms    the same down and up graphs, with the FIFO kept by the host between them: the out counts read back (a
               synchronise), append and pop with torch indexing, the hop counts uploaded
    sep_ms     the separator's slot-list call over the same n with the FIFO's hop counts (l2h_sep_forward_slots_hops), for
               the resampling's share of a tick: device_share = device_ms / (device_ms + sep_ms)
Every tick rewrites the slot list and the packet counts in place (a fresh random list of n), every shape is warmed up
first, and the three are timed alternately, the median of 5 windows of `--reps` ticks (CUDA events).
host_agrees: the two FIFOs, run from fresh states over the same ticks, give the same hop counts and chunks.
Printed as one JSON object with the GPU's name and power limit, which belong with the numbers.
"""
import argparse
import json
import sys

import numpy as np
import torch

from bench_common import L2H_FLAG_GRAPH, alternate, emit, gpu_info, graphed, setup_net
from lookoncetohear_b200 import HopFifo, PacketResampler, synth

T, CAP, PACKET = 3, 1024, 441


class HostFifo:
    """The hop FIFO kept by the host: per slot a linear buffer (the 64-sample carry first) and a fill level on the host"""

    def __init__(self, S, C, dev):
        self.buf = torch.zeros(S, C, 64 + CAP, device=dev)
        self.fill = np.zeros(S, dtype=np.int64)
        self.dev = dev

    def __call__(self, y16, out_counts, sl):
        dev, W = self.dev, self.buf.shape[-1]
        m = out_counts.cpu().numpy().astype(np.int64)               # a synchronise
        fill = self.fill[sl]
        kept = np.minimum(m, CAP - fill)
        rows = np.repeat(np.arange(len(sl)), kept)
        cols = np.arange(rows.size) - np.repeat(np.cumsum(kept) - kept, kept)
        r, c = torch.from_numpy(rows).to(dev), torch.from_numpy(cols).to(dev)
        slot = torch.from_numpy(sl).to(dev)
        self.buf[slot[r], :, torch.from_numpy(64 + fill[rows] + cols).to(dev)] = y16[r, :, c]
        fill = fill + kept
        h = np.minimum(T, fill // 128)
        chunk = self.buf[slot, :, :128 * T + 64]
        src = (torch.arange(W, device=dev)[None] + torch.from_numpy(128 * h).to(dev)[:, None]).clamp(max=W - 1)
        self.buf[slot] = torch.gather(self.buf[slot], 2, src[:, None].expand(-1, self.buf.shape[1], -1))
        self.fill[sl] = fill - 128 * h
        return chunk, torch.from_numpy(h.astype(np.int32)).to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=256, help="slots in the serving state")
    ap.add_argument("--reps", type=int, default=20, help="ticks per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_packet_ticks")
    S, R = args.slots, args.reps
    g = torch.Generator().manual_seed(4410)
    e = synth.embedding(8, seed0=8800)[:, 0].repeat((S + 7) // 8, 1)[:S].contiguous().to(dev)
    big = net.init_buffers(S, dev)
    ws, _ = net._workspace(dev, S, T)
    res = dict(gpu_info(), slots=S, reps_per_window=R, frames=T, cases={})

    for n in (m for m in (16, 64, 256) if m <= S):
        lists = [torch.randperm(S, generator=g)[:n] for _ in range(R)]
        packets = torch.multinomial(torch.tensor([0.3, 0.6, 0.1]), R * n, True, generator=g).view(R, n)
        lists_dev, counts_dev = torch.stack(lists).to(dev, torch.int32), (PACKET * packets).to(dev, torch.int32)
        lists_host = [sl.numpy() for sl in lists]
        x44 = (0.1 * torch.randn(n, 2, 2 * PACKET, generator=g)).to(dev)
        ysep = (0.1 * torch.randn(n, 2, 128 * T, generator=g)).to(dev)
        slots, counts = lists_dev[0].clone(), counts_dev[0].clone()
        b = {k: {"y16": torch.empty(n, 2, 320, device=dev), "oc": torch.empty(n, dtype=torch.int32, device=dev),
                 "chunk": torch.empty(n, 2, 128 * T + 64, device=dev), "hops": torch.zeros(n, dtype=torch.int32, device=dev),
                 "y44": torch.empty(n, 2, 353 * T, device=dev), "oc44": torch.empty(n, dtype=torch.int32, device=dev)}
             for k in ("device", "host")}

        def chain():
            return (PacketResampler(44100, 16000, S, 2, 2 * PACKET, device=dev), HopFifo(S, 2, T, CAP, device=dev),
                    PacketResampler(16000, 44100, S, 2, 128 * T, device=dev))

        dv, hs = chain(), chain()
        host_fifo = HostFifo(S, 2, dev)

        def down(objs, q):
            objs[0](x44, counts, slots, out=q["y16"], out_counts=q["oc"])

        def up(objs, q):
            objs[2](ysep, q["hops"], slots, unit=128, out=q["y44"], out_counts=q["oc44"])

        def device_tick():
            down(dv, b["device"])
            dv[1](b["device"]["y16"], b["device"]["oc"], slots, out=b["device"]["chunk"], hops=b["device"]["hops"])
            up(dv, b["device"])

        def host_tick(i, replay_down, replay_up):
            q = b["host"]
            replay_down()
            chunk, hops = host_fifo(q["y16"], q["oc"], lists_host[i % R])
            q["hops"].copy_(hops)
            replay_up()
            return chunk

        # agreement: fresh states, R ticks of both FIFOs over the same lists and packets
        agree = True
        for i in range(R):
            slots.copy_(lists_dev[i])
            counts.copy_(counts_dev[i])
            device_tick()
            chunk = host_tick(i, lambda: down(hs, b["host"]), lambda: up(hs, b["host"]))
            hd = b["device"]["hops"].tolist()
            agree &= hd == b["host"]["hops"].tolist()
            agree &= all(torch.equal(b["device"]["chunk"][r, :, :128 * h + 64], chunk[r, :, :128 * h + 64])
                         for r, h in enumerate(hd))

        replay_device = graphed(device_tick)
        replay_down, replay_up = graphed(lambda: down(hs, b["host"])), graphed(lambda: up(hs, b["host"]))
        xs, ys = b["device"]["chunk"], torch.empty(n, 2, 128 * T, device=dev)
        ebuf, hops_sep = e[:n].clone(), b["device"]["hops"].clone()
        embs = e[lists_dev.long()]

        def run_device(i):
            slots.copy_(lists_dev[i % R])
            counts.copy_(counts_dev[i % R])
            replay_device()

        def run_host(i):
            slots.copy_(lists_dev[i % R])
            counts.copy_(counts_dev[i % R])
            host_tick(i, replay_down, replay_up)

        def run_sep(i):
            slots.copy_(lists_dev[i % R])
            ebuf.copy_(embs[i % R])
            hops_sep.copy_(b["device"]["hops"])
            net._launch("slots_hops", xs, ebuf, big, ys, T, L2H_FLAG_GRAPH, slots=slots, hops=hops_sep, ws=ws)

        fns = {"device_ms": run_device, "host_ms": run_host, "sep_ms": run_sep}
        for fn in fns.values():                              # warm: every listed slot's gate built, graphs captured
            for i in range(R):
                fn(i)
        torch.cuda.synchronize()
        r = alternate(fns, R)
        r["host_over_device"] = r["host_ms"] / r["device_ms"]
        r["device_share"] = r["device_ms"] / (r["device_ms"] + r["sep_ms"])
        r["host_agrees"] = bool(agree)
        r["mean_hops"] = float(b["device"]["hops"].float().mean())
        res["cases"][f"n{n}"] = r
        print(json.dumps({f"n{n}": r}), file=sys.stderr)
    emit(res, args.out)


if __name__ == "__main__":
    main()
