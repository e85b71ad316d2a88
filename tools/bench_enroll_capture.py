"""Cost of enrollment from listeners' own streams: the per-slot capture inside a serving tick (EnrollCapture,
l2h_enroll_capture), and enrollment from the capture's rings (EmbedTFGridNet.enroll, l2h_embed_forward_slots) against the
path a service has without them.

    python tools/bench_enroll_capture.py [--reps 20] [--out FILE]

Tick, for n = 64 and 256 listeners on a state of n slots, every listener sending 128 samples at 16 kHz per 8 ms tick (a
fresh random slot list each tick, rewritten in place), the FIFO popping up to T = 3 hops:
    tick_ms     one graph replay of HopFifo -> EnrollCapture (5 s rings), then the separator's slot-list call with the
                FIFO's hop counts (l2h_sep_forward_slots_hops, its own cached graph)
    base_ms     the same tick without the capture
    capture_ms  a graph of the capture kernel alone over the same lists
    capture_share = capture_ms / tick_ms
Enrollment, for 1, 8 and 32 listeners of a 32-slot capture holding 5 s each, windows of 3 to 5 s (seeded):
    ring_ms     EmbedTFGridNet.enroll from the rings, into rows of a staging buffer
    host_ms     the windows cut from copies of the streams kept on the host, gathered into a padded [n, 2, n_max] batch,
                uploaded and embedded with EmbedTFGridNet.forward(x, lengths); keeping those copies costs a read-back of
                every tick's audio, which is not counted here
    agree       the two give the same embeddings, bit for bit
Every shape is warmed up first; the tick's three timings alternate, median of 5 windows of `--reps` (CUDA events); each
enrollment timing is the median of `--reps` calls, host clock around work that ends in a device synchronise.
Printed as one JSON object with the GPU's name and power limit, which belong with the numbers.
"""
import argparse
import json
import statistics
import sys
import time

import torch

from bench_common import L2H_FLAG_GRAPH, alternate, emit, gpu_info, graphed, setup_net
from lookoncetohear_b200 import EmbedTFGridNet, EnrollCapture, HopFifo, synth
from lookoncetohear_b200.configs import EMBED_PARAMS

T, HOP, CARRY, SR = 3, 128, 64, 16000


def host_ms(fn, reps):
    """median wall time of fn() followed by a device synchronise (ms)"""
    t = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append(1e3 * (time.perf_counter() - t0))
    return statistics.median(t)


def tick_case(net, dev, n, R, g):
    lists = torch.stack([torch.randperm(n, generator=g) for _ in range(R)]).to(dev, torch.int32)
    x = (0.1 * torch.randn(n, 2, HOP, generator=g)).to(dev)
    e = synth.embedding(n, seed0=8800)[:, 0].to(dev)
    st = net.init_buffers(n, dev)
    ws, _ = net._workspace(dev, n, T)
    fifo, cap = HopFifo(n, 2, T, 1024, device=dev), EnrollCapture(n, 2, 5 * SR, device=dev)
    slots, counts = lists[0].clone(), torch.full((n,), HOP, dtype=torch.int32, device=dev)
    chunk, hops = torch.zeros(n, 2, HOP * T + CARRY, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)
    ys = torch.empty(n, 2, HOP * T, device=dev)
    replay_fc = graphed(lambda: (fifo(x, counts, slots, out=chunk, hops=hops), cap(chunk, slots, hops)))
    replay_f = graphed(lambda: fifo(x, counts, slots, out=chunk, hops=hops))
    replay_c = graphed(lambda: cap(chunk, slots, hops))

    def sep():
        net._launch("slots_hops", chunk, e, st, ys, T, L2H_FLAG_GRAPH, slots=slots, hops=hops, ws=ws)

    def run(replay):
        def f(i):
            slots.copy_(lists[i % R])
            replay()
            if replay is not replay_c:
                sep()
        return f

    fns = {"tick_ms": run(replay_fc), "base_ms": run(replay_f), "capture_ms": run(replay_c)}
    for fn in fns.values():                                  # warm: every slot's gate built, graphs captured
        for i in range(R):
            fn(i)
    torch.cuda.synchronize()
    r = alternate(fns, R)
    r["capture_share"] = r["capture_ms"] / r["tick_ms"]
    r["mean_hops"] = float(hops.float().mean())
    return r


def enroll_case(enet, dev, cap, streams_host, n, R, g):
    S = cap.n_slots
    slots = torch.randperm(S, generator=g)[:n].tolist()
    lens = torch.randint(3 * SR, int(cap.captured.max()) + 1, (n,), generator=g).tolist()
    staging = torch.zeros(S, 256, device=dev)
    out = staging[:n]
    n_max = max(lens)

    def ring():
        enet.enroll(cap, slots, lens, out=out)

    def host():
        x = torch.zeros(n, 2, n_max)
        for b, (s, L) in enumerate(zip(slots, lens)):
            x[b, :, :L] = streams_host[s][:, -L:]
        return enet(x.to(dev), lens)

    with torch.no_grad():
        ring()
        agree = torch.equal(out.view(torch.int32), host().view(torch.int32))
        r = {"ring_ms": host_ms(ring, R), "host_ms": host_ms(host, R)}
    r["host_over_ring"] = r["host_ms"] / r["ring_ms"]
    r["agree"] = bool(agree)
    r["seconds"] = [round(L / SR, 2) for L in lens] if n <= 8 else [round(min(lens) / SR, 2), round(max(lens) / SR, 2)]
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="ticks per timed window, and enrollment calls per median")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_enroll_capture")
    R = args.reps
    g = torch.Generator().manual_seed(5150)
    res = dict(gpu_info(), reps=R, frames=T, ticks={}, enroll={})
    for n in (64, 256):
        res["ticks"][f"n{n}"] = r = tick_case(net, dev, n, R, g)
        print(json.dumps({f"n{n}": r}), file=sys.stderr)

    torch.manual_seed(0)
    enet = EmbedTFGridNet(**EMBED_PARAMS).eval().to(dev)
    S, cap_len, Tc = 32, 5 * SR, 8
    sig = synth.enrollment(S, cap_len, seed0=5200).to(dev)
    cap = EnrollCapture(S, 2, cap_len, device=dev)
    for k in range(cap_len // (HOP * Tc)):                   # 5 s of every stream through the capture
        chunk = torch.zeros(S, 2, HOP * Tc + CARRY, device=dev)
        chunk[:, :, CARRY:] = sig[:, :, HOP * Tc * k:HOP * Tc * (k + 1)]
        cap(chunk, list(range(S)), [Tc] * S)
    fed = HOP * Tc * (cap_len // (HOP * Tc))
    streams_host = [sig[s, :, :fed].cpu() for s in range(S)]
    for n in (1, 8, 32):
        res["enroll"][f"n{n}"] = r = enroll_case(enet, dev, cap, streams_host, n, R, g)
        print(json.dumps({f"enroll_n{n}": r}), file=sys.stderr)
    emit(res, args.out)


if __name__ == "__main__":
    main()
