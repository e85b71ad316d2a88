"""Enrollment in slices (EmbedTFGridNet.enroll_job, l2h_embed_forward_slots_units): what each unit costs on the device,
and how much an enrollment holds up a serving tick, whole or in slices.

    python tools/bench_enroll_slices.py [--reps 20] [--out FILE]

units, for 1, 8 and 32 listeners of 5 s from a 32-slot capture holding 5 s each, at windows 0, 64, 128 and 256:
    unit_ms       the device time of every unit (CUDA events around each step(1); the stream is held by a sleep kernel
                  while the units are enqueued, so the times are device time, not enqueue time), median of 3 jobs
    max_unit_ms   the largest unit; sum_ms their sum; enroll_ms one EmbedTFGridNet.enroll call of the same rows (CUDA
                  events, median of 3); slicing = sum_ms / enroll_ms - 1
ticks, for 64 and 256 listeners: the tick of tools/bench_enroll_capture.py (a graph of HopFifo -> EnrollCapture, then
the separator's slot-list call with the FIFO's hop counts, its own cached graph), every 8 ms:
    alone_ms      the tick alone (median of --reps, CUDA events); alone_worst_ms the worst of them
    then_enroll   tick, then a whole enroll of 1 / 8 listeners on the same stream: when the next tick can start
    side_enroll   ticks launched one after another while an enroll of 1 / 8 listeners runs on a side stream; each tick's
                  duration from its launch (its stream idle) to its end: median and worst over every tick of --reps
                  enrollments
    sliced        an 8-listener job at the default window, step(k) after every tick on the same stream, k the most units
                  whose largest run of k consecutive units (from `units`) fits the tick's idle time 8 ms - alone_worst_ms;
                  tick + step(k) per period, median and worst, and the ticks the job took
Printed as one JSON object with the GPU's name and power limit, which belong with the numbers.
"""
import argparse
import json
import statistics
import sys

import torch

from bench_common import L2H_FLAG_GRAPH, emit, gpu_info, graphed, setup_net
from lookoncetohear_b200 import EmbedTFGridNet, EnrollCapture, HopFifo, synth
from lookoncetohear_b200.configs import EMBED_PARAMS
from lookoncetohear_b200.embed import DEFAULT_WINDOW

T, HOP, CARRY, SR, PERIOD_MS = 3, 128, 64, 16000, 8.0
WINDOWS = (0, 64, 128, 256)


def ev():
    return torch.cuda.Event(enable_timing=True)


def unit_times(enet, cap, slots, lens, window):
    """[ms] the device time of every unit of one job"""
    job = enet.enroll_job(cap, slots, lens, window=window)
    marks = [ev() for _ in range(job.units + 1)]
    torch.cuda._sleep(400_000_000)                    # hold the stream while the host enqueues every unit
    marks[0].record()
    for u in range(job.units):
        job.step()
        marks[u + 1].record()
    torch.cuda.synchronize()
    return [marks[u].elapsed_time(marks[u + 1]) for u in range(job.units)]


def event_ms(fn):
    a, b = ev(), ev()
    torch.cuda._sleep(100_000_000)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def units_case(enet, cap, n, g):
    slots = torch.randperm(cap.n_slots, generator=g)[:n].tolist()
    lens = [5 * SR] * n
    res = {}
    for w in WINDOWS:
        runs = [unit_times(enet, cap, slots, lens, w) for _ in range(3)]
        per = [statistics.median(r[u] for r in runs) for u in range(len(runs[0]))]
        enroll_ms = statistics.median(event_ms(lambda: enet.enroll(cap, slots, lens)) for _ in range(3))
        res[f"w{w}"] = {"units": len(per), "max_unit_ms": max(per), "sum_ms": sum(per), "enroll_ms": enroll_ms,
                        "slicing": sum(per) / enroll_ms - 1, "unit_ms": [round(t, 3) for t in per]}
        print(json.dumps({f"n{n}_w{w}": {k: v for k, v in res[f"w{w}"].items() if k != "unit_ms"}}), file=sys.stderr)
    return res


def tick_setup(net, dev, n, g):
    x = (0.1 * torch.randn(n, 2, HOP, generator=g)).to(dev)
    e = synth.embedding(n, seed0=8800)[:, 0].to(dev)
    st = net.init_buffers(n, dev)
    ws, _ = net._workspace(dev, n, T)
    fifo, cap = HopFifo(n, 2, T, 1024, device=dev), EnrollCapture(n, 2, 5 * SR, device=dev)
    slots, counts = torch.randperm(n, generator=g).to(dev, torch.int32), torch.full((n,), HOP, dtype=torch.int32, device=dev)
    chunk, hops = torch.zeros(n, 2, HOP * T + CARRY, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)
    ys = torch.empty(n, 2, HOP * T, device=dev)
    replay = graphed(lambda: (fifo(x, counts, slots, out=chunk, hops=hops), cap(chunk, slots, hops)))

    def tick():
        replay()
        net._launch("slots_hops", chunk, e, st, ys, T, L2H_FLAG_GRAPH, slots=slots, hops=hops, ws=ws)
    for _ in range(5):
        tick()
    torch.cuda.synchronize()
    return tick


def timed(fn):
    a, b = ev(), ev()
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def ticks_case(net, enet, ecap, dev, n, R, unit_res, g):
    tick = tick_setup(net, dev, n, g)
    alone = [timed(tick) for _ in range(R)]
    r = {"alone_ms": statistics.median(alone), "alone_worst_ms": max(alone), "then_enroll": {}, "side_enroll": {}}
    side = torch.cuda.Stream()
    for m in (1, 8):
        slots = torch.randperm(ecap.n_slots, generator=g)[:m].tolist()
        lens = [5 * SR] * m
        enet.enroll(ecap, slots, lens)
        r["then_enroll"][f"n{m}_ms"] = statistics.median(
            timed(lambda: (tick(), enet.enroll(ecap, slots, lens))) for _ in range(R))
        durs = []
        for _ in range(R):
            torch.cuda.synchronize()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                enet.enroll(ecap, slots, lens)
                done = ev()
                done.record()
            while not done.query():
                durs.append(timed(tick))
        r["side_enroll"][f"n{m}"] = {"median_ms": statistics.median(durs), "worst_ms": max(durs), "ticks": len(durs)}
    # sliced: an 8-listener job at the default window, step(k) after every tick
    per = unit_res["n8"][f"w{DEFAULT_WINDOW}"]["unit_ms"] if f"w{DEFAULT_WINDOW}" in unit_res["n8"] else None
    idle = PERIOD_MS - max(alone)
    k = 1
    if per is not None:
        while k < len(per) and max(sum(per[i:i + k + 1]) for i in range(len(per) - k)) <= idle:
            k += 1
    slots = torch.randperm(ecap.n_slots, generator=g)[:8].tolist()
    lens = [5 * SR] * 8
    periods = []
    for _ in range(3):
        job = enet.enroll_job(ecap, slots, lens)
        ticks = 0
        while not job.done:
            periods.append(timed(lambda: (tick(), job.step(k))))
            ticks += 1
    r["sliced"] = {"window": DEFAULT_WINDOW, "k": k, "idle_ms": idle, "median_ms": statistics.median(periods),
                   "worst_ms": max(periods), "ticks_per_job": ticks}
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="ticks per median, and enrollments per side-stream figure")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_enroll_slices")
    g = torch.Generator().manual_seed(6150)
    res = dict(gpu_info(), reps=args.reps, frames=T, seconds=5, default_window=DEFAULT_WINDOW, units={}, ticks={})

    torch.manual_seed(0)
    enet = EmbedTFGridNet(**EMBED_PARAMS).eval().to(dev)
    S, cap_len, Tc = 32, 5 * SR, 8
    sig = synth.enrollment(S, cap_len, seed0=5200).to(dev)
    ecap = EnrollCapture(S, 2, cap_len, device=dev)
    for k in range(cap_len // (HOP * Tc)):                   # 5 s of every stream through the capture
        chunk = torch.zeros(S, 2, HOP * Tc + CARRY, device=dev)
        chunk[:, :, CARRY:] = sig[:, :, HOP * Tc * k:HOP * Tc * (k + 1)]
        ecap(chunk, list(range(S)), [Tc] * S)
    with torch.no_grad():
        for n in (1, 8, 32):
            enet.enroll(ecap, list(range(n)), [5 * SR] * n)       # warm every shape
            res["units"][f"n{n}"] = units_case(enet, ecap, n, g)
        for n in (64, 256):
            res["ticks"][f"n{n}"] = r = ticks_case(net, enet, ecap, dev, n, args.reps, res["units"], g)
            print(json.dumps({f"ticks_n{n}": r}), file=sys.stderr)
    emit(res, args.out)


if __name__ == "__main__":
    main()
