"""Set-up, CUDA-event timers and result output shared by the serving benchmarks (tools/bench_*.py).

A number from these timers belongs with the GPU it was measured on, so every tool prints gpu_info() beside it."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from lookoncetohear_b200 import Net, synth  # noqa: E402
from lookoncetohear_b200.configs import TSH_PARAMS  # noqa: E402

HOP, LA = 128, 64
L2H_FLAG_GRAPH = 2
LISTENERS = (16, 64, 256)                      # listeners per tick of the stage benchmarks
TICKS = 8                                      # distinct precomputed ticks, cycled


def i32(v, dev):
    return torch.as_tensor(v, dtype=torch.int32).to(dev)


def setup_net(tool):
    """(the seeded separator on cuda:0 with its weights committed, the device); exits when there is no CUDA device"""
    if not torch.cuda.is_available():
        sys.exit(f"{tool}: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    net = Net(**TSH_PARAMS).eval().to(dev)
    net._sync_weights(dev)
    return net, dev


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        info["power_limit_and_max_sm_clock"] = "unavailable"
    return info


def window_ms(fn, reps):
    """device time of `reps` calls fn(0) .. fn(reps - 1), per call (ms)"""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(reps):
        fn(i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def median_ms(fn, reps, windows=5):
    """median over `windows` consecutive windows of window_ms(fn, reps)"""
    return statistics.median([window_ms(fn, reps) for _ in range(windows)])


def alternate(fns, reps, windows=5):
    """{name: median over `windows` of window_ms(fn, reps)}, the fns timed in turn within every window"""
    t = {k: [] for k in fns}
    for _ in range(windows):
        for k, fn in fns.items():
            t[k].append(window_ms(fn, reps))
    return {k: statistics.median(v) for k, v in t.items()}


def graphed(fn):
    """fn() captured as a CUDA graph (after a warm-up call on a side stream); returns the graph's replay"""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def rel_l2(a, b):
    """max over rows of ||a - b|| / ||b||, over the rows b has written (norm > 0)"""
    a, b = a.reshape(a.shape[0], -1).double(), b.reshape(b.shape[0], -1).double()
    nb = b.norm(dim=1)
    live = nb > 0
    return float(((a - b).norm(dim=1)[live] / nb[live]).max()) if bool(live.any()) else 0.0


def emit(res, out=None):
    """print the result as one JSON line, and write it to `out` too if given"""
    line = json.dumps(res)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


def population(n, K=None):
    """(the speakers of each of n listeners, the case's generator, seeded 9700 + n): K each, or without K half the
    listeners with 1, three eighths with 2 and one eighth with 3, in an order drawn from the generator"""
    g = torch.Generator().manual_seed(9700 + n)
    if K is not None:
        return [K] * n, g
    pop = {1: n // 2, 2: 3 * n // 8, 3: n // 8}
    ks = [k for k in (1, 2, 3) for _ in range(pop[k])]
    return [ks[i] for i in torch.randperm(n, generator=g).tolist()], g


class Tick:
    """The multi-voice 16 kHz tick the per-slot stage benchmarks build on: listener i with ks[i] target rows, the R
    records scattered over one state of S = max(256, 1.25 R) records (drawn from g, as are the listeners' slots), T hops
    per tick, every listener advancing T hops (`hops`).  rows(i) rewrites fixed staging buffers with precomputed tick
    i % TICKS of the seeded mixtures and embeddings, then runs the rows call (l2h_sep_forward_targets_rows) on one cached
    engine graph into y [R, 2, 128 T]."""

    def __init__(self, net, dev, ks, g, T):
        self.n, self.ks, self.g, self.T = len(ks), ks, g, T
        self.R = R = sum(ks)
        offsets = [0]
        for k in ks:
            offsets.append(offsets[-1] + k)
        self.S = max(256, R + R // 4)
        self.records = torch.randperm(self.S, generator=g)[:R]
        x_all, _ = synth.mixture(self.n, HOP * T * TICKS, seed0=9800)
        x_all = torch.nn.functional.pad(x_all, (0, LA)).to(dev)
        self.xs = [x_all[..., HOP * T * t:HOP * T * (t + 1) + LA].contiguous() for t in range(TICKS)]
        self.e = synth.embedding(R, seed0=9900)[:, 0].to(dev)
        self.x, self.ea = torch.empty_like(self.xs[0]), torch.empty_like(self.e)
        self.rec, self.off = i32(self.records, dev), i32(offsets, dev)
        self.slots = i32(torch.randperm(self.n, generator=g), dev)
        self.hops = i32([T] * self.n, dev)
        self.y = torch.empty(R, 2, HOP * T, device=dev)
        self.net, self.st = net, net.init_buffers(self.S, dev)
        self.ws, _ = net._workspace(dev, R, T)

    def rows(self, i):
        self.x.copy_(self.xs[i % TICKS]); self.ea.copy_(self.e)
        self.net._launch("targets_rows", self.x, self.ea, self.st, self.y, self.T, L2H_FLAG_GRAPH, slots=self.rec,
                         offsets=self.off, ws=self.ws)

    def result(self, **extra):
        """the case's keys of the JSON result, then `extra`"""
        return dict(listeners=self.n, target_rows=self.R, T=self.T, state_records=self.S, **extra)


def warm_up(fns, reps):
    """every fn(i) for i < reps, in turn: engine graphs, gate memos, every captured graph"""
    for i in range(reps):
        for f in fns.values():
            f(i)
    torch.cuda.synchronize()


def main(tool, case):
    """the command line of a stage benchmark: case(net, dev, n, T, reps) for T = 1 and 3 hops and every count of
    LISTENERS, printed as one JSON object with the GPU's identity"""
    ap = argparse.ArgumentParser()
    ap.add_argument("--hops", type=int, default=20, help="ticks per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net(tool)
    res = dict(gpu_info(), ticks_per_window=args.hops, cases=[])
    with torch.no_grad():
        for T in (1, 3):
            for n in LISTENERS:
                res["cases"].append(case(net, dev, n, T, args.hops))
    emit(res, args.out)
