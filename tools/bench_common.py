"""Set-up, CUDA-event timers and result output shared by the serving benchmarks (tools/bench_*.py).

A number from these timers belongs with the GPU it was measured on, so every tool prints gpu_info() beside it."""
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from lookoncetohear_b200 import Net  # noqa: E402
from lookoncetohear_b200.configs import TSH_PARAMS  # noqa: E402

HOP, LA = 128, 64
L2H_FLAG_GRAPH = 2


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
