"""Cost of adding a speaker to a running listener: the block-0 history a rows tick writes, and the join that replays it.

    python tools/bench_join_targets.py [--reps 20] [--out FILE]

(a) history   one-hop l2h_sep_forward_targets_rows ticks of 16, 64 and 256 listeners with two targets each, with and without
              a 64-frame history (l2h_sep_forward_targets_rows_history), timed alternately: median of 5 windows of `--reps`
              graph replays (L2H_FLAG_GRAPH), every shape warmed up first.  The two ticks' outputs are compared (equal).
(b) join      l2h_sep_join_targets of 1 and 8 records to 8 leads at clock 64, replaying W = 0 (cold), 16, 50 and 64 frames
              of a 64-frame history, graph replays, median of 5 windows.
(c) queued    a join is a call on its listeners' state, ordered with their ticks on one stream: a 256-listener tick with
              history alone, an 8-record 64-frame join into the same state (8 of its leads, 8 spare records, its own
              workspace) alone, and the join followed by the tick, timed alternately, median of 5 windows.
Printed as one JSON object with the GPU's name, power limit and max SM clock, which belong with the numbers.
"""
import argparse
import ctypes

import torch

from bench_common import HOP, LA, L2H_FLAG_GRAPH, alternate, emit, gpu_info, median_ms, setup_net
from lookoncetohear_b200 import _cabi, synth

K, F = 2, 64


def i32(v, dev):
    return torch.as_tensor(v, dtype=torch.int32).to(dev)


class Ticks:
    """n listeners of K targets on records 0 .. n*K - 1 of a state with 8 spare records, fixed buffers, one-hop ticks"""

    def __init__(self, net, dev, n, seed):
        self.net, self.n, self.R = net, n, n * K
        x, _ = synth.mixture(n, HOP * 8, seed0=seed)
        x = torch.nn.functional.pad(x, (0, LA)).to(dev)
        self.xs = [x[..., HOP * t:HOP * (t + 1) + LA].contiguous() for t in range(8)]
        self.e = synth.embedding(self.R + 8, seed0=seed + 1)[:, 0].to(dev)
        self.xb = torch.empty_like(self.xs[0])
        self.rec, self.off = i32(list(range(self.R)), dev), i32([i * K for i in range(n + 1)], dev)
        self.st = net.init_buffers(self.R + 8, dev)
        self.hist = net.target_history(self.st, F)
        self.y = torch.empty(self.R, 2, HOP, device=dev)
        self.ws = net._workspace(dev, self.R, 1)[0].clone()

    def run(self, i, history):
        self.xb.copy_(self.xs[i % 8])
        self.net._launch("targets_rows", self.xb, self.e[:self.R], self.st, self.y, 1, L2H_FLAG_GRAPH, slots=self.rec,
                         offsets=self.off, ws=self.ws, history=self.hist if history else None)


def history_cost(net, dev, reps):
    out = {}
    for n in (16, 64, 256):
        a, b = Ticks(net, dev, n, 9100), Ticks(net, dev, n, 9100)
        for i in range(3):
            a.run(i, True)
            b.run(i, False)
        torch.cuda.synchronize()
        equal = bool(torch.equal(a.y.view(torch.int32), b.y.view(torch.int32)))
        t = alternate({"with": lambda i: a.run(i, True), "without": lambda i: b.run(i, False)}, reps)
        out[f"n{n}"] = {"listeners": n, "target_rows": n * K, "tick_with_history_ms": t["with"],
                        "tick_without_ms": t["without"], "added_ms": t["with"] - t["without"], "outputs_equal": equal}
    return out


def join_cost(net, dev, reps):
    tk = Ticks(net, dev, 8, 9300)
    for i in range(F):                                    # the 8 leads reach clock 64 with full rings
        tk.run(i, True)
    leads = list(range(0, tk.R, K))
    out = {}
    for J in (1, 8):
        recs = i32(list(range(tk.R, tk.R + J)), dev)
        ld = i32(leads[:J], dev)
        y = torch.empty(J, 2, HOP * F, device=dev)
        used = torch.empty(J, dtype=torch.int32, device=dev)
        e = tk.e[tk.R:tk.R + J].contiguous()
        for W in (0, 16, 50, 64):
            def join(_i, W=W):
                net.join_targets(tk.st, recs, ld, e, history=tk.hist, frames=W, out=y, used=used, flags=L2H_FLAG_GRAPH)
            join(0)
            torch.cuda.synchronize()
            assert used.tolist() == [W] * J
            out[f"J{J}_W{W}_ms"] = median_ms(join, reps)
    return out


def queued(net, dev, reps):
    tk = Ticks(net, dev, 256, 9500)
    for i in range(F):                                    # the leads reach clock 64 with full rings
        tk.run(i, True)
    recs, ld = i32(list(range(tk.R, tk.R + 8)), dev), i32(list(range(0, 8 * K, K)), dev)     # 8 spare records, 8 leads
    y, used = torch.empty(8, 2, HOP * F, device=dev), torch.empty(8, dtype=torch.int32, device=dev)
    e = tk.e[tk.R:tk.R + 8].contiguous()
    need = ctypes.c_size_t()
    _cabi.check(_cabi.lib().l2h_sep_workspace_bytes(net._engine(), 8, F, L2H_FLAG_GRAPH, ctypes.byref(need)))
    ws = torch.empty(need.value, dtype=torch.uint8, device=dev)

    def join():
        net.join_targets(tk.st, recs, ld, e, history=tk.hist, frames=F, out=y, used=used, flags=L2H_FLAG_GRAPH, ws=ws)

    def join_then_tick(i):
        join()
        tk.run(F + i, True)
    join_then_tick(0)
    torch.cuda.synchronize()
    assert used.tolist() == [F] * 8
    t = alternate({"tick": lambda i: tk.run(F + i, True), "join_then_tick": join_then_tick, "join": lambda i: join()}, reps)
    return {"tick_ms": t["tick"], "join_then_tick_ms": t["join_then_tick"], "join_ms": t["join"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="calls per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_join_targets")
    res = dict(gpu_info(), reps_per_window=args.reps, history_frames=F, targets_per_listener=K)
    with torch.no_grad():
        res["history"] = history_cost(net, dev, args.reps)
        res["join"] = join_cost(net, dev, args.reps)
        res["queued"] = queued(net, dev, args.reps)
    emit(res, args.out)


if __name__ == "__main__":
    main()
