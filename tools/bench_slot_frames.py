"""Cost of multi-hop calls over a list of a state's records: catching up a backlog, and running listeners at a cadence.

    python tools/bench_slot_frames.py [--slots 256] [--reps 20] [--out FILE]

Calls run as a service runs them: fixed staging buffers, every call a replay of one cached graph (L2H_FLAG_GRAPH), the
list and the rows' embeddings rewritten in place on the device before every call (a fresh random list each time; every
listener keeps its own embedding), over a `--slots`-record state.

  * catch-up, for n = 1, 4, 16 listed listeners with a backlog of k = 2, 4, 8 hops:
      frames_ms   one k-hop l2h_sep_forward_slots_frames call
      chained_ms  k chained one-hop l2h_sep_forward_slots calls over the same list (what a service ran before)
  * cadence, for n = 64, 256 listed listeners and T = 1, 2, 4 hops per call, per hop:
      slots_ms_per_hop  a T-hop slot-list call / T
      dense_ms_per_hop  a T-hop l2h_sep_forward over a state of exactly n streams / T
Every figure is the median over 5 windows of `--reps` calls (or backlogs) timed with CUDA events.  The workspace sizes
of the cadence calls are listed with the part the slot-list calls' (h, c) copy takes.  Printed as one JSON object with
the GPU's name and power limit, which belong with the numbers.
"""
import argparse
import ctypes

import torch

from bench_common import HOP, LA, L2H_FLAG_GRAPH, emit, gpu_info, median_ms, setup_net
from lookoncetohear_b200 import synth, _cabi
from lookoncetohear_b200.configs import TSH_PARAMS

FC = 97 * 64          # floats of one block's h (or c) per record


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=256, help="records in the serving state")
    ap.add_argument("--reps", type=int, default=20, help="calls (catch-up: backlogs) per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_slot_frames")
    S, R = args.slots, args.reps
    catch_up = [(n, k) for n in (1, 4, 16) for k in (2, 4, 8) if n <= S]
    cadence = [(n, T) for n in (64, 256) for T in (1, 2, 4) if n <= S]
    max_t = max([k for _, k in catch_up] + [T for _, T in cadence])
    L, h = _cabi.lib(), net._engine()
    n_blocks = TSH_PARAMS["B"]

    def ws_bytes(n, T):
        b = ctypes.c_size_t()
        _cabi.check(L.l2h_sep_workspace_bytes(h, n, T, 0, ctypes.byref(b)))
        return b.value

    ws = torch.empty(max(ws_bytes(n, T) for n, T in catch_up + cadence + [(S, 1)]), dtype=torch.uint8, device=dev)
    g = torch.Generator().manual_seed(7100)
    x = (0.1 * torch.randn(S, 2, HOP * max_t + LA, generator=g)).to(dev)
    e = synth.embedding(8, seed0=8100)[:, 0].repeat((S + 7) // 8, 1)[:S].contiguous().to(dev)
    y = torch.empty(S, 2, HOP * max_t, device=dev)
    big = net.init_buffers(S, dev)
    res = dict(gpu_info(), slots=S, reps_per_window=R, catch_up={}, cadence={})

    def slot_call(slots, ebuf, n, T, x_off=0):
        """T hops of the n listed rows; x_off: the first hop of x (and y) this call consumes (chained one-hop calls)"""
        net._launch("slots_frames", x[:n, :, HOP * x_off:HOP * (x_off + T) + LA], ebuf, big,
                    y[:n, :, HOP * x_off:HOP * (x_off + T)], T, L2H_FLAG_GRAPH, slots=slots, ws=ws)

    def lists_for(n):
        lists = torch.stack([torch.randperm(S, generator=g)[:n] for _ in range(R)]).to(dev, torch.int32)
        return lists, e[lists.long()], lists[0].clone(), e[lists[0].long()].clone()

    for n, k in catch_up:
        lists, embs, slots, ebuf = lists_for(n)

        def run_frames(i):
            slots.copy_(lists[i % R])
            ebuf.copy_(embs[i % R])
            slot_call(slots, ebuf, n, k)

        def run_chained(i):
            slots.copy_(lists[i % R])
            ebuf.copy_(embs[i % R])
            for j in range(k):
                slot_call(slots, ebuf, n, 1, j)

        for fn in (run_frames, run_chained):          # warm: graph captures, every listed slot's gate built
            for i in range(R):
                fn(i)
        torch.cuda.synchronize()
        r = {"frames_ms": median_ms(run_frames, R), "chained_ms": median_ms(run_chained, R)}
        r["chained_over_frames"] = r["chained_ms"] / r["frames_ms"]
        res["catch_up"][f"n{n}_k{k}"] = r

    for n, T in cadence:
        lists, embs, slots, ebuf = lists_for(n)
        dense = net.init_buffers(n, dev)

        def run_slots(i):
            slots.copy_(lists[i % R])
            ebuf.copy_(embs[i % R])
            slot_call(slots, ebuf, n, T)

        def run_dense(i):
            net._launch("forward", x[:n, :, :HOP * T + LA], e, dense, y[:n, :, :HOP * T], T, L2H_FLAG_GRAPH, ws=ws)

        for fn in (run_slots, run_dense):
            for i in range(R):
                fn(i)
        torch.cuda.synchronize()
        r = {"slots_ms_per_hop": median_ms(run_slots, R) / T, "dense_ms_per_hop": median_ms(run_dense, R) / T}
        r["slots_over_dense"] = r["slots_ms_per_hop"] / r["dense_ms_per_hop"]
        hc = (2 if T > 1 else 0) * n_blocks * n * FC * 4
        r["workspace_bytes"] = ws_bytes(n, T)
        r["hc_copy_bytes"] = hc
        r["hc_copy_share"] = hc / r["workspace_bytes"]
        res["cadence"][f"n{n}_T{T}"] = r
        del dense
    emit(res, args.out)


if __name__ == "__main__":
    main()
