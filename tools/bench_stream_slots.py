"""Cost of per-stream clocks in a 256-slot state (many listeners served from one state).

    python tools/bench_stream_slots.py [--streams 256] [--hops 20] [--out FILE]

Reports, as one JSON object, each figure the median of 5 windows timed with CUDA events:
  * hop_ms_stream_dev   one-hop steps through Net.stream_dev (graph replays; bench.py's batched_streaming path)
  * hop_ms_predict      one-hop Net.predict steps, every slot active (active=None)
  * hop_ms_predict_mask the same with an all-true mask
  * hop_ms_predict_skip the same with a random 10 % of the slots inactive on every hop (a fresh mask per hop)
  * reset_us_1 / reset_us_32   one SepState.reset_streams call of 1 / 32 slots (each slot is a ~6 MB record)
and the GPU's name and power limit, which belong with the numbers.
"""
import argparse

import torch

from bench_common import HOP, LA, emit, gpu_info, median_ms, setup_net
from lookoncetohear_b200 import synth


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=256)
    ap.add_argument("--hops", type=int, default=20, help="hops per timed window")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    net, dev = setup_net("bench_stream_slots")
    B, K = args.streams, args.hops
    g = torch.Generator().manual_seed(5000)
    n_hops = K + 10
    x = (0.1 * torch.randn(B, 2, HOP * n_hops + LA, generator=g)).to(dev)
    e = synth.embedding(8, seed0=6000)[:, 0].repeat((B + 7) // 8, 1)[:B].to(dev)
    chunks = [x[..., HOP * t:HOP * t + HOP + LA].contiguous() for t in range(n_hops)]
    res = dict(gpu_info(), streams=B, hops_per_window=K)

    # graph-replayed one-hop steps, as bench.py's batched_streaming measures them
    st = net.init_buffers(B, dev)
    y = torch.empty(B, 2, HOP * n_hops, device=dev)
    net.stream_dev(x, e, chunks_per_call=1, state=st, n_calls=10, out=y)
    res["hop_ms_stream_dev"] = median_ms(lambda i: net.stream_dev(x[..., HOP * 10:], e, chunks_per_call=1, state=st,
                                                                  n_calls=K, out=y[..., HOP * 10:]), 1) / K

    st = net.init_buffers(B, dev)
    ones = torch.ones(B, dtype=torch.bool, device=dev)
    masks = torch.rand(K, B, generator=g).to(dev) >= 0.1            # a random 10 % of the slots skip each hop
    with torch.no_grad():
        for t in range(3):                                          # warm: gate build, workspace
            net.predict(chunks[t], e, st, pad=False)
            net.predict(chunks[t], e, st, pad=False, active=ones)
        res["hop_ms_predict"] = median_ms(lambda i: net.predict(chunks[i], e, st, pad=False), K)
        res["hop_ms_predict_mask"] = median_ms(lambda i: net.predict(chunks[i], e, st, pad=False, active=ones), K)
        res["hop_ms_predict_skip"] = median_ms(lambda i: net.predict(chunks[i], e, st, pad=False, active=masks[i]), K)
    res["skipped_fraction"] = float(1.0 - masks.float().mean())

    slots32 = torch.randperm(B, generator=g)[:32].tolist()
    st.reset_streams([0])
    res["reset_us_1"] = 1e3 * median_ms(lambda i: st.reset_streams([i % B]), 20)
    res["reset_us_32"] = 1e3 * median_ms(lambda i: st.reset_streams(slots32), 20)
    rec_bytes = st.stride * 4
    res["record_bytes"] = rec_bytes
    res["reset_GBps_32"] = 32 * rec_bytes / (res["reset_us_32"] * 1e-6) / 1e9
    emit(res, args.out)


if __name__ == "__main__":
    main()
