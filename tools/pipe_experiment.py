"""Pipeline sweep: lane counts per stage -> frames/s (device-resident clip, B=1), plus the CPU time the host
spends inside l2h_sep_stream_dev (graph launches) per 500-hop clip.
    python tools/pipe_experiment.py [A:Q:T:O:F:B[:pdl_mask[:midb_hops[:midc_lanes[:hops_per_graph]]]] ...]      lanes of BiLSTM : qkv : attention : attn_out : front : back"""
import os, sys, time, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lookoncetohear_b200 import Net, synth
from lookoncetohear_b200.configs import TSH_PARAMS

dev = torch.device("cuda", 0)
torch.manual_seed(0)
net = Net(**TSH_PARAMS).eval().to(dev)
x, _ = synth.mixture(1, 64000)
x = x.to(dev)
emb = synth.embedding(1)[:, 0].to(dev)
y = torch.empty(1, 2, 64000, device=dev)
combos = sys.argv[1:] or ["12:3:3:4:6:6", "12:3:3:4:4:4", "16:3:3:4:6:6", "12:3:3:4:6:6:16:8", "12:3:3:4:6:6:16:4:2:250"]
names = ("pipeline_lanes", "pipeline_qkv_lanes", "pipeline_attn_lanes", "pipeline_out_lanes", "pipeline_front_lanes",
         "pipeline_back_lanes", "pipeline_pdl", "pipeline_midb_hops", "pipeline_midc_lanes", "pipeline_frames")
for combo in combos:
    vals = [int(v) for v in combo.split(":")]
    defaults = [12, 3, 3, 4, 6, 6, 16, 4, 2, 0]
    vals += defaults[len(vals):]
    for n, v in zip(names, vals):
        net.set_option(n, v)
    best, cpu = None, None
    for it in range(4):
        st = net.init_buffers(1, dev)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        a.record()
        net.stream_dev(x, emb, chunks_per_call=1, state=st, n_calls=500, out=y)
        b.record()
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b)
        if it > 0 and (best is None or ms < best):
            best, cpu = ms, 1e3 * (t1 - t0)
    print(json.dumps({"lanes_A:Q:T:O:F:B": combo, "frames_per_s": round(500 / (best * 1e-3)),
                      "us_per_hop": round(1e3 * best / 500, 2), "host_ms_in_call": round(cpu, 2), "gpu_ms": round(best, 2)}), flush=True)
