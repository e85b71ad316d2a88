"""256 streams x one hop per step (BASELINE configs[4] per-GPU shape): ms per hop-step under engine options.
    python tools/b256_step.py [name=value ...] [-- name=value ...]   (every '--'-separated group is one measurement)"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from lookoncetohear_b200 import Net
from lookoncetohear_b200.configs import TSH_PARAMS

dev = torch.device("cuda", 0)
torch.manual_seed(0)
net = Net(**TSH_PARAMS).eval().to(dev)
groups, cur = [], []
for a in sys.argv[1:]:
    if a == "--":
        groups.append(cur); cur = []
    else:
        cur.append(a)
groups.append(cur)
for g in groups:
    for kv in g:
        k, v = kv.split("=")
        net.set_option(k, int(v))
    ms, gb = bench.measure_batched_streaming(net, dev, 0, 256, 60)
    print(json.dumps({"options": g, "ms_per_hop_step": round(ms / 50, 4), "frames_per_s": round(256 * 50 / (ms * 1e-3))}), flush=True)
    for kv in g:
        k, _ = kv.split("=")
        net.set_option(k, {"pdl": 1, "fuse_ih": 0, "bf16": 0}.get(k, 0))
