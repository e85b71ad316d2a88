"""configs[2] (256 clips of 4 s, bf16 option) against the number of clips per kernel chain: wave quantisation of the recurrences
(tc_lstm: 32 sequences per CTA; lstm_rec4: NSEQ per CTA) decides the best split.   python tools/offline_split_experiment.py"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from lookoncetohear_b200 import Net
from lookoncetohear_b200.configs import TSH_PARAMS

dev = torch.device("cuda", 0)
torch.manual_seed(0)
net = Net(**TSH_PARAMS).eval().to(dev)
for arg in sys.argv[1:] or ["16", "9", "12", "18", "14"]:
    clips, tcmin = (arg.split(":") + ["2048"])[:2]
    clips = int(clips)
    net.set_option("tc_lstm_min", int(tcmin))
    net.max_frames_per_launch = clips * 500 + 100
    net._ws = None
    ms = bench.measure_offline_bf16(net, dev, 256)
    print(json.dumps({"clips_per_chain": clips, "tc_lstm_min": int(tcmin), "ms_per_256_clips": round(ms, 1), "frames_per_s": round(256 * 500 / (ms * 1e-3))}), flush=True)
