"""Minimal target for ncu: a few one-frame (T=1, B=1) chains launched directly (no CUDA graph),
so that `ncu -s <skip> -c <count>` captures exactly one warm chain.
    ncu --set full --import-source on -s 2*L -c L -o prof_chain python tools/prof_chain.py [T] [B]
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from lookoncetohear_b200 import Net, synth
from lookoncetohear_b200.configs import TSH_PARAMS

T = int(sys.argv[1]) if len(sys.argv) > 1 else 1
B = int(sys.argv[2]) if len(sys.argv) > 2 else 1
n_chains = int(sys.argv[3]) if len(sys.argv) > 3 else 4
torch.manual_seed(0)
net = Net(**TSH_PARAMS).eval().cuda()
x, _ = synth.mixture(B, 128 * T * n_chains)
e = synth.embedding(B)[:, 0].cuda()
xp = torch.nn.functional.pad(x, (0, 64)).cuda()
st = net.init_buffers(B, "cuda")
torch.cuda.synchronize()
with torch.no_grad():
    for i in range(n_chains):
        net.predict(xp[..., 128 * T * i:128 * T * (i + 1) + 64], e, st, pad=False)
torch.cuda.synchronize()
print("done", st.header())
