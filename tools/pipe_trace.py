"""Timeline of the pipelined one-hop graph from the device-side trace (l2h_sep_trace_start / _read): per kernel the
duration, the wait between its last dependency finishing and its own start, the start-to-start interval of each stage,
and how many kernels are in flight; then a census of the SM time each stage holds per hop (DESIGN.md 4.2).
python tools/pipe_trace.py [out_prefix]"""
import ctypes, json, os, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from lookoncetohear_b200 import Net, synth, _cabi
from lookoncetohear_b200 import build as _build
from lookoncetohear_b200.configs import TSH_PARAMS

NAMES = ["front", "gemm_ih", "lstm", "mid_a", "mid_b", "mid_c", "qkv", "attn", "attn_out", "back", "mid"]
REC = np.dtype([("t0", "<u8"), ("t1", "<u8"), ("ptr", "<u8"), ("kernel", "<u4"), ("sm", "<u4")])
out_prefix = sys.argv[1] if len(sys.argv) > 1 else os.path.join(tempfile.gettempdir(), "pipe_trace")
dev = torch.device("cuda", 0)
torch.manual_seed(0)
net = Net(**TSH_PARAMS).eval().to(dev)
L = _cabi.lib()
HOPS = 500
x, _ = synth.mixture(1, 128 * HOPS)
x = x.to(dev)
emb = synth.embedding(1)[:, 0].to(dev)
y = torch.empty(1, 2, 128 * HOPS, device=dev)
for _ in range(3):
    net.stream_dev(x, emb, chunks_per_call=1, n_calls=HOPS, out=y)
torch.cuda.synchronize()
CAP = 40 * HOPS
_cabi.check(L.l2h_sep_trace_start(net._engine(), CAP))
st = net.init_buffers(1, dev)
torch.cuda.synchronize()
net.stream_dev(x, emb, chunks_per_call=1, state=st, n_calls=HOPS, out=y)
buf = np.zeros(CAP, dtype=REC)
n = ctypes.c_int32()
_cabi.check(L.l2h_sep_trace_read(net._engine(), buf.ctypes.data_as(ctypes.c_void_p), CAP, ctypes.byref(n)))
_cabi.check(L.l2h_sep_trace_start(net._engine(), 0))
r = buf[:n.value]
r = r[r["t1"] > 0]
ws_base = net._ws.data_ptr()
slot = net._ws.numel() // net.pipeline_frames()
hop = ((r["ptr"].astype(np.int64) - ws_base) // slot).astype(np.int64)
t_origin = int(r["t0"].min())
t0 = (r["t0"].astype(np.int64) - t_origin) / 1e3          # us
t1 = (r["t1"].astype(np.int64) - t_origin) / 1e3
kern = r["kernel"].astype(np.int64)
np.savez_compressed(out_prefix + ".npz", t0=t0, t1=t1, kernel=kern, hop=hop, sm=r["sm"])
total = float(t1.max())
print(json.dumps({"records": int(len(r)), "hops": HOPS, "span_us": round(total, 1), "us_per_hop": round(total / HOPS, 2)}))

# block index of a launch: order of start time among the launches of that kernel for that hop (block b+1 depends on b)
blk = np.zeros(len(r), dtype=np.int64)
for k in range(10):
    for h in np.unique(hop[kern == k]):
        idx = np.where((kern == k) & (hop == h))[0]
        blk[idx[np.argsort(t0[idx])]] = np.arange(len(idx))
key = {(int(kern[i]), int(blk[i]), int(hop[i])): i for i in range(len(r))}
mb = int(np.median(np.diff(np.sort(np.unique(hop[kern == 4]))))) if (kern == 4).sum() > 3 else 1


def dep_end(k, b, h):
    """end time of the latest dependency of launch (kernel k, block b, hop h)"""
    deps = []
    if k == 1: deps = [(0, 0, h)] if b == 0 else [(8, b - 1, h)]
    elif k == 2: deps = [(1, b, h)]
    elif k == 3: deps = [(2, b, h)]
    elif k == 4: deps = [(3, b, h + j) for j in range(mb)] + [(4, b, h - mb)]
    elif k == 5: deps = [(4, b, (h // mb) * mb)]
    elif k == 6: deps = [(5, b, h), (7, b, h - 3)]
    elif k == 7: deps = [(6, b, h), (6, b, h - 1), (6, b, h - 2)]
    elif k == 8: deps = [(7, b, h)]
    elif k == 9: deps = [(8, 2, h - j) for j in range(4)]
    ends = [t1[key[d]] for d in deps if d in key]
    return max(ends) if ends else None


steady = (hop >= 100) & (hop < 400)
print("| stage | launches | duration us (median / p90) | wait after last dependency us (median / p90) | start-to-start per block us (median) |")
print("|---|---|---|---|---|")
for k in range(10):
    m = (kern == k) & steady
    if not m.any():
        continue
    dur = t1[m] - t0[m]
    waits = []
    for i in np.where(m)[0]:
        de = dep_end(k, int(blk[i]), int(hop[i]))
        if de is not None:
            waits.append(t0[i] - de)
    s2s = []
    for b in range(3 if k not in (0, 9) else 1):
        tt = np.sort(t0[m & (blk == b)])
        if len(tt) > 2:
            s2s.append(np.median(np.diff(tt)))
    w = np.array(waits) if waits else np.array([np.nan])
    print("| %s | %d | %.1f / %.1f | %.1f / %.1f | %s |" % (NAMES[k], int(m.sum()), np.median(dur), np.percentile(dur, 90), np.median(w),
                                                    np.percentile(w, 90), ", ".join("%.1f" % v for v in s2s)))
# kernels in flight, sampled every 2 us over the steady part
lo, hi = np.percentile(t0[steady], 5), np.percentile(t0[steady], 95)
ts = np.arange(lo, hi, 2.0)
inflight = np.array([((t0 <= t) & (t1 > t)).sum() for t in ts])
per_stage = {NAMES[k]: round(float(np.mean([((t0 <= t) & (t1 > t) & (kern == k)).sum() for t in ts])), 2) for k in range(10)}
print(json.dumps({"kernels_in_flight_mean": round(float(inflight.mean()), 1), "p10": int(np.percentile(inflight, 10)),
                  "p90": int(np.percentile(inflight, 90)), "mean_in_flight_by_stage": per_stage, "mid_b_hops_per_launch": mb}))
# the pipeline's wavefront: when does hop h leave block b (attn_out end) relative to entering it (gemm start)
for b in range(3):
    lat = [t1[key[(8, b, h)]] - t0[key[(1, b, h)]] for h in range(100, 400) if (8, b, h) in key and (1, b, h) in key]
    if lat:
        print(json.dumps({"block": b, "hop_latency_through_block_us_median": round(float(np.median(lat)), 1)}))

# ---- census: how much SM time each stage holds per hop --------------------------------------------------------------
# A CTA reserves max(smem / 228 KB, threads / 2048, registers / 64 K, 1 / 32) of an SM for as long as it runs.
# Launch geometry of enqueue_pipeline (csrc/sep_engine.cu) at one stream and the default options (4-hop batches):
# stage -> (kernel symbol, CTAs per launch, threads per CTA, dynamic smem bytes, hops per launch per block)
GEOMETRY = {
    "front": ("front_kernel_tIl", 1, 256, 192 * 196 * 4, 1),
    "gemm_ih": ("rows_gemm_kernelILi16ELi64ELi2ELi4E", 25 * 8, 128, (64 * 20 + 64 * 64) * 4, mb),
    "lstm": ("lstm_rec3_kernelILi1ELb1E", 2 * mb, 128, 97 * 1024, mb),
    "mid_a": ("mid_a_kernel", 13, 256, 107264, mb),
    "mid_b": ("mid_b_kernel_tIl", 13, 256, 67840, mb),
    "mid_c": ("mid_c_kernel", 13, 256, 49920, mb),
    "qkv": ("qkv_kernel_tIl", 1, 384, 65216, 1),
    "attn": ("attn_cluster_kernel_tIl", 32, 256, 0, 1),
    "attn_out": ("attn_out_kernel_tIl", 1, 256, 66816, 1),
    "back": ("back_kernel_tIl", 4, 256, 70688, 1),
}
SM_SMEM, SM_THREADS, SM_REGS, SM_CTAS, N_SMS = 228 * 1024, 2048, 65536, 32, 132


def ptxas_usage(log_path):
    """{mangled kernel name: (registers, static smem bytes)} from the -Xptxas -v log of the build"""
    use, cur = {}, None
    for line in open(log_path):
        if "Compiling entry function" in line:
            cur = line.split("'")[1]
        elif cur and "Used" in line and "registers" in line:
            w = line.split()
            regs = int(w[w.index("registers,") - 1])
            smem = int(w[w.index("smem") - 2]) if "smem" in w else 0
            use[cur] = (regs, smem)
            cur = None
    return use


usage = ptxas_usage(os.path.join(_build.LIBDIR, "build.log"))
print("| stage | duration us (median) | CTAs | threads | regs | smem KB per CTA | SM share per CTA | hops per launch | SM us per hop |")
print("|---|---|---|---|---|---|---|---|---|")
total_smus = 0.0
for k, name in enumerate(NAMES[:10]):
    m = (kern == k) & steady
    if not m.any():
        continue
    sym, ctas, threads, dsmem, hops = GEOMETRY[name]
    hits = [(n, u) for n, u in usage.items() if sym in n and "Records" not in n]
    regs, ssmem = hits[0][1]
    smem = dsmem + ssmem + 1024                              # + the 1 KB the SM reserves per CTA
    share = max(smem / SM_SMEM, threads / SM_THREADS, -(-regs * 32 // 256) * 256 * (threads // 32) / SM_REGS, 1 / SM_CTAS)
    dur = float(np.median(t1[m] - t0[m]))
    smus = share * ctas * dur / hops
    total_smus += smus
    print("| %s | %.1f | %d | %d | %d | %.1f | %.3f | %d | %.2f |" % (name, dur, ctas, threads, regs, smem / 1024, share, hops, smus))
us_hop = total / HOPS
print(json.dumps({"sm_us_per_hop": round(total_smus, 1), "us_per_hop": round(us_hop, 2),
                  "machine_fill": round(total_smus / (N_SMS * us_hop), 3)}))
