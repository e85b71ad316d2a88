"""Parity tests proper: the CUDA path, called through the reference-shaped API (which goes through
the C ABI), against the CPU oracle and the committed fixtures.  fp32 gates (BASELINE.json):
rel-L2 <= 1e-3 and |dSI-SDR| <= 0.1 dB."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import Net, synth
from oracle import restate as rs

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
REL_L2 = 1e-3
SISDR_DB = 0.1


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def model(tsh_params, dev):
    torch.manual_seed(0)
    net = Net(**tsh_params).eval()
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    return net.to(dev), sd


def _check(y, y_ref, tgt=None):
    y = y.float().cpu()
    assert y.shape == y_ref.shape
    assert torch.isfinite(y).all()
    err = rs.rel_l2(y, y_ref)
    assert err <= REL_L2, f"rel-L2 {err:.3e}"
    if tgt is not None:
        d = (rs.si_sdr(y, tgt) - rs.si_sdr(y_ref, tgt)).abs().max()
        assert float(d) <= SISDR_DB, f"dSI-SDR {float(d):.4f} dB"


def test_native_library_is_loaded(model):
    from lookoncetohear_b200 import _cabi
    assert _cabi.lib() is not None
    assert "liblookonce_b200.so" in open("/proc/self/maps").read()


@pytest.mark.parametrize("B,N", [(1, 128 * 6), (2, 128 * 14 - 51), (3, 200), (1, 128)])
def test_whole_utterance_vs_oracle(model, dev, B, N):
    net, sd = model
    x, tgt = synth.mixture(B, N, seed0=1000 + N)
    e = synth.embedding(B)
    y_ref = rs.sep_forward(sd, x, e)
    with torch.no_grad():
        y = net(x.to(dev), e.to(dev))
    _check(y, y_ref, tgt)


def test_every_stage_vs_oracle(model, dev):
    net, sd = model
    x, _ = synth.mixture(2, 128 * 5 + 9)
    e = synth.embedding(2)
    taps_ref = {}
    rs.sep_predict(sd, x, e[:, 0], rs.sep_init_state(sd, 2), taps=taps_ref)
    with torch.no_grad():
        _, taps, _ = net.forward_with_taps(x.to(dev), e.to(dev))
    ref = [taps_ref["enc"]] + [taps_ref[f"block{b}{s}"] for b in range(3) for s in ("_intra", "_inter", "")]
    ref[3] = ref[3] * taps_ref["gate"]      # gate folded into block 0's epilogue
    for i, (t, r) in enumerate(zip(taps, ref)):
        assert rs.rel_l2(t.cpu(), r) < 2e-4, f"stage {i}"


def test_golden_fixture(model, dev, tsh_params):
    g = np.load(os.path.join(GOLD, "sep_golden.npz"))
    net, _ = model                                 # seed 0 == fixture seed
    assert int(g["seed"]) == 0
    B, N = int(g["B"]), int(g["N"])
    x, tgt = synth.mixture(B, N)
    e = synth.embedding(B)
    with torch.no_grad():
        y = net(x.to(dev), e.to(dev))
    _check(y, torch.from_numpy(g["y"]), tgt)


def test_golden_fixture_long(model, dev):
    """T = 70 frames > the 50-frame attention window (history wrap inside one call)."""
    g = np.load(os.path.join(GOLD, "sep_golden_long.npz"))
    net, _ = model
    x, _ = synth.mixture(1, int(g["N"]), seed0=1100)
    e = synth.embedding(1, seed0=3100)
    with torch.no_grad():
        y = net(x.to(dev), e.to(dev)).cpu()
    assert rs.rel_l2(y[..., -1024:], torch.from_numpy(g["y_tail"])) <= REL_L2
    assert abs(float(y.pow(2).mean().sqrt()) / float(g["y_rms"]) - 1) < 1e-3


@pytest.mark.parametrize("cpc", [1, 2, 5])
def test_streaming_chunks_vs_whole_and_state(model, dev, cpc):
    """The streaming-buffer API (init_buffers / predict(pad=False)) with 1, 2, 5 chunks per call:
    output equals the whole-utterance oracle, and the final state equals the oracle's state
    (the ring slot rotation is undone by SepState.to_reference)."""
    net, sd = model
    T, B = 60, 2                                    # 60 frames: ring wraps (> 50)
    x, tgt = synth.mixture(B, 128 * T, seed0=77)
    e = synth.embedding(B, seed0=78)
    st_ref = rs.sep_init_state(sd, B)
    y_ref, st_ref = rs.sep_predict(sd, x, e[:, 0], st_ref)
    xp = F.pad(x, (0, 64)).to(dev)
    ed = e[:, 0].to(dev)
    st = net.init_buffers(B, dev)
    outs = []
    with torch.no_grad():
        for i in range(0, T, cpc):
            o, st = net.predict(xp[..., 128 * i:128 * (i + cpc) + 64], ed, st, pad=False)
            outs.append(o)
    _check(torch.cat(outs, -1), y_ref, tgt)
    assert st.header() == (T, T // cpc)
    got = st.to_reference()
    for k in ("conv_buf", "deconv_buf", "istft_buf"):
        assert rs.rel_l2(got[k].cpu(), st_ref[k]) < REL_L2, k
    for i in range(3):
        for k in ("K_buf", "V_buf", "h0", "c0"):
            assert rs.rel_l2(got["gridnet_bufs"][f"buf{i}"][k].cpu(), st_ref["gridnet_bufs"][f"buf{i}"][k]) < REL_L2, (i, k)


def test_mixed_call_sizes_and_embedding_change(model, dev):
    """Calls of different sizes interleaved (3 frames, 1, 1, 7, ...), and the speaker embedding
    changed mid-stream (the device-side gate memo must notice)."""
    net, sd = model
    sizes = [3, 1, 1, 7, 2, 1, 5]
    T = sum(sizes)
    x, _ = synth.mixture(1, 128 * T, seed0=5)
    e1, e2 = synth.embedding(1, seed0=6)[:, 0], synth.embedding(1, seed0=7)[:, 0]
    xp = F.pad(x, (0, 64))
    st_ref = rs.sep_init_state(sd, 1)
    st = net.init_buffers(1, dev)
    t0, ref, got = 0, [], []
    with torch.no_grad():
        for i, n in enumerate(sizes):
            e = e1 if i < 4 else e2
            seg = xp[..., 128 * t0:128 * (t0 + n) + 64]
            r, st_ref = rs.sep_predict(sd, seg, e, st_ref, pad=False)
            o, st = net.predict(seg.to(dev), e.to(dev), st, pad=False)
            ref.append(r)
            got.append(o)
            t0 += n
    _check(torch.cat(got, -1), torch.cat(ref, -1))


def test_linearity_of_front_and_back_is_not_assumed_but_silence_is_exact(model, dev):
    """Size-independent property usable at full size: an all-zero mixture gives the same output
    as the oracle's (bias-only path), and it is independent of the batch position."""
    net, sd = model
    x = torch.zeros(2, 2, 128 * 4)
    e = synth.embedding(2)
    e[1] = e[0]
    with torch.no_grad():
        y = net(x.to(dev), e.to(dev)).cpu()
    assert torch.equal(y[0], y[1])
    _check(y, rs.sep_forward(sd, x, e))


def test_full_size_clip_streaming_equals_whole(model, dev):
    """BASELINE config sizes (4 s clip, T = 500): chunked streaming == one whole-utterance call,
    and both match the oracle run on the same clip."""
    net, sd = model
    x, tgt = synth.mixture(1, 64000)
    e = synth.embedding(1)
    with torch.no_grad():
        y = net(x.to(dev), e.to(dev))
        st = net.init_buffers(1, dev)
        xp = F.pad(x, (0, 64)).to(dev)
        ed = e[:, 0].to(dev)
        ys = torch.cat([net.predict(xp[..., 128 * i:128 * i + 192], ed, st, pad=False)[0] for i in range(500)], -1)
    assert rs.rel_l2(ys.cpu(), y.cpu()) < 1e-4
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    _check(y, rs.sep_forward(sd, x, e), tgt)


def test_batch_split_path(model, dev):
    """forward() splits large batches into independent launches (workspace bound)."""
    net, sd = model
    old = net.max_frames_per_launch
    net.max_frames_per_launch = 8
    try:
        x, _ = synth.mixture(5, 128 * 4)
        e = synth.embedding(5)
        with torch.no_grad():
            y = net(x.to(dev), e.to(dev))
        _check(y, rs.sep_forward(sd, x, e))
    finally:
        net.max_frames_per_launch = old


def test_host_streaming_entry_point(model, dev):
    """l2h_sep_stream_host: pinned host buffers in, pinned host buffers out."""
    net, sd = model
    x, _ = synth.mixture(1, 128 * 20)
    e = synth.embedding(1)
    y_ref = rs.sep_forward(sd, x, e)
    for cpc in (1, 4):
        y = net.stream_host(x, e[:, 0].to(dev), chunks_per_call=cpc)
        _check(y, y_ref)


@pytest.mark.parametrize("cpc", [1, 3])
def test_device_streaming_entry_point(model, dev, cpc):
    """l2h_sep_stream_dev: CUDA-graph replay per call, chunk offset derived from the state's frame
    counter on the device; a second clip continues on the same state (clip_base handling)."""
    net, sd = model
    T = 57
    x, _ = synth.mixture(2, 128 * T, seed0=31)
    e = synth.embedding(2, seed0=32)
    st_ref = rs.sep_init_state(sd, 2)
    y_ref, st_ref = rs.sep_predict(sd, x, e[:, 0], st_ref)
    st = net.init_buffers(2, dev)
    y = net.stream_dev(x.to(dev), e[:, 0].to(dev), chunks_per_call=cpc, state=st)
    _check(y, y_ref)
    x2, _ = synth.mixture(2, 128 * 6, seed0=33)          # next clip, same streams
    y2_ref, _ = rs.sep_predict(sd, x2, e[:, 0], st_ref)
    y2 = net.stream_dev(x2.to(dev), e[:, 0].to(dev), chunks_per_call=cpc, state=st)
    _check(y2, y2_ref)


PIPE_OPTIONS = ("pipeline_lanes", "pipeline_qkv_lanes", "pipeline_attn_lanes", "pipeline_out_lanes", "pipeline_front_lanes",
                "pipeline_back_lanes", "pipeline_pdl", "pipeline_midb_hops", "pipeline_midc_lanes")


@pytest.mark.parametrize("lanes", [None, (16, 4, 4, 4, 8, 6, 1023, 8, 3), (3, 1, 1, 1, 1, 2, 16, 1, 1), (5, 2, 2, 3, 3, 3, 0, 3, 2)],
                         ids=["default", "max-lanes-pdl-all-stages-midb8", "few-lanes-midb1", "odd-lanes-no-pdl-midb3-midc2"])
def test_wavefront_pipeline_equals_sequential(model, dev, lanes):
    """One-hop calls captured as a (block, hop) wavefront graph must reproduce the strictly sequential
    hop-by-hop run bit for bit (same arithmetic, only the schedule and the kernel boundaries of the mid
    section differ), within one graph and across group boundaries (230 hops = 100 + 100 + 30), for several streams and for
    several lane counts per stage (every lane count exercises other event edges); both match the oracle."""
    net, sd = model
    T, B = 230, 3
    x, _ = synth.mixture(B, 128 * T, seed0=91)
    e = synth.embedding(B, seed0=92)
    xd, ed = x.to(dev), e[:, 0].to(dev)
    try:
        if lanes is not None:
            net.set_option("pipeline_frames", 100)        # 230 hops = 100 + 100 + 30; the default takes them as one graph
            for n, v in zip(PIPE_OPTIONS, lanes):
                net.set_option(n, v)
        net.set_option("pipeline", 1)
        y_pipe = net.stream_dev(xd, ed, chunks_per_call=1).cpu()
        st_pipe = net._last_stream_state.to_reference()
        net.set_option("pipeline", 0)
        net.set_option("fused_tail", 0)       # the sequential hops as the same separate kernels the pipeline runs
        y_seq = net.stream_dev(xd, ed, chunks_per_call=1).cpu()
        st_seq = net._last_stream_state.to_reference()
    finally:
        net.set_option("pipeline", 1)
        net.set_option("fused_tail", 1)
        net.reset_options()
    assert torch.equal(y_pipe, y_seq)
    assert torch.equal(st_pipe["gridnet_bufs"]["buf2"]["K_buf"], st_seq["gridnet_bufs"]["buf2"]["K_buf"])
    assert torch.equal(st_pipe["deconv_buf"], st_seq["deconv_buf"])
    y_ref = rs.sep_forward(sd, x[:1, :, :128 * 64], e[:1])
    _check(y_pipe[:1, :, :128 * 64], y_ref)


def test_launch_counter_counts_graph_nodes(model, dev):
    """bench.py's gpu_launches comes from l2h_sep_launch_count: a replayed CUDA graph counts its kernel nodes.  One
    sequential hop = front1 + 3 x (BiLSTM, tail_kernel) + back = 8 kernels (20 as separate kernels: 1 + 3 x 6 + 1); a pipelined 8-hop stream = per hop front + back + 3 x (qkv, attention,
    attn_out), per block and 4-hop batch ONE launch each of W_ih GEMM, BiLSTM, mid_a, mid_b, mid_c, + the header advance + the
    clip-base kernel = 120 (15 kernels per hop; the per-hop stage A and mid_c of round 1 made it 23.75)."""
    import ctypes
    from lookoncetohear_b200 import _cabi
    net, _ = model
    L = _cabi.lib()
    x, _ = synth.mixture(1, 128 * 8, seed0=5)
    e = synth.embedding(1, seed0=6)[:, 0].to(dev)
    xd = F.pad(x, (0, 64)).to(dev)
    st = net.init_buffers(1, dev)
    n = ctypes.c_int64()
    _cabi.check(L.l2h_sep_launch_count(net._engine(), None, 1))
    net.predict(xd[..., :192], e, st, pad=False)
    _cabi.check(L.l2h_sep_launch_count(net._engine(), ctypes.byref(n), 1))
    assert n.value == 8
    net.set_option("fused_tail", 0)
    try:
        net.predict(xd[..., 128:320], e, st, pad=False)
        _cabi.check(L.l2h_sep_launch_count(net._engine(), ctypes.byref(n), 1))
    finally:
        net.set_option("fused_tail", 1)
    assert n.value == 20
    st = net.init_buffers(1, dev)
    _cabi.check(L.l2h_sep_launch_count(net._engine(), None, 1))
    net.stream_dev(x.to(dev), e, chunks_per_call=1, state=st, n_calls=8)
    torch.cuda.synchronize()
    _cabi.check(L.l2h_sep_launch_count(net._engine(), ctypes.byref(n), 1))
    # per hop: front, back, 3 x (qkv, attention, attn_out); per 4-hop batch and block: W_ih GEMM, BiLSTM, mid_a, mid_b, mid_c
    assert n.value == 8 * 11 + 2 * 3 * 5 + 1 + 1


def test_one_hop_cluster_kernel_equals_separate_kernels(model, dev):
    """The latency path (one-hop calls of a few streams) runs everything of a block after the BiLSTM as ONE 16-CTA cluster
    kernel (hop_kernels.cuh: tail_kernel), which also projects the next block's BiLSTM input.  Same arithmetic per element,
    but the LayerNorm statistics are combined from per-tile partials, so not bit-identical: 1e-5 against the separate
    kernels for the output and the carried state over 70 hops (the K/V ring wraps), 1e-3 against the oracle."""
    net, sd = model
    T, B = 70, 2
    x, _ = synth.mixture(B, 128 * T, seed0=291)
    e = synth.embedding(B, seed0=292)
    xd, ed = x.to(dev), e[:, 0].to(dev)
    net.set_option("pipeline", 0)
    try:
        y_fused = net.stream_dev(xd, ed, chunks_per_call=1).cpu()
        st_fused = net._last_stream_state.to_reference()
        net.set_option("fused_tail", 0)
        y_sep = net.stream_dev(xd, ed, chunks_per_call=1).cpu()
        st_sep = net._last_stream_state.to_reference()
    finally:
        net.set_option("fused_tail", 1)
        net.set_option("pipeline", 1)
    assert rs.rel_l2(y_fused, y_sep) < 1e-5
    for i in range(3):
        for k in ("K_buf", "V_buf", "h0", "c0"):
            a, b = st_fused["gridnet_bufs"][f"buf{i}"][k], st_sep["gridnet_bufs"][f"buf{i}"][k]
            assert rs.rel_l2(a, b) < 1e-5, (i, k)
    _check(y_fused[:1], rs.sep_forward(sd, x[:1], e[:1]))
    # the reference-shaped API takes the same path: predict() hop by hop
    st = net.init_buffers(B, dev)
    xp = F.pad(xd, (0, 64))
    with torch.no_grad():
        y_pred = torch.cat([net.predict(xp[..., 128 * i:128 * i + 192], ed, st, pad=False)[0] for i in range(12)], -1).cpu()
    assert rs.rel_l2(y_pred, y_fused[..., :128 * 12]) < 1e-6


def test_one_hop_form_switches_with_the_number_of_streams(model, dev):
    """A one-hop call takes the cluster-kernel form only while all its 16-CTA clusters fit on the device at once (as
    cudaOccupancyMaxActiveClusters reports it); a call with more streams runs the separate kernels.  The same stream must come out the same (1e-5) from a
    4-stream call (cluster form) and from a 12-stream call (separate kernels), state carried over 8 hops."""
    net, _ = model
    B, T = 12, 8
    x, _ = synth.mixture(B, 128 * T, seed0=391)
    e = synth.embedding(B, seed0=392)
    xp = F.pad(x, (0, 64)).to(dev)
    ed = e[:, 0].to(dev)
    st_all, st_few = net.init_buffers(B, dev), net.init_buffers(4, dev)
    with torch.no_grad():
        y_all = torch.cat([net.predict(xp[..., 128 * i:128 * i + 192], ed, st_all, pad=False)[0] for i in range(T)], -1).cpu()
        y_few = torch.cat([net.predict(xp[:4, :, 128 * i:128 * i + 192], ed[:4], st_few, pad=False)[0] for i in range(T)], -1).cpu()
    assert rs.rel_l2(y_all[:4], y_few) < 1e-5


def test_many_frame_front_and_back_kernels_are_bit_identical(model, dev):
    """Calls of several frames start in front_many_kernel and finish in back_many_kernel (one CTA / cluster walks a chunk of a
    stream's frames: filters loaded once, rows staged once, the neighbouring frames' spectra carried) instead of one
    front_kernel CTA and one back_kernel cluster per frame: the same
    arithmetic in the same order, so outputs and the carried tails must be EQUAL -- whole clips, short calls (2, 3, 5 frames
    per call, state threaded through, clip lengths that leave a ragged last call) and a batch."""
    net, _ = model
    x, _ = synth.mixture(3, 128 * 203, seed0=591)
    e = synth.embedding(3, seed0=592)
    xd, ed = x.to(dev), e.to(dev)

    xm, _ = synth.mixture(40, 128 * 4, seed0=593)          # many streams, one hop per call: the same kernels walk (stream) items
    em = synth.embedding(40, seed0=594)[:, 0].to(dev)
    xm = xm.to(dev)

    def run_all():
        outs = [net(xd, ed).cpu(), net(xd[:1, :, :128 * 2], ed[:1]).cpu(), net(xd[:, :, :128 * 3 - 40], ed).cpu()]
        outs.append(net.stream_dev(xm, em, chunks_per_call=1).cpu())
        outs.append(net._last_stream_state.to_reference()["deconv_buf"].cpu())
        for cpc in (2, 3, 5):
            outs.append(net.stream_dev(xd[:, :, :128 * 41], ed[:, 0], chunks_per_call=cpc).cpu())
            ref = net._last_stream_state.to_reference()
            outs += [ref["conv_buf"].cpu(), ref["deconv_buf"].cpu(), ref["istft_buf"].cpu()]
        return outs

    a = run_all()
    net.set_option("back_many", 0)
    try:
        b = run_all()
    finally:
        net.set_option("back_many", 1)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_predict_host_equals_predict(model, dev):
    """Net.predict_host (pinned chunk in, pinned samples out, one C call: H2D, chain, D2H, sync) == Net.predict on device tensors."""
    net, _ = model
    x, _ = synth.mixture(2, 128 * 9, seed0=691)
    e = synth.embedding(2, seed0=692)[:, 0].to(dev)
    xp = F.pad(x, (0, 64))
    st_a, st_b = net.init_buffers(2, dev), net.init_buffers(2, dev)
    chunk = torch.empty(2, 2, 192).pin_memory()
    out = torch.empty(2, 2, 128).pin_memory()
    with torch.no_grad():
        for i in range(9):
            chunk.copy_(xp[..., 128 * i:128 * i + 192])
            ya, _ = net.predict_host(chunk, e, st_a, out=out)
            yb, _ = net.predict(xp[..., 128 * i:128 * i + 192].to(dev), e, st_b, pad=False)
            assert torch.equal(ya, yb.cpu())
    with pytest.raises(ValueError):
        net.predict_host(torch.empty(2, 2, 200).pin_memory(), e, st_a)


def test_init_buffers_in_place(model, dev):
    """init_buffers(out=state) re-initialises a state at its address (the engine's graphs are keyed on it): same pointer,
    header back to zero, and the stream that follows equals one on a new state."""
    net, _ = model
    x, _ = synth.mixture(1, 128 * 6, seed0=491)
    e = synth.embedding(1, seed0=492)[:, 0].to(dev)
    xd = x.to(dev)
    st = net.init_buffers(1, dev)
    y0 = net.stream_dev(xd, e, chunks_per_call=1, state=st).cpu()
    assert st.header()[0] == 6
    st2 = net.init_buffers(1, dev, out=st)
    assert st2.buf.data_ptr() == st.buf.data_ptr() and st2.header() == (0, 0)
    y1 = net.stream_dev(xd, e, chunks_per_call=1, state=st2).cpu()
    assert torch.equal(y0, y1)
    with pytest.raises(ValueError):
        net.init_buffers(2, dev, out=st)


def test_gate_memo_follows_weight_changes(tsh_params, dev):
    """The speaker gate is memoised in the state (the reference recomputes it every call, tfgridnet_causal.py:247-248).
    The memo key is (embedding, weight generation): after load_state_dict with a different embed_to_feats_proj a REUSED
    state with the SAME embedding must produce the new weights' output."""
    torch.manual_seed(21)
    net = Net(**tsh_params).eval().to(dev)
    x, _ = synth.mixture(1, 128 * 6, seed0=31)
    e = synth.embedding(1, seed0=32)
    xp = torch.nn.functional.pad(x, (0, 64)).to(dev)
    st = net.init_buffers(1, dev)
    with torch.no_grad():
        net.predict(xp[..., :192], e[:, 0].to(dev), st, pad=False)                # builds the gate with the old weights
        sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
        sd["tfgridnet.embed_to_feats_proj.0.weight"] = sd["tfgridnet.embed_to_feats_proj.0.weight"] * 1.7 + 0.01
        net.load_state_dict(sd)
        # same state object, same embedding, new weights: continue the stream ...
        y1 = torch.cat([net.predict(xp[..., 128 * i:128 * i + 192], e[:, 0].to(dev), st, pad=False)[0] for i in range(1, 6)], -1).cpu()
    # ... and compare with the oracle continuing from the state after hop 0 with the NEW weights
    sd_cpu = {k: v.cpu() for k, v in sd.items()}
    torch.manual_seed(21)
    sd_old = {k: v.detach().clone() for k, v in Net(**tsh_params).state_dict().items()}
    st_ref = rs.sep_init_state(sd_old, 1)
    rs.sep_predict(sd_old, xp[..., :192].cpu(), e[:, 0], st_ref, pad=False)
    y_ref = torch.cat([rs.sep_predict(sd_cpu, xp[..., 128 * i:128 * i + 192].cpu(), e[:, 0], st_ref, pad=False)[0] for i in range(1, 6)], -1)
    assert rs.rel_l2(y1, y_ref) <= 1e-3
