"""Parity at the shapes of the remaining BASELINE.json configurations, through size-independent
properties where the oracle cannot run the full size in seconds:
  configs[2]  offline batched separation: fp32 at batch 24, and the bf16 tensor-core variant at the full batch 256
  configs[3]  batched enrollment
  configs[4]  batched streaming, many independent streams advancing one hop per step
"""
import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import EmbedTFGridNet, Net, synth
from oracle import restate as rs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def sep(tsh_params, dev):
    torch.manual_seed(0)
    net = Net(**tsh_params).eval()
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    return net.to(dev), sd


def test_offline_batch_of_4s_clips(sep, dev):
    """configs[2] shape per stream (4 s, T = 500), batch 24 (the forward splits it into independent
    launches): every stream must equal its own single-stream run (batch independence), and two of
    them are checked against the oracle."""
    net, sd = sep
    B = 24
    x, tgt = synth.mixture(B, 64000, seed0=400)
    e = synth.embedding(B, seed0=500)
    with torch.no_grad():
        y = net(x.to(dev), e.to(dev)).cpu()
        for b in (0, 7, 23):
            yb = net(x[b:b + 1].to(dev), e[b:b + 1].to(dev)).cpu()
            assert rs.rel_l2(y[b:b + 1], yb) < 1e-5
    torch.set_num_threads(8)
    for b in (3, 17):
        y_ref = rs.sep_forward(sd, x[b:b + 1], e[b:b + 1])
        assert rs.rel_l2(y[b:b + 1], y_ref) <= 1e-3
        d = (rs.si_sdr(y[b:b + 1], tgt[b:b + 1]) - rs.si_sdr(y_ref, tgt[b:b + 1])).abs().max()
        assert float(d) <= 0.1


def test_batched_streaming_many_streams(sep, dev):
    """configs[4] per-GPU shape: 256 independent streams, one 8 ms hop per step.  60 steps (the ring
    wraps); three streams are compared with the oracle, all with the buffered (whole-clip) run."""
    net, sd = sep
    B, T = 256, 60
    x, _ = synth.mixture(B, 128 * T, seed0=600)
    e = synth.embedding(B, seed0=700)
    xd, ed = x.to(dev), e[:, 0].to(dev)
    with torch.no_grad():
        y_stream = net.stream_dev(xd, ed, chunks_per_call=1).cpu()
        y_whole = net(xd, e.to(dev)).cpu()
    assert rs.rel_l2(y_stream, y_whole) < 1e-4
    # the same through the reference-shaped API: one predict() call per hop for all 256 streams
    st = net.init_buffers(B, dev)
    xp = F.pad(xd, (0, 64))
    with torch.no_grad():
        y_pred = torch.cat([net.predict(xp[..., 128 * i:128 * i + 192], ed, st, pad=False)[0] for i in range(8)], -1).cpu()
    assert rs.rel_l2(y_pred, y_whole[..., :128 * 8]) < 1e-4
    for b in (0, 101, 255):
        y_ref = rs.sep_forward(sd, x[b:b + 1], e[b:b + 1])
        assert rs.rel_l2(y_stream[b:b + 1], y_ref) <= 1e-3


def test_batched_enrollment(embed_params, dev):
    """configs[3] shape per utterance (5 s), batch 6: batch independence + oracle on one utterance
    of a shorter length (the CPU oracle needs minutes for a 5 s full-attention clip)."""
    torch.manual_seed(0)
    net = EmbedTFGridNet(**embed_params).eval()
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    net = net.to(dev)
    x = synth.enrollment(6, 80000, seed0=800)
    with torch.no_grad():
        full = net(x.to(dev)).cpu()
        one = net(x[4:5].to(dev)).cpu()
    assert torch.isfinite(full).all()
    assert rs.rel_l2(full[4:5], one) < 1e-5
    xs = synth.enrollment(2, 16000, seed0=900)
    with torch.no_grad():
        o = net(xs.to(dev)).cpu()
    r = rs.embed_forward(sd, xs)
    assert rs.rel_l2(o, r) <= 1e-3 and float(F.cosine_similarity(o, r).min()) >= 0.9999


def test_offline_bf16_batch_256(sep, dev):
    """configs[2] at its full size: 256 clips of 4 s in one forward with the bf16 option: every dense contraction takes
    bf16 WEIGHTS on the tensor cores (activations enter as bf16 hi + lo, two MMA passes; accumulation, LayerNorms,
    recurrent cell state and all element-wise work stay fp32).

    Gate.  north_star asks for |dSI-SDR| <= 0.1 dB.  With random-init weights the network does not separate: SI-SDR of
    its output against the synthetic target is -50 .. -70 dB, where the figure is ill-conditioned (rounding ONLY the
    weights to bf16 on the CPU oracle already moves it by up to 0.28 dB on clip 31 while the output changes by 4e-3).
    The well-conditioned form of the same requirement is asserted instead: the output's SNR against the fp32 oracle's
    output must be >= 36 dB.  An error of that size changes the SI-SDR of ANY estimate whose SI-SDR is <= 20 dB by
    less than 0.1 dB:  dSI-SDR = 10 log10(1 + 10^((SISDR - SNR)/10)) <= 10 log10(1 + 10^-1.6) = 0.108 -> 36.4 dB used.
    Checked on 8 of the 256 clips (the oracle runs them one by one); the raw dSI-SDR values are printed."""
    net, sd = sep
    B = 256
    x, tgt = synth.mixture(B, 64000, seed0=1400)
    e = synth.embedding(B, seed0=1500)
    net.set_option("bf16", 1)
    try:
        with torch.no_grad():
            y = net(x.to(dev), e.to(dev)).cpu()
            for b in (5, 200):
                # with bf16 operands batch independence holds only to rounding amplification: the batched and the
                # single launch pick different recurrence kernels (different fp32 summation order, ~1e-7), and a 1e-7
                # difference that flips a bf16 rounding becomes a 4e-3 relative change of that operand
                yb = net(x[b:b + 1].to(dev), e[b:b + 1].to(dev)).cpu()
                assert rs.rel_l2(y[b:b + 1], yb) < 2e-3
    finally:
        net.set_option("bf16", 0)
    assert torch.isfinite(y).all()
    torch.set_num_threads(8)
    rs.set_fast(True)
    try:
        snr_min, raw = 1e9, []
        for b in (0, 31, 64, 99, 128, 177, 222, 255):
            y_ref = rs.sep_forward(sd, x[b:b + 1], e[b:b + 1])
            snr = float(rs.si_sdr(y[b:b + 1], y_ref).min())                 # output SNR against the fp32 oracle output
            snr_min = min(snr_min, snr)
            raw.append(round(float((rs.si_sdr(y[b:b + 1], tgt[b:b + 1]) - rs.si_sdr(y_ref, tgt[b:b + 1])).abs().max()), 3))
    finally:
        rs.set_fast(False)
    print("bf16 offline: min output SNR vs fp32 oracle %.1f dB; raw |dSI-SDR| vs the synthetic target (SI-SDR ~ -60 dB): %s" % (snr_min, raw))
    assert snr_min >= 36.4, snr_min


def test_enrollment_full_length_vs_oracle(embed_params, dev):
    """configs[3] utterance length (5 s = 80 000 samples, T = 1251 frames, the full T x T attention) against the CPU
    oracle itself, not only through invariances."""
    torch.manual_seed(0)
    net = EmbedTFGridNet(**embed_params).eval()
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    net = net.to(dev)
    x = synth.enrollment(2, 80000, seed0=1700)
    with torch.no_grad():
        o = net(x.to(dev)).cpu()
    torch.set_num_threads(8)
    r = rs.embed_forward(sd, x)
    assert rs.rel_l2(o, r) <= 1e-3, rs.rel_l2(o, r)
    assert float(F.cosine_similarity(o, r).min()) >= 0.9999


def test_enrollment_batch_1024(embed_params, dev):
    """configs[3] at its full batch: 1024 utterances of 5 s through one forward() (the wrapper splits by
    l2h_embed_max_batch).  Every embedding finite; entries on both sides of the split boundaries equal their own
    single-utterance runs."""
    torch.manual_seed(0)
    net = EmbedTFGridNet(**embed_params).eval().to(dev)
    B = 1024
    x = synth.enrollment(8, 80000, seed0=1900).repeat(B // 8, 1, 1)
    x = x * torch.linspace(0.5, 2.0, B)[:, None, None]               # distinct utterances (scale is normalised away inside)
    x[:, :, 1000:1400] *= torch.arange(B)[:, None, None] % 5 + 1        # ... and not only by scale
    with torch.no_grad():
        full = net(x.to(dev)).cpu()
        assert full.shape == (B, 256) and torch.isfinite(full).all()
        for b in (0, 63, 64, 65, 511, 1023):
            one = net(x[b:b + 1].to(dev)).cpu()
            assert rs.rel_l2(full[b:b + 1], one) < 1e-5, b


def test_fused_input_projection_recurrence_option(sep, dev):
    """Engine option "fuse_ih": LayerNorm + W_ih + the recurrence as ONE tensor-core kernel (tc_lstm_x_kernel) for calls
    with >= 4096 sequence-directions.  Off by default; same gates."""
    net, sd = sep
    B = 20
    x, tgt = synth.mixture(B, 128 * 110, seed0=2400)            # 20 x 110 frames: 4400 intra sequence-directions, 1940 inter
    e = synth.embedding(B, seed0=2500)
    with torch.no_grad():
        y0 = net(x.to(dev), e.to(dev)).cpu()
        net.set_option("fuse_ih", 1)
        try:
            y1 = net(x.to(dev), e.to(dev)).cpu()
        finally:
            net.set_option("fuse_ih", 0)
    assert rs.rel_l2(y1, y0) < 1e-4
    for b in (0, 19):
        assert rs.rel_l2(y1[b:b + 1], rs.sep_forward(sd, x[b:b + 1], e[b:b + 1])) <= 1e-3


def _flat_state(ref):
    out = {}
    for k, v in ref.items():
        if isinstance(v, dict):
            out.update({f"{k}.{kk}": vv for kk, vv in _flat_state(v).items()})
        else:
            out[k] = v
    return out


@pytest.mark.parametrize("fuse_ih", [0, 1])
@pytest.mark.parametrize("chunks_per_call", [2, 5])
def test_tensor_core_recurrence_with_carried_state(sep, dev, chunks_per_call, fuse_ih):
    """Streaming calls of several hops run the inter LSTM over T > 1 steps with the (h, c) carried in the state.  With
    option "tc_lstm_min" = 1 that recurrence (and the intra one) runs on the tensor cores (tc_lstm_kernel, or with
    "fuse_ih" tc_lstm_x_kernel) even for 3 streams: output and final state must match the CUDA-core recurrences and the
    oracle."""
    net, sd = sep
    B = 3
    x, _ = synth.mixture(B, 128 * 20, seed0=2600)
    e = synth.embedding(B, seed0=2700)
    xd, ed = x.to(dev), e[:, 0].to(dev)
    with torch.no_grad():
        st0 = net.init_buffers(B, dev)
        y0 = net.stream_dev(xd, ed, chunks_per_call=chunks_per_call, state=st0).cpu()
        s0 = _flat_state(st0.to_reference())
        net.set_option("tc_lstm_min", 1)
        net.set_option("fuse_ih", fuse_ih)
        try:
            st1 = net.init_buffers(B, dev)
            y1 = net.stream_dev(xd, ed, chunks_per_call=chunks_per_call, state=st1).cpu()
            s1 = _flat_state(st1.to_reference())
        finally:
            net.set_option("tc_lstm_min", 4096)
            net.set_option("fuse_ih", 0)
    assert rs.rel_l2(y1, y0) < 1e-4
    for k in s0:
        if s0[k].abs().max() > 0:
            assert rs.rel_l2(s1[k].cpu(), s0[k].cpu()) < 1e-4, k
        else:
            assert torch.equal(s1[k], s0[k]), k
    for b in (0, 2):
        assert rs.rel_l2(y1[b:b + 1], rs.sep_forward(sd, x[b:b + 1], e[b:b + 1])) <= 1e-3
