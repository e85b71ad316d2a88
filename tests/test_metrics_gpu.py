"""On-GPU evaluation epilogue (l2h_eval_metrics) against the formulas of the reference's evaluation loop
(reference src/ts_hear_test.py:139-146): torchmetrics SI-SNR (restated in oracle/restate.py::si_sdr and pinned
by a known-answer test) and torch's cosine_similarity."""
import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import Net, synth
from lookoncetohear_b200.metrics import eval_metrics
from oracle import restate as rs

pytestmark = pytest.mark.gpu


def _ref(outputs, target, mixture, emb, emb_gt):
    s = rs.si_sdr(outputs, target)                          # [B, C]
    si = (s - rs.si_sdr(mixture, target)).mean(dim=1)
    return torch.stack([s.mean(dim=1), si, F.cosine_similarity(emb.double(), emb_gt.double(), dim=-1)], dim=1)


@pytest.mark.parametrize("B,N", [(4, 80000), (1, 1001), (3, 64000)])
def test_metrics_match_reference_formulas(B, N):
    mix, tgt = synth.mixture(B, N, seed0=77)
    g = torch.Generator().manual_seed(5)
    out = tgt * 1.7 + 0.03 * torch.randn(B, 2, N, generator=g) + 0.2        # scaled, offset, noisy estimate
    emb, emb_gt = synth.embedding(B, seed0=10), synth.embedding(B, seed0=20)
    got = eval_metrics(out.cuda(), tgt.cuda(), mix.cuda(), emb.cuda(), emb_gt.cuda()).cpu().double()
    want = _ref(out, tgt, mix, emb[:, 0], emb_gt[:, 0])
    assert torch.allclose(got[:, :2], want[:, :2], atol=2e-3, rtol=0), (got, want)       # dB
    assert torch.allclose(got[:, 2], want[:, 2], atol=1e-6, rtol=0)


def test_metrics_of_separator_output_stay_on_device(tsh_params):
    """The evaluation step end to end: separate, then reduce to 3 floats per mixture without leaving the GPU."""
    torch.manual_seed(0)
    net = Net(**tsh_params).eval().cuda()
    mix, tgt = synth.mixture(2, 128 * 40)
    e = synth.embedding(2)
    with torch.no_grad():
        y = net(mix.cuda(), e.cuda())
        m = eval_metrics(y, tgt.cuda(), mix.cuda(), e.cuda(), e.cuda())
    assert m.is_cuda and m.shape == (2, 3)
    want = _ref(y.cpu(), tgt, mix, e[:, 0], e[:, 0])
    assert torch.allclose(m.cpu().double()[:, :2], want[:, :2], atol=2e-3, rtol=0)
    assert torch.allclose(m.cpu()[:, 2], torch.ones(2), atol=1e-6)
