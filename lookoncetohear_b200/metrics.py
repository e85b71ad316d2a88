"""Evaluation epilogue on the GPU: the per-mixture figures of the reference's evaluation loop
(src/ts_hear_test.py:139-146 -- SI-SNR of the output, SI-SNR improvement over the mixture, cosine similarity of
the enrollment embedding) computed from the separator's DEVICE output by ``l2h_eval_metrics``; only three floats
per mixture cross to the host.  No CPU fallback."""
import torch

from . import _cabi


def eval_metrics(outputs, target, mixture=None, embedding=None, embedding_gt=None):
    """outputs / target / mixture: [B, C, N] CUDA tensors; embedding / embedding_gt: [B, D] or [B, 1, D], both or
    neither.  Returns a [B, 3] CUDA tensor: (output_sisnr, si_snr_i, embedding_sim); si_snr_i is 0 without a mixture,
    embedding_sim 0 without embeddings.  Shapes that do not fit raise ValueError before any launch."""
    if not outputs.is_cuda:
        raise RuntimeError("lookoncetohear_b200.metrics.eval_metrics needs CUDA tensors (no CPU fallback)")
    dev = outputs.device
    est = outputs.contiguous().float()
    tgt = target.to(dev, torch.float32).contiguous()
    if tgt.shape != est.shape:
        raise ValueError(f"target shape {tuple(tgt.shape)} != output shape {tuple(est.shape)}")
    if mixture is not None and tuple(mixture.shape) != tuple(est.shape):
        raise ValueError(f"mixture shape {tuple(mixture.shape)} != output shape {tuple(est.shape)}")
    mix = mixture.to(dev, torch.float32).contiguous() if mixture is not None else None
    B, C, N = est.shape
    if (embedding is None) != (embedding_gt is None):
        raise ValueError("embedding and embedding_gt must be given together")
    emb = emb_gt = None
    D = 0
    if embedding is not None:
        D = embedding.numel() // B if B > 0 else 0
        if D < 1 or embedding.numel() != B * D or embedding_gt.numel() != B * D:
            raise ValueError(f"embedding and embedding_gt must both reshape to [B, D] with B = {B}, got "
                             f"{tuple(embedding.shape)} and {tuple(embedding_gt.shape)}")
        emb = embedding.to(dev, torch.float32).reshape(B, D).contiguous()
        emb_gt = embedding_gt.to(dev, torch.float32).reshape(B, D).contiguous()
    out = torch.empty(B, 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _cabi.check(_cabi.lib().l2h_eval_metrics(
            est.data_ptr(), tgt.data_ptr(), mix.data_ptr() if mix is not None else None, B, C, N,
            emb.data_ptr() if emb is not None else None, emb_gt.data_ptr() if emb_gt is not None else None, D,
            out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
    return out
