"""GPU binaural renderer: mono events + per-ear impulse responses -> binaural events, mixture and target, as the
reference's simulators and dataset do on the CPU (src/datasets/multi_ch_simulator.py:40-61 `SOFASimulator._convolve`;
src/datasets/MixLibriSpeechNoisyEnrollNorm.py:179-202 noise scaling / peak normalisation / mixture), and the band-limited
resampler of the responses and the dataset's audio (`torchaudio.functional.resample` at its defaults,
multi_ch_simulator.py:49, MixLibriSpeechNoisyEnrollNorm.py:69-75).  The arithmetic is `l2h_render_binaural` and
`l2h_resample` (hand-written CUDA).  The streaming forms of the resampler, for the serving front end, are in stream.py.
No CPU fallback."""
import ctypes
import math
import numbers

import torch

from . import _cabi


def _rates(freq, shape, what):
    """An int, or integer rates broadcastable to `shape` -> (contiguous int32 CPU tensor of one rate per row, the lowest
    rate given)."""
    t = torch.as_tensor(freq).detach().cpu()
    if t.dtype == torch.bool or t.is_complex() or (t.is_floating_point() and not bool((t == t.round()).all())):
        raise ValueError(f"{what} must be integer rates in Hz, got {freq}")
    t = t.round().to(torch.int64) if t.is_floating_point() else t.to(torch.int64)
    if t.numel() == 0 or int(t.min()) <= 0 or int(t.max()) >= 2 ** 31:
        raise ValueError(f"{what} must be positive rates below 2**31 Hz, got {freq}")
    try:
        return torch.broadcast_to(t, shape).reshape(-1).to(torch.int32).contiguous(), int(t.min())
    except RuntimeError:
        raise ValueError(f"{what} must be one rate or one per row {tuple(shape)}, got shape {tuple(t.shape)}") from None


def resample(x, orig_freq, new_freq, lowpass_filter_width=6, rolloff=0.99, resampling_method="sinc_interp_hann", beta=None):
    """`torchaudio.functional.resample(x, orig_freq, new_freq)` on the device, for many rows at once.

    x [..., n] CUDA tensor; orig_freq an int, or one rate per row (a sequence or tensor broadcastable to x.shape[:-1]);
    new_freq an int.  Returns [..., ceil(new_freq * n / min(orig_freq))] in x's dtype (computed in fp32): every row
    resampled, rows of higher `orig` zero-padded to the longest.  Rows with orig == new_freq come back unchanged, and if
    all rows have it, x itself is returned.  Only torchaudio's default method is implemented (Hann-windowed sinc,
    lowpass_filter_width=6, rolloff=0.99); the keyword arguments exist so that other settings fail loudly."""
    if resampling_method != "sinc_interp_hann" or lowpass_filter_width != 6 or rolloff != 0.99 or beta is not None:
        raise ValueError("lookoncetohear_b200.resample implements only torchaudio's default resampling "
                         "(resampling_method='sinc_interp_hann', lowpass_filter_width=6, rolloff=0.99, beta=None)")
    if not isinstance(new_freq, numbers.Integral) and not (isinstance(new_freq, float) and new_freq.is_integer()):
        raise ValueError(f"new_freq must be an integer rate in Hz, got {new_freq}")
    new = int(new_freq)
    if not 0 < new < 2 ** 31:
        raise ValueError(f"new_freq must be a positive rate below 2**31 Hz, got {new_freq}")
    if not x.is_cuda:
        raise RuntimeError("lookoncetohear_b200.resample needs a CUDA tensor (no CPU fallback)")
    if not x.is_floating_point() or x.dim() < 1:
        raise ValueError(f"x must be a floating-point tensor [..., n], got {x.dtype} {tuple(x.shape)}")
    lead, n = x.shape[:-1], x.shape[-1]
    rows = math.prod(lead)
    orig, lowest = _rates(orig_freq, lead, "orig_freq")
    if bool((orig == new).all()) and (rows > 0 or lowest == new):
        return x
    n_out = -(-new * n // lowest)                                      # the longest row
    if rows == 0 or n_out == 0:
        return x.new_zeros(*lead, n_out)
    if n_out >= 2 ** 31 or n >= 2 ** 31:
        raise ValueError(f"rows of {n} samples resampled to {n_out} are too long")
    dev = x.device
    xr = x.reshape(rows, n).to(torch.float32).contiguous()
    y = torch.empty(rows, n_out, dtype=torch.float32, device=dev)
    rates = ctypes.cast(orig.data_ptr(), ctypes.POINTER(ctypes.c_int32))       # host table, read during the call
    with torch.cuda.device(dev):
        _cabi.check(_cabi.lib().l2h_resample(xr.data_ptr(), n, n, rows, rates, new, y.data_ptr(), n_out, n_out,
                                             torch.cuda.current_stream(dev).cuda_stream))
    return y.view(*lead, n_out).to(x.dtype)


def render_binaural(srcs, rirs, noise=None, noise_scale=None, rir_sr=None, sr=16000):
    """srcs [B, S, N] mono events at rate `sr`, rirs [B, S, 2, L] impulse responses, noise [B, 2, N] binaural background or
    None, noise_scale [B] or None.  CUDA tensors.  rir_sr None: the responses are at `sr` already.  rir_sr an int, or one
    rate per batch item: the responses are at that rate and are resampled to `sr` on the device first (as the reference's
    `torchaudio.functional.resample(rir, _sr, fs)`); responses whose resampled lengths differ are zero-padded to the
    longest, which leaves the convolution unchanged.
    Returns (events [B, S, 2, N], mixture [B, 2, N], norm [B]); the target of a sample is events[:, tgt_idx]."""
    if not srcs.is_cuda:
        raise RuntimeError("lookoncetohear_b200.render.render_binaural needs CUDA tensors (no CPU fallback)")
    if srcs.dim() != 3:
        raise ValueError(f"srcs must be [B, S, N], got {tuple(srcs.shape)}")
    B, S, N = srcs.shape
    if rirs.dim() != 4 or tuple(rirs.shape[:3]) != (B, S, 2) or rirs.shape[3] < 1:
        raise ValueError(f"rirs must be [B, S, 2, L >= 1] = [{B}, {S}, 2, L], got {tuple(rirs.shape)}")
    if noise is not None and tuple(noise.shape) != (B, 2, N):
        raise ValueError(f"noise must be [B, 2, N] = [{B}, 2, {N}], got {tuple(noise.shape)}")
    if noise_scale is not None and noise_scale.numel() != B:
        raise ValueError(f"noise_scale must have one element per batch item ({B}), got {noise_scale.numel()}")
    dev = srcs.device
    src = srcs.contiguous().float()
    rir = rirs.to(dev, torch.float32).contiguous()
    if rir_sr is not None:
        per_item = torch.as_tensor(rir_sr).detach().cpu().reshape(-1)
        if per_item.numel() not in (1, B):
            raise ValueError(f"rir_sr must be one rate or one per batch item ({B}), got {per_item.numel()}")
        rir = resample(rir, per_item.view(-1, 1, 1), sr)
    L = rir.shape[-1]
    nz = noise.to(dev, torch.float32).contiguous() if noise is not None else None
    ns = noise_scale.to(dev, torch.float32).contiguous() if noise_scale is not None else None
    events = torch.empty(B, S, 2, N, dtype=torch.float32, device=dev)
    mixture = torch.empty(B, 2, N, dtype=torch.float32, device=dev)
    norm = torch.empty(B, dtype=torch.float32, device=dev)
    scratch = torch.empty(B, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _cabi.check(_cabi.lib().l2h_render_binaural(
            src.data_ptr(), rir.data_ptr(), nz.data_ptr() if nz is not None else None,
            ns.data_ptr() if ns is not None else None, B, S, N, L, events.data_ptr(), mixture.data_ptr(), norm.data_ptr(),
            scratch.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))
    return events, mixture, norm
