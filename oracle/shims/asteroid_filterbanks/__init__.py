"""ORACLE SHIM (test infrastructure, never shipped / never on the product path).

Restatement of the one entry point of the un-vendored third-party package
``asteroid-filterbanks`` (pulled in by ``asteroid``, reference requirements.txt:15,
no version pinned) that the reference's separation model calls:

    make_enc_dec('stft', n_filters, kernel_size, stride, window_type=...)
        -- call site reference src/models/tfgridnet_realtime/tfgridnet_causal.py:131-135
    enc(x[B,M,N]) -> [B,M,n_filters+2,T]           -- call site :229
    dec(spec[B,S,n_filters+2,T]) -> [B,S,(T-1)*stride+kernel]   -- call site :272

Restated from the package's published algorithm (STFTFB / Encoder / Decoder), SURVEY.md
Appendix C.1; the package itself is absent from this image, so this part of the parity chain
is "unpinned" (see oracle/README.md).  The engine never regenerates these filters: it reads
them from the state_dict as weights.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


def stft_filters(n_filters: int, kernel_size: int, stride: int) -> torch.Tensor:
    """[n_filters+2, 1, kernel_size] float32: rows 0..N/2 real part, N/2+1.. imaginary part."""
    assert n_filters >= kernel_size
    cutoff = n_filters // 2 + 1
    window = np.hanning(kernel_size + 1)[:-1] ** 0.5          # sqrt periodic Hann
    fm = np.fft.fft(np.eye(n_filters))
    fm = fm / (0.5 * np.sqrt(kernel_size * n_filters / stride))
    lpad = (n_filters - kernel_size) // 2
    rpad = n_filters - kernel_size - lpad
    cols = list(range(lpad, n_filters - rpad))
    filt = np.vstack([np.real(fm[:cutoff, cols]), np.imag(fm[:cutoff, cols])])
    filt[0, :] /= np.sqrt(2)
    filt[n_filters // 2, :] /= np.sqrt(2)
    return torch.from_numpy(filt * window).unsqueeze(1).float()


class _STFTFB(nn.Module):
    def __init__(self, n_filters, kernel_size, stride, **_swallowed):
        super().__init__()
        self.n_filters, self.kernel_size, self.stride = n_filters, kernel_size, stride
        self.n_feats_out = 2 * (n_filters // 2 + 1)
        self.register_buffer("_filters", stft_filters(n_filters, kernel_size, stride))

    def filters(self):
        return self._filters


class Encoder(nn.Module):
    def __init__(self, filterbank):
        super().__init__()
        self.filterbank = filterbank

    def forward(self, wav):
        w = self.filterbank.filters()
        if wav.ndim == 1:
            return F.conv1d(wav[None, None], w, stride=self.filterbank.stride).squeeze(0)
        if wav.ndim == 2:
            return F.conv1d(wav.unsqueeze(1), w, stride=self.filterbank.stride)
        if wav.ndim == 3 and wav.shape[1] == 1:
            return F.conv1d(wav, w, stride=self.filterbank.stride)
        b, ch, n = wav.shape[0], wav.shape[1], wav.shape[-1]
        out = F.conv1d(wav.reshape(-1, 1, n), w, stride=self.filterbank.stride)
        return out.view(b, ch, w.shape[0], -1)


class Decoder(nn.Module):
    def __init__(self, filterbank):
        super().__init__()
        self.filterbank = filterbank

    def forward(self, spec):
        w = self.filterbank.filters()
        if spec.ndim == 2:
            return F.conv_transpose1d(spec.unsqueeze(0), w, stride=self.filterbank.stride).squeeze()
        if spec.ndim == 3:
            return F.conv_transpose1d(spec, w, stride=self.filterbank.stride).squeeze(1)
        lead = spec.shape[:-2]
        out = F.conv_transpose1d(spec.reshape((-1,) + spec.shape[-2:]), w, stride=self.filterbank.stride)
        return out.view(lead + (-1,))


def make_enc_dec(fb_name, n_filters, kernel_size, stride=None, sample_rate=8000.0, **kwargs):
    assert fb_name == "stft", "only the filterbank the reference uses is restated"
    enc = Encoder(_STFTFB(n_filters, kernel_size, stride, **kwargs))
    dec = Decoder(_STFTFB(n_filters, kernel_size, stride, **kwargs))
    return enc, dec
