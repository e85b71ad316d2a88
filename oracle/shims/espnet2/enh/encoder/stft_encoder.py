"""ORACLE SHIM: restatement of espnet2 STFTEncoder (package absent, no version pinned:
reference requirements.txt:19).  Semantics = the Stft.forward the reference vendors at
reference src/models/tfgridnet_orig/stft.py:68-195: torch.stft(center=True -> reflect
pad n_fft//2, periodic Hann, onesided, not normalised); multi-channel input [B,N,M] gives a
complex spectrum [B,T,M,F]."""
import torch


class STFTEncoder(torch.nn.Module):
    def __init__(self, n_fft=512, win_length=None, hop_length=128, window="hann", center=True,
                 normalized=False, onesided=True, use_builtin_complex=True):
        super().__init__()
        self.n_fft, self.win_length = n_fft, win_length or n_fft
        self.hop_length, self.window = hop_length, window
        self.center, self.normalized, self.onesided = center, normalized, onesided

    def forward(self, input, ilens=None):
        bs = input.size(0)
        multi = input.dim() == 3
        if multi:
            input = input.transpose(1, 2).reshape(-1, input.size(1))
        win = getattr(torch, f"{self.window}_window")(self.win_length, dtype=input.dtype,
                                                      device=input.device)
        out = torch.stft(input, n_fft=self.n_fft, win_length=self.win_length,
                         hop_length=self.hop_length, center=self.center, window=win,
                         normalized=self.normalized, onesided=self.onesided, return_complex=True)
        out = out.transpose(1, 2)                      # [B*M, T, F]
        if multi:
            out = out.reshape(bs, -1, out.size(1), out.size(2)).transpose(1, 2)   # [B,T,M,F]
        olens = None
        if ilens is not None:
            pad = self.n_fft // 2 if self.center else 0
            olens = torch.div(ilens + 2 * pad - self.n_fft, self.hop_length, rounding_mode="trunc") + 1
        return out, olens
