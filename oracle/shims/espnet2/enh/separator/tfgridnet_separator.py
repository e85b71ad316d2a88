"""ORACLE SHIM (test infrastructure, never on the product path).

Restatement of ``espnet2.enh.separator.tfgridnet_separator`` -- the base class of the
reference's enrollment network (reference src/models/tfgridnet_orig/tfgridnet.py:8,
``class TFGridNet(TFGridNet)`` :11, ``EmbedTFGridNet`` :88-98).  espnet is an un-vendored,
un-pinned dependency (reference requirements.txt:19) and is absent from this image, so
the constructor and ``GridNetBlock`` are restated from the package's published algorithm
(TF-GridNet, Wang et al. 2022; SURVEY.md Appendix B / C.2).  Only ``__init__`` and
``GridNetBlock.forward`` matter: the reference overrides ``TFGridNet.forward``.

Sanity anchor available offline: the parameter count of ``EmbedTFGridNet`` built on this shim
must equal 2,368,681 (SURVEY.md section 0) -- checked in tests/test_oracle.py.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn import init
from torch.nn.parameter import Parameter

from espnet2.enh.decoder.stft_decoder import STFTDecoder
from espnet2.enh.encoder.stft_encoder import STFTEncoder
from espnet2.enh.separator.abs_separator import AbsSeparator
from espnet2.torch_utils.get_layer_from_string import get_layer


class TFGridNet(AbsSeparator):
    def __init__(self, input_dim, n_srcs=2, n_fft=128, stride=64, window="hann", n_imics=1,
                 n_layers=6, lstm_hidden_units=192, attn_n_head=4, attn_approx_qk_dim=512,
                 emb_dim=48, emb_ks=4, emb_hs=1, activation="prelu", eps=1.0e-5,
                 use_builtin_complex=False, ref_channel=-1):
        super().__init__()
        self.n_srcs = n_srcs
        self.n_layers = n_layers
        self.n_imics = n_imics
        assert n_fft % 2 == 0
        n_freqs = n_fft // 2 + 1
        self.ref_channel = ref_channel

        self.enc = STFTEncoder(n_fft, n_fft, stride, window=window,
                               use_builtin_complex=use_builtin_complex)
        self.dec = STFTDecoder(n_fft, n_fft, stride, window=window)

        t_ksize = 3
        ks, padding = (t_ksize, 3), (t_ksize // 2, 1)
        self.conv = nn.Sequential(
            nn.Conv2d(2 * n_imics, emb_dim, ks, padding=padding),
            nn.GroupNorm(1, emb_dim, eps=eps),
        )
        self.blocks = nn.ModuleList([])
        for _ in range(n_layers):
            self.blocks.append(GridNetBlock(emb_dim, emb_ks, emb_hs, n_freqs, lstm_hidden_units,
                                            n_head=attn_n_head, approx_qk_dim=attn_approx_qk_dim,
                                            activation=activation, eps=eps))
        self.deconv = nn.ConvTranspose2d(emb_dim, n_srcs * 2, ks, padding=padding)

    def forward(self, *a, **k):  # overridden by the reference subclass
        raise NotImplementedError

    @property
    def num_spk(self):
        return self.n_srcs

    @staticmethod
    def pad2(input_tensor, target_len):
        return F.pad(input_tensor, (0, target_len - input_tensor.shape[-1]))


class GridNetBlock(nn.Module):
    def __getitem__(self, key):
        return getattr(self, key)

    def __init__(self, emb_dim, emb_ks, emb_hs, n_freqs, hidden_channels, n_head=4,
                 approx_qk_dim=512, activation="prelu", eps=1e-5):
        super().__init__()
        in_channels = emb_dim * emb_ks
        self.intra_norm = LayerNormalization4D(emb_dim, eps=eps)
        self.intra_rnn = nn.LSTM(in_channels, hidden_channels, 1, batch_first=True, bidirectional=True)
        self.intra_linear = nn.ConvTranspose1d(hidden_channels * 2, emb_dim, emb_ks, stride=emb_hs)
        self.inter_norm = LayerNormalization4D(emb_dim, eps=eps)
        self.inter_rnn = nn.LSTM(in_channels, hidden_channels, 1, batch_first=True, bidirectional=True)
        self.inter_linear = nn.ConvTranspose1d(hidden_channels * 2, emb_dim, emb_ks, stride=emb_hs)

        E = math.ceil(approx_qk_dim * 1.0 / n_freqs)
        assert emb_dim % n_head == 0
        for ii in range(n_head):
            self.add_module("attn_conv_Q_%d" % ii, nn.Sequential(
                nn.Conv2d(emb_dim, E, 1), get_layer(activation)(),
                LayerNormalization4DCF((E, n_freqs), eps=eps)))
            self.add_module("attn_conv_K_%d" % ii, nn.Sequential(
                nn.Conv2d(emb_dim, E, 1), get_layer(activation)(),
                LayerNormalization4DCF((E, n_freqs), eps=eps)))
            self.add_module("attn_conv_V_%d" % ii, nn.Sequential(
                nn.Conv2d(emb_dim, emb_dim // n_head, 1), get_layer(activation)(),
                LayerNormalization4DCF((emb_dim // n_head, n_freqs), eps=eps)))
        self.add_module("attn_concat_proj", nn.Sequential(
            nn.Conv2d(emb_dim, emb_dim, 1), get_layer(activation)(),
            LayerNormalization4DCF((emb_dim, n_freqs), eps=eps)))
        self.emb_dim, self.emb_ks, self.emb_hs, self.n_head = emb_dim, emb_ks, emb_hs, n_head

    def forward(self, x):
        B, C, old_T, old_Q = x.shape
        T = math.ceil((old_T - self.emb_ks) / self.emb_hs) * self.emb_hs + self.emb_ks
        Q = math.ceil((old_Q - self.emb_ks) / self.emb_hs) * self.emb_hs + self.emb_ks
        x = F.pad(x, (0, Q - old_Q, 0, T - old_T))

        input_ = x
        intra_rnn = self.intra_norm(input_)
        intra_rnn = intra_rnn.transpose(1, 2).contiguous().view(B * T, C, Q)
        intra_rnn = F.unfold(intra_rnn[..., None], (self.emb_ks, 1), stride=(self.emb_hs, 1))
        intra_rnn = intra_rnn.transpose(1, 2)
        intra_rnn, _ = self.intra_rnn(intra_rnn)
        intra_rnn = intra_rnn.transpose(1, 2)
        intra_rnn = self.intra_linear(intra_rnn)
        intra_rnn = intra_rnn.view([B, T, C, Q]).transpose(1, 2).contiguous()
        intra_rnn = intra_rnn + input_

        input_ = intra_rnn
        inter_rnn = self.inter_norm(input_)
        inter_rnn = inter_rnn.permute(0, 3, 1, 2).contiguous().view(B * Q, C, T)
        inter_rnn = F.unfold(inter_rnn[..., None], (self.emb_ks, 1), stride=(self.emb_hs, 1))
        inter_rnn = inter_rnn.transpose(1, 2)
        inter_rnn, _ = self.inter_rnn(inter_rnn)
        inter_rnn = inter_rnn.transpose(1, 2)
        inter_rnn = self.inter_linear(inter_rnn)
        inter_rnn = inter_rnn.view([B, Q, C, T]).permute(0, 2, 3, 1).contiguous()
        inter_rnn = inter_rnn + input_

        inter_rnn = inter_rnn[..., :old_T, :old_Q]
        batch = inter_rnn
        all_Q, all_K, all_V = [], [], []
        for ii in range(self.n_head):
            all_Q.append(self["attn_conv_Q_%d" % ii](batch))
            all_K.append(self["attn_conv_K_%d" % ii](batch))
            all_V.append(self["attn_conv_V_%d" % ii](batch))
        Q = torch.cat(all_Q, dim=0)
        K = torch.cat(all_K, dim=0)
        V = torch.cat(all_V, dim=0)
        Q = Q.transpose(1, 2).flatten(start_dim=2)
        K = K.transpose(1, 2).flatten(start_dim=2)
        V = V.transpose(1, 2)
        old_shape = V.shape
        V = V.flatten(start_dim=2)
        emb_dim = Q.shape[-1]
        attn_mat = torch.matmul(Q, K.transpose(1, 2)) / (emb_dim ** 0.5)
        attn_mat = F.softmax(attn_mat, dim=2)
        V = torch.matmul(attn_mat, V)
        V = V.reshape(old_shape).transpose(1, 2)
        emb_dim = V.shape[1]
        batch = V.view([self.n_head, B, emb_dim, old_T, -1]).transpose(0, 1)
        batch = batch.contiguous().view([B, self.n_head * emb_dim, old_T, -1])
        batch = self["attn_concat_proj"](batch)
        return batch + inter_rnn


class LayerNormalization4D(nn.Module):
    def __init__(self, input_dimension, eps=1e-5):
        super().__init__()
        param_size = [1, input_dimension, 1, 1]
        self.gamma = Parameter(torch.Tensor(*param_size).to(torch.float32))
        self.beta = Parameter(torch.Tensor(*param_size).to(torch.float32))
        init.ones_(self.gamma)
        init.zeros_(self.beta)
        self.eps = eps

    def forward(self, x):
        assert x.ndim == 4
        mu_ = x.mean(dim=(1,), keepdim=True)
        std_ = torch.sqrt(x.var(dim=(1,), unbiased=False, keepdim=True) + self.eps)
        return ((x - mu_) / std_) * self.gamma + self.beta


class LayerNormalization4DCF(nn.Module):
    def __init__(self, input_dimension, eps=1e-5):
        super().__init__()
        assert len(input_dimension) == 2
        param_size = [1, input_dimension[0], 1, input_dimension[1]]
        self.gamma = Parameter(torch.Tensor(*param_size).to(torch.float32))
        self.beta = Parameter(torch.Tensor(*param_size).to(torch.float32))
        init.ones_(self.gamma)
        init.zeros_(self.beta)
        self.eps = eps

    def forward(self, x):
        assert x.ndim == 4
        mu_ = x.mean(dim=(1, 3), keepdim=True)
        std_ = torch.sqrt(x.var(dim=(1, 3), unbiased=False, keepdim=True) + self.eps)
        return ((x - mu_) / std_) * self.gamma + self.beta
