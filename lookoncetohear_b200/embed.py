"""Drop-in for ``src.models.tfgridnet_orig.tfgridnet.EmbedTFGridNet`` (reference
tfgridnet_orig/tfgridnet.py:88-127): the enrollment network that turns a noisy binaural "look"
recording into a 256-d speaker embedding.  Select it with ``pl_module_args.model =
"lookoncetohear_b200.embed.EmbedTFGridNet"`` (plugin boundary binaural_embed_pl_module.py:19).

Same constructor keywords and the same parameter names/shapes as the reference class (whose trunk
is espnet2's TFGridNet: conv+GroupNorm, 3 non-causal GridNet blocks with per-head 1x1 convs,
an unused deconv), so a Lightning checkpoint loads unchanged.  The torch modules are parameter
containers only; the forward goes through the C ABI.
"""
import ctypes
import math

import torch
import torch.nn as nn

from . import _cabi


class _Affine4D(nn.Module):
    """gamma/beta holder named like espnet2's LayerNormalization4D / 4DCF."""

    def __init__(self, shape):
        super().__init__()
        self.gamma = nn.Parameter(torch.ones(*shape))
        self.beta = nn.Parameter(torch.zeros(*shape))


class _EmbedBlockParams(nn.Module):
    def __init__(self, emb_dim, emb_ks, n_freqs, hidden, n_head, approx_qk_dim=512):
        super().__init__()
        in_ch = emb_dim * emb_ks
        self.intra_norm = _Affine4D((1, emb_dim, 1, 1))
        self.intra_rnn = nn.LSTM(in_ch, hidden, 1, batch_first=True, bidirectional=True)
        self.intra_linear = nn.ConvTranspose1d(hidden * 2, emb_dim, emb_ks, stride=1)
        self.inter_norm = _Affine4D((1, emb_dim, 1, 1))
        self.inter_rnn = nn.LSTM(in_ch, hidden, 1, batch_first=True, bidirectional=True)
        self.inter_linear = nn.ConvTranspose1d(hidden * 2, emb_dim, emb_ks, stride=1)
        E = math.ceil(approx_qk_dim * 1.0 / n_freqs)
        for ii in range(n_head):
            self.add_module(f"attn_conv_Q_{ii}", nn.Sequential(nn.Conv2d(emb_dim, E, 1), nn.PReLU(),
                                                               _Affine4D((1, E, 1, n_freqs))))
            self.add_module(f"attn_conv_K_{ii}", nn.Sequential(nn.Conv2d(emb_dim, E, 1), nn.PReLU(),
                                                               _Affine4D((1, E, 1, n_freqs))))
            self.add_module(f"attn_conv_V_{ii}", nn.Sequential(nn.Conv2d(emb_dim, emb_dim // n_head, 1), nn.PReLU(),
                                                               _Affine4D((1, emb_dim // n_head, 1, n_freqs))))
        self.attn_concat_proj = nn.Sequential(nn.Conv2d(emb_dim, emb_dim, 1), nn.PReLU(),
                                              _Affine4D((1, emb_dim, 1, n_freqs)))


class EmbedTFGridNet(nn.Module):
    """CUDA (H100) replacement of the reference ``EmbedTFGridNet``."""

    def __init__(self, embed_dim, num_ch, n_fft, stride, num_blocks):
        super().__init__()
        emb_dim, hidden, n_head, emb_ks = 64, 64, 4, 4
        self.n_fft, self.stride, self.num_ch, self.embed_dim = n_fft, stride, num_ch, embed_dim
        self.n_freqs = n_fft // 2 + 1
        self.emb_dim = emb_dim
        self.n_layers = num_blocks
        self.conv = nn.Sequential(nn.Conv2d(2 * num_ch, emb_dim, (3, 3), padding=(1, 1)),
                                  nn.GroupNorm(1, emb_dim, eps=1e-5))
        self.blocks = nn.ModuleList([_EmbedBlockParams(emb_dim, emb_ks, self.n_freqs, hidden, n_head)
                                     for _ in range(num_blocks)])
        self.deconv = nn.ConvTranspose2d(emb_dim, 2, (3, 3), padding=(1, 1))      # unused on this path
        self.embed_proj = nn.Sequential(nn.Linear(self.n_freqs * emb_dim, embed_dim), nn.LayerNorm(embed_dim))
        self._handle = None
        self._dirty = True
        self._ws = None

    def _apply(self, fn, *args, **kwargs):
        self._dirty = True
        return super()._apply(fn, *args, **kwargs)

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        self._dirty = True
        return super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def refresh_weights(self):
        self._dirty = True

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_handle"], d["_ws"], d["_dirty"] = None, None, True
        return d

    def set_option(self, name, value):
        """"bf16": 0 = bf16x3 split products (default, fp32-grade), 1 = bf16 weights x split activations (two MMA passes),
        2 = plain bf16 tensor-core operands (one MMA pass)."""
        _cabi.check(_cabi.lib().l2h_embed_set_option(self._engine(), name.encode(), int(value)))

    def __del__(self):
        try:
            if self._handle is not None:
                _cabi.lib().l2h_embed_destroy(self._handle)
        except Exception:
            pass

    def _engine(self):
        if self._handle is None:
            h = ctypes.c_void_p()
            cfg = _cabi.EmbedConfig(self.embed_dim, self.num_ch, self.n_fft, self.stride, self.n_layers)
            _cabi.check(_cabi.lib().l2h_embed_create(ctypes.byref(cfg), ctypes.byref(h)))
            self._handle = h
        return self._handle

    def _sync_weights(self, device):
        if not self._dirty:
            return
        h, L = self._engine(), _cabi.lib()
        for name, t in self.state_dict().items():
            host = t.detach().to("cpu", torch.float32).contiguous()
            _cabi.check(L.l2h_embed_load_weight(h, name.encode(), host.data_ptr(), host.numel()))
        with torch.cuda.device(device):
            _cabi.check(L.l2h_embed_commit_weights(h, torch.cuda.current_stream(device).cuda_stream))
        self._dirty = False

    def forward(self, input):
        """input [B, M, N] -> [B, embed_dim]   (reference tfgridnet.py:100-127)."""
        if not input.is_cuda:
            raise RuntimeError("lookoncetohear_b200.EmbedTFGridNet runs only on a CUDA (sm_90a) device: "
                               "hand-written CUDA hot path, no CPU fallback")
        dev = input.device
        self._sync_weights(dev)
        x = input.contiguous().float()
        B, M, N = x.shape
        out = torch.empty(B, self.embed_dim, dtype=torch.float32, device=dev)
        L, h = _cabi.lib(), self._engine()
        per = ctypes.c_int32()
        _cabi.check(L.l2h_embed_max_batch(h, N, ctypes.byref(per)))
        per = max(1, per.value)
        for b0 in range(0, B, per):
            nb = min(per, B - b0)
            n = ctypes.c_size_t()
            _cabi.check(L.l2h_embed_workspace_bytes(h, nb, N, ctypes.byref(n)))
            if self._ws is None or self._ws.numel() < n.value or self._ws.device != dev:
                self._ws = torch.empty(n.value, dtype=torch.uint8, device=dev)
            with torch.cuda.device(dev):
                _cabi.check(L.l2h_embed_forward(h, x[b0:].data_ptr(), out[b0:].data_ptr(), nb, N,
                                                self._ws.data_ptr(), self._ws.numel(),
                                                torch.cuda.current_stream(dev).cuda_stream))
        return out
