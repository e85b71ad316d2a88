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
import numbers

import torch
import torch.nn as nn

from . import _cabi
from .net import device_list
from .stream import EnrollCapture


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
        2 = plain bf16 tensor-core operands (one MMA pass).
        "tc_lstm_min" (default 2048): sequence-directions from which a recurrence runs on the tensor cores."""
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

    def max_batch(self, n_samples):
        """Largest batch one engine call takes for utterances padded to n_samples (workspace bound)."""
        per = ctypes.c_int32()
        _cabi.check(_cabi.lib().l2h_embed_max_batch(self._engine(), int(n_samples), ctypes.byref(per)))
        return max(1, per.value)

    def _workspace(self, nb, n, dev):
        """the engine's shared workspace on dev, grown to what a call of nb utterances of n samples needs"""
        ws = ctypes.c_size_t()
        _cabi.check(_cabi.lib().l2h_embed_workspace_bytes(self._engine(), nb, n, ctypes.byref(ws)))
        if self._ws is None or self._ws.numel() < ws.value or self._ws.device != dev:
            self._ws = torch.empty(ws.value, dtype=torch.uint8, device=dev)
        return self._ws

    def _run(self, x, out, lens):
        """One engine call: x [nb, M, n] contiguous on the device, lens None or nb ints, out [nb, embed_dim]."""
        dev = x.device
        nb, _, n = x.shape
        ws = self._workspace(nb, n, dev)
        lens_c = None if lens is None else (ctypes.c_int32 * nb)(*lens)
        with torch.cuda.device(dev):
            _cabi.check(_cabi.lib().l2h_embed_forward_lengths(self._engine(), x.data_ptr(), n, lens_c, nb, out.data_ptr(),
                                                              ws.data_ptr(), ws.numel(),
                                                              torch.cuda.current_stream(dev).cuda_stream))

    def forward(self, input, lengths=None):
        """input [B, M, N] -> [B, embed_dim]   (reference tfgridnet.py:100-127).

        ``lengths`` (optional: B ints, or a 1-D integer tensor on any device) gives each utterance's own sample count,
        192 <= lengths[b] <= N: row b is then the embedding of ``input[b, :, :lengths[b]]`` alone, and the samples past
        it are never read.  A batch larger than one engine call takes is sorted by length and cut into calls padded
        only to their own longest utterance."""
        if not input.is_cuda:
            raise RuntimeError("lookoncetohear_b200.EmbedTFGridNet runs only on a CUDA (sm_90a) device: "
                               "hand-written CUDA hot path, no CPU fallback")
        B, M, N = input.shape
        lens = None if lengths is None else check_lengths(lengths, B, N)
        if lens is not None and all(n == N for n in lens):
            lens = None                                   # equal lengths: the equal-length call
        dev = input.device
        self._sync_weights(dev)
        x = input.contiguous().float()
        out = torch.empty(B, self.embed_dim, dtype=torch.float32, device=dev)
        per = self.max_batch(N)
        if lens is None or B <= per:
            for b0 in range(0, B, per):
                nb = min(per, B - b0)
                self._run(x[b0:b0 + nb], out[b0:b0 + nb], None if lens is None else lens[b0:b0 + nb])
            return out
        for idx, m in group_by_length(lens, self.max_batch):
            ii = torch.tensor(idx, dtype=torch.long, device=dev)
            xc = x[ii, :, :m].contiguous()
            oc = torch.empty(len(idx), self.embed_dim, dtype=torch.float32, device=dev)
            self._run(xc, oc, [lens[i] for i in idx])
            out[ii] = oc
        return out

    def enroll(self, capture, slots, lengths, out=None, used=None):
        """Embed listeners from their own streams: row b is the embedding of the last min(lengths[b], captured) samples
        that slot slots[b] of `capture` (a 2-channel `EnrollCapture`) holds, read from its ring in place on the caller's
        stream, with no host copy of the audio and nothing read back.  It equals, bit for bit, ``forward(x, lengths)``
        of those samples gathered into a batch padded to max(lengths).

        `slots` follows Net.advance_slots: n distinct ints in [0, capture slots) (a sequence or CPU tensor, checked
        here), or a contiguous CUDA int32 tensor of shape (n,) used in place and read when the kernels run, where an
        entry outside the capture marks a row that embeds nothing.  `lengths`: n ints in [192, capture.capacity].

        Returns `out` [n, 256] float32: a new tensor, or the one given, which may be a view with any row stride >= 256 --
        rows of the separator's embedding staging buffer.  A row whose slot captured fewer than 192 samples is not
        written (NaN in a new tensor), so in the staging buffer that listener keeps its embedding.  `used` (a contiguous
        CUDA int32 tensor of shape (n,), optional) receives the samples each row used, 0 for a row not written."""
        dev, slots, n, lens, out, used = self._enroll_args(capture, slots, lengths, out, used)
        n_max = max(lens)
        per = self.max_batch(n_max)
        for b0 in range(0, n, per):
            nb = min(per, n - b0)
            _slots_call(_cabi.lib().l2h_embed_forward_slots, self, capture, slots, lens, out, used, b0, nb, n_max,
                        self._workspace(nb, n_max, dev))
        return out

    def enroll_job(self, capture, slots, lengths, out=None, used=None, window=None):
        """``enroll`` in slices: returns an `EnrollJob` whose ``step(n)`` enqueues the next n units of the enrollment on
        the current stream, so a service can put a bounded amount of enrollment work between its ticks.  Arguments,
        checks and results are those of ``enroll``, bit for bit, whatever the window and however the units are stepped.

        The inter-frame recurrence, the one stage whose length grows with the utterance, runs `window` steps per unit
        (default `DEFAULT_WINDOW`, 0: the whole recurrence is one unit).  The job owns its workspace and keeps its tensors
        alive, so ``enroll``, ``forward`` and other jobs may run between its steps, as may ticks that keep writing the
        capture: the embedding is that of the samples held when the first unit ran.  `used` is final after the first unit
        of each ``max_batch`` cut; `out` rows are written by the last unit of their cut only."""
        if window is None:
            window = DEFAULT_WINDOW
        if isinstance(window, bool) or not isinstance(window, numbers.Integral) or window < 0:
            raise ValueError(f"window must be an int >= 0, got {window!r}")
        dev, slots, n, lens, out, used = self._enroll_args(capture, slots, lengths, out, used)
        return EnrollJob(self, capture, dev, slots, n, lens, out, used, int(window))

    def _enroll_args(self, capture, slots, lengths, out, used):
        """The checks of ``enroll``: (device, slot list tensor, n, lengths, out, used), the weights committed."""
        if not isinstance(capture, EnrollCapture):
            raise TypeError("capture must be an EnrollCapture")
        if capture.channels != self.num_ch:
            raise ValueError(f"enrollment needs a capture of {self.num_ch} channels, got {capture.channels}")
        dev = capture.state.device
        if isinstance(slots, torch.Tensor) and slots.is_cuda:
            n = slots.shape[0] if slots.dim() == 1 else -1
            slots = device_list(slots, dev, n, capture.n_slots, True, "slot")
        else:
            v = torch.as_tensor(slots)
            n = v.shape[0] if v.dim() == 1 else -1
            slots = device_list(v, torch.device("cpu"), n, capture.n_slots, True, "slot").contiguous()
        if n < 1:
            raise ValueError("slots must list at least one slot")
        lens = check_lengths(lengths, n, capture.capacity)
        if out is None:
            out = torch.full((n, self.embed_dim), float("nan"), dtype=torch.float32, device=dev)
        elif (not isinstance(out, torch.Tensor) or out.dtype != torch.float32 or out.device != dev
              or tuple(out.shape) != (n, self.embed_dim) or out.stride(1) != 1 or out.stride(0) < self.embed_dim):
            raise ValueError(f"out must be a float32 tensor [{n}, {self.embed_dim}] on {dev} with unit column stride and a "
                             f"row stride >= {self.embed_dim}")
        if used is None:
            used = torch.empty(n, dtype=torch.int32, device=dev)
        elif (not isinstance(used, torch.Tensor) or used.dtype != torch.int32 or used.device != dev
              or tuple(used.shape) != (n,) or not used.is_contiguous()):
            raise ValueError(f"used must be a contiguous int32 tensor of shape ({n},) on {dev}")
        self._sync_weights(dev)
        return dev, slots, n, lens, out, used


def _slots_call(entry, net, capture, slots, lens, out, used, b0, nb, n_max, ws, *tail):
    """entry (l2h_embed_forward_slots, or ..._units with `tail` = window, first unit, units) over rows b0 .. b0 + nb - 1
    of an enrollment from `capture`: a host or CUDA slot list, the rows' lengths padded to n_max, workspace ws, on the
    current stream of the capture's device"""
    dev = capture.state.device
    sl = slots[b0:b0 + nb]
    sl_host = None if sl.is_cuda else ctypes.cast(sl.data_ptr(), ctypes.POINTER(ctypes.c_int32))
    with torch.cuda.device(dev):
        _cabi.check_args(entry(
            net._engine(), capture.state.data_ptr(), capture.n_slots, capture.capacity, sl_host,
            sl.data_ptr() if sl.is_cuda else None, (ctypes.c_int32 * nb)(*lens[b0:b0 + nb]), nb, n_max,
            out[b0].data_ptr(), out.stride(0), used[b0:].data_ptr(), ws.data_ptr(), ws.numel(), *tail,
            torch.cuda.current_stream(dev).cuda_stream))


# Inter-recurrence steps per unit of an EnrollJob: 0, the whole recurrence as one unit.  Measured at 5 s (DESIGN.md
# section 7, tools/bench_enroll_slices.py), that unit is at most 7 % (8 listeners) to 25 % (1 listener) longer than the
# largest GEMM unit, which no window splits, while windows cost 7-39 % more device time in all.
DEFAULT_WINDOW = 0


class EnrollJob:
    """An enrollment enqueued in slices (``EmbedTFGridNet.enroll_job``).  ``units``: the units of the whole job (those of
    every ``max_batch`` cut, run one cut after another); ``done``: whether all were enqueued; ``step(n=1)`` enqueues the
    next n units on the current stream; ``run()`` enqueues the rest.  ``out`` and ``used`` are the tensors ``enroll``
    would return and fill."""

    def __init__(self, net, capture, dev, slots, n, lens, out, used, window):
        L, h = _cabi.lib(), net._engine()
        self.net, self.capture, self.dev, self.window = net, capture, dev, window
        self.slots, self.lens, self.out, self.used = slots, lens, out, used
        self.n_max = max(lens)
        per = net.max_batch(self.n_max)
        self._cuts = []                                    # (first row, rows, units)
        for b0 in range(0, n, per):
            nb = min(per, n - b0)
            u = ctypes.c_int32()
            _cabi.check_args(L.l2h_embed_slots_units(h, nb, self.n_max, window, ctypes.byref(u)))
            self._cuts.append((b0, nb, u.value))
        ws = ctypes.c_size_t()
        _cabi.check(L.l2h_embed_workspace_bytes(h, self._cuts[0][1], self.n_max, ctypes.byref(ws)))
        self._ws = torch.empty(ws.value, dtype=torch.uint8, device=dev)    # the job's own: shared by its cuts in turn
        self.units = sum(c[2] for c in self._cuts)
        self._next = 0

    @property
    def done(self):
        return self._next >= self.units

    def step(self, n=1):
        """Enqueue the next n units (fewer if fewer remain) on the current stream; returns how many were enqueued."""
        if isinstance(n, bool) or not isinstance(n, numbers.Integral) or n < 1:
            raise ValueError(f"n must be an int >= 1, got {n!r}")
        end = min(self.units, self._next + int(n))
        start, base = self._next, 0
        for b0, nb, units in self._cuts:
            lo, hi = max(start, base), min(end, base + units)
            if lo < hi:
                _slots_call(_cabi.lib().l2h_embed_forward_slots_units, self.net, self.capture, self.slots, self.lens,
                            self.out, self.used, b0, nb, self.n_max, self._ws, self.window, lo - base, hi - lo)
                self._next = hi
            base += units
        return end - start

    def run(self):
        """Enqueue every unit not yet enqueued; returns ``out``."""
        if not self.done:
            self.step(self.units - self._next)
        return self.out


MIN_SAMPLES = 192         # 1 + n // 64 >= 4 STFT frames for the 4-frame unfold


def check_lengths(lengths, batch, n_max):
    """Validate per-utterance lengths on the host: a list of ``batch`` Python ints in [192, n_max], else ValueError."""
    if isinstance(lengths, torch.Tensor):
        if lengths.dim() != 1 or lengths.dtype.is_floating_point or lengths.dtype.is_complex or lengths.dtype == torch.bool:
            raise ValueError(f"lengths must be a 1-D integer tensor, got {lengths.dtype} of shape {tuple(lengths.shape)}")
        lens = [int(v) for v in lengths.tolist()]
    else:
        try:
            lens = list(lengths)
        except TypeError:
            raise ValueError("lengths must be a sequence of ints or a 1-D integer tensor") from None
        for v in lens:
            if isinstance(v, bool) or not isinstance(v, numbers.Integral):
                raise ValueError(f"lengths must be integers, got {v!r}")
        lens = [int(v) for v in lens]
    if len(lens) != batch:
        raise ValueError(f"{len(lens)} lengths for a batch of {batch}")
    for b, v in enumerate(lens):
        if not MIN_SAMPLES <= v <= n_max:
            raise ValueError(f"length {v} of utterance {b} is outside [{MIN_SAMPLES}, {n_max}]")
    return lens


def group_by_length(lengths, max_batch):
    """Cut a batch into engine calls: utterances sorted by length, from the longest down, at most
    ``max_batch(longest in the call)`` per call.  Returns [(indices, pad)]: each call's indices in ascending length and
    the length it is padded to, its own longest."""
    order = sorted(range(len(lengths)), key=lambda i: lengths[i])
    chunks = []
    end = len(order)
    while end > 0:
        m = lengths[order[end - 1]]
        start = max(0, end - max(1, int(max_batch(m))))
        chunks.append((order[start:end], m))
        end = start
    return chunks
