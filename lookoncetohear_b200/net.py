"""Drop-in for ``src.models.tfgridnet_realtime.net.Net`` (reference net.py:20-76).

Select it from the reference's config by pointing ``pl_module_args.model`` at
``lookoncetohear_b200.net.Net`` (the plugin boundary is ``utils.import_attr`` at
ts_hear_embed_pl_module.py:25).  Same constructor keywords, same parameter names and shapes (a
Lightning checkpoint's ``state_dict`` loads unchanged), same ``forward / predict /
init_buffers`` signatures.  The arithmetic is NOT here: every call goes through the C ABI of
``liblookonce_b200.so`` (hand-written sm_90a CUDA).  There is no PyTorch/CPU fallback -- on a
machine without the built library or without a CUDA device the calls raise.

The torch modules held below (nn.Conv2d, nn.LSTM, ...) are used purely as parameter containers,
so names / shapes / default initialisation match the reference; their ``forward`` is never run.
"""
import ctypes
import math

import torch
import torch.nn as nn

from . import _cabi

_HOP_DEFAULT = 128


class _Filterbank(nn.Module):
    """Holds the STFT filter matrix as a buffer named like asteroid's ``filterbank._filters``
    (tfgridnet_causal.py:131-135).  Values: sqrt-periodic-Hann windowed, scaled DFT rows
    (Re rows 0..N/2, then Im rows), as asteroid_filterbanks.STFTFB builds them."""

    def __init__(self, n_filters, kernel_size, stride):
        super().__init__()
        n = torch.arange(kernel_size, dtype=torch.float64)
        k = torch.arange(n_filters // 2 + 1, dtype=torch.float64)
        win = torch.sqrt(0.5 - 0.5 * torch.cos(2 * math.pi * n / kernel_size))
        ang = 2 * math.pi * k[:, None] * n[None, :] / n_filters
        scale = 1.0 / (0.5 * math.sqrt(kernel_size * n_filters / stride))
        filt = torch.cat([torch.cos(ang), -torch.sin(ang)], dim=0) * scale
        filt[0] /= math.sqrt(2.0)
        filt[n_filters // 2] /= math.sqrt(2.0)
        self.register_buffer("_filters", (filt * win).unsqueeze(1).float())


class _Codec(nn.Module):
    def __init__(self, n_filters, kernel_size, stride):
        super().__init__()
        self.filterbank = _Filterbank(n_filters, kernel_size, stride)


class _LN(nn.Module):
    """Same names as the reference's LayerNormalization4D / 4DCF wrappers (``.norm.weight``)."""

    def __init__(self, n):
        super().__init__()
        self.norm = nn.LayerNorm(n)


def _attn_branch(emb_dim, out_dim, ln_dim):
    # indices 0 (Linear), 1 (PReLU), 2 (parameter-less reshape), 3 (LayerNorm) as in the reference
    return nn.Sequential(nn.Linear(emb_dim, out_dim), nn.PReLU(), nn.Identity(), _LN(ln_dim))


class _BlockParams(nn.Module):
    """Parameter container for one GridNetBlock (tfgridnet_causal.py:301-401), same creation
    order as the reference so seeded default init reproduces the same values."""

    def __init__(self, emb_dim, n_freqs, hidden, n_head, approx_qk_dim=512):
        super().__init__()
        E = math.ceil(approx_qk_dim * 1.0 / n_freqs)
        self.intra_norm = _LN(emb_dim)
        self.intra_rnn = nn.LSTM(emb_dim, hidden, 1, batch_first=True, bidirectional=True)
        self.intra_linear = nn.Linear(hidden * 2, emb_dim)
        self.inter_norm = _LN(emb_dim)
        self.inter_rnn = nn.LSTM(emb_dim, hidden, 1, batch_first=True, bidirectional=False)
        self.inter_linear = nn.Linear(hidden, emb_dim)
        self.attn_conv_Q = _attn_branch(emb_dim, E * n_head, n_freqs * E)
        self.attn_conv_K = _attn_branch(emb_dim, E * n_head, n_freqs * E)
        self.attn_conv_V = _attn_branch(emb_dim, (emb_dim // n_head) * n_head, n_freqs * (emb_dim // n_head))
        self.attn_concat_proj = _attn_branch(emb_dim, emb_dim, n_freqs * emb_dim)


class _TFGridNetParams(nn.Module):
    def __init__(self, n_fft, stride, spk_emb_dim, emb_dim, n_layers, n_imics, n_srcs, hidden, n_head):
        super().__init__()
        n_freqs = n_fft // 2 + 1
        self.enc = _Codec(n_fft, n_fft, stride)
        self.dec = _Codec(n_fft, n_fft, stride)
        self.conv = nn.Sequential(nn.Conv2d(2 * n_imics, emb_dim, (3, 3), padding=(0, 1)))
        self.blocks = nn.ModuleList([_BlockParams(emb_dim, n_freqs, hidden, n_head) for _ in range(n_layers)])
        self.embed_to_feats_proj = nn.Sequential(nn.Linear(spk_emb_dim, emb_dim * n_freqs),
                                                 nn.LayerNorm(emb_dim * n_freqs))
        self.deconv = nn.ConvTranspose2d(emb_dim, n_srcs * 2, (3, 3), padding=(2, 1))


class SepState(dict):
    """The streaming state returned by ``Net.init_buffers`` and threaded through ``predict``.

    One contiguous device allocation (header + per-stream records, layout in csrc/sep_layout.h,
    exported through ``l2h_sep_state_offsets``) that the kernels update in place; the dict interface
    is kept because reference callers treat the state as an opaque dict they pass back.
    ``to_reference()`` / ``load_reference()`` convert to / from the reference's nested dict of
    tensors (tfgridnet_causal.py:173-186, :408-427).

    Every stream (slot) has its own frame clock, so the streams of one state need not start together or
    advance on every hop: ``reset_streams`` starts fresh streams in some slots, ``Net.predict(..., active=)``
    advances only some streams, ``copy_streams_from`` moves streams between slots and states.

    A state that ``Net.predict_targets`` runs holds groups of K records, one per target of a mixture.  Only the group's
    lead record (slot i*K) holds the mixture's conv tails and block 0's rings and (h, c), so a non-lead record is not a
    standalone stream: it continues only inside its group.  Resetting or copying whole groups keeps working.
    """

    _OFFSET_NAMES = ("ring", "k_ld", "k_dim", "v_dim", "att", "st_emb", "st_gate", "st_conv", "st_deconv",
                     "st_istft", "st_blk", "bk_k", "bk_v", "bk_h", "bk_c", "bk_stride", "st_pos", "st_calls")

    def __init__(self, buf, batch, n_blocks, header_bytes, stride, offsets, net=None):
        super().__init__()
        self.buf, self.batch, self.n_blocks = buf, batch, n_blocks
        self.header_floats, self.stride = header_bytes // 4, stride
        self.lay = dict(zip(self._OFFSET_NAMES, offsets))
        self._net = net                  # the Net whose engine runs reset_streams / copy_streams_from
        self["buf"] = buf

    # ---- views ------------------------------------------------------------------------------
    def _rec(self):
        return self.buf[self.header_floats:].view(self.batch, self.stride)

    def header(self):
        """(pos, ncalls) of the whole state: frames and calls the predict calls have covered -- synchronises."""
        h = self.buf[:4].view(torch.int64).cpu()
        return int(h[0]), int(h[1])

    def _clocks(self):
        """Views of the per-stream clocks: frames consumed [B] int64, calls [B] int32."""
        r, L = self._rec(), self.lay
        pos = r[:, L["st_pos"]:L["st_pos"] + 2].view(torch.int64)[:, 0]
        calls = r[:, L["st_calls"]:L["st_calls"] + 1].view(torch.int32)[:, 0]
        return pos, calls

    def stream_pos(self):
        """Frames each stream has consumed, a list of `batch` ints -- synchronises."""
        return self._clocks()[0].cpu().tolist()

    def _tails(self, r, par):
        """Current tails of every stream; par: one parity for all streams (views) or a [B] tensor of parities (copies)."""
        L, B = self.lay, self.batch
        sel = (slice(None), par) if isinstance(par, int) else (torch.arange(B, device=r.device), par)
        conv = r[:, L["st_conv"]:L["st_deconv"]].view(B, 2, 2, 4, 97)[sel]            # [B,slot,ch,F]
        deconv = r[:, L["st_deconv"]:L["st_istft"]].view(B, 2, 2, 97, 64)[sel]        # [B,slot,F,C]
        istft = r[:, L["st_istft"]:L["st_blk"]].view(B, 2, 2, 194)[sel]               # [B,ear,2F]
        return conv, deconv, istft

    def _block(self, r, i):
        L, B = self.lay, self.batch
        o = L["st_blk"] + i * L["bk_stride"]
        K = r[:, o + L["bk_k"]:o + L["bk_v"]].view(B, 4, L["ring"], L["k_ld"])
        V = r[:, o + L["bk_v"]:o + L["bk_h"]].view(B, 4, L["ring"], L["v_dim"])
        h = r[:, o + L["bk_h"]:o + L["bk_c"]]
        c = r[:, o + L["bk_c"]:o + L["bk_stride"]]
        return K, V, h, c

    def to_reference(self):
        """Nested dict with the reference's keys and shapes (copies; synchronises)."""
        L, r, B = self.lay, self._rec(), self.batch
        dev = self.buf.device
        pos, calls = self._clocks()
        hist = L["att"] - 1
        conv, deconv, istft = self._tails(r, (calls & 1).long())
        out = dict(conv_buf=conv.permute(0, 2, 1, 3).contiguous(),
                   deconv_buf=deconv.permute(0, 3, 1, 2).contiguous(),
                   istft_buf=istft.unsqueeze(-1).contiguous(), gridnet_bufs={})
        # ring slot of frame n is n % ring; the history rows of stream b are frames pos_b-49 .. pos_b-1 of its own clock
        frames = pos.cpu()[:, None] - hist + torch.arange(hist)[None, :]                  # [B, hist]
        slots = torch.remainder(frames, L["ring"]).to(dev)
        live = (frames >= 0).to(dev, self.buf.dtype)[:, None, :, None]
        rows = torch.arange(B, device=dev)[:, None]
        for i in range(self.n_blocks):
            K, V, h, c = self._block(r, i)
            Kh = K[rows, :, slots].permute(0, 2, 1, 3)                                     # [B, 4, hist, k_ld]
            Vh = V[rows, :, slots].permute(0, 2, 1, 3)
            out["gridnet_bufs"][f"buf{i}"] = dict(
                K_buf=(Kh[..., :L["k_dim"]] * live).reshape(B * 4, hist, L["k_dim"]).contiguous(),
                V_buf=(Vh * live).reshape(B * 4, hist, L["v_dim"]).contiguous(),
                h0=h.reshape(1, B * 97, 64).clone(), c0=c.reshape(1, B * 97, 64).clone())
        return out

    def load_reference(self, ref_state):
        """Import a state in the reference's format (the nested dict ``Net.init_buffers`` /
        ``predict`` of the reference produce) so a stream started on the reference implementation can
        be continued here.  The 49 history rows become frames 0..48 of the rings (pos = 49 for the
        header and every stream)."""
        L, r, B = self.lay, self._rec(), self.batch
        hist = L["att"] - 1
        dev, dt = self.buf.device, self.buf.dtype
        self.buf.zero_()
        hdr = self.buf[:4].view(torch.int64)
        hdr[0] = hist            # pos: frames consumed so far
        hdr[1] = 0               # ncalls: tails live in parity slot 0
        pos, calls = self._clocks()
        pos.fill_(hist)
        calls.fill_(0)
        conv, deconv, istft = self._tails(r, 0)
        conv.copy_(ref_state["conv_buf"].to(dev, dt).permute(0, 2, 1, 3))
        deconv.copy_(ref_state["deconv_buf"].to(dev, dt).permute(0, 2, 3, 1))
        istft.copy_(ref_state["istft_buf"].to(dev, dt)[..., 0])
        for i in range(self.n_blocks):
            K, V, h, c = self._block(r, i)
            g = ref_state["gridnet_bufs"][f"buf{i}"]
            K[:, :, :hist, :L["k_dim"]] = g["K_buf"].to(dev, dt).view(B, 4, hist, L["k_dim"])
            V[:, :, :hist] = g["V_buf"].to(dev, dt).view(B, 4, hist, L["v_dim"])
            h.copy_(g["h0"].to(dev, dt).reshape(B, 97 * 64))
            c.copy_(g["c0"].to(dev, dt).reshape(B, 97 * 64))
        return self

    # ---- serving many listeners ---------------------------------------------------------------
    def _engine_call(self):
        if self._net is None:
            raise ValueError("this state was not made by Net.init_buffers: it has no engine to run on")
        if self.buf.is_cuda:
            self._net._sync_weights(self.buf.device)      # the engine is bound to the device of its weights
        return self._net._engine(), _cabi.lib()

    @staticmethod
    def _slots(slots):
        s = torch.as_tensor(slots, dtype=torch.int64).flatten()
        if s.numel() == 0:
            raise ValueError("no slots given")
        return (ctypes.c_int32 * s.numel())(*s.tolist())

    def reset_streams(self, slots):
        """Start fresh streams in `slots` (a list of slot indices): their records become those of a just-initialised
        state, the other streams keep running undisturbed.  Asynchronous on the current stream."""
        h, L = self._engine_call()
        sl = self._slots(slots)
        with torch.cuda.device(self.buf.device):
            _cabi.check_args(L.l2h_sep_state_reset_streams(h, self.buf.data_ptr(), self.batch, sl, len(sl),
                                                           torch.cuda.current_stream(self.buf.device).cuda_stream))
        return self

    def copy_streams_from(self, src_state, src_slots, dst_slots):
        """Continue stream src_slots[i] of `src_state` in slot dst_slots[i] of this state: its whole record, its clock
        included, is copied, so it goes on exactly as it would have in its old slot.  The states may be the same one, or
        lie on different devices (then the records travel through host memory).  Asynchronous on the current stream."""
        if not isinstance(src_state, SepState) or src_state.stride != self.stride:
            raise ValueError("copy_streams_from: the source must be a SepState of the same network configuration")
        h, L = self._engine_call()
        ss, ds = self._slots(src_slots), self._slots(dst_slots)
        if len(ss) != len(ds):
            raise ValueError("copy_streams_from: src_slots and dst_slots differ in length")
        dev = self.buf.device
        if src_state.buf.device == dev:
            with torch.cuda.device(dev):
                _cabi.check_args(L.l2h_sep_state_copy_streams(h, self.buf.data_ptr(), self.batch, ds, src_state.buf.data_ptr(),
                                                              src_state.batch, ss, len(ss),
                                                              torch.cuda.current_stream(dev).cuda_stream))
            return self
        # another device: the records travel through host memory into a staging state here, then a same-device copy
        # imports them (its argument checks and gate-memo invalidation are the engine's)
        if min(ss) < 0 or max(ss) >= src_state.batch:
            raise ValueError(f"copy_streams_from: a source slot lies outside [0, {src_state.batch})")
        staged = self._net.init_buffers(len(ss), dev)
        staged._rec().copy_(src_state._rec()[list(ss)].cpu().to(dev))
        return self.copy_streams_from(staged, list(range(len(ss))), list(ds))

    def move_lead(self, old, new):
        """Hand the lead of a listener from record old[i] to record new[i], another record of the same listener, so that
        old[i] can be dropped from its rows (l2h_sep_state_move_lead): block 0's rings and (h, c) and the current conv tails
        of old[i] are copied into new[i], whose own blocks 1 .., back tails, gate memo and clock stay.  The clocks must be
        equal (ValueError otherwise); the call waits for the current stream to read them.  Move a TargetHistory's rings
        with it (TargetHistory.move)."""
        h, L = self._engine_call()
        o, nw = self._slots(old), self._slots(new)
        if len(o) != len(nw):
            raise ValueError("move_lead: old and new differ in length")
        with torch.cuda.device(self.buf.device):
            _cabi.check_args(L.l2h_sep_state_move_lead(h, self.buf.data_ptr(), self.batch, o, nw, len(o),
                                                       torch.cuda.current_stream(self.buf.device).cuda_stream))
        return self


class TargetHistory:
    """The block-0 history of a state's listeners (Net.target_history): ``buf`` [state.batch, frames, 97*64] fp32 on the
    state's device, record r's row the ring of the last `frames` frames of block 0's output (before the speaker gate) of
    r as a listener's lead, frame n of r's own clock in slot n mod frames.  advance_target_rows(history=) writes the rings
    of the leads it advances; Net.join_targets replays them.  24.8 KB per frame and record: 64 frames x 256 records take
    407 MB."""

    def __init__(self, state, frames):
        if not isinstance(state, SepState):
            raise TypeError("state must come from Net.init_buffers()")
        if isinstance(frames, bool) or not isinstance(frames, int) or frames < 1:
            raise ValueError(f"a history needs frames >= 1, got {frames!r}")
        self.state, self.frames = state, frames
        self.buf = torch.zeros(state.batch, frames, 97 * 64, dtype=torch.float32, device=state.buf.device)

    def check(self, state):
        """ValueError unless this is a history of `state` of the layout the engine reads"""
        if state is not self.state and state.buf.data_ptr() != self.state.buf.data_ptr():
            raise ValueError("this history belongs to another state")
        shape = (state.batch, self.frames, 97 * 64)
        if (tuple(self.buf.shape) != shape or self.buf.dtype != torch.float32 or not self.buf.is_contiguous()
                or self.buf.device != state.buf.device):
            raise ValueError(f"a history must be a contiguous float32 tensor of shape {shape} on {state.buf.device}, got "
                             f"{tuple(self.buf.shape)} {self.buf.dtype} on {self.buf.device}")

    def reset(self, records):
        """Zero the rings of `records` (a listener starting afresh in them)."""
        r = torch.as_tensor(SepState._slots(records)[:], dtype=torch.int64, device=self.buf.device)
        self.buf.index_fill_(0, r, 0.0)
        return self

    def move(self, src, dst):
        """The ring of record src[i] becomes record dst[i]'s, with SepState.move_lead."""
        s = torch.as_tensor(SepState._slots(src)[:], dtype=torch.int64, device=self.buf.device)
        d = torch.as_tensor(SepState._slots(dst)[:], dtype=torch.int64, device=self.buf.device)
        if s.numel() != d.numel():
            raise ValueError("move: src and dst differ in length")
        self.buf.index_copy_(0, d, self.buf.index_select(0, s))
        return self


# the wording of device_list's errors per list: what its entries are, a wrong count, an entry outside [0, end)
_LIST_WORDS = {"slot": ("integer slot indices", "slots lists {} records for {} input rows",
                        "a slot lies outside [0, {end})"),
               "hop": ("integer hop counts", "hops gives {} counts for {} input rows",
                       "a hop count lies outside [0, {last}] (the call's {last} hops)"),
               "record": ("integer record indices", "records lists {} records for {} target rows",
                          "a record lies outside [0, {end})"),
               "offset": ("integer row offsets", "offsets gives {} entries for {} = input rows + 1",
                          "an offset lies outside [0, {last}] (the call's {last} target rows)"),
               "lead": ("integer record indices", "leads lists {} records for {} joining records",
                        "a lead lies outside [0, {end})"),
               "count": ("integer sample counts", "counts gives {} counts for {} input rows",
                         "a count lies outside [0, {last}] (the units one input row holds)")}


def device_list(values, dev, n, end, distinct, noun):
    """`values` (slots, groups, records, offsets, hop or sample counts of a call of n rows) as the [n] int32 device tensor
    the engine reads (the separator's calls and the streaming resamplers and FIFO).  A CUDA int32 tensor is used as it is
    (its entries are read when the kernels run); anything else is checked here (n ints in [0, end), each listed once if
    `distinct`) and uploaded.  noun: a key of _LIST_WORDS, for the messages."""
    entries, count, outside = _LIST_WORDS[noun]
    if isinstance(values, torch.Tensor) and values.is_cuda:
        if values.dtype != torch.int32 or tuple(values.shape) != (n,) or not values.is_contiguous():
            raise ValueError(f"a CUDA {noun} list must be a contiguous int32 tensor of shape ({n},)")
        if values.device != dev:
            raise ValueError(f"{noun}s must live on the input's device {dev}, not {values.device}")
        return values
    v = torch.as_tensor(values)
    if v.dtype.is_floating_point or v.dtype.is_complex or v.dtype == torch.bool or v.dim() != 1:
        raise ValueError(f"{noun}s must be a sequence or 1-d tensor of {entries}")
    if v.numel() != n:
        raise ValueError(count.format(v.numel(), n))
    if n > 0 and (int(v.min()) < 0 or int(v.max()) >= end):
        raise ValueError(outside.format(end=end, last=end - 1))
    if distinct and len(set(v.tolist())) != n:
        raise ValueError(f"a {noun} is listed twice")
    return v.to(torch.int32).to(dev)


def device_offsets(offsets, dev, n, R):
    """The row offsets of a call of n listeners over R rows as the [n + 1] int32 device tensor: device_list's checks
    (entries in [0, R]), and host lists must also start at 0 and never decrease.  A CUDA tensor is used as it is; the
    kernels clamp its entries as the separator does."""
    values = device_list(offsets, dev, n + 1, R + 1, False, "offset")
    if not (isinstance(offsets, torch.Tensor) and offsets.is_cuda):
        o = torch.as_tensor(offsets).tolist()
        if o[0] != 0 or any(b < a for a, b in zip(o, o[1:])):
            raise ValueError(f"offsets must start at 0 and never decrease, got {o}")
    return values


class Net(nn.Module):
    """CUDA (H100) replacement of the reference ``Net`` (net.py:20-76)."""

    def __init__(self, stft_chunk_size=160, stft_pad_size=120, embed_dim=256, num_ch=2, D=64, B=6, I=1, J=1,
                 L=0, H=128, use_attn=False, lookahead=True, local_atten_len=100, chunk_causal=False,
                 num_src=2):
        super().__init__()
        self.stft_chunk_size = stft_chunk_size
        self.stft_pad_size = stft_pad_size
        self.num_ch = num_ch
        self.lookahead = lookahead
        self.nfft = stft_chunk_size + stft_pad_size
        self._cfg = _cabi.SepConfig(stft_chunk_size, stft_pad_size, embed_dim, num_ch, D, L, I, J, B, H,
                                    local_atten_len, int(bool(use_attn)), int(bool(lookahead)),
                                    int(bool(chunk_causal)), num_src)
        self.num_src, self.embed_dim, self.n_blocks = num_src, embed_dim, B
        self.tfgridnet = _TFGridNetParams(self.nfft, stft_chunk_size, embed_dim, D, B, num_ch, num_src, H,
                                          max(L, 1))
        self._handle = None
        self._dirty = True                      # weights need (re)packing into the engine
        self._ws = None
        # batch*frames per kernel chain: 36 clips of 500 frames (the intra recurrence then has 2 x 18 000 sequences, the inter
        # recurrence 3 492).  Chosen with an earlier tensor-core recurrence on another GPU; not re-measured on the H100
        # (tools/offline_split_experiment.py measures it)
        self.max_frames_per_launch = 18432

    # ---- engine plumbing -------------------------------------------------------------------
    def _engine(self):
        if self._handle is None:
            h = ctypes.c_void_p()
            _cabi.check(_cabi.lib().l2h_sep_create(ctypes.byref(self._cfg), ctypes.byref(h)))
            self._handle = h
        return self._handle

    def __del__(self):
        try:
            if self._handle is not None:
                _cabi.lib().l2h_sep_destroy(self._handle)
        except Exception:
            pass

    def refresh_weights(self):
        """Call after editing parameters in place; load_state_dict / .to() / .cuda() do it themselves."""
        self._dirty = True

    def __getstate__(self):
        # copy.deepcopy / pickle: the native handle, workspace and staging buffers are per-instance
        d = dict(self.__dict__)
        d["_handle"], d["_ws"], d["_dirty"] = None, None, True
        d.pop("_host_stage", None)
        d.pop("_predict_stage", None)
        d.pop("_last_stream_state", None)
        d["_cfg"] = bytes(self._cfg)
        return d

    def __setstate__(self, d):
        d = dict(d)
        d["_cfg"] = _cabi.SepConfig.from_buffer_copy(d["_cfg"])
        self.__dict__.update(d)

    def _apply(self, fn, *args, **kwargs):
        self._dirty = True
        return super()._apply(fn, *args, **kwargs)

    def _sync_weights(self, device):
        """(Re)pack the weights into the engine after construction, load_state_dict or .to()."""
        if not self._dirty:
            return
        tensors = dict(self.state_dict())
        h, L = self._engine(), _cabi.lib()
        for name, t in tensors.items():
            if name.endswith("torch_window"):
                continue
            host = t.detach().to("cpu", torch.float32).contiguous()
            _cabi.check(L.l2h_sep_load_weight(h, name.encode(), host.data_ptr(), host.numel()))
        with torch.cuda.device(device):
            _cabi.check(L.l2h_sep_commit_weights(h, torch.cuda.current_stream(device).cuda_stream))
        self._dirty = False

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        # real asteroid registers an extra (redundant) window buffer on the filterbank; accept it
        for k in [k for k in state_dict if k.startswith(prefix) and k.endswith("filterbank.torch_window")]:
            state_dict.pop(k)
        self._dirty = True
        return super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def _cached_workspace(self, device, size_query, *args):
        """(the net's workspace, grown on `device` to what size_query(handle, *args, &bytes) asks, those bytes)"""
        n = ctypes.c_size_t()
        _cabi.check(size_query(self._engine(), *args, ctypes.byref(n)))
        if self._ws is None or self._ws.numel() < n.value or self._ws.device != device:
            self._ws = torch.empty(n.value, dtype=torch.uint8, device=device)
        return self._ws, n.value

    def _workspace(self, device, batch, frames, flags=0):
        return self._cached_workspace(device, _cabi.lib().l2h_sep_workspace_bytes, batch, frames, flags)

    def _stream_workspace(self, device, batch, chunks_per_call):
        return self._cached_workspace(device, _cabi.lib().l2h_sep_stream_workspace_bytes, batch, chunks_per_call)

    def _launch(self, entry, x, emb, state, y, frames, flags=0, mask=None, slots=None, hops=None, K=1, ws=None,
                offsets=None, history=None):
        """Run the separator forward C entry point `entry` on the current stream of x's device, on the caller's tensors as
        they are (a service's fixed buffers keep the cached graph's key).  entry: "forward", "forward_active", "slots",
        "slots_frames", "slots_hops", "targets", "targets_groups" or "targets_rows" (l2h_sep_forward,
        l2h_sep_forward_<entry>).

        x [rows_x, M, N]; emb [rows, 256]; y [rows, S, N], or for the targets calls [rows_x, K, S, N], passed as its
        [rows, S, N] view; rows = rows_x * K, or for targets_rows the target rows of y.  mask: the [rows] uint8 activity
        mask of forward_active (None: all); slots: the int32 slot list (the group list of targets_groups, the record list
        of targets_rows); offsets: the int32 [rows_x + 1] row offsets of targets_rows; hops: the int32 hop counts (None:
        every row all frames).  ws: a workspace to use, else the net's own, sized for rows and frames.  history: with
        targets_rows, a TargetHistory the call writes (l2h_sep_forward_targets_rows_history).  A rejected argument raises
        ValueError, except on the dense entries, where every error is a RuntimeError."""
        dev = x.device
        self._sync_weights(dev)
        if y.dim() == 4:
            y = y.view(-1, *y.shape[2:])
        if ws is None:
            ws = self._workspace(dev, y.shape[0], frames, flags)[0]
        n = x.shape[0]
        head = (self._engine(), x.data_ptr(), x.stride(0), x.stride(1), x.shape[-1], emb.data_ptr(), state.buf.data_ptr())
        out = (y.data_ptr(), y.stride(0), y.stride(1), y.shape[-1])
        listed = (state.batch, None if slots is None else slots.data_ptr())
        hop_list = None if hops is None else hops.data_ptr()
        with torch.cuda.device(dev):
            tail = (ws.data_ptr(), ws.numel(), flags, torch.cuda.current_stream(dev).cuda_stream)
            if entry == "forward":
                args = (*head, *out, n, frames, *tail)
            elif entry == "forward_active":
                args = (*head, *out, n, frames, *tail, None if mask is None else mask.data_ptr())
            elif entry == "slots":
                args = (*head, *listed, n, *out, *tail)
            elif entry == "slots_frames":
                args = (*head, *listed, n, frames, *out, *tail)
            elif entry == "slots_hops":
                args = (*head, *listed, hop_list, n, frames, *out, *tail)
            elif entry == "targets":
                args = (*head, *out, n, K, frames, *tail)
            elif entry == "targets_rows":
                args = (*head, *listed, offsets.data_ptr(), hop_list, n, y.shape[0], frames, *out, *tail)
                if history is not None:
                    entry = "targets_rows_history"
                    args = (*args, history.buf.data_ptr(), history.frames)
            else:
                args = (*head, *listed, hop_list, n, K, frames, *out, *tail)
            fn = getattr(_cabi.lib(), "l2h_sep_" + entry if entry.startswith("forward") else "l2h_sep_forward_" + entry)
            (_cabi.check if entry.startswith("forward") else _cabi.check_args)(fn(*args))

    def set_option(self, name, value):
        """Engine switches: "pipeline" (wavefront pipelining of one-hop calls), "pdl", "fused_tail", "pipeline_frames"
        and the lanes per pipeline stage: "pipeline_lanes" (BiLSTM), "pipeline_qkv_lanes", "pipeline_midc_lanes",
        "pipeline_attn_lanes", "pipeline_out_lanes", "pipeline_front_lanes", "pipeline_back_lanes".  The full list is in
        include/lookonce_b200.h (l2h_sep_set_option)."""
        _cabi.check(_cabi.lib().l2h_sep_set_option(self._engine(), name.encode(), int(value)))

    def reset_options(self):
        """Pipeline lane counts / hops per graph / PDL stages back to the engine defaults."""
        self.set_option("defaults", 0)

    def pipeline_frames(self):
        k = ctypes.c_int32()
        _cabi.check(_cabi.lib().l2h_sep_pipeline_frames(self._engine(), ctypes.byref(k)))
        return k.value

    @staticmethod
    def _require_cuda(t):
        if not t.is_cuda:
            raise RuntimeError("lookoncetohear_b200.Net runs only on a CUDA (sm_90a) device: the hot path is "
                               "hand-written CUDA with no CPU fallback")

    # ---- reference API ---------------------------------------------------------------------
    def init_buffers(self, batch_size, device, out=None):
        """Fresh streaming state for `batch_size` streams (net.py:40-41 of the reference).  `out`: a SepState of the same batch
        size to re-initialise IN PLACE -- the engine's cached CUDA graphs are keyed on the state's address, so a service that
        resets a stream keeps its graphs warm this way (a new allocation means one more capture + instantiation of the
        clip-sized pipelined graph, ~0.1-0.4 s)."""
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("lookoncetohear_b200.Net.init_buffers: CUDA device required (no CPU fallback)")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        L, h = _cabi.lib(), self._engine()
        n = ctypes.c_size_t()
        _cabi.check(L.l2h_sep_state_bytes(h, batch_size, ctypes.byref(n)))
        hb, stride, offs = self._state_layout()
        if out is not None and (out.batch != batch_size or out.buf.device != device or out.buf.numel() != n.value // 4):
            raise ValueError("init_buffers(out=...): the state to reuse has another batch size, device or layout")
        buf = out.buf if out is not None else torch.empty(n.value // 4, dtype=torch.float32, device=device)
        with torch.cuda.device(device):
            _cabi.check(L.l2h_sep_state_init(h, buf.data_ptr(), batch_size,
                                             torch.cuda.current_stream(device).cuda_stream))
        return SepState(buf, batch_size, self.n_blocks, hb, stride, offs, net=self)

    def _state_layout(self):
        """(header bytes, floats per stream record, record offsets) from the C side."""
        L, h = _cabi.lib(), self._engine()
        hb, stride = ctypes.c_int64(), ctypes.c_int64()
        _cabi.check(L.l2h_sep_state_layout(h, ctypes.byref(hb), ctypes.byref(stride)))
        n = len(SepState._OFFSET_NAMES)
        offs = (ctypes.c_int64 * n)()
        _cabi.check(L.l2h_sep_state_offsets(h, offs, n))
        return hb.value, stride.value, list(offs)

    def _run(self, x, embed, state, frames, out_len, flags=0, active=None, slots=None, hops=None):
        """x [B,M,n] (any length; samples beyond n read as zero), embed [B,256], active: [B] uint8 device mask or None,
        slots: [B] int32 device list of the state's records the rows advance by `frames` hops, or None; hops: with
        slots, [B] int32 device list of the hops each row advances instead (at most `frames`), or None."""
        self._require_cuda(x)
        Bsz = x.shape[0]
        if slots is None and state.batch != Bsz:
            raise ValueError(f"state was built for batch {state.batch}, input has batch {Bsz}")
        y = torch.empty(Bsz, self.num_src, out_len, dtype=torch.float32, device=x.device)
        self._launch("forward_active" if slots is None else "slots_hops", x.contiguous().float(),
                     embed.to(x.device, torch.float32).contiguous(), state, y, frames, flags, mask=active, slots=slots,
                     hops=hops)
        return y

    @staticmethod
    def _active_mask(active, dev, batch):
        """`active` of predict as the [batch] uint8 device tensor the engine reads."""
        if not isinstance(active, torch.Tensor) or active.dtype not in (torch.bool, torch.uint8):
            raise ValueError("active must be a bool or uint8 tensor")
        if active.device != dev:
            raise ValueError(f"active must live on the input's device {dev}, not {active.device}")
        if tuple(active.shape) != (batch,):
            raise ValueError(f"active must have shape ({batch},), got {tuple(active.shape)}")
        return active.contiguous().view(torch.uint8)

    @classmethod
    def _slot_list(cls, slots, dev, n, batch):
        """slots (or groups) of a call of n rows: n distinct ints in [0, batch), or a CUDA int32 list used in place"""
        return device_list(slots, dev, n, batch, True, "slot")

    @classmethod
    def _hop_counts(cls, hops, dev, n, frames):
        """hop counts of a call of n rows and `frames` hops: n ints in [0, frames], or a CUDA int32 list used in place"""
        return device_list(hops, dev, n, frames + 1, False, "hop")

    def _frames(self, n, pad=False, who="pad=False", per=""):
        """(frames, output samples) of a call on n input samples: pad=True rounds up to whole hops and returns n samples;
        pad=False takes 128*T + 64 samples (the look-ahead included) and returns 128*T.  who / per word the ValueError."""
        hop, la = self.stft_chunk_size, self.stft_pad_size
        if pad:
            return (n + hop - 1) // hop, n
        if (n - la) % hop != 0 or n < hop + la:
            raise ValueError(f"{who} needs {hop}*T+{la} samples{per}, got {n}")
        return (n - la) // hop, (n - la) // hop * hop

    def predict(self, x, embed, input_state, pad=True, active=None, slots=None):
        """Reference net.py:54-66.  x [B,M,N]; embed [B,256]; returns (y [B,S,*], state).

        active: None, or for a one-hop call a [B] bool / uint8 CUDA tensor: only the streams with a true entry advance.
        The others are untouched -- record, clock and speaker-gate memo -- and their rows of y are left unwritten.

        slots: None, or for a one-hop call the records of `input_state` the B input rows advance: row i continues stream
        slots[i], and the call costs what B streams cost, whatever the state's size.  Records not listed are not read or
        written.  Either B distinct ints in [0, state.batch) (a sequence or CPU tensor, checked and uploaded), or a CUDA
        int32 tensor used in place: there an entry outside [0, state.batch) marks a row that stores nothing (its y row is
        left unwritten), and listing a slot twice is the caller's error.  Cannot be combined with `active`."""
        hop, la = self.stft_chunk_size, self.stft_pad_size
        frames, out_len = self._frames(x.shape[-1], pad)
        if not isinstance(input_state, SepState):
            raise TypeError("input_state must come from Net.init_buffers()")
        if slots is not None:
            if active is not None:
                raise ValueError("slots and active cannot be combined: skip a stream by leaving it out of the list")
            if frames != 1:
                raise ValueError(f"slots needs a one-hop call ({hop}+{la} samples with pad=False), this call has {frames} hops")
            self._require_cuda(x)
            slots = self._slot_list(slots, x.device, x.shape[0], input_state.batch)
        if active is not None:
            if frames != 1:
                raise ValueError(f"active needs a one-hop call ({hop}+{la} samples with pad=False), this call has {frames} hops")
            self._require_cuda(x)
            active = self._active_mask(active, x.device, x.shape[0])
        y = self._run(x, embed, input_state, frames, out_len, active=active, slots=slots)
        return y, input_state

    def advance_slots(self, x, embed, state, slots, hops=None):
        """Advance record slots[i] of `state` by T hops with row i of x [n, M, 128*T + 64] (the pad=False shape) and
        embed [n, 256]; returns y [n, S, 128*T].  A listener whose chunks arrived late catches up its backlog of T hops
        in one call: the T hops' BiLSTMs run side by side, as in a dense multi-hop predict.

        `slots` is checked as for predict(slots=): n distinct ints in [0, state.batch) (a sequence or CPU tensor, checked
        and uploaded), or a CUDA int32 tensor used in place, where an entry outside [0, state.batch) marks a row that
        stores nothing for all of its hops.  predict(slots=) remains the one-hop form.

        `hops`: None (every row advances T hops), or the hops h_i in [0, T] row i advances, so listeners with different
        backlogs catch up in one call (l2h_sep_forward_slots_hops).  Row i reads only samples 0 .. 128*h_i + 63 of its x
        row and writes only y[i, :, :128*h_i]: its later y samples are left unwritten.  Its record ends exactly where h_i
        hops leave it, and h_i = 0 stores nothing.  Either n ints (a sequence or CPU tensor, checked and uploaded), or a
        contiguous CUDA int32 tensor of shape (n,) used in place, as for `slots`: there an entry outside [0, T] counts
        as 0.  With fixed slot and hop tensors rewritten in place every tick, one cached graph per (n, T) serves every
        mix of backlogs up to T."""
        if x.dim() != 3:
            raise ValueError(f"advance_slots needs x of shape [n, channels, {self.stft_chunk_size}*T+{self.stft_pad_size}], "
                             f"got {tuple(x.shape)}")
        frames, out_len = self._frames(x.shape[-1], who="advance_slots", per=" per row")
        if not isinstance(state, SepState):
            raise TypeError("state must come from Net.init_buffers()")
        if hops is not None:
            hops = self._hop_counts(hops, x.device, x.shape[0], frames)
        self._require_cuda(x)
        slots = self._slot_list(slots, x.device, x.shape[0], state.batch)
        return self._run(x, embed, state, frames, out_len, slots=slots, hops=hops)

    def forward(self, x, embeds, input_state=None, pad=True):
        """Reference net.py:68-76.  x [B,M,N]; embeds [B,1,256] -> [B,S,N]."""
        embeds = embeds[:, 0]
        Bsz = x.shape[0]
        frames = self._frames(x.shape[-1], pad=True)[0]
        # independent streams: split the batch so batch*frames stays inside the workspace bound
        per = max(1, self.max_frames_per_launch // max(frames, 1))
        if input_state is not None or Bsz <= per:
            if input_state is None:
                input_state = self.init_buffers(Bsz, x.device)
            y, _ = self.predict(x, embeds, input_state, pad)
            return y
        outs = []
        for b0 in range(0, Bsz, per):
            xs, es = x[b0:b0 + per], embeds[b0:b0 + per]
            st = self.init_buffers(xs.shape[0], x.device)
            outs.append(self.predict(xs, es, st, pad)[0])
        return torch.cat(outs, dim=0)

    # ---- several targets per mixture ---------------------------------------------------------
    def _targets_shape(self, x, embeds):
        """(B, K) of x [B, M, N] and embeds [B, K, 256], or ValueError."""
        if x.dim() != 3:
            raise ValueError(f"x must have shape [B, channels, N], got {tuple(x.shape)}")
        if (not isinstance(embeds, torch.Tensor) or embeds.dim() != 3 or embeds.shape[0] != x.shape[0]
                or embeds.shape[1] < 1 or embeds.shape[2] != self.embed_dim):
            shape = tuple(embeds.shape) if isinstance(embeds, torch.Tensor) else type(embeds).__name__
            raise ValueError(f"embeds must have shape [B, K, {self.embed_dim}] with B = {x.shape[0]} mixtures and K >= 1 "
                             f"targets, got {shape}")
        return x.shape[0], embeds.shape[1]

    def predict_targets(self, x, embeds, state, pad=True):
        """Extract K enrolled speakers from each of B mixtures in one call (l2h_sep_forward_targets).  x [B,M,N]; embeds
        [B,K,256], one embedding per target; state from init_buffers(B*K), in groups of K records: record i*K + k is target
        k of mixture i.  Returns (y [B,K,S,*], state); `pad` as for predict (pad=False with 128*T + 64 samples is a T-hop
        call).

        The front and block 0 do not depend on the speaker, so they run once per mixture, on the group's lead record
        i*K; the other records of a group never hold them, which makes a non-lead record no standalone stream (see
        SepState).  Each target gets the output of predict on its mixture alone, up to the rounding of one stage in the
        fused one-hop form (include/lookonce_b200.h)."""
        Bsz, K = self._targets_shape(x, embeds)
        frames, out_len = self._frames(x.shape[-1], pad)
        if not isinstance(state, SepState):
            raise TypeError("state must come from Net.init_buffers()")
        if state.batch != Bsz * K:
            raise ValueError(f"state was built for batch {state.batch}, a call of {Bsz} mixtures x {K} targets needs "
                             f"init_buffers({Bsz * K})")
        return self._run_targets("targets", x, embeds, state, frames, out_len), state

    def _run_targets(self, entry, x, embeds, state, frames, out_len, groups=None, hops=None):
        """y [B, K, S, out_len] of the targets call `entry` on x [B, M, N] and embeds [B, K, 256]"""
        self._require_cuda(x)
        Bsz, K = embeds.shape[:2]
        y = torch.empty(Bsz, K, self.num_src, out_len, dtype=torch.float32, device=x.device)
        self._launch(entry, x.contiguous().float(), embeds.to(x.device, torch.float32).reshape(Bsz * K, self.embed_dim)
                     .contiguous(), state, y, frames, slots=groups, hops=hops, K=K)
        return y

    def forward_targets(self, x, embeds):
        """x [B,M,N], embeds [B,K,256] -> [B,K,S,N]: every mixture separated for each of its K targets, on a fresh state,
        padded as forward() pads.  Long batches are split as forward() splits them, counting target rows."""
        Bsz, K = self._targets_shape(x, embeds)
        frames = self._frames(x.shape[-1], pad=True)[0]
        per = max(1, self.max_frames_per_launch // max(frames * K, 1))
        outs = []
        for b0 in range(0, Bsz, per):
            xs, es = x[b0:b0 + per], embeds[b0:b0 + per]
            st = self.init_buffers(xs.shape[0] * K, x.device)
            outs.append(self.predict_targets(xs, es, st)[0])
        return outs[0] if len(outs) == 1 else torch.cat(outs, dim=0)

    def advance_targets(self, x, embeds, state, groups, hops=None):
        """Advance listed groups of a targets state by T hops each (l2h_sep_forward_targets_groups): the slot-list calls of
        advance_slots for listeners who each want K speakers.  x [n, M, 128*T + 64] (the pad=False shape), row i the mixture
        of group groups[i]; embeds [n, K, 256]; state from init_buffers(G*K), in the layout of predict_targets: record
        g*K + k is target k of group g.  Returns y [n, K, S, 128*T].  The front and block 0 run once per listed group, the
        rest once per target; groups not listed are neither read nor written.  T = 1 is the one-hop tick.

        `groups` follows the rules of predict(slots=), counted in groups: n distinct ints in [0, G) (a sequence or CPU tensor,
        checked and uploaded), or a contiguous CUDA int32 tensor of shape (n,) used in place, where an entry outside [0, G)
        marks a group that stores nothing.  `hops` follows advance_slots(hops=): None (every group advances T hops), or the
        hops h_i in [0, T] group i advances; its K rows of y receive only y[i, :, :, :128*h_i].  With fixed tensors rewritten
        in place every tick, one cached graph per (n, K, T) serves every tick.  Reset or copy whole groups of K records
        (reset_streams(range(g*K, g*K + K)))."""
        n, K = self._targets_shape(x, embeds)
        frames, out_len = self._frames(x.shape[-1], who="advance_targets", per=" per row")
        if not isinstance(state, SepState):
            raise TypeError("state must come from Net.init_buffers()")
        if state.batch % K != 0:
            raise ValueError(f"a state of {state.batch} records does not hold groups of {K} targets: use init_buffers(G*{K})")
        if hops is not None:
            hops = self._hop_counts(hops, x.device, n, frames)
        groups = self._slot_list(groups, x.device, n, state.batch // K)
        return self._run_targets("targets_groups", x, embeds, state, frames, out_len, groups, hops)

    def advance_target_rows(self, x, embeds, state, records, offsets, hops=None, history=None):
        """Advance listeners who each enrolled their own number of speakers by T hops each, in one call
        (l2h_sep_forward_targets_rows): advance_targets without its one K for every listener.  x [n, M, 128*T + 64] (the
        pad=False shape), row i listener i's mixture; embeds [R, 256], one row per target row; listener i owns target rows
        offsets[i] .. offsets[i+1]-1, and target row r continues record records[r] of `state`.  Returns y [R, S, 128*T]:
        row r is target row r's speaker.  Rows from offsets[n] on belong to no listener: they store nothing and their y rows
        are left unwritten, so one fixed R carries any number of live targets.

        A listener's lead record, records[offsets[i]], also holds its mixture's front and block 0; its other records never
        do, so reset a listener's records together (reset_streams of all of them) before its first call, or add a record
        to a running listener with join_targets.  Drop a target by leaving its row out of the next call; drop a lead with
        state.move_lead first.  Records need not be adjacent or in order.  Host lists (sequences or CPU tensors) are checked and uploaded: `records` R distinct ints
        in [0, state.batch); `offsets` n + 1 ints from 0, non-decreasing, at most R; `hops` as for advance_targets (None:
        every listener advances T hops; else h_i in [0, T], and listener i's rows receive y[r, :, :128*h_i] only).  CUDA
        int32 tensors are used in place and read when the kernels run: there a record outside the state marks a row that
        stores nothing, and the engine clamps the offsets to be non-decreasing and at most R.  With fixed tensors rewritten in
        place every tick, one cached graph per (n, R, T) serves every mix of listeners.

        history: None, or a TargetHistory of `state` (target_history): the call also writes each listener's advanced
        frames of block 0's output into its lead's ring, for join_targets to replay; y and the state are those of the call
        without it, bit for bit."""
        if x.dim() != 3:
            raise ValueError(f"advance_target_rows needs x of shape [n, channels, {self.stft_chunk_size}*T+"
                             f"{self.stft_pad_size}], got {tuple(x.shape)}")
        if not isinstance(embeds, torch.Tensor) or embeds.dim() != 2 or embeds.shape[1] != self.embed_dim:
            shape = tuple(embeds.shape) if isinstance(embeds, torch.Tensor) else type(embeds).__name__
            raise ValueError(f"embeds must have shape [R, {self.embed_dim}], one row per target row, got {shape}")
        frames, out_len = self._frames(x.shape[-1], who="advance_target_rows", per=" per row")
        if not isinstance(state, SepState):
            raise TypeError("state must come from Net.init_buffers()")
        n, R = x.shape[0], embeds.shape[0]
        if not 0 < n <= R <= state.batch:
            raise ValueError(f"advance_target_rows needs 0 < n <= R <= state.batch, got n = {n} listeners, R = {R} target "
                             f"rows and a state of {state.batch} records")
        dev = x.device
        if hops is not None:
            hops = self._hop_counts(hops, dev, n, frames)
        if history is not None:
            if not isinstance(history, TargetHistory):
                raise TypeError("history must come from Net.target_history()")
            history.check(state)
        records = device_list(records, dev, R, state.batch, True, "record")
        offsets = device_offsets(offsets, dev, n, R)
        self._require_cuda(x)
        y = torch.empty(R, self.num_src, out_len, dtype=torch.float32, device=dev)
        self._launch("targets_rows", x.contiguous().float(), embeds.to(dev, torch.float32).contiguous(), state, y, frames,
                     slots=records, hops=hops, offsets=offsets, history=history)
        return y

    def target_history(self, state, frames):
        """A block-0 history of `frames` frames for the listeners of `state` (TargetHistory), zeroed: pass it to every
        advance_target_rows of those listeners, and join_targets can bring a new target up to a listener's clock."""
        return TargetHistory(state, frames)

    def join_targets(self, state, records, leads, embeds, history=None, frames=None, out=None, used=None, flags=0, ws=None):
        """Add target records to running listeners (l2h_sep_join_targets): record records[j] joins the listener whose lead
        record is leads[j], with embedding embeds[j] ([J, 256]).  The record becomes a fresh record at the lead's clock p
        minus W_j = min(frames, history.frames, p), its gate memo is built, and blocks 1 .. B-1 and the back replay those
        W_j frames of the lead's history, so it ends at clock p, warm.  With a history that covers the whole stream it is
        the record the target would have had from the start.  frames: None (history.frames, or 0 without a history); 0 or
        no history is a cold join (fresh deep state at the lead's clock).  Then list records[j] among the listener's rows
        in the next advance_target_rows.

        Returns (y [J, S, 128*frames], used [J] int32 on the device): row j of y holds the output of the W_j replayed
        frames in its first 128*W_j samples, the rest is left unwritten; used[j] = W_j.  out / used: fixed tensors to write
        instead (a service's buffers keep the cached graph's key with flags=L2H_FLAG_GRAPH).  Host lists are checked:
        records J distinct ints and leads J ints in [0, state.batch), no record equal to any listed lead.  CUDA int32
        tensors are used in place and read when the kernels run: there a record or lead outside the state, a record
        listed twice or a record equal to a listed lead marks a row that stores nothing (used 0).

        ws: a uint8 CUDA tensor of at least l2h_sep_workspace_bytes(J, max(1, min(frames, history.frames))) bytes to use,
        else the net's own workspace, grown if the join needs more than it holds.  The ticks' cached graphs are keyed on
        their workspace, so a service passes its own buffer here (or one to the ticks) and no tick recaptures its graph
        after a join.  A join reads its leads' clocks and rings and counts as a call of its state: enqueue it on the
        stream of that state's ticks, never beside one."""
        if not isinstance(state, SepState):
            raise TypeError("state must come from Net.init_buffers()")
        if not isinstance(embeds, torch.Tensor) or embeds.dim() != 2 or embeds.shape[1] != self.embed_dim:
            shape = tuple(embeds.shape) if isinstance(embeds, torch.Tensor) else type(embeds).__name__
            raise ValueError(f"embeds must have shape [J, {self.embed_dim}], one row per joining record, got {shape}")
        J = embeds.shape[0]
        if not 0 < J <= state.batch:
            raise ValueError(f"join_targets needs 0 < J <= state.batch, got J = {J} and a state of {state.batch} records")
        if history is not None:
            if not isinstance(history, TargetHistory):
                raise TypeError("history must come from Net.target_history()")
            history.check(state)
        if frames is None:
            frames = history.frames if history is not None else 0
        if isinstance(frames, bool) or not isinstance(frames, int) or frames < 0:
            raise ValueError(f"frames must be an int >= 0, got {frames!r}")
        dev = state.buf.device
        # a CUDA list is read when the kernels run: join_start_kernel makes a clashing row store nothing
        if not (isinstance(records, torch.Tensor) and records.is_cuda) and not (isinstance(leads, torch.Tensor) and leads.is_cuda):
            r, l = torch.as_tensor(records).flatten().tolist(), torch.as_tensor(leads).flatten().tolist()
            if set(r) & set(l):
                raise ValueError(f"a joining record is a listed lead: {sorted(set(r) & set(l))}")
        records = device_list(records, dev, J, state.batch, True, "record")
        leads = device_list(leads, dev, J, state.batch, False, "lead")
        replay = min(frames, history.frames) if history is not None else 0
        y = out if out is not None else torch.empty(J, self.num_src, 128 * frames, dtype=torch.float32, device=dev)
        if (not isinstance(y, torch.Tensor) or y.dim() != 3 or y.shape[0] != J or y.shape[1] != self.num_src
                or y.shape[2] < 128 * replay or y.stride(2) != 1 or y.dtype != torch.float32 or y.device != dev):
            shape = (tuple(y.shape), y.dtype, y.device) if isinstance(y, torch.Tensor) else type(y).__name__
            raise ValueError(f"out must be a float32 tensor [J, {self.num_src}, >= {128 * replay}] with unit sample stride on "
                             f"{dev}, got {shape}")
        if used is None:
            used = torch.empty(J, dtype=torch.int32, device=dev)
        elif used.dtype != torch.int32 or tuple(used.shape) != (J,) or used.device != dev or not used.is_contiguous():
            raise ValueError(f"used must be a contiguous int32 tensor of shape ({J},) on {dev}")
        self._require_cuda(state.buf)
        self._sync_weights(dev)
        if ws is None:
            ws, ws_bytes = self._workspace(dev, J, max(1, replay), flags)
        else:
            need = ctypes.c_size_t()
            _cabi.check(_cabi.lib().l2h_sep_workspace_bytes(self._engine(), J, max(1, replay), flags, ctypes.byref(need)))
            if (not isinstance(ws, torch.Tensor) or ws.dtype != torch.uint8 or ws.device != dev or not ws.is_contiguous()
                    or ws.numel() < need.value):
                raise ValueError(f"ws must be a contiguous uint8 tensor of at least {need.value} bytes on {dev}")
            ws_bytes = ws.numel()
        with torch.cuda.device(dev):
            _cabi.check_args(_cabi.lib().l2h_sep_join_targets(
                self._engine(), records.data_ptr(), leads.data_ptr(), embeds.to(dev, torch.float32).contiguous().data_ptr(), J,
                state.buf.data_ptr(), state.batch, None if history is None else history.buf.data_ptr(),
                0 if history is None else history.frames, frames, y.data_ptr() if y.numel() else None, y.stride(0),
                y.stride(1), used.data_ptr(), ws.data_ptr(), ws_bytes, flags,
                torch.cuda.current_stream(dev).cuda_stream))
        return y, used

    def stream_dev(self, x_dev, embed_dev, chunks_per_call=1, state=None, n_calls=None, out=None):
        """Streaming over a device-resident clip (l2h_sep_stream_dev): x_dev [B,M,N] is consumed
        chunks_per_call hops per call with the state carried, every call one CUDA-graph replay.
        Returns y [B,S,N] (device).  Asynchronous."""
        self._require_cuda(x_dev)
        dev = x_dev.device
        self._sync_weights(dev)
        hop = self.stft_chunk_size
        x = x_dev.contiguous().float()
        Bsz, _, n = x.shape
        step = hop * chunks_per_call
        if n_calls is None:
            n_calls = (n + step - 1) // step
        if state is None:
            state = self.init_buffers(Bsz, dev)
        y = out if out is not None else torch.empty(Bsz, self.num_src, n, dtype=torch.float32, device=dev)
        ws, _ = self._stream_workspace(dev, Bsz, chunks_per_call)
        emb = embed_dev.to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            _cabi.check(_cabi.lib().l2h_sep_stream_dev(
                self._engine(), x.data_ptr(), n, emb.data_ptr(), state.buf.data_ptr(), y.data_ptr(), n, Bsz,
                n_calls, chunks_per_call, ws.data_ptr(), ws.numel(), torch.cuda.current_stream(dev).cuda_stream))
        self._last_stream_state = state
        return y

    def stream_host(self, x_host, embed_dev, chunks_per_call=1, state=None, out=None):
        """End-to-end streaming with HOST buffers (l2h_sep_stream_host): x_host [B,M,N] CPU tensor
        (pinned here if it is not); every round copies its samples host->device, runs the one-hop /
        multi-hop chains and copies the new samples back (a round = one call of chunks_per_call hops, or
        with chunks_per_call == 1 a pipelined group of up to pipeline_frames() hops).  Returns
        y [B,S,N] on the host (`out`: a pinned [B,S,>=N] tensor to write into).  Synchronises."""
        dev = embed_dev.device
        self._require_cuda(embed_dev)
        self._sync_weights(dev)
        hop, la = self.stft_chunk_size, self.stft_pad_size
        Bsz, _, n = x_host.shape
        step = hop * chunks_per_call
        n_calls = (n + step - 1) // step
        xh = x_host.contiguous().float()
        if not xh.is_pinned():
            xh = xh.pin_memory()
        grp = max(chunks_per_call, self.pipeline_frames() if chunks_per_call == 1 else 1)
        key = (Bsz, n_calls * step, grp, str(dev))
        cache = getattr(self, "_host_stage", None)
        if cache is None or cache[0] != key:        # staging buffers are reused across calls
            yh_c = torch.empty(Bsz, self.num_src, n_calls * step, dtype=torch.float32).pin_memory()
            xs = torch.empty(Bsz, self.num_ch, hop * grp + la, dtype=torch.float32, device=dev)
            ys = torch.empty(Bsz, self.num_src, hop * grp, dtype=torch.float32, device=dev)
            cache = (key, yh_c, xs, ys)
            self._host_stage = cache
        _, yh_c, xs, ys = cache
        yh = out if out is not None else yh_c
        if not yh.is_pinned() or yh.shape[-1] < n or not yh.is_contiguous():
            raise ValueError("out must be a contiguous pinned [B, S, >= N] float32 tensor")
        if state is None:
            state = self.init_buffers(Bsz, dev)
        ws, _ = self._stream_workspace(dev, Bsz, chunks_per_call)
        emb = embed_dev.to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            _cabi.check(_cabi.lib().l2h_sep_stream_host(
                self._engine(), xh.data_ptr(), n, emb.data_ptr(), state.buf.data_ptr(), yh.data_ptr(),
                yh.shape[-1], Bsz, n_calls, chunks_per_call, xs.data_ptr(), ys.data_ptr(), ws.data_ptr(),
                ws.numel(), torch.cuda.current_stream(dev).cuda_stream))
        self._last_stream_state = state
        return yh[..., :n] if out is not None else yh[..., :n].clone()

    def predict_host(self, x_host, embed_dev, state, out=None):
        """One streaming call with HOST buffers, natively (l2h_sep_stream_host with one call): x_host [B,M,128*T+64] PINNED (the
        chunk plus the 64 look-ahead samples, as predict(..., pad=False) takes it) is copied host->device, the chain runs, the
        128*T new samples per ear are copied back into `out` ([B,S,128*T] pinned; allocated once if None) and the stream is
        synchronised -- the copies, the launch and the wait are one C call instead of four Python-level ops.  Returns (out, state)."""
        dev = embed_dev.device
        self._require_cuda(embed_dev)
        self._sync_weights(dev)
        Bsz, _, n = x_host.shape
        frames, out_len = self._frames(n, who="predict_host")
        if not (x_host.is_pinned() and x_host.is_contiguous() and x_host.dtype == torch.float32):
            raise ValueError("x_host must be a contiguous pinned float32 tensor")
        if not isinstance(state, SepState):
            raise TypeError("state must come from Net.init_buffers()")
        key = (Bsz, frames, str(dev))
        cache = getattr(self, "_predict_stage", None)
        if cache is None or cache[0] != key:
            cache = (key, torch.empty(Bsz, self.num_src, out_len, dtype=torch.float32).pin_memory(),
                     torch.empty(Bsz, self.num_ch, n, dtype=torch.float32, device=dev),
                     torch.empty(Bsz, self.num_src, out_len, dtype=torch.float32, device=dev),
                     self._stream_workspace(dev, Bsz, frames)[0])
            self._predict_stage = cache
        _, yh_c, xs, ys, ws = cache
        emb = embed_dev if (embed_dev.dtype == torch.float32 and embed_dev.is_contiguous()) else embed_dev.to(torch.float32).contiguous()
        yh = out if out is not None else yh_c
        if not yh.is_pinned() or not yh.is_contiguous() or tuple(yh.shape) != (Bsz, self.num_src, out_len):
            raise ValueError("out must be a contiguous pinned [B, S, 128*T] float32 tensor")
        with torch.cuda.device(dev):
            _cabi.check(_cabi.lib().l2h_sep_stream_host(
                self._engine(), x_host.data_ptr(), n, emb.data_ptr(), state.buf.data_ptr(), yh.data_ptr(), out_len, Bsz, 1,
                frames, xs.data_ptr(), ys.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream(dev).cuda_stream))
        return yh, state

    # ---- debugging aid for the parity tests ------------------------------------------------------
    def forward_with_taps(self, x, embeds):
        """Whole-utterance forward that also returns the activations after every stage
        ([B,T,97,64] each): encoder, then per block (after intra, after inter, block output)."""
        embeds = embeds[:, 0]
        frames = self._frames(x.shape[-1], pad=True)[0]
        st = self.init_buffers(x.shape[0], x.device)
        y = self._run(x, embeds, st, frames, x.shape[-1], flags=1)
        off, ns = ctypes.c_int64(), ctypes.c_int32()
        _cabi.check(_cabi.lib().l2h_sep_tap_info(self._engine(), x.shape[0], frames, ctypes.byref(off),
                                                ctypes.byref(ns)))
        n = x.shape[0] * frames * 97 * 64
        wsf = self._ws.view(torch.float32)
        taps = [wsf[off.value + i * n: off.value + (i + 1) * n].view(x.shape[0], frames, 97, 64).clone()
                for i in range(ns.value)]
        return y, taps, st
