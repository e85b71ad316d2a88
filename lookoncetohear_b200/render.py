"""GPU binaural renderer: mono events + per-ear impulse responses -> binaural events, mixture and target, as the
reference's simulators and dataset do on the CPU (src/datasets/multi_ch_simulator.py:40-61 `SOFASimulator._convolve`;
src/datasets/MixLibriSpeechNoisyEnrollNorm.py:179-202 noise scaling / peak normalisation / mixture), and the band-limited
resampler of the responses and the dataset's audio (`torchaudio.functional.resample` at its defaults,
multi_ch_simulator.py:49, MixLibriSpeechNoisyEnrollNorm.py:69-75).  The arithmetic is `l2h_render_binaural` and
`l2h_resample` (hand-written CUDA); and its streaming form for listeners whose devices run at another rate than the
separator's 16 kHz (`StreamResampler`, `l2h_resample_stream`), with pushes of any length (`PacketResampler`,
`l2h_resample_packets`) and the per-slot FIFO that turns them into separator chunks and hop counts (`HopFifo`,
`l2h_hop_fifo`); and the per-slot capture that keeps each listener's recent input for enrollment (`EnrollCapture`,
`l2h_enroll_capture`).  No CPU fallback."""
import ctypes
import math
import numbers

import torch

from . import _cabi
from .net import device_list


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


def _whole(v, what, low=1):
    """v as an int >= low, or ValueError"""
    if isinstance(v, bool) or not isinstance(v, numbers.Integral) or int(v) < low or int(v) >= 2 ** 31:
        raise ValueError(f"{what} must be an integer >= {low} (below 2**31), got {v!r}")
    return int(v)


class StreamResampler:
    """`resample` for streams pushed a block at a time, one state row per (slot, channel): devices at 48, 32, 24 or 8 kHz
    into and out of the 16 kHz separator, every tick one call over the same slot list and hop counts as
    `Net.advance_slots` (l2h_resample_stream).

    Each push of `block` input samples (a multiple of o, the input samples of one period of the reduced rates) yields
    `out_block` = block * new / orig output samples.  The stream's output is `resample` of everything it has been pushed,
    delayed by `delay` samples (zeros before its start), bit for bit; the delay is what the window's taps on the far side
    need (6 samples at 48 -> 16 kHz, 21 at 16 -> 48 kHz).  Each output row first repeats the last `keep` samples of the
    stream's previous output: with keep=64, a push of 384 samples at 48 kHz returns the 192 samples of a one-hop
    `predict(..., pad=False)` chunk.  Equal rates and the 44.1 kHz family (whose 8 ms is no whole number of samples) are
    refused.

    `state` [slots, channels, hist + keep] is a plain float32 tensor on `device`: all zeros is a fresh stream, so a listener
    is reset by zeroing its rows (`reset`) and moved by copying them."""

    def __init__(self, orig_freq, new_freq, slots, channels, block, keep=0, device=None):
        orig, new = _whole(orig_freq, "orig_freq"), _whole(new_freq, "new_freq")
        self.n_slots, self.channels = _whole(slots, "slots"), _whole(channels, "channels")
        self.block, self.keep = _whole(block, "block"), _whole(keep, "keep", 0)
        hist, delay, out_block = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32()
        self._check(_cabi.lib().l2h_resample_stream_layout(orig, new, self.block, self.keep, ctypes.byref(hist),
                                                           ctypes.byref(delay), ctypes.byref(out_block)))
        self.orig_freq, self.new_freq = orig, new
        self.hist, self.delay, self.out_block = hist.value, delay.value, out_block.value
        dev = torch.device("cuda") if device is None else torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError("lookoncetohear_b200.StreamResampler needs a CUDA device (no CPU fallback)")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.state = torch.zeros(self.n_slots, self.channels, self.hist + self.keep, dtype=torch.float32, device=dev)

    @staticmethod
    def _check(rc):
        if rc == 2:                     # a window too large for the kernel: still the caller's sizes
            raise ValueError(_cabi.lib().l2h_last_error().decode())
        _cabi.check_args(rc)

    def __call__(self, x, slots, hops=None, out=None):
        """x [n, channels, block * T] CUDA tensor: row i pushes hops[i] blocks (T without `hops`) into slot slots[i].
        Returns y [n, channels, keep + T * out_block] float32 (`out`, if given): row i receives y[i, :, :keep + h_i *
        out_block], the last keep + h_i * out_block samples of its stream's delayed output; its later samples are left
        unwritten.  A row with h_i = 0, or whose CUDA slot entry lies outside [0, slots), stores nothing: neither its y row
        nor its state rows change.

        `slots` and `hops` follow Net.advance_slots: n distinct ints in [0, slots) and n ints in [0, T] (sequences or CPU
        tensors, checked and uploaded), or contiguous CUDA int32 tensors of shape (n,) used in place and read when the
        kernel runs, so a call captured in a CUDA graph serves any list rewritten in place."""
        dev = self.state.device
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise RuntimeError("StreamResampler needs CUDA tensors (no CPU fallback)")
        if x.device != dev:
            raise ValueError(f"x must live on the state's device {dev}, not {x.device}")
        if (not x.is_floating_point() or x.dim() != 3 or x.shape[0] < 1 or x.shape[1] != self.channels
                or x.shape[2] < self.block or x.shape[2] % self.block):
            raise ValueError(f"x must be a floating-point tensor [n, {self.channels}, {self.block} * T] with n, T >= 1, got "
                             f"{x.dtype} {tuple(x.shape)}")
        n, C, L = x.shape
        T = L // self.block
        y_len = self.keep + T * self.out_block
        if x.dtype != torch.float32 or x.stride(2) != 1 or x.stride(1) < L or x.stride(0) < C * x.stride(1):
            x = x.to(torch.float32).contiguous()
        slots = device_list(slots, dev, n, self.n_slots, True, "slot")
        if hops is not None:
            hops = device_list(hops, dev, n, T + 1, False, "hop")
        if out is None:
            out = torch.empty(n, C, y_len, dtype=torch.float32, device=dev)
        elif (not isinstance(out, torch.Tensor) or out.dtype != torch.float32 or out.device != dev
              or tuple(out.shape) != (n, C, y_len) or out.stride(2) != 1 or out.stride(1) < y_len
              or out.stride(0) < C * out.stride(1)):
            raise ValueError(f"out must be a float32 tensor [{n}, {C}, {y_len}] on {dev} with unit sample stride and rows "
                             "and channels that do not overlap")
        with torch.cuda.device(dev):
            self._check(_cabi.lib().l2h_resample_stream(
                x.data_ptr(), x.stride(0), x.stride(1), out.data_ptr(), out.stride(0), out.stride(1), n, C, T,
                slots.data_ptr(), None if hops is None else hops.data_ptr(), self.state.data_ptr(), self.n_slots,
                self.orig_freq, self.new_freq, self.block, self.keep, torch.cuda.current_stream(dev).cuda_stream))
        return out

    def reset(self, slots):
        """Make the listed slots fresh streams (their state rows zero); the other slots keep their history."""
        idx = torch.as_tensor(slots).cpu().reshape(-1)
        idx = device_list(idx, self.state.device, idx.numel(), self.n_slots, False, "slot")
        self.state.index_fill_(0, idx.long(), 0.0)


def _cuda_device(device, who):
    """the CUDA device a state lives on (the current one for None or "cuda"), or RuntimeError"""
    dev = torch.device("cuda") if device is None else torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError(f"lookoncetohear_b200.{who} needs a CUDA device (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device()) if dev.index is None else dev


def _rows_in(x, dev, channels, who):
    """x [n, channels, L] (n, L >= 1) as float32 on dev with unit sample stride and rows and channels that do not overlap"""
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise RuntimeError(f"{who} needs CUDA tensors (no CPU fallback)")
    if x.device != dev:
        raise ValueError(f"x must live on the state's device {dev}, not {x.device}")
    if not x.is_floating_point() or x.dim() != 3 or x.shape[0] < 1 or x.shape[1] != channels or x.shape[2] < 1:
        raise ValueError(f"x must be a floating-point tensor [n, {channels}, samples] with n, samples >= 1, got "
                         f"{x.dtype} {tuple(x.shape)}")
    if x.dtype != torch.float32 or x.stride(2) != 1 or x.stride(1) < x.shape[2] or x.stride(0) < channels * x.stride(1):
        x = x.to(torch.float32).contiguous()
    return x


def _rows_out(out, shape, dev):
    """`out` checked as a float32 tensor of `shape` on dev with unit sample stride and rows and channels that do not
    overlap, or a new one"""
    if out is None:
        return torch.empty(shape, dtype=torch.float32, device=dev)
    if (not isinstance(out, torch.Tensor) or out.dtype != torch.float32 or out.device != dev or tuple(out.shape) != shape
            or out.stride(2) != 1 or out.stride(1) < shape[2] or out.stride(0) < shape[1] * out.stride(1)):
        raise ValueError(f"out must be a float32 tensor {list(shape)} on {dev} with unit sample stride and rows and channels "
                         "that do not overlap")
    return out


def _ints_out(t, n, dev, what):
    """`t` checked as a contiguous CUDA int32 tensor of shape (n,) on dev, written in place, or a new one"""
    if t is None:
        return torch.empty(n, dtype=torch.int32, device=dev)
    if (not isinstance(t, torch.Tensor) or t.dtype != torch.int32 or t.device != dev or tuple(t.shape) != (n,)
            or not t.is_contiguous()):
        raise ValueError(f"{what} must be a contiguous int32 tensor of shape ({n},) on {dev}")
    return t


def _reset(state, slots):
    """zero the state rows of the listed slots"""
    idx = torch.as_tensor(slots).cpu().reshape(-1)
    idx = device_list(idx, state.device, idx.numel(), state.shape[0], False, "slot")
    state.index_fill_(0, idx.long(), 0.0)


class PacketResampler:
    """`resample` for streams pushed any number of samples at a time, one state row per (slot, channel): devices at 44.1,
    22.05 or 11.025 kHz, and clients that send 10 ms packets at any rate, into and out of the 16 kHz separator
    (l2h_resample_packets).

    A stream that has been pushed N samples in all has returned exactly floor(N * new / orig) samples: the first ones of
    `resample` of everything it was pushed, delayed by `delay` samples (zeros before its start), bit for bit -- the
    output and delay of `StreamResampler` with keep=0 (6 samples at 44.1 -> 16 kHz, 19 at 16 -> 44.1 kHz).  A push of up
    to `max_in` samples returns up to `max_out` samples.  Equal rates are refused.

    `state` [slots, channels, row_floats] is a plain float32 tensor on `device`: all zeros is a fresh stream, so a listener
    is reset by zeroing its rows (`reset`) and moved by copying them."""

    def __init__(self, orig_freq, new_freq, slots, channels, max_in, device=None):
        orig, new = _whole(orig_freq, "orig_freq"), _whole(new_freq, "new_freq")
        self.n_slots, self.channels = _whole(slots, "slots"), _whole(channels, "channels")
        self.max_in = _whole(max_in, "max_in")
        row, delay, max_out = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32()
        StreamResampler._check(_cabi.lib().l2h_resample_packets_layout(orig, new, self.max_in, ctypes.byref(row),
                                                                       ctypes.byref(delay), ctypes.byref(max_out)))
        self.orig_freq, self.new_freq = orig, new
        self.delay, self.max_out = delay.value, max_out.value
        dev = _cuda_device(device, "PacketResampler")
        self.state = torch.zeros(self.n_slots, self.channels, row.value, dtype=torch.float32, device=dev)

    def __call__(self, x, counts, slots, unit=1, out=None, out_counts=None):
        """x [n, channels, max_in] CUDA tensor: row i pushes its first counts[i] * unit samples into slot slots[i].
        Returns (y [n, channels, max_out] float32, out_counts [n] int32 CUDA) (`out` and `out_counts`, if given, written
        in place): row i receives y[i, :, :out_counts[i]], the samples of its stream's delayed output its push makes
        final; its later samples are left unwritten.  A row that pushes nothing, or whose CUDA slot entry lies outside
        [0, slots), stores nothing and gets out count 0.

        `slots` follows Net.advance_slots: n distinct ints in [0, slots), or a contiguous CUDA int32 tensor of shape (n,)
        used in place and read when the kernel runs.  `counts` likewise: n ints in [0, max_in // unit], or a CUDA int32
        tensor (HopFifo's hops, with unit=128, on the way out of the separator), where an entry whose count * unit lies
        outside [0, max_in] counts as 0.  So a call captured in a CUDA graph serves any lists rewritten in place."""
        dev = self.state.device
        x = _rows_in(x, dev, self.channels, "PacketResampler")
        n, C, L = x.shape
        if L != self.max_in:
            raise ValueError(f"x rows must hold max_in = {self.max_in} samples, got {L}")
        unit = _whole(unit, "unit")
        slots = device_list(slots, dev, n, self.n_slots, True, "slot")
        counts = device_list(counts, dev, n, self.max_in // unit + 1, False, "count")
        out = _rows_out(out, (n, C, self.max_out), dev)
        out_counts = _ints_out(out_counts, n, dev, "out_counts")
        with torch.cuda.device(dev):
            StreamResampler._check(_cabi.lib().l2h_resample_packets(
                x.data_ptr(), x.stride(0), x.stride(1), out.data_ptr(), out.stride(0), out.stride(1), n, C, L,
                counts.data_ptr(), unit, out_counts.data_ptr(), slots.data_ptr(), self.state.data_ptr(), self.n_slots,
                self.orig_freq, self.new_freq, torch.cuda.current_stream(dev).cuda_stream))
        return out, out_counts

    def reset(self, slots):
        """Make the listed slots fresh streams (their state rows zero); the other slots keep their history."""
        _reset(self.state, slots)


class HopFifo:
    """A per-slot FIFO that turns 16 kHz pieces of any length into the separator's chunks and per-row hop counts on the
    device (l2h_hop_fifo), so a tick of packets needs no count read back to the host.

    A slot's signal is 64 zeros, then every sample appended since it was reset.  Each call appends a row's samples to its
    slot, then pops h = min(frames, floor(held / 128)) hops of the samples held past the 64-sample carry: the chunk is the
    next 128 h + 64 samples of the signal, the `Net.advance_slots` input of h hops, and the last 64 stay as the next
    chunk's start.  With 48 kHz pushes of 384 samples through `PacketResampler` this gives exactly the chunks of
    `StreamResampler(48000, 16000, ..., keep=64)`.  Samples past `capacity` are dropped and counted in `dropped`.

    `state` [slots, channels, 3 + 64 + capacity] is a float32 tensor on `device` (three int32 words in its first floats):
    all zeros is an empty FIFO, so a listener is reset by zeroing its rows (`reset`) and moved by copying them."""

    HOP, CARRY = 128, 64

    def __init__(self, slots, channels, frames, capacity, device=None):
        self.n_slots, self.channels = _whole(slots, "slots"), _whole(channels, "channels")
        self.frames, self.capacity = _whole(frames, "frames"), _whole(capacity, "capacity")
        row = ctypes.c_int32()
        _cabi.check_args(_cabi.lib().l2h_hop_fifo_layout(self.capacity, ctypes.byref(row)))
        dev = _cuda_device(device, "HopFifo")
        self.state = torch.zeros(self.n_slots, self.channels, row.value, dtype=torch.float32, device=dev)

    def __call__(self, x, counts, slots, unit=1, out=None, hops=None):
        """x [n, channels, L] CUDA tensor: row i appends its first counts[i] * unit samples to slot slots[i], then pops
        its hops.  Returns (chunk [n, channels, 128 * frames + 64] float32, hops [n] int32 CUDA) (`out` and `hops`, if
        given, written in place): row i receives chunk[i, :, :128 * hops[i] + 64]; its later samples are left unwritten.
        A row whose CUDA slot entry lies outside [0, slots) stores nothing and gets 0 hops, so (slots, hops) go straight
        to `Net.advance_slots(chunk, embed, state, slots, hops=hops)`.  A row with count 0 still pops the hops its slot
        holds.

        `slots` and `counts` follow PacketResampler: host lists are checked (counts in [0, L // unit]) and uploaded, CUDA
        int32 tensors are used in place, where a count whose count * unit lies outside [0, L] counts as 0."""
        dev = self.state.device
        x = _rows_in(x, dev, self.channels, "HopFifo")
        n, C, L = x.shape
        unit = _whole(unit, "unit")
        slots = device_list(slots, dev, n, self.n_slots, True, "slot")
        counts = device_list(counts, dev, n, L // unit + 1, False, "count")
        out = _rows_out(out, (n, C, self.HOP * self.frames + self.CARRY), dev)
        hops = _ints_out(hops, n, dev, "hops")
        with torch.cuda.device(dev):
            _cabi.check_args(_cabi.lib().l2h_hop_fifo(
                x.data_ptr(), x.stride(0), x.stride(1), L, counts.data_ptr(), unit, out.data_ptr(), out.stride(0),
                out.stride(1), hops.data_ptr(), n, C, self.frames, slots.data_ptr(), self.state.data_ptr(), self.n_slots,
                self.capacity, torch.cuda.current_stream(dev).cuda_stream))
        return out, hops

    @property
    def dropped(self):
        """[slots] int64: the samples each slot has dropped since its reset (capacity overflows)"""
        return self.state[:, 0, 2].view(torch.int32).long()

    @property
    def held(self):
        """[slots] int64: the samples each slot holds past its 64-sample carry"""
        return self.state[:, 0, 1].view(torch.int32).long()

    def reset(self, slots):
        """Make the listed slots empty FIFOs with a zero carry; the other slots keep what they hold."""
        _reset(self.state, slots)


class EnrollCapture:
    """Per-slot capture of each listener's recent 16 kHz input on the device (l2h_enroll_capture), so a "look" can be
    enrolled from the stream itself (`EmbedTFGridNet.enroll`) with no copy of the audio kept on the host.

    Each call appends the hops' new samples of a row's chunk, samples 64 .. 64 + 128 h - 1 (no look-ahead repeat), to its
    slot; a slot keeps its last `capacity` samples and counts what it captured since reset, capped at `capacity`
    (`captured`).  It takes the chunk, slots and hops that `HopFifo` hands `Net.advance_slots`, so it runs in the same
    tick and the same CUDA graph.

    `state` [slots, channels, 2 + capacity] is a float32 tensor on `device` (two int32 words in its first floats): all
    zeros is an empty capture, so a listener is reset by zeroing its rows (`reset`) and moved by copying them.  `capacity`
    must hold the 192 samples of the shortest enrollment."""

    HOP, CARRY = 128, 64

    def __init__(self, slots, channels, capacity, device=None):
        self.n_slots, self.channels = _whole(slots, "slots"), _whole(channels, "channels")
        self.capacity = _whole(capacity, "capacity")
        row = ctypes.c_int32()
        _cabi.check_args(_cabi.lib().l2h_enroll_capture_layout(self.capacity, ctypes.byref(row)))
        dev = _cuda_device(device, "EnrollCapture")
        self.state = torch.zeros(self.n_slots, self.channels, row.value, dtype=torch.float32, device=dev)

    def __call__(self, chunk, slots, hops):
        """chunk [n, channels, 128 * T + 64] CUDA tensor: row i appends samples 64 .. 64 + 128 * hops[i] - 1 to slot
        slots[i].  A row whose CUDA slot entry lies outside [0, slots), or whose CUDA hop entry lies outside [1, T],
        stores nothing.

        `slots` and `hops` follow Net.advance_slots: n distinct ints in [0, slots) and n ints in [0, T] (sequences or CPU
        tensors, checked and uploaded), or contiguous CUDA int32 tensors of shape (n,) used in place and read when the
        kernel runs (HopFifo's hops), so a call captured in a CUDA graph serves any lists rewritten in place."""
        dev = self.state.device
        chunk = _rows_in(chunk, dev, self.channels, "EnrollCapture")
        n, C, L = chunk.shape
        if L < self.HOP + self.CARRY or (L - self.CARRY) % self.HOP:
            raise ValueError(f"chunk rows must hold 128 * T + 64 samples with T >= 1, got {L}")
        T = (L - self.CARRY) // self.HOP
        slots = device_list(slots, dev, n, self.n_slots, True, "slot")
        hops = device_list(hops, dev, n, T + 1, False, "hop")
        with torch.cuda.device(dev):
            _cabi.check_args(_cabi.lib().l2h_enroll_capture(
                chunk.data_ptr(), chunk.stride(0), chunk.stride(1), n, C, T, slots.data_ptr(), hops.data_ptr(),
                self.state.data_ptr(), self.n_slots, self.capacity, torch.cuda.current_stream(dev).cuda_stream))

    @property
    def captured(self):
        """[slots] int32 CUDA view of the state: the samples each slot captured since its reset, capped at capacity"""
        return self.state[:, 0, 1].view(torch.int32)

    def reset(self, slots):
        """Make the listed slots empty captures; the other slots keep what they hold."""
        _reset(self.state, slots)


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
