"""The per-slot stages of the serving front end, each one hand-written CUDA call per tick over the same slot list as
`Net.advance_slots`: streaming resampling for listeners whose devices run at another rate than the separator's 16 kHz
(`StreamResampler`, `l2h_resample_stream`), with pushes of any length (`PacketResampler`, `l2h_resample_packets`), the
per-slot FIFO that turns 16 kHz pieces into separator chunks and hop counts (`HopFifo`, `l2h_hop_fifo`), and the
per-slot capture that keeps each listener's recent input for enrollment (`EnrollCapture`, `l2h_enroll_capture`),
the per-listener mixer that sums the separated voices and the ambient mixture into one row with fades (`TargetMixer`,
`l2h_target_mix`), the per-listener look-ahead limiter that keeps the output under a ceiling with one gain for both
ears (`Limiter`, `l2h_limiter`), the per-row leveler that brings each voice to one loudness with one gain for both
ears (`Leveler`, `l2h_leveler`), the per-listener multiband compressor that fits the output to each ear's hearing
(`BandCompressor`, `l2h_band_compressor`), and the per-slot jitter buffer that puts a device's packets back in sequence
order and conceals lost ones (`JitterBuffer`, `l2h_jitter_buffer`).

Each stage keeps a float32 state [slots, channels, row floats] on a CUDA device.  All zeros is a fresh slot, so a
listener is reset by zeroing its rows (`reset`) and moved by copying them.  No CPU fallback."""
import ctypes
import math
import numbers

import torch

from . import _cabi
from .net import device_list, device_offsets


def _whole(v, what, low=1):
    """v as an int >= low, or ValueError"""
    if isinstance(v, bool) or not isinstance(v, numbers.Integral) or int(v) < low or int(v) >= 2 ** 31:
        raise ValueError(f"{what} must be an integer >= {low} (below 2**31), got {v!r}")
    return int(v)


def _real(v, what, ok=math.isfinite, must="a finite number"):
    """v as a float when it is a real number, not a bool, that passes `ok` (by default: finite; a range test also
    refuses NaN), else ValueError "{what} must be {must}"."""
    if isinstance(v, bool) or not isinstance(v, numbers.Real) or not ok(v):
        raise ValueError(f"{what} must be {must}, got {v!r}")
    return float(v)


def _check(rc):
    """_cabi.check_args, with error 2 (a window too large for the kernel: still the caller's sizes) a ValueError too"""
    if rc == 2:
        raise ValueError(_cabi.lib().l2h_last_error().decode())
    _cabi.check_args(rc)


def _layout(query, *args, outs=1):
    """the `outs` int32 values a layout query writes after its arguments"""
    vals = [ctypes.c_int32() for _ in range(outs)]
    _check(query(*args, *[ctypes.byref(v) for v in vals]))
    return [v.value for v in vals]


class _SlotStage:
    """What the stages share: the slots and channels of the state, its allocation on a CUDA device, `reset`, and the
    checks of the row tensors a call reads and writes."""

    HOP, CARRY = 128, 64      # a separator chunk of h hops: 64 samples carried from the last chunk, then 128 h new ones
    HOP_S = 128 / 16000       # seconds per hop of the 16 kHz grid

    def __init__(self, slots, channels):
        self.n_slots, self.channels = _whole(slots, "slots"), _whole(channels, "channels")

    def _allocate(self, row_floats, device, rows=None):
        """a zero state of `rows` (else n_slots) rows of row_floats on `device` (the current CUDA device for None or
        "cuda")"""
        dev = torch.device("cuda") if device is None else torch.device(device)
        if dev.type != "cuda":
            raise RuntimeError(f"lookoncetohear_b200.{type(self).__name__} needs a CUDA device (no CPU fallback)")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.state = torch.zeros(rows or self.n_slots, self.channels, row_floats, dtype=torch.float32, device=dev)

    def reset(self, slots):
        """Make the listed slots fresh (their state rows zero); the other slots keep what they hold."""
        self.state.index_fill_(0, self._indices(slots, self.n_slots, "slot"), 0.0)

    def _indices(self, values, end, noun, distinct=False, need=None):
        """host indices into [0, end) (each listed once if `distinct`), checked and uploaded as an int64 tensor on the
        state's device; `need` names a call that needs at least one"""
        idx = torch.as_tensor(values).cpu().reshape(-1)
        if need and idx.numel() < 1:
            raise ValueError(f"{need} needs at least one {noun}")
        return device_list(idx, self.state.device, idx.numel(), end, distinct, noun).long()

    def _hops(self, hops, n, T):
        """an optional hop list of n rows in [0, T], as device_list uploads it"""
        return None if hops is None else device_list(hops, self.state.device, n, T + 1, False, "hop")

    def _run(self, entry, *args):
        """the C entry `entry` called on the state's device and its current stream, each tensor argument passed as its
        data pointer"""
        dev = self.state.device
        with torch.cuda.device(dev):
            args = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
            _check(getattr(_cabi.lib(), entry)(*args, torch.cuda.current_stream(dev).cuda_stream))

    def _rows_in(self, x, block=None):
        """x [n, channels, L] (n, L >= 1; L a multiple of `block` if given) as float32 on the state's device with unit
        sample stride and rows and channels that do not overlap"""
        dev, C = self.state.device, self.channels
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise RuntimeError(f"{type(self).__name__} needs CUDA tensors (no CPU fallback)")
        if x.device != dev:
            raise ValueError(f"x must live on the state's device {dev}, not {x.device}")
        unit = block or 1
        if (not x.is_floating_point() or x.dim() != 3 or x.shape[0] < 1 or x.shape[1] != C or x.shape[2] < unit
                or x.shape[2] % unit):
            shape, count = ("samples", "samples") if block is None else (f"{block} * T", "T")
            raise ValueError(f"x must be a floating-point tensor [n, {C}, {shape}] with n, {count} >= 1, got "
                             f"{x.dtype} {tuple(x.shape)}")
        if x.dtype != torch.float32 or x.stride(2) != 1 or x.stride(1) < x.shape[2] or x.stride(0) < C * x.stride(1):
            x = x.to(torch.float32).contiguous()
        return x

    def _rows_out(self, out, shape):
        """`out` checked as a float32 tensor of `shape` on the state's device with unit sample stride and rows and
        channels that do not overlap, or a new one"""
        dev = self.state.device
        if out is None:
            return torch.empty(shape, dtype=torch.float32, device=dev)
        if (not isinstance(out, torch.Tensor) or out.dtype != torch.float32 or out.device != dev
                or tuple(out.shape) != shape or out.stride(2) != 1 or out.stride(1) < shape[2]
                or out.stride(0) < shape[1] * out.stride(1)):
            raise ValueError(f"out must be a float32 tensor {list(shape)} on {dev} with unit sample stride and rows and "
                             "channels that do not overlap")
        return out

    def _ints_out(self, t, n, what):
        """`t` checked as a contiguous CUDA int32 tensor of shape (n,) on the state's device, written in place, or a new
        one"""
        dev = self.state.device
        if t is None:
            return torch.empty(n, dtype=torch.int32, device=dev)
        if (not isinstance(t, torch.Tensor) or t.dtype != torch.int32 or t.device != dev or tuple(t.shape) != (n,)
                or not t.is_contiguous()):
            raise ValueError(f"{what} must be a contiguous int32 tensor of shape ({n},) on {dev}")
        return t


class StreamResampler(_SlotStage):
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
        super().__init__(slots, channels)
        self.block, self.keep = _whole(block, "block"), _whole(keep, "keep", 0)
        self.hist, self.delay, self.out_block = _layout(_cabi.lib().l2h_resample_stream_layout, orig, new, self.block,
                                                        self.keep, outs=3)
        self.orig_freq, self.new_freq = orig, new
        self._allocate(self.hist + self.keep, device)

    def __call__(self, x, slots, hops=None, out=None):
        """x [n, channels, block * T] CUDA tensor: row i pushes hops[i] blocks (T without `hops`) into slot slots[i].
        Returns y [n, channels, keep + T * out_block] float32 (`out`, if given): row i receives y[i, :, :keep + h_i *
        out_block], the last keep + h_i * out_block samples of its stream's delayed output; its later samples are left
        unwritten.  A row with h_i = 0, or whose CUDA slot entry lies outside [0, slots), stores nothing: neither its y row
        nor its state rows change.

        `slots` and `hops` follow Net.advance_slots: n distinct ints in [0, slots) and n ints in [0, T] (sequences or CPU
        tensors, checked and uploaded), or contiguous CUDA int32 tensors of shape (n,) used in place and read when the
        kernel runs, so a call captured in a CUDA graph serves any list rewritten in place."""
        x = self._rows_in(x, self.block)
        dev = self.state.device
        n, C, L = x.shape
        T = L // self.block
        slots = device_list(slots, dev, n, self.n_slots, True, "slot")
        hops = self._hops(hops, n, T)
        out = self._rows_out(out, (n, C, self.keep + T * self.out_block))
        self._run("l2h_resample_stream", x, x.stride(0), x.stride(1), out, out.stride(0), out.stride(1), n, C, T, slots,
                  hops, self.state, self.n_slots, self.orig_freq, self.new_freq, self.block, self.keep)
        return out


class PacketResampler(_SlotStage):
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
        super().__init__(slots, channels)
        self.max_in = _whole(max_in, "max_in")
        row, self.delay, self.max_out = _layout(_cabi.lib().l2h_resample_packets_layout, orig, new, self.max_in, outs=3)
        self.orig_freq, self.new_freq = orig, new
        self._allocate(row, device)

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
        x = self._rows_in(x)
        dev = self.state.device
        n, C, L = x.shape
        if L != self.max_in:
            raise ValueError(f"x rows must hold max_in = {self.max_in} samples, got {L}")
        unit = _whole(unit, "unit")
        slots = device_list(slots, dev, n, self.n_slots, True, "slot")
        counts = device_list(counts, dev, n, self.max_in // unit + 1, False, "count")
        out = self._rows_out(out, (n, C, self.max_out))
        out_counts = self._ints_out(out_counts, n, "out_counts")
        self._run("l2h_resample_packets", x, x.stride(0), x.stride(1), out, out.stride(0), out.stride(1), n, C, L, counts,
                  unit, out_counts, slots, self.state, self.n_slots, self.orig_freq, self.new_freq)
        return out, out_counts


class HopFifo(_SlotStage):
    """A per-slot FIFO that turns 16 kHz pieces of any length into the separator's chunks and per-row hop counts on the
    device (l2h_hop_fifo), so a tick of packets needs no count read back to the host.

    A slot's signal is 64 zeros, then every sample appended since it was reset.  Each call appends a row's samples to its
    slot, then pops h = min(frames, floor(held / 128)) hops of the samples held past the 64-sample carry: the chunk is the
    next 128 h + 64 samples of the signal, the `Net.advance_slots` input of h hops, and the last 64 stay as the next
    chunk's start.  With 48 kHz pushes of 384 samples through `PacketResampler` this gives exactly the chunks of
    `StreamResampler(48000, 16000, ..., keep=64)`.  Samples past `capacity` are dropped and counted in `dropped`.

    `state` [slots, channels, 3 + 64 + capacity] is a float32 tensor on `device` (three int32 words in its first floats):
    all zeros is an empty FIFO, so a listener is reset by zeroing its rows (`reset`) and moved by copying them."""

    def __init__(self, slots, channels, frames, capacity, device=None):
        super().__init__(slots, channels)
        self.frames, self.capacity = _whole(frames, "frames"), _whole(capacity, "capacity")
        self._allocate(*_layout(_cabi.lib().l2h_hop_fifo_layout, self.capacity), device)

    def __call__(self, x, counts, slots, unit=1, out=None, hops=None):
        """x [n, channels, L] CUDA tensor: row i appends its first counts[i] * unit samples to slot slots[i], then pops
        its hops.  Returns (chunk [n, channels, 128 * frames + 64] float32, hops [n] int32 CUDA) (`out` and `hops`, if
        given, written in place): row i receives chunk[i, :, :128 * hops[i] + 64]; its later samples are left unwritten.
        A row whose CUDA slot entry lies outside [0, slots) stores nothing and gets 0 hops, so (slots, hops) go straight
        to `Net.advance_slots(chunk, embed, state, slots, hops=hops)`.  A row with count 0 still pops the hops its slot
        holds.

        `slots` and `counts` follow PacketResampler: host lists are checked (counts in [0, L // unit]) and uploaded, CUDA
        int32 tensors are used in place, where a count whose count * unit lies outside [0, L] counts as 0."""
        x = self._rows_in(x)
        dev = self.state.device
        n, C, L = x.shape
        unit = _whole(unit, "unit")
        slots = device_list(slots, dev, n, self.n_slots, True, "slot")
        counts = device_list(counts, dev, n, L // unit + 1, False, "count")
        out = self._rows_out(out, (n, C, self.HOP * self.frames + self.CARRY))
        hops = self._ints_out(hops, n, "hops")
        self._run("l2h_hop_fifo", x, x.stride(0), x.stride(1), L, counts, unit, out, out.stride(0), out.stride(1), hops, n,
                  C, self.frames, slots, self.state, self.n_slots, self.capacity)
        return out, hops

    @property
    def dropped(self):
        """[slots] int64: the samples each slot has dropped since its reset (capacity overflows)"""
        return self.state[:, 0, 2].view(torch.int32).long()

    @property
    def held(self):
        """[slots] int64: the samples each slot holds past its 64-sample carry"""
        return self.state[:, 0, 1].view(torch.int32).long()


class EnrollCapture(_SlotStage):
    """Per-slot capture of each listener's recent 16 kHz input on the device (l2h_enroll_capture), so a "look" can be
    enrolled from the stream itself (`EmbedTFGridNet.enroll`) with no copy of the audio kept on the host.

    Each call appends the hops' new samples of a row's chunk, samples 64 .. 64 + 128 h - 1 (no look-ahead repeat), to its
    slot; a slot keeps its last `capacity` samples and counts what it captured since reset, capped at `capacity`
    (`captured`).  It takes the chunk, slots and hops that `HopFifo` hands `Net.advance_slots`, so it runs in the same
    tick and the same CUDA graph.

    `state` [slots, channels, 2 + capacity] is a float32 tensor on `device` (two int32 words in its first floats): all
    zeros is an empty capture, so a listener is reset by zeroing its rows (`reset`) and moved by copying them.  `capacity`
    must hold the 192 samples of the shortest enrollment."""

    def __init__(self, slots, channels, capacity, device=None):
        super().__init__(slots, channels)
        self.capacity = _whole(capacity, "capacity")
        self._allocate(*_layout(_cabi.lib().l2h_enroll_capture_layout, self.capacity), device)

    def __call__(self, chunk, slots, hops):
        """chunk [n, channels, 128 * T + 64] CUDA tensor: row i appends samples 64 .. 64 + 128 * hops[i] - 1 to slot
        slots[i].  A row whose CUDA slot entry lies outside [0, slots), or whose CUDA hop entry lies outside [1, T],
        stores nothing.

        `slots` and `hops` follow Net.advance_slots: n distinct ints in [0, slots) and n ints in [0, T] (sequences or CPU
        tensors, checked and uploaded), or contiguous CUDA int32 tensors of shape (n,) used in place and read when the
        kernel runs (HopFifo's hops), so a call captured in a CUDA graph serves any lists rewritten in place."""
        chunk = self._rows_in(chunk)
        dev = self.state.device
        n, C, L = chunk.shape
        if L < self.HOP + self.CARRY or (L - self.CARRY) % self.HOP:
            raise ValueError(f"chunk rows must hold 128 * T + 64 samples with T >= 1, got {L}")
        T = (L - self.CARRY) // self.HOP
        slots = device_list(slots, dev, n, self.n_slots, True, "slot")
        hops = device_list(hops, dev, n, T + 1, False, "hop")
        self._run("l2h_enroll_capture", chunk, chunk.stride(0), chunk.stride(1), n, C, T, slots, hops, self.state,
                  self.n_slots, self.capacity)

    @property
    def captured(self):
        """[slots] int32 CUDA view of the state: the samples each slot captured since its reset, capped at capacity"""
        return self.state[:, 0, 1].view(torch.int32)


class TargetMixer(_SlotStage):
    """Per-listener mixing of the separated voices on the device (l2h_target_mix): each listener's target rows of
    `Net.advance_target_rows`, each scaled by its record's gain, plus optionally its unprocessed mixture scaled by its
    slot's ambient gain ("transparency"), summed into one row per listener for the up-resampler and the client.

    Every gain is a ramp: set_gains / set_ambient fade it to a new value over `fade` samples along a raised cosine, so a
    joined voice fades in and a dropped one fades out instead of clicking.  The gain of a sample depends only on the
    ramp and the sample's position since the ramp started: how the ramp is cut into ticks and hop counts never changes a
    bit of the output, and a ramp advances only by the samples its listener mixes.

    `state` [records + slots, channels, 4] is a float32 tensor on `device`: one ramp per separator record, then one per
    listener slot.  All zeros is a fresh row, a record at gain 1 and a slot at ambient gain 0, so rows are reset by
    zeroing them (`reset`) and moved by copying them."""

    GAIN_MAX = 16.0

    def __init__(self, records, slots, channels, device=None):
        super().__init__(slots, channels)
        self.n_records = _whole(records, "records")
        if self.n_records + self.n_slots >= 2 ** 31:
            raise ValueError("records + slots must be below 2**31")
        self._allocate(*_layout(_cabi.lib().l2h_target_mix_layout), device, rows=self.n_records + self.n_slots)

    def reset(self, records=(), slots=()):
        """Make the listed records (gain 1) and slots (ambient gain 0) fresh; the other rows keep their ramps."""
        rows = [self._indices(values, end, noun) + base
                for values, end, noun, base in ((records, self.n_records, "record", 0),
                                                (slots, self.n_slots, "slot", self.n_records))
                if torch.as_tensor(values).numel()]
        if rows:
            self.state.index_fill_(0, torch.cat(rows), 0.0)

    def __call__(self, y, records, offsets, slots, hops=None, chunk=None, out=None):
        """y [R, channels, 128 * T] CUDA tensor, the target rows of Net.advance_target_rows; listener row i owns target
        rows offsets[i] .. offsets[i+1]-1, target row r has record records[r]'s gain, and slots[i] is the listener's
        slot.  Returns out [n, channels, 128 * T] float32 (`out`, if given, written in place): row i receives, for
        s < 128 h (h = hops[i], T without hops), the sum in row order of its live target rows times their gains, plus
        chunk[i, :, s] times its slot's ambient gain when `chunk` is given.  Its later samples are left unwritten.

        chunk [n, channels, 128 * T + 64] is the separator's input of the same call: its first 128 h samples are exactly
        the stretch of the mixture that y's rows estimate, with the same 64-sample look-ahead delay, so the ambient term
        needs no buffer of its own.  A term enters only the samples where its gain is nonzero, so one target at gain 1
        returns its y row bit for bit, NaN in a muted term's samples never reaches out, and a term whose gain is 0 over
        the call is not read.  A listener with no live term gets zeros (-0).

        Lists follow Net.advance_target_rows: host lists are checked and uploaded (`records` R distinct ints in
        [0, records); `offsets` n + 1 ints from 0, non-decreasing, at most R; `slots` n distinct ints in [0, slots);
        `hops` n ints in [0, T]); contiguous CUDA int32 tensors are used in place and read when the kernel runs, where a
        record outside the mixer marks a row that is skipped, the offsets are clamped as the separator clamps them, and
        a slot outside the mixer or a hop count outside [1, T] marks a listener that stores nothing and advances no
        ramp.  So a call captured in a CUDA graph with the FIFO, the separator and the up-resampler serves any lists
        rewritten in place.  The output of Net.advance_targets, y [n, K, S, 128 T], is y.view(n K, S, 128 T) with offsets
        i K and records g_i K + k."""
        y = self._rows_in(y, self.HOP)
        dev = self.state.device
        R, C, L = y.shape
        T = L // self.HOP
        n = len(slots) if not isinstance(slots, torch.Tensor) else slots.numel()
        if not 0 < n <= R:
            raise ValueError(f"a mix needs 0 < n <= R, got n = {n} listeners and R = {R} target rows")
        records = device_list(records, dev, R, self.n_records, True, "record")
        offsets = device_offsets(offsets, dev, n, R)
        slots = device_list(slots, dev, n, self.n_slots, True, "slot")
        hops = self._hops(hops, n, T)
        if chunk is not None:
            chunk = self._rows_in(chunk)
            if tuple(chunk.shape) != (n, C, L + self.CARRY):
                raise ValueError(f"chunk must have shape [{n}, {C}, {L + self.CARRY}] (the separator's input of the call, "
                                 f"with y's channels), got {tuple(chunk.shape)}")
        out = self._rows_out(out, (n, C, L))
        ck = (None, 0, 0) if chunk is None else (chunk, chunk.stride(0), chunk.stride(1))
        self._run("l2h_target_mix", y, y.stride(0), y.stride(1), *ck, out, out.stride(0), out.stride(1), n, R, C, T, records,
                  offsets, hops, slots, self.state, self.n_records, self.n_slots)
        return out

    def set_gains(self, records, gains, fade=0, start=None):
        """Fade the gains of the listed records to `gains` over `fade` samples (0: at once), starting at `start`, or,
        without it, at the gain of the last sample each record mixed, so changing a ramp halfway never jumps.  Join a
        voice with set_gains([b], [1.0], fade=480, start=0.0); drop one with set_gains([b], [0.0], fade=480), keep
        listing b until fading[b] is false, then leave its row out.

        `gains`, `fade` and `start` are numbers or one per record.  Host values are checked (gains and starts finite, in
        [0, 16]; fades ints >= 0) and uploaded; CUDA tensors (int32 records and fades, float32 gains and starts, shape
        (n,)) are used in place and read when the kernel runs, so a set can be captured in a CUDA graph.  Enqueue a set
        on the mixer's stream between its calls."""
        self._set(records, self.n_records, "record", 0, gains, fade, start)

    def set_ambient(self, slots, gains, fade=0, start=None):
        """set_gains for the ambient gains of the listed slots (the share of the unprocessed mixture each listener hears;
        0 when fresh)."""
        self._set(slots, self.n_slots, "slot", self.n_records, gains, fade, start)

    def _set(self, rows, end, noun, base, gains, fade, start):
        dev = self.state.device
        n = rows.numel() if isinstance(rows, torch.Tensor) else len(rows)
        if n < 1:
            raise ValueError(f"set needs at least one {noun}")
        rows = device_list(rows, dev, n, end, True, noun)
        # record b is state row b, slot s is state row records + s; a CUDA entry outside [0, end) stays outside the state
        rows = torch.where((rows >= 0) & (rows < end), rows + base, -1).to(torch.int32)
        gains = self._values(gains, n, torch.float32, "gains")
        fades = self._values(fade, n, torch.int32, "fade")
        starts = None if start is None else self._values(start, n, torch.float32, "start")
        self._run("l2h_target_mix_set", self.state, self.n_records, self.n_slots, self.channels, rows, n, gains, starts,
                  fades)

    def _values(self, v, n, dtype, what):
        """v as an [n] `dtype` tensor on the state's device: a CUDA tensor used in place, else numbers checked and
        uploaded (a single number for every entry)"""
        dev = self.state.device
        if isinstance(v, torch.Tensor) and v.is_cuda:
            if v.dtype != dtype or tuple(v.shape) != (n,) or not v.is_contiguous() or v.device != dev:
                raise ValueError(f"a CUDA {what} tensor must be a contiguous {dtype} tensor of shape ({n},) on {dev}")
            return v
        vals = v.tolist() if isinstance(v, torch.Tensor) else v
        vals = list(vals) if isinstance(vals, (list, tuple)) else [vals] * n
        if len(vals) != n:
            raise ValueError(f"{what} gives {len(vals)} values for {n} entries")
        if dtype == torch.int32:
            vals = [_whole(f, what, 0) for f in vals]
            if max(vals) >= 2 ** 31 - 1:
                raise ValueError(f"{what} must be below 2**31 - 1 samples")
        else:
            for g in vals:
                _real(g, what, lambda g: 0.0 <= g <= self.GAIN_MAX, f"finite numbers in [0, {self.GAIN_MAX:g}]")
        return torch.tensor(vals, dtype=dtype).to(dev)

    def _words(self):
        """(g0, g1, F, p, set) of channel 0 of every row, p clamped into [0, F]"""
        w = self.state[:, 0]
        f1 = w[:, 2].view(torch.int32)
        F = (f1 - 1).clamp(min=0)
        p = torch.minimum(w[:, 3].view(torch.int32).clamp(min=0), F)
        return w[:, 0], w[:, 1], F, p, f1 > 0

    @property
    def level(self):
        """[records + slots] float32 CUDA tensor: the gain of the last sample each row mixed (entry b: record b; entry
        records + s: slot s's ambient gain), computed on the device, never synchronising.  It follows the kernel's ramp
        up to the rounding of torch's cos against the kernel's cospif."""
        g0, g1, F, p, is_set = self._words()
        x = p.float() / F.clamp(min=1).float()
        ramp = g0 + (g1 - g0) * (1.0 - torch.cos(math.pi * x)) * 0.5
        lvl = torch.where(p >= F, g1, ramp)
        rest = torch.zeros_like(lvl)
        rest[:self.n_records] = 1.0
        return torch.where(is_set, lvl, rest)

    @property
    def fading(self):
        """[records + slots] bool CUDA tensor: the rows whose ramp has samples left to mix, never synchronising"""
        _, _, F, p, is_set = self._words()
        return is_set & (p < F)


class Limiter(_SlotStage):
    """A per-slot look-ahead peak limiter on the device (l2h_limiter): each listener's output kept under `ceiling`, with
    one gain for all channels at each sample, so the interaural level ratios the binaural output carries are preserved.
    Place it after the up-resampler, on the samples the device plays: band-limited upsampling of a signal limited at
    16 kHz can overshoot the ceiling between its samples.

    Every written sample satisfies |y| <= ceiling exactly, whatever the input.  Output is the slot's signal delayed by
    La = round(lookahead * rate) samples (La / rate of added latency; 44 samples at 44.1 kHz for the 1 ms default), times
    a gain that is exactly 1 while no reduction is pending, so below the ceiling y is the delayed input bit for bit.  A
    peak is met by a gain reduction that starts La samples ahead of it, and the reduction then recovers at `release` dB
    per second.  The gain is computed in an integer log domain, so cutting a stream into other pushes changes no bit of
    the output or the state.  A non-finite sample is written as 0 and mutes the output around it; the gain then recovers
    at the release rate from about 900 dB of reduction, and `reset` ends the mute at once.

    `state` [slots, channels, 4 + 3 La] is a float32 tensor on `device`: all zeros is a fresh slot, so a listener is reset
    by zeroing its rows (`reset`) and moved by copying them."""

    Q = 65536                                  # log-gain quanta per octave of amplitude (l2h_limiter)
    MUTE = 150 * Q                             # the cap of a reduction, a gain of exactly 0
    DB_PER_OCTAVE = 20 * math.log10(2)

    def __init__(self, slots, channels, rate, ceiling=10 ** (-1 / 20), lookahead=0.001, release=80.0, device=None):
        super().__init__(slots, channels)
        self.rate = _whole(rate, "rate")
        self.ceiling = self._level(ceiling, "ceiling")
        _real(lookahead, "lookahead", lambda s: 0 <= s < 2 ** 31 / self.rate, "a number of seconds >= 0")
        _real(release, "release", lambda r: 0 < r < math.inf, "a positive number of dB per second")
        self.lookahead = round(lookahead * self.rate)
        self.release_step = max(1, round(release / self.DB_PER_OCTAVE * self.Q / self.rate))
        if self.release_step > self.MUTE:
            raise ValueError(f"release {release!r} dB/s recovers more than the whole range in one sample")
        self._allocate(*_layout(_cabi.lib().l2h_limiter_layout, self.channels, self.lookahead), device)

    @staticmethod
    def _level(v, what, zero=False):
        """v rounded to float32, where it must be a positive normal number (or 0 if `zero`), or ValueError"""
        must = "a positive amplitude that float32 holds as a normal number"
        f = float(torch.tensor(_real(v, what, must=must), dtype=torch.float32))
        if not (2.0 ** -126 <= f < math.inf or (zero and v == 0)):
            raise ValueError(f"{what} must be {must}, got {v!r}")
        return f

    def __call__(self, x, counts, slots, unit=1, out=None):
        """x [n, channels, L] CUDA tensor: row i pushes its first counts[i] * unit samples into slot slots[i] and receives
        as many back, y[i, :, :counts[i] * unit]: its slot's signal delayed by La samples times the linked gain.  Returns
        y [n, channels, L] float32 (`out`, if given, written in place; it must not overlap x).  Its later samples are left
        unwritten.

        `counts`/`unit` follow the packet stages: lim(y44, n44, slots) after PacketResampler up,
        lim(y48, hops, slots, unit=384) after a 48 kHz StreamResampler up, lim(mix, hops, slots, unit=128) on the mixer's
        16 kHz output.  Host lists are checked (slots n distinct ints in [0, slots), counts n ints in [0, L // unit]) and
        uploaded; contiguous CUDA int32 tensors are used in place and read when the kernel runs, where a slot outside
        [0, slots) or a count * unit outside [0, L] marks a row that stores nothing (neither its out row nor its state
        rows change).  So a call captured in the tick's CUDA graph serves any lists rewritten in place."""
        x = self._rows_in(x)
        dev = self.state.device
        n, C, L = x.shape
        unit = _whole(unit, "unit")
        slots = device_list(slots, dev, n, self.n_slots, True, "slot")
        counts = device_list(counts, dev, n, L // unit + 1, False, "count")
        out = self._rows_out(out, (n, C, L))
        self._run("l2h_limiter", x, x.stride(0), x.stride(1), L, counts, unit, out, out.stride(0), out.stride(1), n, C, slots,
                  self.state, self.n_slots, self.ceiling, self.lookahead, self.release_step)
        return out

    def set_ceiling(self, slots, values):
        """Give the listed slots their own ceilings (a hearing-safety cap per user): `values` one number or one per slot,
        positive finite amplitudes, or 0 for the limiter's `ceiling`.  It applies to the samples pushed after the set.
        Enqueued on the current stream; `reset` returns a slot to the default."""
        idx = self._indices(slots, self.n_slots, "slot", True, "set_ceiling")
        n = idx.numel()
        vals = values.tolist() if isinstance(values, torch.Tensor) else values
        vals = list(vals) if isinstance(vals, (list, tuple)) else [vals] * n
        if len(vals) != n:
            raise ValueError(f"values gives {len(vals)} ceilings for {n} slots")
        vals = [self._level(v, "a ceiling", zero=True) for v in vals]
        self.state[idx, 0, 1] = torch.tensor(vals, dtype=torch.float32).to(self.state.device)

    @property
    def reduction(self):
        """[slots] float32 CUDA view of the state: the dB of gain reduction at the last sample each slot wrote"""
        return self.state[:, 0, 3]

    @property
    def limited(self):
        """[slots] int32 CUDA view of the state: the samples each slot wrote with a gain reduction since its reset
        (saturating at 2**31 - 1)"""
        return self.state[:, 0, 2].view(torch.int32)


class Leveler(_SlotStage):
    """A per-row loudness leveler on the device (l2h_leveler): each voice a listener hears brought to one loudness, with
    one gain for all channels, so the interaural level ratios the binaural output carries are preserved.  A row is a
    separator record (level the target rows of `Net.advance_target_rows` before the mixer, so voices that are 15-20 dB
    apart in the mixture reach the mixer at one level), or a listener slot (level the mixer's sum, records = slots).

    It works on the separator's 16 kHz grid, hop by hop, with no look-ahead and no added delay.  Each hop's loudness is
    measured as BS.1770 defines it (K-weighted mean square, summed over the channels, in LUFS).  Hops that pass the
    absolute `gate` and, once the row has an estimate, the `relative` gate below it update the estimate: the plain mean
    of the first hops, then an exponential average over `window` seconds.  Pauses and a silent target's residual fail
    the gate and never pull the gain up.  The gain (dB) stays at 0 until the row has `settle` seconds of gated hops, then
    takes clamp(target - estimate, min_gain, max_gain) at once, and afterwards follows it at most `rise` dB/s up and
    `fall` dB/s down.  The gain is interpolated in dB across each hop.  A hop's result depends only on the row's state and
    its samples, so cutting hops into other ticks changes no bit; with min_gain = max_gain = 0 the output is the input bit
    for bit.  A hop with a non-finite sample is not measured and leaves the state as it was.

    The defaults are choices, not values tuned on trained separator output.

    `state` [rows, channels, 7] is a float32 tensor on `device`: all zeros is a fresh row, so rows are reset by zeroing
    them (`reset`) and moved by copying them."""

    def __init__(self, rows, channels, target=-20.0, gate=-50.0, relative=-20.0, window=3.0, settle=0.256,
                 min_gain=-12.0, max_gain=12.0, rise=3.0, fall=10.0, device=None):
        super().__init__(rows, channels)
        num = {k: _real(v, k) for k, v in (("target", target), ("gate", gate), ("relative", relative),
                                                   ("window", window), ("settle", settle), ("min_gain", min_gain),
                                                   ("max_gain", max_gain), ("rise", rise), ("fall", fall))}
        if num["relative"] > 0:
            raise ValueError(f"relative must be at most 0 LU, got {relative!r}")
        if num["window"] <= 0 or num["settle"] <= 0:
            raise ValueError(f"window and settle must be positive seconds, got {window!r} and {settle!r}")
        if not -40.0 <= num["min_gain"] <= num["max_gain"] <= 40.0:
            raise ValueError(f"the gain range must satisfy -40 <= min_gain <= max_gain <= 40 dB, got {min_gain!r}, "
                             f"{max_gain!r}")
        if num["rise"] < 0 or num["fall"] < 0:
            raise ValueError(f"rise and fall must be dB/s >= 0, got {rise!r} and {fall!r}")
        self.target, self.gate, self.relative = num["target"], num["gate"], num["relative"]
        self.min_gain, self.max_gain = num["min_gain"], num["max_gain"]
        self.alpha = -math.expm1(-self.HOP_S / num["window"])
        self.settle_hops = max(1, round(num["settle"] / self.HOP_S))
        self.rise_step, self.fall_step = num["rise"] * self.HOP_S, num["fall"] * self.HOP_S
        if self.settle_hops >= 2 ** 31 or self.alpha <= 0:
            raise ValueError(f"settle {settle!r} s or window {window!r} s is out of range")
        self._allocate(*_layout(_cabi.lib().l2h_leveler_layout, self.channels), device)

    def __call__(self, y, records, offsets=None, hops=None, out=None):
        """y [R, channels, 128 * T] CUDA tensor: row r is leveled with the state of row records[r].  Returns out [R,
        channels, 128 * T] float32 (`out`, if given, written in place; out=y levels y in place): listener i owns rows
        offsets[i] .. offsets[i+1]-1 (without offsets, row i alone) and its rows receive their first 128 h samples, h =
        hops[i] (T without hops).  Their later samples, and rows that store nothing, are left unwritten.

        Lists follow TargetMixer: host lists are checked and uploaded (`records` R distinct ints in [0, rows); `offsets`
        n + 1 ints from 0, non-decreasing, at most R; `hops` n ints in [0, T], n = R without offsets); contiguous CUDA
        int32 tensors are used in place and read when the kernel runs, where a record outside the leveler marks a row
        that stores nothing and advances nothing, the offsets are clamped as the separator clamps them, rows from
        offsets[n] on store nothing, and a hop count outside [1, T] stores nothing.  So a call captured in a CUDA graph
        with the FIFO, the separator and the mixer serves any lists rewritten in place.  Before the mixer:
        lev(y, records, offsets, hops=hops, out=y); on the mixer's sum: lev(mix, slots, hops=hops, out=mix)."""
        y = self._rows_in(y, self.HOP)
        dev = self.state.device
        R, C, L = y.shape
        T = L // self.HOP
        records = device_list(records, dev, R, self.n_slots, True, "record")
        if offsets is None:
            n = R
        else:
            n = (offsets.numel() if isinstance(offsets, torch.Tensor) else len(offsets)) - 1
            if not 0 < n <= R:
                raise ValueError(f"offsets must hold n + 1 entries with 0 < n <= R = {R}, got {n + 1}")
            offsets = device_offsets(offsets, dev, n, R)
        if n > self.n_slots:
            raise ValueError(f"a call of {n} listeners needs n <= rows = {self.n_slots}")
        hops = self._hops(hops, n, T)
        out = self._rows_out(out, (R, C, L))
        self._run("l2h_leveler", y, y.stride(0), y.stride(1), out, out.stride(0), out.stride(1), n, R, C, T, records,
                  offsets, hops, self.state, self.n_slots, self.target, self.gate, self.relative, self.alpha,
                  self.settle_hops, self.min_gain, self.max_gain, self.rise_step, self.fall_step)
        return out

    @property
    def loudness(self):
        """[rows] float32 CUDA tensor: the loudness (LUFS) of each row's estimate, -inf before its first gated hop;
        computed on the device, never synchronising"""
        w = self.state[:, 0]
        lufs = -0.691 + 10.0 * torch.log10(w[:, 0].clamp(min=torch.finfo(torch.float32).tiny))
        return torch.where(w[:, 1].view(torch.int32) > 0, lufs, torch.full_like(lufs, -math.inf))

    @property
    def gain(self):
        """[rows] float32 CUDA view of the state: each row's gain in dB at the last sample it wrote"""
        return self.state[:, 0, 2]


class BandCompressor(_SlotStage):
    """A per-slot multiband compressor on the device (l2h_band_compressor): each listener's output fitted to their hearing,
    with a gain per band and per ear and compression per band ("wide dynamic range compression") that is the same for
    both ears, so the dynamics keep the interaural level differences the binaural output carries.  Hearing loss depends on
    frequency and often differs between the ears; a profile sets both per listener (`set_profile`).

    It runs on the mixer's 16 kHz sum, one row per slot: cmp(mix, slots, hops=hops, out=mix).  The separated audio holds
    nothing above 8 kHz, so 16 kHz loses nothing and is the cheapest place for it; the limiter stays after the
    up-resampler.  The bank (`design`) splits the band at `edges` Hz into linear-phase FIR bands of `taps` taps that sum
    to a delay of `delay` = (taps - 1) / 2 samples: 64 samples (4 ms) at the defaults, five octave-wide bands.  Per hop
    of 128 samples each band's level, averaged over the channels, drives a detector that follows it with time constants
    `attack` (level rising) and `release` (falling) in seconds; a band's compression is slope * max(0, level - knee) dB
    with slope = 1 - 1 / ratio, and ear c's band b takes clamp(gain_cb - compression_b, -40, 40) dB at the hop's end,
    interpolated in dB across the hop.  While every gain of a slot is 0 dB, as in a fresh slot, the output is the input
    delayed by `delay` samples, bit for bit.  A hop's result depends only on the slot's state and its samples, so cutting
    hops into other ticks changes no bit.  A non-finite sample, or one of magnitude 2^32 or more, enters as 0, and its hop
    is not measured.

    `bank` chooses the filters: "fir" (the default, above), or "lr4" / "lr8", a Linkwitz-Riley crossover tree of order 4
    or 8 (`design_lr`; l2h_band_compressor_lr) whose bands sum to an allpass: flat in magnitude, with a delay that is
    short and falls with frequency (1.83 ms at 250 Hz down to 0.19 ms at 6 kHz for "lr4" at the default edges, against
    the FIR bank's 4 ms), for weaker band separation and a non-linear phase (INTEGRATION.md, "Choosing the compressor's
    bank").  An LR bank has no pure delay (`delay` is 0) and no bypass: at 0 dB its output is the allpass cascade of the
    input.  `taps` applies to the FIR bank only.

    `taps` is the bank on the device: [bands, taps] float32 FIR taps, or [bands, S, 5] float32 second-order sections for
    an LR bank.  `state` [slots, channels, row] is a float32 tensor on `device` (row = 5 bands + taps - 1 for the FIR
    bank, 5 bands + 2 bands S for an LR bank): all zeros is a fresh slot with a flat 0 dB profile and no compression, so
    a listener is reset by zeroing its rows (`reset`) and moved by copying them."""

    RATE = 16000
    RANGE = 40.0                                # the gains' clamp, dB
    BANKS = {"fir": None, "lr4": 4, "lr8": 8}   # bank -> LR order

    def __init__(self, slots, channels, edges=(500, 1000, 2000, 4000), taps=129, attack=0.005, release=0.08,
                 device=None, bank="fir"):
        super().__init__(slots, channels)
        if not isinstance(bank, str) or bank not in self.BANKS:
            raise ValueError(f"bank must be one of {', '.join(map(repr, self.BANKS))}, got {bank!r}")
        self.bank, self.order = bank, self.BANKS[bank]
        if self.order is None:
            table = self.design(edges, taps)
            self.bands, self.n_taps = table.shape
            self.delay = (self.n_taps - 1) // 2
        else:
            if isinstance(taps, bool) or taps != 129:
                raise ValueError(f"taps applies to the FIR bank only, got taps={taps!r} with bank={bank!r}")
            table = self.design_lr(edges, self.order)
            self.bands, self.n_taps, self.delay = table.shape[0], None, 0
        self.edges = tuple(float(e) for e in torch.as_tensor(edges, dtype=torch.float32).reshape(-1).tolist())
        def coef_of(tau):                       # the per-hop step of a detector with time constant tau seconds
            return -math.expm1(-self.HOP_S / tau)

        coef = {}
        for what, tau in (("attack", attack), ("release", release)):
            _real(tau, what, lambda t: 0 < t < math.inf and float(torch.tensor(coef_of(t), dtype=torch.float32)) > 0,
                  "a positive number of seconds")
            coef[what] = coef_of(tau)
        self.attack, self.release = float(attack), float(release)
        self.attack_coef, self.release_coef = coef["attack"], coef["release"]
        if self.order is None:
            self._allocate(*_layout(_cabi.lib().l2h_band_compressor_layout, self.channels, self.bands, self.n_taps), device)
        else:
            self._allocate(*_layout(_cabi.lib().l2h_band_compressor_lr_layout, self.channels, self.bands, self.order),
                           device)
        self._bank = torch.zeros(max(1, table.numel()), device=self.state.device)   # one band: a pointer to no words
        self._bank[:table.numel()].copy_(table.reshape(-1))
        self.taps = self._bank[:table.numel()].view(table.shape)

    @staticmethod
    def _edges(edges):
        """edges as a contiguous float32 CPU tensor of at most 15 entries, or ValueError"""
        try:
            e = torch.as_tensor(edges, dtype=torch.float32).reshape(-1).contiguous()
        except (TypeError, ValueError, RuntimeError):
            raise ValueError(f"edges must be a sequence of numbers of Hz, got {edges!r}") from None
        if isinstance(edges, (str, bytes)) or e.numel() >= 16:
            raise ValueError(f"edges must be at most 15 numbers of Hz (at most 16 bands), got {edges!r}")
        return e

    @staticmethod
    def design_lr(edges=(500, 1000, 2000, 4000), order=4):
        """The Linkwitz-Riley bank of K = len(edges) + 1 bands cut at `edges` Hz (rising strictly inside (0, 8000)) with
        crossovers of `order` 4 or 8, as a [K, S, 5] float32 CPU tensor of second-order sections (b0, b1, b2, a1, a2),
        S = order / 2 (K - 1) (l2h_band_compressor_lr_design): at each edge LP = (Butterworth low-pass)^2, HP =
        (Butterworth high-pass)^2 of order / 2, as scipy.signal.butter designs them at fs=16000, and AP the allpass on the
        same poles; band j is the HPs of the edges below it, its own LP (every band but the last) and the APs of the edges
        above that, padded with identity sections, computed in float64, so the bands sum to the product of the APs."""
        e = BandCompressor._edges(edges)
        if isinstance(order, bool) or order not in (4, 8):
            raise ValueError(f"order must be 4 or 8, got {order!r}")
        N = int(order)
        S = N // 2 * e.numel()
        buf = torch.empty(max(1, (e.numel() + 1) * S * 5), dtype=torch.float32)    # one band: no sections, no words
        _check(_cabi.lib().l2h_band_compressor_lr_design(e.numel() + 1, e.data_ptr() if e.numel() else None, N,
                                                         buf.data_ptr()))
        return buf[:(e.numel() + 1) * S * 5].view(e.numel() + 1, S, 5)

    @staticmethod
    def design(edges=(500, 1000, 2000, 4000), taps=129):
        """The bank of K = len(edges) + 1 bands cut at `edges` Hz (rising strictly inside (0, 8000)), each a linear-phase
        FIR of `taps` taps (odd, 33 to 255), as a [K, taps] float32 CPU tensor (l2h_band_compressor_design): with LP_j =
        scipy.signal.firwin(taps, edge_j, fs=16000), band 0 is LP_1, band j is LP_{j+1} - LP_j and the last band is a
        delay of (taps - 1) / 2 samples minus LP_{K-1}, computed in float64, so the bands sum to that delay."""
        e = BandCompressor._edges(edges)
        L = _whole(taps, "taps")
        out = torch.empty(e.numel() + 1, L, dtype=torch.float32)
        _check(_cabi.lib().l2h_band_compressor_design(e.numel() + 1, e.data_ptr() if e.numel() else None, L,
                                                      out.data_ptr()))
        return out

    def __call__(self, y, slots, hops=None, out=None):
        """y [n, channels, 128 * T] CUDA tensor, the mixer's sum: row i is compressed with the state of slot slots[i].
        Returns out [n, channels, 128 * T] float32 (`out`, if given, written in place; out=y compresses y in place): row
        i receives its first 128 h samples, h = hops[i] (T without hops).  Its later samples, and rows that store nothing,
        are left unwritten.

        Lists follow Leveler on the mixer's sum: host lists are checked and uploaded (`slots` n distinct ints in
        [0, slots), `hops` n ints in [0, T]); contiguous CUDA int32 tensors are used in place and read when the kernel
        runs, where a slot outside [0, slots) or a hop count outside [1, T] marks a row that stores nothing and advances
        nothing.  So a call captured in the tick's CUDA graph serves any lists rewritten in place."""
        y = self._rows_in(y, self.HOP)
        dev = self.state.device
        n, C, L = y.shape
        T = L // self.HOP
        slots = device_list(slots, dev, n, self.n_slots, True, "slot")
        hops = self._hops(hops, n, T)
        out = self._rows_out(out, (n, C, L))
        entry, shape = ("l2h_band_compressor", self.n_taps) if self.order is None else ("l2h_band_compressor_lr", self.order)
        self._run(entry, y, y.stride(0), y.stride(1), out, out.stride(0), out.stride(1), n, C, T, slots, hops, self._bank,
                  self.bands, shape, self.state, self.n_slots, self.attack_coef, self.release_coef)
        return out

    def set_profile(self, slots, gains, knees=0.0, ratios=1.0):
        """Fit the listed slots: `gains` in dB per band, [K] for every slot and both ears, [n, K] per slot for both ears,
        or [n, channels, K] per slot and ear, each in [-40, 40]; `knees` in dBFS and `ratios` >= 1 per band, each a
        number, [K] or [n, K].  A band compresses by (1 - 1 / ratio) dB per dB its level lies above its knee.  Enqueued on
        the current stream; it takes effect from the next hop, across one hop's dB ramp, and `reset` returns a slot to
        the flat profile."""
        dev, K, C = self.state.device, self.bands, self.channels
        rows = self._indices(slots, self.n_slots, "slot", True, "set_profile")
        n = rows.numel()
        g = self._table(gains, "gains", n, [(K,), (n, K), (n, C, K)], lambda v: -self.RANGE <= v <= self.RANGE,
                        f"dB in [{-self.RANGE:g}, {self.RANGE:g}]")
        kn = self._table(knees, "knees", n, [(), (K,), (n, K)], math.isfinite, "finite dBFS")
        ra = self._table(ratios, "ratios", n, [(), (K,), (n, K)], lambda v: v >= 1, "ratios >= 1")
        g = (g.reshape(1, 1, K) if g.dim() == 1 else g.reshape(n, -1, K)).expand(n, C, K)
        kn, ra = ((t.expand(K) if t.dim() == 0 else t).reshape(-1, K).expand(n, K) for t in (kn, ra))
        self.state[rows, :, :K] = g.float().to(dev)
        self.state[rows, 0, 3 * K:4 * K] = kn.float().to(dev)
        self.state[rows, 0, 4 * K:5 * K] = (1.0 - 1.0 / ra).float().to(dev)

    @staticmethod
    def _table(v, what, n, shapes, ok, must):
        """v as a float64 CPU tensor of one of `shapes` whose every entry is `must` (passes `ok`), or ValueError"""
        try:
            t = torch.as_tensor(v.detach().cpu() if isinstance(v, torch.Tensor) else v, dtype=torch.float64)
        except (TypeError, ValueError, RuntimeError):
            t = None
        if t is None or tuple(t.shape) not in shapes or isinstance(v, bool):
            raise ValueError(f"{what} must be numbers of shape {' or '.join(str(list(s)) for s in shapes)}, got {v!r}")
        for x in t.reshape(-1).tolist():
            _real(x, f"every entry of {what}", ok, must)
        return t

    @property
    def level(self):
        """[slots, bands] float32 CUDA tensor: each band's detector level in dBFS (a full-scale sine reads -3.01), -inf
        before the slot's first measured hop; computed on the device, never synchronising"""
        K = self.bands
        return 10.0 * torch.log10(self.state[:, 0, 2 * K:3 * K])

    @property
    def gain(self):
        """[slots, channels, bands] float32 CUDA view of the state: each band's gain in dB at the last sample written"""
        return self.state[:, :, self.bands:2 * self.bands]


class JitterBuffer(_SlotStage):
    """A per-slot jitter buffer on the device (l2h_jitter_buffer): the first stage of a tick for devices that send packets
    of `packet` samples at `rate` Hz with RTP's 16-bit sequence numbers over a lossy network.  It puts the packets back in
    sequence order, drops late and duplicate ones, and conceals lost ones, so every later stage sees one continuous
    stream at the device's rate: jb(x, seqs, counts, slots) -> (y, out_counts), then PacketResampler (unit=packet) or,
    for a 16 kHz device, HopFifo (unit=packet).

    Arrivals are processed one at a time in row order.  `next` is the sequence number of the next packet to decide (the
    first packet of a fresh slot sets it), and d = (s - next) mod 2**16 taken in [-2**15, 2**15).  A packet with d < 0 is
    late, one already held a duplicate, and one with d >= `window` restarts the slot (the held packets are dropped, next
    := s, and the packet fades in).  Others are held.  Then, while next is held it is released; while it is missing and a
    packet at least `depth` + 1 past it is held, it is declared lost and released as concealment.  In-order traffic is
    therefore released on arrival, bit for bit with no added delay, and `depth` is the reordering a gap waits for.  A
    call writes at most `max_out` released packets per row; the rest wait (a backlog of up to `window` packets) and are
    written first by the slot's next call.  Decisions depend on the arrivals alone: cutting them into other calls, or
    another max_out, moves only where the output is cut.

    A lost packet repeats the last pitch period (2.5-15 ms, found by normalised autocorrelation over the last 20 ms of
    the channel sum, one lag for all channels) at gain 1 for 10 ms, falling linearly to 0 at 60 ms and silent after; the
    first real packet after a run or a restart fades in from the continuing concealment along a raised cosine over
    min(4 ms, packet).  A non-finite sample, or one of magnitude 2**32 or more, enters as 0.

    With `deadline` (microseconds; l2h_jitter_buffer_timed) the buffer also releases on time: every call takes `now`,
    the server's clock in microseconds, and a missing packet is declared lost either by the rule above or once its
    deadline has passed, whichever comes first.  A slot anchors its clock on the highest packet it has placed: packet s
    is expected at the anchor's arrival time plus (s - anchor) packet periods, and the packet at next expires once now
    lies `deadline` past that.  After its arrivals, each call releases every expired packet as a loss (counted in `lost`
    and `expired`), so a gap in a device's uplink is concealed as it happens.  Once the concealment has gone silent (60 ms
    of packets past the anchor) the slot releases nothing more, and its next arrival at or past next restarts it, so a
    long outage adds no latency.  A slot's deadlines are checked only in calls that list it: list every live slot in
    every tick, with count 0 when it sent nothing.  With a deadline no call reaches, the output is the untimed buffer's.

    With `deadline=(lo, hi)` (l2h_jitter_buffer_adaptive) each slot draws its own deadline from the measured lateness of
    its packets: a packet's lateness is its arrival time minus the time the anchor expects it, and a slot keeps a
    64-bin histogram of it over about the last 5 s of packets, in exact integer arithmetic.  Once per call the slot's
    deadline becomes the smallest bin edge that leaves at most `late_rate` of the measured packets later than it,
    clamped to [lo, hi]; it is `hi` until 1 / late_rate packets have been measured.  A slot's first packet, duplicates,
    restarts and arrivals while the slot is stalled are not measured; late packets are.  Each call may take `arrivals`,
    the packets' arrival times on the server's clock (else each arrives at `now`).  `deadline_us` reads each slot's
    current deadline.  With lo == hi and no arrival times the output is the timed buffer's at that deadline.

    `state` [slots, channels, row] is a float32 tensor on `device`: all zeros is a fresh slot, so a listener is reset by
    zeroing its rows (`reset`) and moved by copying them.  The counters are int32 views that never synchronise."""

    SEQ = 1 << 16
    LOST, LATE, DUPLICATE, DROPPED, RESTARTS, HELD, PITCH = 6, 7, 8, 9, 10, 11, 12   # head words of channel 0
    EXPIRED = 15

    def __init__(self, slots, channels, rate, packet, depth=1, window=16, max_out=4, device=None, deadline=None,
                 late_rate=None):
        super().__init__(slots, channels)
        self.rate, self.packet = _whole(rate, "rate"), _whole(packet, "packet")
        self.depth, self.window = _whole(depth, "depth", 0), _whole(window, "window")
        self.max_out = _whole(max_out, "max_out")
        self.adaptive = isinstance(deadline, (tuple, list))
        if self.adaptive:
            if len(deadline) != 2:
                raise ValueError(f"an adaptive deadline is a pair (lo, hi) of microseconds, got {deadline!r}")
            lo, hi = _whole(deadline[0], "deadline lo", 0), _whole(deadline[1], "deadline hi", 0)
            if lo > hi:
                raise ValueError(f"deadline (lo, hi) needs lo <= hi, got {deadline!r}")
            self.deadline = (lo, hi)
            self.late_rate = _real(0.02 if late_rate is None else late_rate, "late_rate", lambda v: 0 < v <= 0.5,
                                   "a number in (0, 0.5]")
        else:
            if late_rate is not None:
                raise ValueError("late_rate is given only with an adaptive deadline=(lo, hi)")
            self.deadline = None if deadline is None else _whole(deadline, "deadline", 0)
            self.late_rate = None
        if self.depth >= self.window:
            raise ValueError(f"depth must be below window = {self.window} packets, got {depth!r}")
        query = _cabi.lib().l2h_jitter_buffer_adaptive_layout if self.adaptive else _cabi.lib().l2h_jitter_buffer_layout
        self._allocate(*_layout(query, self.channels, self.rate, self.packet, self.depth, self.window, self.max_out),
                       device)

    def __call__(self, x, seqs, counts, slots, out=None, out_counts=None, now=None, arrivals=None):
        """x [n, channels, M * packet] CUDA tensor: row i pushes its packets j < counts[i], x[i, :, j P:(j + 1) P], with
        sequence numbers seqs[i, j], into slot slots[i].  Returns (y [n, channels, max_out * packet] float32, out_counts [n]
        int32 CUDA) (`out` and `out_counts`, if given, written in place): row i receives y[i, :, :out_counts[i] * packet],
        its slot's next packets in sequence order; its later samples are left unwritten.

        `now` is required exactly when the buffer has a deadline: the server's clock in microseconds, a host int (taken
        mod 2**32) or a CUDA int32 tensor of shape (1,) used in place and read when the kernel runs.

        `arrivals` (adaptive deadline only; optional) [n, M]: each packet's arrival time on the same clock, in
        microseconds, a host integer array (taken mod 2**32, checked and uploaded) or a contiguous CUDA int32 tensor
        used in place and read when the kernel runs.  An arrival after `now` is taken as now; without `arrivals` every
        packet arrives at now.

        Host lists are checked and uploaded (`slots` n distinct ints in [0, slots), `counts` n ints in [0, M], `seqs` [n, M]
        int32 values whose first counts[i] entries of row i lie in [0, 65535], so a short row may be padded with -1; with
        counts on the device every entry is checked); contiguous CUDA int32 tensors are used in place and read when the kernel runs, where a slot
        outside [0, slots) or a count outside [0, M] marks a row that stores nothing and gets out count 0, and a sequence
        number outside [0, 65535] marks a packet that is skipped.  So a call captured in the tick's CUDA graph serves any
        lists rewritten in place."""
        x = self._rows_in(x, self.packet)
        now = self._now(now)
        dev = self.state.device
        n, C, L = x.shape
        M = L // self.packet
        arrivals = self._arrivals(arrivals, n, M)
        slots = device_list(slots, dev, n, self.n_slots, True, "slot")
        host_counts = None if isinstance(counts, torch.Tensor) and counts.is_cuda else counts
        counts = device_list(counts, dev, n, M + 1, False, "count")
        seqs = self._seqs(seqs, n, M, host_counts)
        out = self._rows_out(out, (n, C, self.max_out * self.packet))
        out_counts = self._ints_out(out_counts, n, "out_counts")
        args = (x, x.stride(0), x.stride(1), M, seqs, counts, out, out.stride(0), out.stride(1), out_counts, n, C, slots,
                self.state, self.n_slots, self.rate, self.packet, self.depth, self.window, self.max_out)
        if now is None:
            self._run("l2h_jitter_buffer", *args)
        elif self.adaptive:
            self._run("l2h_jitter_buffer_adaptive", *args, now, arrivals, *self.deadline, self.late_rate)
        else:
            self._run("l2h_jitter_buffer_timed", *args, now, self.deadline)
        return out, out_counts

    def _arrivals(self, arrivals, n, M):
        """the [n, M] int32 arrival times on the state's device (None: every packet arrives at now): a CUDA tensor used
        in place, else integers taken mod 2**32 and uploaded; ValueError without an adaptive deadline"""
        if arrivals is None:
            return None
        if not self.adaptive:
            raise ValueError("arrivals are given only to a JitterBuffer with an adaptive deadline=(lo, hi)")
        dev = self.state.device
        if isinstance(arrivals, torch.Tensor) and arrivals.is_cuda:
            if (arrivals.dtype != torch.int32 or tuple(arrivals.shape) != (n, M) or not arrivals.is_contiguous()
                    or arrivals.device != dev):
                raise ValueError(f"a CUDA arrivals tensor must be a contiguous int32 tensor of shape ({n}, {M}) on {dev}")
            return arrivals
        try:
            v = torch.as_tensor(arrivals)
        except (TypeError, ValueError, RuntimeError, OverflowError):
            raise ValueError("arrivals must be integers of microseconds (each within int64)") from None
        if v.dtype.is_floating_point or v.dtype.is_complex or v.dtype == torch.bool or tuple(v.shape) != (n, M):
            raise ValueError(f"arrivals must be integers of shape ({n}, {M}), got {tuple(v.shape)} {v.dtype}")
        w = v.to(torch.int64).remainder(2 ** 32)
        return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32).contiguous().to(dev)

    def _now(self, now):
        """the clock of a call as a CUDA int32 tensor of shape (1,) on the state's device (None without a deadline), or
        ValueError"""
        if self.deadline is None:
            if now is not None:
                raise ValueError("now is given to a JitterBuffer without a deadline")
            return None
        dev = self.state.device
        if isinstance(now, torch.Tensor) and now.is_cuda:
            if now.dtype != torch.int32 or tuple(now.shape) != (1,) or now.device != dev:
                raise ValueError(f"a CUDA now tensor must be an int32 tensor of shape (1,) on {dev}")
            return now
        if now is None:
            raise ValueError("a JitterBuffer with a deadline needs now, the server's clock in microseconds")
        if isinstance(now, bool) or not isinstance(now, numbers.Integral):
            raise ValueError(f"now must be an int of microseconds or a CUDA int32 tensor of shape (1,), got {now!r}")
        v = int(now) % 2 ** 32
        return torch.tensor([v - 2 ** 32 if v >= 2 ** 31 else v], dtype=torch.int32).to(dev)

    def _seqs(self, seqs, n, M, counts=None):
        """the [n, M] int32 sequence numbers on the state's device: a CUDA tensor used in place, else checked (the
        entries each row pushes, given host `counts`, else all of them) and uploaded"""
        dev = self.state.device
        if isinstance(seqs, torch.Tensor) and seqs.is_cuda:
            if seqs.dtype != torch.int32 or tuple(seqs.shape) != (n, M) or not seqs.is_contiguous() or seqs.device != dev:
                raise ValueError(f"a CUDA seqs tensor must be a contiguous int32 tensor of shape ({n}, {M}) on {dev}")
            return seqs
        v = torch.as_tensor(seqs)
        if v.dtype.is_floating_point or v.dtype.is_complex or v.dtype == torch.bool or tuple(v.shape) != (n, M):
            raise ValueError(f"seqs must be integers of shape ({n}, {M}), got {tuple(v.shape)} {v.dtype}")
        if v.numel() and (int(v.min()) < -2 ** 31 or int(v.max()) >= 2 ** 31):
            raise ValueError("sequence numbers must be int32 values")
        pushed = torch.ones(n, M, dtype=torch.bool) if counts is None else \
            torch.arange(M)[None] < torch.as_tensor(counts).reshape(n, 1)
        if bool(((v < 0) | (v >= self.SEQ))[pushed].any()):
            raise ValueError("the sequence numbers of pushed packets must lie in [0, 65535]")
        return v.to(torch.int32).contiguous().to(dev)

    def _word(self, k):
        return self.state[:, 0, k].view(torch.int32)

    @property
    def lost(self):
        """[slots] int32 CUDA view: packets declared lost and concealed since the slot's reset (saturating)"""
        return self._word(self.LOST)

    @property
    def late(self):
        """[slots] int32 CUDA view: packets that arrived after their turn and were dropped (saturating)"""
        return self._word(self.LATE)

    @property
    def duplicate(self):
        """[slots] int32 CUDA view: packets that arrived while the same number was held and were dropped (saturating)"""
        return self._word(self.DUPLICATE)

    @property
    def dropped(self):
        """[slots] int32 CUDA view: held packets a restart discarded, and released ones a full backlog discarded
        (saturating)"""
        return self._word(self.DROPPED)

    @property
    def restarts(self):
        """[slots] int32 CUDA view: arrivals beyond the window that restarted the slot (saturating)"""
        return self._word(self.RESTARTS)

    @property
    def held(self):
        """[slots] int32 CUDA view: packets stored and waiting for their turn"""
        return self._word(self.HELD)

    @property
    def next(self):
        """[slots] int32 CUDA view: the sequence number of the next packet to decide (released packets a call has not
        written yet, `max_out` per row, play before it)"""
        return self._word(1)

    @property
    def pitch(self):
        """[slots] int32 CUDA view: the lag, in samples, of the last concealment run (0 before the first)"""
        return self._word(self.PITCH)

    @property
    def deadline_us(self):
        """[slots] int32 CUDA view (adaptive deadline only): each slot's deadline in microseconds, as its last call
        found it from the slot's statistics (0 before the slot's first packet); read it beside `expired` and `late`"""
        if not self.adaptive:
            raise ValueError("deadline_us belongs to a JitterBuffer with an adaptive deadline=(lo, hi)")
        return self._word(self.state.shape[2] - 1)

    @property
    def expired(self):
        """[slots] int32 CUDA view: packets declared lost because their deadline passed, a part of `lost` (saturating;
        0 without a deadline)"""
        return self._word(self.EXPIRED)
