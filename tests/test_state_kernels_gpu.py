"""The kernels that own a separator state's records (csrc/sep_kernels.cuh: state_init, reset_streams, advance_header,
set_clip_base; csrc/targets_kernels.cuh: join_start, history_put, history_get, move_lead) launched directly through
the engine's launchers, every output against an exact reference (kernels/harness.py).

Cases.  The layouts of 1 and 3 blocks, records GAP floats apart.  state_init: batch 1 and 3, each record larger than one
grid-stride pass of its 592 x 256 threads.  reset_streams: unsorted lists on the real layouts, and lists of 1,
RESET_MAX_SLOTS and RESET_MAX_SLOTS + 1 slots on a synthetic 264-float stride (the kernel addresses records only
through it).  advance_header: 300 streams (the 256-thread loop wraps), the header clock crossing 2^32, a record clock
crossing 2^32, a call count wrapping past 2^31 - 1, done non-zero.  set_clip_base: header clock 2^40 + 7.
join_start (kernels/harness.py::join_start_case): lead clocks 0, 1, 49, 50, 51, 2^31 - 1, 2^31 + 3, 2^32 - 1, 2^32 + 5
and 2^40 + 7 against w_max 0, 1 and 50; a record listed twice, a record that is another row's lead or its own, records
and leads -1, batch and 2^31 - 1, two rows on one lead; used_out present and absent.  history_put and history_get
(history_put_case, history_get_case): rings of F = 1, 7, 50, 64 at clocks around 2^31, 2^32 and 2^40; ragged hop counts
(0, -1, T + 1, more than F); leads -1, batch, 2^31 - 1; used 0, 1, T - 1, T, T + 1, -1.  An end-to-end history: ragged
ticks of a lead starting at 2^32 - 4, one longer than the ring, then join_start and history_get must replay exactly the
lead's frames p - W .. p - 1, whatever the slot arithmetic.  move_lead: all four parity combinations of source and
destination, and MOVE_MAX_PAIRS + 1 pairs over 962 one-block records (about 2 GB, freed after the case).  The product
library's launch counter moves by one per launch of init, reset (1, 960, 961 slots) and move_lead (1, 481 pairs).

Oracle.  Each state sits between guards of the sentinel 0x7FC0DEAD, every float the reference does not write holds the
sentinel or seeded random bits, and the whole buffer must equal the reference bit for bit.  Every list the kernels
write is compared exactly.

Mutants (each must differ from the kernel on every case that names it): state_init counting records from float 0 and
leaving the embedding 0; reset keeping the clock words and skipping the slots past the first chunk; advance_header
carrying clocks in 32 bits and keeping done; join_start giving clock p, W unclamped, no lead clash, no record clash;
history_put keeping the first F frames of a long tick, taking the slot from the clock after the tick or from 32 bits;
history_get taking the slot from the lead's clock, not zeroing frames past used, or from 32 bits; move_lead copying
the tails into the source's parity and copying blocks 1 and up.

Measured on one NVIDIA H100 80GB HBM3 (700 W power limit): every output bit-exact and every mutant caught on its cases.
Run with test_embed_slot_kernels_gpu.py, the two modules took 8 s (17 s with interpreter start-up) and peaked at
1.89 GiB of device memory, in the 962-record cases.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from kernels import harness as kh
from kernels.scaffold import SENTINEL, Guarded, Records, bits, dev, is_sentinel  # noqa: F401

pytestmark = pytest.mark.gpu

GAP = 132                   # floats between two records (a multiple of 4: the kernels read float4s)
SYN_STRIDE = 264            # a synthetic record: the SPK embedding floats, the clock words and a tail
INT_MAX = kh.INT_MAX
CAUGHT = {}


def caught(key, mutants):
    CAUGHT.setdefault(key, set()).update(mutants)
    print(f"[{key}] bit-exact; mutants caught: {sorted(mutants)}")


@pytest.fixture(scope="module")
def limits(dev):
    return kh.state_limits()


@pytest.fixture(params=[1, 3], ids=["blocks1", "blocks3"])
def layout(request, dev):
    return kh.sep_layout(request.param), request.param


def i32(v, dev):
    return torch.tensor(v, dtype=torch.int32, device=dev)


def host(t):
    return bits(t).cpu().numpy()


def upload(t, a):
    t.copy_(torch.from_numpy(np.ascontiguousarray(a)).view(torch.float32).to(t.device))


def random_bits(n, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(-2 ** 31, 2 ** 31, (n,), generator=g, device=dev, dtype=torch.int64).to(torch.int32)


def set_clock(a, o, lay, clock, calls=None):
    kh.put64(a, o + lay["ST_POS"], clock)
    if calls is not None:
        a[o + lay["ST_CALLS"]] = calls


def launches(fn):
    n0 = kh.lib().kh_launch_count()
    assert fn() == 0
    return kh.lib().kh_launch_count() - n0


# ---- state_init / reset_streams --------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3])
def test_state_init(B, layout, dev):
    lay, _ = layout
    st = Records(lay, B, dev, GAP)
    assert lay["STREAM_STRIDE"] > 592 * 256                   # one record is more than one grid-stride pass
    assert launches(lambda: kh.state_init(st.t, st.ss, B)) == 1
    torch.cuda.synchronize()
    got = host(st.t)
    assert st.buf.ok() and np.array_equal(got, kh.state_init_ref(st.hdr, st.ss, B))
    for m in kh.STATE_INIT_MUTANTS:
        assert not np.array_equal(got, kh.state_init_ref(st.hdr, st.ss, B, mutant=m)), m
    caught("state_init", kh.STATE_INIT_MUTANTS)


def test_reset_streams_layouts(layout, dev):
    lay, _ = layout
    batch, slots = 6, [4, 0, 2]
    st = Records(lay, batch, dev, GAP)
    a = host(st.t)
    for b in range(batch):
        set_clock(a, st.hdr + b * st.ss, lay, kh.CLOCKS[b + 2], 2 * b + 1)
    upload(st.t, a)
    assert launches(lambda: kh.reset_streams(st.t, st.ss, batch, slots)) == 1
    torch.cuda.synchronize()
    got = host(st.t)
    assert st.buf.ok() and np.array_equal(got, kh.reset_streams_ref(a, st.hdr, st.ss, lay, slots))
    assert not np.array_equal(got, kh.reset_streams_ref(a, st.hdr, st.ss, lay, slots, mutant="clock_kept"))
    caught("reset_streams", {"clock_kept"})


@pytest.mark.parametrize("which", ["one", "max", "max_plus_1"])
def test_reset_streams_chunks(which, limits, dev):
    lim = limits["RESET_MAX_SLOTS"]
    n = {"one": 1, "max": lim, "max_plus_1": lim + 1}[which]
    lay = dict(ST_CALLS=kh.sep_layout(1)["ST_CALLS"], ST_POS=kh.sep_layout(1)["ST_POS"])
    hdr, batch = 16, lim + 5
    buf = Guarded((hdr + batch * SYN_STRIDE,), dev)
    bits(buf.t).copy_(random_bits(buf.t.numel(), 71 + n, dev))
    a = host(buf.t)
    for b in range(batch):
        set_clock(a, hdr + b * SYN_STRIDE, lay, kh.CLOCKS[b % len(kh.CLOCKS)], b)
    upload(buf.t, a)
    slots = [int(s) for s in np.random.default_rng(n).permutation(batch)[:n]]
    assert launches(lambda: kh.reset_streams(buf.t, SYN_STRIDE, batch, slots)) == math.ceil(n / lim)
    torch.cuda.synchronize()
    got = host(buf.t)
    assert buf.ok() and np.array_equal(got, kh.reset_streams_ref(a, hdr, SYN_STRIDE, lay, slots))
    muts = {"clock_kept"} | ({"first_chunk_only"} if n > lim else set())
    for m in muts:
        assert not np.array_equal(got, kh.reset_streams_ref(a, hdr, SYN_STRIDE, lay, slots, mutant=m)), m
    caught("reset_streams", muts)


def test_reset_streams_refuses_bad_slots(dev):
    buf = Guarded((16 + 4 * SYN_STRIDE,), dev)
    n0 = kh.lib().kh_launch_count()
    for slots in ([4], [-1], [0, INT_MAX]):
        assert kh.reset_streams(buf.t, SYN_STRIDE, 4, slots) != 0, slots
    assert kh.reset_streams(buf.t, SYN_STRIDE + 2, 4, [0]) != 0
    assert kh.lib().kh_launch_count() == n0 and is_sentinel(buf.whole)


# ---- advance_header / set_clip_base ----------------------------------------------------------------------------------
@pytest.mark.parametrize("form", ["synthetic300", "layout"])
def test_advance_header(form, dev):
    lay = kh.sep_layout(1)
    if form == "synthetic300":
        hdr, ss, batch, n = 16, SYN_STRIDE, 310, 300
    else:
        hdr, ss, batch, n = 16, lay["STREAM_STRIDE"] + GAP, 4, 3
    buf = Guarded((hdr + batch * ss,), dev)
    bits(buf.t).copy_(random_bits(buf.t.numel(), 81, dev))
    a = host(buf.t)
    kh.put64(a, kh.HDR_POS, 2 ** 32 - 3)
    kh.put64(a, kh.HDR_NCALLS, 2 ** 31 + 11)
    a[kh.HDR_DONE] = 7
    for b in range(batch):
        set_clock(a, hdr + b * ss, lay, kh.CLOCKS[b % len(kh.CLOCKS)], INT_MAX if b == 1 else b)
    upload(buf.t, a)
    assert launches(lambda: kh.advance_header(buf.t, ss, n, 5)) == 1
    torch.cuda.synchronize()
    got = host(buf.t)
    assert buf.ok() and np.array_equal(got, kh.advance_header_ref(a, hdr, ss, lay, n, 5))
    for m in kh.ADVANCE_MUTANTS:
        assert not np.array_equal(got, kh.advance_header_ref(a, hdr, ss, lay, n, 5, mutant=m)), m
    caught("advance_header", kh.ADVANCE_MUTANTS)


def test_set_clip_base(dev):
    buf = Guarded((16 + SYN_STRIDE,), dev)
    bits(buf.t).copy_(random_bits(buf.t.numel(), 91, dev))
    a = host(buf.t)
    kh.put64(a, kh.HDR_POS, 2 ** 40 + 7)
    upload(buf.t, a)
    assert launches(lambda: kh.set_clip_base(buf.t)) == 1
    torch.cuda.synchronize()
    got = host(buf.t)
    assert buf.ok() and np.array_equal(got, kh.set_clip_base_ref(a)) and kh.get64(got, kh.HDR_CLIP) == 2 ** 40 + 7


# ---- join_start ------------------------------------------------------------------------------------------------------
def clocked_state(lay, batch, clocks, dev, seed=None, calls=None):
    st = Records(lay, batch, dev, GAP)
    if seed is not None:
        bits(st.t).copy_(random_bits(st.t.numel(), seed, dev))
    a = host(st.t)
    for b, c in enumerate(clocks):
        set_clock(a, st.hdr + b * st.ss, lay, c, None if calls is None else calls[b])
    upload(st.t, a)
    return st, a


def join_expected(a, st, lay, ref):
    exp = a.copy()
    for s, start in ref["start"].items():
        exp[st.hdr + s * st.ss:st.hdr + (s + 1) * st.ss] = kh.fresh_record(st.ss, lay, start)
    return exp


@pytest.mark.parametrize("with_used_out", [True, False], ids=["used_out", "no_used_out"])
@pytest.mark.parametrize("w_max", [0, 1, 50])
def test_join_start(w_max, with_used_out, layout, dev):
    lay, _ = layout
    c = kh.join_start_case(w_max)
    J, batch = len(c["records"]), c["batch"]
    st, a = clocked_state(lay, batch, c["clocks"], dev)
    lists, used_out = Guarded((3 * J,), dev), Guarded((J,), dev)
    assert launches(lambda: kh.join_start(st.t, st.ss, batch, i32(c["records"], dev), i32(c["leads"], dev), w_max, J, lists.t,
                                          used_out.t if with_used_out else None)) == 1
    torch.cuda.synchronize()
    assert lists.ok() and used_out.ok() and st.buf.ok()
    got_lists, got = host(lists.t).tolist(), host(st.t)
    ref = kh.join_start_ref(c["records"], c["leads"], c["clocks"], batch, w_max)
    assert got_lists == ref["rec"] + ref["used"] + ref["owner"]
    assert host(used_out.t).tolist() == (ref["used"] if with_used_out else [SENTINEL] * J)
    assert np.array_equal(got, join_expected(a, st, lay, ref))
    for m in c["catches"]:
        mr = kh.join_start_ref(c["records"], c["leads"], c["clocks"], batch, w_max, mutant=m)
        assert got_lists != mr["rec"] + mr["used"] + mr["owner"] or not np.array_equal(got, join_expected(a, st, lay, mr)), m
    caught("join_start", c["catches"])


# ---- history_put / history_get ---------------------------------------------------------------------------------------
def frame_words(shape, seed, dev):
    """seeded non-NaN bit patterns (0 <= bits < 2^30)"""
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(0, 2 ** 30, shape, generator=g, device=dev, dtype=torch.int32)


@pytest.mark.parametrize("F", kh.HIST_F)
def test_history_put(F, layout, dev):
    lay, _ = layout
    c = kh.history_put_case(F)
    T, batch, M = c["T"], c["batch"], len(c["leads"])
    st, _ = clocked_state(lay, batch, c["clocks"], dev)
    before = st.snapshot()
    hist = Guarded((batch, F, kh.FC), dev)
    X0 = frame_words((M, T, kh.FC), 100 + F, dev)
    lead_t, hops_t = i32(c["leads"], dev), i32(c["hops"], dev)
    assert kh.history_put(X0.view(torch.float32), st.t, kh.records_map(st.ss, lead_t, batch, hops_t, T), hist.t, F, M) == 0
    torch.cuda.synchronize()
    assert hist.ok() and st.same_outside(st.index(), before)
    got, x0 = host(hist.t), X0.cpu().numpy()
    h0 = np.full((batch, F, kh.FC), SENTINEL, dtype=np.int32)
    assert np.array_equal(got, kh.history_put_ref(h0, x0, c["leads"], c["hops"], c["clocks"], F, T, batch))
    for m in c["catches"]:
        assert not np.array_equal(got, kh.history_put_ref(h0, x0, c["leads"], c["hops"], c["clocks"], F, T, batch, m)), m
    caught("history_put", c["catches"])


@pytest.mark.parametrize("F", kh.HIST_F)
def test_history_get(F, layout, dev):
    lay, _ = layout
    c = kh.history_get_case(F)
    T, batch, J = c["T"], c["batch"], len(c["rec"])
    st, _ = clocked_state(lay, batch, c["clocks"], dev)
    before = st.snapshot()
    H = frame_words((batch, F, kh.FC), 200 + F, dev)
    X0 = Guarded((J, T, kh.FC), dev)
    rec_t, used_t = i32(c["rec"], dev), i32(c["used"], dev)
    assert kh.history_get(H.view(torch.float32), F, st.t, kh.records_map(st.ss, rec_t, batch, used_t, T), i32(c["leads"], dev),
                          X0.t, J) == 0
    torch.cuda.synchronize()
    assert X0.ok() and st.same_outside(st.index(), before)
    got, h = host(X0.t), H.cpu().numpy()
    assert np.array_equal(got, kh.history_get_ref(h, c["rec"], c["used"], c["leads"], c["clocks"], F, T, batch))
    for m in c["catches"]:
        assert not np.array_equal(got, kh.history_get_ref(h, c["rec"], c["used"], c["leads"], c["clocks"], F, T, batch, m)), m
    caught("history_get", c["catches"])


@pytest.mark.parametrize("F", [7, 50])
def test_history_end_to_end(F, dev):
    """ragged ticks of lead 0 from clock 2^32 - 4 (one tick longer than the ring), the clock advanced between ticks as
    finish_call would, then a join of three rows on it at w_max = F and 3: each row replays exactly frames p - W .. p - 1
    of the lead, in order.  Frame n's element e holds the word n * 8192 + e (n counted from the first tick)."""
    lay = kh.sep_layout(1)
    batch, p0 = 5, 2 ** 32 - 4
    st, _ = clocked_state(lay, batch, [p0] + [0] * (batch - 1), dev, calls=[0] * batch)
    hist = Guarded((batch, F, kh.FC), dev)
    e = torch.arange(kh.FC, dtype=torch.int32, device=dev)
    n = 0
    for h in (3, 1, F + 2, 2, 5):
        X0 = ((n + torch.arange(h, dtype=torch.int32, device=dev))[:, None] * 8192 + e)[None]
        lead_t = i32([0], dev)
        assert kh.history_put(X0.view(torch.float32), st.t, kh.records_map(st.ss, lead_t, batch, None, h), hist.t, F, 1) == 0
        n += h
        pos = st.pos(0)
        pos += h
        st.calls(0).add_(1)
    torch.cuda.synchronize()
    assert hist.ok() and int(st.pos(0)) == p0 + n
    for w_max in (F, 3):
        J = 3
        lists = Guarded((3 * J,), dev)
        leads = i32([0] * J, dev)
        assert kh.join_start(st.t, st.ss, batch, i32([1, 2, 3], dev), leads, w_max, J, lists.t, None) == 0
        li = bits(lists.t)
        X = Guarded((J, w_max, kh.FC), dev)
        assert kh.history_get(hist.t, F, st.t, kh.records_map(st.ss, li[:J], batch, li[J:2 * J], w_max), leads, X.t, J) == 0
        torch.cuda.synchronize()
        assert X.ok() and li[J:2 * J].tolist() == [w_max] * J
        exp = ((n - w_max + torch.arange(w_max, dtype=torch.int32, device=dev))[:, None] * 8192 + e)
        for j in range(J):
            assert int(st.pos(1 + j)) == p0 + n - w_max
            assert torch.equal(bits(X.t[j]), exp), (F, w_max, j)
    print(f"[history end to end F={F}] {n} frames from clock {p0}: replays exact")


# ---- move_lead -------------------------------------------------------------------------------------------------------
def test_move_lead_parities(layout, dev):
    lay, nb = layout
    batch = 8
    calls = [4, 6, 5, 7, 0, 1, 2, 3]             # pairs i -> i + 4: parities (0, 0), (0, 1), (1, 0), (1, 1)
    st, a = clocked_state(lay, batch, [2 ** 32 + 5] * batch, dev, seed=101, calls=calls)
    src, dst = [0, 1, 2, 3], [4, 5, 6, 7]
    assert launches(lambda: kh.move_lead(st.t, st.ss, batch, src, dst)) == 1
    torch.cuda.synchronize()
    got = host(st.t)
    assert st.buf.ok() and np.array_equal(got, kh.move_lead_ref(a, st.hdr, st.ss, lay, nb, src, dst))
    muts = {"src_parity"} | ({"all_blocks"} if nb > 1 else set())
    for m in muts:
        assert not np.array_equal(got, kh.move_lead_ref(a, st.hdr, st.ss, lay, nb, src, dst, mutant=m)), m
    caught("move_lead", muts)


def test_move_lead_two_chunks(limits, dev):
    """MOVE_MAX_PAIRS + 1 pairs (two launches) over 962 one-block records: each destination's block 0 and current conv
    tails are its source's, everything else of it keeps the sentinel, and the source keeps its bits"""
    lay = kh.sep_layout(1)
    n = limits["MOVE_MAX_PAIRS"] + 1
    batch = 2 * n
    st = Records(lay, batch, dev, GAP)
    blk, conv, cp = lay["ST_BLK"], lay["ST_CONV"], kh.CONV_PARITY
    span = lay["BK_STRIDE"]
    for i in range(n):                            # sources 0 .. n-1: random block 0 and tails; destinations n .. 2n-1
        r = bits(st.rec(i))
        r[blk:blk + span].copy_(random_bits(span, 1000 + i, dev))
        r[conv:conv + 2 * cp].copy_(random_bits(2 * cp, 5000 + i, dev))
        r[lay["ST_CALLS"]] = i % 2
        bits(st.rec(n + i))[lay["ST_CALLS"]] = (i // 2) % 2
    src, dst = list(range(n)), [n + (i * 7) % n for i in range(n)]
    assert launches(lambda: kh.move_lead(st.t, st.ss, batch, src, dst)) == 2
    torch.cuda.synchronize()
    assert st.buf.ok()
    sent = torch.tensor(SENTINEL, dtype=torch.int32, device=dev)
    for i, d in zip(src, dst):
        s, r = bits(st.rec(i)), bits(st.rec(d))
        pa, pb = i % 2, int(r[lay["ST_CALLS"]]) & 1
        assert torch.equal(r[blk:blk + span], s[blk:blk + span]), (i, d)
        assert torch.equal(r[conv + pb * cp:conv + (pb + 1) * cp], s[conv + pa * cp:conv + (pa + 1) * cp]), (i, d)
        keep = torch.ones(st.ss, dtype=torch.bool, device=dev)
        keep[blk:blk + span] = False
        keep[conv + pb * cp:conv + (pb + 1) * cp] = False
        keep[lay["ST_CALLS"]] = False
        assert bool((r[keep] == sent).all()), (i, d, "destination written outside block 0 and its current tails")
        assert torch.equal(s[blk:blk + span], random_bits(span, 1000 + i, dev)), (i, "source written")
    del st
    torch.cuda.empty_cache()
    print(f"[move_lead {n} pairs] two launches, exact")


def test_move_lead_refuses_bad_pairs(dev):
    lay = kh.sep_layout(1)
    st = Records(lay, 2, dev, GAP)
    n0 = kh.lib().kh_launch_count()
    assert kh.move_lead(st.t, st.ss, 2, [0], [2]) != 0 and kh.move_lead(st.t, st.ss, 2, [-1], [1]) != 0
    assert kh.move_lead(st.t, lay["ST_BLK"], 2, [0], [1]) != 0
    assert kh.lib().kh_launch_count() == n0 and is_sentinel(st.buf.whole)


# ---- the product library's launch counter ----------------------------------------------------------------------------
def test_engine_launch_counts(limits, dev):
    """l2h_sep_launch_count moves by one per launch of init, reset and move_lead: ceil(n / RESET_MAX_SLOTS) for a reset
    of n slots and ceil(n / MOVE_MAX_PAIRS) for a move of n pairs (a one-block engine, 962 records)"""
    from lookoncetohear_b200 import Net, _cabi
    from lookoncetohear_b200.configs import TSH_PARAMS
    net = Net(**dict(TSH_PARAMS, B=1))
    L, h = _cabi.lib(), net._engine()
    rl, ml = limits["RESET_MAX_SLOTS"], limits["MOVE_MAX_PAIRS"]
    batch = 2 * (ml + 1)
    ss = kh.sep_layout(1)["STREAM_STRIDE"]
    state = torch.empty(16 + batch * ss, dtype=torch.float32, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    arr = lambda v: (ctypes.c_int32 * len(v))(*v)
    count = ctypes.c_int64()

    def moved(call):
        _cabi.check(L.l2h_sep_launch_count(h, None, 1))
        _cabi.check(call())
        _cabi.check(L.l2h_sep_launch_count(h, ctypes.byref(count), 1))
        return count.value

    assert moved(lambda: L.l2h_sep_state_init(h, state.data_ptr(), batch, s)) == 1
    for n in (1, rl, rl + 1):
        assert moved(lambda: L.l2h_sep_state_reset_streams(h, state.data_ptr(), batch, arr(list(range(n))), n, s)) == \
            math.ceil(n / rl), n
    for n in (1, ml + 1):
        assert moved(lambda: L.l2h_sep_state_move_lead(h, state.data_ptr(), batch, arr(list(range(n))),
                                                       arr(list(range(n, 2 * n))), n, s)) == math.ceil(n / ml), n
    torch.cuda.synchronize()
    del state
    torch.cuda.empty_cache()


def test_summary(dev):
    import subprocess
    index = torch.cuda.current_device()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(index)],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    print(f"\ndevice: {torch.cuda.get_device_name(index)}, power limit {pl}; peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    for k in sorted(CAUGHT):
        print(f"{k}: exact; mutants caught {sorted(CAUGHT[k])}")
    named = {"state_init": kh.STATE_INIT_MUTANTS, "reset_streams": kh.RESET_MUTANTS, "advance_header": kh.ADVANCE_MUTANTS,
             "join_start": kh.JOIN_MUTANTS, "history_put": kh.HIST_PUT_MUTANTS, "history_get": kh.HIST_GET_MUTANTS,
             "move_lead": kh.MOVE_MUTANTS}
    for k, ms in named.items():
        assert CAUGHT.get(k, set()) == set(ms), (k, CAUGHT.get(k))
