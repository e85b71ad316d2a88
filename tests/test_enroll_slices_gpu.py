"""Enrollment in slices on the GPU (l2h_embed_forward_slots_units / EmbedTFGridNet.enroll_job): the embeddings and `used`
of every job equal those of EmbedTFGridNet.enroll with the same arguments, bit for bit, for windows 0, 1, 7, 64 and one
longer than the recurrence, for steps of one unit, seeded random partitions and run() at once, with host and device slot
lists, at equal and mixed lengths, in every recurrence kernel the padded batch picks (lstm_rec's preloaded, ring and 2- and
4-sequence forms, and tc_lstm).  Serving: FIFO -> capture -> advance_slots ticks between the units, two jobs interleaved
with each other and with enroll and forward calls, a job over several max_batch cuts; and one row against the oracle."""
import pytest
import torch

from lookoncetohear_b200 import EmbedTFGridNet, EnrollCapture, HopFifo, synth
from oracle import restate as rs
from serving_util import bits, dev, i32, model  # noqa: F401

pytestmark = pytest.mark.gpu

HEAD, HOP, CARRY = 2, 128, 64
NAN = float("nan")
WINDOWS = (0, 1, 7, 64, 100000)
S, CAPACITY = 24, 16000
SHORT, OUTSIDE = 23, 24                         # a slot that captured under 192 samples; a device entry outside


@pytest.fixture(scope="module")
def embed(embed_params, dev):
    torch.manual_seed(0)
    net = EmbedTFGridNet(**embed_params).eval()
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    return net.to(dev), sd


def _fill(cap, sig, totals, fed, T=8):
    """push slot s's signal up to totals[s] samples (multiples of 128), T hops per call of every slot at once"""
    n = cap.n_slots
    while any(f < t for f, t in zip(fed, totals)):
        hops = [min(T, (t - f) // HOP) for f, t in zip(fed, totals)]
        chunk = torch.full((n, 2, HOP * T + CARRY), NAN, device=sig.device)
        for s, h in enumerate(hops):
            chunk[s, :, CARRY:CARRY + HOP * h] = sig[s, :, fed[s]:fed[s] + HOP * h]
            fed[s] += HOP * h
        cap(chunk, list(range(n)), hops)


@pytest.fixture(scope="module")
def capture(dev):
    """24 slots of a 1 s capture, each fed 1-2.5 s (wrapped), slot 23 only 128 samples"""
    g = torch.Generator().manual_seed(1200)
    totals = [HOP * int(k) for k in torch.randint(CAPACITY // HOP, 5 * CAPACITY // (2 * HOP), (S,), generator=g)]
    totals[SHORT] = 128
    sig = synth.enrollment(S, max(totals), seed0=1300).to(dev)
    cap = EnrollCapture(S, 2, CAPACITY, device=dev)
    _fill(cap, sig, totals, [0] * S)
    return cap


def ring_last(cap, s, L):
    w = int(cap.state[s, 0, 0].view(torch.int32))
    idx = (w - L + torch.arange(L, device=cap.state.device)) % cap.capacity
    return cap.state[s][:, HEAD + idx]


# lengths per case, chosen so that the inter recurrence of the padded batch (65 sequences per utterance, two directions)
# takes each kernel form in turn: lstm_rec3 with the gate input preloaded (one short utterance) or streamed (two long
# ones), lstm_rec4 with more sequences per CTA (3 and 5 utterances), and tc_lstm (17 utterances: >= 2048 seq-dirs)
CASES = {
    "b1_short": [3000],
    "b2_long": [16000, 9000],
    "b3_mixed": [700, 12000, 5000],
    "b5_equal": [8000] * 5,
    "b17_tc": [192, 2000, 1500] + [1000 + 50 * i for i in range(14)],
}


def _slots(case, n, on_dev, dev):
    g = torch.Generator().manual_seed(len(case) * 31 + n)
    pick = torch.randperm(SHORT, generator=g)[:n].tolist()
    if n >= 3:
        pick[1] = SHORT                                        # captured too little: its row is left as it was
        if on_dev:
            pick[2] = OUTSIDE                                  # outside the capture: embeds nothing
    return i32(pick, dev) if on_dev else pick


def _partition(total, kind, seed):
    if kind == "ones":
        return [1] * total
    if kind == "run":
        return []
    g = torch.Generator().manual_seed(seed)
    parts, left = [], total
    while left:
        k = min(left, int(torch.randint(1, 12, (1,), generator=g)))
        parts.append(k)
        left -= k
    return parts


def _reference(net, cap, slots, lens, n, dev):
    staging = torch.randn(2 * n + 1, 256, generator=torch.Generator().manual_seed(n)).to(dev)
    used = torch.full((n,), -3, dtype=torch.int32, device=dev)
    with torch.no_grad():
        net.enroll(cap, slots, lens, out=staging[1::2], used=used)
    return staging, used


@pytest.mark.parametrize("case", list(CASES))
def test_job_equals_enroll(embed, capture, dev, case):
    net, _ = embed
    lens = CASES[case]
    n = len(lens)
    for wi, window in enumerate(WINDOWS):
        for kind, on_dev in (("ones", False), ("random", True), ("run", wi % 2 == 0)):
            slots = _slots(case, n, on_dev, dev)
            want, want_used = _reference(net, capture, slots, lens, n, dev)
            staging = torch.randn(2 * n + 1, 256, generator=torch.Generator().manual_seed(n)).to(dev)
            used = torch.full((n,), -3, dtype=torch.int32, device=dev)
            job = net.enroll_job(capture, slots, lens, out=staging[1::2], used=used, window=window)
            assert job.out is not None and job.units >= 11 and not job.done
            for k in _partition(job.units, kind, 100 * wi + n):
                assert job.step(k) == k
            assert job.run() is job.out and job.done
            assert job.step(3) == 0
            assert torch.equal(used, want_used), (case, window, kind)
            assert torch.equal(bits(staging), bits(want)), (case, window, kind)
            if n >= 3:
                assert want_used[1].item() == 0
                if on_dev:
                    assert want_used[2].item() == 0


def test_rows_and_used_between_units(embed, capture, dev):
    """`used` is final after unit 0; the rows keep their old values until the last unit"""
    net, _ = embed
    lens = [9000, 300, 16000]
    slots = [4, SHORT, 7]
    out = torch.full((3, 256), 7.0, device=dev)
    used = torch.zeros(3, dtype=torch.int32, device=dev)
    job = net.enroll_job(capture, slots, lens, out=out, used=used, window=64)
    job.step()
    torch.cuda.synchronize()
    assert used.tolist() == [9000, 0, 16000]
    job.step(job.units - 2)
    torch.cuda.synchronize()
    assert (out == 7.0).all()
    job.step()
    assert (out[1] == 7.0).all() and not (out[0] == 7.0).any() and not (out[2] == 7.0).any()


def test_tc_lstm_option_small_batch(embed_params, capture, dev):
    """tc_lstm_min = 1: a 2-utterance batch whose recurrences all run on the tensor cores"""
    torch.manual_seed(0)
    net = EmbedTFGridNet(**embed_params).eval().to(dev)
    net.set_option("tc_lstm_min", 1)
    lens, slots = [11000, 4000], [3, 9]
    want, want_used = _reference(net, capture, slots, lens, 2, dev)
    for window in (7, 64):
        staging = torch.randn(5, 256, generator=torch.Generator().manual_seed(2)).to(dev)
        used = torch.zeros(2, dtype=torch.int32, device=dev)
        job = net.enroll_job(capture, slots, lens, out=staging[1::2], used=used, window=window)
        for k in _partition(job.units, "random", window):
            job.step(k)
        assert torch.equal(used, want_used) and torch.equal(bits(staging), bits(want)), window


def test_ticks_between_units(model, embed, dev):
    """Four listeners stream through FIFO -> capture -> advance_slots.  A job enrolling three of them steps a few units
    after every tick, so the ticks keep writing the rings under it.  It returns the embedding of the windows the capture
    held when its first unit ran, and the ticks' outputs and the capture equal a run without the job, bit for bit."""
    sep, _ = model
    enet, _ = embed
    S4, slots, T, cap_len = 6, [2, 0, 3, 5], 2, 12000
    n = len(slots)
    ticks = cap_len // (HOP * T) + 45
    x, _ = synth.mixture(n, HOP * T * ticks, seed0=9300)
    x = x.to(dev)
    E = synth.embedding(n, seed0=9400)[:, 0].to(dev)
    sl, cnt = i32(slots, dev), i32([HOP * T] * n, dev)

    def objs():
        return HopFifo(S4, 2, T, 4096, device=dev), EnrollCapture(S4, 2, cap_len, device=dev), sep.init_buffers(S4, dev)

    def tick(o, t):
        fifo, cap, st = o
        chunk, hops = fifo(x[:, :, HOP * T * t:HOP * T * (t + 1)], cnt, sl)
        cap(chunk, sl, hops)
        return sep.advance_slots(chunk, E, st, sl, hops=hops)

    live, twin = objs(), objs()
    start = cap_len // (HOP * T) + 2
    ys_live, ys_twin = [], []
    with torch.no_grad():
        for t in range(start):
            tick(live, t)
            tick(twin, t)
        snap = EnrollCapture(S4, 2, cap_len, device=dev)
        snap.state.copy_(live[1].state)
        who, lens = [0, 5, 3], [cap_len, 5000, 700]
        want, want_used = _reference(enet, snap, who, lens, 3, dev)
        staging = torch.randn(7, 256, generator=torch.Generator().manual_seed(3)).to(dev)
        used = torch.full((3,), -3, dtype=torch.int32, device=dev)
        job = enet.enroll_job(live[1], who, lens, out=staging[1::2], used=used, window=1)
        t = start
        while not job.done:
            job.step(20)
            ys_live.append(tick(live, t).clone())
            ys_twin.append(tick(twin, t).clone())
            t += 1
    assert t - start > 20                                        # 20+ ticks wrote 5000+ samples to every ring under the job
    assert not torch.equal(live[1].state, snap.state)
    assert torch.equal(used, want_used)
    assert torch.equal(bits(staging), bits(want))
    assert torch.equal(bits(live[1].state), bits(twin[1].state))
    assert torch.equal(bits(torch.cat(ys_live, -1)), bits(torch.cat(ys_twin, -1)))


def test_jobs_interleave(embed, capture, dev):
    """two jobs stepped in turn, with enroll and forward calls (which use the net's shared workspace) between steps"""
    net, _ = embed
    a_args = ([1, 2, 3, 4], [16000, 3000, 9000, 9000])
    b_args = (i32([5, 6, OUTSIDE], dev), [5000, 5000, 5000])
    wa, wa_used = _reference(net, capture, *a_args, 4, dev)
    wb, wb_used = _reference(net, capture, *b_args, 3, dev)
    sa = torch.randn(9, 256, generator=torch.Generator().manual_seed(4)).to(dev)
    sb = torch.randn(7, 256, generator=torch.Generator().manual_seed(3)).to(dev)
    ua, ub = torch.zeros(4, dtype=torch.int32, device=dev), torch.zeros(3, dtype=torch.int32, device=dev)
    ja = net.enroll_job(capture, *a_args, out=sa[1::2], used=ua, window=7)
    jb = net.enroll_job(capture, *b_args, out=sb[1::2], used=ub, window=64)
    x = synth.enrollment(2, 6000, seed0=77).to(dev)
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        fwd_want = net(x)
        k = 0
        while not (ja.done and jb.done):
            (ja if k % 2 == 0 else jb).step(int(torch.randint(1, 6, (1,), generator=g)))
            if k % 7 == 3:
                net.enroll(capture, [10, 11], [4000, 15000])
            if k % 11 == 5:
                assert torch.equal(bits(net(x)), bits(fwd_want))
            k += 1
    assert torch.equal(ua, wa_used) and torch.equal(bits(sa), bits(wa))
    assert torch.equal(ub, wb_used) and torch.equal(bits(sb), bits(wb))


def test_job_over_max_batch_cuts(embed, capture, dev):
    """max_batch of 2: five rows in three cuts, their units run one cut after another, stepped across the cuts' edges"""
    net, _ = embed
    lens = [16000, 2000, 9000, 700, 12000]
    slots = [8, SHORT, 12, 13, 14]
    net.max_batch = lambda n_samples: 2
    try:
        want, want_used = _reference(net, capture, slots, lens, 5, dev)
        for window in (0, 64):
            staging = torch.randn(11, 256, generator=torch.Generator().manual_seed(5)).to(dev)
            used = torch.zeros(5, dtype=torch.int32, device=dev)
            job = net.enroll_job(capture, slots, lens, out=staging[1::2], used=used, window=window)
            assert len(job._cuts) == 3 and job.units == sum(c[2] for c in job._cuts)
            per_cut = job._cuts[0][2]
            job.step(per_cut - 1)
            job.step(2)                                          # the last unit of cut 0 and the first of cut 1
            for k in _partition(job.units - job._next, "random", window):
                job.step(k)
            assert job.done
            assert torch.equal(used, want_used) and torch.equal(bits(staging), bits(want)), window
    finally:
        del net.max_batch


def test_one_row_against_oracle(embed, capture, dev):
    net, sd = embed
    lens, slots = [6000, 16000], [15, 16]
    job = net.enroll_job(capture, slots, lens, window=64)
    with torch.no_grad():
        out = job.run().cpu()
    x = ring_last(capture, 15, 6000)[None].cpu()
    r0 = rs.embed_forward(sd, x)
    assert rs.rel_l2(out[0:1], r0) <= 1e-3, rs.rel_l2(out[0:1], r0)
