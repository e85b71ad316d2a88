"""The kernels of an enrollment from a capture (csrc/embed_kernels.cuh): eslot_rows_kernel, eput_rows_kernel, and
estd_kernel / efront_kernel over the capture ring's sample map (XRing), launched directly through the engine's launchers.

Cases.  eslot_rows (kernels/harness.py::eslot_rows_case): host and device slot lists of 1, SLOT_ROWS_PER_LAUNCH and
SLOT_ROWS_PER_LAUNCH + 1 rows (one and two launches) over a capture of 500 slots of capacity 1000; raw captured counts
negative, 0, 191, 192, above capacity and +-(2^31 - 1); lengths below MIN_SAMPLES, above capacity, 0 and negative; on
device lists also slots -1, n_slots and 2^31 - 1.  eput_rows: row strides 256 and 300, live and dead rows.  The ring map
(ring_cases): write positions 0, n - 1, n, capacity - 1 and one past the ring, n == capacity, capacity == MIN_SAMPLES,
and rows that are not live.

Oracle.  slots_out, lens and used equal eslot_rows_ref exactly, and the guard floats around them keep the sentinel
0x7FC0DEAD; eput_rows leaves dead rows and the gaps between rows at the sentinel.  The ring map is checked against the
dense map the kernels also run (XDense) on the same utterances unwrapped into a padded [B][2][N] copy: for every live row,
inv_std and every frame of X must be bit-identical (the kernel code is the same; only the sample map differs).  The
GroupNorm sums are double atomics, one per CTA, whose order varies between launches: they must agree within the
reordering bound 2 T u64 sum_t |partial_t|.  A row that is not live must give inv_std = 0 and a finite X.

Mutants (each must differ on every case that names it): eslot_rows keeping rows below MIN_SAMPLES live and not clamping
the captured count; eput_rows writing dead rows; the ring map with the start not wrapped (the dense map's inv_std over
that unwrapping must differ from the ring's on every call with a wrapping row).

Measured on one NVIDIA H100 80GB HBM3 (700 W power limit): every list, row and ring-map output exact, the GroupNorm sums
within their reordering bound, and every mutant caught.  Run with test_state_kernels_gpu.py, the two modules took 8 s.
"""
import pytest
import torch

from kernels import harness as kh
from kernels.scaffold import SENTINEL, Guarded, bits, dev, is_sentinel  # noqa: F401

pytestmark = pytest.mark.gpu

CAUGHT = {}


def caught(key, mutants):
    CAUGHT.setdefault(key, set()).update(mutants)
    print(f"[{key}] exact; mutants caught: {sorted(mutants)}")


@pytest.fixture(scope="module")
def limits(dev):
    return kh.state_limits()


def i32(v, dev):
    return torch.tensor(v, dtype=torch.int32, device=dev)


def capture_buf(n_slots, capacity, heads, dev, seed):
    """a capture [n_slots][2][EC_HEAD + capacity] of seeded samples; heads[s] = (wpos, captured) of slot s, written to
    both channels' head words"""
    g = torch.Generator().manual_seed(seed)
    cap = torch.randn(n_slots, 2, 2 + capacity, generator=g)
    hw = torch.tensor(heads, dtype=torch.int64)
    cap_bits = cap.view(torch.int32)
    cap_bits[:, :, 0] = hw[:, 0, None].to(torch.int32)
    cap_bits[:, :, 1] = hw[:, 1, None].to(torch.int32)
    return Guarded((n_slots, 2, 2 + capacity), dev, cap)


# ---- eslot_rows ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("device", [False, True], ids=["host_list", "device_list"])
@pytest.mark.parametrize("which", ["one", "max", "max_plus_1"])
def test_eslot_rows(which, device, limits, dev):
    lim = limits["SLOT_ROWS_PER_LAUNCH"]
    n = {"one": 1, "max": lim, "max_plus_1": lim + 1}[which]
    c = kh.eslot_rows_case(n, device, lim)
    capture = capture_buf(c["n_slots"], c["capacity"], [(s % 7, v) for s, v in enumerate(c["captured"])], dev, 3)
    outs = [Guarded((n,), dev) for _ in range(3)]
    n0 = kh.lib().kh_launch_count()
    rc = kh.eslot_rows(None if device else c["slots"], i32(c["slots"], dev) if device else None, c["lens"], n, capture.t,
                       c["n_slots"], c["capacity"], *(o.t for o in outs))
    assert rc == 0 and kh.lib().kh_launch_count() - n0 == -(-n // lim)
    torch.cuda.synchronize()
    assert all(o.ok() for o in outs) and capture.ok()
    got = dict(zip(("slots", "lens", "used"), (bits(o.t).cpu().tolist() for o in outs)))
    args = (c["slots"], c["lens"], c["captured"], c["n_slots"], c["capacity"], limits["MIN_SAMPLES"])
    assert got == kh.eslot_rows_ref(*args)
    for m in c["catches"]:
        assert got != kh.eslot_rows_ref(*args, mutant=m), m
    caught("eslot_rows", c["catches"])


def test_eslot_rows_refuses_bad_host_slots(dev):
    capture = capture_buf(4, 200, [(0, 0)] * 4, dev, 4)
    outs = [Guarded((1,), dev) for _ in range(3)]
    n0 = kh.lib().kh_launch_count()
    for s in (-1, 4, kh.INT_MAX):
        assert kh.eslot_rows([s], None, [192], 1, capture.t, 4, 200, *(o.t for o in outs)) != 0, s
    assert kh.lib().kh_launch_count() == n0 and all(is_sentinel(o.whole) for o in outs)


# ---- eput_rows -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row_stride", [256, 300])
def test_eput_rows(row_stride, dev):
    used = [200, 0, 192, -1, 0, 5000, 1]
    B = len(used)
    g = torch.Generator().manual_seed(row_stride)
    src = torch.randn(B, 256, generator=g)
    dst = Guarded((B * row_stride,), dev)
    assert kh.eput_rows(src.to(dev), dst.t, row_stride, i32(used, dev), B) == 0
    torch.cuda.synchronize()
    assert dst.ok()
    got = bits(dst.t).cpu().numpy()
    import numpy as np
    d0 = np.full(B * row_stride, SENTINEL, dtype=np.int32)
    s = bits(src).numpy()
    assert np.array_equal(got, kh.eput_rows_ref(d0, s, used, row_stride))
    assert not np.array_equal(got, kh.eput_rows_ref(d0, s, used, row_stride, mutant="dead_written"))
    caught("eput_rows", {"dead_written"})


# ---- estd / efront over the capture ring -----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def w(dev):
    from test_embed_kernels_gpu import Weights
    return Weights(dev)


def dense_copy(rings, c, N, mutant=None):
    """x [B][2][N]: row b the utterance of its slot's ring, zero padded"""
    x = torch.zeros(len(c["rows"]), 2, N)
    for b, (wpos, n, _) in enumerate(c["rows"]):
        x[b, :, :n] = torch.from_numpy(kh.ring_utterance(rings[b].numpy(), wpos, n, c["capacity"], mutant))
    return x


@pytest.mark.parametrize("case", kh.ring_cases(192), ids=lambda c: c["name"])
def test_ring_map(case, limits, w, dev):
    c, ms = case, limits["MIN_SAMPLES"]
    assert ms == 192
    rows, cap = c["rows"], c["capacity"]
    B = len(rows)
    N = max(n for _, n, _ in rows)
    T = kh.e_frames(N)
    heads = [(wpos, cap) for wpos, _, _ in rows]              # one slot per row, a full ring
    capture = capture_buf(B, cap, heads, dev, 7)
    rings = capture.t[:, :, 2:].cpu()
    slots, lens = i32(list(range(B))[::-1], dev), [n for _, n, _ in rows]
    # the ring rows are listed in reverse, so row b reads slot B - 1 - b
    order = list(range(B))[::-1]
    rows_r = [rows[s] for s in order]
    used = i32([n if live else 0 for _, n, live in rows_r], dev)
    lens_r = i32([lens[s] for s in order], dev)
    cr = dict(c, rows=rows_r)
    x = dense_copy([rings[s] for s in order], cr, N)
    xd = x.to(dev)
    out = {}
    for form in ("ring", "dense"):
        inv = Guarded((B,), dev)
        X = Guarded((B, T, kh.E_NF, kh.E_CH), dev)
        gn = torch.zeros(2 * B, dtype=torch.float64, device=dev)
        if form == "ring":
            assert kh.estd_ring(capture.t, cap, slots, used, N, lens_r, inv.t, B) == 0
            assert kh.efront_ring(w.c, capture.t, cap, slots, used, N, lens_r, inv.t, X.t, gn, B, T) == 0
        else:
            assert kh.estd(xd, N, lens_r, inv.t, B) == 0
            assert kh.efront(w.c, xd, N, lens_r, inv.t, X.t, gn, B, T) == 0
        torch.cuda.synchronize()
        assert inv.ok() and X.ok() and capture.ok()
        out[form] = (inv.t.clone(), X.t.clone(), gn.clone())
    (ir, Xr, gr), (id_, Xd, gd) = out["ring"], out["dense"]
    for b, (wpos, n, live) in enumerate(rows_r):
        if not live:
            assert float(ir[b]) == 0.0 and bool(torch.isfinite(Xr[b]).all()), b
            continue
        assert torch.equal(bits(ir[b]), bits(id_[b])), (c["name"], b, "inv_std")
        assert torch.equal(bits(Xr[b]), bits(Xd[b])), (c["name"], b, "X")
        part = Xd[b].double().sum(dim=(1, 2)).abs().sum(), Xd[b].double().square().sum()
        for k in range(2):
            bound = 2 * T * 2.0 ** -53 * float(part[k]) + 1e-300
            assert abs(float(gr[2 * b + k]) - float(gd[2 * b + k])) <= bound, (c["name"], b, k)
    # the unwrapped mutant: the dense map over that copy gives another inv_std on a wrapping row
    xm = dense_copy([rings[s] for s in order], cr, N, mutant="no_wrap").to(dev)
    im = Guarded((B,), dev)
    assert kh.estd(xm, N, lens_r, im.t, B) == 0
    torch.cuda.synchronize()
    wraps = [b for b, (wpos, n, live) in enumerate(rows_r) if live and min(max(wpos, 0), cap - 1) < n]
    assert wraps and any(not torch.equal(bits(ir[b]), bits(im.t[b])) for b in wraps)
    caught("ring_map", {"no_wrap"})


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
    named = {"eslot_rows": kh.SLOT_ROWS_MUTANTS, "eput_rows": kh.PUT_ROWS_MUTANTS, "ring_map": kh.RING_MUTANTS}
    for k, ms in named.items():
        assert CAUGHT.get(k, set()) == set(ms), (k, CAUGHT.get(k))
