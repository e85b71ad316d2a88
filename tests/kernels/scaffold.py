"""What the kernel-level GPU tests share: the NaN sentinel and guarded buffers, error / bound ratios and the ledger that
checks and summarises them, the `dev` and `lay` fixtures, and views of the records of a separator state.

A test module imports the fixtures it uses by name (`from kernels.scaffold import dev, lay`), so that pytest finds them.
"""
import math
import subprocess

import pytest
import torch

from kernels import harness as kh

SENTINEL = 0x7FC0DEAD          # a quiet NaN with a payload no kernel produces
SENSITIVITY = 10.0             # every mutant must miss its bound by at least this factor
GUARD = 4096                   # sentinel floats on each side of a guarded buffer: a multiple of 128, so that the buffer
                               # keeps the 512-byte alignment of a fresh allocation, which the kernels' TMA descriptors need


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    kh.lib()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def lay(request, dev):
    """the separator state layout of the requesting module's N_BLOCKS blocks"""
    return kh.sep_layout(request.module.N_BLOCKS)


def sentinel(n, dev):
    return torch.full((n,), SENTINEL, dtype=torch.int32, device=dev).view(torch.float32)


def bits(t):
    return t.contiguous().view(torch.int32)


def is_sentinel(t):
    return bool((bits(t) == SENTINEL).all())


class Guarded:
    """`t`: a buffer of `shape` floats (init: its values, else the sentinel) between GUARD sentinel floats on each side"""

    def __init__(self, shape, dev, init=None):
        n = math.prod(shape)
        self.whole = sentinel(n + 2 * GUARD, dev)
        self.t = self.whole[GUARD:GUARD + n].view(shape)
        if init is not None:
            self.t.copy_(torch.as_tensor(init).reshape(shape))

    def ok(self):
        """both guards still hold the sentinel, bit for bit"""
        return is_sentinel(self.whole[:GUARD]) and is_sentinel(self.whole[-GUARD:])


def ratio(got, ref, bound):
    """max |got - ref| / bound: 0 where got equals ref exactly (so 0 / 0 is 0), inf where a bound of 0 is missed, and 0
    over no elements; tensors or numpy arrays"""
    got, ref = (torch.as_tensor(v).double().cpu() for v in (got, ref))
    d = (got - ref).abs()
    r = d / torch.as_tensor(bound, dtype=torch.float64)
    r[d == 0] = 0
    return float(r.max()) if r.numel() else 0.0


class Ledger:
    """The worst error / bound and the smallest mutant error / bound per key, over the checks of one test module."""

    def __init__(self):
        self.worst, self.margin = {}, {}

    def check(self, key, errs, mutants):
        """errs: one error / bound, or {output: error / bound}; mutants: {mutant: error / bound}.  Every error must be
        within its bound, and every mutant at least SENSITIVITY bounds away."""
        named = errs if isinstance(errs, dict) else {None: errs}
        self.worst[key] = max(self.worst.get(key, 0.0), *named.values())
        if mutants:
            self.margin[key] = min(self.margin.get(key, math.inf), *mutants.values())
        print(f"[{key}] err / bound " + ", ".join(f"{v:.3f}" if k is None else f"{k} {v:.3f}" for k, v in named.items())
              + "; mutants / bound: " + ", ".join(f"{m} {v:.1f}" for m, v in mutants.items()))
        for k, v in named.items():
            assert v <= 1.0, (key, k, v)
        for m, v in mutants.items():
            assert v >= SENSITIVITY, (key, m, v)

    def summary(self):
        """prints the device, its power limit and every key's worst error and smallest mutant margin; asserts them again"""
        index = torch.cuda.current_device()
        try:
            pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(index)],
                                capture_output=True, text=True, timeout=30).stdout.strip()
        except (OSError, subprocess.SubprocessError):
            pl = "unknown"
        print(f"\ndevice: {torch.cuda.get_device_name(index)}, power limit {pl}")
        for k, v in sorted(self.worst.items()):
            print(f"worst {k}: {v:.3f} x bound; smallest mutant margin {self.margin.get(k, math.nan):.1f}")
        assert all(v <= 1.0 for v in self.worst.values()) and all(v >= SENSITIVITY for v in self.margin.values())


class Records:
    """A separator state in a guarded buffer: the header, then `batch` records STREAM_STRIDE + gap floats apart, every
    float the sentinel.  Each view is of the live state t, or of `t` when given (a snapshot)."""

    def __init__(self, lay, batch, dev, gap=0):
        self.lay, self.batch = lay, batch
        self.hdr, self.ss = lay["HEADER_BYTES"] // 4, lay["STREAM_STRIDE"] + gap
        self.buf = Guarded((self.hdr + batch * self.ss,), dev)
        self.t = self.buf.t

    def rec(self, b, t=None):
        t = self.t if t is None else t
        return t[self.hdr + b * self.ss:self.hdr + (b + 1) * self.ss]

    def field(self, b, name, shape, t=None):
        """record b's floats at layout offset `name` (or at a float offset) as a [shape] view"""
        o = self.lay[name] if isinstance(name, str) else name
        return self.rec(b, t)[o:o + math.prod(shape)].view(shape)

    def pos(self, b, t=None):
        """the record's clock (ST_POS, frames consumed), int64 [1]"""
        return self.field(b, "ST_POS", (2,), t).view(torch.int64)

    def calls(self, b, t=None):
        return self.field(b, "ST_CALLS", (1,), t).view(torch.int32)

    def gen(self, b, t=None):
        """the weight generation the record's gate was built with, int32 [1]"""
        return self.field(b, "ST_GEN", (1,), t).view(torch.int32)

    def gate(self, b, t=None):
        return self.field(b, "ST_GATE", (kh.NF, kh.CH), t)

    def emb(self, b, t=None):
        return self.field(b, "ST_EMB", (kh.SPK,), t)

    def conv(self, b, t=None):
        return self.field(b, "ST_CONV", (2, 2, 4, kh.NF), t)

    def deconv(self, b, t=None):
        return self.field(b, "ST_DECONV", (2, 2, kh.NF, kh.CH), t)

    def istft(self, b, t=None):
        return self.field(b, "ST_ISTFT", (2, 2, kh.NROW), t)

    def hc(self, b, blk, which, t=None):
        """block blk's carried h or c (which = 'h' or 'c'), [97][64]"""
        o = self.lay["ST_BLK"] + blk * self.lay["BK_STRIDE"] + self.lay["BK_H" if which == "h" else "BK_C"]
        return self.field(b, o, (kh.NF, kh.CH), t)

    def ring(self, b, blk, which, t=None):
        """block blk's K ring (which = 'k': [4][56][584]) or V ring ('v': [4][56][1552]); frame n's row of head h is
        [h, kh.Ring.slot(n)]"""
        n = kh.QK_LD if which == "k" else kh.V_DIM
        return self.field(b, kh.Ring(self.lay).row(blk, which, 0, 0), (kh.NHEAD, kh.RING, n), t)

    def snapshot(self):
        return self.t.clone()

    def index(self, *views):
        """the flat indices into t of the floats of views of t (float32 views: other dtypes count other units)"""
        out = [torch.zeros(0, dtype=torch.int64)]
        for v in views:
            i = torch.tensor(v.storage_offset() - self.t.storage_offset())
            for n, s in zip(v.shape, v.stride()):
                i = i[..., None] + s * torch.arange(n)
            out.append(i.reshape(-1))
        return torch.cat(out)

    def same_outside(self, indices, before):
        """the state equals `before` bit for bit outside the flat indices `indices`, and both its guards hold"""
        exp = before.clone()
        indices = indices.to(self.t.device)
        exp[indices] = self.t[indices]
        return self.buf.ok() and torch.equal(bits(self.t), bits(exp))
