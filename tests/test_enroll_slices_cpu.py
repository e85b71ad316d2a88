"""Host-side checks of enrollment in slices, no device: the two entry points are built, exported and declared, and the
header states the contract; a pure-Python model of the unit plan against l2h_embed_slots_units over batches, lengths and
windows; and every refusal of l2h_embed_slots_units, l2h_embed_forward_slots_units (returned before anything is enqueued)
and EmbedTFGridNet.enroll_job."""
import ctypes

import pytest
import torch

from lookoncetohear_b200 import EmbedTFGridNet, EnrollCapture, EnrollJob
from lookoncetohear_b200.embed import DEFAULT_WINDOW
from serving_util import FAKE_DEV, declaration, header

HEAD = 2
ENTRIES = ("l2h_embed_slots_units", "l2h_embed_forward_slots_units")


@pytest.fixture(scope="module")
def lib():
    from lookoncetohear_b200 import build, _cabi
    build.build()
    return _cabi.lib()


@pytest.fixture(scope="module")
def handle(lib, embed_params):
    net = EmbedTFGridNet(**embed_params)            # weights never committed
    h = net._engine()
    yield h
    del net


def test_entries_exported_and_declared(lib):
    from lookoncetohear_b200 import _cabi
    hdr = header()
    for name in ENTRIES:
        assert hasattr(lib, name), name
        assert name in _cabi.declared_symbols(), name
        assert declaration(hdr, name)[0] is not None, name
    text = " ".join(w for w in hdr.split() if w != "*")
    for phrase in ("exactly once, in order", "the same workspace", "used_dev is final after unit 0",
                   "written by the last unit only", "window < 0", "a unit range outside the plan",
                   "host slot lists are checked on every call"):
        assert phrase in text, phrase


def model_units(n_blocks, n_max, window):
    """the plan of embed_engine.cu: unit 0 (front), per block 3 intra + 2 inter + the inter recurrence's windows + 3
    attention units, and the head"""
    steps = 1 + n_max // 64 - 3
    windows = 1 if window == 0 or window >= steps else -(-steps // window)
    return 1 + n_blocks * (3 + 2 + windows + 3) + 1


@pytest.mark.parametrize("batch", [1, 8, 300])
@pytest.mark.parametrize("n_max", [192, 255, 256, 1000, 48000, 80000, 80063])
@pytest.mark.parametrize("window", [0, 1, 7, 64, 128, 1247, 1248, 1249, 100000])
def test_unit_count_matches_model(lib, handle, embed_params, batch, n_max, window):
    u = ctypes.c_int32(-5)
    assert lib.l2h_embed_slots_units(handle, batch, n_max, window, ctypes.byref(u)) == 0
    assert u.value == model_units(embed_params["num_blocks"], n_max, window)


def test_unit_count_examples(embed_params):
    nb = embed_params["num_blocks"]
    # 5 s at 16 kHz: T = 1251 frames, 1248 inter steps
    assert model_units(nb, 80000, 0) == 2 + 9 * nb
    assert model_units(nb, 80000, 1248) == 2 + 9 * nb
    assert model_units(nb, 80000, 1247) == 2 + 10 * nb
    assert model_units(nb, 80000, 128) == 2 + 18 * nb
    assert model_units(nb, 80000, 1) == 2 + 1256 * nb
    assert isinstance(DEFAULT_WINDOW, int) and DEFAULT_WINDOW >= 0


def test_slots_units_refusals(lib, handle):
    u = ctypes.c_int32(-5)
    assert lib.l2h_embed_slots_units(None, 1, 1000, 0, ctypes.byref(u)) == 1
    assert lib.l2h_embed_slots_units(handle, 1, 1000, 0, None) == 1
    assert lib.l2h_embed_slots_units(handle, 0, 1000, 0, ctypes.byref(u)) == 1
    assert lib.l2h_embed_slots_units(handle, 1, 191, 0, ctypes.byref(u)) == 1
    assert lib.l2h_embed_slots_units(handle, 1, 1000, -1, ctypes.byref(u)) == 1
    assert u.value == -5


def _units_call(lib, h, lens, slots=(0, 1), on_dev=False, S=4, cap=1000, n_max=None, stride=256, used=FAKE_DEV,
                ws_bytes=None, both=False, neither=False, window=0, first=0, n=1):
    B = len(lens)
    n_max = max(lens, default=1000) if n_max is None else n_max
    if ws_bytes is None:
        w = ctypes.c_size_t()
        assert lib.l2h_embed_workspace_bytes(h, max(B, 1), max(n_max, 192), ctypes.byref(w)) == 0
        ws_bytes = w.value
    sh = (ctypes.c_int32 * len(slots))(*slots)
    s_host = None if (on_dev or neither) else sh
    s_dev = FAKE_DEV if (on_dev or both) and not neither else None
    ln = (ctypes.c_int32 * max(B, 1))(*lens)
    return lib.l2h_embed_forward_slots_units(h, FAKE_DEV, S, cap, s_host, s_dev, ln, B, n_max, FAKE_DEV, stride, used,
                                             FAKE_DEV, ws_bytes, window, first, n, None)


def test_forward_slots_units_argument_errors(lib, handle, embed_params):
    total = model_units(embed_params["num_blocks"], 1000, 4)
    # all good but the weights: error 4 once every argument passed, for every unit range inside the plan
    for first, n in ((0, 1), (0, total), (total - 1, 1), (3, 5)):
        assert _units_call(lib, handle, [1000, 192], window=4, first=first, n=n) == 4, (first, n)
    assert _units_call(lib, handle, [1000, 192], on_dev=True, window=0, first=0, n=9) == 4
    # the unit range and the window
    for first, n in ((-1, 1), (0, 0), (0, -1), (total, 1), (total - 1, 2), (0, total + 1), (2**31 - 1, 1)):
        assert _units_call(lib, handle, [1000, 192], window=4, first=first, n=n) == 1, (first, n)
    assert _units_call(lib, handle, [1000, 192], window=4, first=total - 1, n=2) == 1
    assert b"outside the plan" in lib.l2h_last_error()
    assert _units_call(lib, handle, [1000, 192], window=-1) == 1
    assert b"window" in lib.l2h_last_error()
    assert _units_call(lib, handle, [1000, 192], window=0, first=model_units(embed_params["num_blocks"], 1000, 0)) == 1
    # every error of l2h_embed_forward_slots, on a call of a later unit too
    for first in (0, 5):
        kw = {"window": 4, "first": first}
        assert _units_call(lib, None, [1000, 192], ws_bytes=1 << 40, **kw) == 1
        assert _units_call(lib, handle, [1000, 192], used=None, **kw) == 1
        assert _units_call(lib, handle, [1000, 192], both=True, **kw) == 1
        assert _units_call(lib, handle, [1000, 192], neither=True, **kw) == 1
        assert _units_call(lib, handle, [1000, 192], slots=(0, 4), **kw) == 1
        assert _units_call(lib, handle, [1000, 192], slots=(-1, 0), **kw) == 1
        assert _units_call(lib, handle, [1000, 192], slots=(2, 2), **kw) == 1
        assert b"twice" in lib.l2h_last_error()
        assert _units_call(lib, handle, [1000, 191], **kw) == 1
        assert _units_call(lib, handle, [1000, 192], n_max=999, **kw) == 1
        assert _units_call(lib, handle, [1000, 192], cap=999, **kw) == 1
        assert _units_call(lib, handle, [1000, 192], cap=191, n_max=191, **kw) == 1
        assert _units_call(lib, handle, [1000, 192], stride=255, **kw) == 1
        assert _units_call(lib, handle, [1000, 192], S=0, **kw) == 1
        assert _units_call(lib, handle, [1000] * 5, slots=(0, 1, 2, 3, 4), S=4, **kw) == 1
        assert _units_call(lib, handle, [], slots=(), **kw) == 1
        assert _units_call(lib, handle, [1000, 192], ws_bytes=1024, **kw) == 1


def _host_capture(S=4, C=2, cap=1000):
    """an EnrollCapture whose state lives in host memory, for the Python argument checks (no engine call is reached)"""
    c = EnrollCapture.__new__(EnrollCapture)
    c.n_slots, c.channels, c.capacity = S, C, cap
    c.state = torch.zeros(S, C, HEAD + cap)
    return c


def test_enroll_job_python_checks(embed_params):
    net = EmbedTFGridNet(**embed_params)
    cap = _host_capture()
    for w in (-1, 1.5, True, "8"):
        with pytest.raises(ValueError, match="window"):
            net.enroll_job(cap, [0, 1], [500, 500], window=w)
    with pytest.raises(TypeError):
        net.enroll_job(object(), [0], [500])
    with pytest.raises(ValueError, match="channels"):
        net.enroll_job(_host_capture(C=1), [0], [500])
    for slots in ([0, 0], [0, 4], [-1, 1], [0.5, 1], [[0, 1]], []):
        with pytest.raises(ValueError):
            net.enroll_job(cap, slots, [500] * max(len(slots), 1))
    for lens in ([500], [500, 191], [500, 1001], [500, 2.5]):
        with pytest.raises(ValueError):
            net.enroll_job(cap, [0, 1], lens)
    with pytest.raises(ValueError, match="out"):
        net.enroll_job(cap, [0, 1], [500, 500], out=torch.zeros(2, 255))
    with pytest.raises(ValueError, match="out"):
        net.enroll_job(cap, [0, 1], [500, 500], out=torch.zeros(256, 2).t())
    with pytest.raises(ValueError, match="used"):
        net.enroll_job(cap, [0, 1], [500, 500], used=torch.zeros(2, dtype=torch.int64))
    with pytest.raises(ValueError, match="used"):
        net.enroll_job(cap, [0, 1], [500, 500], used=torch.zeros(3, dtype=torch.int32))


def test_enroll_job_step_refusals():
    job = EnrollJob.__new__(EnrollJob)
    job.units, job._next = 10, 0
    for n in (0, -1, 1.5, True, None):
        with pytest.raises(ValueError, match="n must be"):
            job.step(n)
    assert not job.done
    job._next = 10
    assert job.done
