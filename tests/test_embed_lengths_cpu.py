"""Host-side checks of per-utterance enrollment lengths, no device: the argument errors of
l2h_embed_forward_lengths (returned before the weights are checked and before any device work), the length
validation and the grouping of a large batch into calls."""
import ctypes

import pytest
import torch

from lookoncetohear_b200.embed import EmbedTFGridNet, check_lengths, group_by_length


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


def _call(lib, h, n_max, lens, batch, x=16, emb=16, ws=16, ws_bytes=None):
    """Never-dereferenced stand-in device addresses: every call here must stop at argument checking."""
    if ws_bytes is None:
        n = ctypes.c_size_t()
        assert lib.l2h_embed_workspace_bytes(h, max(batch, 1), max(n_max, 192), ctypes.byref(n)) == 0
        ws_bytes = n.value
    arr = None if lens is None else (ctypes.c_int32 * len(lens))(*lens)
    return lib.l2h_embed_forward_lengths(h, x, n_max, arr, batch, emb, ws, ws_bytes, None)


def test_argument_errors_return_1(lib, handle):
    assert _call(lib, None, 1000, [1000], 1, ws_bytes=1 << 40) == 1
    assert _call(lib, handle, 1000, [1000], 1, x=None) == 1
    assert _call(lib, handle, 1000, [1000], 1, emb=None) == 1
    assert _call(lib, handle, 1000, [1000], 1, ws=None) == 1
    assert _call(lib, handle, 1000, [], 0) == 1
    assert _call(lib, handle, 1000, None, -1) == 1
    assert _call(lib, handle, 1000, [1000, 191], 2) == 1
    assert _call(lib, handle, 1000, [1001, 500], 2) == 1
    assert _call(lib, handle, 1000, [500, -3], 2) == 1
    assert b"outside [192, n_max = 1000]" in lib.l2h_last_error()
    assert _call(lib, handle, 191, None, 1) == 1
    assert b"at least 192 samples" in lib.l2h_last_error()
    assert _call(lib, handle, 1000, [1000, 500], 2, ws_bytes=64) == 1


def test_valid_arguments_reach_the_weights_check(lib, handle):
    """Valid arguments on an uncommitted handle: the argument checks pass and the call stops at the weights (4)."""
    assert _call(lib, handle, 1000, [1000, 192, 577], 3) == 4
    assert _call(lib, handle, 1000, None, 3) == 4
    assert _call(lib, handle, 192, [192], 1) == 4


def test_workspace_and_max_batch_count_the_lengths(lib, handle):
    a, b = ctypes.c_size_t(), ctypes.c_size_t()
    assert lib.l2h_embed_workspace_bytes(handle, 1, 80000, ctypes.byref(a)) == 0
    assert lib.l2h_embed_workspace_bytes(handle, 40, 80000, ctypes.byref(b)) == 0
    assert b.value > a.value > 0
    mb = ctypes.c_int32()
    assert lib.l2h_embed_max_batch(handle, 80000, ctypes.byref(mb)) == 0 and mb.value >= 1


@pytest.mark.parametrize("bad", [[4800, 4800], [191, 4800, 4800], [4800, 4801, 4800], [4800, 2400.0, 4800],
                                 [4800, "4800", 4800], [4800, True, 4800], 4800,
                                 torch.tensor([4800.0, 4800.0, 4800.0]), torch.tensor([[4800, 4800, 4800]])])
def test_check_lengths_rejects(bad):
    with pytest.raises(ValueError):
        check_lengths(bad, 3, 4800)


def test_check_lengths_accepts_ints_and_integer_tensors():
    import numpy as np
    assert check_lengths([192, 4800, 1000], 3, 4800) == [192, 4800, 1000]
    assert check_lengths(torch.tensor([192, 4800, 1000], dtype=torch.int32), 3, 4800) == [192, 4800, 1000]
    assert check_lengths(np.array([192, 4800, 1000]), 3, 4800) == [192, 4800, 1000]


def test_cpu_input_is_refused_before_lengths(embed_params):
    net = EmbedTFGridNet(**embed_params)
    with pytest.raises(RuntimeError):
        net(torch.zeros(2, 2, 4800), lengths=[4800, 1000])


def _fake_max_batch(n):
    return max(1, 100_000 // n)                     # fewer utterances per call the longer they are


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_grouping(seed):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(192, 80001, (97,), generator=g).tolist()
    chunks = group_by_length(lens, _fake_max_batch)
    seen = [i for idx, _ in chunks for i in idx]
    assert sorted(seen) == list(range(len(lens)))                       # every utterance exactly once
    for idx, pad in chunks:
        assert 1 <= len(idx) <= _fake_max_batch(pad)                     # at most max_batch(longest in the call)
        assert pad == max(lens[i] for i in idx)                          # padded to its own longest only
        assert [lens[i] for i in idx] == sorted(lens[i] for i in idx)
    # calls taken from the longest down: no call's shortest is shorter than a later call's longest
    for (a, _), (b, pb) in zip(chunks, chunks[1:]):
        assert min(lens[i] for i in a) >= pb
    # scattering the results back by index restores the input order
    out = [None] * len(lens)
    for idx, _ in chunks:
        for i in idx:
            out[i] = lens[i]
    assert out == lens


def test_grouping_single_call_and_ties():
    assert group_by_length([500, 300, 400], lambda n: 8) == [([1, 2, 0], 500)]
    chunks = group_by_length([300] * 5, lambda n: 2)
    assert [len(i) for i, _ in chunks] == [2, 2, 1] and all(p == 300 for _, p in chunks)
