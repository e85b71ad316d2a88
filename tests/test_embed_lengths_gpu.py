"""Enrollment utterances of different lengths in one call (EmbedTFGridNet.forward(x, lengths) ->
l2h_embed_forward_lengths): row b must be the embedding of x[b, :, :lengths[b]] computed alone.

Per-utterance reference calls pick their recurrence kernels from their own size (tensor cores from 2048
sequence-directions), so a short utterance alone can run the CUDA-core recurrence while the padded batch runs the
tensor-core one.  The 1e-5 comparisons therefore also run with the choice pinned ("tc_lstm_min"), which makes both
sides use the same recurrence arithmetic; the default choice is compared as well."""
import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import EmbedTFGridNet, synth
from oracle import restate as rs

pytestmark = pytest.mark.gpu

# B < 16: the inter recurrence of the batch runs on the CUDA cores (lstm_rec); the intra one on the tensor cores
LENS_SMALL = [80000, 32000, 4800, 192, 64 * 9 + 5, 50000]
# B >= 16: both recurrences of the batch run on the tensor cores (tc_lstm); short utterances keep the oracle cheap
LENS_LARGE = [192, 6400] + torch.randint(192, 6401, (18,), generator=torch.Generator().manual_seed(11)).tolist()
ALWAYS_TC, NEVER_TC = 1, 1 << 30


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def make(embed_params, dev):
    """Seeded nets on the device, one per option set (options are per engine handle)."""
    cache = {}

    def get(**opts):
        key = tuple(sorted(opts.items()))
        if key not in cache:
            torch.manual_seed(0)
            net = EmbedTFGridNet(**embed_params).eval()
            sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
            net = net.to(dev)
            for k, v in opts.items():
                net.set_option(k, v)
            cache[key] = (net, sd)
        return cache[key]
    return get


def _batch(lens, seed0):
    """[B, 2, max(lens)] with real signal past every length (it must not be read)."""
    return synth.enrollment(len(lens), max(lens), seed0=seed0)


def _alone(net, x, lens, dev):
    with torch.no_grad():
        return torch.cat([net(x[i:i + 1, :, :n].to(dev)) for i, n in enumerate(lens)]).cpu()


def _rows_close(o, r, tol):
    for i in range(o.shape[0]):
        err = rs.rel_l2(o[i:i + 1], r[i:i + 1])
        assert err <= tol, (i, err)


@pytest.mark.parametrize("lens", [LENS_SMALL, LENS_LARGE], ids=["B6", "B20"])
def test_mixed_lengths_vs_alone_and_oracle(make, dev, lens):
    net, sd = make()
    x = _batch(lens, 3000 + len(lens))
    with torch.no_grad():
        o = net(x.to(dev), lengths=lens).cpu()
    assert torch.isfinite(o).all()
    _rows_close(o, _alone(net, x, lens, dev), 1e-5)
    for i, n in enumerate(lens):
        r = rs.embed_forward(sd, x[i:i + 1, :, :n])
        assert rs.rel_l2(o[i:i + 1], r) <= 1e-3, (i, n, rs.rel_l2(o[i:i + 1], r))
        assert float(F.cosine_similarity(o[i:i + 1], r).min()) >= 0.9999, (i, n)


@pytest.mark.parametrize("tcmin", [ALWAYS_TC, NEVER_TC], ids=["tc_lstm", "lstm_rec"])
@pytest.mark.parametrize("lens", [LENS_SMALL, LENS_LARGE], ids=["B6", "B20"])
def test_mixed_lengths_vs_alone_same_recurrence(make, dev, lens, tcmin):
    net, _ = make(tc_lstm_min=tcmin)
    x = _batch(lens, 3100 + len(lens))
    with torch.no_grad():
        o = net(x.to(dev), lengths=lens).cpu()
    _rows_close(o, _alone(net, x, lens, dev), 1e-5)


def test_mixed_lengths_plain_bf16(make, dev):
    """bf16 = 2 (one MMA pass): the padded batch against per-utterance calls under the same options.  The recurrence is
    pinned to the tensor cores, whose arithmetic per sequence does not depend on the batch.  The CUDA-core family picks
    one of several kernel variants from the sequence count, and their float sums are ordered differently; plain bf16
    GEMMs downstream turn those last-bit differences into ~1e-4 even for an utterance of the full length, which has no
    padding at all."""
    net, _ = make(bf16=2, tc_lstm_min=ALWAYS_TC)
    x = _batch(LENS_SMALL, 3200)
    with torch.no_grad():
        o = net(x.to(dev), lengths=LENS_SMALL).cpu()
    assert torch.isfinite(o).all()
    _rows_close(o, _alone(net, x, LENS_SMALL, dev), 1e-5)


@pytest.mark.parametrize("lens", [LENS_SMALL, LENS_LARGE], ids=["B6", "B20"])
def test_padding_is_never_read(make, dev, lens):
    net, _ = make()
    x = _batch(lens, 3300)
    xz, xn = x.clone(), x.clone()
    for i, n in enumerate(lens):
        xz[i, :, n:] = 0.0
        xn[i, :, n:] = float("nan")
    with torch.no_grad():
        oz = net(xz.to(dev), lengths=lens)
        on = net(xn.to(dev), lengths=torch.tensor(lens, dtype=torch.int32, device=dev))
    assert torch.isfinite(on).all()
    assert torch.equal(on, oz)


def test_equal_lengths_take_the_equal_length_path(make, dev):
    net, _ = make()
    x = synth.enrollment(3, 4800, seed0=3400).to(dev)
    with torch.no_grad():
        a = net(x)
        b = net(x, lengths=[4800] * 3)
        c = net(x, lengths=torch.full((3,), 4800, dtype=torch.int64))
    assert torch.equal(a, b) and torch.equal(a, c)


def test_chunked_batch_scatters_back_in_order(make, dev):
    """More utterances than one call takes: sorted, cut into calls padded to their own longest, scattered back."""
    net, _ = make(tc_lstm_min=NEVER_TC)
    lens = LENS_LARGE
    x = _batch(lens, 3500)
    with torch.no_grad():
        whole = net(x.to(dev), lengths=lens).cpu()
        net.max_batch = lambda n: 3                       # instance attribute: this net only
        try:
            chunked = net(x.to(dev), lengths=lens).cpu()
        finally:
            del net.max_batch
    _rows_close(chunked, whole, 1e-5)
    _rows_close(chunked, _alone(net, x, lens, dev), 1e-5)


@pytest.mark.parametrize("bad", [[4800, 4800], [191, 4800, 4800], [4800, 4801, 4800], [4800, 2400.0, 4800],
                                 torch.tensor([4800.0, 4800.0, 4800.0]), torch.tensor([[4800, 4800, 4800]])])
def test_bad_lengths_raise(make, dev, bad):
    net, _ = make()
    x = synth.enrollment(3, 4800).to(dev)
    with pytest.raises(ValueError):
        net(x, lengths=bad)
