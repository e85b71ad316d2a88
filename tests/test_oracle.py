"""Pin the oracle (oracle/restate.py) against committed fixtures generated from the reference's own code
(tests/golden/make_golden.py: outputs, final streaming state and seeded weights of the reference modules, large
tensors as fixed seeded samples plus their norms).  The reference repo has no golden vectors of its own
(SURVEY.md section 4)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lookoncetohear_b200 import EmbedTFGridNet, Net, synth
from oracle import restate as rs

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PINS = np.load(os.path.join(GOLD, "ref_pins.npz"))


def _pinned(name, t, tol):
    """The full tensor t against the reference's: same shape, sampled values and norm within rel. tolerance tol."""
    assert tuple(t.shape) == tuple(PINS[name + "/shape"]), name
    flat = t.reshape(-1)
    idx = torch.from_numpy(PINS[name + "/idx"].astype(np.int64))
    assert rs.rel_l2(flat[idx], torch.from_numpy(PINS[name + "/val"])) < tol, name
    norm = float(PINS[name + "/norm"])
    assert abs(float(flat.double().norm()) - norm) <= tol * norm, name


def _wsum(sd):
    return np.array([float(sum(v.double().abs().sum() for v in sd.values())),
                     float(sum((v.double() ** 2).sum() for v in sd.values()))])


def _seeded_sd(tsh_params, seed):
    torch.manual_seed(seed)
    return {k: v.detach().clone() for k, v in Net(**tsh_params).state_dict().items()}


def test_seeded_init_matches_reference(tsh_params, embed_params):
    for tag, cls, params in (("init_sep", Net, tsh_params), ("init_embed", EmbedTFGridNet, embed_params)):
        torch.manual_seed(0)
        mine = cls(**params).state_dict()
        keys = [str(k) for k in PINS[f"{tag}/keys"]]
        assert keys == list(mine), tag
        for i, k in enumerate(keys):
            flat = mine[k].reshape(-1)
            got = flat[torch.from_numpy(PINS[f"{tag}/idx"][i].astype(np.int64))]
            assert torch.allclose(got, torch.from_numpy(PINS[f"{tag}/val"][i]), atol=1e-7, rtol=0), k
            assert abs(float(flat.double().norm()) - float(PINS[f"{tag}/norm"][i])) <= 1e-6 * float(PINS[f"{tag}/norm"][i]), k


def test_param_counts(tsh_params, embed_params):
    for tag, net in (("init_sep", Net(**tsh_params)), ("init_embed", EmbedTFGridNet(**embed_params))):
        assert sum(p.numel() for p in net.parameters()) == int(PINS[f"{tag}/n_params"])
    assert int(PINS["init_sep/n_params"]) == 2_037_960 and int(PINS["init_embed/n_params"]) == 2_368_681


def test_restatement_equals_reference_forward_and_state(tsh_params):
    sd = _seeded_sd(tsh_params, 3)
    x, _ = synth.mixture(2, 128 * 9 + 77, seed0=50)
    e = synth.embedding(2, seed0=60)
    st = rs.sep_init_state(sd, 2)
    y, st = rs.sep_predict(sd, x, e[:, 0], st)
    assert rs.rel_l2(y, torch.from_numpy(PINS["fwd3/y"])) < 5e-6
    for k in ("conv_buf", "deconv_buf", "istft_buf"):
        _pinned(f"fwd3/{k}", st[k], 5e-6)
    for i in range(3):
        for k in ("K_buf", "V_buf", "h0", "c0"):
            _pinned(f"fwd3/buf{i}/{k}", st["gridnet_bufs"][f"buf{i}"][k], 5e-6)


def test_restatement_fp64_floor(tsh_params):
    sd = _seeded_sd(tsh_params, 1)
    x, _ = synth.mixture(1, 128 * 8)
    e = synth.embedding(1)
    y64 = rs.sep_forward(rs.cast_sd(sd, torch.float64), x.double(), e.double())
    assert rs.rel_l2(y64, torch.from_numpy(PINS["fwd1/y"])) < 5e-6


def test_embed_restatement_equals_reference(embed_params):
    torch.manual_seed(2)
    sd = {k: v.detach().clone() for k, v in EmbedTFGridNet(**embed_params).state_dict().items()}
    o = rs.embed_forward(sd, synth.enrollment(2, 5000))
    r = torch.from_numpy(PINS["emb2/emb"])
    assert rs.rel_l2(o, r) < 5e-5
    assert float(F.cosine_similarity(o, r).min()) > 0.99999


def test_restatement_streaming_equals_whole(tsh_params):
    sd = _seeded_sd(tsh_params, 5)
    x, _ = synth.mixture(1, 128 * 7)
    e = synth.embedding(1)
    y = rs.sep_forward(sd, x, e)
    st = rs.sep_init_state(sd, 1)
    xp = F.pad(x, (0, 64))
    ys = torch.cat([rs.sep_predict(sd, xp[..., 128 * i:128 * i + 192], e[:, 0], st, pad=False)[0]
                    for i in range(7)], -1)
    assert rs.rel_l2(ys, y) < 5e-6


def test_fast_timing_mode_equals_explicit_loop(tsh_params):
    sd = _seeded_sd(tsh_params, 6)
    x, _ = synth.mixture(1, 128 * 5)
    e = synth.embedding(1)
    y = rs.sep_forward(sd, x, e)
    rs.set_fast(True)
    try:
        yf = rs.sep_forward(sd, x, e)
    finally:
        rs.set_fast(False)
    assert rs.rel_l2(yf, y) < 5e-6


def test_golden_sep(tsh_params):
    g = np.load(os.path.join(GOLD, "sep_golden.npz"))
    sd = _seeded_sd(tsh_params, int(g["seed"]))
    assert np.allclose(_wsum(sd), g["wsum"], rtol=1e-9), "seeded init differs from the build that made the fixture"
    B, N = int(g["B"]), int(g["N"])
    x, _ = synth.mixture(B, N)
    e = synth.embedding(B)
    st = rs.sep_init_state(sd, B)
    y, st = rs.sep_predict(sd, x, e[:, 0], st)
    assert rs.rel_l2(y, torch.from_numpy(g["y"])) < 5e-6
    assert rs.rel_l2(st["gridnet_bufs"]["buf2"]["h0"], torch.from_numpy(g["h0_buf2"])) < 5e-6


def test_golden_embed(embed_params):
    g = np.load(os.path.join(GOLD, "embed_golden.npz"))
    from lookoncetohear_b200.embed import EmbedTFGridNet
    torch.manual_seed(int(g["seed"]))
    sd = {k: v.detach().clone() for k, v in EmbedTFGridNet(**embed_params).state_dict().items()}
    assert np.allclose(_wsum(sd), g["wsum"], rtol=1e-9)
    o = rs.embed_forward(sd, synth.enrollment(2, int(g["n"])))
    assert rs.rel_l2(o, torch.from_numpy(g["emb"])) < 5e-5


def test_si_sdr_known_answer():
    t = torch.sin(torch.arange(1000.) * 0.1)[None]
    n = torch.cos(torch.arange(1000.) * 0.37)[None]
    n = n - (n * t).sum() / (t * t).sum() * t          # orthogonal noise
    p = 3.0 * t + 0.3 * n * (t.norm() / n.norm()) * 3.0
    assert abs(float(rs.si_sdr(p, t)) - 20 * np.log10(1 / 0.3)) < 1e-3


def test_stft_shim_equals_the_stft_the_reference_vendors():
    """The one piece of espnet2 arithmetic the reference DOES carry -- Stft.forward, src/models/tfgridnet_orig/
    stft.py:68-195, identical to what espnet2's STFTEncoder calls -- pins the shim the enrollment oracle uses
    (oracle/shims/espnet2/enh/encoder/stft_encoder.py): same frames, same bins, same values, same output lengths."""
    import sys
    shims = os.path.join(os.path.dirname(os.path.dirname(GOLD)), "oracle", "shims")
    if shims not in sys.path:
        sys.path.insert(0, shims)
    from espnet2.enh.encoder.stft_encoder import STFTEncoder
    for i, (n_fft, hop, n) in enumerate(((128, 64, 5000), (128, 64, 4999), (192, 128, 3001))):
        x = synth.enrollment(3, n).transpose(1, 2).contiguous()          # [B, N, M] as EmbedTFGridNet.forward passes it
        ilens = torch.tensor([n, n, n])
        got, gl_out = STFTEncoder(n_fft, n_fft, hop, window="hann")(x, ilens)                             # complex [B,T,M,F]
        assert got.shape[1] == 1 + n // hop
        assert torch.equal(gl_out, torch.from_numpy(PINS[f"stft{i}/olens"]))
        _pinned(f"stft{i}/spec", torch.view_as_real(got), 1e-6)
