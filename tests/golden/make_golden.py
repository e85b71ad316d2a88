"""Generate the committed fixtures from the REFERENCE ITSELF (a checkout of vb000/LookOnceToHear):

    LOOKONCE_REFERENCE=<checkout> python tests/golden/make_golden.py

Weights are not stored (8 MB): they are the PyTorch default init under torch.manual_seed(seed),
which the reference modules and the engine's parameter containers reproduce identically
(tests/test_oracle.py::test_seeded_init_matches_reference); a checksum of the weights is stored
so that an RNG drift between torch builds is detected rather than misread as a parity failure.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from lookoncetohear_b200 import synth  # noqa: E402
from oracle import ref_loader as rl  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def weight_checksum(sd):
    return np.array([float(sum(v.double().abs().sum() for v in sd.values())),
                     float(sum((v.double() ** 2).sum() for v in sd.values()))])


def sample(t, k, seed):
    """A fixed, seeded sample of at most k elements of t: (flat indices, values, L2 norm of the whole tensor)."""
    flat = t.detach().reshape(-1)
    g = torch.Generator().manual_seed(seed)
    idx = torch.randperm(flat.numel(), generator=g)[:k].sort().values if flat.numel() > k else torch.arange(flat.numel())
    return idx.numpy().astype(np.int32), flat[idx].numpy(), float(flat.double().norm())


def ref_pins():
    """What the reference-pinning tests compare against (tests/test_oracle.py, tests/test_ckpt.py): outputs and
    state of the reference modules on the tests' seeded inputs, and the vendored STFT; large tensors as samples."""
    import importlib
    pins = {}

    def put(name, t, k=512, seed=0):
        pins[name + "/idx"], pins[name + "/val"], pins[name + "/norm"] = sample(t, k, seed)
        pins[name + "/shape"] = np.array(t.shape)

    # seeded default init of both networks: 16 sampled values and the norm of every state_dict entry
    for tag, net in (("init_sep", rl.reference_net(0)), ("init_embed", rl.reference_embed_net(0))):
        sd = net.state_dict()
        rows = []
        for i, v in enumerate(sd.values()):
            flat = v.reshape(-1)
            g = torch.Generator().manual_seed(i)
            idx = torch.randperm(flat.numel(), generator=g)[:16] if flat.numel() >= 16 else torch.arange(16) % flat.numel()
            rows.append((idx.numpy().astype(np.int32), flat[idx].numpy(), float(flat.double().norm())))
        pins[f"{tag}/keys"] = np.array(list(sd))
        pins[f"{tag}/idx"] = np.stack([r[0] for r in rows])
        pins[f"{tag}/val"] = np.stack([r[1] for r in rows])
        pins[f"{tag}/norm"] = np.array([r[2] for r in rows])
        pins[f"{tag}/n_params"] = np.array(sum(p.numel() for p in net.parameters()))
    # forward + final state, seed 3, B = 2, ragged length
    net = rl.reference_net(3)
    x, _ = synth.mixture(2, 128 * 9 + 77, seed0=50)
    e = synth.embedding(2, seed0=60)
    with torch.no_grad():
        pins["fwd3/y"] = net(x, e).numpy()
        st = net.init_buffers(2, "cpu")
        _, st = net.predict(x, e[:, 0], st)
    for k in ("conv_buf", "deconv_buf", "istft_buf"):
        put(f"fwd3/{k}", st[k])
    for i in range(3):
        for k in ("K_buf", "V_buf", "h0", "c0"):
            put(f"fwd3/buf{i}/{k}", st["gridnet_bufs"][f"buf{i}"][k], 512, 10 * i)
    # forward, seed 1, B = 1 (the fp64 floor of the restatement)
    net = rl.reference_net(1)
    x, _ = synth.mixture(1, 128 * 8)
    with torch.no_grad():
        pins["fwd1/y"] = net(x, synth.embedding(1)).numpy()
    # enrollment, seed 2
    en = rl.reference_embed_net(2)
    with torch.no_grad():
        pins["emb2/emb"] = en(synth.enrollment(2, 5000)).numpy()
    # checkpoint -> outputs on the GPU: the reference network of seed 13 on a 12-hop clip
    net = rl.reference_net(13)
    x, _ = synth.mixture(1, 128 * 12)
    with torch.no_grad():
        pins["ckpt13/y"] = net(x, synth.embedding(1)).numpy()
    pins["ckpt13/wsum"] = weight_checksum(net.state_dict())
    # the STFT the reference vendors (src/models/tfgridnet_orig/stft.py)
    Stft = importlib.import_module("src.models.tfgridnet_orig.stft").Stft
    for i, (n_fft, hop, n) in enumerate(((128, 64, 5000), (128, 64, 4999), (192, 128, 3001))):
        xs = synth.enrollment(3, n).transpose(1, 2).contiguous()
        ref, olens = Stft(n_fft=n_fft, win_length=n_fft, hop_length=hop, window="hann")(xs, torch.tensor([n, n, n]))
        put(f"stft{i}/spec", ref, 1024, 100 + i)
        pins[f"stft{i}/olens"] = olens.numpy()
    np.savez_compressed(os.path.join(HERE, "ref_pins.npz"), **pins)


def main():
    torch.set_num_threads(8)
    # ---- separation: whole utterance (ragged length) + chunked streaming, B=2 ----------------
    seed = 0
    net = rl.reference_net(seed)
    B, N = 2, 128 * 14 - 51
    x, tgt = synth.mixture(B, N)
    e = synth.embedding(B)
    with torch.no_grad():
        y = net(x, e)
        st = net.init_buffers(B, "cpu")
        xp = torch.nn.functional.pad(x, (0, 128 * 14 - N + 64))
        ys = torch.cat([net.predict(xp[..., 128 * i:128 * i + 192], e[:, 0], st, pad=False)[0] for i in range(14)], -1)
    np.savez_compressed(os.path.join(HERE, "sep_golden.npz"), seed=seed, B=B, N=N, y=y.numpy(),
                        y_stream=ys.numpy(), h0_buf2=st["gridnet_bufs"]["buf2"]["h0"].numpy(),
                        istft_buf=st["istft_buf"].numpy(), wsum=weight_checksum(net.state_dict()))
    # ---- separation: longer than the attention window (T = 70 > 50), B=1, keep only a digest ---
    N2 = 128 * 70
    x2, _ = synth.mixture(1, N2, seed0=1100)
    e2 = synth.embedding(1, seed0=3100)
    with torch.no_grad():
        y2 = net(x2, e2)
    np.savez_compressed(os.path.join(HERE, "sep_golden_long.npz"), seed=seed, N=N2, y_tail=y2[..., -1024:].numpy(),
                        y_rms=float(y2.pow(2).mean().sqrt()), y_sum=float(y2.double().sum()))
    # ---- enrollment ------------------------------------------------------------------------------
    en = rl.reference_embed_net(seed)
    xe = synth.enrollment(2, 4800)
    with torch.no_grad():
        emb = en(xe)
    np.savez_compressed(os.path.join(HERE, "embed_golden.npz"), seed=seed, n=4800, emb=emb.numpy(),
                        wsum=weight_checksum(en.state_dict()))
    # ---- state_dict key names and shapes of both reference modules (checkpoint compatibility, SURVEY 8f-1) ----
    import json
    keys = {"sep": {k: list(v.shape) for k, v in net.state_dict().items()},
            "embed": {k: list(v.shape) for k, v in en.state_dict().items()}}
    with open(os.path.join(HERE, "ckpt_keys.json"), "w") as f:
        json.dump(keys, f, indent=0, sort_keys=True)
    ref_pins()
    print("written", os.listdir(HERE))


if __name__ == "__main__":
    main() if "--pins-only" not in sys.argv else ref_pins()
