"""ORACLE (test infrastructure): import the reference's own modules, unmodified, by path.

Works only where a reference checkout exists; its path is taken from the environment variable
LOOKONCE_REFERENCE.  Only the fixture generator (tests/golden/make_golden.py) uses it: the tests check against
oracle/restate.py + the committed fixtures under tests/golden/, which were generated from the reference.

The reference's two third-party packages that are absent from this image (asteroid_filterbanks,
espnet2 -- SURVEY.md section 8c) are satisfied by the restatements in oracle/shims/.
Nothing is copied from the reference: its files are executed where they lie.
"""
import importlib
import json
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_SHIMS = os.path.join(_HERE, "shims")


def reference_root():
    c = os.environ.get("LOOKONCE_REFERENCE")
    if c and os.path.isfile(os.path.join(c, "src", "models", "tfgridnet_realtime", "net.py")):
        return c
    return None


def available():
    return reference_root() is not None


def _prepare():
    root = reference_root()
    if root is None:
        raise RuntimeError("reference checkout not found: set LOOKONCE_REFERENCE to its path")
    for p in (root, _SHIMS):
        if p not in sys.path:
            sys.path.insert(0, p)
    try:  # typeguard >= 3 dropped check_argument_types (used by the vendored stft.py:8,45)
        import typeguard
        if not hasattr(typeguard, "check_argument_types"):
            typeguard.check_argument_types = lambda *a, **k: True
    except ImportError:
        pass
    return root


def load_config(name):
    """name: 'tsh' or 'embed' -> model_params dict of configs/<name>.json."""
    root = _prepare()
    with open(os.path.join(root, "configs", f"{name}.json")) as f:
        return json.load(f)["pl_module_args"]["model_params"]


def reference_net(seed=0, **overrides):
    """The reference separation model (src.models.tfgridnet_realtime.net.Net), eval mode."""
    import torch
    _prepare()
    mod = importlib.import_module("src.models.tfgridnet_realtime.net")
    params = dict(load_config("tsh"))
    params.update(overrides)
    torch.manual_seed(seed)
    return mod.Net(**params).eval()


def reference_embed_net(seed=0, **overrides):
    """The reference enrollment model (src.models.tfgridnet_orig.tfgridnet.EmbedTFGridNet)."""
    import torch
    _prepare()
    mod = importlib.import_module("src.models.tfgridnet_orig.tfgridnet")
    params = dict(load_config("embed"))
    params.update(overrides)
    torch.manual_seed(seed)
    return mod.EmbedTFGridNet(**params).eval()
