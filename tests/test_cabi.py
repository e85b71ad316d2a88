"""CPU-side checks of the drop-in boundary: the C-ABI library builds, loads, and exports every
symbol include/*.h declares; host-only entry points behave (no compute calls without a GPU)."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from lookoncetohear_b200 import build, _cabi
    build.build()
    return _cabi.lib()


def _declared():
    names = []
    inc = os.path.join(ROOT, "include")
    for fn in os.listdir(inc):
        if fn.endswith(".h"):
            txt = open(os.path.join(inc, fn)).read()
            txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
            names += re.findall(r"\b(l2h_[a-z0-9_]+)\s*\(", txt)
    return sorted(set(names))


def test_every_declared_symbol_is_exported(lib):
    names = _declared()
    assert len(names) >= 14
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/ but not exported"


def test_binding_covers_header(lib):
    from lookoncetohear_b200 import _cabi
    assert set(_declared()) == set(_cabi.declared_symbols())


def test_create_rejects_other_configs(lib):
    from lookoncetohear_b200 import _cabi
    bad = _cabi.SepConfig(160, 120, 256, 2, 64, 4, 1, 1, 3, 64, 50, 1, 1, 1, 2)
    h = ctypes.c_void_p()
    assert lib.l2h_sep_create(ctypes.byref(bad), ctypes.byref(h)) != 0
    assert b"unsupported" in lib.l2h_last_error()


def test_weight_table_matches_reference_state_dict(lib, tsh_params):
    """Every key of the (mirror) state_dict is accepted, the expected count is reached, unknown
    names and wrong sizes are refused -- all host-side, no GPU."""
    from lookoncetohear_b200 import Net
    net = Net(**tsh_params)
    h = net._engine()
    for k, v in net.state_dict().items():
        host = v.detach().float().contiguous()
        assert lib.l2h_sep_load_weight(h, k.encode(), host.data_ptr(), host.numel()) == 0, k
    ne, nl = ctypes.c_int32(), ctypes.c_int32()
    assert lib.l2h_sep_weights_expected(h, ctypes.byref(ne), ctypes.byref(nl)) == 0
    assert ne.value == nl.value == len(net.state_dict())
    z = torch.zeros(4)
    assert lib.l2h_sep_load_weight(h, b"tfgridnet.nope", z.data_ptr(), 4) == 2
    assert lib.l2h_sep_load_weight(h, b"tfgridnet.deconv.bias", z.data_ptr(), 3) == 1


def test_state_and_workspace_sizes(lib, tsh_params):
    from lookoncetohear_b200 import Net
    net = Net(**tsh_params)
    h = net._engine()
    n = ctypes.c_size_t()
    assert lib.l2h_sep_state_bytes(h, 1, ctypes.byref(n)) == 0
    # reference state is 5,222,480 B/stream (SURVEY 3.3); ours adds the cached gate, the padded
    # K rows, seven extra ring slots (RING = 56 for a 49-row history) and the double-buffered tails
    assert 5_222_480 < n.value < 6_100_000
    n2 = ctypes.c_size_t()
    assert lib.l2h_sep_state_bytes(h, 3, ctypes.byref(n2)) == 0
    assert (n2.value - 64) == 3 * (n.value - 64)
    w = ctypes.c_size_t()
    assert lib.l2h_sep_workspace_bytes(h, 1, 1, 0, ctypes.byref(w)) == 0 and w.value > 0


def test_cpu_tensors_are_refused(tsh_params):
    """No CPU fallback: the module raises instead of computing on the host."""
    from lookoncetohear_b200 import Net
    net = Net(**tsh_params)
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 2, 256), torch.zeros(1, 1, 256))
    with pytest.raises(RuntimeError):
        net.init_buffers(1, "cpu")


def test_mirror_module_matches_reference_layout(tsh_params):
    from lookoncetohear_b200 import Net
    net = Net(**tsh_params)
    assert sum(p.numel() for p in net.parameters()) == 2_037_960          # SURVEY section 0
    sd = net.state_dict()
    assert tuple(sd["tfgridnet.enc.filterbank._filters"].shape) == (194, 1, 192)
    assert tuple(sd["tfgridnet.blocks.2.attn_conv_V.3.norm.weight"].shape) == (1552,)
    assert tuple(sd["tfgridnet.embed_to_feats_proj.0.weight"].shape) == (6208, 256)


def test_embed_weight_table_matches_reference_state_dict(lib, embed_params):
    from lookoncetohear_b200 import EmbedTFGridNet
    net = EmbedTFGridNet(**embed_params)
    assert sum(p.numel() for p in net.parameters()) == 2_368_681          # SURVEY section 0
    h = net._engine()
    for k, v in net.state_dict().items():
        host = v.detach().float().contiguous()
        assert lib.l2h_embed_load_weight(h, k.encode(), host.data_ptr(), host.numel()) == 0, k
    ne, nl = ctypes.c_int32(), ctypes.c_int32()
    assert lib.l2h_embed_weights_expected(h, ctypes.byref(ne), ctypes.byref(nl)) == 0
    assert ne.value == nl.value == len(net.state_dict())
    z = torch.zeros(4)
    assert lib.l2h_embed_load_weight(h, b"blocks.0.nope", z.data_ptr(), 4) == 2
    assert lib.l2h_embed_load_weight(h, b"conv.0.bias", z.data_ptr(), 4) == 1
    n = ctypes.c_size_t()
    assert lib.l2h_embed_workspace_bytes(h, 1, 80000, ctypes.byref(n)) == 0 and n.value > 0
    mb = ctypes.c_int32()
    assert lib.l2h_embed_max_batch(h, 80000, ctypes.byref(mb)) == 0 and mb.value >= 1
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 2, 8000))


def test_weight_info_enumerates_the_state_dict(lib, tsh_params):
    """l2h_sep_weight_info walks exactly the reference state_dict keys (minus buffers the engine ignores) with
    their element counts -- what a non-Python host iterates over (examples/stream_clip.cpp)."""
    from lookoncetohear_b200 import Net
    net = Net(**tsh_params)
    h = net._engine()
    ne = ctypes.c_int32()
    assert lib.l2h_sep_weights_expected(h, ctypes.byref(ne), None) == 0
    sd = {k: v.numel() for k, v in net.state_dict().items()}
    seen = {}
    for i in range(ne.value):
        name, numel = ctypes.c_char_p(), ctypes.c_int64()
        assert lib.l2h_sep_weight_info(h, i, ctypes.byref(name), ctypes.byref(numel)) == 0
        seen[name.value.decode()] = numel.value
    assert seen == sd
    assert lib.l2h_sep_weight_info(h, ne.value, None, None) != 0


def test_cpp_host_example_builds(lib, tmp_path):
    """examples/stream_clip.cpp (a host with no Python and no torch) compiles and links against the header and the
    library; without a GPU it must stop at its first CUDA call with an error, not compute anything."""
    import shutil
    import subprocess
    gxx = shutil.which("g++")
    cuda = "/usr/local/cuda"
    if gxx is None or not os.path.exists(os.path.join(cuda, "include", "cuda_runtime.h")):
        pytest.skip("g++ / CUDA headers not available")
    libdir = os.path.join(ROOT, "lookoncetohear_b200", "lib")
    exe = str(tmp_path / "stream_clip")
    cmd = [gxx, "-O1", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(cuda, "include"),
           os.path.join(ROOT, "examples", "stream_clip.cpp"), "-L", libdir, "-llookonce_b200",
           "-L", os.path.join(cuda, "lib64"), "-lcudart", "-Wl,-rpath," + libdir, "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    if not torch.cuda.is_available():
        r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
        assert r.returncode != 0 and "l2h_sep_commit_weights" in r.stderr


def test_every_engine_option_is_documented_in_the_header():
    """l2h_sep_set_option takes its switches by name: the engine accepts exactly the names below, and every one must appear in
    the header's description of the call (and no environment variable may select a code path: the only getenv allowed in
    csrc/ would be none)."""
    src = open(os.path.join(ROOT, "lookoncetohear_b200", "csrc", "sep_engine.cu")).read()
    hdr = open(os.path.join(ROOT, "include", "lookonce_b200.h")).read()
    names = sorted(set(re.findall(r'n == "([a-z_0-9]+)"', src)))
    assert set(names) == {
        "defaults", "pipeline", "pipeline_frames", "pipeline_lanes", "pipeline_pdl", "pipeline_gemm_shape", "pipeline_midb_hops",
        "pipeline_qkv_lanes", "pipeline_midc_lanes", "pipeline_attn_lanes", "pipeline_out_lanes", "pipeline_front_lanes",
        "pipeline_back_lanes", "pdl", "fused_tail", "back_many", "tc_pdl", "tc_lstm_min", "fuse_ih", "bf16"}
    for n in names:
        assert f'"{n}"' in hdr, f'option "{n}" is accepted by l2h_sep_set_option but not documented in include/lookonce_b200.h'
    csrc = os.path.join(ROOT, "lookoncetohear_b200", "csrc")
    for fn in os.listdir(csrc):
        assert "getenv" not in open(os.path.join(csrc, fn)).read(), f"{fn}: environment switches are not part of the interface"
