"""The kernel harness library (tests/kernels/) and the float64 references the kernel-level GPU tests
(test_umma_gemm_gpu.py, test_lstm_kernels_gpu.py, test_attention_kernels_gpu.py, test_front_back_kernels_gpu.py,
test_embed_kernels_gpu.py, test_rows_gemm_kernels_gpu.py, test_mid_kernels_gpu.py, test_tail_kernel_gpu.py,
test_targets_kernels_gpu.py, test_state_kernels_gpu.py, test_embed_slot_kernels_gpu.py) rely on.  The enrollment references (estd64, efront64, egn64, eqkv_ln64, softmax64,
eattn_out64, ehead64) are pinned to oracle/restate.py; each of their mutants is shown to miss the reference by more than
10x its bound, and einter_mask_expected's mutants to change it.  No device needed."""
import ctypes
import math

import torch

from kernels import harness as kh


def test_harness_builds_and_exports():
    L = kh.lib()
    for s in kh.SYMBOLS:
        assert hasattr(L, s), s


def test_ctypes_mirrors_match_the_c_structs():
    L = kh.lib()
    for fn, cls in kh.MIRRORS.items():
        assert getattr(L, fn)() == ctypes.sizeof(cls), (fn, cls.__name__)


def _plan(n_chunks, N, passes=3, ldc=None):
    d = kh.Gemm()
    d.a0.channels, d.a0.n_pos, d.a0.n_inner, d.a0.n_outer = 64 * n_chunks, 130, 1, 1
    d.n_chunks, d.rows_per_seq, d.nseq, d.N, d.K, d.passes = n_chunks, 130, 1, N, 64 * n_chunks, passes
    d.ldc = N if ldc is None else ldc
    d.c_seq_stride = 130 * d.ldc
    return kh.gemm_plan(d)


def test_gemm_plan_resident_switch():
    """umma::launch's own plan (no device needed): with bf16x3 the weight slab stays resident in shared memory up to
    2 k-chunks at BN = 128 and up to 5 at BN = 64; beyond, A and B stream through a ring of at least two operand slots.
    test_umma_gemm_gpu.py runs k-chunk counts on both sides of both switch points."""
    for N, bn, last in ((256, 128, 2), (64, 64, 5)):
        for k in (1, last, last + 1, 65, 96):
            p = _plan(k, N)
            assert p is not None and p.BN == bn, (N, k)
            assert p.b_resident == int(k <= last), (N, k, p.b_resident)
            if not p.b_resident:
                assert p.nop >= 2, (N, k, p.nop)
    assert _plan(97, 64) is None and _plan(0, 64) is None and _plan(1, 64, passes=4) is None


def test_gemm_plan_vec_ok():
    """the float4 epilogue is chosen from the row alignment alone: a ragged N with padded rows keeps it"""
    assert _plan(1, 70, ldc=72).vec_ok == 1
    assert _plan(1, 70).vec_ok == 0
    assert _plan(1, 64).vec_ok == 1


def test_lstm_reference_equals_torch_lstm():
    """lstm_ref over the packed gate layout (columns j*4+q) equals torch.nn.LSTM in float64, both directions, with a
    carried (h0, c0) on the forward direction."""
    torch.manual_seed(0)
    nseq, L, F = 5, 7, 16
    for reverse in (False, True):
        m = torch.nn.LSTM(F, 64, batch_first=True).double()
        x = torch.randn(nseq, L, F, dtype=torch.float64)
        h0 = 0.5 * torch.randn(1, nseq, 64, dtype=torch.float64)
        c0 = 0.5 * torch.randn(1, nseq, 64, dtype=torch.float64)
        # lstm_ref carries state on direction 0 only: the reverse direction starts from zero
        with torch.no_grad():
            if reverse:
                want, (hn, cn) = m(x.flip(1))
                want = want.flip(1)
            else:
                want, (hn, cn) = m(x, (h0, c0))
        w_ih, w_hh = m.weight_ih_l0.detach(), m.weight_hh_l0.detach()
        b = (m.bias_ih_l0 + m.bias_hh_l0).detach()
        gx = (x.reshape(-1, F) @ w_ih.T + b)[:, _perm()]           # rows seq*L + step
        d = 1 if reverse else 0
        gx2 = torch.zeros(nseq * L, 512, dtype=torch.float64)
        gx2[:, d * 256:(d + 1) * 256] = gx
        whh = torch.zeros(2, 256, 64, dtype=torch.float64)
        whh[d] = kh.packed_from_torch(w_hh)
        hs, fin = kh.lstm_ref(gx2, whh, nseq, L, d + 1, lambda s, t: s * L + t,
                              h0=None if reverse else h0[0], c0=None if reverse else c0[0])
        got = hs[d].transpose(0, 1)                                    # [nseq][L][64]
        assert torch.allclose(got, want, rtol=0, atol=1e-12)
        assert torch.allclose(fin[d][0], hn[0], rtol=0, atol=1e-12)
        assert torch.allclose(fin[d][1], cn[0], rtol=0, atol=1e-12)


def _perm():
    return torch.tensor([q * 64 + j for j in range(64) for q in range(4)])


def test_packed_from_torch_is_the_gate_permutation():
    w = torch.arange(256 * 3, dtype=torch.float64).view(256, 3)
    assert torch.equal(kh.packed_from_torch(w), w[_perm()])


def test_bf16_split_reproduces_fp32():
    """hi = rn_bf16(x) (torch rounds to nearest even, like __float2bfloat16_rn), lo = rn_bf16(x - hi): hi + lo equals x
    to 2^-17 relative (lo carries 8 more significant bits), and |lo| <= 2^-9 |x|."""
    torch.manual_seed(1)
    x = torch.cat([torch.randn(100000), torch.randn(1000) * 1e-20, torch.randn(1000) * 1e20,
                   torch.tensor([1.0, -1.0, 0.0, 1 + 2 ** -8, 1 + 3 * 2 ** -8])])
    hi, lo = kh.split_bf16(x)
    r = hi.double() + lo.double()
    nz = x != 0
    rel = ((r - x.double()).abs() / x.double().abs())[nz]
    assert float(rel.max()) <= 2.0 ** -17
    assert bool(((lo.double().abs() <= 2.0 ** -8 * x.double().abs()) | ~nz).all())
    # round to nearest EVEN at ties (bf16 ulp at 1 is 2^-7): 1 + 2^-8 -> 1, 1 + 3 * 2^-8 -> 1 + 2^-6
    assert float(hi[-2]) == 1.0 and float(hi[-1]) == 1.0 + 2 ** -6


def test_split_product_passes():
    """passes = 3 is exact on small-integer inputs (every operand is its own hi); on general inputs each pass count is
    within its documented scale of the exact product and passes = 3 < 2 < 1 in error."""
    torch.manual_seed(2)
    a = torch.randint(-4, 5, (33, 200)).float()
    b = torch.randint(-4, 5, (17, 200)).float()
    exact = a.double() @ b.double().T
    assert torch.equal(kh.split_product(a, b, 3), exact)
    a, b = torch.randn(64, 256), torch.randn(48, 256)
    exact = a.double() @ b.double().T
    P = a.double().abs() @ b.double().abs().T
    err = {p: float(((kh.split_product(a, b, p) - exact).abs() / P).max()) for p in (1, 2, 3)}
    assert err[3] <= 3 * 2.0 ** -17 and err[2] <= 2.0 ** -8 and err[1] <= 2.0 ** -7
    assert err[3] < err[2] / 20 and err[2] < err[1]


# ---- the attention section ------------------------------------------------------------------------------------------
def test_sep_layout_matches_the_product_library(tsh_params):
    """the harness's state layout (kh_sep_layout) is the one the product library reports, so the state buffers the
    attention, front and back tests build are the engine's"""
    from lookoncetohear_b200 import Net, build, _cabi
    build.build()
    net = Net(**tsh_params)
    h, L = net._engine(), _cabi.lib()
    offs = (ctypes.c_int64 * 18)()
    assert L.l2h_sep_state_offsets(h, offs, 18) == 0
    hb, stride = ctypes.c_int64(), ctypes.c_int64()
    assert L.l2h_sep_state_layout(h, ctypes.byref(hb), ctypes.byref(stride)) == 0
    one = kh.sep_layout(1)
    n_blocks = (stride.value - one["ST_BLK"]) // one["BK_STRIDE"]
    names = {"RING": 0, "QK_LD": 1, "QK_DIM": 2, "V_DIM": 3, "ATT": 4, "ST_EMB": 5, "ST_GATE": 6, "ST_CONV": 7,
             "ST_DECONV": 8, "ST_ISTFT": 9, "ST_BLK": 10, "BK_K": 11, "BK_V": 12, "BK_H": 13, "BK_C": 14, "BK_STRIDE": 15,
             "ST_POS": 16, "ST_CALLS": 17}
    want = {n: offs[i] for n, i in names.items()}
    # the weight generation of the gate memo is the word before the stream's call count
    want.update(HEADER_BYTES=hb.value, STREAM_STRIDE=stride.value, ST_GEN=offs[17] - 1)
    assert kh.sep_layout(n_blocks) == want
    assert (kh.RING, kh.QK_LD, kh.QK_DIM, kh.V_DIM, kh.ATT) == tuple(offs[:5])


def test_ring_model():
    """frame n in slot n mod 56; a window and its 6 spare slots cover the ring once, also across the wrap, for
    negative frames and above 2^31; rows are laid out head by head, K ring then V ring, block by block"""
    lay = kh.sep_layout(2)
    ring = kh.Ring(lay)
    for n in (0, 1, 48, 49, 50, 55, 56, 57, 111, 2 ** 31 + 7):
        w, sp = ring.window(n), ring.spare(n)
        assert len(w) == kh.ATT and w[-1] == n and len(sp) == kh.RING - kh.ATT and sp[-1] == n - kh.ATT
        assert sorted(ring.slot(m) for m in w + sp) == list(range(kh.RING))
    assert ring.slot(-1) == 55 and ring.slot(56) == 0 and ring.slot(2 ** 31 + 7) == 23
    blk1 = lay["ST_BLK"] + lay["BK_STRIDE"]
    assert ring.row(1, "k", 0, 0) == blk1 + lay["BK_K"]
    assert ring.row(1, "k", 1, 57) == blk1 + lay["BK_K"] + (kh.RING + 1) * kh.QK_LD
    assert ring.row(1, "k", 3, 55) + kh.QK_LD == blk1 + lay["BK_V"]
    assert ring.row(1, "v", 3, -1) + kh.V_DIM == blk1 + lay["BK_H"]
    assert ring.row(0, "v", 2, 2 ** 31 + 7) == lay["ST_BLK"] + lay["BK_V"] + (2 * kh.RING + 23) * kh.V_DIM


def test_window_attention_is_the_reference_loop():
    """attention64 over window_mask equals the model's loop (oracle/restate.py::sep_block): Kall = [K_buf (49 zero rows
    of a fresh stream) ; k], query t attends to rows t .. t+49"""
    torch.manual_seed(3)
    T, H = 7, 2
    q = torch.randn(T, H, kh.QK_DIM, dtype=torch.float64)
    k = torch.randn(T, H, kh.QK_DIM, dtype=torch.float64)
    v = torch.randn(T, H, kh.V_DIM, dtype=torch.float64)
    Kall = torch.cat([torch.zeros(kh.ATT - 1, H, kh.QK_DIM, dtype=torch.float64), k])
    Vall = torch.cat([torch.zeros(kh.ATT - 1, H, kh.V_DIM, dtype=torch.float64), v])
    want = torch.stack([torch.einsum("hj,jhd->hd", torch.softmax(
        torch.einsum("hd,jhd->hj", q[t], Kall[t:t + kh.ATT]) / math.sqrt(kh.QK_DIM), -1), Vall[t:t + kh.ATT])
        for t in range(T)])
    frames = list(range(-(kh.ATT - 1), T))
    got = kh.attention64(q, Kall, Vall, kh.window_mask(list(range(T)), frames))
    assert torch.allclose(got, want, rtol=0, atol=1e-12)


def test_mutated_references_differ():
    """each mutated reference the attention tests use moves a small case (scores ~ N(0, 1)) by more than 10x the
    kernels' bounds at such scores (<= 2e-5), so the sensitivity checks cannot pass vacuously"""
    g = torch.Generator().manual_seed(5)
    N = 3
    X = torch.randn(N, kh.NF, kh.CH, generator=g)
    w = (torch.rand(64, kh.NQKV, generator=g) * 2 - 1) * 0.25
    bias = 0.1 * torch.randn(kh.NQKV, generator=g)
    slopes = torch.tensor([0.25, -0.1, 0.05, 0.2])
    ln = [(1 + 0.2 * torch.randn(n, generator=g), 0.2 * torch.randn(n, generator=g)) for n in (kh.QK_DIM, kh.QK_DIM, kh.V_DIM)]
    P = kh.qkv_proj64(X, w, bias, slopes)
    ref = kh.qkv_ln64(P, *ln)
    assert [tuple(t.shape) for t in ref] == [(N, 4, kh.QK_DIM), (N, 4, kh.QK_DIM), (N, 4, kh.V_DIM)]
    for mut in (kh.qkv_ln64(P, *ln, unbiased=True), kh.qkv_ln64(P, *ln, heads_transposed=True),
                kh.qkv_ln64(kh.qkv_proj64(X, w, bias, slopes, swap_qk_slopes=True), *ln)):
        assert max(float((a - b).abs().max()) for a, b in zip(mut, ref)) > 1e-3
    # attention: frames -3 .. 60 of one stream (zero rows before 0), queries at frames 1 and 55
    n = 64
    kf = list(range(-3, n - 3))
    K = torch.randn(n, 4, kh.QK_LD, generator=g, dtype=torch.float64)
    V = torch.randn(n, 4, kh.V_DIM, generator=g, dtype=torch.float64)
    K[:3], V[:3] = 0, 0
    q = torch.randn(2, 4, kh.QK_LD, generator=g, dtype=torch.float64)
    qf = [1, 55]
    ref = kh.merge_heads64(kh.attention64(q, K, V, kh.window_mask(qf, kf)))
    muts = [kh.attention64(q, K, V, kh.window_mask(qf, kf, -kh.ATT, -1)),
            kh.attention64(q, K, V, kh.window_mask(qf, kf, -(kh.ATT - 2))),
            kh.attention64(q, K, V, kh.window_mask(qf, kf, -kh.ATT)),
            kh.attention64(q, K, V, kh.window_mask(qf, kf, mask_before_start=True)),
            kh.attention64(q, K, V, kh.window_mask(qf, kf), scale=1 / math.sqrt(kh.QK_LD))]
    for m in muts:
        assert float((kh.merge_heads64(m) - ref).abs().max()) > 1e-3
    o = kh.attention64(q, K, V, kh.window_mask(qf, kf))
    assert float((kh.merge_heads64(o, transposed=True) - ref).abs().max()) > 1e-3
    # the head merge: channel h*16 + c of bin f is feature f*16 + c of head h
    assert torch.equal(ref[1, 5, 2 * 16 + 3], o[1, 2, 5 * 16 + 3])
    # attention output: LayerNorm over the frame's 6208 values, then the gate
    Pp = torch.randn(N, kh.NF, kh.CH, generator=g)
    Xr = torch.randn(N, kh.NF, kh.CH, generator=g)
    gate = 1 + 0.5 * torch.randn(N, kh.NF, kh.CH, generator=g)
    lg, lb = 1 + 0.2 * torch.randn(kh.FC, generator=g), 0.2 * torch.randn(kh.FC, generator=g)
    ref = kh.ln_frame_res64(Pp, Xr, lg, lb, gate)
    for mut in (dict(per_bin=True), dict(gate_first=True), dict(unbiased=True)):
        assert float((kh.ln_frame_res64(Pp, Xr, lg, lb, gate, **mut) - ref).abs().max()) > 3e-4, mut


# ---- the front and the back -----------------------------------------------------------------------------------------
def _net_sd(tsh_params, seed=0):
    from lookoncetohear_b200 import Net
    torch.manual_seed(seed)
    return Net(**tsh_params).state_dict()


def _fb(sd64):
    g = lambda k: sd64["tfgridnet." + k]
    return dict(Wa=g("enc.filterbank._filters")[:, 0], Wc=g("conv.0.weight"), bc=g("conv.0.bias"),
                Wd=g("deconv.weight"), bd=g("deconv.bias"), Ws=g("dec.filterbank._filters")[:, 0],
                We=g("embed_to_feats_proj.0.weight"), be=g("embed_to_feats_proj.0.bias"),
                lg=g("embed_to_feats_proj.1.weight"), lb=g("embed_to_feats_proj.1.bias"))


def test_front_and_back_references_are_the_model(tsh_params):
    """over three consecutive calls of 1, 2 and 5 frames of one stream, front64 and back64 (fed the tails of the model's
    state, in the kernels' layouts) reproduce oracle/restate.py::sep_core: the encoder output taps["enc"], the new
    conv / deconv / iSTFT tails, and the 128 T samples of the output before the look-ahead; gate64 is taps["gate"]"""
    from oracle import restate
    sd = _net_sd(tsh_params)
    sd["tfgridnet.embed_to_feats_proj.1.weight"] = 1 + 0.3 * torch.randn(kh.FC)
    sd["tfgridnet.embed_to_feats_proj.1.bias"] = 0.3 * torch.randn(kh.FC)
    sd64 = restate.cast_sd(sd, torch.float64)
    w = _fb(sd64)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, kh.HOP * 8 + kh.LOOKAHEAD, generator=g, dtype=torch.float64)
    emb = torch.randn(kh.SPK, generator=g, dtype=torch.float64)
    state = restate.sep_init_state(sd64, 1, dtype=torch.float64)
    pos = 0
    for T in (1, 2, 5):
        conv_tail = state["conv_buf"][0].permute(1, 0, 2)                 # [4][2][97] -> [2 frames][4][97]
        deconv_tail = state["deconv_buf"][0].permute(1, 2, 0)             # [64][2][97] -> [2][97][64]
        istft_tail = state["istft_buf"][0, :, :, 0]                       # [2 ears][194]
        end = kh.HOP * (pos + T) + kh.LOOKAHEAD
        taps = {}
        y, state = restate.sep_core(sd64, x[None, :, kh.HOP * pos:end], emb[None], state, taps=taps)
        f = kh.front64(x, end, kh.HOP * pos, T, conv_tail, w["Wa"], w["Wc"], w["bc"])
        assert torch.allclose(f["X"], taps["enc"][0], rtol=0, atol=1e-12)
        assert torch.allclose(f["tail"], state["conv_buf"][0].permute(1, 0, 2), rtol=0, atol=1e-12)
        b = kh.back64(taps["block2"][0], deconv_tail, istft_tail, w["Wd"], w["bd"], w["Ws"])
        assert torch.allclose(b["y"], y[0, :, :kh.HOP * T], rtol=0, atol=1e-12)
        assert torch.equal(b["deconv_tail"], state["deconv_buf"][0].permute(1, 2, 0))
        assert torch.allclose(b["istft_tail"], state["istft_buf"][0, :, :, 0], rtol=0, atol=1e-12)
        gate, _ = kh.gate64(emb, w["We"], w["be"], w["lg"], w["lb"])
        assert torch.allclose(gate, taps["gate"][0, 0], rtol=0, atol=1e-12)
        pos += T


def test_front_and_back_mutants_differ(tsh_params):
    """every mutated reference the front / back tests use moves a small case far from the reference (by more than 1 %
    of the largest value): the kernels' bounds are ~1e-5 of it, so the >= 10x margins cannot pass vacuously.  The
    gate's unbiased variance moves a value by |LN| / 12416 only: more than 12x gate64's own bound somewhere."""
    from oracle import restate
    w = _fb(restate.cast_sd(_net_sd(tsh_params), torch.float64))
    g = torch.Generator().manual_seed(8)
    T = 3
    x = torch.randn(2, 2000, generator=g, dtype=torch.float64)
    ct, ct2 = torch.randn(2, 2, 4, kh.NF, generator=g, dtype=torch.float64)
    dt, dt2 = torch.randn(2, 2, kh.NF, kh.CH, generator=g, dtype=torch.float64)
    it, it2 = torch.randn(2, 2, kh.NROW, generator=g, dtype=torch.float64)
    X = torch.randn(T, kh.NF, kh.CH, generator=g, dtype=torch.float64)
    front = lambda s0=300, tail=ct, **m: kh.front64(x, 1900, s0, T, tail, w["Wa"], w["Wc"], w["bc"], **m)
    ref = front()
    for m in (dict(shift=1), dict(reim_interleaved=True), dict(conv_flip_time=True), dict(edge_clamp=True),
              dict(tail=ct2), dict(s0=300 + kh.HOP * 5)):
        mut = front(**m)
        d = max(float((mut[k] - ref[k]).abs().max()) for k in ("X", "tail"))
        assert d > 1e-2 * float(ref["X"].abs().max()), m
    # the edge clamp changes bins 0 and 96 only
    mut = front(edge_clamp=True)
    assert torch.equal(mut["X"][:, 1:-1], ref["X"][:, 1:-1])
    back = lambda d=dt, i=it, **m: kh.back64(X, d, i, w["Wd"], w["bd"], w["Ws"], **m)
    ref = back()
    for m in (dict(plain_conv=True), dict(swap_ear_ri=True), dict(ola="dropped"), dict(ola="wrong_half"),
              dict(carry_istft=False), dict(d=dt2), dict(i=it2)):
        mut = back(**m)
        d = max(float((mut[k] - ref[k]).abs().max()) for k in ("y", "istft_tail"))
        assert d > 1e-2 * float(ref["y"].abs().max()), m
    # the overlap-add mutants change the first 64 samples of each frame only
    assert torch.equal(back(ola="dropped")["y"].view(2, T, kh.HOP)[..., kh.LOOKAHEAD:], ref["y"].view(2, T, kh.HOP)[..., kh.LOOKAHEAD:])
    e = torch.randn(kh.SPK, generator=g, dtype=torch.float64)
    lg, lb = 1 + 0.3 * torch.randn(kh.FC, generator=g), 0.3 * torch.randn(kh.FC, generator=g)
    ref, bound = kh.gate64(e, w["We"], w["be"], lg, lb)
    for m in (dict(cf_order=True), dict(unbiased=True)):
        mut, _ = kh.gate64(e, w["We"], w["be"], lg, lb, **m)
        assert float(((mut - ref).abs() / bound).max()) > 12, m


def test_front_back_packing_round_trips(tsh_params):
    """pack_front_back gives the kernels' layouts; unpacked again they are the state-dict tensors bit for bit, and the
    two pad columns of the transposed analysis filters hold the pad value"""
    sd = _net_sd(tsh_params)
    p = kh.pack_front_back(sd)
    shapes = dict(wat=(192, 196), ws=(194, 192), wc=(64, 36), bc=(64,), we=(kh.FC, 256), be=(kh.FC,), lne_g=(kh.FC,),
                  lne_b=(kh.FC,), wd=(64, 4, 9), bd=(4,))
    assert {k: tuple(v.shape) for k, v in p.items()} == shapes
    assert bool(p["wat"][:, 194:].isnan().all()) and not bool(p["wat"][:, :194].isnan().any())
    for k, v in kh.unpack_front_back(p).items():
        assert torch.equal(v, sd[k]), k
    assert torch.equal(p["wat"][5, 100], sd["tfgridnet.enc.filterbank._filters"][100, 0, 5])
    assert torch.equal(p["wd"][7, 3, 2 * 3 + 1], sd["tfgridnet.deconv.weight"][7, 3, 2, 1])


# ---- the enrollment network's own kernels ---------------------------------------------------------------------------
def test_embed_layout():
    """the constants the enrollment tests build their buffers from are the kernels' own"""
    lay = kh.embed_layout()
    assert lay == dict(NFFT=kh.E_NFFT, HOP=kh.E_HOP, NF=kh.E_NF, CH=kh.E_CH, QK=kh.E_QK, VDIM=kh.E_VDIM, FC=kh.E_FC,
                       NQKV=kh.E_NQKV, DFT_LD=kh.E_DFT_LD, EAOUT_SMEM=(64 * 68 + 64 * 64 + 65 * 64) * 4,
                       LENS_PER_LAUNCH=kh.E_LENS_PER_LAUNCH)


def _embed_sd(embed_params, seed=0):
    """a seeded EmbedTFGridNet's state dict with random affine parameters (the defaults are ones and zeros, under which
    swapped or transposed gains would go unseen)"""
    from lookoncetohear_b200 import EmbedTFGridNet
    torch.manual_seed(seed)
    sd = {k: v.detach().clone() for k, v in EmbedTFGridNet(**embed_params).state_dict().items()}
    g = torch.Generator().manual_seed(seed + 1)
    for k, v in sd.items():
        if k.endswith((".gamma", "conv.1.weight", "embed_proj.1.weight")):
            sd[k] = 1 + 0.3 * torch.randn(v.shape, generator=g)
        elif k.endswith((".beta", "conv.1.bias", "embed_proj.1.bias")):
            sd[k] = 0.3 * torch.randn(v.shape, generator=g)
    return sd


def _embed_front(x, n, T, sd64):
    """estd64 -> efront64 -> egn64 of one utterance x [2][>= n]"""
    inv, _ = kh.estd64(x, n)
    f = kh.efront64(x, n, T, inv, sd64["conv.0.weight"], sd64["conv.0.bias"])
    X, _ = kh.egn64(f["X"], f["sums"], kh.e_frames(n), sd64["conv.1.weight"], sd64["conv.1.bias"])
    return X, f


def test_embed_references_are_the_model(embed_params):
    """the chained references reproduce oracle/restate.py::embed_forward and embed_block to 1e-12: estd64 -> efront64 ->
    egn64 the encoder output taps["enc"], eqkv_ln64 -> softmax64 -> eattn_out64 the attention section of every block
    (its input is embed_block's output with the attention's LayerNorm affine zeroed), ehead64 the embedding; for a batch
    of equal lengths and for an utterance of a padded batch alone (its rows t >= T_b are exactly zero)"""
    from oracle import restate
    sd = _embed_sd(embed_params)
    sd64 = restate.cast_sd(sd, torch.float64)
    pk = kh.pack_embed(sd64, embed_params["num_blocks"])
    g = torch.Generator().manual_seed(21)
    N, n = 700, 450
    x = torch.randn(2, 2, N, generator=g)
    T = kh.e_frames(N)
    for xb, nb in ((x, N), (x[1:2, :, :n], n)):
        taps = {}
        emb = restate.embed_forward(sd64, xb.double(), taps=taps)
        for b in range(xb.shape[0]):
            X, _ = _embed_front(x[1 if nb == n else b], nb, T, sd64)
            Tb = kh.e_frames(nb)
            assert torch.allclose(X[:Tb], taps["enc"][b], rtol=0, atol=1e-12)
            assert bool((X[Tb:] == 0).all())
            for blk in range(embed_params["num_blocks"]):
                Xin = taps["enc"][b:b + 1] if blk == 0 else taps[f"block{blk - 1}"][b:b + 1]
                sdz = dict(sd64)
                p = f"blocks.{blk}.attn_concat_proj.2."
                sdz[p + "gamma"], sdz[p + "beta"] = torch.zeros_like(sd64[p + "gamma"]), torch.zeros_like(sd64[p + "beta"])
                X2 = restate.embed_block(sdz, f"blocks.{blk}.", Xin)[0]
                got = kh.eattention64(X2, {k: v.double() for k, v in pk.items()}, blk)
                assert torch.allclose(got, taps[f"block{blk}"][b], rtol=0, atol=1e-12)
            Xl = taps[f"block{embed_params['num_blocks'] - 1}"][b]
            HD = Xl.permute(0, 2, 1).reshape(Tb, -1) @ sd64["embed_proj.0.weight"].T + sd64["embed_proj.0.bias"]
            out, _ = kh.ehead64(HD, Tb, sd64["embed_proj.1.weight"], sd64["embed_proj.1.bias"])
            assert torch.allclose(out, emb[b], rtol=0, atol=1e-12)


def _far(mut, ref, bound, k=10):
    """mut differs from ref by more than k times the bound somewhere"""
    return float(((mut.double() - ref.double()).abs() / bound.clamp_min(1e-300)).max()) > k


def test_embed_mutants_differ(embed_params):
    """every mutated reference the enrollment kernel tests use misses the reference by more than 10x its bound on a
    small case, so their >= 10x margins cannot pass vacuously"""
    from oracle import restate
    sd64 = restate.cast_sd(_embed_sd(embed_params), torch.float64)
    pk = {k: v.double() for k, v in kh.pack_embed(sd64).items()}
    g = torch.Generator().manual_seed(22)
    N, n = 1000, 450
    x = torch.randn(2, N, generator=g).float()
    inv, ib = kh.estd64(x, n)
    for m in (dict(unbiased=False), dict(mic0_only=True)):
        assert _far(kh.estd64(x, n, **m)[0], inv, ib), m
    T = kh.e_frames(N)
    Wc, bc = sd64["conv.0.weight"], sd64["conv.0.bias"]
    ref = kh.efront64(x, n, T, inv, Wc, bc)
    for m in (dict(edge_repeat=True), dict(reflect_at=N), dict(symmetric_hann=True), dict(reim_interleaved=True),
              dict(conv_flip_time=True)):
        assert _far(kh.efront64(x, n, T, inv, Wc, bc, **m)["X"], ref["X"], ref["X_bound"]), m
    Tb = kh.e_frames(n)
    X = torch.randn(T, kh.E_NF, kh.E_CH, generator=g).double()
    sums = torch.stack([X[:Tb].sum(), (X[:Tb] ** 2).sum()])
    gg, gb = sd64["conv.1.weight"], sd64["conv.1.bias"]
    ref, bound = kh.egn64(X, sums, Tb, gg, gb)
    assert torch.equal(ref[Tb:], X[Tb:])
    for m in (dict(padded_count=True), dict(unbiased=True)):
        assert _far(kh.egn64(X, sums, Tb, gg, gb, **m)[0], ref, bound), m
    QKV = torch.randn(5, kh.E_NF, kh.E_NQKV, generator=g).double()
    ln = [pk["0." + k] for k in ("gq", "bq", "gk", "bk", "gv", "bv")]
    ref = kh.eqkv_ln64(QKV, *ln)
    for m in (dict(per_bin=True), dict(heads_transposed=True), dict(swap_qk_gains=True)):
        mut = kh.eqkv_ln64(QKV, *ln, **m)
        assert any(_far(mut[k][0], ref[k][0], ref[k][1]) for k in "QKV"), m
    # softmax: 4 utterances of different lengths (z % 4 picks another utterance's length for most heads)
    lens, Tp = [450, 1000, 300, 700], 64
    S = 3 * torch.randn(4 * kh.E_NH * T, Tp, generator=g)
    ncols = kh.softmax_row_lens(4 * kh.E_NH, T, lens, T)
    ref, bound = kh.softmax64(S, ncols)
    assert _far(kh.softmax64(S, kh.softmax_row_lens(4 * kh.E_NH, T, lens, T, by_mod=True))[0], ref, bound)
    assert _far(kh.softmax64(S, ncols, zero_pad=False)[0], ref, bound)
    O = torch.randn(3, kh.E_NH, kh.E_VDIM, generator=g).double()
    Xr = torch.randn(3, kh.E_NF, kh.E_CH, generator=g).double()
    a = [pk["0." + k] for k in ("wp_t", "bp", "slope_p", "gp", "bpn")]
    ref, bound = kh.eattn_out64(O, Xr, *a)
    for m in (dict(heads_cf=True), dict(ignore_slope=True), dict(ln_per_bin=True)):
        assert _far(kh.eattn_out64(O, Xr, *a, **m)[0], ref, bound), m
    HD = torch.randn(T, 256, generator=g).double()
    hg, hb = sd64["embed_proj.1.weight"], sd64["embed_proj.1.bias"]
    ref, bound = kh.ehead64(HD, Tb, hg, hb)
    for m in (dict(div_T=True), dict(mean_before_ln=True)):
        assert _far(kh.ehead64(HD, Tb, hg, hb, **m)[0], ref, bound), m
    # the inter mask: exact, so any change is a miss; the longest utterance is left as it is
    steps = T - 3
    lens = lens[:2]
    gx = torch.randn(2 * kh.E_NF, steps, 512, generator=g)
    ref = kh.einter_mask_expected(gx, lens, steps)
    assert torch.equal(ref.view(2, kh.E_NF, steps, 512)[1], gx.view(2, kh.E_NF, steps, 512)[1])
    assert bool(ref.view(2, kh.E_NF, steps, 512)[0, :, Tb - 3:, 0::4].isneginf().all())
    assert torch.equal(ref.view(2, kh.E_NF, steps, 512)[0, :, :Tb - 3], gx.view(2, kh.E_NF, steps, 512)[0, :, :Tb - 3])
    for m in (dict(start=4), dict(start=2), dict(fwd_only=True), dict(pad=(float("-inf"), 0.0, float("-inf"), 0.0))):
        assert not torch.equal(kh.einter_mask_expected(gx, lens, steps, **m), ref), m


# ---- the rows GEMM and the one-hop middle section (test_rows_gemm_kernels_gpu.py, test_mid_kernels_gpu.py) -----------
def _mid_params(seed=0):
    """random block weights in the engine's stored layouts (W^T, gate columns j*4 + q), distinct PReLU slopes"""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: scale * torch.randn(*s, generator=g)
    return dict(wl1_t=r(128, 64, scale=128 ** -0.5), bl1=r(64, scale=0.3), ln2_g=1 + r(64, scale=0.2),
                ln2_b=r(64, scale=0.2), wih2_t=r(64, 256, scale=0.25), whh2_t=r(64, 256, scale=0.25), b2=r(256, scale=0.3),
                wl2_t=r(64, 64, scale=0.125), bl2=r(64, scale=0.3), wqkv_t=r(64, kh.NQKV, scale=0.125),
                bqkv=r(kh.NQKV, scale=0.3), slopes=torch.tensor([0.25, -0.3, 0.6, 0.1]))


def _torch_gate_rows(w):
    """engine gate columns j*4 + q of W^T [K][256] -> torch.nn.LSTMCell rows q*64 + j of W [256][K]"""
    return w.T.reshape(64, 4, -1).transpose(0, 1).reshape(256, -1)


def test_rows_gemm_reference_is_layer_norm_and_linear():
    torch.manual_seed(1)
    A, Wt, b, R = torch.randn(37, 64), torch.randn(64, 256) / 8, torch.randn(256), torch.randn(37, 256)
    ln = torch.nn.LayerNorm(64).double()
    with torch.no_grad():
        ln.weight.copy_(1 + 0.2 * torch.randn(64))
        ln.bias.copy_(0.2 * torch.randn(64))
        lin = torch.nn.Linear(64, 256).double()
        lin.weight.copy_(Wt.T)
        lin.bias.copy_(b)
        want = lin(ln(A.double())) + R.double()
    got, bound = kh.rows_gemm64(A, Wt, b, (ln.weight.float(), ln.bias.float()), R)
    assert torch.allclose(got, want, rtol=0, atol=1e-12)
    assert bool((bound > 0).all())
    # windowed rows: sequence s, row p at s * seq_stride + p * ld
    assert kh.rows_offsets(5, 64, 2, 1000).tolist() == [0, 64, 1000, 1064, 2000]
    assert kh.rows_offsets(3, 72).tolist() == [0, 72, 144]


def test_mid_references_are_the_torch_modules():
    """mid64 is nn.Linear(128, 64) + residual, nn.LayerNorm(64), nn.LSTMCell(64, 64) (gates permuted to j*4 + q),
    nn.Linear(64, 64) + residual and nn.Linear(64, 112) + nn.PReLU per Q / K / V group; mid_b64 over hops is the
    LSTMCell stepped; lstm_cell64 is the LSTMCell's cell from given pre-activations."""
    p = _mid_params()
    torch.manual_seed(2)
    n = 23
    Y, X, h, c = torch.randn(n, 128), torch.randn(n, 64), 0.5 * torch.randn(n, 64), torch.randn(n, 64)
    d = lambda t: t.double()
    with torch.no_grad():
        l1 = torch.nn.Linear(128, 64).double()
        l1.weight.copy_(p["wl1_t"].T); l1.bias.copy_(p["bl1"])
        ln = torch.nn.LayerNorm(64).double()
        ln.weight.copy_(p["ln2_g"]); ln.bias.copy_(p["ln2_b"])
        cell = torch.nn.LSTMCell(64, 64).double()
        cell.weight_ih.copy_(_torch_gate_rows(p["wih2_t"])); cell.weight_hh.copy_(_torch_gate_rows(p["whh2_t"]))
        cell.bias_ih.copy_(_torch_gate_rows(p["b2"][None, :])[:, 0]); cell.bias_hh.zero_()
        l2 = torch.nn.Linear(64, 64).double()
        l2.weight.copy_(p["wl2_t"].T); l2.bias.copy_(p["bl2"])
        lq = torch.nn.Linear(64, kh.NQKV).double()
        lq.weight.copy_(p["wqkv_t"].T); lq.bias.copy_(p["bqkv"])
        X1 = d(X) + l1(d(Y))
        h2, c2 = cell(ln(X1), (d(h), d(c)))
        X2 = X1 + l2(h2)
        Z = lq(X2)
        P = torch.cat([torch.nn.PReLU(init=float(p["slopes"][i])).double()(Z[:, a:b])
                       for i, (a, b) in enumerate(((0, 24), (24, 48), (48, kh.NQKV)))], 1)
        r = kh.mid64(Y, X, h, c, p)
        for k, want in (("X1", X1), ("h", h2), ("c", c2), ("X2", X2), ("P", P)):
            assert torch.allclose(r[k], want, rtol=0, atol=1e-12), k
            assert bool((r[k + "_b"] > 0).all()), k
        # three hops of mid_b from the same GI rows
        GIs = torch.stack([kh.mid_a64(torch.randn(n, 128), torch.randn(n, 64), p)[2].float() for _ in range(3)])
        H, _, (hs, _, cs, _) = kh.mid_b64(GIs, h, c, p)
        hh, cc = d(h), d(c)
        for j in range(3):
            g = d(GIs[j]) + hh @ d(p["whh2_t"])
            cell_only = torch.nn.LSTMCell(256, 64, bias=False).double()
            cell_only.weight_ih.copy_(_torch_gate_rows(torch.eye(256)))
            cell_only.weight_hh.zero_()
            hh, cc = cell_only(g, (hh, cc))
            assert torch.allclose(H[j], hh, rtol=0, atol=1e-12)
        assert torch.allclose(hs, hh, rtol=0, atol=1e-12) and torch.allclose(cs, cc, rtol=0, atol=1e-12)
        gates = 2 * torch.randn(n, 256)
        hl, _, cl, _ = kh.lstm_cell64(gates, c)
        hw, cw = cell_only(d(gates), (torch.zeros(n, 64, dtype=torch.float64), d(c)))
        assert torch.allclose(hl, hw, rtol=0, atol=1e-12) and torch.allclose(cl, cw, rtol=0, atol=1e-12)


def test_mid_pack_round_trips_through_mid_widx():
    """kh_mid_pack (the engine's own packing at commit) puts W^T[k][n] of each matrix at region + mid_widx(KS, N, k, n)
    and zero in every padding float"""
    lay = kh.mid_layout()
    assert lay["MID_RT"] == 8 and lay["NUM_SMS"] == 132
    p = _mid_params(3)
    mats = [p[k] for k in ("wl1_t", "wih2_t", "whh2_t", "wl2_t", "wqkv_t")]
    packed = kh.mid_pack(*mats)
    for got, want in zip(kh.mid_unpack(packed, lay), mats):
        assert torch.equal(got, want)
    used = torch.zeros(lay["MID_PACK"], dtype=torch.bool)
    for region, K, N, ks in kh.MID_MATRICES:
        used[lay[region] + kh.mid_widx(ks, N, torch.arange(K)[:, None], torch.arange(N)[None, :])] = True
    assert int(used.sum()) == sum(K * N for _, K, N, _ in kh.MID_MATRICES)
    assert bool((packed[~used] == 0).all())


def _ratio(a, b, bound):
    return float(((a - b).abs() / bound).max())


def test_rows_gemm_and_mid_mutants_differ():
    """every mutated reference the GPU tests use misses the reference by >= 10x its bound, on at least one of the outputs
    of the kernel it stands for, on test-like data; the eps placement shows on a row of small spread"""
    torch.manual_seed(4)
    A = torch.randn(40, 64)
    A[3] = 0.5 + 0.01 * torch.randn(64)
    Wt, b, R = torch.randn(64, 64) / 8, 0.3 * torch.randn(64), torch.randn(40, 64)
    ln = (1 + 0.2 * torch.randn(64), 0.2 * torch.randn(64))
    ref, bound = kh.rows_gemm64(A, Wt, b, ln, R)
    for m in ("unbiased", "eps_outside", "no_transpose", "drop_bias", "drop_residual"):
        assert _ratio(kh.rows_gemm64(A, Wt, b, ln, R, **{m: True})[0], ref, bound) >= 10, m
    assert _ratio(ref[:-16], ref[16:], bound[16:]) >= 10                 # rows offset by one 16-row tile
    p = _mid_params(5)
    n = 97
    Y, X, h, c = torch.randn(n, 128), torch.randn(n, 64), 0.5 * torch.randn(n, 64), torch.randn(n, 64)
    Y[7] = 0
    X[7] = 0.4 - p["bl1"] + 0.01 * torch.randn(64)                        # X1 of row 7: spread 0.01
    r = kh.mid64(Y, X, h, c, p)
    muts = dict(unbiased=("h", "c", "P"), eps_outside=("h", "c", "P"), swap_if=("h", "c", "P"), drop_c=("h", "c", "P"),
                whh_new_h=("h", "c", "P"), drop_residual=("X2", "P"), drop_bias=("X2", "P"), slope_groups=("P",))
    for m, keys in muts.items():
        mr = kh.mid64(Y, X, h, c, p, **{m: (20, 48) if m == "slope_groups" else True})
        assert max(_ratio(mr[k], r[k], r[k + "_b"]) for k in keys) >= 10, m
    GIs = torch.stack([kh.mid_a64(torch.randn(n, 128), torch.randn(n, 64), p)[2].float() for _ in range(3)])
    H, Hb, (hs, hb, cs, cb) = kh.mid_b64(GIs, h, c, p)
    H2 = kh.mid_b64(GIs, h, c, p, no_advance=True)[0]
    assert _ratio(H2[1:], H[1:], Hb[1:]) >= 10
    _, _, (hs2, _, cs2, _) = kh.mid_b64(GIs, h, c, p, store_first=True)
    assert _ratio(hs2, hs, hb) >= 10 and _ratio(cs2, cs, cb) >= 10
    gates = 2 * torch.randn(n, 256)
    hl, hlb, cl, clb = kh.lstm_cell64(gates, c)
    for m in ("swap_if", "drop_c"):
        hm, _, cm, _ = kh.lstm_cell64(gates, c, **{m: True})
        assert _ratio(hm, hl, hlb) >= 10 and _ratio(cm, cl, clb) >= 10, m


# ---- the fused one-hop tail (test_tail_kernel_gpu.py) ------------------------------------------------------------------
def _tail_block(sd64, blk):
    """block blk's weights in the engine's stored layouts (sep_engine.cu: W^T, gate columns j*4 + q, slopes Q K V proj)"""
    g = lambda k: sd64[f"tfgridnet.blocks.{blk}." + k]
    pk = kh.packed_from_torch
    p = dict(wl1_t=g("intra_linear.weight").T, bl1=g("intra_linear.bias"), ln2_g=g("inter_norm.norm.weight"),
             ln2_b=g("inter_norm.norm.bias"), wih2_t=pk(g("inter_rnn.weight_ih_l0")).T,
             whh2_t=pk(g("inter_rnn.weight_hh_l0")).T, b2=pk(g("inter_rnn.bias_ih_l0") + g("inter_rnn.bias_hh_l0")),
             wl2_t=g("inter_linear.weight").T, bl2=g("inter_linear.bias"),
             wqkv_t=torch.cat([g(f"attn_conv_{n}.0.weight") for n in "QKV"]).T,
             bqkv=torch.cat([g(f"attn_conv_{n}.0.bias") for n in "QKV"]),
             slopes=torch.stack([g(f"attn_conv_{n}.1.weight")[0] for n in "QKV"] + [g("attn_concat_proj.1.weight")[0]]),
             wp_t=g("attn_concat_proj.0.weight").T, bp=g("attn_concat_proj.0.bias"),
             lnp_g=g("attn_concat_proj.3.norm.weight"), lnp_b=g("attn_concat_proj.3.norm.bias"))
    for n in "QKV":
        p[f"ln{n.lower()}_g"], p[f"ln{n.lower()}_b"] = g(f"attn_conv_{n}.3.norm.weight"), g(f"attn_conv_{n}.3.norm.bias")
    ih = (g("intra_norm.norm.weight"), g("intra_norm.norm.bias"),
          torch.cat([pk(g("intra_rnn.weight_ih_l0")).T, pk(g("intra_rnn.weight_ih_l0_reverse")).T], 1),
          torch.cat([pk(g("intra_rnn.bias_ih_l0") + g("intra_rnn.bias_hh_l0")),
                     pk(g("intra_rnn.bias_ih_l0_reverse") + g("intra_rnn.bias_hh_l0_reverse"))]))
    return p, ih


def _intra(sd64, blk, X):
    """the block's intra BiLSTM output [97][128] of X [97][64] (oracle/restate.py::sep_block's first half)"""
    from oracle import restate
    g = lambda k: sd64[f"tfgridnet.blocks.{blk}." + k]
    A = restate._ln(X, g("intra_norm.norm.weight"), g("intra_norm.norm.bias"))[None]
    yf, _, _ = restate._lstm_seq(A, g("intra_rnn.weight_ih_l0"), g("intra_rnn.weight_hh_l0"), g("intra_rnn.bias_ih_l0"),
                                 g("intra_rnn.bias_hh_l0"))
    yb, _, _ = restate._lstm_seq(A, g("intra_rnn.weight_ih_l0_reverse"), g("intra_rnn.weight_hh_l0_reverse"),
                                 g("intra_rnn.bias_ih_l0_reverse"), g("intra_rnn.bias_hh_l0_reverse"), reverse=True)
    return torch.cat([yf[0], yb[0]], -1)


def _ring_rows(buf):
    """the oracle's K_buf / V_buf [4][49][n] (frames pos - 49 .. pos - 1) as tail64's rows of frames pos - 50 .. pos - 1"""
    k, v = buf["K_buf"].permute(1, 0, 2), buf["V_buf"].permute(1, 0, 2)
    return torch.cat([torch.zeros_like(k[:1]), k]), torch.cat([torch.zeros_like(v[:1]), v])


def test_tail_reference_is_the_model(tsh_params):
    """tail64 (and tail_chain64 over 3 hops) reproduces oracle/restate.py::sep_block for T = 1 with carried buffers: the
    block output, the new K_buf / V_buf rows and (h0, c0); its GX is the next block's intra input projection of that
    output (the gate applied first, as sep_core applies it to the next block's input)"""
    from oracle import restate
    sd64 = restate.cast_sd(_net_sd(tsh_params, seed=3), torch.float64)
    hp = restate.sep_hparams(sd64)
    p, _ = _tail_block(sd64, 0)
    _, ih1 = _tail_block(sd64, 1)
    g = torch.Generator().manual_seed(11)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    buf = dict(K_buf=r(4, 49, kh.QK_DIM), V_buf=r(4, 49, kh.V_DIM), h0=0.5 * r(1, kh.NF, 64), c0=r(1, kh.NF, 64))
    gate = 1 + 0.5 * r(kh.NF, 64)
    X = [r(kh.NF, 64) for _ in range(3)]
    Y = [_intra(sd64, 0, x) for x in X]
    hk, hv = _ring_rows(buf)
    chain = kh.tail_chain64(Y, X, buf["h0"][0], buf["c0"][0], p, hk, hv, gates=[gate] * 3, nxt=ih1)
    one = kh.tail64(Y[0], X[0], buf["h0"][0], buf["c0"][0], p, hk, hv, gate, ih1)
    for t in range(3):
        want = restate.sep_block(sd64, "tfgridnet.blocks.0.", X[t][None, None], buf, hp, 50)[0, 0]
        got = chain[t]
        for k, ref in (("X", want * gate), ("K", buf["K_buf"][:, -1]), ("V", buf["V_buf"][:, -1]), ("h", buf["h0"][0]),
                       ("c", buf["c0"][0])):
            assert torch.allclose(got[k], ref, rtol=0, atol=1e-12), (t, k)
            assert bool((got[k + "_b"] > 0).all()), (t, k)
            if t == 0:
                assert torch.equal(one[k], got[k]), k
        # the next block's intra gates of its input (the gated output): columns d*256 + j*4 + q
        A = restate._ln(want * gate, ih1[0], ih1[1])
        blk1 = lambda k: sd64["tfgridnet.blocks.1." + k]
        gx = torch.cat([kh.packed_from_torch((A @ blk1(f"intra_rnn.weight_ih_l0{s}").T + blk1(f"intra_rnn.bias_ih_l0{s}")
                                              + blk1(f"intra_rnn.bias_hh_l0{s}")).T).T for s in ("", "_reverse")], 1)
        assert torch.allclose(got["GX"], gx, rtol=0, atol=1e-12), t
    assert torch.allclose(kh.chan_ln64(X[0].reshape(-1)[:kh.NF * 6], p["lnq_g"], p["lnq_b"], 6),
                          kh.layer_norm64(X[0].reshape(-1)[:kh.NF * 6], p["lnq_g"], p["lnq_b"]), rtol=0, atol=1e-12)


def test_tail_mutants_differ():
    """every mutated tail64 misses the reference by >= 10x its bound on at least one output (X, K, V, h, c or GX), on
    test-like data: a young stream's window (zero rows), X1 of small spread on rows 7 and 96, a K head of mean >> spread"""
    p = _mid_params(6)
    g = torch.Generator().manual_seed(8)
    r = lambda *s, scale=1.0: scale * torch.randn(*s, generator=g)
    p.update(lnq_g=1 + r(kh.QK_DIM, scale=0.2), lnq_b=r(kh.QK_DIM, scale=0.2), lnk_g=1 + r(kh.QK_DIM, scale=0.2),
             lnk_b=r(kh.QK_DIM, scale=0.2), lnv_g=1 + r(kh.V_DIM, scale=0.2), lnv_b=r(kh.V_DIM, scale=0.2),
             wp_t=r(64, 64, scale=0.25), bp=r(64, scale=0.1), lnp_g=1 + r(kh.FC, scale=0.2), lnp_b=r(kh.FC, scale=0.2))
    p["bqkv"][36:42] = 5.0                                  # K head 2: mean 5, spread ~0.1
    p["wqkv_t"][:, 36:42] *= 0.1
    Y, X, h, c = r(kh.NF, 128), r(kh.NF, 64), r(kh.NF, 64, scale=0.5), r(kh.NF, 64)
    for f in (7, 96):
        Y[f] = 0
        X[f] = 0.4 - p["bl1"] + 0.01 * r(64)
    hk, hv = torch.zeros(50, kh.NHEAD, kh.QK_DIM), torch.zeros(50, kh.NHEAD, kh.V_DIM)
    hk[20:], hv[20:] = r(30, kh.NHEAD, kh.QK_DIM), r(30, kh.NHEAD, kh.V_DIM)     # frames before the start: zero rows
    gate = 1 + 0.5 * r(kh.NF, 64)
    gate[::5] *= -1
    nxt = (1 + r(64, scale=0.2), r(64, scale=0.2), r(64, 512, scale=0.125), r(512, scale=0.3))
    stale = (r(kh.NHEAD, kh.QK_DIM), r(kh.NHEAD, kh.V_DIM))
    ref = kh.tail64(Y, X, h, c, p, hk, hv, gate, nxt)
    keys = ("X", "K", "V", "h", "c", "GX")
    for name, kw in list(kh.TAIL_MUTANTS.items()) + [("stale", dict(stale=stale))]:
        mr = kh.tail64(Y, X, h, c, p, hk, hv, gate, nxt, **kw)
        assert max(_ratio(mr[k], ref[k], ref[k + "_b"]) for k in keys) >= 10, name


def test_target_lists_reference_is_the_plain_definition():
    """On a valid list (monotone offsets inside [0, rows], every record in the state) target_lists_ref is the obvious
    reading: listener i owns rows offsets[i] .. offsets[i+1]-1, each storing through its own record."""
    import random
    g = random.Random(3)
    n, rows, batch = 40, 150, 200
    off = sorted(g.randrange(rows - 10) for _ in range(n - 1))
    off = [0] + off + [rows - 10]
    recs = g.sample(range(batch), rows)
    hops = [g.randrange(4) for _ in range(n)]
    ref = kh.target_lists_ref(recs, off, None, hops, n, 0, rows, batch)
    owner = [next((i for i in range(n) if off[i] <= r < off[i + 1]), -1) for r in range(rows)]
    assert ref["owner"] == owner and ref["start"] == off
    assert ref["rec"] == [recs[r] if owner[r] >= 0 else -1 for r in range(rows)]
    assert ref["rec_hops"] == [hops[i] if i >= 0 else 0 for i in owner]
    assert ref["lead"] == [recs[off[i]] if off[i] < off[i + 1] else -1 for i in range(n)]
    grp = kh.target_lists_ref(None, None, [2, -1, 0], None, 3, 4, 12, 12)
    assert grp["rec"] == [8, 9, 10, 11, -1, -1, -1, -1, 0, 1, 2, 3] and grp["lead"] == [8, -1, 0] and grp["start"] is None


def test_target_lists_mutants_differ():
    """Every mutant of target_lists_ref differs from the reference on each case of the GPU test
    (test_targets_kernels_gpu.py) that names it, and every mutant is named by some case."""
    named = set()
    for c in kh.target_lists_cases():
        args = (c["records"], c["offsets"], c["groups"], c["hops"], c["n"], c["K"], c["rows"], c["batch"])
        ref = kh.target_lists_ref(*args)
        for m in c["catches"]:
            assert kh.target_lists_ref(*args, mutant=m) != ref, (c["name"], m)
        named |= c["catches"]
        assert c["rows"] >= c["n"]
    assert named == set(kh.TARGET_LISTS_MUTANTS)


def test_gate_fanout_reference_and_mutants():
    """gate_fanout_ref copies X0 of the owner (mixture 0 for no owner) times the row's gate; the owner r % K mutant differs
    on a dense fan-out of 3 x 3 rows, the gated unowned row on a listed one with apply_gate"""
    g = torch.Generator().manual_seed(5)
    X0 = torch.randn(3, 2, kh.NF, kh.CH, generator=g)
    gates = 1 + 0.5 * torch.randn(9, kh.NF, kh.CH, generator=g)
    out = kh.gate_fanout_ref(X0, gates, None, 3, 1)
    assert torch.equal(out[4], X0[1] * gates[4][None])
    assert not torch.equal(kh.gate_fanout_ref(X0, gates, None, 3, 0, mutant="owner_mod"), kh.gate_fanout_ref(X0, gates, None, 3, 0))
    owner = [0, -1, 2, 1, -1, 0, 2, 1, 0]
    lst = kh.gate_fanout_ref(X0, gates, owner, 3, 1)
    assert torch.equal(lst[1], X0[0]) and torch.equal(lst[2], X0[2] * gates[2][None])
    assert not torch.equal(kh.gate_fanout_ref(X0, gates, owner, 3, 1, mutant="gate_unowned"), lst)
    assert torch.equal(kh.gate_fanout_ref(X0, gates, owner, 3, 0), torch.stack([X0[max(i, 0)] for i in owner]))


def test_row_frames_is_the_kernels_rule():
    assert [kh.row_frames([-1, 0, 1, 3, 4, kh.INT_MAX, -kh.INT_MAX], b, 3) for b in range(7)] == [0, 0, 1, 3, 0, 0, 0]
    assert kh.row_frames(None, 0, 5) == 5


# ---- the state-record kernels and the enrollment rows of a capture (test_state_kernels_gpu.py,
# test_embed_slot_kernels_gpu.py) ---------------------------------------------------------------------------------------
_LAY = dict(ST_CALLS=257, ST_POS=258, ST_GEN=256, ST_BLK=300, BK_STRIDE=40, ST_CONV=264)


def _state(hdr, ss, B, seed):
    import numpy as np
    return np.random.default_rng(seed).integers(-2 ** 31, 2 ** 31, hdr + B * ss, dtype=np.int64).astype(np.int32)


def test_state_references_are_the_plain_definition():
    """state_init, reset, advance_header and set_clip_base references against element loops on small synthetic
    layouts, and each of their mutants changes them"""
    import numpy as np
    hdr, ss, B = 16, 300, 3
    ref = kh.state_init_ref(hdr, ss, B)
    loop = [0] * hdr + [kh.NAN_BITS if o < kh.SPK else 0 for b in range(B) for o in range(ss)]
    assert ref.tolist() == loop
    for m in kh.STATE_INIT_MUTANTS:
        assert not np.array_equal(kh.state_init_ref(hdr, ss, B, mutant=m), ref), m
    st = _state(hdr, ss, 5, 1)
    out = kh.reset_streams_ref(st, hdr, ss, _LAY, [3, 1])
    for b in range(5):
        r = out[hdr + b * ss:hdr + (b + 1) * ss].tolist()
        if b in (3, 1):
            assert r == [kh.NAN_BITS] * kh.SPK + [0] * (ss - kh.SPK)
        else:
            assert r == st[hdr + b * ss:hdr + (b + 1) * ss].tolist()
    assert not np.array_equal(kh.reset_streams_ref(st, hdr, ss, _LAY, [3, 1], mutant="clock_kept"), out)
    st = _state(hdr, ss, 5, 2)
    for i, c in ((0, 2 ** 32 - 3), (hdr + 2 * ss + 258, 2 ** 32 - 1)):
        kh.put64(st, i, c)
    st[hdr + 2 * ss + 257] = 2 ** 31 - 1
    out = kh.advance_header_ref(st, hdr, ss, _LAY, 3, 5)
    assert kh.get64(out, 0) == 2 ** 32 + 2 and kh.get64(out, 2) == kh.get64(st, 2) + 1 and out[6] == 0
    assert kh.get64(out, hdr + 2 * ss + 258) == 2 ** 32 + 4 and out[hdr + 2 * ss + 257] == -2 ** 31
    assert np.array_equal(out[hdr + 3 * ss:], st[hdr + 3 * ss:])
    for m in kh.ADVANCE_MUTANTS:
        assert not np.array_equal(kh.advance_header_ref(st, hdr, ss, _LAY, 3, 5, mutant=m), out), m
    cb = kh.set_clip_base_ref(st)
    assert kh.get64(cb, kh.HDR_CLIP) == kh.get64(st, kh.HDR_POS) and np.array_equal(cb[6:], st[6:])


def test_reset_first_chunk_mutant_needs_a_second_chunk():
    import numpy as np
    lim = kh.state_limits()["RESET_MAX_SLOTS"]
    hdr, ss = 16, 264
    st = _state(hdr, ss, lim + 1, 3)
    slots = list(range(lim + 1))[::-1]
    ref = kh.reset_streams_ref(st, hdr, ss, _LAY, slots)
    assert np.array_equal(kh.reset_streams_ref(st, hdr, ss, _LAY, slots[:lim], mutant="first_chunk_only"),
                          kh.reset_streams_ref(st, hdr, ss, _LAY, slots[:lim]))
    assert not np.array_equal(kh.reset_streams_ref(st, hdr, ss, _LAY, slots, mutant="first_chunk_only"), ref)


def test_join_start_reference_and_mutants():
    """join_start_ref against the rule written out per row, on every case of the GPU test; each mutant differs on the
    cases that name it, and every mutant is named"""
    named = set()
    for w_max in (0, 1, 50):
        c = kh.join_start_case(w_max)
        recs, leads, batch = c["records"], c["leads"], c["batch"]
        ref = kh.join_start_ref(recs, leads, c["clocks"], batch, w_max)
        for j, (s, l) in enumerate(zip(recs, leads)):
            live = recs.count(s) == 1 and s not in leads and 0 <= s < batch and 0 <= l < batch
            W = min(w_max, c["clocks"][l]) if live else 0
            assert (ref["rec"][j], ref["used"][j], ref["owner"][j]) == ((s, W, j) if live else (-1, 0, -1)), (w_max, j)
            if live:
                assert ref["start"][s] == c["clocks"][l] - W
        assert sum(r >= 0 for r in ref["rec"]) == 12
        for m in c["catches"]:
            assert kh.join_start_ref(recs, leads, c["clocks"], batch, w_max, mutant=m) != ref, (w_max, m)
        named |= c["catches"]
    assert named == set(kh.JOIN_MUTANTS)


def test_history_references_and_mutants():
    """history_put_ref writes listener i's frame t to slot (clock + t) mod F for its last min(h, F) frames;
    history_get_ref reads them back by the row's own clock.  A put of one frame per tick then a get equals the frames in
    order, and every mutant differs on the cases that name it."""
    import numpy as np
    named_put, named_get = set(), set()
    for F in kh.HIST_F:
        c = kh.history_put_case(F)
        T, batch = c["T"], c["batch"]
        X0 = np.arange(len(c["leads"]) * T, dtype=np.int32).reshape(len(c["leads"]), T, 1) + 1
        hist = np.zeros((batch, F, 1), dtype=np.int32)
        ref = kh.history_put_ref(hist, X0, c["leads"], c["hops"], c["clocks"], F, T, batch)
        for i, l in enumerate(c["leads"]):
            h = kh.row_frames(c["hops"], i, T)
            if 0 <= l < batch and h > 0:
                for t in range(max(0, h - F), h):
                    assert ref[l, (c["clocks"][l] + t) % F, 0] == X0[i, t, 0]
        for m in c["catches"]:
            assert not np.array_equal(kh.history_put_ref(hist, X0, c["leads"], c["hops"], c["clocks"], F, T, batch, m), ref), (F, m)
        named_put |= c["catches"]
        g = kh.history_get_case(F)
        H = np.arange(g["batch"] * F, dtype=np.int32).reshape(g["batch"], F, 1) + 1
        got = kh.history_get_ref(H, g["rec"], g["used"], g["leads"], g["clocks"], F, g["T"], g["batch"])
        for j, s in enumerate(g["rec"]):
            h = kh.row_frames(g["used"], j, g["T"])
            for t in range(g["T"]):
                live = 0 <= s < g["batch"] and t < h
                assert got[j, t, 0] == (H[g["leads"][j], (g["clocks"][s] + t) % F, 0] if live else 0), (F, j, t)
        for m in g["catches"]:
            assert not np.array_equal(kh.history_get_ref(H, g["rec"], g["used"], g["leads"], g["clocks"], F, g["T"], g["batch"],
                                                         m), got), (F, m)
        named_get |= g["catches"]
    assert named_put == set(kh.HIST_PUT_MUTANTS) and named_get == set(kh.HIST_GET_MUTANTS)
    # round trip: ticks of one frame starting at 2^32 - 4 put into a ring of 7, then read back from clock p - W
    F, p0, n = 7, 2 ** 32 - 4, 10
    hist = np.zeros((1, F, 1), dtype=np.int32)
    for k in range(n):
        hist = kh.history_put_ref(hist, np.full((1, 1, 1), 100 + k, dtype=np.int32), [0], None, [p0 + k], F, 1, 1)
    W = 5
    back = kh.history_get_ref(hist, [0], [W], [0], [p0 + n - W], F, W, 1)
    assert back[0, :, 0].tolist() == [100 + k for k in range(n - W, n)]


def test_move_lead_reference_and_mutants():
    import numpy as np
    lay = dict(_LAY, ST_BLK=320, BK_STRIDE=20, ST_CONV=264)
    hdr, ss, nb = 16, 320 + 3 * 20, 3
    st = _state(hdr, ss, 4, 4)
    for b, calls in enumerate((2, 5, 7, 4)):
        st[hdr + b * ss + lay["ST_CALLS"]] = calls
    for src, dst in ((0, 1), (1, 3), (2, 0), (1, 2)):
        ref = kh.move_lead_ref(st, hdr, ss, lay, nb, [src], [dst], conv_parity=8)
        exp = st.copy()
        a, b = hdr + src * ss, hdr + dst * ss
        exp[b + 320:b + 340] = st[a + 320:a + 340]
        pa, pb = st[a + lay["ST_CALLS"]] & 1, st[b + lay["ST_CALLS"]] & 1
        exp[b + 264 + 8 * pb:b + 272 + 8 * pb] = st[a + 264 + 8 * pa:a + 272 + 8 * pa]
        assert np.array_equal(ref, exp), (src, dst)
        assert not np.array_equal(kh.move_lead_ref(st, hdr, ss, lay, nb, [src], [dst], mutant="all_blocks", conv_parity=8), ref)
        assert np.array_equal(kh.move_lead_ref(st, hdr, ss, lay, nb, [src], [dst], mutant="src_parity", conv_parity=8), ref) == (pa == pb)


def test_eslot_rows_reference_and_mutants():
    lim = kh.state_limits()
    named = set()
    for n in (1, lim["SLOT_ROWS_PER_LAUNCH"], lim["SLOT_ROWS_PER_LAUNCH"] + 1):
        for device in (False, True):
            c = kh.eslot_rows_case(n, device, lim["SLOT_ROWS_PER_LAUNCH"])
            args = (c["slots"], c["lens"], c["captured"], c["n_slots"], c["capacity"], lim["MIN_SAMPLES"])
            ref = kh.eslot_rows_ref(*args)
            for i, (s, ln) in enumerate(zip(c["slots"], c["lens"])):
                cap = min(max(c["captured"][s], 0), c["capacity"]) if 0 <= s < c["n_slots"] else 0
                u = min(ln, cap)
                use = u if u >= lim["MIN_SAMPLES"] else 0
                assert (ref["slots"][i], ref["lens"][i], ref["used"][i]) == \
                    (s if 0 <= s < c["n_slots"] else 0, use or lim["MIN_SAMPLES"], use)
            assert device or all(0 <= s < c["n_slots"] for s in c["slots"])
            for m in c["catches"]:
                assert kh.eslot_rows_ref(*args, mutant=m) != ref, (n, device, m)
            named |= c["catches"]
    assert named == set(kh.SLOT_ROWS_MUTANTS)
    import numpy as np
    dst = np.zeros(3 * 300, dtype=np.int32)
    src = np.arange(3 * 256, dtype=np.int32).reshape(3, 256) + 1
    out = kh.eput_rows_ref(dst, src, [5, 0, 192], 300)
    assert out[:256].tolist() == src[0].tolist() and not out[300:900 - 44 - 256].any() and out[600:856].tolist() == src[2].tolist()
    assert not np.array_equal(kh.eput_rows_ref(dst, src, [5, 0, 192], 300, mutant="dead_written"), out)


def test_ring_utterance_is_the_last_samples_written():
    """Write samples 1, 2, ... into a ring one at a time, as the capture does: the utterance of the last n samples is
    n consecutive values ending at the last one written, whatever the write position; the unwrapped mutant differs exactly
    when the utterance wraps"""
    import numpy as np
    for cap in (192, 1000):
        for total in (cap - 1, cap, cap + 37, 3 * cap + 5):
            rings = np.zeros((2, cap), dtype=np.int64)
            for k in range(1, total + 1):
                rings[0, (k - 1) % cap], rings[1, (k - 1) % cap] = k, -k
            wpos = total % cap
            for n in (192, cap // 2 + 1, min(cap, total)):
                if n > min(cap, total):
                    continue
                u = kh.ring_utterance(rings, wpos, n, cap)
                assert u[0].tolist() == list(range(total - n + 1, total + 1)) and u[1].tolist() == [-v for v in u[0]]
                assert np.array_equal(kh.ring_utterance(rings, wpos, n, cap, mutant="no_wrap"), u) == (wpos >= n)
    for c in kh.ring_cases(192):
        assert any(w < n for w, n, live in c["rows"] if live), c["name"]
