"""Vector-quantised feature fields: csrc/vq.cu (f3dgs_vq_assign, _plan, _update, _codebook_grad, _decode,
_decode_f16out), codebook.kmeans / decode / CodePlan, GaussianState.quantize_features and the compressed PLY layout.

The yardstick is tests/ref_vq.py: numpy float64 distances and Lloyd iterations.  The assignment is checked against the
error bound the header states, the segment means and sums within 1 float32 ulp of float64, decode bitwise."""
import ctypes
import os
import tempfile

import numpy as np
import pytest
import torch

import ref_vq as ref

INT_MAX = 2**31 - 1


# ---------------------------------------------------------------------------------------------------- C ABI (CPU)
@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    p, i = ctypes.c_void_p, ctypes.c_int
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_launch_count.restype = ctypes.c_ulonglong
    L.f3dgs_vq_scratch_bytes.restype = ctypes.c_size_t
    L.f3dgs_vq_scratch_bytes.argtypes = [i, i]
    L.f3dgs_vq_assign.argtypes = [i, i, i, p, p, p, p]
    L.f3dgs_vq_plan.argtypes = [i, i, p, p, p]
    L.f3dgs_vq_update.argtypes = [i, i, i, p, p, p, p, p]
    L.f3dgs_vq_codebook_grad.argtypes = [i, i, i, p, p, p, p]
    L.f3dgs_vq_decode.argtypes = [i, i, i, p, p, p, p]
    L.f3dgs_vq_decode_f16out.argtypes = [i, i, i, p, p, p, p]
    return L


def _rejected(lib, name, call, msg):
    """call() is rejected with `name: ...msg...`, also right after another entry point failed"""
    lib.f3dgs_vq_decode(-1, 1, 1, None, None, None, None)
    assert call() == -1
    err = lib.f3dgs_last_error()
    assert err.startswith(name + b": ") and msg in err, (name, err)


BAD_SIZES = [(-1, 4, 8), (10, 0, 8), (10, 65537, 8), (10, 4, 0), (10, 4, 4097)]


def test_cabi_rejects_bad_arguments_before_touching_cuda(lib):
    n0 = lib.f3dgs_launch_count()
    P, K, D = 10, 4, 8
    x, c, code, scr, w, out = 0x1000000, 0x2000000, 0x3000000, 0x4000000, 0x5000000, 0x6000000

    fn, name = lib.f3dgs_vq_assign, b"f3dgs_vq_assign"
    for s in BAD_SIZES:
        _rejected(lib, name, lambda: fn(*s, x, c, code, None), b"bad sizes")
    for k in range(3):
        a = [x, c, code]
        a[k] = None
        _rejected(lib, name, lambda: fn(P, K, D, *a, None), b"NULL")
    for a in ([x, c, x + 4 * D * 3], [x, c, c + 8], [x, c, x - 16]):
        _rejected(lib, name, lambda: fn(P, K, D, *a, None), b"overlap")
    assert fn(0, K, D, None, None, None, None) == 0

    fn, name = lib.f3dgs_vq_plan, b"f3dgs_vq_plan"
    for s in ((-1, 4), (10, 0), (10, 65537)):
        _rejected(lib, name, lambda: fn(*s, code, scr, None), b"bad sizes")
    _rejected(lib, name, lambda: fn(P, K, None, scr, None), b"NULL")
    _rejected(lib, name, lambda: fn(P, K, code, None, None), b"NULL")
    _rejected(lib, name, lambda: fn(P, K, scr + 300, scr, None), b"overlap")
    _rejected(lib, name, lambda: fn(P, K, code, code - 256, None), b"overlap")
    assert fn(0, K, None, None, None) == 0

    fn, name = lib.f3dgs_vq_update, b"f3dgs_vq_update"
    for s in BAD_SIZES:
        _rejected(lib, name, lambda: fn(*s, x, w, scr, c, None), b"bad sizes")
    for k in (0, 2, 3):  # weights may be NULL
        a = [x, w, scr, c]
        a[k] = None
        _rejected(lib, name, lambda: fn(P, K, D, *a, None), b"NULL")
    for a in ([x, w, scr, x + 64], [x, w, scr, w - 4], [x, w, scr, scr + 256], [x, c + 4, scr, c]):
        _rejected(lib, name, lambda: fn(P, K, D, *a, None), b"overlap")
    assert fn(0, K, D, None, None, None, None, None) == 0

    fn, name = lib.f3dgs_vq_codebook_grad, b"f3dgs_vq_codebook_grad"
    for s in BAD_SIZES:
        _rejected(lib, name, lambda: fn(*s, x, scr, out, None), b"bad sizes")
    for k in range(3):
        a = [x, scr, out]
        a[k] = None
        _rejected(lib, name, lambda: fn(P, K, D, *a, None), b"NULL")
    for a in ([x, scr, x + 4], [x, scr, scr + 1000]):
        _rejected(lib, name, lambda: fn(P, K, D, *a, None), b"overlap")
    assert fn(0, K, D, None, None, None, None) == 0

    for fn, name, es in ((lib.f3dgs_vq_decode, b"f3dgs_vq_decode", 4), (lib.f3dgs_vq_decode_f16out,
                                                                          b"f3dgs_vq_decode_f16out", 2)):
        for s in BAD_SIZES:
            _rejected(lib, name, lambda: fn(*s, c, code, out, None), b"bad sizes")
        for k in range(3):
            a = [c, code, out]
            a[k] = None
            _rejected(lib, name, lambda: fn(P, K, D, *a, None), b"NULL")
        for a in ([c, code, c + 4 * D], [c, code, code - es * D * P + 4]):
            _rejected(lib, name, lambda: fn(P, K, D, *a, None), b"overlap")
        assert fn(0, K, D, None, None, None, None) == 0

    assert lib.f3dgs_vq_scratch_bytes(0, 4) == 0 and lib.f3dgs_vq_scratch_bytes(-3, 4) == 0
    assert lib.f3dgs_vq_scratch_bytes(10, 0) == 0 and lib.f3dgs_vq_scratch_bytes(10, 65537) == 0
    assert lib.f3dgs_launch_count() == n0  # nothing was launched


def test_header_states_the_assignment_bound():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    h = open(os.path.join(root, "include", "f3dgs_b200.h")).read()
    assert "(4 (2u + u^2) + 4 g (1 + u)^2) ||x|| cmax + 2 g cmax^2" in h and "g = (D + 8) 2^-22" in h
    # the leading term is 2^-8 + 2^-20, the issue's 2^-8 ||x|| max ||c|| plus the square of the rounding
    u = 2.0 ** -11
    assert 4 * (2 * u + u * u) == 2.0 ** -8 + 2.0 ** -20


# ---------------------------------------------------------------------------------------------------- PLY (CPU)
def _ply_fields(P, rng):
    return (rng.standard_normal((P, 3)), rng.standard_normal((P, 1, 3)), rng.standard_normal((P, 15, 3)),
            rng.standard_normal((P, 1)), rng.standard_normal((P, 3)), rng.standard_normal((P, 4)))


@pytest.mark.parametrize("P,K,C", [(301, 17, 16), (50, 1, 1), (40, 65536, 2), (2, 3, 4)])
def test_ply_compressed_round_trip(P, K, C):
    from diff_gaussian_rasterization import io as ply

    rng = np.random.default_rng(P + K + C)
    fields = _ply_fields(P, rng)
    book = rng.standard_normal((K, C)).astype(np.float32)
    book[0, 0] = -0.0
    code = rng.integers(0, K, P).astype(np.int32)
    if P:
        code[-1] = K - 1
    with tempfile.TemporaryDirectory() as d:
        full, comp = os.path.join(d, "full.ply"), os.path.join(d, "comp.ply")
        ply.save_ply(full, *fields, book[code][:, None, :])
        ply.save_ply(comp, *fields, None, semantic_codebook=torch.from_numpy(book), semantic_code=torch.from_numpy(code))
        a, b = ply.load_ply(full), ply.load_ply(comp)
        # the data: 4 C - 2 bytes less per vertex, 4 K C more; the header: two more lines
        extra_header = len("property ushort semantic_code\n") + len(f"element semantic_codebook {K}\n")
        assert os.path.getsize(full) - os.path.getsize(comp) == P * (4 * C - 2) - 4 * K * C - extra_header
    assert "semantic_codebook" not in a and "semantic_code" not in a
    assert b["semantic_codebook"].dtype == np.float32 and b["semantic_code"].dtype == np.int32
    assert b["semantic_codebook"].tobytes() == book.tobytes() and np.array_equal(b["semantic_code"], code)
    assert b["semantic_feature"].shape == (P, 1, C)
    assert b["semantic_feature"].tobytes() == book[code][:, None, :].tobytes()
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k


def test_ply_rejects_inconsistent_codebooks():
    from diff_gaussian_rasterization import io as ply

    rng = np.random.default_rng(0)
    fields = _ply_fields(5, rng)
    book = np.zeros((3, 2), np.float32)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "x.ply")
        with pytest.raises(ValueError):
            ply.save_ply(path, *fields, None, semantic_codebook=book)
        with pytest.raises(ValueError):
            ply.save_ply(path, *fields, None, semantic_codebook=book, semantic_code=np.array([0, 1, 2, 3, 0]))
        with pytest.raises(ValueError):
            ply.save_ply(path, *fields, None, semantic_codebook=book, semantic_code=np.zeros(4, np.int32))


# ---------------------------------------------------------------------------------------------------- GPU helpers
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bits(t):
    return t.detach().contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16).cpu()


def _ulp32(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


# ---------------------------------------------------------------------------------------------------- assign
@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 3, 128, 512, 4096])
def test_assign_within_the_stated_bound(D):
    from diff_gaussian_rasterization import codebook as vq

    P, K = (3001, 301) if D <= 512 else (701, 133)
    g = _gen(D)
    x = torch.randn(P, D, device="cuda", generator=g)
    c = torch.randn(K, D, device="cuda", generator=g) * 0.7
    code = vq.assign(x, c)
    xn, cn, kn = x.cpu().numpy(), c.cpu().numpy(), code.cpu().numpy()
    assert kn.dtype == np.int32 and kn.min() >= 0 and kn.max() < K
    d = ref.distances(xn, cn)
    gap = d[np.arange(P), kn] - d.min(1)
    bound = ref.assign_bound(xn, cn)
    assert (gap <= bound).all(), float((gap / bound).max())
    if D > 1:  # the rounding decides only near-ties (at D = 1 the 301 codes are packed too densely for this)
        assert (kn == ref.assign(xn, cn)).mean() > 0.9
    assert torch.equal(vq.assign(x, c), code)  # bitwise reproducible


@pytest.mark.gpu
def test_assign_ties_go_to_the_lower_index_and_nan_rows_to_code_0():
    from diff_gaussian_rasterization import codebook as vq

    P, K, D = 2000, 200, 64
    g = _gen(1)
    c = torch.randn(K, D, device="cuda", generator=g)
    dup = torch.arange(100, 200, device="cuda")
    c[dup] = c[dup - 100]  # rows 100.. duplicate rows 0..
    x = c[torch.randint(0, K, (P,), device="cuda", generator=g)] + 0.01 * torch.randn(P, D, device="cuda", generator=g)
    x[7] = float("nan")
    code = vq.assign(x, c)
    assert int(code.max()) < 100
    assert int(code[7]) == 0
    exact = ref.assign(x[:7].cpu().numpy(), c.cpu().numpy())
    assert np.array_equal(code[:7].cpu().numpy(), exact)


# ---------------------------------------------------------------------------------------------------- update / grad
def _codes(P, K, seed, empty=()):
    g = _gen(seed)
    code = torch.randint(0, K, (P,), device="cuda", generator=g, dtype=torch.int32)
    for k in empty:
        code[code == k] = (k + 1) % K
    return code


@pytest.mark.gpu
@pytest.mark.parametrize("P,K,D,weighted", [(5000, 37, 3, True), (100_003, 1000, 128, False),
                                            (20_011, 4096, 1, True), (3000, 7, 513, True)])
def test_update_and_grad_match_float64(P, K, D, weighted):
    from diff_gaussian_rasterization.codebook import CodePlan

    g = _gen(P)
    x = torch.randn(P, D, device="cuda", generator=g) * 3 + 1
    w = torch.rand(P, device="cuda", generator=g) if weighted else None
    code = _codes(P, K, P + 1, empty=(0, K // 2))
    c0 = torch.randn(K, D, device="cuda", generator=g)
    plan = CodePlan(code, K)
    c = plan.update(c0.clone(), x, w)
    xn, kn = x.cpu().numpy(), code.cpu().numpy().astype(np.int64)
    wn = None if w is None else w.cpu().numpy()
    s, sw = ref.segment_sum(xn, kn, K, wn)
    mean = ref.update(c0.cpu().numpy(), xn, kn, wn)
    got = c.cpu().numpy().astype(np.float64)
    nz = sw > 0
    assert np.all(np.abs(got - mean)[nz] <= _ulp32(mean)[nz])
    assert not nz[0] and not nz[K // 2]
    assert torch.equal(_bits(c[~torch.from_numpy(nz).cuda()]), _bits(c0[~torch.from_numpy(nz).cuda()]))
    dx = torch.randn(P, D, device="cuda", generator=g)
    gr = plan.grad(dx)
    gs, _ = ref.segment_sum(dx.cpu().numpy(), kn, K)
    assert np.all(np.abs(gr.cpu().numpy().astype(np.float64) - gs) <= _ulp32(gs))
    assert np.all(gr.cpu().numpy()[~nz] == 0)
    # bitwise reproducible, a second plan included
    assert torch.equal(_bits(CodePlan(code, K).update(c0.clone(), x, w)), _bits(c))
    assert torch.equal(_bits(plan.grad(dx)), _bits(gr))


@pytest.mark.gpu
def test_every_row_in_one_code():
    from diff_gaussian_rasterization.codebook import CodePlan

    P, K, D = 1_000_003, 5, 64
    g = _gen(3)
    x = torch.randn(P, D, device="cuda", generator=g)
    code = torch.full((P,), 3, dtype=torch.int32, device="cuda")
    plan = CodePlan(code, K)
    c0 = torch.randn(K, D, device="cuda", generator=g)
    c = plan.update(c0.clone(), x)
    gr = plan.grad(x)
    torch.cuda.synchronize()
    x64 = x.double()
    s = x64.sum(0)
    assert torch.all((c[3].double() - s / P).abs() <= torch.from_numpy(_ulp32((s / P).cpu().numpy())).cuda())
    assert torch.all((gr[3].double() - s).abs() <= torch.from_numpy(_ulp32(s.cpu().numpy())).cuda())
    keep = torch.tensor([0, 1, 2, 4], device="cuda")
    assert torch.equal(_bits(c[keep]), _bits(c0[keep])) and bool((gr[keep] == 0).all())


@pytest.mark.gpu
def test_out_of_range_codes_and_bad_weights_write_nothing(built):
    from diff_gaussian_rasterization import _C
    from diff_gaussian_rasterization.codebook import CodePlan

    L = ctypes.CDLL(built)
    L.f3dgs_vq_codebook_grad.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 4
    P, K, D = 4000, 16, 8
    g = _gen(5)
    x = torch.randn(P, D, device="cuda", generator=g)
    c0 = torch.randn(K, D, device="cuda", generator=g)
    for bad in (K, -1):
        code = _codes(P, K, 6)
        code[1234] = bad
        plan = CodePlan(code, K)
        c = plan.update(c0.clone(), x)
        out = torch.full((K, D), 7.0, device="cuda")
        torch.cuda.synchronize()
        assert L.f3dgs_vq_codebook_grad(P, K, D, x.data_ptr(), plan.scratch.data_ptr(), out.data_ptr(), None) == 0
        torch.cuda.synchronize()
        assert torch.equal(_bits(c), _bits(c0)) and bool((out == 7.0).all())
    plan = CodePlan(_codes(P, K, 7), K)
    for v in (float("nan"), float("inf"), -1.0):
        w = torch.ones(P, device="cuda")
        w[99] = v
        c = c0.clone()
        _C.vq_update(x, w, plan.scratch, c)  # past the Python check: the device check refuses
        assert torch.equal(_bits(c), _bits(c0))
    assert not torch.equal(_bits(plan.update(c0.clone(), x, torch.ones(P, device="cuda"))), _bits(c0))


# ---------------------------------------------------------------------------------------------------- decode
@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 3, 8, 12, 128, 4096])
def test_decode_is_the_gather_bitwise(D):
    from diff_gaussian_rasterization import codebook as vq

    P, K = 10_007, 97
    g = _gen(D)
    c = torch.randn(K, D, device="cuda", generator=g) * 1000
    c[0, 0] = 65520.0  # rounds to inf in float16
    c[1, 0] = 2.0 ** -25  # rounds to the even zero
    code = torch.randint(0, K, (P,), device="cuda", generator=g, dtype=torch.int32)
    assert torch.equal(_bits(vq.decode(c, code)), _bits(c[code.long()]))
    assert torch.equal(_bits(vq.decode(c, code, torch.float16)), _bits(c.half()[code.long()]))
    out = torch.empty(P, D, device="cuda", dtype=torch.float16)
    assert vq.decode(c, code, torch.float16, out=out).data_ptr() == out.data_ptr()
    assert torch.equal(_bits(out), _bits(c.half()[code.long()]))


# ---------------------------------------------------------------------------------------------------- kmeans
def _blobs(P, K, D, seed, first):
    """K well-separated blobs; row first[j] (kmeans' initial pick j) lies in blob j, so each code starts in its own blob
    and no row is near a tie"""
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((K, D)) * 20
    lab = rng.integers(0, K, P)
    lab[first] = np.arange(K)
    return (centres[lab] + rng.standard_normal((P, D))).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("weighted", [False, True])
def test_kmeans_matches_lloyd_on_blobs(weighted):
    from diff_gaussian_rasterization import kmeans

    P, K, D, iters = 20_000, 24, 16, 6
    first = torch.randperm(P, generator=torch.Generator().manual_seed(4))[:K].numpy()
    xn = _blobs(P, K, D, 0, first)
    x = torch.from_numpy(xn).cuda()
    w = torch.rand(P, device="cuda", generator=_gen(1)) + 0.5 if weighted else None
    cb, code = kmeans(x, K, iters=iters, weights=w, generator=torch.Generator().manual_seed(4))
    rc, rcode = ref.lloyd(xn, xn[first], iters, None if w is None else w.cpu().numpy())
    assert cb.shape == (K, D) and cb.dtype == torch.float32 and code.dtype == torch.int32
    assert np.array_equal(code.cpu().numpy(), rcode)
    assert np.allclose(cb.cpu().numpy(), rc, rtol=1e-5, atol=1e-5)
    cb2, code2 = kmeans(x, K, iters=iters, weights=w, generator=torch.Generator().manual_seed(4))
    assert torch.equal(_bits(cb2), _bits(cb)) and torch.equal(code2, code)
    cb3, _ = kmeans(x, K, iters=iters, weights=w, generator=torch.Generator().manual_seed(5))
    assert not torch.equal(cb3, cb)


@pytest.mark.gpu
def test_kmeans_rejects_bad_arguments():
    from diff_gaussian_rasterization import kmeans

    x = torch.randn(10, 4, device="cuda")
    with pytest.raises(ValueError):
        kmeans(x, 11)
    with pytest.raises(ValueError):
        kmeans(x, 0)
    with pytest.raises(ValueError):
        kmeans(x, 3, weights=torch.full((10,), float("nan"), device="cuda"))
    with pytest.raises(ValueError):
        kmeans(x, 3, weights=-torch.ones(10, device="cuda"))
    with pytest.raises(ValueError):
        kmeans(x.double(), 3)


# ---------------------------------------------------------------------------------------------------- GaussianState
def _state(sc, feature_dtype=torch.float32):
    import scenegen
    from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid

    t = scenegen.to_torch(sc, "cuda")
    return GaussianState(t["means3D"].clone(), t["shs"][:, :1].contiguous(), t["shs"][:, 1:].contiguous(),
                         inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                         t["rotations"].clone(), t["semantic_feature"].clone(), feature_dtype=feature_dtype)


def _settings(sc, cam):
    import scenegen
    from diff_gaussian_rasterization import GaussianRasterizationSettings

    return GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, "cuda"))


def _render(rs, a, features):
    from diff_gaussian_rasterization import GaussianRasterizer

    means2D = torch.zeros_like(a["means3D"], requires_grad=True)
    return GaussianRasterizer(rs)(means3D=a["means3D"], means2D=means2D, opacities=a["opacities"], shs=a["shs"],
                                  semantic_feature=features, scales=a["scales"], rotations=a["rotations"])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["f32", "f16"])
def test_quantized_state_renders_the_decoded_field(dtype):
    import scenegen

    sc = scenegen.make_config("small128", views=1)
    st = _state(sc, dtype)
    P, C = st.P, sc.C
    rep = st.quantize_features(64, iters=4, generator=torch.Generator().manual_seed(0))
    assert st.codebook.shape == (64, C) and st.code.shape == (P,) and st.code.dtype == torch.int32
    assert st.raw["semantic_feature"].numel() == 0 and st.exp_avg["semantic_feature"].numel() == 0
    assert rep["after"] < rep["before"]
    a = st.activate()
    assert a["semantic_feature"].dtype == dtype and a["semantic_feature"].shape == (P, 1, C)
    rs = _settings(sc, sc.cameras[0])
    feat = st.codebook[st.code.long()].reshape(P, 1, C)
    _, f_state, _, _ = _render(rs, a, a["semantic_feature"])
    _, f_ref, _, _ = _render(rs, a, feat.to(dtype))
    assert f_state.dtype == dtype and torch.equal(_bits(f_state), _bits(f_ref))


LRS = dict(xyz=0.0, f_dc=0.0, f_rest=0.0, opacity=0.0, scaling=0.0, rotation=0.0, semantic_feature=0.05)


@pytest.mark.gpu
def test_quantized_fine_tuning_matches_autograd():
    """Five steps of ViewBatch forward, feature L1, backward, all_reduce and step() on the codebook, against
    codebook.requires_grad_(), features codebook[code] through the rasterizer and torch.optim.Adam(eps=1e-15)."""
    import scenegen

    sc = scenegen.make_config("small", views=2)
    st = _state(sc)
    st.quantize_features(32, iters=3, generator=torch.Generator().manual_seed(1))
    P, C = st.P, sc.C
    book = st.codebook.clone().requires_grad_(True)
    code = st.code.long()
    opt = torch.optim.Adam([book], lr=LRS["semantic_feature"], eps=1e-15)
    rs = [_settings(sc, cam) for cam in sc.cameras]
    g = _gen(11)
    H, W = sc.cameras[0].image_height, sc.cameras[0].image_width
    tg = [torch.rand(C, H, W, device="cuda", generator=g) for _ in rs]
    fixed = {k: v.clone() for k, v in st.activate().items() if k != "semantic_feature"}
    for step in range(5):
        st.activate()
        vb = st.batch()
        vb.zero_()
        for v, r in enumerate(rs):
            color, feat, radii, depth, ctx = vb.forward(r)
            vb.backward(ctx, torch.zeros_like(color), torch.sign(feat - tg[v]) / feat.numel(), torch.zeros_like(depth),
                        last=v == len(rs) - 1)
        vb.all_reduce()
        st.step(LRS)

        opt.zero_grad()
        loss = 0.0
        for v, r in enumerate(rs):
            _, feat, _, _ = _render(r, fixed, book[code].reshape(P, 1, C))
            loss = loss + (feat - tg[v]).abs().mean()
        loss.backward()
        opt.step()
        err = (st.codebook - book.detach()).abs()
        assert float(err.max()) <= 8 * LRS["semantic_feature"] * (step + 1) + 1e-6, (step, float(err.max()))
        close = torch.isclose(st.codebook, book.detach(), rtol=1e-4, atol=1e-6)
        assert float((~close).float().mean()) <= 2e-3, (step, float((~close).float().mean()))
    for k, v in fixed.items():  # lr 0: nothing else moved
        assert torch.equal(st.act[k], v), k


@pytest.mark.gpu
def test_quantized_prune_densify_relocate_and_dequantize():
    import scenegen
    from diff_gaussian_rasterization import GaussianScores  # noqa: F401  (exported next to kmeans)

    sc = scenegen.make_config("small", views=1)
    st = _state(sc)
    st.quantize_features(16, iters=2, generator=torch.Generator().manual_seed(2))
    P = st.P
    code0, book = st.code.clone(), st.codebook.clone()
    keep = torch.rand(P, device="cuda", generator=_gen(3)) > 0.3
    assert st.prune(keep) == int(keep.sum())
    assert torch.equal(st.code, code0[keep])
    a = st.activate()
    assert torch.equal(_bits(a["semantic_feature"].reshape(st.P, -1)), _bits(book[st.code.long()]))
    with pytest.raises(ValueError):
        st.densify_and_prune(0.0002, 0.005, 1.0, 20)
    with pytest.raises(ValueError):
        st.relocate_and_add(st.P + 100)
    with pytest.raises(ValueError):
        st.quantize_features(8)
    st.dequantize()
    sf = st.raw["semantic_feature"]
    assert sf.shape == (st.P, 1, sc.C) and torch.equal(_bits(sf.reshape(st.P, -1)), _bits(book[code0[keep].long()]))
    assert st.code is None and st.codebook is None
    assert bool((st.exp_avg["semantic_feature"] == 0).all()) and st.steps["semantic_feature"] == 0
    with pytest.raises(ValueError):
        st.dequantize()
