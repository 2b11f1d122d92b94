"""Training float16 feature fields: float16 feature maps and scaled float16 map gradients through the feature loss, the
backward and Adam (f3dgs_backward[_accum]_f16, f3dgs_feature_resize_fwd_f16[_f16gt], f3dgs_feature_resize_bwd_f16,
f3dgs_adam_step_f16out; feature_head's grad_dtype / ScaledGrad, ViewBatch, GaussianState(feature_dtype=...)).

A float16 map gradient h with scale s stands for the float32 gradient s * float(h), so every float16 path has an exact
float32 twin: the backward against the float32 backward of h.float() * s (equal up to the order of its float atomics),
the resize forward bitwise against the float32 one of the upcast map, the resize backward bitwise against
(resize_bwd(dout) * out_scale).half(), and Adam's float16 copy bitwise against param.half().  The scale matters: at a
config-3-like ratio the L1 feature gradient is ~1.9e-8, and a plain float16 cast of it is all zeros.
CPU part (`-m "not gpu"`): every new symbol rejects bad arguments before any CUDA call.
"""
import ctypes

import numpy as np
import pytest
import torch

import parity
import scenegen

GEOM = ("means3D", "opacities", "shs", "scales", "rotations")
c_f, c_p, c_i, c_sz = ctypes.c_float, ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_launch_count.restype = ctypes.c_ulonglong
    fp = lambda k: [c_p] * k  # noqa: E731
    L.f3dgs_backward_f16.argtypes = ([c_i] * 5 + [c_p, c_i, c_i] + fp(5) + [c_f, c_p, c_p] + fp(3) + [c_f, c_f]
                                     + fp(5) + [c_p, c_f, c_p] + fp(11) + [c_i, c_p])
    L.f3dgs_backward_accum_f16.argtypes = ([c_i] * 5 + [c_p, c_i, c_i] + fp(4) + [c_f, c_p, c_p] + fp(3) + [c_f, c_f]
                                           + fp(5) + [c_p, c_f, c_p] + fp(12) + [c_p, c_i, c_p])
    L.f3dgs_feature_resize_fwd_f16.argtypes = [c_i] * 5 + [c_p, c_p, c_f, c_p, c_p, c_p]
    L.f3dgs_feature_resize_fwd_f16_f16gt.argtypes = [c_i] * 5 + [c_p, c_p, c_f, c_p, c_p, c_p]
    L.f3dgs_feature_resize_bwd_f16.argtypes = [c_i] * 5 + [c_p, c_f, c_p, c_p]
    L.f3dgs_adam_step_f16out.argtypes = [c_i, c_sz, c_i] + fp(5) + [c_f] * 4 + [c_i, c_p]
    return L


def _rejected(lib, fn, msg, *args):
    assert fn(*args) == -1, (fn.__name__, msg)
    err = lib.f3dgs_last_error()
    assert err.startswith(fn.__name__.encode() + b": ") and msg in err, (fn.__name__, msg, err)


# ---- CPU: C ABI validation (fake addresses, never dereferenced: every call below fails validation)
def test_half_training_symbols_reject_bad_arguments_before_touching_cuda(lib):
    launches = lib.f3dgs_launch_count()
    A = lambda k: k << 24  # noqa: E731  (distinct fake device addresses, 16 MiB apart)
    P, C, W, H = 10, 4, 64, 64
    nan, inf = float("nan"), float("inf")

    def bwd(P=P, C=C, W=W, H=H, geom=A(1), fpix=A(2), scale=1.0, dsf=A(3)):
        return (P, 1, 4, 100, C, A(4), W, H, A(5), A(6), None, None, A(7), 1.0, A(8), None, A(9), A(10), A(11),
                0.5, 0.5, None, geom, A(12), A(13), A(14), fpix, scale, A(15), A(16), A(17), A(18), A(19), dsf, A(20),
                A(21), A(22), A(23), A(24), A(25), 0, None)

    f = lib.f3dgs_backward_f16
    _rejected(lib, f, b"bad sizes", *bwd(P=-1))
    _rejected(lib, f, b"bad sizes", *bwd(C=4097))
    _rejected(lib, f, b"bad sizes", *bwd(W=0))
    _rejected(lib, f, b"missing forward buffers", *bwd(geom=None))
    _rejected(lib, f, b"NULL gradient pointer", *bwd(fpix=None))
    for s in (0.0, -0.0, nan, inf, -inf):
        _rejected(lib, f, b"dL_dfeaturepix_scale must be finite and nonzero", *bwd(scale=s))
    _rejected(lib, f, b"overlaps dL_dfeaturepix", *bwd(dsf=A(2) + C * W * H * 2 - 4))
    assert f(*bwd(P=0)) == 0

    def acc(P=P, C=C, scratch=A(30), fpix=A(2), scale=1.0, dsf=A(3)):
        return (P, 1, 4, 100, C, A(4), W, H, A(5), A(6), None, A(7), 1.0, A(8), None, A(9), A(10), A(11), 0.5, 0.5,
                None, A(12), A(13), A(14), A(15), fpix, scale, A(16), scratch, A(17), None, dsf, A(18), None, A(19),
                A(20), A(21), None, None, None, None, 0, None)

    f = lib.f3dgs_backward_accum_f16
    _rejected(lib, f, b"bad sizes", *acc(P=-1))
    _rejected(lib, f, b"bad sizes", *acc(C=-1))
    _rejected(lib, f, b"NULL scratch", *acc(scratch=None))
    _rejected(lib, f, b"NULL gradient pointer", *acc(fpix=None))
    for s in (0.0, nan, inf):
        _rejected(lib, f, b"dL_dfeaturepix_scale must be finite and nonzero", *acc(scale=s))
    _rejected(lib, f, b"overlaps dL_dfeaturepix", *acc(dsf=A(2) - P * C * 4 + 4))
    assert f(*acc(P=0)) == 0

    Hg, Wg = 28, 28
    for f, gt in ((lib.f3dgs_feature_resize_fwd_f16, None), (lib.f3dgs_feature_resize_fwd_f16_f16gt, A(3))):
        _rejected(lib, f, b"bad sizes", C, 0, W, Hg, Wg, A(1), gt, 1.0, A(2), None, None)
        _rejected(lib, f, b"bad sizes", -1, H, W, Hg, Wg, A(1), gt, 1.0, A(2), None, None)
        _rejected(lib, f, b"NULL pointer", C, H, W, Hg, Wg, None, gt, 1.0, A(2), None, None)
        _rejected(lib, f, b"NULL pointer", C, H, W, Hg, Wg, A(1), gt, 1.0, None, None, None)
        # a 2-byte map: out overlaps it only within C*H*W*2 bytes
        _rejected(lib, f, b"out overlaps feature_map", C, H, W, Hg, Wg, A(1), gt, 1.0, A(1) + C * H * W * 2 - 4, None,
                  None)
        assert f(0, H, W, Hg, Wg, None, None, 1.0, None, None, None) == 0
    f = lib.f3dgs_feature_resize_fwd_f16_f16gt
    _rejected(lib, f, b"gt is required", C, H, W, Hg, Wg, A(1), None, 1.0, A(2), None, None)
    _rejected(lib, f, b"out overlaps feature_map or gt", C, H, W, Hg, Wg, A(1), A(3), 1.0, A(3) + C * Hg * Wg * 2 - 4,
              None, None)

    f = lib.f3dgs_feature_resize_bwd_f16
    _rejected(lib, f, b"bad sizes", C, H, W, 0, Wg, A(1), 1.0, A(2), None)
    _rejected(lib, f, b"NULL pointer", C, H, W, Hg, Wg, None, 1.0, A(2), None)
    _rejected(lib, f, b"NULL pointer", C, H, W, Hg, Wg, A(1), 1.0, None, None)
    for s in (0.0, nan, inf):
        _rejected(lib, f, b"out_scale must be finite and nonzero", C, H, W, Hg, Wg, A(1), s, A(2), None)
    _rejected(lib, f, b"overlaps dout", C, H, W, Hg, Wg, A(1), 1.0, A(1) - C * H * W * 2 + 2, None)
    assert f(0, H, W, Hg, Wg, None, 1.0, None, None) == 0

    f = lib.f3dgs_adam_step_f16out
    n = 1000
    for kind in (1, 2, 3, 4, 5, 6, -1):  # every kind but F3DGS_PARAM_IDENTITY
        _rejected(lib, f, b"kind must be F3DGS_PARAM_IDENTITY", kind, n, 1, A(1), A(2), A(3), A(4), A(5), 1e-3, 0.9,
                  0.999, 1e-15, 1, None)
    _rejected(lib, f, b"step < 1", 0, n, 1, A(1), A(2), A(3), A(4), A(5), 1e-3, 0.9, 0.999, 1e-15, 0, None)
    for k in range(5):
        ptrs = [A(1), A(2), A(3), A(4), A(5)]
        ptrs[k] = None
        _rejected(lib, f, b"NULL pointer", 0, n, 1, *ptrs, 1e-3, 0.9, 0.999, 1e-15, 1, None)
    for k in range(4):  # param_f16 overlapping each float32 buffer in turn
        _rejected(lib, f, b"param_f16 overlaps", 0, n, 1, A(1), A(2), A(3), A(4), A(k + 1) + n * 4 - 2, 1e-3, 0.9,
                  0.999, 1e-15, 1, None)
    assert f(0, 0, 1, A(1), A(2), A(3), A(4), A(5), 1e-3, 0.9, 0.999, 1e-15, 1, None) == 0
    assert lib.f3dgs_launch_count() == launches


# =================================================================================================== GPU
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bits(x):
    return x.view(torch.int16) if x.dtype == torch.float16 else x.view(torch.int32)


def _viol(a, b, extra=None):
    """Worst |a - b| over the gradient tolerance of the parity bar (+ `extra`), <= 1 passes (as test_half_features)."""
    a, b = a.double(), b.double()
    tol = parity.RTOL * b.abs() + parity.GRAD_ATOL_REL * b.abs().max() + 1e-30
    if extra is not None:
        tol = tol + extra
    return float(((a - b).abs() / tol).max())


def _half_ulp(x):
    """Half a float16 ulp at |x| (subnormal spacing below 2^-14)."""
    e = torch.floor(torch.log2(x.double().abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 11)


def _scene(name, C):
    if name == "small513":
        sc = scenegen.make_scene(P=3000, W=150, H=100, C=0, sh_degree=1, seed=5)
    else:
        sc = scenegen.make_config(name)
    t = scenegen.to_torch(sc, "cuda")
    t["semantic_feature"] = torch.randn(sc.P, 1, C, device="cuda", generator=_gen(C))
    return sc, t


def _settings(sc):
    from diff_gaussian_rasterization import GaussianRasterizationSettings

    return GaussianRasterizationSettings(**parity.settings(sc, sc.cameras[0], "cuda"))


def _accum(t, rs, gc, gf, gd, **kw):
    """One ViewBatch forward + accumulating backward; -> the flat buffer's gradients and statistics."""
    from diff_gaussian_rasterization.parallel import ViewBatch

    vb = ViewBatch({k: t[k] for k in ("means3D", "scales", "rotations", "opacities", "shs", "semantic_feature")})
    vb.zero_()
    _, _, _, _, ctx = vb.forward(rs)
    vb.backward(ctx, gc, gf, gd, **kw)
    out = {k: v.clone() for k, v in vb.grads.items()}
    out["grad_accum"], out["denom"] = vb.grad_accum.clone(), vb.denom.clone()
    return out


def _check_bwd(g16, g32, label):
    v = _viol(g16["semantic_feature"], g32["semantic_feature"])
    worst = {k: _viol(g16[k], g32[k]) for k in GEOM + ("grad_accum",)}
    print(f"[{label}] dL/dfeature viol {v:.3g}; " + ", ".join(f"{k}={x:.3g}" for k, x in worst.items()))
    assert float(g32["semantic_feature"].abs().max()) > 0
    assert v <= 1.0
    for k, x in worst.items():
        assert x <= 1.0, (k, x)
    assert torch.equal(g16["denom"], g32["denom"])


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["aligned", "odd_offset"])
@pytest.mark.parametrize("s", [2.0 ** -20, 3e-8])
@pytest.mark.parametrize("name,C", [("small", 16), ("small128", 128), ("small200", 200), ("small513", 513)])
def test_accum_backward_f16_is_the_float_backward_of_the_scaled_map(name, C, s, layout):
    """small/small128: W % 4 == 0 (8-byte loads); small200/small513: W = 150 (scalar loads); odd_offset: the map one
    element into its storage (scalar loads); C = 513: four 128-channel chunks and a one-channel tail."""
    sc, t = _scene(name, C)
    rs = _settings(sc)
    H, W = rs.image_height, rs.image_width
    g = _gen(C + 1)
    gc, gd = torch.randn(3, H, W, device="cuda", generator=g), torch.randn(1, H, W, device="cuda", generator=g)
    h = torch.randn(C, H, W, device="cuda", generator=g).half()
    if layout == "odd_offset":
        base = torch.empty(C * H * W + 1, device="cuda", dtype=torch.float16)
        base[1:] = h.flatten()
        h = base[1:].view(C, H, W)
        assert h.is_contiguous() and h.data_ptr() % 8 != 0
    from diff_gaussian_rasterization.feature_head import ScaledGrad

    g16 = _accum(t, rs, gc, ScaledGrad(h, s), gd)
    g32 = _accum(t, rs, gc, h.float() * s, gd)
    _check_bwd(g16, g32, f"{name} C={C} s={s:g} {layout}")


@pytest.mark.gpu
@pytest.mark.parametrize("name,C", [("small", 16), ("small128", 128), ("small200", 200), ("small513", 513)])
def test_backward_f16_binding_is_the_float_backward_of_the_upcast_map(name, C):
    """rasterize_gaussians_backward with a float16 dL/dfeature_map calls f3dgs_backward_f16 with scale 1."""
    from diff_gaussian_rasterization import _C

    sc, t = _scene(name, C)
    rs = _settings(sc)
    H, W = rs.image_height, rs.image_width
    g = _gen(C + 2)
    gc, gd = torch.randn(3, H, W, device="cuda", generator=g), torch.randn(1, H, W, device="cuda", generator=g)
    h = torch.randn(C, H, W, device="cuda", generator=g).half()
    e = torch.Tensor([])
    R, _, _, _, radii, geom, binning, img = _C.rasterize_gaussians(
        rs.bg, t["means3D"], e, t["semantic_feature"], t["opacities"], t["scales"], t["rotations"], 1.0, e,
        rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, H, W, t["shs"], rs.sh_degree, rs.campos, False, False)

    def bwd(gf):
        out = _C.rasterize_gaussians_backward(rs.bg, t["means3D"], radii, e, t["semantic_feature"], t["scales"],
                                              t["rotations"], 1.0, e, rs.viewmatrix, rs.projmatrix, rs.tanfovx,
                                              rs.tanfovy, gc, gf, gd, t["shs"], rs.sh_degree, rs.campos, geom, R,
                                              binning, img, False)
        return dict(zip(("means2D", "colors", "semantic_feature", "opacities", "means3D", "cov3D", "shs", "scales",
                         "rotations"), out))

    g16, g32 = bwd(h), bwd(h.float())
    assert g16["semantic_feature"].dtype == torch.float32
    v = _viol(g16["semantic_feature"], g32["semantic_feature"])
    worst = {k: _viol(g16[k], g32[k]) for k in GEOM + ("means2D",)}
    print(f"[{name} C={C}] dL/dfeature viol {v:.3g}; " + ", ".join(f"{k}={x:.3g}" for k, x in worst.items()))
    assert v <= 1.0 and all(x <= 1.0 for x in worst.values()), worst


@pytest.mark.gpu
def test_accum_binding_rejects_a_scale_on_a_float32_gradient():
    sc, t = _scene("small", 16)
    rs = _settings(sc)
    H, W = rs.image_height, rs.image_width
    z = torch.zeros
    with pytest.raises(RuntimeError, match="feature_grad_scale != 1 needs a float16"):
        _accum(t, rs, z(3, H, W, device="cuda"), (z(16, H, W, device="cuda"), 0.5), z(1, H, W, device="cuda"))


RESIZES = [(108, 192, 48, 85), (96, 150, 64, 100), (40, 60, 80, 121), (50, 70, 1, 31), (50, 70, 23, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("H,W,Hg,Wg", RESIZES, ids=["down2.25", "down1.5", "up2", "Hg1", "Wg1"])
def test_resize_fwd_of_a_half_map_is_the_float_resize_of_the_upcast_map(H, W, Hg, Wg):
    from diff_gaussian_rasterization import _C

    C = 24
    g = _gen(H * W)
    fm = torch.randn(C, H, W, device="cuda", generator=g).half()
    gt = torch.randn(C, Hg, Wg, device="cuda", generator=g)
    for target in (gt, gt.half(), torch.empty(0, device="cuda")):
        o16, l16 = _C.feature_resize_fwd(fm, target, Hg, Wg, 0.37)
        o32, l32 = _C.feature_resize_fwd(fm.float(), target, Hg, Wg, 0.37)
        assert o16.dtype == torch.float32 and torch.equal(_bits(o16), _bits(o32))
        if target.numel():
            # the loss is one float atomic per block: equal up to their order
            assert torch.allclose(l16, l32, rtol=1e-5, atol=0)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W,Hg,Wg", [(108, 193, 48, 85), (97, 151, 64, 100), (41, 61, 80, 121)],
                         ids=["one_tap", "generic_down", "generic_up"])
def test_resize_bwd_f16_is_the_float_gradient_scaled_and_rounded(H, W, Hg, Wg):
    from diff_gaussian_rasterization import _C

    C = 12
    dout = torch.randn(C, Hg, Wg, device="cuda", generator=_gen(W))
    ref = _C.feature_resize_bwd(dout, H, W)
    for out_scale in (1.0, 3e-3, 7.5e4, -2.0 ** 17):  # the last two overflow 65504 for part of the elements
        h = _C.feature_resize_bwd(dout, H, W, torch.float16, out_scale)
        want = (ref * out_scale).half()
        assert h.dtype == torch.float16 and torch.equal(_bits(h), _bits(want)), out_scale
    assert bool(torch.isinf(_C.feature_resize_bwd(dout, H, W, torch.float16, 7.5e4)).any())
    with pytest.raises(RuntimeError, match="out_scale != 1 needs dtype float16"):
        _C.feature_resize_bwd(dout, H, W, torch.float32, 2.0)


@pytest.mark.gpu
def test_adam_step_f16out_is_adam_step_and_a_half_cast():
    from diff_gaussian_rasterization import _C

    n = 100003
    g = _gen(9)
    p0 = torch.randn(n, device="cuda", generator=g) * 10
    pa, pb = p0.clone(), p0.clone()
    ma, va = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    mb, vb = ma.clone(), va.clone()
    h = torch.empty(n, device="cuda", dtype=torch.float16)
    for step in range(1, 6):
        grad = torch.randn(n, device="cuda", generator=g)
        _C.adam_step(0, pa, grad, ma, va, 1, 1e-2, 0.9, 0.999, 1e-15, step)
        _C.adam_step(0, pb, grad, mb, vb, 1, 1e-2, 0.9, 0.999, 1e-15, step, h)
        for x, y in ((pa, pb), (ma, mb), (va, vb)):
            assert torch.equal(_bits(x), _bits(y))
        assert torch.equal(_bits(h), _bits(pb.half()))
    with pytest.raises(RuntimeError, match="kind must be F3DGS_PARAM_IDENTITY"):
        _C.adam_step(1, pb, grad, mb, vb, 1, 1e-2, 0.9, 0.999, 1e-15, 6, h)


@pytest.mark.gpu
def test_scaled_half_gradient_survives_where_a_plain_cast_underflows():
    """Config-3-like ratio: C = 128, 1920x1080 map, teacher at 1/2.25 (853x480): the L1 gradient is ~1.9e-8."""
    from diff_gaussian_rasterization import feature_head as fh

    C, H, W = 128, 1080, 1920
    Hg, Wg = round(H / 2.25), round(W / 2.25)
    g = _gen(3)
    fm = torch.randn(C, H, W, device="cuda", generator=g).half()
    gt = torch.randn(C, Hg, Wg, device="cuda", generator=g).half()
    l32, g32 = fh.feature_l1_loss_and_grad(fm.float(), gt)
    l16, sg = fh.feature_l1_loss_and_grad(fm, gt, grad_dtype=torch.float16)
    assert isinstance(sg, fh.ScaledGrad) and sg.grad.dtype == torch.float16 and sg.grad.shape == (C, H, W)
    assert sg.scale == 1.0 / (C * Hg * Wg)
    assert not g32.half().any()  # the plain cast: all zeros
    assert torch.allclose(l16, l32, rtol=1e-5, atol=0)
    s = sg.scale
    got = sg.grad.float() * s
    tol = (_half_ulp(g32 / s) + 1e-6 * (g32 / s).abs()) * s
    bad = int(((got.double() - g32.double()).abs() > tol).sum())
    print(f"scale {s:.3g}; |g32| max {float(g32.abs().max()):.3g}; elements beyond half an ulp: {bad}")
    assert bad == 0
    # the nonzero pattern: every element float16 can hold at this scale is nonzero, and no zero of g32 becomes nonzero
    assert not bool(((got != 0) & (g32 == 0)).any())
    assert bool((got != 0)[g32.abs() >= s * 2.0 ** -24].all())
    assert float((got != 0).float().mean()) > 0.5


@pytest.mark.gpu
def test_decoded_loss_f16_gradient_matches_the_float_gradient():
    from diff_gaussian_rasterization import feature_head as fh

    Cin, Cout, H, W = 32, 64, 135, 240
    Hg, Wg = 60, 107
    g = _gen(4)
    fm = torch.randn(Cin, H, W, device="cuda", generator=g).half()
    gt = torch.randn(Cout, Hg, Wg, device="cuda", generator=g)
    w, b = torch.randn(Cout, Cin, 1, 1, device="cuda", generator=g) * 0.1, torch.randn(Cout, device="cuda", generator=g)
    l32, g32, dw32, db32 = fh.decoded_feature_l1_loss_and_grad(fm.float(), gt, w, b, 0.5)
    l16, sg, dw16, db16 = fh.decoded_feature_l1_loss_and_grad(fm, gt, w, b, 0.5, grad_dtype=torch.float16)
    assert torch.equal(l16, l32) and torch.equal(dw16, dw32) and torch.equal(db16, db32)
    assert sg.scale == 0.5 / (Cout * Hg * Wg) and sg.grad.dtype == torch.float16
    got = sg.grad.float() * sg.scale
    tol = (_half_ulp(g32 / sg.scale) + 1e-6 * (g32 / sg.scale).abs()) * sg.scale
    assert bool(((got.double() - g32.double()).abs() <= tol).all())


@pytest.mark.gpu
def test_autograd_feature_losses_reject_half_maps():
    from diff_gaussian_rasterization import feature_head as fh

    fm = torch.randn(8, 20, 30, device="cuda").half().requires_grad_(True)
    gt = torch.randn(8, 10, 15, device="cuda")
    with pytest.raises(RuntimeError, match="ViewBatch"):
        fh.feature_l1_loss(fm, gt)
    w = torch.randn(4, 8, device="cuda")
    with pytest.raises(RuntimeError, match="ViewBatch"):
        fh.decoded_feature_l1_loss(fm, torch.randn(4, 10, 15, device="cuda"), w)


def _train(feature_dtype, steps=50, C=16):
    """Colour + feature loss with Adam on a small scene against a synthetic teacher, from one seed."""
    from diff_gaussian_rasterization import _C, feature_head as fh
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid

    sc = scenegen.make_scene(P=3000, W=128, H=96, C=0, sh_degree=1, views=3, seed=21)
    t = scenegen.to_torch(sc, "cuda")
    P, M = sc.P, 4
    shs = t["shs"][:, :M].contiguous()
    teacher_sf = torch.randn(P, 1, C, device="cuda", generator=_gen(77))
    state = GaussianState(t["means3D"].clone(), shs[:, :1].clone(), shs[:, 1:].clone(),
                          inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                          t["rotations"].clone(), torch.zeros(P, 1, C, device="cuda"), feature_dtype=feature_dtype)
    views = [GaussianRasterizationSettings(**parity.settings(sc, cam, "cuda")) for cam in sc.cameras]
    H, W = views[0].image_height, views[0].image_width
    Hg, Wg = round(H / 2.25), round(W / 2.25)
    e = torch.Tensor([])
    teachers, colours = [], []
    for rs in views:  # the teacher: the same geometry rendered with target features and colours, resized
        _, col, fm, *_ = _C.rasterize_gaussians(rs.bg, t["means3D"], e, teacher_sf, t["opacities"], t["scales"],
                                               t["rotations"], 1.0, e, rs.viewmatrix, rs.projmatrix, rs.tanfovx,
                                               rs.tanfovy, H, W, (shs * 0.5).contiguous(), rs.sh_degree, rs.campos,
                                               False, False)
        teachers.append(_C.feature_resize_fwd(fm, e, Hg, Wg, 0.0)[0])
        colours.append(col)
    lrs = dict(xyz=1.6e-5, f_dc=2.5e-3, f_rest=1.25e-4, opacity=0.05, scaling=5e-3, rotation=1e-3, semantic_feature=0.03)
    grad_dtype = torch.float16 if feature_dtype == torch.float16 else None
    curve = []
    for _ in range(steps):
        state.activate()
        vb = state.batch()
        vb.zero_()
        lf_sum = 0.0
        for i, rs in enumerate(views):
            color, feat, _, depth, ctx = vb.forward(rs)
            assert feat.dtype == feature_dtype
            g_color = torch.sign(color - colours[i]) / color.numel()
            lf, gfeat = fh.feature_l1_loss_and_grad(feat, teachers[i], 1.0, grad_dtype=grad_dtype)
            vb.backward(ctx, g_color, gfeat, torch.zeros_like(depth), last=i == len(views) - 1)
            lf_sum += float(lf)
        vb.all_reduce()
        state.step(lrs)
        curve.append(lf_sum / len(views))
    if feature_dtype == torch.float16:
        assert state.raw["semantic_feature"].dtype == torch.float32
        assert torch.equal(_bits(state.act["semantic_feature"]), _bits(state.raw["semantic_feature"].half()))
    return curve


@pytest.mark.gpu
def test_half_feature_training_follows_float_training():
    c32 = _train(torch.float32)
    c16 = _train(torch.float16)
    print("step  float32 feature loss  float16 feature loss")
    for i in range(0, len(c32), 5):
        print(f"{i:4d}  {c32[i]:.6f}  {c16[i]:.6f}")
    print(f"last  {c32[-1]:.6f}  {c16[-1]:.6f}")
    assert c32[-1] <= 0.5 * c32[0] and c16[-1] <= 0.5 * c16[0]
    assert abs(c16[-1] - c32[-1]) <= 0.05 * c32[-1]


@pytest.mark.gpu
def test_gaussian_state_keeps_the_half_copy_through_densification():
    from diff_gaussian_rasterization.trainer import GaussianState

    g = np.random.default_rng(0)
    pts, cols = g.uniform(-1, 1, (500, 3)), g.uniform(0, 1, (500, 3))
    st = GaussianState.from_point_cloud(pts, cols, 8, feature_dtype=torch.float16)
    assert st.act["semantic_feature"].dtype == torch.float16 and st.raw["semantic_feature"].dtype == torch.float32
    st.raw["semantic_feature"].normal_()
    ga = torch.rand(st.P, device="cuda") * 1e-3
    st.densify_and_prune(2e-4, 0.005, 1.0, False, ga, torch.ones(st.P, device="cuda"),
                         torch.Generator(device="cuda").manual_seed(0))
    assert st.act["semantic_feature"].shape == st.raw["semantic_feature"].shape
    assert torch.equal(_bits(st.act["semantic_feature"]), _bits(st.raw["semantic_feature"].half()))
    with pytest.raises(ValueError, match="feature_dtype"):
        GaussianState.from_point_cloud(pts, cols, 8, feature_dtype=torch.bfloat16)


def _peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


@pytest.mark.gpu
def test_half_viewbatch_step_saves_a_float32_map_of_memory():
    from diff_gaussian_rasterization import feature_head as fh
    from diff_gaussian_rasterization.parallel import ViewBatch

    C, W, H = 512, 960, 544
    sc = scenegen.make_scene(P=20000, W=W, H=H, C=0, sh_degree=1, seed=11)
    t = scenegen.to_torch(sc, "cuda")
    rs = _settings(sc)
    gt = torch.rand(C, round(H / 2.25), round(W / 2.25), device="cuda", generator=_gen(1))
    sf32 = torch.randn(sc.P, 1, C, device="cuda", generator=_gen(2))
    peaks = {}
    for dt in (torch.float32, torch.float16):
        params = {k: t[k] for k in ("means3D", "scales", "rotations", "opacities", "shs")}
        params["semantic_feature"] = sf32.to(dt)
        vb = ViewBatch(params)
        gd = torch.zeros(1, H, W, device="cuda")
        gc = torch.zeros(3, H, W, device="cuda")

        def step():
            vb.zero_()
            _, feat, _, _, ctx = vb.forward(rs)
            _, gf = fh.feature_l1_loss_and_grad(feat, gt, grad_dtype=dt if dt == torch.float16 else None)
            vb.backward(ctx, gc, gf, gd, last=True)

        step()  # warm-up
        peaks[dt] = _peak(step)
        del vb, params
    map32 = C * H * W * 4
    print(f"peak: float32 {peaks[torch.float32] / 2**20:.1f} MiB, float16 {peaks[torch.float16] / 2**20:.1f} MiB, "
          f"float32 map {map32 / 2**20:.1f} MiB")
    assert peaks[torch.float32] - peaks[torch.float16] >= 0.9 * map32


@pytest.mark.gpu
def test_autograd_backward_of_a_half_render_makes_no_float32_map():
    from diff_gaussian_rasterization import GaussianRasterizer

    C, W, H = 512, 960, 544
    sc = scenegen.make_scene(P=20000, W=W, H=H, C=0, sh_degree=1, seed=11)
    t = scenegen.to_torch(sc, "cuda", requires_grad=True)
    sf16 = torch.randn(sc.P, 1, C, device="cuda", generator=_gen(5)).half().requires_grad_(True)
    rast = GaussianRasterizer(_settings(sc))
    gf = torch.randn(C, H, W, device="cuda", generator=_gen(6)).half()

    def run():
        means2D = torch.zeros_like(t["means3D"], requires_grad=True)
        color, feat, radii, depth = rast(means3D=t["means3D"], means2D=means2D, opacities=t["opacities"],
                                         shs=t["shs"], semantic_feature=sf16, scales=t["scales"],
                                         rotations=t["rotations"])
        return feat

    feat = run()
    feat.backward(gf)  # warm-up
    feat = run()
    grew = _peak(lambda: feat.backward(gf))
    map32 = C * H * W * 4
    print(f"backward peak growth {grew / 2**20:.1f} MiB, float32 map {map32 / 2**20:.1f} MiB")
    assert sf16.grad.dtype == torch.float16
    assert grew < 0.5 * map32
