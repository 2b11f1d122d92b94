"""Feature lifting: blend-weighted back-projection of 2-D feature maps onto Gaussians (f3dgs_lift_features_accum[_f16],
the backward composite's lift mode, feature_head.FeatureLift).

The lift is the identity  feature_sum = dL_dsemantic_feature, weight_sum = dL_dcolors[:, 0]  of a full backward with
dL/dfeature_map = F, dL/dcolor = the planes (1, 0, 0) and dL/ddepth = 0, which the CPU oracle and the device backward
both provide; the lift computes it without the geometric gradients.
CPU part (`-m "not gpu"`): both C symbols reject malformed calls before any CUDA call.
"""
import ctypes
import functools

import numpy as np
import pytest
import torch

import parity
import scenegen

c_p, c_i = ctypes.c_void_p, ctypes.c_int
SYMS = ("f3dgs_lift_features_accum", "f3dgs_lift_features_accum_f16")


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_launch_count.restype = ctypes.c_ulonglong
    for s in SYMS:
        getattr(L, s).argtypes = [c_i] * 5 + [c_p] * 7
    return L


# ---- CPU: C ABI validation (fake addresses, never dereferenced: every call below fails validation)
@pytest.mark.parametrize("sym,esize", [(SYMS[0], 4), (SYMS[1], 2)])
def test_lift_rejects_malformed_calls_before_touching_cuda(lib, sym, esize):
    f = getattr(lib, sym)
    launches = lib.f3dgs_launch_count()
    A = lambda k: k << 28  # noqa: E731  (distinct fake device addresses, 256 MiB apart)
    P, R, C, W, H = 1000, 5000, 16, 64, 48

    def call(P=P, R=R, C=C, W=W, H=H, geom=A(1), binning=A(2), img=A(3), fmap=A(4), fsum=A(5), wsum=A(6)):
        return f(P, R, C, W, H, geom, binning, img, fmap, fsum, wsum, None)

    def rejected(msg, **kw):
        assert call(**kw) == -1, (sym, kw)
        err = lib.f3dgs_last_error()
        assert err.startswith(sym.encode() + b": ") and msg in err, (sym, kw, err)

    for kw in (dict(P=-1), dict(R=-1), dict(W=0), dict(H=0), dict(C=0), dict(C=-3), dict(C=4097)):
        rejected(b"bad sizes", **kw)
    for k in ("geom", "binning", "img"):
        rejected(b"missing forward buffers", **{k: None})
    for k in ("fmap", "fsum", "wsum"):
        rejected(b"NULL pointer", **{k: None})
    nmap = C * W * H * esize
    rejected(b"must not overlap", fsum=A(4) + nmap - 4)      # feature_sum runs into the map's last element
    rejected(b"must not overlap", fsum=A(4) - P * C * 4 + 4)  # feature_sum ends in the map's first element
    rejected(b"must not overlap", wsum=A(4) + nmap - 4)
    rejected(b"must not overlap", wsum=A(5) + P * C * 4 - 4)  # weight_sum inside feature_sum
    rejected(b"must not overlap", fsum=A(6) - P * C * 4 + 4)
    # the limit itself passes the size check (the call then stops at the missing map)
    rejected(b"NULL pointer", C=4096, fmap=None)
    # nothing to blend: nothing is launched and nothing is read
    assert call(P=0) == 0 and call(R=0) == 0
    assert lib.f3dgs_launch_count() == launches


# =================================================================================================== GPU
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _settings(sc, cam=None):
    from diff_gaussian_rasterization import GaussianRasterizationSettings

    return GaussianRasterizationSettings(**parity.settings(sc, cam or sc.cameras[0], "cuda"))


def _forward(t, rs):
    """f3dgs_forward at C = 0 with zero colours, as FeatureLift.add does -> (R, radii, geom, binning, img)."""
    from diff_gaussian_rasterization import _C

    e = torch.empty(0, device="cuda")
    P = t["means3D"].shape[0]
    R, _, _, _, radii, geom, binning, img = _C.rasterize_gaussians(
        rs.bg, t["means3D"], torch.zeros(P, 3, device="cuda"), e, t["opacities"], t["scales"], t["rotations"],
        rs.scale_modifier, e, rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width,
        e, rs.sh_degree, rs.campos, rs.prefiltered, False)
    return R, radii, geom, binning, img


def _lift(t, rs, fmap, fwd=None):
    """One view through the native lift -> (feature_sum [P,C], weight_sum [P])."""
    from diff_gaussian_rasterization import _C

    R, _, geom, binning, img = fwd or _forward(t, rs)
    P, C = t["means3D"].shape[0], fmap.shape[0]
    fs, ws = torch.zeros(P, C, device="cuda"), torch.zeros(P, device="cuda")
    _C.lift_features_accum(geom, R, binning, img, fmap, fs, ws)
    return fs, ws


def _composition(t, rs, fmap, fwd=None):
    """The same sums from a full backward: dL/dfeature_map = F, dL/dcolor = (1, 0, 0) planes, dL/ddepth = 0."""
    from diff_gaussian_rasterization import _C

    R, radii, geom, binning, img = fwd or _forward(t, rs)
    P, (C, H, W) = t["means3D"].shape[0], fmap.shape
    e = torch.empty(0, device="cuda")
    gc = torch.zeros(3, H, W, device="cuda")
    gc[0] = 1.0
    out = _C.rasterize_gaussians_backward(
        rs.bg, t["means3D"], radii, torch.zeros(P, 3, device="cuda"), torch.empty(P, 1, C, device="cuda"),
        t["scales"], t["rotations"], rs.scale_modifier, e, rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, gc,
        fmap, torch.zeros(1, H, W, device="cuda"), e, rs.sh_degree, rs.campos, geom, R, binning, img, False)
    return out[2].reshape(P, C), out[1][:, 0].contiguous()


def _close(a, b, rtol=1e-5, floor=1e-6):
    """Float-reduction-order tolerance: rtol relative plus an absolute floor of `floor` x max|b|."""
    a, b = a.double(), b.double()
    tol = rtol * b.abs() + floor * float(b.abs().max()) + 1e-30
    return float(((a - b).abs() / tol).max())


# ---- 1. the CPU oracle
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny", "small", "small200"])
def test_lift_equals_the_oracle_backward_identity(name):
    import oracle

    sc = scenegen.make_config(name)
    cam = sc.cameras[0]
    H, W, C = cam.image_height, cam.image_width, sc.C
    F = np.random.Generator(np.random.PCG64(7)).standard_normal((C, H, W), dtype=np.float32)
    gc = np.zeros((3, H, W), np.float32)
    gc[0] = 1.0
    fwd = oracle.forward(sc, cam)
    g = oracle.backward(sc, cam, fwd, gc, F, np.zeros((1, H, W), np.float32))
    t = scenegen.to_torch(sc, "cuda")
    fs, ws = _lift(t, _settings(sc), torch.from_numpy(F).cuda())
    # the oracle's expf differs from CUDA's by <= 2 ulp: a pixel at the 1/255 or 1e-4 threshold may blend one Gaussian
    # more or less; such ties widen the bar 50x, as the gradient parity tests do (parity.compare, tie_tolerant)
    ours = parity.run_ours(sc, cam)
    ties = int((ours["n_contrib"] != fwd["n_contrib"].astype(np.int64)).sum())
    assert ties <= max(2, int(1e-4 * H * W)), ties
    widen = 50.0 if ties else 1.0
    rf = parity.float_mismatch(fs.cpu().numpy(), g["semantic_feature"].reshape(sc.P, C), parity.RTOL * widen,
                               parity.GRAD_ATOL_REL * widen)
    rw = parity.float_mismatch(ws.cpu().numpy(), g["colors"][:, 0], parity.RTOL * widen, parity.GRAD_ATOL_REL * widen)
    print(f"[{name}] ties={ties} feature_sum viol={rf[0]:.3g} weight_sum viol={rw[0]:.3g}")
    assert rf[0] <= 1.0 and rw[0] <= 1.0
    assert float(ws.max()) > 0


# ---- 2. the full-backward composition on the device, config-2-sized
@functools.lru_cache(maxsize=2)
def _c2(W, H):
    sc = scenegen.make_scene(P=300_000, W=W, H=H, C=0, sh_degree=3, seed=2)
    return sc, scenegen.to_torch(sc, "cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["aligned", "w_odd", "misaligned_view"])
@pytest.mark.parametrize("C", [1, 3, 16, 128, 200, 513])
def test_lift_equals_the_full_backward_composition(C, layout):
    """aligned: 800x800 (4-pixel vector loads of the map); w_odd: W = 803 (scalar loads); misaligned_view: the map one
    element into its storage (scalar loads)."""
    sc, t = _c2(803 if layout == "w_odd" else 800, 800)
    rs = _settings(sc)
    H, W = rs.image_height, rs.image_width
    fmap = torch.randn(C, H, W, device="cuda", generator=_gen(C))
    if layout == "misaligned_view":
        base = torch.empty(C * H * W + 1, device="cuda")
        base[1:] = fmap.flatten()
        fmap = base[1:].view(C, H, W)
        assert fmap.is_contiguous() and fmap.data_ptr() % 16 != 0
    fwd = _forward(t, rs)
    fs, ws = _lift(t, rs, fmap, fwd)
    fs_ref, ws_ref = _composition(t, rs, fmap, fwd)
    vf, vw = _close(fs, fs_ref), _close(ws, ws_ref)
    print(f"[C={C} {layout}] R={fwd[0]} feature_sum viol={vf:.3g} weight_sum viol={vw:.3g}")
    assert vf <= 1.0 and vw <= 1.0
    assert float(ws.max()) > 0 and float(fs.abs().max()) > 0


# ---- 3. float16 maps
@pytest.mark.gpu
@pytest.mark.parametrize("C,W", [(16, 160), (128, 160), (200, 150), (513, 150)])
def test_half_map_lifts_as_its_exact_upcast(C, W):
    sc = scenegen.make_scene(P=4000, W=W, H=112, C=0, sh_degree=1, seed=C)
    t = scenegen.to_torch(sc, "cuda")
    rs = _settings(sc)
    h = torch.randn(C, rs.image_height, rs.image_width, device="cuda", generator=_gen(C)).half()
    fwd = _forward(t, rs)
    fs16, ws16 = _lift(t, rs, h, fwd)
    fs32, ws32 = _lift(t, rs, h.float(), fwd)
    v, vw = _close(fs16, fs32), _close(ws16, ws32)  # the sums' float atomics have no fixed order
    print(f"[C={C} W={W}] float16 map viol={v:.3g} weight_sum viol={vw:.3g}")
    assert v <= 1.0 and vw <= 1.0


# ---- 4. properties
def _prop_scene(C=0, seed=41, P=5000):
    sc = scenegen.make_scene(P=P, W=150, H=100, C=C, sh_degree=1, seed=seed)
    return sc, scenegen.to_torch(sc, "cuda")


@pytest.mark.gpu
def test_constant_map_lifts_to_itself_and_weights_do_not_depend_on_the_map():
    from diff_gaussian_rasterization.feature_head import FeatureLift

    sc, t = _prop_scene()
    rs = _settings(sc)
    H, W = rs.image_height, rs.image_width
    F0 = torch.randn(24, device="cuda", generator=_gen(1))
    lift = FeatureLift(t["means3D"], t["opacities"], t["scales"], t["rotations"], 24)
    lift.add(rs, F0[:, None, None].expand(24, H, W).contiguous())
    feats, w = lift.result()
    assert feats.shape == (sc.P, 1, 24) and w.shape == (sc.P,)
    seen = w > 0
    assert int(seen.sum()) > 0.5 * sc.P
    assert torch.allclose(feats[seen, 0], F0.expand(int(seen.sum()), 24), rtol=1e-5, atol=1e-6)
    # weight_sum: the same for every C and map
    for C, seed in ((1, 2), (77, 3), (300, 4)):
        _, ws = _lift(t, rs, torch.randn(C, H, W, device="cuda", generator=_gen(seed)))
        assert torch.allclose(ws, w, rtol=1e-6, atol=0), C


@pytest.mark.gpu
def test_unseen_gaussians_get_zero_weight_and_feature():
    from diff_gaussian_rasterization.feature_head import FeatureLift

    sc, t = _prop_scene(seed=42)
    P = sc.P
    t["opacities"][: P // 10] = 0.002  # alpha < 1/255 everywhere: never blended
    t["means3D"][P // 10: P // 5, 1] += 40.0  # far above the view: radii == 0
    rs = _settings(sc)
    R, radii, *_ = _forward(t, rs)
    culled = radii == 0
    assert bool(culled[P // 10: P // 5].all())
    lift = FeatureLift(t["means3D"], t["opacities"], t["scales"], t["rotations"], 8)
    lift.add(rs, torch.randn(8, rs.image_height, rs.image_width, device="cuda", generator=_gen(5)))
    feats, w = lift.result()
    unseen = culled.clone()
    unseen[: P // 10] = True
    assert bool((w[unseen] == 0).all()) and bool((feats[unseen] == 0).all())
    # a threshold drops the weakly seen ones too, and never gives NaN
    f2, _ = lift.result(min_weight=float(w[w > 0].median()))
    assert bool(torch.isfinite(f2).all()) and bool((f2[w <= float(w[w > 0].median())] == 0).all())


@pytest.mark.gpu
def test_two_views_accumulate_to_the_sum_of_their_lifts():
    from diff_gaussian_rasterization.feature_head import FeatureLift

    sc = scenegen.make_scene(P=5000, W=150, H=100, C=0, sh_degree=1, views=2, seed=43)
    t = scenegen.to_torch(sc, "cuda")
    views = [_settings(sc, cam) for cam in sc.cameras]
    maps = [torch.randn(40, 100, 150, device="cuda", generator=_gen(10 + i)) for i in range(2)]
    both = FeatureLift(t["means3D"], t["opacities"], t["scales"], t["rotations"], 40)
    for rs, m in zip(views, maps):
        both.add(rs, m)
    sums = [_lift(t, rs, m) for rs, m in zip(views, maps)]
    assert _close(both.feature_sum[:, 0], sums[0][0] + sums[1][0]) <= 1.0
    assert _close(both.weight_sum, sums[0][1] + sums[1][1]) <= 1.0
    # the flat buffer holds both
    P = sc.P
    assert both.flat.data_ptr() == both.feature_sum.data_ptr()
    assert both.weight_sum.data_ptr() == both.flat.data_ptr() + P * 40 * 4 and both.flat.numel() == P * 41


@pytest.mark.gpu
def test_widest_features():
    sc, t = _prop_scene(P=1500, seed=44)
    rs = _settings(sc)
    fmap = torch.randn(4096, rs.image_height, rs.image_width, device="cuda", generator=_gen(6))
    fwd = _forward(t, rs)
    fs, ws = _lift(t, rs, fmap, fwd)
    fs_ref, ws_ref = _composition(t, rs, fmap, fwd)
    assert _close(fs, fs_ref) <= 1.0 and _close(ws, ws_ref) <= 1.0


@pytest.mark.gpu
def test_lift_rejects_mismatched_maps():
    from diff_gaussian_rasterization import _C
    from diff_gaussian_rasterization.feature_head import FeatureLift

    sc, t = _prop_scene(P=500, seed=45)
    rs = _settings(sc)
    lift = FeatureLift(t["means3D"], t["opacities"], t["scales"], t["rotations"], 8)
    with pytest.raises(ValueError, match="C = 8"):
        lift.add(rs, torch.zeros(9, 100, 150, device="cuda"))
    with pytest.raises(ValueError, match="image_height=50, image_width=75"):
        lift.add(rs, torch.zeros(8, 50, 75, device="cuda"))
    with pytest.raises(ValueError, match="float32 or float16"):
        lift.add(rs, torch.zeros(8, 100, 150, device="cuda", dtype=torch.float64))
    with pytest.raises(ValueError, match="C must be"):
        FeatureLift(t["means3D"], t["opacities"], t["scales"], t["rotations"], 0)
    R, _, geom, binning, img = _forward(t, rs)
    fm = torch.zeros(8, 100, 150, device="cuda")
    with pytest.raises(RuntimeError, match="feature_sum"):
        _C.lift_features_accum(geom, R, binning, img, fm, torch.zeros(sc.P, 7, device="cuda"),
                               torch.zeros(sc.P, device="cuda"))
    flat = torch.zeros(sc.P * 9, device="cuda")
    with pytest.raises(RuntimeError, match="must not overlap"):
        _C.lift_features_accum(geom, R, binning, img, fm, flat[: sc.P * 8], flat[sc.P * 8 - 1: sc.P * 9 - 1])
    # a teacher at its own resolution: the settings at that size
    lift.add(rs._replace(image_height=50, image_width=75), torch.ones(8, 50, 75, device="cuda"))
    f, w = lift.result()
    assert float(w.max()) > 0 and torch.allclose(f[w > 0], torch.ones_like(f[w > 0]), rtol=1e-5)


# ---- 5. end to end: lifted fields render, train and densify through the existing paths
def _state_of(sc, t, sf, feature_dtype):
    from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid

    shs = t["shs"][:, :4].contiguous()
    return GaussianState(t["means3D"].clone(), shs[:, :1].clone(), shs[:, 1:].clone(),
                         inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                         t["rotations"].clone(), sf, feature_dtype=feature_dtype)


def _feature_loss(state, views, teachers, grad_dtype=None, train_steps=0):
    """Mean feature L1 over the views; with train_steps, that many Adam steps on the feature loss first."""
    from diff_gaussian_rasterization import feature_head as fh

    lrs = dict(xyz=1.6e-5, f_dc=2.5e-3, f_rest=1.25e-4, opacity=0.05, scaling=5e-3, rotation=1e-3, semantic_feature=0.03)
    for step in range(train_steps + 1):
        state.activate()
        vb = state.batch()
        vb.zero_()
        total = 0.0
        for i, rs in enumerate(views):
            color, feat, radii, depth, ctx = vb.forward(rs)
            lf, gfeat = fh.feature_l1_loss_and_grad(feat, teachers[i], 1.0, grad_dtype=grad_dtype)
            total += float(lf)
            if step < train_steps:
                vb.backward(ctx, torch.zeros_like(color), gfeat, torch.zeros_like(depth), last=i == len(views) - 1)
        if step < train_steps:
            vb.all_reduce()
            state.step(lrs)
    return total / len(views)


@pytest.mark.gpu
@pytest.mark.parametrize("feature_dtype", [torch.float32, torch.float16], ids=["float32", "float16"])
def test_lifted_field_renders_trains_and_densifies(feature_dtype):
    from diff_gaussian_rasterization import _C
    from diff_gaussian_rasterization.feature_head import FeatureLift

    C = 32
    sc = scenegen.make_scene(P=4000, W=128, H=96, C=0, sh_degree=1, views=6, seed=46)
    t = scenegen.to_torch(sc, "cuda")
    views = [_settings(sc, cam) for cam in sc.cameras]
    H, W = views[0].image_height, views[0].image_width
    field = torch.randn(sc.P, 1, C, device="cuda", generator=_gen(47))  # the seeded per-Gaussian field
    e = torch.Tensor([])
    teachers = []
    for rs in views:  # teachers: renders of that field, as a float16 teacher map is stored
        fm = _C.rasterize_gaussians(rs.bg, t["means3D"], e, field, t["opacities"], t["scales"], t["rotations"], 1.0, e,
                                    rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, H, W, t["shs"],
                                    rs.sh_degree, rs.campos, False, False)[2]
        teachers.append(fm.half() if feature_dtype == torch.float16 else fm)
    grad_dtype = torch.float16 if feature_dtype == torch.float16 else None

    zero = _state_of(sc, t, torch.zeros(sc.P, 1, C, device="cuda"), feature_dtype)
    lift = FeatureLift.from_state(zero)
    for rs, tm in zip(views, teachers):
        lift.add(rs, tm)
    feats, w = lift.result()
    assert feats.shape == (sc.P, 1, C) and feats.dtype == torch.float32
    lifted = _state_of(sc, t, feats, feature_dtype)

    l_zero = _feature_loss(zero, views, teachers, grad_dtype)
    l_lift = _feature_loss(lifted, views, teachers, grad_dtype)
    print(f"[{feature_dtype}] feature L1: zero field {l_zero:.4f}, lifted field {l_lift:.4f}")
    assert l_lift < l_zero
    # training from the lifted field keeps lowering the loss, and densification carries the field along
    l_trained = _feature_loss(lifted, views, teachers, grad_dtype, train_steps=20)
    print(f"[{feature_dtype}] after 20 steps from the lifted field {l_trained:.4f}")
    assert l_trained < l_lift
    P0 = lifted.P
    ga = torch.rand(P0, device="cuda", generator=_gen(48)) * 1e-3
    P1 = lifted.densify_and_prune(2e-4, 0.005, 1.0, False, ga, torch.ones(P0, device="cuda"), _gen(49))
    assert P1 > 0 and lifted.raw["semantic_feature"].shape == (P1, 1, C)
    assert bool(torch.isfinite(lifted.raw["semantic_feature"]).all())
    _feature_loss(lifted, views, teachers, grad_dtype, train_steps=1)
