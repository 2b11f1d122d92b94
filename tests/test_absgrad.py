"""AbsGS's absolute-gradient densification statistic (f3dgs_backward_absgrad / f3dgs_backward_accum_absgrad,
f3dgs_densify_plan_absgrad, AbsGradGaussianRasterizer, ViewBatch(absgrad=True), densify_and_prune(abs_grad=...)).

For view v and Gaussian i, dL_dmean2D_abs[i] = (sum_p |t_x|, sum_p |t_y|, 0) over the pixels p the view blends i into,
t_ip pixel p's term of dL/dmean2D_i.  The yardsticks are tests/ref_absgrad.py: a float64 model of the per-pixel terms
(blend_weights.composite_model's loss with one leaf per pair) within composite_model's mean-2D bar, and the PyTorch
restatement of AbsGS's split rule.  Everything else the new entries write must be bitwise what their counterparts write.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import blend_weights as bw
import ref_absgrad
import scenegen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F16 = 0, 1


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_launch_count.restype = ctypes.c_ulonglong
    L.f3dgs_backward_scratch_bytes.restype = ctypes.c_size_t
    return L


# ------------------------------------------------------------------------------------------------------------ CPU
def test_header_declares_and_library_exports_the_entries(lib):
    header = open(os.path.join(ROOT, "include", "f3dgs_b200.h")).read()
    for name in ("f3dgs_backward_absgrad", "f3dgs_backward_accum_absgrad", "f3dgs_densify_plan_absgrad"):
        assert f"int {name}(" in header, name
        assert hasattr(lib, name), name
    assert "#define F3DGS_ABI_VERSION 2" in header


def _fake(i, fake=1 << 40):
    return ctypes.c_void_p(fake + i * (1 << 20))


def _assign_args(P=5, planes=(None, None), absb=40):
    """f3dgs_backward_absgrad's arguments with distinct fake device addresses (the checks fail first); outputs are
    _fake(15) .. _fake(25), dL_dcamera _fake(26)."""
    f, null = ctypes.c_float, ctypes.c_void_p(0)
    p = lambda i: _fake(i) if i is not None else null  # noqa: E731
    return [P, 0, 1, 10, 4, _fake(0), 64, 64, _fake(1), _fake(2), null, _fake(50), F32, _fake(3), f(1.0), _fake(4),
            null, _fake(5), _fake(6), _fake(7), f(0.5), f(0.5), _fake(8), _fake(9), _fake(10), _fake(11), _fake(12),
            _fake(13), F32, f(1.0), _fake(14), _fake(15), _fake(16), _fake(17), _fake(18), _fake(19), _fake(20),
            _fake(21), _fake(22), _fake(23), _fake(24), _fake(25), 0, null, _fake(26), 0, p(planes[0]), p(planes[1]),
            p(absb)]


def _accum_args(P=5, planes=(None, None), absb=40, gaa=41, ga=22, dn=23):
    """f3dgs_backward_accum_absgrad's arguments: scratch _fake(30), outputs _fake(15) .. _fake(21), grad_accum
    _fake(22), denom _fake(23), dL_dcamera _fake(26)."""
    f, null = ctypes.c_float, ctypes.c_void_p(0)
    p = lambda i: _fake(i) if i is not None else null  # noqa: E731
    return [P, 0, 1, 10, 4, _fake(0), 64, 64, _fake(1), _fake(2), null, _fake(50), F32, _fake(3), f(1.0), _fake(4),
            null, _fake(5), _fake(6), _fake(7), f(0.5), f(0.5), _fake(8), _fake(9), _fake(10), _fake(11), _fake(12),
            _fake(13), F32, f(1.0), _fake(14), _fake(30), _fake(15), null, _fake(16), _fake(17), null, _fake(18),
            _fake(19), _fake(20), _fake(21), p(ga), p(dn), null, 0, null, _fake(26), 0, p(planes[0]), p(planes[1]),
            p(absb), p(gaa)]


def test_cabi_rejects_every_invalid_argument_before_any_cuda_call(lib):
    n0 = lib.f3dgs_launch_count()
    err = lambda: lib.f3dgs_last_error().decode()  # noqa: E731
    for name, mk in (("f3dgs_backward_absgrad", _assign_args), ("f3dgs_backward_accum_absgrad", _accum_args)):
        fn = getattr(lib, name)
        assert fn(*mk(absb=None)) == -1 and err() == f"{name}: NULL dL_dmean2D_abs"
        for planes in ((60, None), (None, 61)):
            assert fn(*mk(planes=planes)) == -1 and "dL_dalpha and dL_dinvdepth go together" in err(), planes
        outs = (15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26) if name == "f3dgs_backward_absgrad" else \
            (30, 15, 16, 17, 18, 19, 20, 21, 22, 23, 26)
        for i in outs:  # the statistic inside each other output (the camera gradient and the scratch included)
            assert fn(*mk(absb=i)) == -1 and "dL_dmean2D_abs overlaps another output" in err(), (name, i, err())
        assert fn(*mk(planes=(40, 61))) == -1 and "overlap" in err()  # a plane gradient inside the statistic
        assert fn(*mk(P=-1)) == -1
        assert fn(*mk(P=0)) == 0  # nothing to do
    fn = lib.f3dgs_backward_accum_absgrad
    name = "f3dgs_backward_accum_absgrad"
    assert fn(*_accum_args(ga=None, dn=None)) == -1 and err() == f"{name}: grad_accum_abs needs grad_accum and denom"
    for i in (30, 15, 16, 17, 18, 19, 20, 21, 22, 23, 26, 40):
        assert fn(*_accum_args(gaa=i)) == -1 and "grad_accum_abs overlaps another output" in err(), (i, err())
    plan = lib.f3dgs_densify_plan_absgrad
    plan.argtypes = [ctypes.c_int] + [ctypes.c_void_p] * 4 + [ctypes.c_float] * 4 + [ctypes.c_void_p] * 4 + \
        [ctypes.c_float]
    ga, dn, op, sc, scr, cnt, gaa = 0x1000000, 0x2000000, 0x3000000, 0x4000000, 0x80000000, 0x90000000, 0x5000000
    th = (2e-4, 0.04, 0.005, 0.4)
    assert plan(-1, ga, dn, op, sc, *th, scr, cnt, None, gaa, 4e-4) == -1 and b"bad sizes" in lib.f3dgs_last_error()
    assert plan(10, ga, dn, op, sc, *th, scr, cnt, None, None, 4e-4) == -1 and b"NULL" in lib.f3dgs_last_error()
    assert plan(10, ga, dn, op, sc, *th, scr, scr + 64, None, gaa, 4e-4) == -1
    assert b"overlaps" in lib.f3dgs_last_error()
    assert lib.f3dgs_launch_count() == n0


def test_restated_split_rule_on_hand_made_statistics():
    """AbsGS: clone on the norm of the summed gradient (small Gaussians), split on the summed norms (large ones)."""
    ga = torch.tensor([3e-4, 3e-4, 1e-5, 1e-5, 0.0, 1e-3, 1e-5])
    gaa = torch.tensor([3e-4, 3e-4, 5e-3, 5e-3, 0.0, 1e-3, 5e-3])
    dn = torch.tensor([1.0, 1.0, 1.0, 1.0, 0.0, 2.0, 0.0])
    smax = torch.tensor([0.01, 0.5, 0.01, 0.5, 0.5, 0.5, 0.5])
    scaling = smax[:, None].repeat(1, 3)
    clone, split = ref_absgrad.absgs_masks(ga, gaa, dn, scaling, 2e-4, 4e-3, 0.037)
    # row 0: clone; 1: large, its abs statistic below abs_grad: nothing; 2: small, collision-free norm small: nothing;
    # 3: large with colliding gradients (small norm, large abs sum): split; 4: 0 / 0 -> 0; 5: 5e-4 < 4e-3; 6: x / 0
    assert clone.tolist() == [True, False, False, False, False, False, False]
    assert split.tolist() == [False, False, False, True, False, False, True]


def test_python_surface():
    import inspect

    import diff_gaussian_rasterization as dgr
    from diff_gaussian_rasterization.parallel import ViewBatch
    from diff_gaussian_rasterization.trainer import GaussianState

    assert "AbsGradGaussianRasterizer" in dgr.__all__ and "AbsGradGaussianRasterizer" in dgr.__doc__
    assert issubclass(dgr.AbsGradGaussianRasterizer, dgr.GaussianRasterizer)
    assert list(inspect.signature(dgr.AbsGradGaussianRasterizer.__init__).parameters) == [
        "self", "raster_settings", "feature_geometry", "antialiasing"]
    assert inspect.signature(dgr.AbsGradGaussianRasterizer.forward).parameters["means2D_abs"].default is None
    assert hasattr(dgr._C, "rasterize_gaussians_backward_absgrad")
    assert inspect.signature(ViewBatch.__init__).parameters["absgrad"].default is False
    assert inspect.signature(GaussianState.__init__).parameters["absgrad"].default is False
    p = inspect.signature(GaussianState.densify_and_prune).parameters
    assert p["abs_grad"].default is None and p["grad_accum_abs"].default is None
    with pytest.raises(ValueError):
        ViewBatch(dict(means3D=torch.zeros(4, 3)), densify_stats=False, absgrad=True)


# ------------------------------------------------------------------------------------------------------------ GPU
def _backward(v, ups, absgrad, camera=False, feature_geometry=False, planes=None, half=False, antialiasing=False):
    """The binding's assigning backward of a test_geometry_grads.View: rasterize_gaussians_backward_absgrad, or the
    counterpart entry that has the same options without the statistic -> its tuple."""
    from diff_gaussian_rasterization import _C

    gc, gf, gd = (u if isinstance(u, torch.Tensor) else torch.from_numpy(u).cuda() for u in ups)
    if half:
        gf = gf.half()
    b = v.base
    args = (v.bg, v.d["means3D"], b["radii"], v.cols, v.feats, v.scales, v.rots, v.mod, v.cov, v.vm, v.pm,
            v.cam.tanfovx, v.cam.tanfovy, gc, gf, gd, v.shs, v.D, v.cp, b["geom"], v.R, b["binning"], b["img"], False)
    sf = v.feats if feature_geometry else None
    if absgrad:
        ga, gi = planes if planes is not None else (None, None)
        return _C.rasterize_gaussians_backward_absgrad(*args, dL_dout_alpha=ga, dL_dout_invdepth=gi, camera=camera,
                                                       semantic_feature=sf, antialiasing=antialiasing)
    if planes is not None:
        return _C.rasterize_gaussians_backward_alpha_invdepth(*args, *planes, camera=camera, semantic_feature=sf,
                                                              antialiasing=antialiasing)
    if antialiasing:
        return _C.rasterize_gaussians_backward_antialiased(*args, camera=camera, semantic_feature=sf)
    if feature_geometry:
        return _C.rasterize_gaussians_backward_feature_geometry(*args, camera)
    if camera:
        return _C.rasterize_gaussians_backward_camera(*args)
    return _C.rasterize_gaussians_backward(*args)


def _view(name, planes=False, antialiasing=False):
    from test_geometry_grads import View, _scene

    sc, cam, kw = _scene(name)
    return View(sc, cam, planes=planes, antialiasing=antialiasing, **kw)


def _model_ratio(ours, ref, bar):
    return float(bw._ratio((ours[:, :2].double().cpu() - ref.cpu()).abs(), bar.cpu()).max())


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["default", "antialiased", "planes", "feature_geometry"])
@pytest.mark.parametrize("name", ["small", "needles", "layers129"])
def test_statistic_matches_the_float64_model(name, mode):
    """Per Gaussian, dL_dmean2D_abs against the sums of |per-pixel term| of the float64 model, within composite_model's
    mean-2D bar.  With feature geometry: the colour walk's sums plus the feature walk's."""
    v = _view(name, planes=mode in ("planes", "antialiased"), antialiasing=mode == "antialiased")
    P, W, H, HW = v.P, v.W, v.H, v.W * v.H
    rec = v.base["rec"]
    for seed in (5, 6):
        gc, gf, gd = (torch.from_numpy(u).cuda() for u in bw.upstream(H, W, v.C, seed))
        Gc, Gd = gc.reshape(3, HW).t(), gd.reshape(HW)
        bgp = Gc.double() * v.bg.double()
        bg_dot = (bgp.sum(1), bgp.abs().sum(1))
        dfn, length, planes = bw.colour_depth_dots(rec, Gc, Gd), 4, None
        if mode == "planes":
            g = torch.Generator().manual_seed(seed)
            gA, gI = (torch.randn(1, H, W, generator=g).cuda() for _ in range(2))
            planes = (gA, gI)
            dfn, length = ref_absgrad.planes_dfn(rec, Gc, Gd, gI), 5
            bg_dot = (bg_dot[0] - gA.reshape(-1).double(), bg_dot[1] + gA.reshape(-1).double().abs())
        out = _backward(v, (gc, gf, gd), True, planes=planes, feature_geometry=mode == "feature_geometry",
                        antialiasing=mode == "antialiased")
        ours = out[12]
        ref = ref_absgrad.abs_mean2d_model(v.pairs, v.w, rec, P, dfn, bg_dot)
        _, bar = bw.composite_model(v.pairs, v.w, rec, P, dfn, length, bg_dot)
        bar = bar[:, :2]
        if mode == "feature_geometry":
            fd = ref_absgrad.feature_dfn(v.feats.reshape(P, v.C), gf.reshape(v.C, HW))
            ref = ref + ref_absgrad.abs_mean2d_model(v.pairs, v.w, rec, P, fd)
            bar = bar + bw.composite_model(v.pairs, v.w, rec, P, fd, v.C)[1][:, :2]
        r = _model_ratio(ours, ref, bar)
        print(f"[{name} {mode} seed {seed}] worst |err|/bar = {r:.3g}")
        assert r <= 1.0
        assert bool((ours[:, 2] == 0).all()) and bool((ours[v.base["radii"] == 0] == 0).all())
        # the statistic bounds the summed gradient's magnitude (within the rounding of sums over <= 16 k pixels)
        assert bool((ours[:, :2] >= out[0][:, :2].abs() * (1 - 1e-3)).all())
        # negative control: the largest statistic of the model scaled by 1.5 fails the bar
        worst = int(torch.argmax(ref[:, 0]))
        bad = ref.clone()
        bad[worst, 0] *= 1.5
        assert _model_ratio(ours, bad, bar) > 1.0


def _single_pixel_scene(W=64, H=48, seed=0):
    """_block_scene's layout with faint 0.3 px Gaussians whose centres sit 0.3 px off a pixel centre: each blends into
    that one pixel (alpha < 1/255 on its neighbours), with a nonzero 2-D mean gradient there."""
    from test_camera_grad import _block_scene

    sc, cam = _block_scene(W, H, C=0, deg=1, seed=seed)
    nb = sc.P // 2
    rng = np.random.default_rng(seed)
    by, bx = np.divmod(np.arange(nb), W // 8)
    px = np.concatenate([8 * bx + 2.3, 8 * bx + 5.3])
    py = np.concatenate([4 * by + 1.2, 4 * by + 2.2])
    z = np.concatenate([np.full(nb, 3.8), np.full(nb, 4.1)]) + rng.uniform(-0.05, 0.05, 2 * nb)
    vx = ((2 * px + 1) / W - 1) * cam.tanfovx * z
    vy = ((2 * py + 1) / H - 1) * cam.tanfovy * z
    view = np.stack([vx, vy, z, np.ones_like(z)], 1)
    sc.means3D = (view @ np.linalg.inv(cam.viewmatrix.astype(np.float64)))[:, :3].astype(np.float32)
    sc.opacities = rng.uniform(0.0045, 0.006, (2 * nb, 1)).astype(np.float32)
    return sc, cam


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["single_pixel", "small"])
def test_one_pixel_gaussians_give_the_absolute_gradient_bitwise(scene):
    """A Gaussian blended into exactly one pixel (GaussianScores.pixel_count == 1) has one term: dL_dmean2D_abs is
    |dL_dmean2D| bitwise.  Culled rows and the third column are 0."""
    from diff_gaussian_rasterization import _C
    from test_geometry_grads import View, _scene

    if scene == "single_pixel":
        sc, cam = _single_pixel_scene()
        sc.bg = np.array([0.2, 0.3, 0.4], np.float32)
        kw = {}
    else:
        sc, cam, kw = _scene(scene)
    v = View(sc, cam, weights=False, **kw)
    P = v.P
    ws, mw, pc = torch.zeros(P, device="cuda"), torch.zeros(P, device="cuda"), torch.zeros(P, dtype=torch.int64,
                                                                                          device="cuda")
    _C.gaussian_scores_accum(v.base["geom"], v.R, v.base["binning"], v.base["img"], v.W, v.H, ws, mw, pc)
    one = pc == 1
    if scene == "single_pixel":
        assert int(one.sum()) >= P // 2, int(one.sum())
    out = _backward(v, bw.upstream(v.H, v.W, v.C, 3), True)
    ours, mean2D = out[12], out[0]
    assert torch.equal(ours[one][:, :2], mean2D[one][:, :2].abs())
    if scene == "single_pixel":
        assert bool((ours[one][:, :2] > 0).any())
    assert bool((ours[:, 2] == 0).all())
    assert bool((ours[v.base["radii"] == 0] == 0).all()) and bool((ours[pc == 0] == 0).all())


def _settings(sc, cam):
    from diff_gaussian_rasterization import GaussianRasterizationSettings

    return GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, torch.device("cuda")))


COMBOS = [(h, c, f, a, p) for h in (False, True) for c in (False, True) for f in (False, True) for a in (False, True)
          for p in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("half,camera,fgeom,aa,planes", COMBOS)
def test_every_other_output_is_bitwise_the_counterparts(half, camera, fgeom, aa, planes):
    """On test_camera_grad._block_scene, whose reductions do not depend on atomic order: every other output of both new
    entries equals the counterpart entry's, and the accumulating entry's statistic equals the assigning one's."""
    from diff_gaussian_rasterization.parallel import ViewBatch
    from test_camera_grad import _block_scene
    from test_geometry_grads import View

    sc, cam = _block_scene()
    v = View(sc, cam, weights=False, planes=aa, antialiasing=aa)
    g = torch.Generator().manual_seed(11)
    H, W = v.H, v.W
    ups = tuple(torch.from_numpy(u).cuda() for u in scenegen.upstream_grads(H, W, v.C, 9))
    pl = tuple(torch.randn(1, H, W, generator=g).cuda() for _ in range(2)) if planes else None
    kw = dict(camera=camera, feature_geometry=fgeom, planes=pl, half=half, antialiasing=aa)
    ref = _backward(v, ups, False, **kw)
    new = _backward(v, ups, True, **kw)
    n = 12 if (planes or aa or fgeom or camera) else 9
    for i in range(n):
        a, b = ref[i], new[i]
        assert (a is None) == (b is None), i
        if a is not None:
            assert torch.equal(a, b), i
    abs_assign = new[12]
    assert bool(abs_assign.abs().sum() > 0)

    # the accumulating entry through ViewBatch
    params = dict(means3D=v.d["means3D"], scales=v.d["scales"], rotations=v.d["rotations"],
                  opacities=v.d["opacities"], shs=v.d["shs"],
                  semantic_feature=v.feats.half() if half else v.feats)
    rs = _settings(sc, cam)
    gf = ups[1].half() if half else ups[1]
    flats, cams = [], []
    for absgrad in (False, True):
        vb = ViewBatch(params, absgrad=absgrad)
        vb.zero_()
        if planes:
            *_, ctx = vb.forward_alpha_invdepth(rs, antialiasing=aa)
        else:
            *_, ctx = vb.forward(rs, antialiasing=aa)
        cg = vb.backward(ctx, ups[0], gf, ups[2], camera=camera, feature_geometry=fgeom,
                         g_alpha=pl[0] if planes else None, g_invdepth=pl[1] if planes else None)
        flats.append(vb.flat[:vb.n_param + 2 * vb.P].clone())
        cams.append(cg)
        if absgrad:
            assert vb.grad_accum_abs.data_ptr() == vb.flat.data_ptr() + (vb.n_param + 2 * vb.P) * 4
            if not half:  # the float16 features give the float16 forward's buffers: the same walk, another call
                assert torch.equal(vb.mean2D_abs, abs_assign)
            vis = ctx.radii > 0
            assert torch.allclose(vb.grad_accum_abs, vb.mean2D_abs[:, :2].norm(dim=1) * vis, rtol=1e-6, atol=0)
    assert torch.equal(flats[0], flats[1])
    if camera:
        for x, y in zip(cams[0], cams[1]):
            assert torch.equal(x, y)


def _collision_state(absgrad=True):
    """One large Gaussian at the origin, seen head-on and centred on the image: under a constant upstream colour
    gradient its per-pixel 2-D mean terms cancel in pairs."""
    from diff_gaussian_rasterization.trainer import GaussianState

    dev = torch.device("cuda")
    st = GaussianState(torch.zeros(1, 3, device=dev), torch.full((1, 1, 3), 0.8, device=dev),
                       torch.zeros(1, 0, 3, device=dev), torch.full((1, 1), 2.0, device=dev),
                       torch.full((1, 3), float(np.log(0.25)), device=dev),
                       torch.tensor([[1.0, 0.0, 0.0, 0.0]], device=dev), torch.zeros(1, 1, 0, device=dev),
                       absgrad=absgrad)
    cam = scenegen.make_camera(64, 64, np.array([0.0, 0.0, 3.0]))
    sc = scenegen.make_scene(1, 64, 64, 0, sh_degree=0)
    sc.bg = np.zeros(3, np.float32)
    return st, _settings(sc, cam)


@pytest.mark.gpu
def test_gradient_collision_splits_only_with_the_abs_statistic():
    st, rs = _collision_state()
    vb = st.batch()
    vb.zero_()
    st.activate()
    _, _, radii, _, ctx = vb.forward(rs)
    assert int(radii[0]) > 8
    H, W = rs.image_height, rs.image_width
    vb.backward(ctx, torch.ones(3, H, W, device="cuda"), None, torch.zeros(1, H, W, device="cuda"))
    g, ga = float(vb.grad_accum[0]), float(vb.grad_accum_abs[0])
    print(f"|dL/dmean2D| = {g:.3g}, sum |t| = {ga:.3g}")
    assert g < 1e-3 * ga
    thr = float(np.sqrt(max(g, 1e-30) * ga))  # between the two
    extent = 1.0  # dense_scale 0.01 < 0.25: a large Gaussian
    a, _ = _collision_state()
    a.batch().flat.copy_(vb.flat)
    assert a.densify_and_prune(thr, 0.005, extent, None, abs_grad=thr) == 2
    b, _ = _collision_state()
    b.batch().flat.copy_(vb.flat)
    assert b.densify_and_prune(thr, 0.005, extent, None) == 1
    c, _ = _collision_state(absgrad=False)
    with pytest.raises(ValueError):
        c.densify_and_prune(thr, 0.005, extent, None, abs_grad=thr)


@pytest.mark.gpu
def test_accumulation_over_three_views():
    """grad_accum_abs is the sum of the per-view norms of mean2D_abs where radii > 0; denom is bitwise that of
    absgrad=False and the rest of the flat buffer agrees within the order of the composite's float atomics (this scene's
    reductions depend on it; test_every_other_output_is_bitwise_the_counterparts compares bitwise where they do not);
    the slice lies inside vb.flat."""
    from diff_gaussian_rasterization.parallel import ViewBatch

    sc = scenegen.make_scene(300, 96, 64, 8, sh_degree=1, views=3, seed=4)
    d = scenegen.to_torch(sc, torch.device("cuda"))
    params = {k: d[k] for k in ("means3D", "scales", "rotations", "opacities", "shs", "semantic_feature")}
    out = {}
    for absgrad in (False, True):
        vb = ViewBatch(params, absgrad=absgrad)
        vb.zero_()
        expect = torch.zeros(sc.P, device="cuda")
        for i, cam in enumerate(sc.cameras):
            color, feat, radii, depth, ctx = vb.forward(_settings(sc, cam))
            gc, gf, gd = (torch.from_numpy(u).cuda() for u in scenegen.upstream_grads(cam.image_height,
                                                                                    cam.image_width, 8, 20 + i))
            vb.backward(ctx, gc, gf, gd)
            if absgrad:
                expect += vb.mean2D_abs[:, :2].norm(dim=1) * (radii > 0)
                assert bool((vb.mean2D_abs[radii == 0] == 0).all())
        out[absgrad] = vb
        if absgrad:
            assert torch.allclose(vb.grad_accum_abs, expect, rtol=1e-6, atol=0)
            assert bool((vb.grad_accum_abs >= vb.grad_accum * (1 - 1e-5)).all())
            o = vb.n_param + 2 * vb.P
            assert vb.flat.numel() == o + vb.P
            assert vb.grad_accum_abs.data_ptr() == vb.flat[o:].data_ptr()
    a, b = out[False], out[True]
    assert torch.equal(a.denom, b.denom)
    n = a.flat.numel()
    assert torch.allclose(a.flat, b.flat[:n], rtol=1e-4, atol=1e-5 * float(a.flat.abs().max()))


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 16])
@pytest.mark.parametrize("C", [0, 3, 128])
@pytest.mark.parametrize("P", [1, 1000, 200_000])
def test_densify_with_abs_grad_matches_the_restatement(P, C, M):
    from test_densify import EXTENT, MAX_GRAD, MIN_OPACITY, assert_matches, clone_state, gen, make_state

    st, ga, dn = make_state(P, C, M, seed=P + 7 * C + M + 1)
    g = torch.Generator().manual_seed(P + C)
    gaa = (ga + torch.rand(P, generator=g).cuda() * dn * 6e-4).contiguous()
    abs_grad = 5e-4
    for screen in (None, 20):
        a, b = clone_state(st), clone_state(st)
        ga_, gb_ = gen(3), gen(3)
        na = a.densify_and_prune(MAX_GRAD, MIN_OPACITY, EXTENT, screen, grad_accum=ga, denom=dn, generator=ga_,
                                 abs_grad=abs_grad, grad_accum_abs=gaa)
        info = {}
        nb = ref_absgrad.densify_and_prune(b, MAX_GRAD, abs_grad, MIN_OPACITY, EXTENT, screen, ga, gaa, dn,
                                           generator=gb_, info=info)
        assert_matches(a, b, na, nb, info, ga_, gb_)
        if P >= 1000:
            # the rule changes the plan: AbsGS splits Gaussians the 3DGS rule leaves alone, and vice versa
            scaling = torch.exp(st.raw["scaling"])
            _, split = ref_absgrad.absgs_masks(ga, gaa, dn, scaling, MAX_GRAD, abs_grad, st.percent_dense * EXTENT)
            g3 = ga / dn
            g3[g3.isnan()] = 0
            split3 = (g3 >= MAX_GRAD) & (scaling.max(1).values > st.percent_dense * EXTENT)
            assert bool((split & ~split3).any()) and bool((split3 & ~split).any())


@pytest.mark.gpu
def test_densify_with_abs_grad_makes_one_host_sync_and_none_changes_nothing():
    from test_densify import EXTENT, MAX_GRAD, MIN_OPACITY, _count_syncs, assert_matches, clone_state, gen, make_state
    import ref_densify

    st, ga, dn = make_state(20_000, 32, 16, seed=3)
    gaa = ga * 3
    a = clone_state(st)
    g = gen(2)
    syncs = _count_syncs(lambda: a.densify_and_prune(MAX_GRAD, MIN_OPACITY, EXTENT, 20, grad_accum=ga, denom=dn,
                                                     generator=g, abs_grad=1e-3, grad_accum_abs=gaa))
    assert len(syncs) == 1, syncs
    # abs_grad=None ignores a given statistic: bitwise the 3DGS plan
    a, b = clone_state(st), clone_state(st)
    ga_, gb_ = gen(4), gen(4)
    na = a.densify_and_prune(MAX_GRAD, MIN_OPACITY, EXTENT, 20, grad_accum=ga, denom=dn, generator=ga_,
                             grad_accum_abs=gaa)
    info = {}
    nb = ref_densify.densify_and_prune(b, MAX_GRAD, MIN_OPACITY, EXTENT, 20, grad_accum=ga, denom=dn, generator=gb_,
                                       info=info)
    assert_matches(a, b, na, nb, info, ga_, gb_)


@pytest.mark.gpu
@pytest.mark.parametrize("antialiasing", [False, True])
@pytest.mark.parametrize("feature_geometry", [False, True])
def test_autograd_rasterizer(antialiasing, feature_geometry):
    """AbsGradGaussianRasterizer: means2D_abs.grad is the binding's statistic and every other gradient, the camera's
    included, is GaussianRasterizer's (AntialiasedGaussianRasterizer's)."""
    import diff_gaussian_rasterization as dgr

    sc = scenegen.make_scene(200, 80, 64, 8, sh_degree=2, seed=7)
    cam = sc.cameras[0]
    d = scenegen.to_torch(sc, torch.device("cuda"))
    gc, gf, gd = (torch.from_numpy(u).cuda() for u in scenegen.upstream_grads(64, 80, 8, 3))

    def run(cls, absgrad):
        rs = _settings(sc, cam)
        rs = rs._replace(viewmatrix=rs.viewmatrix.clone().requires_grad_())
        leaves = {k: d[k].clone().requires_grad_() for k in ("means3D", "shs", "semantic_feature", "opacities",
                                                             "scales", "rotations")}
        m2 = torch.zeros(sc.P, 3, device="cuda", requires_grad=True)
        m2a = torch.zeros(sc.P, 3, device="cuda", requires_grad=True)
        if cls is dgr.AbsGradGaussianRasterizer:
            r = cls(rs, feature_geometry=feature_geometry, antialiasing=antialiasing)
        elif antialiasing:
            r = dgr.AntialiasedGaussianRasterizer(rs, feature_geometry=feature_geometry)
        else:
            r = dgr.GaussianRasterizer(rs, feature_geometry=feature_geometry)
        kw = dict(means2D_abs=m2a) if absgrad else {}
        color, feat, radii, depth = r(means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"],
                                      shs=leaves["shs"], semantic_feature=leaves["semantic_feature"],
                                      scales=leaves["scales"], rotations=leaves["rotations"], **kw)
        ((color * gc).sum() + (feat * gf).sum() + (depth * gd).sum()).backward()
        grads = {k: v.grad for k, v in leaves.items()}
        grads["means2D"], grads["viewmatrix"] = m2.grad, rs.viewmatrix.grad
        return (color, feat, radii, depth), grads, m2a.grad

    base_out, base, _ = run(dgr.GaussianRasterizer, False)
    out, new, abs_grad = run(dgr.AbsGradGaussianRasterizer, True)
    for x, y in zip(base_out, out):
        assert torch.equal(x, y)
    for k in base:
        # the composite reduces with float atomics: equal up to their order
        s = float(base[k].abs().max())
        assert torch.allclose(base[k], new[k], rtol=1e-4, atol=1e-5 * s + 1e-12), k
    assert abs_grad is not None and bool((abs_grad[:, :2] > 0).any()) and bool((abs_grad[:, 2] == 0).all())
    # the binding's statistic for the same view
    from diff_gaussian_rasterization import _C

    e = torch.empty(0, device="cuda")
    rs = _settings(sc, cam)
    fwd = _C.rasterize_gaussians_antialiased if antialiasing else _C.rasterize_gaussians
    R, color, feat, depth, radii, geom, binning, img = fwd(
        rs.bg, d["means3D"], e, d["semantic_feature"], d["opacities"], d["scales"], d["rotations"], 1.0, e,
        rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, 64, 80, d["shs"], 2, rs.campos, False, False)
    ref = _C.rasterize_gaussians_backward_absgrad(
        rs.bg, d["means3D"], radii, e, d["semantic_feature"], d["scales"], d["rotations"], 1.0, e, rs.viewmatrix,
        rs.projmatrix, rs.tanfovx, rs.tanfovy, gc, gf, gd, d["shs"], 2, rs.campos, geom, R, binning, img, False,
        semantic_feature=d["semantic_feature"] if feature_geometry else None, antialiasing=antialiasing)[12]
    s = float(ref.abs().max())
    assert torch.allclose(abs_grad, ref, rtol=1e-4, atol=1e-5 * s)


@pytest.mark.gpu
def test_absgs_training_loop():
    """AbsGS's reference loop: autograd with screenspace_points and screenspace_points_abs, add_densification_stats on
    both (torch.norm of the first two columns where visible), then densify_and_prune with abs_grad on those statistics."""
    import diff_gaussian_rasterization as dgr
    from diff_gaussian_rasterization.trainer import GaussianState

    sc = scenegen.make_scene(400, 64, 48, 0, sh_degree=0, views=3, seed=12)
    d = scenegen.to_torch(sc, torch.device("cuda"))
    xyz = d["means3D"].clone().requires_grad_()
    P = sc.P
    ga, gaa, dn = (torch.zeros(P, 1, device="cuda") for _ in range(3))
    for cam in sc.cameras:
        rs = _settings(sc, cam)
        pts = torch.zeros(P, 3, device="cuda", requires_grad=True)
        pts_abs = torch.zeros(P, 3, device="cuda", requires_grad=True)
        color, _, radii, _ = dgr.AbsGradGaussianRasterizer(rs)(
            means3D=xyz, means2D=pts, means2D_abs=pts_abs, opacities=d["opacities"], shs=d["shs"], scales=d["scales"],
            rotations=d["rotations"])
        color.square().mean().backward()
        f = radii > 0
        ga[f] += torch.norm(pts.grad[f, :2], dim=-1, keepdim=True)
        gaa[f] += torch.norm(pts_abs.grad[f, :2], dim=-1, keepdim=True)
        dn[f] += 1
    assert bool((gaa >= ga * (1 - 1e-5)).all()) and bool((gaa > ga).any())
    st = GaussianState(d["means3D"], d["shs"][:, :1].contiguous(), d["shs"][:, 1:].contiguous(),
                       torch.logit(d["opacities"]), torch.log(d["scales"]), d["rotations"],
                       torch.zeros(P, 1, 0, device="cuda"))
    thr = float(torch.quantile((gaa / dn)[dn > 0], 0.8))
    n = st.densify_and_prune(1e9, 0.005, 1.0, None, grad_accum=ga.reshape(-1), denom=dn.reshape(-1),
                             abs_grad=thr, grad_accum_abs=gaa.reshape(-1))
    assert n > P
