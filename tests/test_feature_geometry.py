"""Feature gradients into geometry: the opt-in feature term of dL/dalpha (f3dgs_backward_feature_geometry,
f3dgs_backward_accum_feature_geometry, rasterize_gaussians_backward_feature_geometry, GaussianRasterizer(...,
feature_geometry=True), ViewBatch.backward(..., feature_geometry=True)).

The colour term is reference-validated, and the feature term is the same recurrence with one channel d_ip = f_i . G_p
and no background.  So with colours_precomp = X, features = X (or k stacked copies of X, each with G / k), background
0, the feature-geometry backward of (dL/dpix = 0, dL/dfeature = G) must give the geometric gradients of the ordinary
backward of (dL/dpix = G, dL/dfeature = 0), camera included.

The independent oracle is a float64 torch autograd model of the term over the composite's own records and blended
pairs (blend_weights.composite_model), with a per-Gaussian bar derived there; a dropped pair exceeds it.

CPU: the entries' argument checks.  GPU: the model against generic random features at C = 1, 5, 40, 130, 132 (scalar and
16-byte row loads, the 32-, 64- and 128-channel kernels), with the camera gradient against camera_grad_model; the
identity above, each side against the model, on the regime scenes at C = 3, 39, 129 and 2049; additivity, zero map gradients and the unaffected outputs on every new entry, float16
features and maps; the old path's zero camera gradient on a feature-only loss; autograd, view batches; and a pose
recovered from a feature map alone.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import scenegen

F32, F16 = 0, 1  # F3DGS_F32, F3DGS_F16
OUTS = ("mean2D", "conic", "opacity", "color", "feat", "mean3D", "cov3D", "sh", "scale", "rot", "dz")
GEOM = ("mean2D", "conic", "opacity", "mean3D", "cov3D", "scale", "rot", "camera")
UNAFFECTED = ("feat", "color", "dz")


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_backward_scratch_bytes.restype = ctypes.c_size_t
    return L


# ------------------------------------------------------------------------------------------------------------ CPU
def _fake(i, fake=1 << 40):
    return ctypes.c_void_p(fake + i * (1 << 20))


def _assign_args(P=5, C=4, sf=50, sf_dtype=F32, map_dtype=F32, scale=1.0, camera=None):
    """f3dgs_backward_feature_geometry's arguments with distinct fake device addresses (the checks fail first)."""
    f, null = ctypes.c_float, ctypes.c_void_p(0)
    sfp = _fake(sf) if sf is not None else null
    return [P, 0, 1, 10, C, _fake(0), 64, 64, _fake(1), _fake(2), null, sfp, sf_dtype, _fake(3), f(1.0), _fake(4), null,
            _fake(5), _fake(6), _fake(7), f(0.5), f(0.5), _fake(8), _fake(9), _fake(10), _fake(11), _fake(12),
            _fake(13), map_dtype, f(scale), _fake(14), _fake(15), _fake(16), _fake(17), _fake(18), _fake(19), _fake(20),
            _fake(21), _fake(22), _fake(23), _fake(24), _fake(25), 0, null, camera if camera is not None else null]


def _accum_args(P=5, C=4, sf=50, sf_dtype=F32, map_dtype=F32, scale=1.0, camera=None):
    f, null = ctypes.c_float, ctypes.c_void_p(0)
    sfp = _fake(sf) if sf is not None else null
    return [P, 0, 1, 10, C, _fake(0), 64, 64, _fake(1), _fake(2), null, sfp, sf_dtype, _fake(3), f(1.0), _fake(4),
            null, _fake(5), _fake(6), _fake(7), f(0.5), f(0.5), _fake(8), _fake(9), _fake(10), _fake(11), _fake(12),
            _fake(13), map_dtype, f(scale), _fake(14), _fake(30), _fake(15), null, _fake(16), _fake(17), null, _fake(18),
            _fake(19), _fake(20), _fake(21), _fake(22), _fake(23), null, 0, null,
            camera if camera is not None else null]


@pytest.mark.parametrize("entry", ["f3dgs_backward_feature_geometry", "f3dgs_backward_accum_feature_geometry"])
def test_entries_reject_bad_arguments_before_any_launch(lib, entry):
    fn = getattr(lib, entry)
    mk = _assign_args if "accum" not in entry else _accum_args
    err = lambda: lib.f3dgs_last_error().decode()  # noqa: E731
    assert fn(*mk(sf=None)) == -1 and err() == f"{entry}: NULL semantic_feature"
    for kw in (dict(sf_dtype=2), dict(map_dtype=-1)):
        assert fn(*mk(**kw)) == -1 and err() == f"{entry}: unknown dtype code", kw
    for s in (0.0, float("inf"), float("nan")):
        assert fn(*mk(map_dtype=F16, scale=s)) == -1 and "dL_dfeaturepix_scale must be finite and nonzero" in err(), s
    outs = (15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25) if "accum" not in entry else (30, 15, 16, 17, 18, 19, 20, 21,
                                                                                      22, 23)
    for i in outs:  # semantic_feature inside each output (and the accumulating entry's scratch)
        assert fn(*mk(sf=i)) == -1, i
        assert "semantic_feature overlaps an output" in err(), (i, err())
    assert fn(*mk(sf_dtype=F16, sf=15)) == -1 and "overlaps" in err()
    assert fn(*mk(camera=_fake(50))) == -1 and "overlaps" in err()  # the camera gradient is an output too
    # the counterpart's own checks still apply; C == 0 needs no features; P == 0 is a no-op
    assert fn(*mk(P=-1)) == -1
    assert fn(*mk(P=0)) == 0


def test_python_surface():
    import inspect

    import diff_gaussian_rasterization as dgr
    from diff_gaussian_rasterization.parallel import ViewBatch

    assert hasattr(dgr._C, "rasterize_gaussians_backward_feature_geometry")
    assert list(inspect.signature(dgr.GaussianRasterizer.__init__).parameters) == ["self", "raster_settings",
                                                                                    "feature_geometry"]
    assert list(inspect.signature(dgr.rasterize_gaussians_feature_geometry).parameters) == list(
        inspect.signature(dgr.rasterize_gaussians).parameters)
    assert inspect.signature(ViewBatch.backward).parameters["feature_geometry"].default is False


# ------------------------------------------------------------------------------------------------------------ GPU
def _forward(sc, cam, feats, colors=None):
    """Forward through the binding -> dict of what the backward entries need."""
    from diff_gaussian_rasterization import _C

    dev = torch.device("cuda")
    d = scenegen.to_torch(sc, dev)
    e = torch.empty(0, device=dev)
    vm, pm, cp = (torch.tensor(a, device=dev).contiguous() for a in (cam.viewmatrix, cam.projmatrix, cam.campos))
    bg = torch.zeros(3, device=dev) if colors is not None else d["bg"]
    shs = e if colors is not None else d["shs"]
    cols = colors if colors is not None else e
    R, color, fmap, depth, radii, geom, binning, img = _C.rasterize_gaussians(
        bg, d["means3D"], cols, feats, d["opacities"], d["scales"], d["rotations"], 1.0, e, vm, pm, cam.tanfovx,
        cam.tanfovy, cam.image_height, cam.image_width, shs, sc.sh_degree, cp, False, False)
    return dict(sc=sc, cam=cam, d=d, bg=bg, shs=shs, cols=cols, feats=feats, vm=vm, pm=pm, cp=cp, R=R, radii=radii,
                geom=geom, binning=binning, img=img, fmap=fmap, P=sc.P, M=sc.shs.shape[1] if colors is None else 0,
                C=feats.shape[-1] if feats.numel() else 0)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None and t.numel() else 0)


def _assign(lib, f, gc, gf, gd, new, camera=False, gf_half=False, scale=1.0):
    """One assigning backward through ctypes: new -> f3dgs_backward_feature_geometry (features of f's forward), else
    f3dgs_backward(_f16)(_cam) -> dict of outputs."""
    dev = torch.device("cuda")
    P, M, C, sc, cam = f["P"], f["M"], f["C"], f["sc"], f["cam"]
    o = {k: torch.zeros(P, n, device=dev) for k, n in (("mean2D", 3), ("conic", 4), ("opacity", 1), ("color", 3),
                                                        ("feat", C), ("mean3D", 3), ("cov3D", 6), ("scale", 3),
                                                        ("rot", 4), ("dz", 1))}
    o["sh"] = torch.zeros(P, M, 3, device=dev)
    o["camera"] = torch.zeros(35, device=dev)
    d, W, H = f["d"], cam.image_width, cam.image_height
    head = [P, sc.sh_degree, M, f["R"], C, _ptr(f["bg"]), W, H, _ptr(d["means3D"]), _ptr(f["shs"]), _ptr(f["cols"])]
    mid = [_ptr(d["scales"]), ctypes.c_float(1.0), _ptr(d["rotations"]), ctypes.c_void_p(0), _ptr(f["vm"]),
           _ptr(f["pm"]), _ptr(f["cp"]), ctypes.c_float(cam.tanfovx), ctypes.c_float(cam.tanfovy), _ptr(f["radii"]),
           _ptr(f["geom"]), _ptr(f["binning"]), _ptr(f["img"]), _ptr(gc)]
    tail = [_ptr(gd)] + [_ptr(o[k]) for k in OUTS] + [0, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)]
    sf = f["feats"]
    if new:
        args = head + [_ptr(sf), F16 if sf.dtype == torch.float16 else F32] + mid + \
            [_ptr(gf), F16 if gf_half else F32, ctypes.c_float(scale)] + tail + [_ptr(o["camera"]) if camera else
                                                                                 ctypes.c_void_p(0)]
        entry = "f3dgs_backward_feature_geometry"
    else:
        args = head + [ctypes.c_void_p(0)] + mid + [_ptr(gf)] + ([ctypes.c_float(scale)] if gf_half else []) + tail
        entry = "f3dgs_backward" + ("_cam" if camera else "") + ("_f16" if gf_half else "")
        if camera:
            args.append(_ptr(o["camera"]))
    rc = getattr(lib, entry)(*args)
    assert rc == 0, lib.f3dgs_last_error()
    torch.cuda.synchronize()
    return o


def _accum(lib, f, gc, gf, gd, new, camera=False, repeat=1):
    """The accumulating entry (new: _feature_geometry) `repeat` times into zeroed buffers -> dict of outputs."""
    dev = torch.device("cuda")
    P, M, C, sc, cam = f["P"], f["M"], f["C"], f["sc"], f["cam"]
    o = {k: torch.zeros(P, n, device=dev) for k, n in (("opacity", 1), ("feat", C), ("mean3D", 3), ("scale", 3),
                                                        ("rot", 4), ("mean2D", 3), ("grad_accum", 1), ("denom", 1))}
    o["sh"] = torch.zeros(P, M, 3, device=dev)
    o["camera"] = torch.zeros(35, device=dev)
    scratch = torch.empty(lib.f3dgs_backward_scratch_bytes(P), dtype=torch.uint8, device=dev)
    d, W, H = f["d"], cam.image_width, cam.image_height
    head = [P, sc.sh_degree, M, f["R"], C, _ptr(f["bg"]), W, H, _ptr(d["means3D"]), _ptr(f["shs"]), ctypes.c_void_p(0)]
    mid = [_ptr(d["scales"]), ctypes.c_float(1.0), _ptr(d["rotations"]), ctypes.c_void_p(0), _ptr(f["vm"]),
           _ptr(f["pm"]), _ptr(f["cp"]), ctypes.c_float(cam.tanfovx), ctypes.c_float(cam.tanfovy), _ptr(f["radii"]),
           _ptr(f["geom"]), _ptr(f["binning"]), _ptr(f["img"]), _ptr(gc)]
    tail = [_ptr(gd), _ptr(scratch), _ptr(o["opacity"]), ctypes.c_void_p(0), _ptr(o["feat"]), _ptr(o["mean3D"]),
            ctypes.c_void_p(0), _ptr(o["sh"]), _ptr(o["scale"]), _ptr(o["rot"]), _ptr(o["mean2D"]),
            _ptr(o["grad_accum"]), _ptr(o["denom"]), ctypes.c_void_p(0), 0,
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)]
    sf = f["feats"]
    for _ in range(repeat):
        if new:
            args = head + [_ptr(sf), F16 if sf.dtype == torch.float16 else F32] + mid + [_ptr(gf), F32,
                                                                                        ctypes.c_float(1.0)] + tail
            args.append(_ptr(o["camera"]) if camera else ctypes.c_void_p(0))
            entry = "f3dgs_backward_accum_feature_geometry"
        else:
            args = head + mid + [_ptr(gf)] + tail
            entry = "f3dgs_backward_accum" + ("_cam" if camera else "")
            if camera:
                args.append(_ptr(o["camera"]))
        rc = getattr(lib, entry)(*args)
        assert rc == 0, lib.f3dgs_last_error()
    torch.cuda.synchronize()
    return o


def _grads(cam, C, seed=7):
    dev = torch.device("cuda")
    return tuple(torch.from_numpy(a).to(dev) for a in scenegen.upstream_grads(cam.image_height, cam.image_width, C,
                                                                              seed))


def _close(a, b, label, rel=1e-4):
    """Within rounding of float32 reductions whose order differs: per entry against the larger magnitude and a floor at
    the tensor's scale."""
    a, b = a.double().cpu(), b.double().cpu()
    scale = float(torch.maximum(a.abs().max(), b.abs().max())) if a.numel() else 0.0
    bar = rel * torch.maximum(a.abs(), b.abs()) + 1e-5 * scale + 1e-30
    ratio = float(((a - b).abs() / bar).max()) if a.numel() else 0.0
    assert ratio <= 1.0, (label, ratio)
    return ratio


def _block_scene(C=8):
    from test_camera_grad import _block_scene as blocks

    return blocks(C=C)


def _identity_scene(name):
    from test_gpu_regimes import anisotropic, make

    if name == "small":
        sc = scenegen.make_config("small")
        return sc, sc.cameras[0]
    if name == "fx_ne_fy":
        sc, cam = make("inside", 0)
        return sc, anisotropic(cam, 0.7)
    return make(name, 0)


def _feature_model(view, dfn, C):
    """blend_weights.composite_model of the feature term (no background) on a view of test_blend_weights.DeviceView."""
    import blend_weights as bw

    return bw.composite_model(view.pairs, view.w, view.base["rec"], view.P, dfn, C)


def _geom6(o):
    """The composite's six geometric gradients of an _assign result, in composite_model's order."""
    import blend_weights as bw

    return bw.geom6(o["mean2D"], o["conic"], o["opacity"])


def _model_ratio(ours, ref, bar):
    import blend_weights as bw

    err = (ours.double().to(ref.device) - ref).abs()
    return float(bw._ratio(err, bar).max())


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 13, 43, 683])
@pytest.mark.parametrize("name", ["small", "inside", "needles", "fx_ne_fy"])
def test_feature_term_is_the_colour_term_of_the_same_values(lib, name, k):
    """colours_precomp = X, features = k copies of X with G / k each, background 0: the feature-geometry backward of
    (0, G) and the ordinary backward of (G, 0) both match the float64 model of their own inputs (_feature_model) within
    its per-Gaussian bar.  C = 3k: 3 (one 32-channel chunk), 39 (one 64-channel chunk), 129 (two 128-channel chunks, the
    last one channel wide), 2049 (seventeen, the last one channel wide)."""
    from test_blend_weights import DeviceView

    dev = torch.device("cuda")
    sc, cam = _identity_scene(name)
    view = DeviceView(sc, cam, 512)
    P, H, W = sc.P, cam.image_height, cam.image_width
    gen = torch.Generator().manual_seed(11)
    X = torch.rand(P, 3, generator=gen).to(dev)
    G = torch.randn(3, H, W, generator=gen).to(dev)
    feats = X.repeat(1, k).reshape(P, 1, 3 * k).contiguous()
    f = _forward(sc, cam, feats, colors=X)
    zc, zd = torch.zeros(3, H, W, device=dev), torch.zeros(1, H, W, device=dev)
    zf = torch.zeros(3 * k, H, W, device=dev)
    gk = G / k  # float32, as the feature path reads it
    gf = gk.repeat(k, 1, 1).contiguous()
    ref = _assign(lib, f, G, zf, zd, new=False)
    ours = _assign(lib, f, zc, gf, zd, new=True)

    def dots(g, copies):  # k copies of X . g at every pair, in float64
        Xd, g = X.double(), g.reshape(3, -1).double()
        return lambda gid, pix: (copies * (Xd[gid] * g[:, pix].t()).sum(1),
                                 copies * (Xd[gid].abs() * g[:, pix].t().abs()).sum(1))

    colour_model = _feature_model(view, dots(G, 1), 3)
    feature_model = _feature_model(view, dots(gk, k), 3 * k)
    r_ref = _model_ratio(_geom6(ref), *colour_model)
    r_ours = _model_ratio(_geom6(ours), *feature_model)
    print(f"[{name} C={3 * k}] worst |err|/bar: feature term {r_ours:.3g}, colour term {r_ref:.3g}")
    assert r_ref <= 1.0 and r_ours <= 1.0, (r_ours, r_ref)
    assert bool(ref["opacity"].abs().sum() > 0)
    assert bool((ours["color"] == 0).all()) and bool((ours["dz"] == 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 5, 40, 130, 132])
def test_feature_term_against_the_float64_model(lib, C):
    """Generic random features and map gradient on small scenes (40 Gaussians, 64x48): the native dL/dmean2D, dL/dconic
    and dL/dopacity of a feature-only loss against _feature_model, and the camera gradient against camera_grad_model on
    those intermediates within test_camera_grad's bars.  C = 1, 5, 130 read feature rows one channel at a time; C = 40
    (the 64-channel kernel) and 132 (two 128-channel chunks) with 16-byte loads."""
    import camera_grad_model as cgm
    from test_blend_weights import DeviceView
    from test_cabi_gpu import Layout

    dev = torch.device("cuda")
    for seed in (1, 2, 3):
        sc = scenegen.make_scene(40, 64, 48, C, sh_degree=1, seed=seed)
        cam = sc.cameras[0]
        P, W, H = sc.P, cam.image_width, cam.image_height
        view = DeviceView(sc, cam, 64)
        feats = torch.from_numpy(np.ascontiguousarray(sc.features)).to(dev)
        f = _forward(sc, cam, feats)
        gf = torch.randn(C, H, W, generator=torch.Generator().manual_seed(seed)).to(dev)
        zc, zd = torch.zeros(3, H, W, device=dev), torch.zeros(1, H, W, device=dev)
        o = _assign(lib, f, zc, gf, zd, new=True, camera=True)
        Fd, Gd = feats.reshape(P, C).double(), gf.reshape(C, -1).double()

        def dots(gid, pix):
            return (Fd[gid] * Gd[:, pix].t()).sum(1), (Fd[gid].abs() * Gd[:, pix].t().abs()).sum(1)

        ref, bar = _feature_model(view, dots, C)
        r = _model_ratio(_geom6(o), ref, bar)
        assert bool(ref[:, 5].abs().sum() > 0)
        # negative control: the model without one (Gaussian, pixel) pair of the Gaussian that blends the most pixels
        def dropped(gid, pix):
            d, dabs = dots(gid, pix)
            on = torch.nonzero(gid == torch.bincount(gid).argmax()).reshape(-1)
            d = d.clone()
            d[on[torch.argmax(d[on].abs())]] = 0.0
            return d, dabs

        assert _model_ratio(_geom6(o), *_feature_model(view, dropped, C)) > 1.0

        L = Layout()
        assert lib.f3dgs_get_layout(P, W, H, f["R"], ctypes.byref(L)) == 0
        cov = f["geom"][L.geom_cov3d:L.geom_cov3d + P * 24].view(torch.float32).view(P, 6).cpu()
        t = cgm.terms(sc.means3D, cov, f["vm"].cpu(), f["pm"].cpu(), f["cp"].cpu(),
                      [o["mean2D"].cpu(), o["conic"].cpu(), torch.zeros(P, 3), torch.zeros(P)], W, H, cam.tanfovx,
                      cam.tanfovy, sc.sh_degree, shs=sc.shs, visible=(f["radii"] > 0).cpu())
        cref, scale = cgm.camera_vector(t), cgm.camera_scale(t)
        cbar = 1e-5 * scale + 1e-7 * float(cgm.camera_scale(t, needles=False).max())
        ours = o["camera"].cpu().double()
        rc = float(((ours - cref).abs() / cbar).max())
        print(f"[C={C} seed={seed}] worst |err|/bar: composite {r:.3g}, camera {rc:.3g}")
        assert r <= 1.0 and rc <= 1.0, (r, rc)
        assert bool(ours.abs().sum() > 0)


@pytest.mark.gpu
@pytest.mark.parametrize("camera", [False, True])
def test_zero_map_gradient_and_unaffected_outputs_are_bitwise(lib, camera):
    """On a view whose composite reduces each per-Gaussian value with one atomic (so two runs agree bitwise): with a zero
    map gradient every output of the new entries is the old entry's; with any map gradient dL/dfeature, dL/dcolor and
    dL/dz are."""
    dev = torch.device("cuda")
    sc, cam = _block_scene()
    f = _forward(sc, cam, scenegen.to_torch(sc, dev)["semantic_feature"])
    gc, gf, gd = _grads(cam, 8)
    old = _assign(lib, f, gc, gf, gd, new=False, camera=camera)
    zero = _assign(lib, f, gc, torch.zeros_like(gf), gd, new=True, camera=camera)
    old0 = _assign(lib, f, gc, torch.zeros_like(gf), gd, new=False, camera=camera)
    for k in OUTS + ("camera",):
        assert torch.equal(zero[k], old0[k]), k
    new = _assign(lib, f, gc, gf, gd, new=True, camera=camera)
    for k in UNAFFECTED:
        assert torch.equal(new[k], old[k]), k
    assert not torch.equal(new["opacity"], old["opacity"])
    # accumulating entries, called twice into the same buffers
    old = _accum(lib, f, gc, gf, gd, new=False, camera=camera, repeat=2)
    zero = _accum(lib, f, gc, torch.zeros_like(gf), gd, new=True, camera=camera, repeat=2)
    old0 = _accum(lib, f, gc, torch.zeros_like(gf), gd, new=False, camera=camera, repeat=2)
    for k in old0:
        assert torch.equal(zero[k], old0[k]), k
    new = _accum(lib, f, gc, gf, gd, new=True, camera=camera, repeat=2)
    assert torch.equal(new["feat"], old["feat"])
    assert not torch.equal(new["opacity"], old["opacity"])
    assert not torch.equal(new["grad_accum"], old["grad_accum"])  # the densification statistics see the term


@pytest.mark.gpu
@pytest.mark.parametrize("scene", ["blocks", "small"])
@pytest.mark.parametrize("camera", [False, True])
def test_additivity(lib, scene, camera):
    """new(Gc, Gf) = old(Gc, 0) + new(0, Gf) within rounding, for the assigning and accumulating entries.  On the
    one-atomic view the Gaussians are isotropic with identity rotations, so their scale and rotation gradients are
    rounding noise of cancelling terms: there only the composite's outputs, dL/dmeans3D and the camera are compared."""
    dev = torch.device("cuda")
    if scene == "blocks":
        sc, cam = _block_scene()
    else:
        sc = scenegen.make_config("small")
        cam = sc.cameras[0]
    f = _forward(sc, cam, scenegen.to_torch(sc, dev)["semantic_feature"])
    gc, gf, gd = _grads(cam, f["C"])
    zc, zd = torch.zeros_like(gc), torch.zeros_like(gd)
    both = _assign(lib, f, gc, gf, gd, new=True, camera=camera)
    colour = _assign(lib, f, gc, torch.zeros_like(gf), gd, new=False, camera=camera)
    feature = _assign(lib, f, zc, gf, zd, new=True, camera=camera)
    keys = [k for k in GEOM if (camera or k != "camera") and (scene == "small" or k not in ("cov3D", "scale", "rot"))]
    for k in keys:
        _close(both[k], colour[k] + feature[k], (scene, "assign", k))
    assert bool(feature["opacity"].abs().sum() > 0)
    both = _accum(lib, f, gc, gf, gd, new=True, camera=camera)
    colour = _accum(lib, f, gc, torch.zeros_like(gf), gd, new=False, camera=camera)
    feature = _accum(lib, f, zc, gf, zd, new=True, camera=camera)
    for k in [k for k in ("opacity", "mean3D", "mean2D", "camera", "scale", "rot") if k in keys]:
        _close(both[k], colour[k] + feature[k], (scene, "accum", k))


@pytest.mark.gpu
def test_float16_features_and_scaled_float16_map(lib):
    """float16 features with a float16 map h and scale s: bitwise the float32 call on the upcast features and the map
    s * float(h) (on the one-atomic view)."""
    dev = torch.device("cuda")
    sc, cam = _block_scene()
    d = scenegen.to_torch(sc, dev)
    h16 = d["semantic_feature"].half()
    gc, gf, gd = _grads(cam, 8)
    s = 3.0e-3
    gh = (gf / s).half()
    a = _assign(lib, _forward(sc, cam, h16), gc, gh, gd, new=True, camera=True, gf_half=True, scale=s)
    b = _assign(lib, _forward(sc, cam, h16.float()), gc, gh.float() * s, gd, new=True, camera=True)
    for k in OUTS + ("camera",):
        assert torch.equal(a[k], b[k]), k


@pytest.mark.gpu
def test_feature_only_loss_moves_the_camera_only_on_the_new_path(lib):
    dev = torch.device("cuda")
    sc = scenegen.make_config("small")
    cam = sc.cameras[0]
    f = _forward(sc, cam, scenegen.to_torch(sc, dev)["semantic_feature"])
    gc, gf, gd = _grads(cam, f["C"])
    zc, zd = torch.zeros_like(gc), torch.zeros_like(gd)
    old = _assign(lib, f, zc, gf, zd, new=False, camera=True)
    assert bool((old["camera"] == 0).all()) and bool((old["mean3D"] == 0).all())
    new = _assign(lib, f, zc, gf, zd, new=True, camera=True)
    assert bool(new["camera"].abs().sum() > 0) and bool(new["mean3D"].abs().sum() > 0)


@pytest.mark.gpu
def test_autograd_and_binding(lib):
    """GaussianRasterizer(feature_geometry=True) through autograd gives the binding's and the C entry's gradients; the
    default rasterizer gives the old ones (on the one-atomic view, bitwise)."""
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer, _C

    dev = torch.device("cuda")
    sc, cam = _block_scene()
    gc, gf, gd = _grads(cam, 8)
    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))
    e = torch.Tensor([])
    results = {}
    for fg in (False, True):
        d = scenegen.to_torch(sc, dev, requires_grad=True)
        m2 = torch.zeros_like(d["means3D"], requires_grad=True)
        color, fmap, radii, depth = GaussianRasterizer(rs, feature_geometry=fg)(
            means3D=d["means3D"], means2D=m2, opacities=d["opacities"], shs=d["shs"],
            semantic_feature=d["semantic_feature"], scales=d["scales"], rotations=d["rotations"])
        ((color * gc).sum() + (fmap * gf).sum() + (depth * gd).sum()).backward()
        results[fg] = (d, m2)
    D = {k: v.detach() for k, v in scenegen.to_torch(sc, dev).items()}
    R, color, fmap, depth, rad, geom, binning, img = _C.rasterize_gaussians(
        rs.bg, D["means3D"], e, D["semantic_feature"], D["opacities"], D["scales"], D["rotations"], 1.0, e,
        rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, cam.image_height, cam.image_width, D["shs"],
        rs.sh_degree, rs.campos, False, False)
    args = (rs.bg, D["means3D"], rad, e, D["semantic_feature"], D["scales"], D["rotations"], 1.0, e, rs.viewmatrix,
            rs.projmatrix, rs.tanfovx, rs.tanfovy, gc, gf, gd, D["shs"], rs.sh_degree, rs.campos, geom, R, binning,
            img, False)
    ref_old = _C.rasterize_gaussians_backward(*args)
    ref_new = _C.rasterize_gaussians_backward_feature_geometry(*args, False)
    assert all(x is None for x in ref_new[9:])
    cam_new = _C.rasterize_gaussians_backward_feature_geometry(*args, True)
    for fg, ref in ((False, ref_old), (True, ref_new)):
        d, m2 = results[fg]
        for key, g in zip(("means3D", "semantic_feature", "shs", "opacities", "scales", "rotations"),
                          (ref[4], ref[2], ref[6], ref[3], ref[7], ref[8])):
            assert torch.equal(d[key].grad, g), (fg, key)
        assert torch.equal(m2.grad, ref[0])
    for i in range(9):
        assert torch.equal(cam_new[i], ref_new[i]), i
    assert not torch.equal(ref_new[3], ref_old[3])
    f = _forward(sc, cam, D["semantic_feature"])
    c_entry = _assign(lib, f, gc, gf, gd, new=True, camera=True)
    assert torch.equal(c_entry["camera"][:16], cam_new[9].reshape(16))
    assert torch.equal(c_entry["opacity"], ref_new[3])


@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
def test_view_batch(lib, half):
    """ViewBatch.backward(feature_geometry=True, camera=True, last=True) over three views: the flat buffer is the sum of
    the views' assigning feature-geometry calls, and each camera gradient is that view's (bitwise on the one-atomic
    view, where the sum over views is the only reordering).  With float16 features and a ScaledGrad map, against the
    float32 call on the upcast inputs."""
    from diff_gaussian_rasterization import GaussianRasterizationSettings, _C
    from diff_gaussian_rasterization.feature_head import ScaledGrad
    from diff_gaussian_rasterization.parallel import ViewBatch

    dev = torch.device("cuda")
    sc, cam = _block_scene()
    d = scenegen.to_torch(sc, dev)
    if half:
        d["semantic_feature"] = d["semantic_feature"].half()
    params = {k: d[k] for k in ("means3D", "scales", "rotations", "opacities", "shs", "semantic_feature")}
    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))
    ups = [_grads(cam, 8, seed=s) for s in (1, 2, 3)]
    s = 1e-2
    if half:
        ups = [(gc, (gf / s).half(), gd) for gc, gf, gd in ups]
    vb = ViewBatch(params)
    vb.zero_()
    cams, ctxs = [], []
    for i, (gc, gf, gd) in enumerate(ups):
        color, feat, radii, depth, ctx = vb.forward(rs)
        g = ScaledGrad(gf, s) if half else gf
        cams.append(vb.backward(ctx, gc, g, gd, camera=True, last=i == 2, feature_geometry=True))
        ctxs.append(ctx)
    vb.all_reduce()
    torch.cuda.synchronize()
    e = torch.Tensor([])
    sf = params["semantic_feature"].float()
    total = {k: torch.zeros_like(params[k], dtype=torch.float32) for k in ("opacities", "means3D", "scales",
                                                                           "rotations", "semantic_feature")}
    for (gc, gf, gd), ctx, cg in zip(ups, ctxs, cams):
        gmap = gf.float() * s if half else gf
        ref = _C.rasterize_gaussians_backward_feature_geometry(
            rs.bg, params["means3D"], ctx.radii, e, sf, params["scales"], params["rotations"], 1.0, e, rs.viewmatrix,
            rs.projmatrix, rs.tanfovx, rs.tanfovy, gc, gmap, gd, params["shs"], rs.sh_degree, rs.campos, ctx.geom,
            ctx.num_rendered, ctx.binning, ctx.img, False, True)
        for x, y in zip(cg, ref[9:]):
            assert torch.equal(x, y)
        for key, idx in (("opacities", 3), ("means3D", 4), ("scales", 7), ("rotations", 8), ("semantic_feature", 2)):
            total[key] += ref[idx].reshape(total[key].shape)
    for key, t in total.items():
        _close(vb.grads[key].float(), t, key, rel=1e-5)


@pytest.mark.gpu
def test_pose_recovery_from_features_alone():
    """Render a C = 16 feature map at a true pose, start 1 degree and 2 % of the camera distance off, and run 100 Adam
    steps on an se3_exp delta of the L2 distance between rendered and target feature maps, colour weight 0, through
    GaussianRasterizer(feature_geometry=True).  It must end within 0.25 degrees and 0.015 (scene units; the camera is
    3.5 away) of the true pose; an H100 ends at 0.049 degrees and 0.0026.  The old path gives this loss no camera
    gradient at all."""
    from diff_gaussian_rasterization import GaussianRasterizer
    from diff_gaussian_rasterization.camera import se3_exp, settings_from_w2c

    dev = torch.device("cuda")
    sc = scenegen.make_scene(3000, 160, 120, 16, sh_degree=1, seed=5, target_radius_px=8.0)
    cam = sc.cameras[0]
    W, H = cam.image_width, cam.image_height
    d = scenegen.to_torch(sc, dev)
    w2c_true = torch.tensor(cam.viewmatrix, device=dev).t().contiguous()

    def render(w2c, fg=True):
        rs = settings_from_w2c(w2c, cam.tanfovx, cam.tanfovy, H, W, d["bg"], sh_degree=sc.sh_degree)
        m2 = torch.zeros_like(d["means3D"])
        return GaussianRasterizer(rs, feature_geometry=fg)(
            means3D=d["means3D"], means2D=m2, opacities=d["opacities"], shs=d["shs"],
            semantic_feature=d["semantic_feature"], scales=d["scales"], rotations=d["rotations"])[1]

    with torch.no_grad():
        target = render(w2c_true)
    dist = float(torch.linalg.norm(torch.tensor(cam.campos)))
    axis = torch.tensor([0.3, -0.8, 0.5], device=dev)
    axis = axis / axis.norm()
    xi0 = torch.cat([0.02 * dist * torch.tensor([0.6, 0.0, -0.8], device=dev), math.radians(1.0) * axis])
    w2c0 = se3_exp(xi0) @ w2c_true

    def errors(w2c):
        D = w2c @ torch.linalg.inv(w2c_true)
        ang = math.degrees(math.acos(max(-1.0, min(1.0, (float(torch.trace(D[:3, :3])) - 1) / 2))))
        return ang, float(torch.linalg.norm(torch.linalg.inv(w2c)[:3, 3] - torch.linalg.inv(w2c_true)[:3, 3]))

    xi = torch.zeros(6, device=dev, requires_grad=True)
    ((render(se3_exp(xi) @ w2c0, fg=False) - target) ** 2).mean().backward()
    assert bool((xi.grad == 0).all())
    opt = torch.optim.Adam([xi], lr=2e-3)
    a0, t0 = errors(w2c0)
    for _ in range(100):
        opt.zero_grad()
        ((render(se3_exp(xi) @ w2c0) - target) ** 2).mean().backward()
        opt.step()
    a1, t1 = errors((se3_exp(xi) @ w2c0).detach())
    print(f"rotation error {a0:.3f} -> {a1:.4f} deg, centre error {t0:.4f} -> {t1:.5f}")
    assert a1 <= 0.25 and t1 <= 0.015, (a0, a1, t0, t1)
