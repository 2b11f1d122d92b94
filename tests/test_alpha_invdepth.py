"""Opacity and inverse-depth maps: f3dgs_forward_alpha_invdepth / f3dgs_backward[_accum]_alpha_invdepth and their torch,
autograd and view-batch surfaces.

    alpha     A_p = 1 - T_final,p          (bitwise 1 - final_T)
    invdepth  I_p = sum_i w_ip / z_i       (w = alpha T, z the record's view depth, 1/z correctly rounded)

The forward is checked bitwise against the forward without the planes (colour, feature map, depth, radii, R, final_T,
n_contrib, the splat records), every pixel of both planes is written (outputs prefilled with NaN), alpha is 1 - final_T
bitwise, and both planes satisfy the per-pixel blend-weight identities of blend_weights.py.

The backward adds, per pixel p with gA = dL/dA_p and gI = dL/dI_p,
    dL/dalpha_i += gA T_final / (1 - alpha_i)                       (the background term with bg.dL/dpix - gA)
    dL/dalpha_i += T_i (1/z_i - B_i) gI,  B_i = alpha_{i+1}/z_{i+1} + (1 - alpha_{i+1}) B_{i+1}
    dL/dz_i     -= sum_p w_ip gI / z_i^2
It is checked per Gaussian against blend_weights.composite_model run with d = c.Gc + z Gd + gI / z and
bg_dot = bg.Gc - gA, dL/dz against its blend-weight identity, and the preprocess outputs against camera_grad_model's
chain.  With gA = gI = 0 every output is bitwise that of the counterpart entry (on the block scene, whose reductions do not
depend on the order of the float atomics).
"""
import ctypes
import inspect
import os
import re

import numpy as np
import pytest
import torch

import blend_weights as bw
import scenegen

F32, F16 = 0, 1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _t(a, dev="cpu"):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None and t.numel() else 0)


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_backward_scratch_bytes.restype = ctypes.c_size_t
    L.f3dgs_launch_count.restype = ctypes.c_ulonglong
    return L


# ------------------------------------------------------------------------------------------------------------ the model
def planes_dfn(rec, Gc, Gd, GI, F=None, Gf=None):
    """colour_depth_dots with the inverse-depth term: d = c.Gc + z Gd + GI / z per pair (GI [HW] float32), and with the
    feature term f.Gf when F [P,C] (the rows the backward reads, as float32 values) and Gf [HW,C] (the map gradient as
    the composite scales it) are given"""
    base = bw.colour_depth_dots(rec, Gc, Gd)
    rz = 1.0 / rec[:, 11].double()
    GI = GI.double().reshape(-1)
    if F is not None:
        F, Gf = F.to(GI.device), Gf.to(GI.device)

    def dfn(gid, pix):
        d, dabs = base(gid, pix)
        t = rz[gid] * GI[pix]
        d, dabs = d + t, dabs + t.abs()
        if F is not None:
            fs, fa = bw.pair_dots(F, Gf, gid, pix)
            d, dabs = d + fs, dabs + fa
        return d, dabs

    return dfn


def planes_model(pairs, w, rec, P, bg, Gc, Gd, GA, GI, F=None, Gf=None):
    """(ref, bar) of the six geometric values with the planes' terms (and the feature term, see planes_dfn).
    Gc [HW,3], Gd, GA, GI [HW]."""
    bgp = Gc.double() * bg.double().to(Gc.device)
    GA = GA.double().reshape(-1)
    # 5 products in d, and the reciprocal's rounding; C more with the feature term
    return bw.composite_model(pairs, w, rec, P, planes_dfn(rec, Gc, Gd, GI, F, Gf), 6 + (0 if F is None else F.shape[1]),
                              (bgp.sum(1) - GA, bgp.abs().sum(1) + GA.abs()))


def dz_check(Wt, rec, ours, Gd, GI, rows=None):
    """dL/dz_g = sum_p w (Gd_p - GI_p / z_g^2) per Gaussian -> worst ratio over the Gaussians `rows` (default all)"""
    P = ours.numel()
    r1, a1, n1 = Wt.terms(Gd.reshape(-1, 1))
    r2, a2, n2 = Wt.terms(GI.reshape(-1, 1))
    z = rec[:, 11].double().reshape(-1, 1).to(r1.device)
    iz2 = torch.where(z > 0, 1.0 / (z * z), torch.zeros_like(z))  # culled Gaussians: z = 0 in the record, no pairs
    return bw.gaussian_ratio(ours.reshape(P, 1).to(r1.device), (r1 - r2 * iz2, a1 + a2 * iz2, n1 + n2 * iz2), Wt.m,
                             rows)


def test_negative_controls_the_model_flags_a_dropped_term():
    """On an oracle view: a result without the 1/z term, or without gA, is outside the planes model's bar; the model of
    zero plane gradients is the default backward's model."""
    from test_blend_weights import _oracle_view

    sc, cam, f, pairs, w = _oracle_view("small")
    rec = _t(bw.oracle_records(f))
    H, W, P = cam.image_height, cam.image_width, sc.P
    gc, _, gd = bw.upstream(H, W, 0, 5)
    rng = np.random.default_rng(6)
    ga, gi = (rng.standard_normal((H * W,)).astype(np.float32) for _ in range(2))
    Gc, Gd, GA, GI = _t(gc).reshape(3, -1).t(), _t(gd).reshape(-1), _t(ga), _t(gi)
    bg = torch.tensor(sc.bg)
    ref, bar = planes_model(pairs, w, rec, P, bg, Gc, Gd, GA, GI)
    no_invd, _ = planes_model(pairs, w, rec, P, bg, Gc, Gd, GA, torch.zeros_like(GI))
    no_ga, _ = planes_model(pairs, w, rec, P, bg, Gc, Gd, torch.zeros_like(GA), GI)
    for label, x in (("no 1/z term", no_invd), ("no gA", no_ga)):
        worst = float(bw._ratio((x - ref).abs(), bar).max())
        print(f"[{label}] worst |err|/bar {worst:.3g}")
        assert worst > 1.0, label
    zero, _ = planes_model(pairs, w, rec, P, bg, Gc, Gd, torch.zeros_like(GA), torch.zeros_like(GI))
    bgp = Gc.double() * bg.double()
    default, _ = bw.composite_model(pairs, w, rec, P, bw.colour_depth_dots(rec, Gc, Gd), 4,
                                    (bgp.sum(1), bgp.abs().sum(1)))
    assert torch.allclose(zero, default, rtol=1e-12, atol=0)
    # dL/dz: dropping the plane's term is flagged too
    Wt = bw.Weights(pairs, w, P)
    r1, _, _ = Wt.terms(Gd.reshape(-1, 1))
    assert dz_check(Wt, rec, r1.float().reshape(-1), Gd, GI) > 1.0


# -------------------------------------------------------------------------------------------------------- CPU surface
def test_header_declares_the_entries():
    src = open(f"{ROOT}/include/f3dgs_b200.h").read()
    for name, tail in (("f3dgs_forward_alpha_invdepth", r"int antialiasing,\s*float\* out_alpha,\s*float\* out_invdepth"),
                       ("f3dgs_backward_alpha_invdepth", r"float\* dL_dcamera,\s*int antialiasing,\s*const float\* "
                                                         r"dL_dalpha,\s*const float\* dL_dinvdepth"),
                       ("f3dgs_backward_accum_alpha_invdepth", r"float\* dL_dcamera,\s*int antialiasing,\s*const float\* "
                                                               r"dL_dalpha,\s*const float\* dL_dinvdepth")):
        assert re.search(r"int " + name + r"\([^;]*" + tail + r"\);", src), name
    assert "#define F3DGS_ABI_VERSION 2" in src


def test_python_surface():
    import diff_gaussian_rasterization as dgr
    from diff_gaussian_rasterization import _C
    from diff_gaussian_rasterization.parallel import ViewBatch

    sig = inspect.signature(dgr.AlphaInvDepthGaussianRasterizer.__init__)
    assert list(sig.parameters) == ["self", "raster_settings", "feature_geometry", "antialiasing"]
    assert sig.parameters["feature_geometry"].default is False and sig.parameters["antialiasing"].default is False
    assert issubclass(dgr.AlphaInvDepthGaussianRasterizer, dgr.GaussianRasterizer)
    sig = inspect.signature(dgr.rasterize_gaussians_alpha_invdepth)
    assert list(sig.parameters) == list(inspect.signature(dgr.rasterize_gaussians).parameters) + [
        "feature_geometry", "antialiasing"]
    assert all(sig.parameters[k].default is False for k in ("feature_geometry", "antialiasing"))
    sig = inspect.signature(ViewBatch.backward)
    assert list(sig.parameters)[-2:] == ["g_alpha", "g_invdepth"]
    assert sig.parameters["g_alpha"].default is None and sig.parameters["g_invdepth"].default is None
    assert list(inspect.signature(ViewBatch.forward_alpha_invdepth).parameters) == ["self", "rs", "antialiasing"]
    doc = _C.rasterize_gaussians_alpha_invdepth.__doc__
    assert "debug: bool, antialiasing: bool = False" in doc
    doc = _C.rasterize_gaussians_backward_alpha_invdepth.__doc__
    assert ("dL_dout_alpha: torch.Tensor, dL_dout_invdepth: torch.Tensor, camera: bool = False, "
            "semantic_feature: torch.Tensor | None = None, antialiasing: bool = False") in doc
    doc = _C.rasterize_gaussians_backward_accum.__doc__
    assert "dL_dout_alpha: torch.Tensor | None = None, dL_dout_invdepth: torch.Tensor | None = None" in doc


def test_entries_check_their_arguments_before_any_launch(lib):
    from test_antialiasing import ACCUM_OUTS, BWD_OUTS, _accum_args, _bwd_args, _fake

    null = ctypes.c_void_p(0)
    n0 = lib.f3dgs_launch_count()
    planes = [_fake(40), _fake(41)]
    for name, mk, outs in (("f3dgs_backward_alpha_invdepth", _bwd_args, BWD_OUTS),
                           ("f3dgs_backward_accum_alpha_invdepth", _accum_args, ACCUM_OUTS)):
        fn = getattr(lib, name)
        for k in (0, 1):  # a NULL plane gradient
            for aa in (0, 1):
                pl = list(planes)
                pl[k] = null
                assert fn(*mk(5), aa, *pl) == -1
                assert lib.f3dgs_last_error() == (name + ": NULL dL_dalpha / dL_dinvdepth").encode()
        for k in (0, 1):  # a plane gradient overlapping an output
            for i in outs:
                a = mk(5)
                pl = list(planes)
                pl[k] = ctypes.c_void_p(a[i].value + 4)
                assert fn(*a, 0, *pl) == -1, (name, i)
                assert b"dL_dalpha / dL_dinvdepth overlap an output" in lib.f3dgs_last_error(), (name, i)
            a = mk(5)
            pl = list(planes)
            pl[k] = ctypes.c_void_p(a[-1].value or _fake(30).value)  # dL_dcamera
            a[-1] = ctypes.c_void_p(pl[k].value)
            assert fn(*a, 0, *pl) == -1 and b"overlap" in lib.f3dgs_last_error(), name
        assert fn(*mk(5, sf_dtype=9), 0, *planes) == -1 and b"unknown dtype code" in lib.f3dgs_last_error()
        assert fn(*mk(0), 0, *planes) == 0  # P == 0

    alloc = ctypes.CFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t)(lambda ctx, n: None)
    f = ctypes.c_float
    p = _fake

    def fwd(dtype=F32):
        return [alloc, null, alloc, null, alloc, null, 5, 0, 1, 4, p(0), 64, 64, p(1), p(2), null, p(3), dtype, p(5),
                p(6), f(1.0), p(7), null, p(8), p(9), p(10), f(0.5), f(0.5), 0, p(11), p(12), p(13), p(14), 0, null]

    fn = lib.f3dgs_forward_alpha_invdepth
    for k in (0, 1):
        pl = list(planes)
        pl[k] = null
        assert fn(*fwd(), 0, *pl) == -1
        assert lib.f3dgs_last_error() == b"f3dgs_forward_alpha_invdepth: NULL out_alpha / out_invdepth"
    assert fn(*fwd(dtype=5), 1, *planes) == -1 and b"unknown dtype code" in lib.f3dgs_last_error()
    for k in (0, 1):
        for i in (29, 30, 31, 32):  # out_color, out_feature_map, out_depth, radii
            pl = list(planes)
            a = fwd()
            pl[k] = ctypes.c_void_p(a[i].value + 8)
            assert fn(*a, 0, *pl) == -1, i
            assert b"out_alpha / out_invdepth overlap another output" in lib.f3dgs_last_error(), i
    assert fn(*fwd(), 0, planes[0], ctypes.c_void_p(planes[0].value + 4)) == -1  # with each other
    assert lib.f3dgs_launch_count() == n0


# ------------------------------------------------------------------------------------------------------------ GPU: forward
def _forward_ctypes(lib, sc, cam, sf, aa, dev="cuda"):
    """f3dgs_forward_alpha_invdepth with NaN-prefilled outputs and torch-owned buffers -> dict"""
    d = scenegen.to_torch(sc, dev)
    H, W, P = cam.image_height, cam.image_width, sc.P
    C = sf.shape[-1] if sf.numel() else 0
    keep = []

    def grow(ctx, n):
        keep.append(torch.empty(max(int(n), 1), dtype=torch.uint8, device=dev))
        return keep[-1].data_ptr()

    alloc = ctypes.CFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t)(grow)
    nan = lambda *s, dt=torch.float32: torch.full(s, float("nan"), dtype=dt, device=dev)  # noqa: E731
    o = dict(color=nan(3, H, W), fmap=nan(C, H, W, dt=sf.dtype), depth=nan(1, H, W), alpha=nan(1, H, W),
             invdepth=nan(1, H, W), radii=torch.full((P,), -7, dtype=torch.int32, device=dev))
    vm, pm, cp = (torch.tensor(a, device=dev).contiguous() for a in (cam.viewmatrix, cam.projmatrix, cam.campos))
    bg = torch.tensor(sc.bg, device=dev)
    f = ctypes.c_float
    sfp = sf.contiguous()
    R = lib.f3dgs_forward_alpha_invdepth(
        alloc, None, alloc, None, alloc, None, P, sc.sh_degree, d["shs"].shape[1], C, _ptr(bg), W, H,
        _ptr(d["means3D"]), _ptr(d["shs"]), None, _ptr(sfp), F16 if sf.dtype == torch.float16 else F32,
        _ptr(d["opacities"]), _ptr(d["scales"]), f(1.0), _ptr(d["rotations"]), None, _ptr(vm), _ptr(pm), _ptr(cp),
        f(cam.tanfovx), f(cam.tanfovy), 0, _ptr(o["color"]), _ptr(o["fmap"]), _ptr(o["depth"]), _ptr(o["radii"]), 0,
        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream), int(aa), _ptr(o["alpha"]), _ptr(o["invdepth"]))
    assert R >= 0, lib.f3dgs_last_error()
    torch.cuda.synchronize()
    o["R"], (o["geom"], o["img"], o["binning"]) = R, keep[:3]  # the allocators' call order
    return o


def _plain_forward(sc, cam, sf, aa, dev="cuda"):
    from diff_gaussian_rasterization import _C

    d = scenegen.to_torch(sc, dev)
    e = torch.empty(0, device=dev)
    fn = _C.rasterize_gaussians_antialiased if aa else _C.rasterize_gaussians
    vm, pm, cp = (torch.tensor(a, device=dev) for a in (cam.viewmatrix, cam.projmatrix, cam.campos))
    R, color, fmap, depth, radii, geom, binning, img = fn(
        torch.tensor(sc.bg, device=dev), d["means3D"], e, sf, d["opacities"], d["scales"], d["rotations"], 1.0, e, vm,
        pm, cam.tanfovx, cam.tanfovy, cam.image_height, cam.image_width, d["shs"], sc.sh_degree, cp, False, False)
    return dict(R=R, color=color, fmap=fmap, depth=depth, radii=radii, geom=geom, binning=binning, img=img)


def _views(o, sc, cam):
    from diff_gaussian_rasterization import _C

    return _C.debug_views(o["geom"], o["binning"], o["img"], sc.P, cam.image_width, cam.image_height, o["R"])


@pytest.mark.gpu
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("C", [0, 3, 32, 64, 128, 200])
def test_forward_is_the_plain_forward_plus_the_planes(lib, C, dtype, aa):
    from test_geometry_grads import _scene

    if C == 0 and dtype == torch.float16:
        pytest.skip("no features: one kernel for both element types")
    sc, cam, _ = _scene("inside")
    sf = (torch.randn(sc.P, 1, C, generator=torch.Generator().manual_seed(C)).to("cuda", dtype) if C
          else torch.empty(0, device="cuda"))
    new = _forward_ctypes(lib, sc, cam, sf, aa)
    ref = _plain_forward(sc, cam, sf, aa)
    assert new["R"] == ref["R"]
    for k in ("color", "fmap", "depth", "radii"):
        assert torch.equal(new[k], ref[k]), k
    vis = ref["radii"] > 0  # the preprocess writes no record for a culled Gaussian
    for a, b, k in zip(_views(new, sc, cam), _views(ref, sc, cam), ("point_list", "ranges", "n_contrib", "final_T",
                                                                      "rec")):
        assert torch.equal(a[vis] if k == "rec" else a, b[vis] if k == "rec" else b), k
    final_T = _views(new, sc, cam)[3]
    assert not bool(new["alpha"].isnan().any()) and not bool(new["invdepth"].isnan().any())
    assert torch.equal(new["alpha"].reshape(final_T.shape), 1 - final_T)
    assert bool((new["invdepth"] >= 0).all()) and bool((new["invdepth"] <= 5.0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "inside", "needles", "layers129", "opaque"])
def test_planes_match_the_blend_weight_identities(lib, name):
    from test_geometry_grads import _view

    v = _view(name)
    new = _forward_ctypes(lib, v.sc, v.cam, v.feats, False)
    for k in ("color", "depth"):
        assert torch.equal(new[k], v.base[k]), k
    Wt = bw.Weights(v.pairs, v.w, v.P)
    HW = v.W * v.H
    dev = v.pairs.pix.device
    rec = v.base["rec"].to(dev)
    T = v.base["final_T"].reshape(HW, 1).double().to(dev)
    # 1 - T: T's own rounding (n_p roundings relative to T) shows up absolutely in the difference
    r_alpha = Wt.per_pixel(new["alpha"].reshape(HW, 1).to(dev), torch.ones(v.P, 1, dtype=torch.float64, device=dev),
                           torch.zeros_like(T), T)
    r_invd = Wt.per_pixel(new["invdepth"].reshape(HW, 1).to(dev), 1.0 / rec[:, 11:12].double())
    print(f"[{name}] worst |err|/bar: alpha {r_alpha:.3g}, invdepth {r_invd:.3g}")
    assert r_alpha <= 1.0 and r_invd <= 1.0


# ----------------------------------------------------------------------------------------------------------- GPU: backward
def _backward_planes(lib, v, ups, ga, gi, buffers=None, sf=None, aa=0, map_scale=None, camera=False, accum=None):
    """f3dgs_backward_alpha_invdepth on the View v (buffers: another forward's dict with geom/binning/img/R/radii).
    ups, ga, gi: numpy arrays or tensors.  sf: the feature rows of the feature term (float32 or float16), or None.
    map_scale: ups[1] is a float16 map h standing for map_scale * float(h) (else a float32 map).  camera: also
    dL_dcamera (35 floats, "camera").  accum: a dict of buffers to add into with f3dgs_backward_accum_alpha_invdepth
    instead (opacity, feat, means3D, sh, scales, rotations, mean2D (dL_dmean2D_out), grad_accum, denom; colors /
    cov3D when precomputed; camera when camera)."""
    dev = torch.device("cuda")
    gc, gf, gd, ga, gi = (torch.as_tensor(u).to(dev) for u in (*ups, ga, gi))
    P, M = v.P, v.M
    b = v.base if buffers is None else buffers
    z = lambda *s: torch.zeros(*s, device=dev)  # noqa: E731
    sr = v.scales.numel() > 0
    null = ctypes.c_void_p(0)
    f = ctypes.c_float
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    args = [P, v.D, M, b["R"], v.C, _ptr(v.bg), v.W, v.H, _ptr(v.d["means3D"]), _ptr(v.shs), _ptr(v.cols),
            _ptr(sf), F16 if sf is not None and sf.dtype == torch.float16 else F32, _ptr(v.scales), f(v.mod),
            _ptr(v.rots), _ptr(v.cov), _ptr(v.vm), _ptr(v.pm), _ptr(v.cp), f(v.cam.tanfovx), f(v.cam.tanfovy),
            _ptr(b["radii"]), _ptr(b["geom"]), _ptr(b["binning"]), _ptr(b["img"]), _ptr(gc), _ptr(gf),
            F32 if map_scale is None else F16, f(1.0 if map_scale is None else map_scale), _ptr(gd)]
    if accum is None:
        o = dict(mean2D=z(P, 3), conic=z(P, 4), opacity=z(P), color=z(P, 3), feat=z(P, v.C), means3D=z(P, 3),
                 cov3D=z(P, 6), sh=z(P, M, 3), scales=z(P, 3), rotations=z(P, 4), dz=z(P))
        if camera:
            o["camera"] = z(35)
        args += [_ptr(o["mean2D"]), _ptr(o["conic"]), _ptr(o["opacity"]), _ptr(o["color"]), _ptr(o["feat"]),
                 _ptr(o["means3D"]), _ptr(o["cov3D"]), _ptr(o["sh"]) if M else null,
                 _ptr(o["scales"]) if sr else null, _ptr(o["rotations"]) if sr else null, _ptr(o["dz"]), 0, stream]
        entry = lib.f3dgs_backward_alpha_invdepth
    else:
        o = accum
        scratch = torch.empty(lib.f3dgs_backward_scratch_bytes(P), dtype=torch.uint8, device=dev)
        args += [_ptr(scratch), _ptr(o["opacity"]), _ptr(o["colors"]) if v.cols.numel() else null, _ptr(o["feat"]),
                 _ptr(o["means3D"]), _ptr(o["cov3D"]) if v.cov.numel() else null, _ptr(o["sh"]) if M else null,
                 _ptr(o["scales"]) if sr else null, _ptr(o["rotations"]) if sr else null, _ptr(o["mean2D"]),
                 _ptr(o["grad_accum"]), _ptr(o["denom"]), null, 0, stream]
        entry = lib.f3dgs_backward_accum_alpha_invdepth
    args += [_ptr(o["camera"]) if camera else null, int(aa), _ptr(ga), _ptr(gi)]
    rc = entry(*args)
    assert rc == 0, lib.f3dgs_last_error()
    torch.cuda.synchronize()
    return o


def _plane_grads(H, W, seed, dynamic=False):
    rng = np.random.default_rng(seed)
    g = [rng.standard_normal((1, H, W)).astype(np.float32) for _ in range(2)]
    if dynamic:
        g = [x * (10.0 ** rng.uniform(-6.0, 0.0, (1, H, W))).astype(np.float32) for x in g]
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "inside", "needles", "plane", "layers129", "opaque", "fx!=fy",
                                  "cov3D_precomp"])
def test_backward_matches_the_model(lib, name):
    from test_geometry_grads import _report, _upstreams, _view, preprocess_check

    v = _view(name)
    HW = v.W * v.H
    rec = v.base["rec"]
    Wt = bw.Weights(v.pairs, v.w, v.P)
    for i, (label, ups) in enumerate(_upstreams(v.H, v.W, v.C, 71)):
        ga, gi = _plane_grads(v.H, v.W, 90 + i, dynamic=label == "dynamic range")
        o = _backward_planes(lib, v, ups, ga, gi)
        dev = v.pairs.pix.device
        Gc, Gd = _t(ups[0]).reshape(3, HW).t().to(dev), _t(ups[2]).reshape(HW).to(dev)
        GA, GI = _t(ga).reshape(HW).to(dev), _t(gi).reshape(HW).to(dev)
        ref, bar = planes_model(v.pairs, v.w, rec, v.P, v.bg, Gc, Gd, GA, GI)
        g6 = bw.geom6(o["mean2D"], o["conic"], o["opacity"]).double().to(ref.device)
        r = bw._ratio((g6 - ref).abs(), bar).max(0).values
        worst = {k: float(x) for k, x in zip(("dL_dmean2D.x", "dL_dmean2D.y", "dL_dconic.a", "dL_dconic.b",
                                              "dL_dconic.c", "dL_dopacity"), r)}
        worst["dL_dcolor"] = Wt.per_gaussian(o["color"].reshape(v.P, 3), Gc)
        worst["dL_dz"] = dz_check(Wt, rec, o["dz"], Gd, GI)
        worst.update(preprocess_check(v.chain(o), v.outputs(o), v.visible))
        _report(f"{name} planes {label}", worst)


# ------------------------------------------------------------------------------------------------- GPU: bitwise identities
def _block():
    from test_camera_grad import _block_scene

    sc, cam = _block_scene()
    sc.bg = np.array([0.3, 0.6, 0.9], np.float32)
    return sc, cam


def _bargs(sc, cam, f, sf, ups, dev="cuda"):
    """rasterize_gaussians_backward's 24 positional arguments for the forward dict f"""
    d = scenegen.to_torch(sc, dev)
    e = torch.empty(0, device=dev)
    gc, gf, gd = ups
    vm, pm, cp = (torch.tensor(a, device=dev) for a in (cam.viewmatrix, cam.projmatrix, cam.campos))
    return (torch.tensor(sc.bg, device=dev), d["means3D"], f["radii"], e, sf, d["scales"], d["rotations"], 1.0, e, vm,
            pm, cam.tanfovx, cam.tanfovy, gc, gf, gd, d["shs"], sc.sh_degree, cp, f["geom"], f["R"], f["binning"],
            f["img"], False)


def _equal(a, b, label):
    for i, (x, y) in enumerate(zip(a, b)):
        assert (x is None and y is None) or torch.equal(x, y), (label, i)


@pytest.mark.gpu
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("C", [0, 8, 200])
def test_zero_plane_gradients_give_the_counterparts_bits(lib, C, aa):
    from diff_gaussian_rasterization import _C

    sc, cam = _block()
    dev = torch.device("cuda")
    H, W = cam.image_height, cam.image_width
    sf = torch.randn(sc.P, 1, C, generator=torch.Generator().manual_seed(1)).to(dev) if C else torch.empty(0, device=dev)
    f = _plain_forward(sc, cam, sf, aa)
    z = torch.zeros(1, H, W, device=dev)
    gc, gf, gd = (_t(u, dev) for u in bw.upstream(H, W, C, 3))
    for half in (False, True):
        g = (gc, gf.half() if half else gf, gd)
        a = _bargs(sc, cam, f, sf, g)
        new = lambda **kw: _C.rasterize_gaussians_backward_alpha_invdepth(*a, z, z, antialiasing=aa, **kw)  # noqa
        if aa:
            _equal(new(), _C.rasterize_gaussians_backward_antialiased(*a), "antialiased")
            _equal(new(camera=True), _C.rasterize_gaussians_backward_antialiased(*a, camera=True), "aa camera")
            _equal(new(semantic_feature=sf), _C.rasterize_gaussians_backward_antialiased(*a, semantic_feature=sf),
                   "aa feature geometry")
        else:
            _equal(new()[:9], _C.rasterize_gaussians_backward(*a), "default")
            _equal(new(camera=True), _C.rasterize_gaussians_backward_camera(*a), "camera")
            _equal(new(semantic_feature=sf), _C.rasterize_gaussians_backward_feature_geometry(*a, False),
                   "feature geometry")
            _equal(new(semantic_feature=sf, camera=True), _C.rasterize_gaussians_backward_feature_geometry(*a, True),
                   "feature geometry camera")
    # the accumulating entry (ViewBatch) with zero planes, and with g_alpha = g_invdepth = None, against the call
    # without them; the planes forward's buffers against the plain forward's.  With and without the camera, and with
    # features that the feature term leaves out (the _antialiased / plain accumulating counterparts)
    from diff_gaussian_rasterization.parallel import ViewBatch

    d = scenegen.to_torch(sc, dev)
    params = dict(means3D=d["means3D"], scales=d["scales"], rotations=d["rotations"], opacities=d["opacities"],
                  shs=d["shs"], semantic_feature=sf if C else None)
    rs = _settings(sc, cam)
    for camera, fg in [(True, bool(C)), (False, bool(C))] + ([(True, False)] if C else []):
        outs = []
        for planes in (None, "none", "zeros"):
            vb = ViewBatch(params)
            ctx = (vb.forward_alpha_invdepth(rs, antialiasing=aa) if planes else vb.forward(rs, antialiasing=aa))[-1]
            kw = dict(g_alpha=z, g_invdepth=z) if planes == "zeros" else {}
            for half in (False, True):
                g = gf.half() if half else gf
                cam_g = vb.backward(ctx, gc, g if C else None, gd, camera=camera, feature_geometry=fg, **kw)
                outs.append((vb.flat.clone(), torch.cat([cam_g.viewmatrix.reshape(-1), cam_g.projmatrix.reshape(-1),
                                                         cam_g.campos]) if camera else None))
        # outs: (without planes, None planes, zero planes) x (float32 map, then float16 map added into the same buffer)
        for i, o in enumerate(outs[2:]):
            assert torch.equal(outs[i % 2][0], o[0]), (camera, fg, i)
            assert not camera or torch.equal(outs[i % 2][1], o[1]), (camera, fg, i)


def _settings(sc, cam, dev="cuda", **over):
    from diff_gaussian_rasterization import GaussianRasterizationSettings

    kw = scenegen.settings_kwargs(sc, cam, torch.device(dev))
    kw.update(over)
    return GaussianRasterizationSettings(**kw)


@pytest.mark.gpu
@pytest.mark.parametrize("aa", [False, True])
def test_either_forwards_buffers_go_to_the_backward(lib, aa):
    """The buffers of the plain forward and of the planes forward give the new backward bitwise-equal gradients; the
    accumulating entry into zeros gives the assigning entry's bits (block scene)."""
    from diff_gaussian_rasterization import _C

    sc, cam = _block()
    dev = torch.device("cuda")
    H, W = cam.image_height, cam.image_width
    sf = torch.randn(sc.P, 1, 8, generator=torch.Generator().manual_seed(2)).to(dev)
    plain = _plain_forward(sc, cam, sf, aa)
    planes = _forward_ctypes(lib, sc, cam, sf, aa)
    ups = tuple(_t(u, dev) for u in bw.upstream(H, W, 8, 4))
    ga, gi = (_t(x, dev) for x in _plane_grads(H, W, 5))
    r = [_C.rasterize_gaussians_backward_alpha_invdepth(*_bargs(sc, cam, f, sf, ups), ga, gi, camera=True,
                                                         antialiasing=aa) for f in (plain, planes)]
    _equal(r[0], r[1], "buffers")
    assert bool(r[0][3].abs().sum() > 0)
    # accumulating entry into zeros == assigning entry, through ViewBatch
    from diff_gaussian_rasterization.parallel import ViewBatch

    d = scenegen.to_torch(sc, dev)
    vb = ViewBatch(dict(means3D=d["means3D"], scales=d["scales"], rotations=d["rotations"], opacities=d["opacities"],
                        shs=d["shs"], semantic_feature=sf))
    rs = _settings(sc, cam)
    *_, ctx = vb.forward_alpha_invdepth(rs, antialiasing=aa)
    m2d = torch.zeros(sc.P, 3, device=dev)
    cg = vb.backward(ctx, *ups, means2D_out=m2d, camera=True, g_alpha=ga, g_invdepth=gi)
    g = vb.grads
    ref = r[0]
    for k, x in (("means3D", ref[4]), ("opacities", ref[3]), ("shs", ref[6]), ("scales", ref[7]),
                 ("rotations", ref[8]), ("semantic_feature", ref[2])):
        assert torch.equal(g[k].reshape(x.shape), x), k
    assert torch.equal(m2d, ref[0])
    assert torch.equal(torch.cat([cg.viewmatrix.reshape(-1), cg.projmatrix.reshape(-1), cg.campos]),
                       torch.cat([ref[9].reshape(-1), ref[10].reshape(-1), ref[11]]))
    # the densification statistics carry the planes' terms
    assert torch.allclose(vb.grad_accum, ref[0][:, :2].norm(dim=1), rtol=1e-6, atol=0)
    no_planes = _C.rasterize_gaussians_backward_antialiased(*_bargs(sc, cam, plain, sf, ups), camera=True) if aa else \
        _C.rasterize_gaussians_backward_camera(*_bargs(sc, cam, plain, sf, ups))
    assert not torch.equal(no_planes[0], ref[0]) and not torch.equal(no_planes[3], ref[3])
    assert not torch.allclose(vb.grad_accum, no_planes[0][:, :2].norm(dim=1), rtol=1e-6, atol=0)


@pytest.mark.gpu
def test_view_batch_sums_three_views(lib):
    from diff_gaussian_rasterization import _C
    from diff_gaussian_rasterization.parallel import ViewBatch

    sc = scenegen.make_config("small")
    dev = torch.device("cuda")
    d = scenegen.to_torch(sc, dev)
    vb = ViewBatch(dict(means3D=d["means3D"], scales=d["scales"], rotations=d["rotations"], opacities=d["opacities"],
                        shs=d["shs"], semantic_feature=d["semantic_feature"]))
    cams = [scenegen.make_camera(96, 64, np.array(p)) for p in ([0.2, 0.1, 4.0], [-0.4, 0.3, 3.6], [0.1, -0.5, 4.4])]
    tot = {k: 0 for k in ("means3D", "opacities", "semantic_feature")}
    for i, cam in enumerate(cams):
        H, W = cam.image_height, cam.image_width
        color, feat, radii, depth, alpha, invdepth, ctx = vb.forward_alpha_invdepth(_settings(sc, cam))
        ups = tuple(_t(u, dev) for u in bw.upstream(H, W, sc.C, 20 + i))
        ga, gi = (_t(x, dev) for x in _plane_grads(H, W, 30 + i))
        vb.backward(ctx, *ups, g_alpha=ga, g_invdepth=gi)
        f = dict(R=ctx.num_rendered, radii=ctx.radii, geom=ctx.geom, binning=ctx.binning, img=ctx.img)
        r = _C.rasterize_gaussians_backward_alpha_invdepth(*_bargs(sc, cam, f, d["semantic_feature"], ups), ga, gi)
        for k, x in (("means3D", r[4]), ("opacities", r[3]), ("semantic_feature", r[2])):
            tot[k] = tot[k] + x
    for k, x in tot.items():
        got = vb.grads[k].reshape(x.shape)
        scale = x.abs().max()
        assert bool(scale > 0)
        assert torch.allclose(got, x, rtol=1e-4, atol=1e-5 * float(scale)), k


# ---------------------------------------------------------------------------------------------------------- GPU: autograd
@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("antialiasing", [False, True])
@pytest.mark.parametrize("feature_geometry", [False, True])
@pytest.mark.parametrize("camera", [False, True])
def test_autograd_equals_the_binding(lib, camera, feature_geometry, antialiasing, half):
    """half: float16 features, whose float16 feature map's gradient reaches the binding as float16"""
    import diff_gaussian_rasterization as dgr
    from diff_gaussian_rasterization import _C

    sc, cam = _block()
    dev = torch.device("cuda")
    H, W = cam.image_height, cam.image_width
    d = scenegen.to_torch(sc, dev, requires_grad=True)
    if half:
        d["semantic_feature"] = d["semantic_feature"].detach().half().requires_grad_()
    rs = _settings(sc, cam)
    if camera:
        rs = rs._replace(viewmatrix=rs.viewmatrix.clone().requires_grad_(), projmatrix=rs.projmatrix.clone(
        ).requires_grad_(), campos=rs.campos.clone().requires_grad_())
    ups = [_t(u, dev) for u in bw.upstream(H, W, sc.C, 8)] + [_t(x, dev) for x in _plane_grads(H, W, 9)]
    if half:
        ups[1] = ups[1].half()
    ras = dgr.AlphaInvDepthGaussianRasterizer(rs, feature_geometry=feature_geometry, antialiasing=antialiasing)
    outs = ras(means3D=d["means3D"], means2D=torch.zeros_like(d["means3D"]), opacities=d["opacities"], shs=d["shs"],
               semantic_feature=d["semantic_feature"], scales=d["scales"], rotations=d["rotations"])
    color, fmap, radii, depth, alpha, invdepth = outs
    assert fmap.dtype == d["semantic_feature"].dtype
    loss = sum((o * g).sum() for o, g in zip((color, depth, alpha, invdepth), ups[:1] + ups[2:]))
    # the feature map's gradient is ups[1] in the map's own dtype
    loss = loss + (fmap * ups[1]).sum()
    cam_t = [rs.viewmatrix, rs.projmatrix, rs.campos] if camera else []
    keys = ("means3D", "opacities", "shs", "scales", "rotations", "semantic_feature")
    got = torch.autograd.grad(loss, [d[k] for k in keys] + cam_t)
    sf = d["semantic_feature"].detach()
    f = _plain_forward(sc, cam, sf, antialiasing)
    r = _C.rasterize_gaussians_backward_alpha_invdepth(
        *_bargs(sc, cam, f, sf, ups[:3]), ups[3], ups[4], camera=camera,
        semantic_feature=sf if feature_geometry else None, antialiasing=antialiasing)
    want = (r[4], r[3], r[6], r[7], r[8], r[2]) + tuple(r[9:12] if camera else ())
    for k, a, b in zip(keys + ("viewmatrix", "projmatrix", "campos"), got, want):
        assert a.dtype == (sf.dtype if k == "semantic_feature" else torch.float32), k
        assert torch.equal(a.reshape(b.shape), b.to(a.dtype)), k
    # a loss on colour only: GaussianRasterizer's gradients
    outs2 = (dgr.AntialiasedGaussianRasterizer if antialiasing else dgr.GaussianRasterizer)(
        rs, feature_geometry=feature_geometry)(means3D=d["means3D"], means2D=torch.zeros_like(d["means3D"]), opacities=d["opacities"], shs=d["shs"],
        semantic_feature=d["semantic_feature"], scales=d["scales"], rotations=d["rotations"])
    outs = ras(means3D=d["means3D"], means2D=torch.zeros_like(d["means3D"]), opacities=d["opacities"], shs=d["shs"],
               semantic_feature=d["semantic_feature"], scales=d["scales"], rotations=d["rotations"])
    for o in (outs, outs2):
        assert torch.equal(o[0], outs2[0])
    ga = torch.autograd.grad((outs[0] * ups[0]).sum(), [d[k] for k in keys[:5]] + cam_t)
    gb = torch.autograd.grad((outs2[0] * ups[0]).sum(), [d[k] for k in keys[:5]] + cam_t)
    for a, b in zip(ga, gb):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_mask_and_inverse_depth_losses_train():
    """A few dozen Adam steps on a mask loss on alpha plus an inverse-depth L1 against a perturbed scene's render lower
    the loss."""
    import diff_gaussian_rasterization as dgr

    sc = scenegen.make_config("small")
    cam = sc.cameras[0]
    dev = torch.device("cuda")
    rs = _settings(sc, cam)
    tgt = scenegen.to_torch(sc, dev)
    ras = dgr.AlphaInvDepthGaussianRasterizer(rs)

    def render(d):
        return ras(means3D=d["means3D"], means2D=torch.zeros_like(d["means3D"]), opacities=d["opacities"],
                   colors_precomp=torch.full_like(d["means3D"], 0.5), scales=d["scales"], rotations=d["rotations"])

    with torch.no_grad():
        _, _, _, _, mask, inv_t = render(tgt)
    g = torch.Generator().manual_seed(4)
    d = {k: v.clone() for k, v in tgt.items()}
    d["means3D"] += 0.05 * torch.randn(d["means3D"].shape, generator=g).to(dev)
    d["opacities"] = torch.logit(d["opacities"].clamp(0.02, 0.98)) + 0.5 * torch.randn(d["opacities"].shape,
                                                                                      generator=g).to(dev)
    params = [d["means3D"].requires_grad_(), d["opacities"].requires_grad_()]
    opt = torch.optim.Adam(params, lr=5e-3)
    losses = []
    for _ in range(40):
        dd = dict(d, opacities=torch.sigmoid(d["opacities"]))
        _, _, _, _, alpha, invdepth = render(dd)
        loss = (alpha - mask).abs().mean() + (invdepth - inv_t).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    print(f"loss {losses[0]:.4g} -> {losses[-1]:.4g}")
    assert losses[-1] < 0.9 * losses[0]
