"""Depth distortion loss: f3dgs_forward_distortion / f3dgs_backward[_accum]_distortion and their torch, autograd and
view-batch surfaces.

For pixel p over the pairs i = 1..n it blends, in blend order, with w_i = alpha_i T_i and z_i the record's view depth:
    L_p = sum_i sum_j w_i w_j |z_i - z_j| = 2 sum_i w_i (z_i A_i - D_i),  A_i = sum_{j<i} w_j,  D_i = sum_{j<i} w_j z_j
(z is non-decreasing along each tile list, so the prefix-sum form is the pairwise sum).  dL_p/dw_i = c_i
= 2 [z_i (A_i - Abar_i) + Dbar_i - D_i] with the sums over the later pairs Abar_i, Dbar_i, and dL_p/dz_i
= 2 w_i (A_i - Abar_i): blend order is the tie-breaking subgradient.  Since L_p is a sum of w_i c_i-weighted terms in the
weights, its gradients with respect to the geometry are composite_model's with d_i = g_p c_i (c_i held fixed): the
composite's colour recurrence on c.

The forward is checked bitwise against the forward without the plane, and the plane per pixel against the float64 model
on the extracted weights, within  K u (n_p + 4) 2 sum_i w_i (z_i (1 + A_i) + D_i): the float32 1 - T of the i-th pair
differs from A_i by up to 2 u n_p (T's unwound roundings, T <= 1), Dp from D_i by n_p u relative, and the n_p terms'
products and sum add (n_p + 4) u relative to their magnitudes.  The backward is checked per Gaussian against
composite_model with d = c.Gc + z Gd + g c_i and dL/dz against its sum over pixels.
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
def blended(pairs, w, rec):
    """The blended pairs in blend order -> (pix, gid, w, z, first) in float64; first = index of the pixel's first pair"""
    keep = w > 0
    sel = pairs.widx[keep]
    pix, gid = pairs.pix[sel], pairs.gid[sel]
    _, counts = torch.unique_consecutive(pix, return_counts=True)
    first = torch.repeat_interleave(torch.cumsum(counts, 0) - counts, counts)
    return pix, gid, w[keep].double(), rec.to(pix.device)[gid, 11].double(), first


def prefix_sums(w, z, pix, first, HW):
    """(A, D, Abar, Dbar) per pair: the sums of w and w z over the pixel's earlier and later pairs"""
    A, D = bw._seg_excl_cumsum(w, first), bw._seg_excl_cumsum(w * z, first)
    tw = torch.zeros(HW, dtype=w.dtype, device=w.device).index_add(0, pix, w)
    td = torch.zeros(HW, dtype=w.dtype, device=w.device).index_add(0, pix, w * z)
    return A, D, tw[pix] - A - w, td[pix] - D - w * z


def distortion_model(pairs, w, rec):
    """(L [HW], bar [HW]) in float64 from the extracted weights: the prefix-sum form and the forward's bar (module
    docstring)"""
    HW = pairs.HW
    pix, _, wv, z, first = blended(pairs, w, rec)
    A, D, _, _ = prefix_sums(wv, z, pix, first, HW)
    L = torch.zeros(HW, dtype=torch.float64, device=pix.device).index_add(0, pix, 2 * wv * (z * A - D))
    mag = torch.zeros(HW, dtype=torch.float64, device=pix.device).index_add(0, pix, 2 * wv * (z * (1 + A) + D))
    return L, bw.K * bw.U * (pairs.n.double() + 4) * mag


def brute_force(pairs, w, rec):
    """sum_ij w_i w_j |z_i - z_j| per pixel over every ordered pair of blended pairs, in float64"""
    HW = pairs.HW
    pix, _, wv, z, first = blended(pairs, w, rec)
    n = torch.zeros(HW, dtype=torch.long, device=pix.device).index_add(0, pix, torch.ones_like(pix))[pix]
    I = torch.repeat_interleave(torch.arange(pix.numel(), device=pix.device), n)
    J = first[I] + (torch.arange(I.numel(), device=pix.device) - torch.repeat_interleave(torch.cumsum(n, 0) - n, n))
    t = wv[I] * wv[J] * (z[I] - z[J]).abs()
    return torch.zeros(HW, dtype=torch.float64, device=pix.device).index_add(0, pix[I], t)


def dist_dfn(pairs, w, rec, G, form="l1"):
    """dfn of composite_model for the distortion alone: per blended pair d = g_p c_i, c_i = dL_p/dw_i of the L1 form
    (form="no_abar": without the later pairs' z_i Abar_i, a negative control; "squared": 2DGS's
    sum_ij w_i w_j (z_i - z_j)^2), and dabs the magnitudes c's float32 evaluation is bounded by: the unwound T's absolute
    error (up to 2 u n_p) times z_i, and the running sums' errors relative to D_tot.  Pairs are matched by position:
    composite_model's (pix, gid) are the blended pairs in the same order."""
    pix, gid, wv, z, first = blended(pairs, w, rec)
    A, D, Abar, Dbar = prefix_sums(wv, z, pix, first, pairs.HW)
    if form == "l1":
        c = 2 * (z * (A - Abar) + Dbar - D)
    elif form == "no_abar":
        c = 2 * (z * A + Dbar - D)
    else:  # sum_j w_j (z_i - z_j)^2 = z^2 W - 2 z M1 + M2 over the pixel's other pairs, twice
        tw = A + Abar
        m1 = D + Dbar
        m2 = torch.zeros(pairs.HW, dtype=torch.float64, device=pix.device).index_add(0, pix, wv * z * z)[pix] - \
            wv * z * z
        c = 2 * (z * z * tw - 2 * z * m1 + m2)
    g = G.double().reshape(-1).to(pix.device)[pix]
    cabs = 2 * (z * (1 + A + Abar) + 2 * (D + Dbar + wv * z))
    d, dabs = g * c, g.abs() * cabs

    def dfn(gid_, pix_):
        assert torch.equal(gid_, gid) and torch.equal(pix_, pix)
        return d, dabs

    return dfn, (pix, gid, wv, z, A, Abar, g)


def full_dfn(pairs, w, rec, Gc, Gd, G, form="l1"):
    """colour and depth (colour_depth_dots) plus the distortion's d"""
    base = bw.colour_depth_dots(rec, Gc, Gd)
    ddfn, parts = dist_dfn(pairs, w, rec, G, form)

    def dfn(gid, pix):
        d0, a0 = base(gid, pix)
        d1, a1 = ddfn(gid, pix)
        return d0 + d1, a0 + a1

    return dfn, parts


def backward_model(pairs, w, rec, P, bg, Gc, Gd, G, form="l1"):
    """(ref, bar) of the six geometric values with the distortion's term, and the dL/dz terms (ref, sum |.|, sum
    |.| (2 n_p + 4)) [P,1] of gaussian_ratio"""
    dfn, (pix, gid, wv, z, A, Abar, g) = full_dfn(pairs, w, rec, Gc, Gd, G, form)
    bgp = Gc.double() * bg.double().to(Gc.device)
    # 4 products for colour and depth; c takes about ten more operations per pair
    ref, bar = bw.composite_model(pairs, w, rec, P, dfn, 14, (bgp.sum(1), bgp.abs().sum(1)))
    Wt = bw.Weights(pairs, w, P)
    r, a, an = Wt.terms(Gd.reshape(-1, 1))
    t = 2 * wv * (A - Abar) * g
    ta = 2 * wv * (1 + A + Abar) * g.abs()
    n = pairs.n.double()[pix]
    z0 = torch.zeros(P, 1, dtype=torch.float64, device=pix.device)
    dz = (r + z0.index_add(0, gid, t[:, None]), a + z0.index_add(0, gid, ta[:, None]),
          an + z0.index_add(0, gid, (ta * (2 * n + 4))[:, None]))
    return ref, bar, dz, Wt.m


# --------------------------------------------------------------------------------------------------------------- CPU
def _oracle(name):
    from test_blend_weights import _oracle_view

    sc, cam, f, pairs, w = _oracle_view(name)
    return sc, cam, _t(bw.oracle_records(f)), pairs, w


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_prefix_sums_are_the_pairwise_sum(name):
    sc, cam, rec, pairs, w = _oracle(name)
    pix, _, _, z, first = blended(pairs, w, rec)
    # z is non-decreasing along each pixel's blend order
    same = torch.arange(z.numel()) > first
    assert bool((z[1:][same[1:]] >= z[:-1][same[1:]]).all())
    L, _ = distortion_model(pairs, w, rec)
    ref = brute_force(pairs, w, rec)
    assert bool((ref > 0).any())
    # the segmented prefix sums come from one float64 cumsum over the image: exact to ~1e-16 of the image's total
    assert torch.allclose(L, ref, rtol=1e-9, atol=1e-9)


def test_autograd_model_matches_finite_differences():
    """The L1 form's gradients (c_i through the weights' alphas, and dL/dz) against central differences of the
    float64 prefix-sum model, on a few random pixels with ties in z"""
    rng = np.random.default_rng(3)
    for n in (1, 2, 5, 9):
        al = torch.tensor(rng.uniform(0.05, 0.9, n)).requires_grad_()
        z = torch.tensor(np.sort(np.round(rng.uniform(1.0, 3.0, n), 1))).requires_grad_()

        def loss(al, z):
            T = torch.cumprod(torch.cat([torch.ones(1, dtype=al.dtype), 1 - al[:-1]]), 0)
            wv = al * T
            A = torch.cumsum(wv, 0) - wv
            D = torch.cumsum(wv * z, 0) - wv * z
            return 2 * (wv * (z * A - D)).sum()

        ga, gz = torch.autograd.grad(loss(al, z), [al, z])
        with torch.no_grad():
            T = torch.cumprod(torch.cat([torch.ones(1, dtype=al.dtype), 1 - al[:-1]]), 0)
            wv = al * T
            A = torch.cumsum(wv, 0) - wv
            Abar = wv.sum() - A - wv
            D = torch.cumsum(wv * z, 0) - wv * z
            Dbar = (wv * z).sum() - D - wv * z
            c = 2 * (z * (A - Abar) + Dbar - D)
            B = torch.zeros(n, dtype=al.dtype)
            for i in range(n - 2, -1, -1):
                B[i] = al[i + 1] * c[i + 1] + (1 - al[i + 1]) * B[i + 1]
            assert torch.allclose(ga, T * (c - B), rtol=1e-10, atol=1e-12)
            assert torch.allclose(gz, 2 * wv * (A - Abar), rtol=1e-10, atol=1e-12)
            h = 1e-6
            for i in range(n):
                e = torch.zeros(n, dtype=al.dtype)
                e[i] = h
                fd = (loss(al + e, z) - loss(al - e, z)) / (2 * h)
                assert abs(float(fd - ga[i])) <= 1e-7 * max(1.0, abs(float(fd))), (n, i)
                # z: away from ties only (at a tie the model takes blend order, a one-sided derivative)
                zi = z.clone()
                if not bool(((zi - zi[i]).abs()[torch.arange(n) != i] < 2 * h).any()):
                    fd = (loss(al, z + e) - loss(al, z - e)) / (2 * h)
                    assert abs(float(fd - gz[i])) <= 1e-7 * max(1.0, abs(float(fd))), (n, i)


def test_windowed_pairs_give_the_whole_image_values():
    import oracle

    sc, cam, rec, pairs, w = _oracle("small")
    f = oracle.forward(sc, cam)
    pl, rg, nc = (_t(f[k].astype(np.int64)) for k in ("point_list", "ranges", "n_contrib"))
    tiles = torch.tensor([0, 3, 7])
    win = bw.Pairs(pl, rg, nc, cam.image_width, cam.image_height, tiles=tiles)
    # the window's walked pairs are a subsequence of the whole image's, in the same order
    key = pairs.pix[pairs.widx] * (1 << 20) + pairs.pos[pairs.widx]
    wkey = win.pix[win.widx] * (1 << 20) + win.pos[win.widx]
    ww = w[torch.searchsorted(key, wkey)]
    L, _ = distortion_model(pairs, w, rec)
    Lw, _ = distortion_model(win, ww, rec)
    # equal up to the rounding of the two images' float64 prefix sums (see test_prefix_sums_are_the_pairwise_sum)
    assert torch.allclose(Lw[win.pixels], L[win.pixels], rtol=1e-9, atol=1e-9) and bool((Lw[win.pixels] > 0).any())
    inside = bw.contained(pl, rg, sc.P, tiles)
    Gc, Gd = torch.zeros(pairs.HW, 3), torch.zeros(pairs.HW)
    G = _t(np.random.default_rng(1).standard_normal(pairs.HW).astype(np.float32))
    bg = torch.tensor(sc.bg)
    ref, _, dz, _ = backward_model(pairs, w, rec, sc.P, bg, Gc, Gd, G)
    refw, _, dzw, _ = backward_model(win, ww, rec, sc.P, bg, Gc, Gd, G)
    assert bool(inside.any())
    assert torch.allclose(refw[inside], ref[inside], rtol=1e-8, atol=1e-9)
    assert torch.allclose(dzw[0][inside], dz[0][inside], rtol=1e-8, atol=1e-9)


def test_negative_controls_fail_the_bar():
    """A model without the Abar term, and 2DGS's squared form, are outside the L1 model's bar."""
    sc, cam, rec, pairs, w = _oracle("small")
    HW, P = pairs.HW, sc.P
    rng = np.random.default_rng(6)
    G = _t(rng.standard_normal(HW).astype(np.float32))
    Gc, Gd = torch.zeros(HW, 3), torch.zeros(HW)
    bg = torch.tensor(sc.bg)
    ref, bar, dz, m = backward_model(pairs, w, rec, P, bg, Gc, Gd, G)
    for form in ("no_abar", "squared"):
        x, _, dzx, _ = backward_model(pairs, w, rec, P, bg, Gc, Gd, G, form)
        worst = float(bw._ratio((x - ref).abs(), bar).max())
        print(f"[{form}] worst |err|/bar {worst:.3g}")
        assert worst > 1.0, form
    assert bw.gaussian_ratio(dz[0] * 0, dz, m) > 1.0  # dropping the dL/dz term is flagged


def test_header_declares_the_entries():
    src = open(f"{ROOT}/include/f3dgs_b200.h").read()
    for name, tail in (("f3dgs_forward_distortion", r"void\* cuda_stream,\s*int antialiasing,\s*float\* out_distortion"),
                       ("f3dgs_backward_distortion", r"float\* dL_dcamera,\s*int antialiasing,\s*const float\* depth,"
                                                     r"\s*const float\* dL_ddistortion,\s*float\* dL_dmean2D_abs"),
                       ("f3dgs_backward_accum_distortion", r"float\* dL_dcamera,\s*int antialiasing,\s*const float\* "
                                                           r"depth,\s*const float\* dL_ddistortion,\s*float\* "
                                                           r"dL_dmean2D_abs,\s*float\* grad_accum_abs")):
        assert re.search(r"int " + name + r"\([^;]*" + tail + r"\);", src), name
        # the rest is the counterpart's argument list
        base = name.replace("distortion", "antialiased")
        body = re.search(r"int " + name + r"\(([^;]*)\);", src).group(1)
        body0 = re.search(r"int " + base + r"\(([^;]*)\);", src).group(1)
        norm = lambda s: re.sub(r"\s+", " ", s)  # noqa: E731
        assert norm(body).startswith(norm(body0)), name


def test_python_surface():
    import diff_gaussian_rasterization as dgr
    from diff_gaussian_rasterization import _C
    from diff_gaussian_rasterization.parallel import ViewBatch

    assert "rasterize_gaussians_distortion" in dgr.__all__ and "DistortionGaussianRasterizer" in dgr.__all__
    sig = inspect.signature(dgr.DistortionGaussianRasterizer.__init__)
    assert list(sig.parameters) == ["self", "raster_settings", "feature_geometry", "antialiasing"]
    sig = inspect.signature(dgr.rasterize_gaussians_distortion)
    assert list(sig.parameters) == list(inspect.signature(dgr.rasterize_gaussians).parameters) + [
        "feature_geometry", "antialiasing"]
    sig = inspect.signature(ViewBatch.backward)
    assert list(sig.parameters)[-3:] == ["g_distortion", "g_alpha", "g_invdepth"]
    assert sig.parameters["g_distortion"].default is None
    assert list(inspect.signature(ViewBatch.forward_distortion).parameters) == ["self", "rs", "antialiasing"]
    assert "debug: bool, antialiasing: bool = False" in _C.rasterize_gaussians_distortion.__doc__
    assert ("depth: torch.Tensor, dL_ddistortion: torch.Tensor, camera: bool = False, semantic_feature: "
            "torch.Tensor | None = None, antialiasing: bool = False, dL_dmean2D_abs: torch.Tensor | None = None"
            ) in _C.rasterize_gaussians_backward_distortion.__doc__
    assert ("depth: torch.Tensor | None = None, g_distortion: torch.Tensor | None = None"
            in _C.rasterize_gaussians_backward_accum.__doc__)


def test_view_batch_rejects_misuse():
    from diff_gaussian_rasterization.parallel import ViewBatch, _ViewCtx

    vb = ViewBatch.__new__(ViewBatch)
    ctx = _ViewCtx()
    ctx.depth = None
    g = torch.zeros(1, 4, 4)
    with pytest.raises(ValueError, match="forward_distortion"):
        vb.backward(ctx, None, None, None, g_distortion=g)
    ctx.depth = g
    with pytest.raises(ValueError, match="g_alpha"):
        vb.backward(ctx, None, None, None, g_alpha=g, g_distortion=g)


def test_entries_check_their_arguments_before_any_launch(lib):
    from test_antialiasing import ACCUM_OUTS, BWD_OUTS, _accum_args, _bwd_args, _fake

    null = ctypes.c_void_p(0)
    n0 = lib.f3dgs_launch_count()
    ins = [_fake(40), _fake(41)]  # depth, dL_ddistortion
    for name, mk, outs, tail in (("f3dgs_backward_distortion", _bwd_args, BWD_OUTS, [null]),
                                 ("f3dgs_backward_accum_distortion", _accum_args, ACCUM_OUTS, [null, null])):
        fn = getattr(lib, name)
        for k in (0, 1):
            pl = list(ins)
            pl[k] = null
            assert fn(*mk(5), 0, *pl, *tail) == -1
            assert lib.f3dgs_last_error() == (name + ": NULL depth / dL_ddistortion").encode()
            for i in outs:  # an input plane overlapping an output
                a = mk(5)
                pl = list(ins)
                pl[k] = ctypes.c_void_p(a[i].value + 4)
                assert fn(*a, 1, *pl, *tail) == -1, (name, i)
                assert b"depth / dL_ddistortion overlap an output" in lib.f3dgs_last_error(), (name, i)
        # the statistic overlapping another output
        a = mk(5)
        t = list(tail)
        t[0] = ctypes.c_void_p(a[outs[0]].value + 4)
        assert fn(*a, 0, *ins, *t) == -1 and b"dL_dmean2D_abs overlaps another output" in lib.f3dgs_last_error()
        assert fn(*mk(5, sf_dtype=9), 0, *ins, *tail) == -1 and b"unknown dtype code" in lib.f3dgs_last_error()
        assert fn(*mk(0), 0, *ins, *tail) == 0  # P == 0
    assert lib.f3dgs_backward_accum_distortion(*_accum_args(5), 0, *ins, null, _fake(50)) == -1
    assert b"grad_accum_abs needs dL_dmean2D_abs" in lib.f3dgs_last_error()

    alloc = ctypes.CFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t)(lambda ctx, n: None)
    f = ctypes.c_float
    p = _fake

    def fwd(dtype=F32):
        return [alloc, null, alloc, null, alloc, null, 5, 0, 1, 4, p(0), 64, 64, p(1), p(2), null, p(3), dtype, p(5),
                p(6), f(1.0), p(7), null, p(8), p(9), p(10), f(0.5), f(0.5), 0, p(11), p(12), p(13), p(14), 0, null]

    fn = lib.f3dgs_forward_distortion
    assert fn(*fwd(), 0, null) == -1
    assert lib.f3dgs_last_error() == b"f3dgs_forward_distortion: NULL out_distortion"
    assert fn(*fwd(dtype=5), 1, ins[0]) == -1 and b"unknown dtype code" in lib.f3dgs_last_error()
    for i in (29, 30, 31, 32):  # out_color, out_feature_map, out_depth, radii
        a = fwd()
        assert fn(*a, 0, ctypes.c_void_p(a[i].value + 8)) == -1, i
        assert b"out_distortion overlaps another output" in lib.f3dgs_last_error(), i
    assert lib.f3dgs_launch_count() == n0


# ------------------------------------------------------------------------------------------------------------ GPU: forward
def _forward_ctypes(lib, sc, cam, sf, aa, dev="cuda"):
    """f3dgs_forward_distortion with NaN-prefilled outputs and torch-owned buffers -> dict"""
    d = scenegen.to_torch(sc, dev)
    H, W, P = cam.image_height, cam.image_width, sc.P
    C = sf.shape[-1] if sf.numel() else 0
    keep = []

    def grow(ctx, n):
        keep.append(torch.empty(max(int(n), 1), dtype=torch.uint8, device=dev))
        return keep[-1].data_ptr()

    alloc = ctypes.CFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t)(grow)
    nan = lambda *s, dt=torch.float32: torch.full(s, float("nan"), dtype=dt, device=dev)  # noqa: E731
    o = dict(color=nan(3, H, W), fmap=nan(C, H, W, dt=sf.dtype), depth=nan(1, H, W), distortion=nan(1, H, W),
             radii=torch.full((P,), -7, dtype=torch.int32, device=dev))
    vm, pm, cp = (torch.tensor(a, device=dev).contiguous() for a in (cam.viewmatrix, cam.projmatrix, cam.campos))
    bg = torch.tensor(sc.bg, device=dev)
    f = ctypes.c_float
    sfp = sf.contiguous()
    R = lib.f3dgs_forward_distortion(
        alloc, None, alloc, None, alloc, None, P, sc.sh_degree, d["shs"].shape[1], C, _ptr(bg), W, H,
        _ptr(d["means3D"]), _ptr(d["shs"]), None, _ptr(sfp), F16 if sf.dtype == torch.float16 else F32,
        _ptr(d["opacities"]), _ptr(d["scales"]), f(1.0), _ptr(d["rotations"]), None, _ptr(vm), _ptr(pm), _ptr(cp),
        f(cam.tanfovx), f(cam.tanfovy), 0, _ptr(o["color"]), _ptr(o["fmap"]), _ptr(o["depth"]), _ptr(o["radii"]), 0,
        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream), int(aa), _ptr(o["distortion"]))
    assert R >= 0, lib.f3dgs_last_error()
    torch.cuda.synchronize()
    o["R"], (o["geom"], o["img"], o["binning"]) = R, keep[:3]  # the allocators' call order
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("C", [0, 32, 128, 256])
def test_forward_is_the_plain_forward_plus_the_plane(lib, C, dtype, aa):
    from test_alpha_invdepth import _plain_forward, _views
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
    vis = ref["radii"] > 0
    vn, vr = _views(new, sc, cam), _views(ref, sc, cam)
    for a, b, k in zip(vn, vr, ("point_list", "ranges", "n_contrib", "final_T", "rec")):
        assert torch.equal(a[vis] if k == "rec" else a, b[vis] if k == "rec" else b), k
    dist = new["distortion"]
    assert not bool(dist.isnan().any()) and bool((dist >= 0).all())
    assert bool((dist.reshape(-1)[vn[2].reshape(-1) == 0] == 0).all())  # nothing blended: 0
    # record depths are non-decreasing along every tile list
    pl, rg, rec = vn[0].long(), vn[1].long(), vn[4]
    z = rec[pl, 11]
    L = rg[:, 1] - rg[:, 0]
    tile = torch.repeat_interleave(torch.arange(L.numel(), device=pl.device), L)  # the lists are in tile order
    assert tile.numel() == pl.numel() and bool((z > 0).all())
    same = tile[1:] == tile[:-1]
    assert bool((z[1:][same] >= z[:-1][same]).all())


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "inside", "needles", "layers129", "opaque"])
def test_plane_matches_the_model_per_pixel(lib, name):
    from test_geometry_grads import _view

    v = _view(name)
    new = _forward_ctypes(lib, v.sc, v.cam, v.feats, False)
    for k in ("color", "depth"):
        assert torch.equal(new[k], v.base[k]), k
    dev = v.pairs.pix.device
    L, bar = distortion_model(v.pairs, v.w, v.base["rec"].to(dev))
    ours = new["distortion"].reshape(-1).to(dev).double()
    r = float(bw._ratio((ours - L).abs(), bar).max())
    print(f"[{name}] distortion worst |err|/bar {r:.3g}, max L {float(L.max()):.3g}")
    assert r <= 1.0 and bool((L > 0).any())


def _block():
    from test_alpha_invdepth import _block as blk

    return blk()


@pytest.mark.gpu
def test_two_gaussian_pixels(lib):
    """The block scene: every pixel blends at most the two Gaussians of its block, so L_p = 2 w1 w2 (z2 - z1)."""
    from diff_gaussian_rasterization import _C
    from test_alpha_invdepth import _plain_forward, _views

    sc, cam = _block()
    H, W, P = cam.image_height, cam.image_width, sc.P
    e = torch.empty(0, device="cuda")
    new = _forward_ctypes(lib, sc, cam, e, False)
    pl, rg, nc, final_T, rec = _views(new, sc, cam)
    pairs = bw.Pairs(pl, rg, nc, W, H)

    def render(g0, C):
        sf = torch.zeros(P, 1, C, device="cuda")
        sf[g0:g0 + C, 0] = torch.eye(C, device="cuda")
        return _plain_forward(sc, cam, sf, False)["fmap"].reshape(C, -1)

    w = bw.extract(pairs, P, render, 256)
    pix, gid, wv, z, first = blended(pairs, w, rec)
    n = torch.zeros(pairs.HW, dtype=torch.long, device=pix.device).index_add(0, pix, torch.ones_like(pix))
    assert int(n.max()) == 2 and int((n == 2).sum()) > 100
    two = (n[pix] == 2) & (torch.arange(pix.numel(), device=pix.device) == first)
    i = torch.nonzero(two).reshape(-1)
    want = 2 * wv[i] * wv[i + 1] * (z[i + 1] - z[i])
    assert bool((want > 0).all())
    L, bar = distortion_model(pairs, w, rec)
    assert torch.allclose(L[pix[i]], want, rtol=1e-8, atol=1e-12)  # the model's prefix sums: one float64 cumsum
    got = new["distortion"].reshape(-1).double()
    r = float(bw._ratio((got[pix[i]] - want).abs(), bar[pix[i]]).max())
    print(f"two-Gaussian pixels: {i.numel()}, worst |err|/bar {r:.3g}")
    assert r <= 1.0
    assert bool((got[pix[n[pix] == 1]] == 0).all())


# ----------------------------------------------------------------------------------------------------------- GPU: backward
def _bargs(sc, cam, f, sf, ups, dev="cuda"):
    from test_alpha_invdepth import _bargs as b

    return b(sc, cam, f, sf, ups, dev)


def _dist_grad(H, W, seed, dynamic=False):
    rng = np.random.default_rng(seed)
    g = rng.standard_normal((1, H, W)).astype(np.float32)
    if dynamic:
        g = g * (10.0 ** rng.uniform(-6.0, 0.0, (1, H, W))).astype(np.float32)
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "inside", "needles", "plane", "layers129", "opaque", "fx!=fy",
                                  "cov3D_precomp"])
def test_backward_matches_the_model(lib, name):
    from test_geometry_grads import _report, _upstreams, _view, preprocess_check

    v = _view(name)
    HW = v.W * v.H
    rec = v.base["rec"]
    dev = v.pairs.pix.device
    Wt = bw.Weights(v.pairs, v.w, v.P)
    for i, (label, ups) in enumerate(_upstreams(v.H, v.W, v.C, 71)):
        g = _dist_grad(v.H, v.W, 90 + i, dynamic=label == "dynamic range")
        ug = [_t(u, "cuda") for u in ups]
        z = lambda *s: torch.zeros(*s, device="cuda")  # noqa: E731
        m = dict(mean2D=z(v.P, 3), conic=z(v.P, 4), opacity=z(v.P), color=z(v.P, 3), feat=z(v.P, v.C),
                 means3D=z(v.P, 3), cov3D=z(v.P, 6), sh=z(v.P, v.M, 3), scales=z(v.P, 3), rotations=z(v.P, 4),
                 dz=z(v.P))
        _ctypes_backward(lib, v, ug, _t(g, "cuda"), m)
        Gc, Gd = ug[0].reshape(3, HW).t().to(dev), ug[2].reshape(HW).to(dev)
        G = _t(g).reshape(HW).to(dev)
        ref, bar, dz, mcount = backward_model(v.pairs, v.w, rec.to(dev), v.P, v.bg, Gc, Gd, G)
        g6 = bw.geom6(m["mean2D"], m["conic"], m["opacity"]).double().to(ref.device)
        rr = bw._ratio((g6 - ref).abs(), bar).max(0).values
        worst = {k: float(x) for k, x in zip(("dL_dmean2D.x", "dL_dmean2D.y", "dL_dconic.a", "dL_dconic.b",
                                              "dL_dconic.c", "dL_dopacity"), rr)}
        worst["dL_dcolor"] = Wt.per_gaussian(m["color"].reshape(v.P, 3), Gc)
        worst["dL_dz"] = bw.gaussian_ratio(m["dz"].reshape(v.P, 1).to(dev), dz, mcount)
        worst.update(preprocess_check(v.chain(m), v.outputs(m), v.visible))
        _report(f"{name} distortion {label}", worst)
        # negative controls: the ablated models are outside the bar of ours (not on the planar scene, whose pixels
        # blend Gaussians of nearly one depth, where every form of the loss is nearly 0)
        if label == "N(0,1)" and name != "plane":
            for form in ("no_abar", "squared"):
                x, _, _, _ = backward_model(v.pairs, v.w, rec.to(dev), v.P, v.bg, Gc, Gd, G, form)
                assert float(bw._ratio((g6 - x).abs(), bar).max()) > 1.0, form


def _ctypes_backward(lib, v, ug, g, o):
    """f3dgs_backward_distortion into the zeroed dict o (v: test_geometry_grads.View)"""
    gc, gf, gd = ug
    null = ctypes.c_void_p(0)
    f = ctypes.c_float
    sr = v.scales.numel() > 0
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    b = v.base
    args = [v.P, v.D, v.M, b["R"], v.C, _ptr(v.bg), v.W, v.H, _ptr(v.d["means3D"]), _ptr(v.shs), _ptr(v.cols), null,
            F32, _ptr(v.scales), f(v.mod), _ptr(v.rots), _ptr(v.cov), _ptr(v.vm), _ptr(v.pm), _ptr(v.cp),
            f(v.cam.tanfovx), f(v.cam.tanfovy), _ptr(b["radii"]), _ptr(b["geom"]), _ptr(b["binning"]), _ptr(b["img"]),
            _ptr(gc), _ptr(gf), F32, f(1.0), _ptr(gd), _ptr(o["mean2D"]), _ptr(o["conic"]), _ptr(o["opacity"]),
            _ptr(o["color"]), _ptr(o["feat"]), _ptr(o["means3D"]), _ptr(o["cov3D"]), _ptr(o["sh"]) if v.M else null,
            _ptr(o["scales"]) if sr else null, _ptr(o["rotations"]) if sr else null, _ptr(o["dz"]), 0, stream, null,
            0, _ptr(b["depth"]), _ptr(g), null]
    rc = lib.f3dgs_backward_distortion(*args)
    assert rc == 0, lib.f3dgs_last_error()
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("C", [0, 8, 200])
def test_zero_gradient_gives_the_counterparts_bits(lib, C, aa):
    """g = 0: every output of the assigning and the accumulating entry is bitwise the counterpart's (block scene)"""
    from diff_gaussian_rasterization import _C
    from diff_gaussian_rasterization.parallel import ViewBatch
    from test_alpha_invdepth import _equal, _plain_forward, _settings

    sc, cam = _block()
    dev = torch.device("cuda")
    H, W = cam.image_height, cam.image_width
    sf = torch.randn(sc.P, 1, C, generator=torch.Generator().manual_seed(1)).to(dev) if C else torch.empty(0, device=dev)
    f = _plain_forward(sc, cam, sf, aa)
    z = torch.zeros(1, H, W, device=dev)
    gc, gf, gd = (_t(u, dev) for u in bw.upstream(H, W, C, 3))
    for half in (False, True):
        a = _bargs(sc, cam, f, sf, (gc, gf.half() if half else gf, gd))
        new = lambda **kw: _C.rasterize_gaussians_backward_distortion(*a, f["depth"], z, antialiasing=aa, **kw)  # noqa
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
        # with the AbsGS statistic: _absgrad's bits
        m_abs = torch.zeros(sc.P, 3, device=dev)
        r = new(camera=True, dL_dmean2D_abs=m_abs)
        ra = _C.rasterize_gaussians_backward_absgrad(*a, camera=True, antialiasing=aa)
        _equal(r, ra[:12], "absgrad")
        assert torch.equal(m_abs, ra[12])
    d = scenegen.to_torch(sc, dev)
    params = dict(means3D=d["means3D"], scales=d["scales"], rotations=d["rotations"], opacities=d["opacities"],
                  shs=d["shs"], semantic_feature=sf if C else None)
    rs = _settings(sc, cam)
    for camera, fg, absgrad in ((True, bool(C), False), (False, False, True)):
        outs = []
        for dist in (False, True):
            vb = ViewBatch(params, absgrad=absgrad)
            ctx = vb.forward_distortion(rs, antialiasing=aa)[-1] if dist else vb.forward(rs, antialiasing=aa)[-1]
            cg = vb.backward(ctx, gc, gf if C else None, gd, camera=camera, feature_geometry=fg,
                             g_distortion=z if dist else None)
            outs.append((vb.flat.clone(), None if cg is None else torch.cat([cg.viewmatrix.reshape(-1),
                                                                              cg.projmatrix.reshape(-1), cg.campos]),
                         None if vb.mean2D_abs is None else vb.mean2D_abs.clone()))
        _equal(outs[0], outs[1], ("accum", camera, fg, absgrad))


@pytest.mark.gpu
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("antialiasing", [False, True])
@pytest.mark.parametrize("feature_geometry", [False, True])
@pytest.mark.parametrize("camera", [False, True])
def test_autograd_and_view_batch_equal_the_binding(lib, camera, feature_geometry, antialiasing, half):
    """DistortionGaussianRasterizer's gradients are the binding's bits; ViewBatch (float16 rows with a ScaledGrad map
    when half, and absgrad) sums the same over three views; colour-only losses keep GaussianRasterizer's bits."""
    import diff_gaussian_rasterization as dgr
    from diff_gaussian_rasterization import _C
    from diff_gaussian_rasterization.parallel import ViewBatch
    from test_alpha_invdepth import _plain_forward, _settings

    sc, cam = _block()
    dev = torch.device("cuda")
    H, W = cam.image_height, cam.image_width
    d = scenegen.to_torch(sc, dev, requires_grad=True)
    if half:
        d["semantic_feature"] = d["semantic_feature"].detach().half().requires_grad_()
    rs = _settings(sc, cam)
    if camera:
        rs = rs._replace(viewmatrix=rs.viewmatrix.clone().requires_grad_(),
                         projmatrix=rs.projmatrix.clone().requires_grad_(), campos=rs.campos.clone().requires_grad_())
    ups = [_t(u, dev) for u in bw.upstream(H, W, sc.C, 8)] + [_t(_dist_grad(H, W, 9), dev)]
    if half:
        ups[1] = ups[1].half()
    ras = dgr.DistortionGaussianRasterizer(rs, feature_geometry=feature_geometry, antialiasing=antialiasing)
    kw = dict(means3D=d["means3D"], means2D=torch.zeros_like(d["means3D"]), opacities=d["opacities"], shs=d["shs"],
              semantic_feature=d["semantic_feature"], scales=d["scales"], rotations=d["rotations"])
    color, fmap, radii, depth, distortion = ras(**kw)
    loss = (color * ups[0]).sum() + (fmap * ups[1]).sum() + (depth * ups[2]).sum() + (distortion * ups[3]).sum()
    cam_t = [rs.viewmatrix, rs.projmatrix, rs.campos] if camera else []
    keys = ("means3D", "opacities", "shs", "scales", "rotations", "semantic_feature")
    got = torch.autograd.grad(loss, [d[k] for k in keys] + cam_t)
    sf = d["semantic_feature"].detach()
    f = _plain_forward(sc, cam, sf, antialiasing)
    assert torch.equal(depth, f["depth"])
    r = _C.rasterize_gaussians_backward_distortion(
        *_bargs(sc, cam, f, sf, ups[:3]), f["depth"], ups[3], camera=camera,
        semantic_feature=sf if feature_geometry else None, antialiasing=antialiasing)
    want = (r[4], r[3], r[6], r[7], r[8], r[2]) + tuple(r[9:12] if camera else ())
    for k, a, b in zip(keys + ("viewmatrix", "projmatrix", "campos"), got, want):
        assert torch.equal(a.reshape(b.shape), b.to(a.dtype)), k
    # the distortion moves geometry
    plain = _C.rasterize_gaussians_backward_distortion(
        *_bargs(sc, cam, f, sf, ups[:3]), f["depth"], torch.zeros_like(ups[3]), antialiasing=antialiasing,
        semantic_feature=sf if feature_geometry else None)
    assert not torch.equal(plain[3], r[3])
    # a colour-only loss: the counterpart rasterizer's gradients
    base = (dgr.AntialiasedGaussianRasterizer if antialiasing else dgr.GaussianRasterizer)(
        rs, feature_geometry=feature_geometry)
    o1, o2 = ras(**kw), base(**kw)
    assert torch.equal(o1[0], o2[0]) and torch.equal(o1[3], o2[3])
    ga = torch.autograd.grad((o1[0] * ups[0]).sum(), [d[k] for k in keys[:5]] + cam_t)
    gb = torch.autograd.grad((o2[0] * ups[0]).sum(), [d[k] for k in keys[:5]] + cam_t)
    for a, b in zip(ga, gb):
        assert torch.equal(a, b)
    # ViewBatch: the sum over three views equals the binding's sum; absgrad's statistic is the binding's
    P = sc.P
    dd = {k: v.detach() for k, v in d.items()}
    params = dict(means3D=dd["means3D"], scales=dd["scales"], rotations=dd["rotations"], opacities=dd["opacities"],
                  shs=dd["shs"], semantic_feature=dd["semantic_feature"])
    vb = ViewBatch(params, absgrad=True)
    tot = {k: 0 for k in ("means3D", "opacities", "semantic_feature")}
    for i in range(3):
        gv = [_t(u, dev) for u in bw.upstream(H, W, sc.C, 30 + i)] + [_t(_dist_grad(H, W, 40 + i), dev)]
        gmap = gv[1].half() if half else gv[1]  # float16 rows render a float16 map; its gradient as a ScaledGrad
        color, feat, radii, depth, distortion, ctx = vb.forward_distortion(rs, antialiasing=antialiasing)
        assert ctx.depth is depth
        cg = vb.backward(ctx, gv[0], (gmap, 1.0) if half else gmap, gv[2], camera=camera,
                         feature_geometry=feature_geometry, g_distortion=gv[3])
        fv = dict(R=ctx.num_rendered, radii=ctx.radii, geom=ctx.geom, binning=ctx.binning, img=ctx.img)
        m_abs = torch.zeros(P, 3, device=dev)
        rv = _C.rasterize_gaussians_backward_distortion(
            *_bargs(sc, cam, fv, dd["semantic_feature"], (gv[0], gmap, gv[2])), depth, gv[3],
            camera=camera, semantic_feature=dd["semantic_feature"] if feature_geometry else None,
            antialiasing=antialiasing, dL_dmean2D_abs=m_abs)
        assert torch.allclose(vb.mean2D_abs, m_abs, rtol=1e-6, atol=0)
        if camera:
            assert torch.equal(torch.cat([cg.viewmatrix.reshape(-1), cg.projmatrix.reshape(-1), cg.campos]),
                               torch.cat([rv[9].reshape(-1), rv[10].reshape(-1), rv[11]]))
        for k, x in (("means3D", rv[4]), ("opacities", rv[3]), ("semantic_feature", rv[2])):
            tot[k] = tot[k] + x
    for k, x in tot.items():
        got = vb.grads[k].reshape(x.shape)
        sc_ = float(x.abs().max())
        assert sc_ > 0
        assert torch.allclose(got, x, rtol=1e-4, atol=1e-5 * sc_), k


@pytest.mark.gpu
def test_distortion_loss_trains():
    """On a two-layer scene with fixed colour, Adam steps on the distortion alone lower its sum and keep opacities
    finite."""
    import diff_gaussian_rasterization as dgr
    from test_alpha_invdepth import _settings

    sc, cam = _block()
    dev = torch.device("cuda")
    rs = _settings(sc, cam)
    d = scenegen.to_torch(sc, dev)
    ras = dgr.DistortionGaussianRasterizer(rs)
    # wider Gaussians so that both layers blend over many pixels
    raw_s = torch.log(d["scales"] * 3.0).requires_grad_()
    raw_o = torch.logit(d["opacities"].clamp(0.02, 0.98) * 4).requires_grad_()
    means = d["means3D"].clone().requires_grad_()
    opt = torch.optim.Adam([raw_s, raw_o, means], lr=1e-2)
    sums = []
    for _ in range(40):
        out = ras(means3D=means, means2D=torch.zeros_like(means), opacities=torch.sigmoid(raw_o),
                  colors_precomp=torch.full_like(means, 0.5), scales=torch.exp(raw_s), rotations=d["rotations"])
        loss = out[4].sum()
        opt.zero_grad()
        loss.backward()
        opt.step()
        sums.append(float(loss))
        assert bool(torch.isfinite(raw_o).all())
    print(f"distortion sum {sums[0]:.4g} -> {sums[-1]:.4g}")
    assert sums[0] > 0 and sums[-1] < 0.8 * sums[0]


@pytest.mark.gpu
def test_accumulating_binding_rejects_an_empty_depth_plane():
    """The depth plane is an input the backward reads: an empty or missing one is an error, never zeros."""
    from diff_gaussian_rasterization import _C
    from diff_gaussian_rasterization.parallel import ViewBatch
    from test_alpha_invdepth import _settings

    sc, cam = _block()
    dev = torch.device("cuda")
    H, W = cam.image_height, cam.image_width
    d = scenegen.to_torch(sc, dev)
    vb = ViewBatch(dict(means3D=d["means3D"], scales=d["scales"], rotations=d["rotations"], opacities=d["opacities"],
                        shs=d["shs"]))
    *_, ctx = vb.forward_distortion(_settings(sc, cam))
    g = torch.ones(1, H, W, device=dev)
    gc, _, gd = (_t(u, dev) for u in bw.upstream(H, W, 0, 3))
    for depth in (torch.empty(0, device=dev), torch.zeros(H * W - 1, device=dev)):
        ctx.depth = depth
        with pytest.raises(RuntimeError, match="depth must have H \\* W"):
            vb.backward(ctx, gc, None, gd, g_distortion=g)
    f = dict(R=ctx.num_rendered, radii=ctx.radii, geom=ctx.geom, binning=ctx.binning, img=ctx.img)
    with pytest.raises(RuntimeError, match="depth must have H \\* W"):
        _C.rasterize_gaussians_backward_distortion(*_bargs(sc, cam, f, torch.empty(0, device=dev), (gc, e := torch.empty(
            0, device=dev), gd)), e, g)
    assert bool((vb.flat == 0).all())  # nothing was launched into the buffers
