"""Antialiased rendering: the opacity compensation of the 0.3 px^2 dilation (f3dgs_forward_antialiased,
f3dgs_backward_antialiased, f3dgs_backward_accum_antialiased, rasterize_gaussians_antialiased,
AntialiasedGaussianRasterizer, ViewBatch.forward(antialiasing=True), FeatureLift(antialiasing=True)).

The model is a float64 restatement of the antialiased preprocess, on camera_grad_model's conventions: (means3D, cov3D or
scale / rotation, opacity, camera) -> (NDC mean, conic, op_eff, colour, depth), with
    det0 = a0 c0 - b^2,  det = (a0 + 0.3)(c0 + 0.3) - b^2,  op_eff = opacity * sqrt(max(2.5e-5, det0 / det)).
CPU: the model's op_eff gradient against central differences, the resolution consistency the compensation exists for,
and the C entries' argument checks.  GPU: the antialiased render is bitwise the default render on op_eff; the native
backward matches the model pushed through by autograd from the composite's own per-Gaussian gradients; bitwise checks on
a view whose composite does not depend on atomic order; autograd, view batches, lifting and an end-to-end resolution
check.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import camera_grad_model as cgm
import scenegen
from camera_grad_model import cov3d_from_scale_rot

torch.set_default_dtype(torch.float32)
MIN_RATIO = 2.5e-5
F32, F16 = 0, 1


# ------------------------------------------------------------------------------------------------------------ model
def aa_quantities(means3D, cov3D, opacity, vm, pm, campos, W, H, tanfovx, tanfovy, deg=0, shs=None, colors=None):
    """-> (ndc [P,2], conic (A, B, C), op_eff [P], colour [P,3], depth [P], (a0, b, c0)), float64, differentiable.  The
    conventions (clamped Jacobian entries detached, 1e-7 in the screen mean, the conic's 1/(det^2 + 1e-7)) are
    camera_grad_model's."""
    P = means3D.shape[0]
    vm = vm.expand(P, 16) if vm.dim() == 1 else vm
    pm = pm.expand(P, 16) if pm.dim() == 1 else pm
    campos = campos.expand(P, 3) if campos.dim() == 1 else campos
    p = torch.cat([means3D, torch.ones_like(means3D[:, :1])], 1)

    def row(m, r):
        return (m[:, r::4] * p).sum(1)

    hx, hy, hw = row(pm, 0), row(pm, 1), row(pm, 3)
    p_w = 1.0 / (hw + 1e-7)
    ndc = torch.stack([hx * p_w, hy * p_w], 1)
    tx, ty, tz = row(vm, 0), row(vm, 1), row(vm, 2)
    fx, fy = W / (2.0 * tanfovx), H / (2.0 * tanfovy)
    limx, limy = 1.3 * tanfovx, 1.3 * tanfovy
    rx, ry = tx / tz, ty / tz
    cx, cy = (rx < -limx) | (rx > limx), (ry < -limy) | (ry > limy)
    tx = torch.where(cx, (rx.clamp(-limx, limx) * tz).detach(), tx)
    ty = torch.where(cy, (ry.clamp(-limy, limy) * tz).detach(), ty)
    zero = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, zero, -fx * tx / (tz * tz)], 1),
                     torch.stack([zero, fy / tz, -fy * ty / (tz * tz)], 1)], 1)
    Wr = torch.stack([vm[:, 0:3], vm[:, 4:7], vm[:, 8:11]], 1)
    T = J @ Wr.transpose(1, 2)
    c = cov3D
    V = torch.stack([torch.stack([c[:, 0], c[:, 1], c[:, 2]], 1), torch.stack([c[:, 1], c[:, 3], c[:, 4]], 1),
                     torch.stack([c[:, 2], c[:, 4], c[:, 5]], 1)], 1)
    S = T @ V @ T.transpose(1, 2)
    a0, b, c0 = S[:, 0, 0], S[:, 0, 1], S[:, 1, 1]
    A, B, C = cgm._Conic.apply(a0 + 0.3, b, c0 + 0.3)
    ratio = (a0 * c0 - b * b) / ((a0 + 0.3) * (c0 + 0.3) - b * b)
    op_eff = opacity.reshape(-1) * torch.sqrt(torch.clamp(ratio, min=MIN_RATIO))
    if colors is None:
        d = means3D - campos
        d = d / d.norm(dim=1, keepdim=True)
        colors = cgm.sh_color(deg, shs, d).clamp_min(0.0)
    return ndc, (A, B, C), op_eff, colors, row(vm, 2), (a0, b, c0)


def _f64(a):
    return torch.as_tensor(np.asarray(a) if not isinstance(a, torch.Tensor) else a.cpu()).double()


def model_gradients(sc, cam, grads, idx, mod=1.0, cov=None, colors=None):
    """Float64 gradients of sum(q . grads) over the Gaussians `idx`, for grads = (dL_dmean2D, dL_dconic, dL/dop_eff,
    dL_dcolor, dL_dz) of the composite.  cov: [P,6] precomputed covariances (else scale / rotation).  -> dict of full
    [P, ...] tensors (0 outside idx), with kappa and eig_ratio of the dilated 2-D covariance."""
    P = sc.P
    m = _f64(sc.means3D)[idx].clone().requires_grad_()
    op = _f64(sc.opacities).reshape(-1)[idx].clone().requires_grad_()
    vm, pm, cp = (_f64(a).reshape(-1).clone().requires_grad_() for a in (cam.viewmatrix, cam.projmatrix, cam.campos))
    leaves = [m, op, vm, pm, cp]
    if cov is None:
        # as in the reference backward, dL_dscale is the gradient of the modified scale (scale_modifier * scale)
        s = (_f64(sc.scales)[idx] * mod).clone().requires_grad_()
        r = _f64(sc.rotations)[idx].clone().requires_grad_()
        cv = cov3d_from_scale_rot(s, r)
        leaves += [s, r]
    else:
        cv = _f64(cov)[idx].clone().requires_grad_()
        leaves += [cv]
    q = aa_quantities(m, cv, op, vm, pm, cp, cam.image_width, cam.image_height, cam.tanfovx, cam.tanfovy,
                      sc.sh_degree, shs=None if colors is not None else _f64(sc.shs)[idx],
                      colors=None if colors is None else _f64(colors)[idx])
    ndc, (A, B, C), op_eff, col, depth, _ = q
    g = [_f64(x).reshape(P, -1)[idx] for x in grads]
    L = ((ndc * g[0][:, :2]).sum() + (A * g[1][:, 0] + 2 * B * g[1][:, 1] + C * g[1][:, 3]).sum()
         + (op_eff * g[2][:, 0]).sum() + (col * g[3]).sum() + (depth * g[4][:, 0]).sum())
    out_g = torch.autograd.grad(L, leaves, allow_unused=True)
    names = ["means3D", "opacity", "vm", "pm", "campos"] + (["scales", "rotations"] if cov is None else ["cov3D"])
    widths = dict(means3D=3, opacity=1, scales=3, rotations=4, cov3D=6)
    out = {}
    for k, v in zip(names, out_g):
        if k in widths:
            full = torch.zeros(P, widths[k], dtype=torch.float64)
            if v is not None:
                full[idx] = v.reshape(len(idx), -1)
            out[k] = full
        else:
            out[k] = torch.zeros(3 if k == "campos" else 16, dtype=torch.float64) if v is None else v
    out["camera"] = torch.cat([out["vm"], out["pm"], out["campos"]])
    A, B, C = (x.detach() for x in (A, B, C))
    mid, d = 0.5 * (A + C), torch.sqrt(0.25 * (A - C) ** 2 + B * B)
    for k, v in (("kappa", (A * C + B * B) / (A * C - B * B)), ("eig_ratio", (mid + d) / (mid - d))):
        out[k] = torch.zeros(P, dtype=torch.float64)
        out[k][idx] = v
    return out


# ------------------------------------------------------------------------------------------------------------ CPU
def test_model_op_eff_gradient_matches_central_differences():
    """d op_eff / d(opacity, 2-D covariance) of the model (the backward's formula, by autograd) against central
    differences, for well-resolved, sub-pixel and clamped Gaussians (where rho is constant: only dL/dopacity)."""
    torch.manual_seed(0)
    for a0, b, c0 in [(4.0, 1.0, 3.0), (0.25, 0.05, 0.2), (0.02, 0.0, 0.01), (1e-6, 0.0, 1e-6)]:
        x = torch.tensor([0.7, a0, b, c0], dtype=torch.float64, requires_grad=True)

        def f(v):
            det0 = v[1] * v[3] - v[2] * v[2]
            det = (v[1] + 0.3) * (v[3] + 0.3) - v[2] * v[2]
            return v[0] * torch.sqrt(torch.clamp(det0 / det, min=MIN_RATIO))

        g = torch.autograd.grad(f(x), x)[0]
        # the kernel's closed form (include/f3dgs_b200.h)
        a, c = a0 + 0.3, c0 + 0.3
        det0, det = a0 * c0 - b * b, a * c - b * b
        rho = math.sqrt(max(MIN_RATIO, det0 / det))
        h = 0.5 * 0.7 * rho if det0 / det > MIN_RATIO else 0.0
        closed = torch.tensor([rho, h * (c0 / det0 - c / det) if h else 0.0, 2 * h * b * (1 / det - 1 / det0) if h else 0.0,
                               h * (a0 / det0 - a / det) if h else 0.0], dtype=torch.float64)
        for j in range(4):
            eps = 1e-7 * max(1.0, abs(float(x[j].detach())))
            e = torch.zeros(4, dtype=torch.float64)
            e[j] = eps
            fd = (f(x.detach() + e) - f(x.detach() - e)) / (2 * eps)
            assert abs(float(fd - g[j])) <= 1e-6 * max(1.0, abs(float(g[j]))), (a0, j, float(fd), float(g[j]))
        assert torch.allclose(g, closed, rtol=1e-10, atol=1e-12), (g, closed)
        if det0 / det <= MIN_RATIO:
            assert float(g[1:].abs().max()) == 0.0


def _isolated(W, H, n=6, seed=3):
    """n isolated sub-pixel Gaussians (screen std. dev. 0.2 - 0.5 px at W x H), one per 32 x 32 cell, in front of a
    camera at the origin looking down +z."""
    rng = np.random.default_rng(seed)
    cam = scenegen.make_camera(W, H, np.array([0.0, 0.0, -5.0]))
    focal = W / (2 * cam.tanfovx)
    sc = scenegen.make_scene(n, W, H, 0, sh_degree=0, seed=seed)
    z = 5.0 + rng.uniform(-0.5, 0.5, n)
    cx = (np.arange(n) % (W // 32)) * 32 + 16.3
    cy = (np.arange(n) // (W // 32)) * 32 + 16.6
    vx, vy = ((2 * cx + 1) / W - 1) * cam.tanfovx * z, ((2 * cy + 1) / H - 1) * cam.tanfovy * z
    world = np.stack([vx, vy, z, np.ones(n)], 1) @ np.linalg.inv(cam.viewmatrix.astype(np.float64))
    sc.means3D = world[:, :3].astype(np.float32)
    sc.scales = (rng.uniform(0.2, 0.5, (n, 3)) * z[:, None] / focal).astype(np.float32)
    q = rng.standard_normal((n, 4))
    sc.rotations = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    sc.opacities = rng.uniform(0.6, 0.9, (n, 1)).astype(np.float32)
    sc.cameras = [cam]
    return sc, cam


def _scaled_camera(cam, k):
    """The camera at 1/k of its resolution (same field of view): a pixel covers k x k pixels of cam."""
    c = scenegen.make_camera(cam.image_width // k, cam.image_height // k, np.array([0.0, 0.0, -5.0]))
    c.viewmatrix, c.projmatrix, c.campos = cam.viewmatrix, cam.projmatrix, cam.campos
    c.tanfovx, c.tanfovy = cam.tanfovx, cam.tanfovy
    return c


def model_coverage(sc, cam, antialiasing):
    """Per Gaussian, the sum over the pixels of `cam` of alpha (the composite's alpha = min(0.99, op exp(-power)), cut
    below 1/255; the Gaussians are isolated, so T = 1), in float64, with the undilated integral op * 2 pi sqrt(det0) in
    the same pixels, the dilation's growth sqrt(det / det0) and the bar of the antialiased sum against the integral."""
    W, H = cam.image_width, cam.image_height
    P = sc.P
    cov = cov3d_from_scale_rot(_f64(sc.scales), _f64(sc.rotations))
    ndc, (A, B, C), op_eff, _, _, (a0, b, c0) = aa_quantities(
        _f64(sc.means3D), cov, _f64(sc.opacities), _f64(cam.viewmatrix).reshape(16), _f64(cam.projmatrix).reshape(16),
        _f64(cam.campos), W, H, cam.tanfovx, cam.tanfovy, 0, colors=torch.zeros(P, 3, dtype=torch.float64))
    op = op_eff if antialiasing else _f64(sc.opacities).reshape(-1)
    px = ((ndc[:, 0] + 1.0) * W - 1.0) * 0.5
    py = ((ndc[:, 1] + 1.0) * H - 1.0) * 0.5
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    cover = torch.zeros(P, dtype=torch.float64)
    for i in range(P):
        dx, dy = px[i] - xs, py[i] - ys
        power = -0.5 * (A[i] * dx * dx + C[i] * dy * dy) - B[i] * dx * dy
        alpha = torch.clamp(op[i] * torch.exp(power), max=0.99)
        alpha = torch.where((power <= 0) & (alpha >= 1.0 / 255.0), alpha, torch.zeros_like(alpha))
        cover[i] = alpha.sum()
    det0 = a0 * c0 - b * b
    det = (a0 + 0.3) * (c0 + 0.3) - b * b
    lam_min = 0.5 * (a0 + c0 + 0.6) - torch.sqrt(0.25 * (a0 - c0) ** 2 + b * b)
    # bar of the AA sum against the undilated integral: the mass the 1/255 cut removes (a fraction t = 1 / (255 op_eff)
    # of a Gaussian's integral outside its level set; sampled on the grid, at most 2 t), and the error of sampling the
    # Gaussian on the unit grid (Poisson summation: 4 exp(-2 pi^2 lambda_min) for lambda_min >= 0.3)
    bar = 2.0 / (255.0 * op_eff) + 4.0 * torch.exp(-2 * math.pi ** 2 * lam_min) + 1e-3
    return cover, _f64(sc.opacities).reshape(-1) * 2 * math.pi * torch.sqrt(det0), torch.sqrt(det / det0), bar


def test_model_resolution_consistency():
    """Sub-pixel Gaussians at 1x, 1/2x and 1/4x: with the compensation, the coverage (sum of alpha x pixel area) stays
    at the undilated integral within the bar the model gives; without it, it grows by the dilation's sqrt(det/det0)."""
    sc, cam = _isolated(192, 64)
    for k in (1, 2, 4):
        c = _scaled_camera(cam, k)
        aa, integral, growth, bar = model_coverage(sc, c, True)
        plain, _, _, _ = model_coverage(sc, c, False)
        # coverage and integral are both in pixels of c; times k^2 both are in pixels of cam, so the ratio is the same
        rel = (aa / integral - 1.0).abs()
        assert bool((rel <= bar).all()), (k, rel, bar)
        assert bool((plain / integral >= 0.9 * growth).all()), (k, plain / integral, growth)
        if k == 4:
            assert bool((growth > 5).all()), growth


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    return L


def _fake(i, off=0):
    return ctypes.c_void_p((1 << 40) + i * (1 << 20) + off)


def _bwd_args(P, C=4, sf_dtype=F32, map_dtype=F32, scale=1.0, sf=True):
    """f3dgs_backward_antialiased's arguments with distinct fake device addresses (the checks fail before any use;
    outputs at BWD_OUTS, dL_dopacity at BWD_OPACITY, dL_dcamera last)."""
    f, null = ctypes.c_float, ctypes.c_void_p(0)
    p = _fake
    return [P, 0, 1, 10, C, p(0), 64, 64, p(1), p(2), null, p(3) if sf else null, sf_dtype, p(4), f(1.0), p(5), null,
            p(6), p(7), p(8), f(0.5), f(0.5), p(9), p(10), p(11), p(12), p(13), p(14), map_dtype, f(scale), p(31),
            p(15), p(16), p(17), p(18), p(19), p(20), p(21), p(22), p(23), p(24), p(25), 0, null, null]


def _accum_args(P, C=4, sf_dtype=F32, map_dtype=F32, scale=1.0, sf=True):
    """f3dgs_backward_accum_antialiased's arguments (outputs at ACCUM_OUTS, dL_dopacity at ACCUM_OPACITY)."""
    f, null = ctypes.c_float, ctypes.c_void_p(0)
    p = _fake
    return [P, 0, 1, 10, C, p(0), 64, 64, p(1), p(2), null, p(3) if sf else null, sf_dtype, p(4), f(1.0), p(5), null,
            p(6), p(7), p(8), f(0.5), f(0.5), p(9), p(10), p(11), p(12), p(13), p(14), map_dtype, f(scale), p(31),
            p(30), p(15), null, p(17), p(18), null, p(20), p(21), p(22), p(23), p(24), p(25), null, 0, null, null]
# argument indices of the outputs: dL_dmean2D .. dL_dz of the assigning entry (32: dL_dconic .. 33 is dL_dopacity)
BWD_OUTS, BWD_OPACITY = (31, 32, 34, 35, 36, 37, 38, 39, 40, 41), 33
# scratch, dL_dsemantic_feature, dL_dmean3D, dL_dsh, dL_dscale, dL_drot, dL_dmean2D_out, grad_accum, denom
ACCUM_OUTS, ACCUM_OPACITY = (31, 34, 35, 37, 38, 39, 40, 41, 42), 32


def test_backward_entries_check_their_arguments(lib):
    for name, mk, opacity_at, outs in (("f3dgs_backward_antialiased", _bwd_args, BWD_OPACITY, BWD_OUTS),
                                       ("f3dgs_backward_accum_antialiased", _accum_args, ACCUM_OPACITY, ACCUM_OUTS)):
        fn = getattr(lib, name)
        for kw in (dict(sf_dtype=7), dict(map_dtype=-1)):
            assert fn(*mk(5, **kw)) == -1
            assert lib.f3dgs_last_error() == (name + ": unknown dtype code").encode()
        a = mk(5, map_dtype=F16, scale=float("inf"))
        assert fn(*a) == -1 and b"dL_dfeaturepix_scale must be finite and nonzero" in lib.f3dgs_last_error()
        assert fn(*mk(5, map_dtype=F16, scale=0.0)) == -1
        for i in (opacity_at, outs[2]):  # dL_dopacity, dL_dmean3D
            a = mk(5)
            a[i] = ctypes.c_void_p(0)
            assert fn(*a) == -1 and b"NULL gradient pointer" in lib.f3dgs_last_error(), (name, lib.f3dgs_last_error())
        # semantic_feature overlapping an output
        for i in outs:
            a = mk(5)
            a[11] = ctypes.c_void_p(a[i].value + 4)
            assert fn(*a) == -1, (name, i)
            assert b"semantic_feature overlaps an output" in lib.f3dgs_last_error(), (name, i, lib.f3dgs_last_error())
        # dL_dcamera overlapping an output
        for i in outs:
            a = mk(5)
            a[-1] = ctypes.c_void_p(a[i].value + 4)
            assert fn(*a) == -1, (name, i)
            assert b"dL_dcamera overlaps another output" in lib.f3dgs_last_error(), (name, i)
        # dL_dopacity, which the preprocess backward writes, overlapping another output
        for i in outs:
            if i == opacity_at:
                continue
            a = mk(5, sf=False)
            a[opacity_at] = ctypes.c_void_p(a[i].value + 4)
            assert fn(*a) == -1, (name, i)
            assert b"overlaps" in lib.f3dgs_last_error(), (name, i, lib.f3dgs_last_error())
        assert fn(*mk(0)) == 0  # P == 0


def test_forward_entry_checks_its_arguments(lib):
    null = ctypes.c_void_p(0)
    alloc = ctypes.CFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t)(lambda ctx, n: None)
    f = ctypes.c_float
    p = _fake

    def args(dtype=F32, opac=p(5)):
        return [alloc, null, alloc, null, alloc, null, 5, 0, 1, 4, p(0), 64, 64, p(1), p(2), null, p(3), dtype, opac,
                p(6), f(1.0), p(7), null, p(8), p(9), p(10), f(0.5), f(0.5), 0, p(11), p(12), p(13), null, 0, null]

    assert lib.f3dgs_forward_antialiased(*args(dtype=3)) == -1
    assert lib.f3dgs_last_error() == b"f3dgs_forward_antialiased: unknown dtype code"
    assert lib.f3dgs_forward_antialiased(*args(opac=null)) == -1
    assert lib.f3dgs_last_error() == b"f3dgs_forward_antialiased: NULL required pointer"
    a = args()
    a[16] = null  # semantic_feature with C = 4
    assert lib.f3dgs_forward_antialiased(*a) == -1 and b"semantic_feature" in lib.f3dgs_last_error()


def test_python_surface():
    import inspect

    import diff_gaussian_rasterization as dgr
    from diff_gaussian_rasterization.feature_head import FeatureLift
    from diff_gaussian_rasterization.parallel import ViewBatch

    for n in ("rasterize_gaussians_antialiased", "rasterize_gaussians_backward_antialiased"):
        assert hasattr(dgr._C, n)
    assert dgr.AntialiasedGaussianRasterizer.antialiasing and not dgr.GaussianRasterizer.antialiasing
    assert issubclass(dgr.AntialiasedGaussianRasterizer, dgr.GaussianRasterizer)
    assert inspect.signature(ViewBatch.forward).parameters["antialiasing"].default is False
    assert inspect.signature(FeatureLift.__init__).parameters["antialiasing"].default is False


# ------------------------------------------------------------------------------------------------------------ GPU
def _ptr(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None and t.numel() else 0)


def _forward(sc, cam, aa, C=0, fdtype=torch.float32, opacities=None, mod=1.0, cov_precomp=False, colors_precomp=False,
             seed=7, cov_override=None):
    from diff_gaussian_rasterization import _C

    dev = torch.device("cuda")
    d = scenegen.to_torch(sc, dev)
    e = torch.empty(0, device=dev)
    vm, pm, cp = (torch.tensor(a, device=dev).contiguous() for a in (cam.viewmatrix, cam.projmatrix, cam.campos))
    feats = (torch.randn(sc.P, 1, C, generator=torch.Generator().manual_seed(seed)).to(dev).to(fdtype) if C else e)
    cov = (cov3d_from_scale_rot(_f64(sc.scales), _f64(sc.rotations), mod).float().to(dev) if cov_precomp else e)
    if cov_override is not None:
        cov = cov_override.float().to(dev).contiguous()
    cols = torch.rand(sc.P, 3, generator=torch.Generator().manual_seed(seed + 1)).to(dev) if colors_precomp else e
    shs = e if colors_precomp else d["shs"]
    s_, r_ = (e, e) if cov_precomp else (d["scales"], d["rotations"])
    op = d["opacities"] if opacities is None else opacities
    fn = _C.rasterize_gaussians_antialiased if aa else _C.rasterize_gaussians
    R, color, fmap, depth, radii, geom, binning, img = fn(
        d["bg"], d["means3D"], cols, feats, op, s_, r_, mod, cov, vm, pm, cam.tanfovx, cam.tanfovy,
        cam.image_height, cam.image_width, shs, sc.sh_degree, cp, False, False)
    pl, ranges, n_contrib, final_T, rec = _C.debug_views(geom, binning, img, sc.P, cam.image_width, cam.image_height, R)
    return dict(d=d, R=R, color=color, fmap=fmap, depth=depth, radii=radii, geom=geom, binning=binning, img=img,
                point_list=pl, n_contrib=n_contrib, final_T=final_T, rec=rec, feats=feats, cov=cov, cols=cols, shs=shs,
                scales=s_, rots=r_, vm=vm, pm=pm, cp=cp, mod=mod, op=op)


def _backward(lib, sc, cam, f, entry, feature_geometry=False, half_map=False, camera=False, seed=1234, scale=1.0):
    """One C backward entry on the buffers of forward f -> dict of outputs.  entry: f3dgs_backward_feature_geometry,
    f3dgs_backward_antialiased or f3dgs_backward_accum_antialiased (all read features by dtype code)."""
    dev = torch.device("cuda")
    P, M, C = sc.P, sc.shs.shape[1], (f["feats"].shape[-1] if f["feats"].numel() else 0)
    W, H = cam.image_width, cam.image_height
    gc, gf, gd = (torch.from_numpy(a).to(dev) for a in scenegen.upstream_grads(H, W, C, seed))
    gmap = (gf / scale).half() if half_map else gf
    z = lambda *s: torch.zeros(*s, device=dev)  # noqa: E731
    o = dict(mean2D=z(P, 3), conic=z(P, 4), opacity=z(P), color=z(P, 3), feat=z(P, C), mean3D=z(P, 3), cov3D=z(P, 6),
             sh=z(P, M, 3), scale=z(P, 3), rot=z(P, 4), dz=z(P), camera=z(35))
    sf = f["feats"] if feature_geometry else None
    d = f["d"]
    null = ctypes.c_void_p(0)
    head = [P, sc.sh_degree, M, f["R"], C, _ptr(d["bg"]), W, H, _ptr(d["means3D"]), _ptr(f["shs"]), _ptr(f["cols"]),
            _ptr(sf), F16 if sf is not None and sf.dtype == torch.float16 else F32, _ptr(f["scales"]),
            ctypes.c_float(f["mod"]), _ptr(f["rots"]), _ptr(f["cov"]), _ptr(f["vm"]), _ptr(f["pm"]), _ptr(f["cp"]),
            ctypes.c_float(cam.tanfovx), ctypes.c_float(cam.tanfovy), _ptr(f["radii"]), _ptr(f["geom"]),
            _ptr(f["binning"]), _ptr(f["img"]), _ptr(gc), _ptr(gmap), F16 if half_map else F32,
            ctypes.c_float(scale if half_map else 1.0), _ptr(gd)]
    has_sh, has_sr = f["shs"].numel() > 0, f["scales"].numel() > 0
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    cam_ptr = _ptr(o["camera"]) if camera else null
    if "accum" in entry:
        import diff_gaussian_rasterization as dgr

        scratch = torch.empty(int(dgr._C.backward_scratch_bytes(P)), dtype=torch.uint8, device=dev)
        args = head + [_ptr(scratch), _ptr(o["opacity"]), _ptr(o["color"]) if f["cols"].numel() else null,
                       _ptr(o["feat"]), _ptr(o["mean3D"]), _ptr(o["cov3D"]) if f["cov"].numel() else null,
                       _ptr(o["sh"]) if has_sh else null, _ptr(o["scale"]) if has_sr else null,
                       _ptr(o["rot"]) if has_sr else null, _ptr(o["mean2D"]), null, null, null, 0, stream, cam_ptr]
    else:
        args = head + [_ptr(o["mean2D"]), _ptr(o["conic"]), _ptr(o["opacity"]), _ptr(o["color"]), _ptr(o["feat"]),
                       _ptr(o["mean3D"]), _ptr(o["cov3D"]), _ptr(o["sh"]) if has_sh else null,
                       _ptr(o["scale"]) if has_sr else null, _ptr(o["rot"]) if has_sr else null, _ptr(o["dz"]), 0,
                       stream, cam_ptr]
    if entry == "f3dgs_backward":  # float32 features and map, no dtype codes or map scale
        assert not half_map
        del args[29], args[28], args[12]
    rc = getattr(lib, entry)(*args)
    assert rc == 0, lib.f3dgs_last_error()
    torch.cuda.synchronize()
    return o


def _scenes():
    from test_blend_weights import SCENES

    out = {k: SCENES[k]() for k in ("small", "needles", "layers129", "opaque")}
    sc = scenegen.make_scene(600, 96, 40, 0, sh_degree=3, seed=21)
    cam = scenegen.make_camera(96, 96, np.array([0.0, 0.4, 3.2]), fovx_deg=50.0)
    cam.tanfovy = float(np.float32(cam.tanfovy * 0.7))  # fx != fy
    out["fx!=fy"] = (sc, cam)
    out["inside"] = (sc, scenegen.make_camera(96, 40, np.array([0.1, 0.05, 0.2]), fovx_deg=75.0))
    for deg in range(4):
        s = scenegen.make_scene(400, 96, 64, 0, sh_degree=deg, seed=10 + deg)
        out[f"deg{deg}"] = (s, s.cameras[0])
    return out


@pytest.fixture(scope="module")
def glib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    return L


@pytest.fixture(scope="module")
def scenes():
    return _scenes()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "needles", "layers129", "opaque", "inside", "fx!=fy", "deg3"])
@pytest.mark.parametrize("fdtype", [torch.float32, torch.float16])
def test_render_is_the_default_render_on_effective_opacities(scenes, name, fdtype):
    sc, cam = scenes[name]
    a = _forward(sc, cam, True, C=8, fdtype=fdtype)
    op_eff = a["rec"][:, 7:8].contiguous()
    b = _forward(sc, cam, False, C=8, fdtype=fdtype, opacities=torch.where(a["radii"][:, None] > 0, op_eff,
                                                                           a["d"]["opacities"]))
    for k in ("color", "fmap", "depth", "radii", "final_T", "n_contrib", "point_list"):
        assert torch.equal(a[k], b[k]), (name, k)
    assert a["R"] == b["R"]
    # rec.op against the model, within a few ulp scaled by the conditioning of det0 = a0 c0 - b^2
    vis = (a["radii"] > 0).cpu()
    idx = vis.nonzero().flatten()
    cov = cov3d_from_scale_rot(_f64(sc.scales), _f64(sc.rotations))[idx]
    _, _, op_eff_m, _, _, (a0, b0, c0) = aa_quantities(
        _f64(sc.means3D)[idx], cov, _f64(sc.opacities)[idx], _f64(cam.viewmatrix).reshape(16),
        _f64(cam.projmatrix).reshape(16), _f64(cam.campos), cam.image_width, cam.image_height, cam.tanfovx,
        cam.tanfovy, 0, colors=torch.zeros(len(idx), 3, dtype=torch.float64))
    det0 = a0 * c0 - b0 * b0
    cond = (a0.abs() * c0.abs() + b0 * b0) / det0.abs().clamp_min(1e-300)
    # det0 / det is clamped at 2.5e-5; near the clamp the float32 ratio may land on either side
    cond = torch.where(det0 / ((a0 + 0.3) * (c0 + 0.3) - b0 * b0) < 4 * MIN_RATIO, torch.full_like(cond, 1e30), cond)
    u = 2.0 ** -24
    bar = 64 * u * (1.0 + cond) * op_eff_m
    # a needle's 2-D covariance (eigenvalue ratio > 100 after the dilation) carries float32 errors of the projection
    # that a bar on det0's cancellation does not bound; as parity.tie_aware_compare does, those are not compared here
    a_, c_ = a0 + 0.3, c0 + 0.3
    mid, dd = 0.5 * (a_ + c_), torch.sqrt(0.25 * (a_ - c_) ** 2 + b0 * b0)
    well = (mid + dd) / (mid - dd) <= 100.0
    err = (a["rec"][:, 7].cpu().double()[idx] - op_eff_m).abs()
    ratio = float((err / bar)[well].max()) if bool(well.any()) else 0.0
    print(f"[{name}] op_eff worst |err|/bar = {ratio:.3g}")
    assert ratio <= 1.0
    assert bool((a["rec"][:, 7].cpu()[idx] <= torch.as_tensor(sc.opacities).reshape(-1)[idx]).all())


def _check_against_model(lib, sc, cam, label, entry="f3dgs_backward_antialiased", C=0, feature_geometry=False,
                         half_map=False, camera=True, mod=1.0, cov_precomp=False, colors_precomp=False, cov_override=None):
    """The native AA backward against the model pushed through by autograd from the composite's per-Gaussian gradients
    of the default backward on the effective opacities."""
    kw = dict(C=C, mod=mod, cov_precomp=cov_precomp, colors_precomp=colors_precomp, cov_override=cov_override)
    a = _forward(sc, cam, True, **kw)
    eff = torch.where(a["radii"][:, None] > 0, a["rec"][:, 7:8].contiguous(), a["d"]["opacities"])
    b = _forward(sc, cam, False, opacities=eff, **kw)
    ref = _backward(lib, sc, cam, b, "f3dgs_backward_feature_geometry" if feature_geometry else "f3dgs_backward",
                    feature_geometry=feature_geometry, half_map=half_map, scale=1e-3)
    ours = _backward(lib, sc, cam, a, entry, feature_geometry=feature_geometry, half_map=half_map, camera=camera,
                     scale=1e-3)
    vis = (a["radii"] > 0).cpu()
    idx = vis.nonzero().flatten()
    grads = [ref[k].cpu() for k in ("mean2D", "conic", "opacity", "color", "dz")]
    m = model_gradients(sc, cam, grads, idx, mod=mod, cov=a["cov"].cpu() if cov_precomp else None,
                        colors=a["cols"].cpu() if colors_precomp else None)
    well = m["eig_ratio"] <= 100.0
    k = m["kappa"].clamp_min(1.0)
    worst = 0.0
    # dL/dopacity = rho g, and rho is a function of the 2-D covariance: it is weighted like the others
    pairs = [("opacity", "opacity", True), ("mean3D", "means3D", True)]
    pairs += [("cov3D", "cov3D", True)] if cov_precomp else [("scale", "scales", True), ("rot", "rotations", True)]
    for nk, mk_, through_cov in pairs:
        n = ours[nk].cpu().double().reshape(sc.P, -1)
        r = m[mk_]
        rows = well if through_cov else torch.ones_like(well)
        floor = 1e-6 * float(r[rows].abs().max()) + 1e-12 if bool(rows.any()) else 1e-12
        bar = 1e-4 * (k if through_cov else torch.ones_like(k))[:, None] * r.abs().sum(1, keepdim=True) + floor
        ratio = ((n - r).abs() / bar)[rows]
        worst = max(worst, float(ratio.max()) if ratio.numel() else 0.0)
        assert float(ratio.max() if ratio.numel() else 0.0) <= 1.0, (label, nk, float(ratio.max()))
    if camera:
        t = cgm.terms(sc.means3D, (a["cov"].cpu() if cov_precomp else
                                   cov3d_from_scale_rot(_f64(sc.scales), _f64(sc.rotations), mod)).double(),
                      a["vm"].cpu(), a["pm"].cpu(), a["cp"].cpu(), [ref[x].cpu() for x in ("mean2D", "conic", "color", "dz")],
                      cam.image_width, cam.image_height, cam.tanfovx, cam.tanfovy, sc.sh_degree,
                      shs=None if colors_precomp else sc.shs, colors=a["cols"].cpu() if colors_precomp else None,
                      visible=vis)
        # camera_grad_model's scale of the non-AA terms, plus the AA term's own magnitude (it passes through the conic
        # backward's covariance chain, weighted as the vm_cov share is)
        scale = cgm.camera_scale(t) + (m["camera"] - cgm.camera_vector(t)).abs() * float(k[well].max() if bool(well.any()) else 1.0)
        bar = 1e-5 * scale + 1e-7 * float(cgm.camera_scale(t, needles=False).max())
        ratio = float(((ours["camera"].cpu().double() - m["camera"]).abs() / bar).max())
        worst = max(worst, ratio)
        assert ratio <= 1.0, (label, "camera", ratio)
    print(f"[{label}] visible={len(idx)} needles={int((~well[idx]).sum())} worst |err|/bar = {worst:.3g}")
    return a, ref, ours, m


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "needles", "layers129", "opaque", "inside", "fx!=fy", "deg0", "deg1", "deg2",
                                  "deg3"])
def test_backward_matches_the_model(glib, scenes, name):
    sc, cam = scenes[name]
    _check_against_model(glib, sc, cam, name, mod=1.3 if name == "fx!=fy" else 1.0)


@pytest.mark.gpu
def test_backward_matches_the_model_with_precomputed_covariance_and_colours(glib, scenes):
    sc, cam = scenes["fx!=fy"]
    _check_against_model(glib, sc, cam, "cov3D_precomp", cov_precomp=True)
    _check_against_model(glib, sc, cam, "colors_precomp", colors_precomp=True)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["f3dgs_backward_antialiased", "f3dgs_backward_accum_antialiased"])
def test_degenerate_covariances_give_finite_gradients(glib, scenes, entry):
    """A zero cov3D_precomp and a rank-1 one along the camera's x axis: the undilated 2-D covariance is singular
    (det0 = 0), rho is clamped and constant, so these Gaussians get no rho term, and every output of the view,
    the camera gradient included, stays finite and matches the model (which differentiates through the clamp)."""
    sc, cam = scenes["small"]
    f = _forward(sc, cam, False, cov_precomp=True)
    vis = (f["radii"] > 0).cpu().nonzero().flatten()
    i0, i1 = int(vis[0]), int(vis[1])
    cov = f["cov"].cpu().double().clone()
    cov[i0] = 0.0
    e = torch.tensor(cam.viewmatrix, dtype=torch.float64).reshape(16)[[0, 4, 8]]  # the camera's x axis in the world
    tz = float((torch.tensor(cam.viewmatrix, dtype=torch.float64).reshape(16)[2::4]
                * torch.cat([_f64(sc.means3D)[i1], torch.ones(1, dtype=torch.float64)])).sum())
    s = 2.0 * tz / (cam.image_width / (2 * cam.tanfovx))  # 2 px along x on screen
    E = s * s * torch.outer(e, e)
    cov[i1] = torch.stack([E[0, 0], E[0, 1], E[0, 2], E[1, 1], E[1, 2], E[2, 2]])
    a, ref, ours, m = _check_against_model(glib, sc, cam, "degenerate", entry=entry, cov_precomp=True,
                                           cov_override=cov)
    assert int(a["radii"][i0]) > 0 and int(a["radii"][i1]) > 0
    for k, v in ours.items():
        assert bool(torch.isfinite(v).all()), k
    for i in (i0, i1):
        assert float(m["eig_ratio"][i]) <= 100.0  # compared by _check_against_model, not skipped as a needle
        assert float(a["rec"][i, 7]) == pytest.approx(float(sc.opacities[i, 0]) * math.sqrt(MIN_RATIO), rel=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["accum", "no_camera", "feature_geometry", "feature_geometry_f16_map"])
def test_backward_variants_match_the_model(glib, scenes, variant):
    sc, cam = scenes["small"]
    kw = dict(accum=dict(entry="f3dgs_backward_accum_antialiased"), no_camera=dict(camera=False),
              feature_geometry=dict(C=8, feature_geometry=True),
              feature_geometry_f16_map=dict(C=8, feature_geometry=True, half_map=True))[variant]
    _check_against_model(glib, sc, cam, variant, **kw)


@pytest.mark.gpu
def test_block_view_is_bitwise(glib):
    """On _block_scene (each Gaussian reduced by one atomic onto zero): the composite's outputs equal the default
    backward's on effective opacities, repeated runs are identical, the camera twin changes nothing else, and one view
    accumulated into zeros equals the assigning entry."""
    from test_camera_grad import _block_scene

    sc, cam = _block_scene()
    a = _forward(sc, cam, True, C=8)
    eff = torch.where(a["radii"][:, None] > 0, a["rec"][:, 7:8].contiguous(), a["d"]["opacities"])
    b = _forward(sc, cam, False, C=8, opacities=eff)
    ref = _backward(glib, sc, cam, b, "f3dgs_backward")
    runs = [_backward(glib, sc, cam, a, "f3dgs_backward_antialiased", camera=c) for c in (False, True, True)]
    for k in ("color", "feat", "dz", "mean2D", "conic"):
        assert torch.equal(runs[0][k], ref[k]), k
    for k in ("mean2D", "conic", "opacity", "color", "feat", "mean3D", "cov3D", "sh", "scale", "rot", "dz"):
        assert torch.equal(runs[0][k], runs[1][k]) and torch.equal(runs[1][k], runs[2][k]), k
    assert torch.equal(runs[1]["camera"], runs[2]["camera"]) and bool(runs[1]["camera"].abs().sum() > 0)
    acc = _backward(glib, sc, cam, a, "f3dgs_backward_accum_antialiased", camera=True)
    acc0 = _backward(glib, sc, cam, a, "f3dgs_backward_accum_antialiased", camera=False)
    for k in ("opacity", "feat", "mean3D", "sh", "scale", "rot", "mean2D", "camera"):
        assert torch.equal(acc[k], runs[1][k]), k
        if k != "camera":
            assert torch.equal(acc0[k], acc[k]), k
    # the compensation is not a no-op here: 0.3 px Gaussians lose about half their opacity
    assert bool((a["rec"][:, 7] < 0.8 * a["d"]["opacities"].reshape(-1)).all())


def _settings(sc, cam, dev):
    from diff_gaussian_rasterization import GaussianRasterizationSettings

    return GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))


@pytest.mark.gpu
def test_autograd_and_view_batches(scenes):
    import diff_gaussian_rasterization as dgr
    from diff_gaussian_rasterization import _C
    from diff_gaussian_rasterization.parallel import ViewBatch

    dev = torch.device("cuda")
    sc = scenegen.make_scene(300, 96, 64, 8, sh_degree=2, views=2, seed=5)
    d = scenegen.to_torch(sc, dev)
    names = ("means3D", "scales", "rotations", "opacities", "shs", "semantic_feature")
    params = {k: d[k].clone().requires_grad_() for k in names}
    total = {k: torch.zeros_like(v) for k, v in params.items()}
    seeds = (11, 12)
    for cam, seed in zip(sc.cameras, seeds):
        rs = _settings(sc, cam, dev)
        r = dgr.AntialiasedGaussianRasterizer(rs)
        color, feat, radii, depth = r(means3D=params["means3D"], means2D=torch.zeros_like(params["means3D"]),
                                      opacities=params["opacities"], shs=params["shs"],
                                      semantic_feature=params["semantic_feature"], scales=params["scales"],
                                      rotations=params["rotations"])
        gc, gf, gd = (torch.from_numpy(x).to(dev) for x in scenegen.upstream_grads(cam.image_height, cam.image_width,
                                                                                    sc.C, seed))
        g = torch.autograd.grad((color * gc).sum() + (feat * gf).sum() + (depth * gd).sum(), list(params.values()))
        # the binding, directly
        e = torch.Tensor([])
        out = _C.rasterize_gaussians_antialiased(rs.bg, d["means3D"], e, d["semantic_feature"], d["opacities"],
                                                 d["scales"], d["rotations"], rs.scale_modifier, e, rs.viewmatrix,
                                                 rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width,
                                                 d["shs"], rs.sh_degree, rs.campos, False, False)
        R, c2, f2, d2, radii2, geom, binning, img = out
        assert torch.equal(c2, color.detach()) and torch.equal(radii2, radii)
        bw = _C.rasterize_gaussians_backward_antialiased(
            rs.bg, d["means3D"], radii2, e, d["semantic_feature"], d["scales"], d["rotations"], rs.scale_modifier, e,
            rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, gc, gf, gd, d["shs"], rs.sh_degree, rs.campos, geom,
            R, binning, img, False)
        assert bw[9] is None and len(bw) == 12
        ref = dict(means3D=bw[4], opacities=bw[3], shs=bw[6], scales=bw[7], rotations=bw[8], semantic_feature=bw[2])
        for k, v in zip(names, g):
            assert torch.allclose(v, ref[k].reshape(v.shape), rtol=1e-4, atol=1e-5 * float(ref[k].abs().max()) + 1e-12), k
            total[k] += v
    vb = ViewBatch({k: d[k] for k in names}, densify_stats=False)
    vb.zero_()
    for i, (cam, seed) in enumerate(zip(sc.cameras, seeds)):
        rs = _settings(sc, cam, dev)
        color, feat, radii, depth, ctx = vb.forward(rs, antialiasing=True)
        assert ctx.antialiasing
        gc, gf, gd = (torch.from_numpy(x).to(dev) for x in scenegen.upstream_grads(cam.image_height, cam.image_width,
                                                                                    sc.C, seed))
        vb.backward(ctx, gc, gf, gd, last=(i == 1))
    # a side stream that waits on the last view's event sees the final opacity slice (a sanity check of the ordering)
    side = torch.cuda.Stream()
    side.wait_event(vb._ev)
    with torch.cuda.stream(side):
        seen = vb.grads["opacities"].clone()
    torch.cuda.synchronize()
    for k in names:
        scale = float(total[k].abs().max())
        assert torch.allclose(vb.grads[k], total[k], rtol=1e-4, atol=1e-5 * scale + 1e-12), k
    assert torch.equal(seen, vb.grads["opacities"])


@pytest.mark.gpu
def test_coverage_across_resolutions_end_to_end():
    """The model's coverage prediction (test_model_resolution_consistency) against the rendered 1 - final_T."""
    sc, cam = _isolated(192, 64)
    for k in (1, 2, 4):
        c = _scaled_camera(cam, k)
        f = _forward(sc, c, True)
        aa, integral, _, bar = model_coverage(sc, c, True)
        # each Gaussian sits alone in its 32 x 32 cell (at any of the scales): sum 1 - final_T per cell
        ft = 1.0 - f["final_T"].cpu().double()
        cell = 32 // k
        got = torch.stack([ft[(i // (192 // 32)) * cell:(i // (192 // 32) + 1) * cell,
                              (i % (192 // 32)) * cell:(i % (192 // 32) + 1) * cell].sum() for i in range(sc.P)])
        assert torch.allclose(got, aa, rtol=1e-4, atol=1e-6), (k, got, aa)
        assert bool(((got / integral - 1).abs() <= bar).all()), (k, got / integral)


@pytest.mark.gpu
def test_feature_lift_on_effective_opacities():
    from diff_gaussian_rasterization.feature_head import FeatureLift
    from test_camera_grad import _block_scene

    dev = torch.device("cuda")
    for label, (sc, cam) in (("small", (scenegen.make_config("small"), None)), ("block", _block_scene())):
        cam = cam or sc.cameras[0]
        d = scenegen.to_torch(sc, dev)
        rs = _settings(sc, cam, dev)
        fmap = torch.randn(5, cam.image_height, cam.image_width, generator=torch.Generator().manual_seed(2)).to(dev)
        a = FeatureLift(d["means3D"], d["opacities"], d["scales"], d["rotations"], 5, antialiasing=True)
        a.add(rs, fmap)
        f = _forward(sc, cam, True)
        eff = torch.where(f["radii"][:, None] > 0, f["rec"][:, 7:8].contiguous(), d["opacities"])
        b = FeatureLift(d["means3D"], eff, d["scales"], d["rotations"], 5)
        b.add(rs, fmap)
        torch.cuda.synchronize()
        if label == "block":
            assert torch.equal(a.flat, b.flat)
        else:
            scale = float(b.flat.abs().max())
            assert torch.allclose(a.flat, b.flat, rtol=1e-5, atol=1e-5 * scale), label
