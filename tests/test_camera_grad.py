"""Camera gradients: dL/dviewmatrix, dL/dprojmatrix and dL/dcampos from the backward preprocess (f3dgs_backward_cam and
its twins, rasterize_gaussians_backward_camera, _RasterizeGaussiansCamera, ViewBatch.backward(camera=True)).

CPU: the float64 model of camera_grad_model.py against the CPU oracle's preprocess backward, central differences and the
rigid-motion identities, and the C entries' argument checks.  GPU: the native camera gradient against the model on the composite's own per-Gaussian
gradients, bitwise equality of every other output with the twin entries, determinism, autograd through a pose, view
batches, and an end-to-end pose recovery.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import camera_grad_model as cgm
import scenegen

torch.set_default_dtype(torch.float32)


# ------------------------------------------------------------------------------------------------------------ helpers
def _cov3d(scales, rotations, mod=1.0):
    s = np.asarray(scales, np.float64) * mod
    r, x, y, z = np.asarray(rotations, np.float64).T
    R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                  np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                  np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], 1)
    M = s[:, :, None] * R  # rows of S R
    Sig = np.einsum("pki,pkj->pij", M, M)
    return np.stack([Sig[:, 0, 0], Sig[:, 0, 1], Sig[:, 0, 2], Sig[:, 1, 1], Sig[:, 1, 2], Sig[:, 2, 2]], 1)


def _small_case(seed, deg, P=40, W=64, H=48, inside=False):
    sc = scenegen.make_scene(P, W, H, 0, sh_degree=deg, seed=seed)
    cam = sc.cameras[0]
    if inside:
        cam = scenegen.make_camera(W, H, np.array([0.1, 0.05, 0.2]))
    rng = np.random.default_rng(seed + 100)
    grads = (rng.standard_normal((P, 3)), rng.standard_normal((P, 4)), rng.standard_normal((P, 3)),
             rng.standard_normal((P,)))
    return sc, cam, grads, _cov3d(sc.scales, sc.rotations)


def _visible_unclamped(sc, cam, margin=0.9):
    vm = torch.tensor(cam.viewmatrix, dtype=torch.float64).reshape(16)
    p = torch.cat([torch.tensor(sc.means3D, dtype=torch.float64), torch.ones(sc.P, 1, dtype=torch.float64)], 1)
    t = [(vm[r::4] * p).sum(1) for r in range(3)]
    return ((t[2] > 0.2) & ((t[0] / t[2]).abs() < margin * 1.3 * cam.tanfovx)
            & ((t[1] / t[2]).abs() < margin * 1.3 * cam.tanfovy))


def _model_loss(sc, cam, grads, cov, deg, vm, pm, cp, visible, colors=None, means=None, cv=None):
    f = lambda a: torch.as_tensor(a, dtype=torch.float64)  # noqa: E731
    idx = visible.nonzero().flatten()
    means = f(sc.means3D)[idx] if means is None else means
    cv = f(cov)[idx] if cv is None else cv
    q = cgm.screen_quantities(means, cv, vm, pm, cp, cam.image_width, cam.image_height, cam.tanfovx, cam.tanfovy,
                              deg, shs=None if colors is not None else f(sc.shs)[idx],
                              colors=None if colors is None else f(colors)[idx])
    g = [f(x)[idx] for x in grads]
    return cgm.contract(q, g[0], g[1], g[2], g[3])


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("case", ["deg0", "deg1", "deg2", "deg3", "cov3D_precomp", "colors_precomp", "inside"])
def test_model_matches_the_oracle_preprocess_backward(case):
    """Pins the model to the validated chain: fed the CPU oracle's per-Gaussian intermediates (dL_dmean2D, dL_dconic,
    dL_dcolor, dL_dz of oracle.backward) and the forward's float32 cov3D, the model's dL/dmeans3D and dL/dcov3D are the
    oracle's (oracle_preprocess_backward, the reference's preprocess backward restated in C).  That ties its forward --
    the J and W layout, the 1e-7 conventions, the conic, the SH direction and the clamps -- to the reference's, which
    the camera gradient is then the other contraction of.  Float32 bar per Gaussian, scaled by the conditioning of its
    2-D covariance; conics with an eigenvalue ratio above 100 are skipped, as parity does for the covariance path."""
    import oracle

    deg = int(case[3]) if case.startswith("deg") else 3
    seed = {"cov3D_precomp": 11, "colors_precomp": 12, "inside": 13}.get(case, 5 + deg)
    sc = scenegen.make_scene(300 if case == "inside" else 80, 64, 48, 0, sh_degree=deg, seed=seed)
    cam = scenegen.make_camera(64, 48, np.array([0.1, 0.05, 0.2])) if case == "inside" else sc.cameras[0]
    rng = np.random.default_rng(seed)
    cols = rng.uniform(0, 1, (sc.P, 3)).astype(np.float32) if case == "colors_precomp" else None
    cov = _cov3d(sc.scales, sc.rotations).astype(np.float32) if case == "cov3D_precomp" else None
    fwd = oracle.forward(sc, cam, colors_precomp=cols, cov3D_precomp=cov)
    gc, gf, gd = scenegen.upstream_grads(cam.image_height, cam.image_width, 0, seed)
    g = oracle.backward(sc, cam, fwd, gc, gf, gd, colors_precomp=cols, cov3D_precomp=cov)
    vis = torch.from_numpy(fwd["radii"] > 0)
    t = cgm.terms(sc.means3D, fwd["cov3D"], cam.viewmatrix, cam.projmatrix, cam.campos,
                  (g["means2D"], g["conic"], g["colors"], g["dz"]), cam.image_width, cam.image_height, cam.tanfovx,
                  cam.tanfovy, deg, shs=None if cols is not None else sc.shs, colors=cols, visible=vis)
    well = vis & (t["eig_ratio"] <= 100)
    assert int(well.sum()) >= 20
    k = t["kappa"].clamp_min(1.0)[:, None]
    worst = {}
    for key, ours in (("means3D", g["means3D"]), ("cov3D", g["cov3D"])):
        m, o = t[key][well], torch.from_numpy(ours).double()[well]
        bar = 1e-4 * k[well] * m.abs().amax(1, keepdim=True) + 1e-6 * float(m.abs().max())
        worst[key] = float(((m - o).abs() / bar).max())
        assert bool((o[~well[well]] == 0).all())
    print(f"[{case}] visible={int(vis.sum())} compared={int(well.sum())} worst |err|/bar: {worst}")
    assert max(worst.values()) <= 1.0, worst
    assert bool((torch.from_numpy(g["means3D"])[~vis] == 0).all())


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_model_camera_gradient_matches_central_differences(deg):
    sc, cam, grads, cov = _small_case(deg + 1, deg)
    vis = _visible_unclamped(sc, cam)
    assert int(vis.sum()) > 5
    t = cgm.terms(sc.means3D, cov, cam.viewmatrix, cam.projmatrix, cam.campos, grads, cam.image_width,
                  cam.image_height, cam.tanfovx, cam.tanfovy, deg, shs=sc.shs, visible=vis)
    g = cgm.camera_vector(t)
    base = [torch.tensor(a, dtype=torch.float64).reshape(-1) for a in (cam.viewmatrix, cam.projmatrix, cam.campos)]
    fd = torch.zeros(35, dtype=torch.float64)
    h = 1e-6
    for j in range(35):
        which, k = (0, j) if j < 16 else ((1, j - 16) if j < 32 else (2, j - 32))
        vals = []
        for s in (1, -1):
            cam_t = [b.clone() for b in base]
            cam_t[which][k] += s * h
            vals.append(float(_model_loss(sc, cam, grads, cov, deg, *cam_t, vis)))
        fd[j] = (vals[0] - vals[1]) / (2 * h)
    scale = cgm.camera_scale(t)
    err = (g - fd).abs()
    assert bool((err <= 1e-6 * scale + 1e-6).all()), (err / (scale + 1e-12)).max()
    for j in (3, 7, 11, 15, 16 + 2, 16 + 6, 16 + 10, 16 + 14):  # entries the forward never reads
        assert g[j] == 0
    if deg == 0:
        assert bool((g[32:] == 0).all())


def _rigid_residuals(sc, cam, grads, cov, deg, colors=None, with_rotation=False):
    """d/d(delta, omega) of the loss when the world and the camera move together; zero if the gradients are right."""
    vis = torch.as_tensor(_visible_unclamped(sc, cam, margin=10.0))
    t = cgm.terms(sc.means3D, cov, cam.viewmatrix, cam.projmatrix, cam.campos, grads, cam.image_width,
                  cam.image_height, cam.tanfovx, cam.tanfovy, deg, shs=None if colors is not None else sc.shs,
                  colors=colors, visible=vis)
    vm = torch.tensor(cam.viewmatrix, dtype=torch.float64).reshape(16)
    pm = torch.tensor(cam.projmatrix, dtype=torch.float64).reshape(16)
    cp = torch.tensor(cam.campos, dtype=torch.float64)
    gvm, gpm, gcp = t["vm"].sum(0), t["pm"].sum(0), t["campos"].sum(0)
    out, scale = [], []
    for k in range(3):  # translation: sum_i dL/dp_i[k] - sum_r dL/dvm[12+r] vm[4k+r] - ... + dL/dcampos[k]
        terms = [t["means3D"][:, k].sum(), -sum(gvm[12 + r] * vm[4 * k + r] for r in range(4)),
                 -sum(gpm[12 + r] * pm[4 * k + r] for r in range(4)), gcp[k]]
        out.append(sum(terms))
        scale.append(t["means3D"][:, k].abs().sum() + sum(abs(x) for x in terms[1:]))
    if with_rotation:
        pts = torch.tensor(sc.means3D, dtype=torch.float64)
        cv = torch.as_tensor(cov, dtype=torch.float64)
        V = torch.stack([torch.stack([cv[:, 0], cv[:, 1], cv[:, 2]], 1), torch.stack([cv[:, 1], cv[:, 3], cv[:, 4]], 1),
                         torch.stack([cv[:, 2], cv[:, 4], cv[:, 5]], 1)], 1)
        for j in range(3):
            K = torch.zeros(3, 3, dtype=torch.float64)
            a, b = [(1, 2), (2, 0), (0, 1)][j]
            K[b, a], K[a, b] = 1.0, -1.0  # hat(e_j)
            dp = pts @ K.t()
            dV = K @ V + V @ K.t()
            dcv = torch.stack([dV[:, 0, 0], dV[:, 0, 1], dV[:, 0, 2], dV[:, 1, 1], dV[:, 1, 2], dV[:, 2, 2]], 1)
            dG = torch.zeros(4, 4, dtype=torch.float64)
            dG[:3, :3] = K.t()
            dvm = -(dG @ vm.reshape(4, 4)).reshape(16)
            dpm = -(dG @ pm.reshape(4, 4)).reshape(16)
            dcp = K @ cp
            terms = [(t["means3D"] * dp).sum(), (t["cov3D"] * dcv).sum(), (gvm * dvm).sum(), (gpm * dpm).sum(),
                     (gcp * dcp).sum()]
            out.append(sum(terms))
            scale.append((t["means3D"] * dp).abs().sum() + (t["cov3D"] * dcv).abs().sum() + (gvm * dvm).abs().sum()
                         + (gpm * dpm).abs().sum() + (gcp * dcp).abs().sum())
    return torch.stack(out), torch.stack(scale)


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("deg", [0, 3])
def test_model_satisfies_the_translation_identity(seed, deg):
    sc, cam, grads, cov = _small_case(seed, deg)
    res, scale = _rigid_residuals(sc, cam, grads, cov, deg)
    assert bool((res.abs() <= 1e-9 * scale).all()), (res, scale)


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("colors", [False, True])
def test_model_satisfies_the_rotation_identities(seed, colors):
    """Rotations move cov3D_precomp with the points; the SH colour is not rotation-invariant, so colours are given or
    SH degree is 0."""
    sc, cam, grads, cov = _small_case(seed, 0)
    col = np.random.default_rng(seed).uniform(0, 1, (sc.P, 3)) if colors else None
    res, scale = _rigid_residuals(sc, cam, grads, cov, 0, colors=col, with_rotation=True)
    assert res.numel() == 6
    assert bool((res.abs() <= 1e-9 * scale).all()), (res, scale)


def test_model_inside_camera_translation_identity():
    sc, cam, grads, cov = _small_case(7, 3, inside=True)
    res, scale = _rigid_residuals(sc, cam, grads, cov, 3)
    assert bool((res.abs() <= 1e-9 * scale).all()), (res, scale)


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    return L


def _backward_args(P, fake, C=4):
    """Arguments of f3dgs_backward with distinct fake device addresses (the checks below fail before any is used)."""
    f = ctypes.c_float
    p = lambda i: ctypes.c_void_p(fake + i * (1 << 20))  # noqa: E731
    null = ctypes.c_void_p(0)
    return [P, 0, 1, 10, C, p(0), 64, 64, p(1), p(2), null, null, p(3), f(1.0), p(4), null, p(5), p(6), p(7), f(0.5),
            f(0.5), p(8), p(9), p(10), p(11), p(12), p(13), p(14), p(15), p(16), p(17), p(18), p(19), p(20), p(21),
            p(22), p(23), p(24), p(25), 0, null]


def test_cam_entries_reject_null_or_overlapping_camera_gradient(lib):
    fake = 1 << 40
    args = _backward_args(5, fake)
    null = ctypes.c_void_p(0)
    assert lib.f3dgs_backward_cam(*args, null) == -1
    assert lib.f3dgs_last_error() == b"f3dgs_backward_cam: NULL dL_dcamera"
    for i in (15, 16, 17, 19, 20, 21, 23, 24, 25):  # dL_dmean2D, dL_dconic, .. dL_dz (each output of the call)
        inside = ctypes.c_void_p(fake + i * (1 << 20) + 8)
        assert lib.f3dgs_backward_cam(*args, inside) == -1, i
        assert b"dL_dcamera overlaps another output" in lib.f3dgs_last_error(), i
    assert lib.f3dgs_backward_cam(*_backward_args(0, fake), ctypes.c_void_p(fake + 15 * (1 << 20))) == 0  # P == 0

    f16 = args[:26] + [ctypes.c_float(1.0)] + args[26:]
    assert lib.f3dgs_backward_cam_f16(*f16, null) == -1
    assert lib.f3dgs_last_error() == b"f3dgs_backward_cam_f16: NULL dL_dcamera"
    assert lib.f3dgs_backward_cam_f16(*f16, ctypes.c_void_p(fake + 20 * (1 << 20))) == -1
    assert b"overlaps" in lib.f3dgs_last_error()


def test_accum_cam_entries_reject_null_or_overlapping_camera_gradient(lib):
    fake = 1 << 40
    p = lambda i: ctypes.c_void_p(fake + i * (1 << 20))  # noqa: E731
    f = ctypes.c_float
    null = ctypes.c_void_p(0)
    args = [5, 0, 1, 10, 4, p(0), 64, 64, p(1), p(2), null, p(3), f(1.0), p(4), null, p(5), p(6), p(7), f(0.5),
            f(0.5), p(8), p(9), p(10), p(11), p(12), p(13), p(14), p(30), p(15), null, p(16), p(17), null, p(18),
            p(19), p(20), p(21), p(22), p(23), null, 0, null]
    assert lib.f3dgs_backward_accum_cam(*args, null) == -1
    assert lib.f3dgs_last_error() == b"f3dgs_backward_accum_cam: NULL dL_dcamera"
    for i in (30, 15, 16, 17, 18, 19, 20, 21, 22, 23):  # scratch, then every accumulated output
        assert lib.f3dgs_backward_accum_cam(*args, ctypes.c_void_p(fake + i * (1 << 20) + 4)) == -1, i
        assert b"dL_dcamera overlaps another output" in lib.f3dgs_last_error(), i
    f16 = args[:26] + [f(1.0)] + args[26:]
    assert lib.f3dgs_backward_accum_cam_f16(*f16, null) == -1
    assert lib.f3dgs_last_error() == b"f3dgs_backward_accum_cam_f16: NULL dL_dcamera"


def test_se3_exp_is_a_rigid_transform_with_the_right_derivative():
    from diff_gaussian_rasterization.camera import se3_exp

    xi = torch.tensor([0.1, -0.2, 0.3, 0.2, -0.1, 0.25], dtype=torch.float64)
    T = se3_exp(xi)
    R = T[:3, :3]
    assert torch.allclose(R @ R.t(), torch.eye(3, dtype=torch.float64), atol=1e-12)
    assert torch.allclose(torch.linalg.det(R), torch.tensor(1.0, dtype=torch.float64))
    assert torch.allclose(T, torch.linalg.matrix_exp(_twist(xi)), atol=1e-12)
    z = torch.zeros(6, dtype=torch.float64, requires_grad=True)
    J = torch.autograd.functional.jacobian(se3_exp, z)
    for j in range(6):
        e = torch.zeros(6, dtype=torch.float64)
        e[j] = 1.0
        assert torch.allclose(J[..., j], _twist(e), atol=1e-12)


def _twist(xi):
    M = torch.zeros(4, 4, dtype=torch.float64)
    a, b, c = xi[3:6]
    M[:3, :3] = torch.tensor([[0, -c, b], [c, 0, -a], [-b, a, 0]], dtype=torch.float64)
    M[:3, 3] = xi[:3]
    return M


def test_settings_from_w2c_matches_the_reference_camera():
    """viewmatrix, projmatrix and campos bitwise as the reference Camera builds them from the same float32 w2c."""
    from diff_gaussian_rasterization.camera import settings_from_w2c

    cam = scenegen.make_camera(64, 48, np.array([1.0, 0.5, 3.0]))
    w2c = torch.tensor(cam.viewmatrix).t().contiguous()
    rs = settings_from_w2c(w2c, cam.tanfovx, cam.tanfovy, 48, 64, torch.zeros(3))
    # the reference: world_view_transform = w2c^T, full_proj = bmm(world_view, P^T), centre = inverse()[3, :3]
    znear, zfar = 0.01, 100.0
    top, right = cam.tanfovy * znear, cam.tanfovx * znear
    P = torch.zeros(4, 4)
    P[0, 0] = 2.0 * znear / (2 * right)
    P[1, 1] = 2.0 * znear / (2 * top)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    wv = w2c.transpose(0, 1)
    assert torch.equal(rs.viewmatrix, wv)
    assert torch.equal(rs.projmatrix, wv.unsqueeze(0).bmm(P.transpose(0, 1).unsqueeze(0)).squeeze(0))
    assert torch.equal(rs.campos, wv.inverse()[3, :3])
    assert torch.allclose(rs.campos, torch.tensor(cam.campos), atol=1e-5)
    assert torch.allclose(rs.projmatrix, torch.tensor(cam.projmatrix), atol=1e-5)


# ------------------------------------------------------------------------------------------------------------ GPU
def _native(lib, sc, cam, entry="f3dgs_backward_cam", mod=1.0, feature_dtype=None, C=0, seed=1234, cov_precomp=False,
            colors_precomp=False):
    """Forward through the binding, then the C entry `entry` through ctypes on torch memory -> dict of outputs."""
    from diff_gaussian_rasterization import _C

    dev = torch.device("cuda")
    d = scenegen.to_torch(sc, dev)
    P, M = sc.P, sc.shs.shape[1]
    W, H = cam.image_width, cam.image_height
    vm, pm, cp = (torch.tensor(a, device=dev).contiguous() for a in (cam.viewmatrix, cam.projmatrix, cam.campos))
    feats = torch.randn(P, 1, C, generator=torch.Generator().manual_seed(seed)).to(dev) if C else torch.empty(0, device=dev)
    if feature_dtype is not None and C:
        feats = feats.to(feature_dtype)
    e = torch.empty(0, device=dev)
    cov = torch.tensor(_cov3d(sc.scales, sc.rotations, mod), dtype=torch.float32, device=dev) if cov_precomp else e
    cols = torch.rand(P, 3, generator=torch.Generator().manual_seed(seed + 1)).to(dev) if colors_precomp else e
    shs = e if colors_precomp else d["shs"]
    sc_, rot_ = (e, e) if cov_precomp else (d["scales"], d["rotations"])
    R, color, fmap, depth, radii, geom, binning, img = _C.rasterize_gaussians(
        d["bg"], d["means3D"], cols, feats, d["opacities"], sc_, rot_, mod, cov, vm, pm, cam.tanfovx, cam.tanfovy, H, W,
        shs, sc.sh_degree, cp, False, False)
    gc, gf, gd = (torch.from_numpy(a).to(dev) for a in scenegen.upstream_grads(H, W, C, seed))
    out = dict(R=R, radii=radii, geom=geom, feats=feats, cov=cov, cols=cols, vm=vm, pm=pm, cp=cp,
               mean2D=torch.zeros(P, 3, device=dev), conic=torch.zeros(P, 4, device=dev),
               opacity=torch.zeros(P, device=dev), color=torch.zeros(P, 3, device=dev),
               feat=torch.zeros(P, C, device=dev), mean3D=torch.zeros(P, 3, device=dev),
               cov3D=torch.zeros(P, 6, device=dev), sh=torch.zeros(P, M, 3, device=dev),
               scale=torch.zeros(P, 3, device=dev), rot=torch.zeros(P, 4, device=dev), dz=torch.zeros(P, device=dev),
               camera=torch.zeros(35, device=dev))
    ptr = lambda t: ctypes.c_void_p(t.data_ptr() if t.numel() else 0)  # noqa: E731
    half = entry.endswith("_f16")
    gfm = gf.half() if half else gf
    fn = getattr(lib, entry)
    args = [P, sc.sh_degree, M, R, C, ptr(d["bg"]), W, H, ptr(d["means3D"]), ptr(shs), ptr(cols), ptr(e), ptr(sc_),
            ctypes.c_float(mod), ptr(rot_), ptr(cov), ptr(vm), ptr(pm), ptr(cp), ctypes.c_float(cam.tanfovx),
            ctypes.c_float(cam.tanfovy), ptr(radii), ptr(geom), ptr(binning), ptr(img), ptr(gc), ptr(gfm)]
    if half:
        args.append(ctypes.c_float(1.0))
    args += [ptr(gd), ptr(out["mean2D"]), ptr(out["conic"]), ptr(out["opacity"]), ptr(out["color"]), ptr(out["feat"]),
             ptr(out["mean3D"]), ptr(out["cov3D"]), ptr(out["sh"]) if M and not colors_precomp else ctypes.c_void_p(0),
             ptr(out["scale"]) if not cov_precomp else ctypes.c_void_p(0),
             ptr(out["rot"]) if not cov_precomp else ctypes.c_void_p(0), ptr(out["dz"]), 0,
             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)]
    if "_cam" in entry:
        args.append(ptr(out["camera"]))
    rc = fn(*args)
    assert rc == 0, lib.f3dgs_last_error()
    torch.cuda.synchronize()
    return out


def _model_check(lib, sc, cam, label, **kw):
    o = _native(lib, sc, cam, **kw)
    P = sc.P
    from test_cabi_gpu import Layout

    L = Layout()
    assert lib.f3dgs_get_layout(P, cam.image_width, cam.image_height, o["R"], ctypes.byref(L)) == 0
    if kw.get("cov_precomp"):
        cov = o["cov"].cpu()
    else:  # the forward's own float32 covariance, as the backward reads it
        cov = o["geom"][L.geom_cov3d:L.geom_cov3d + P * 24].view(torch.float32).view(P, 6).cpu()
    vis = (o["radii"] > 0).cpu()
    t = cgm.terms(sc.means3D, cov, o["vm"].cpu(), o["pm"].cpu(), o["cp"].cpu(),
                  [o[k].cpu() for k in ("mean2D", "conic", "color", "dz")], cam.image_width, cam.image_height,
                  cam.tanfovx, cam.tanfovy, sc.sh_degree, shs=None if kw.get("colors_precomp") else sc.shs,
                  colors=o["cols"].cpu() if kw.get("colors_precomp") else None, visible=vis)
    ref, scale = cgm.camera_vector(t), cgm.camera_scale(t)
    ours = o["camera"].cpu().double()
    bar = 1e-5 * scale + 1e-7 * float(cgm.camera_scale(t, needles=False).max())  # floor: the well-conditioned scale
    ratio = float(((ours - ref).abs() / bar).max())
    n_ill = int((t["eig_ratio"] > 100).sum())
    print(f"[{label}] visible={int(vis.sum())} needles (eigenvalue ratio > 100) = {n_ill} worst |err|/bar = {ratio:.3g}")
    assert ratio <= 1.0, (label, ours, ref)
    for j in (3, 7, 11, 15, 18, 22, 26, 30):
        assert ours[j] == 0
    return o, t


@pytest.fixture(scope="module")
def glib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    return L


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "needles", "layers129", "opaque"])
def test_native_camera_gradient_matches_the_model_on_blend_weight_views(glib, name):
    from test_blend_weights import SCENES

    sc, cam = SCENES[name]()
    _model_check(glib, sc, cam, name)


@pytest.mark.gpu
@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_native_camera_gradient_matches_the_model_per_sh_degree(glib, deg):
    sc = scenegen.make_scene(400, 96, 64, 0, sh_degree=deg, seed=10 + deg)
    _model_check(glib, sc, sc.cameras[0], f"deg{deg}")


@pytest.mark.gpu
def test_native_camera_gradient_inside_the_scene_with_fx_ne_fy_and_scale_modifier(glib):
    sc = scenegen.make_scene(600, 96, 40, 0, sh_degree=3, seed=21)
    cam = scenegen.make_camera(96, 40, np.array([0.1, 0.05, 0.2]), fovx_deg=75.0)
    _model_check(glib, sc, cam, "inside")
    cam2 = scenegen.make_camera(96, 96, np.array([0.0, 0.4, 3.2]), fovx_deg=50.0)
    cam2.tanfovy = float(np.float32(cam2.tanfovy * 0.7))  # fx != fy
    _model_check(glib, sc, cam2, "fx!=fy mod=1.3", mod=1.3)
    _model_check(glib, sc, cam2, "cov/colors precomp", cov_precomp=True, colors_precomp=True)


def _block_scene(W=64, H=48, C=8, deg=3, seed=0):
    """Two small, faint Gaussians in the middle of every 8x4 pixel block, one in front of the other: each blends into
    its own block only (its alpha is below 1/255 on every pixel outside it), so the backward composite reduces each of
    its per-Gaussian gradients with ONE red.global.add onto zero.  Those intermediates (dL_dmean2D, dL_dconic,
    dL_dcolor, dL_dz, dL_dopacity, dL_dsemantic_feature) then do not depend on the order of the float atomics, and two
    backwards of this view give bitwise-equal intermediates, as a run-to-run check needs."""
    cam = scenegen.make_camera(W, H, np.array([0.3, 0.2, 4.0]))
    nb = (W // 8) * (H // 4)
    sc = scenegen.make_scene(2 * nb, W, H, C, sh_degree=deg, seed=seed)
    rng = np.random.default_rng(seed)
    by, bx = np.divmod(np.arange(nb), W // 8)
    px = np.concatenate([8 * bx + 3.5 - 1.0, 8 * bx + 3.5 + 1.0])
    py = np.concatenate([4 * by + 1.5, 4 * by + 1.5])
    z = np.concatenate([np.full(nb, 3.8), np.full(nb, 4.1)]) + rng.uniform(-0.05, 0.05, 2 * nb)
    vx = ((2 * px + 1) / W - 1) * cam.tanfovx * z
    vy = ((2 * py + 1) / H - 1) * cam.tanfovy * z
    view = np.stack([vx, vy, z, np.ones_like(z)], 1)
    world = view @ np.linalg.inv(cam.viewmatrix.astype(np.float64))
    focal = W / (2 * cam.tanfovx)
    sc.means3D = world[:, :3].astype(np.float32)
    sc.scales = np.repeat((0.3 * z / focal)[:, None], 3, 1).astype(np.float32)  # 0.3 px: 2-D variance 0.39 px^2
    sc.rotations = np.tile(np.array([1.0, 0.0, 0.0, 0.0], np.float32), (2 * nb, 1))
    sc.opacities = rng.uniform(0.05, 0.12, (2 * nb, 1)).astype(np.float32)
    sc.cameras = [cam]
    return sc, cam


MID = ("mean2D", "conic", "color", "dz")  # the composite's per-Gaussian intermediates the preprocess reads


@pytest.mark.gpu
@pytest.mark.parametrize("pair", [("f3dgs_backward", "f3dgs_backward_cam"),
                                  ("f3dgs_backward_f16", "f3dgs_backward_cam_f16")])
def test_cam_entries_leave_every_other_output_bitwise_unchanged_and_are_deterministic(glib, pair):
    """On a view whose composite intermediates come back bitwise equal (_block_scene): every output of the _cam entry
    is bitwise its twin's, and two _cam calls give bitwise-equal camera gradients.  On an ordinary view, whose
    composite reduces with unordered float atomics, the outputs agree within rounding."""
    sc, cam = _block_scene()
    runs = [_native(glib, sc, cam, entry=e, C=8) for e in (pair[0], pair[1], pair[1])]
    for k in MID:
        assert torch.equal(runs[0][k], runs[1][k]) and torch.equal(runs[1][k], runs[2][k]), k
    for k in MID + ("opacity", "feat", "mean3D", "cov3D", "sh", "scale", "rot"):
        assert torch.equal(runs[0][k], runs[1][k]) and torch.equal(runs[0][k], runs[2][k]), k
    assert torch.equal(runs[1]["camera"], runs[2]["camera"])
    assert bool((runs[0]["camera"] == 0).all()) and bool(runs[1]["camera"].abs().sum() > 0)
    sc, cam = scenegen.make_config("small"), None
    cam = sc.cameras[0]
    a, b = (_native(glib, sc, cam, entry=e, C=8) for e in pair)
    for k in MID + ("opacity", "feat", "mean3D", "cov3D", "sh", "scale", "rot"):
        scale = float(a[k].abs().max()) if a[k].numel() else 0.0
        assert torch.allclose(a[k], b[k], rtol=1e-4, atol=1e-5 * scale + 1e-12), k


@pytest.mark.gpu
def test_float16_features_give_the_float32_camera_gradient(glib):
    """The feature map does not feed the geometry: with float16 features and a float16 map gradient the intermediates,
    and so the camera gradient, are bitwise those of float32 features."""
    sc, cam = _block_scene()
    a = _native(glib, sc, cam, entry="f3dgs_backward_cam", C=8)
    b = _native(glib, sc, cam, entry="f3dgs_backward_cam_f16", C=8, feature_dtype=torch.float16)
    for k in MID:
        assert torch.equal(a[k], b[k]), k
    assert torch.equal(a["camera"], b["camera"])


@pytest.mark.gpu
def test_translation_identity_on_native_gradients(glib):
    sc = scenegen.make_scene(500, 96, 64, 0, sh_degree=3, seed=31)
    cam = sc.cameras[0]
    o = _native(glib, sc, cam)
    g = o["camera"].cpu().double()
    vm, pm = o["vm"].cpu().double().reshape(16), o["pm"].cpu().double().reshape(16)
    gm = o["mean3D"].cpu().double()
    for k in range(3):
        terms = torch.stack([gm[:, k].sum(), -sum(g[12 + r] * vm[4 * k + r] for r in range(4)),
                             -sum(g[16 + 12 + r] * pm[4 * k + r] for r in range(4)), g[32 + k]])
        scale = gm[:, k].abs().sum() + terms[1:].abs().sum()
        assert abs(float(terms.sum())) <= 1e-5 * float(scale) + 1e-7, (k, terms)


@pytest.mark.gpu
def test_autograd_through_a_pose_matches_the_explicit_chain(glib):
    """w2c.grad through settings_from_w2c and _RasterizeGaussiansCamera is bitwise the binding's camera gradient pulled
    back through settings_from_w2c; without a camera tensor requiring grad the call is _RasterizeGaussians, with every
    output and gradient bitwise the binding's rasterize_gaussians_backward.  On _block_scene, so that separate
    backwards give bitwise-equal intermediates."""
    from diff_gaussian_rasterization import GaussianRasterizer, _RasterizeGaussians, _RasterizeGaussiansCamera, _C
    from diff_gaussian_rasterization.camera import settings_from_w2c

    dev = torch.device("cuda")
    sc, cam = _block_scene()
    W, H = cam.image_width, cam.image_height
    gc, gf, gd = (torch.from_numpy(a).to(dev) for a in scenegen.upstream_grads(H, W, sc.features.shape[-1]))
    e = torch.Tensor([])

    def render(d, rs):
        m2 = torch.zeros_like(d["means3D"], requires_grad=True)
        out = GaussianRasterizer(rs)(means3D=d["means3D"], means2D=m2, opacities=d["opacities"], shs=d["shs"],
                                     semantic_feature=d["semantic_feature"], scales=d["scales"],
                                     rotations=d["rotations"])
        return out, m2

    def native(d, rs, fn):
        D = {k: v.detach() for k, v in d.items()}
        R, color, fmap, depth, rad, geom, binning, img = _C.rasterize_gaussians(
            rs.bg, D["means3D"], e, D["semantic_feature"], D["opacities"], D["scales"], D["rotations"], 1.0, e,
            rs.viewmatrix.detach(), rs.projmatrix.detach(), rs.tanfovx, rs.tanfovy, H, W, D["shs"], rs.sh_degree,
            rs.campos.detach(), False, False)
        return (color, fmap, depth), fn(rs.bg, D["means3D"], rad, e, D["semantic_feature"], D["scales"],
                                        D["rotations"], 1.0, e, rs.viewmatrix.detach(), rs.projmatrix.detach(),
                                        rs.tanfovx, rs.tanfovy, gc, gf, gd, D["shs"], rs.sh_degree,
                                        rs.campos.detach(), geom, R, binning, img, False)

    d = scenegen.to_torch(sc, dev, requires_grad=True)
    w2c = torch.tensor(cam.viewmatrix, device=dev).t().contiguous().requires_grad_()
    rs = settings_from_w2c(w2c, cam.tanfovx, cam.tanfovy, H, W, d["bg"], sh_degree=sc.sh_degree)
    (color, fmap, radii, depth), _ = render(d, rs)
    assert type(color.grad_fn).__name__.startswith(_RasterizeGaussiansCamera.__name__)
    ((color * gc).sum() + (fmap * gf).sum() + (depth * gd).sum()).backward()
    _, grads = native(d, rs, _C.rasterize_gaussians_backward_camera)
    w2 = w2c.detach().clone().requires_grad_()
    rs2 = settings_from_w2c(w2, cam.tanfovx, cam.tanfovy, H, W, d["bg"], sh_degree=sc.sh_degree)
    torch.autograd.backward([rs2.viewmatrix, rs2.projmatrix, rs2.campos], [grads[9], grads[10], grads[11]])
    assert torch.equal(w2c.grad, w2.grad), (w2c.grad, w2.grad)
    assert bool(w2c.grad.abs().sum() > 0)
    for k, g in zip(("means3D", "shs", "opacities", "scales", "rotations"), (grads[4], grads[6], grads[3], grads[7],
                                                                               grads[8])):
        assert torch.equal(d[k].grad, g), k

    # no camera tensor requiring grad: _RasterizeGaussians, bitwise the binding's outputs and gradients
    d2 = scenegen.to_torch(sc, dev, requires_grad=True)
    rsd = rs._replace(viewmatrix=rs.viewmatrix.detach(), projmatrix=rs.projmatrix.detach(), campos=rs.campos.detach())
    (c2, f2, r2, z2), m2 = render(d2, rsd)
    assert type(c2.grad_fn).__name__ == _RasterizeGaussians.__name__ + "Backward"
    ((c2 * gc).sum() + (f2 * gf).sum() + (z2 * gd).sum()).backward()
    images, ref = native(d2, rsd, _C.rasterize_gaussians_backward)
    for x, y in zip((c2, f2, z2), images):
        assert torch.equal(x.detach(), y)
    for k, g in zip(("means3D", "semantic_feature", "shs", "opacities", "scales", "rotations"),
                    (ref[4], ref[2], ref[6], ref[3], ref[7], ref[8])):
        assert torch.equal(d2[k].grad, g), k
    assert torch.equal(m2.grad, ref[0])


@pytest.mark.gpu
def test_view_batch_camera_gradients(glib):
    """ViewBatch.backward(camera=True) on three views of _block_scene (one camera, three upstream gradients): the flat
    buffer and the densification statistics are bitwise those of camera=False, and each view's CameraGrad is bitwise
    the binding's rasterize_gaussians_backward_camera for that view."""
    from diff_gaussian_rasterization import GaussianRasterizationSettings, _C
    from diff_gaussian_rasterization.parallel import ViewBatch

    dev = torch.device("cuda")
    sc, cam = _block_scene()
    d = scenegen.to_torch(sc, dev)
    params = {k: d[k] for k in ("means3D", "scales", "rotations", "opacities", "shs", "semantic_feature")}
    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))
    ups = [tuple(torch.from_numpy(a).to(dev) for a in
                 scenegen.upstream_grads(cam.image_height, cam.image_width, sc.features.shape[-1], seed=s))
           for s in (1, 2, 3)]
    runs = []
    for camera in (False, True):
        vb = ViewBatch(params)
        vb.zero_()
        cams = []
        for gc, gf, gd in ups:
            color, feat, radii, depth, ctx = vb.forward(rs)
            cams.append((vb.backward(ctx, gc, gf, gd, camera=camera), ctx))
        torch.cuda.synchronize()
        runs.append((vb.flat.clone(), cams))
    assert torch.equal(runs[0][0], runs[1][0])  # parameter gradients, grad_accum and denom
    assert all(c is None for c, _ in runs[0][1])
    e = torch.Tensor([])
    for (cg, ctx), (gc, gf, gd) in zip(runs[1][1], ups):
        assert cg.viewmatrix.shape == (4, 4) and cg.projmatrix.shape == (4, 4) and cg.campos.shape == (3,)
        ref = _C.rasterize_gaussians_backward_camera(
            rs.bg, params["means3D"], ctx.radii, e, params["semantic_feature"], params["scales"], params["rotations"],
            1.0, e, rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, gc, gf, gd, params["shs"], rs.sh_degree,
            rs.campos, ctx.geom, ctx.num_rendered, ctx.binning, ctx.img, False)
        for x, y in zip(cg, ref[9:]):
            assert torch.equal(x, y)
    # the binding checks the buffer it is given
    cg, ctx = runs[1][1][0]
    gc, gf, gd = ups[0]
    none = torch.empty(0, device=dev)
    with pytest.raises(RuntimeError, match="camera_grad"):
        _C.rasterize_gaussians_backward_accum(
            rs.bg, params["means3D"], ctx.radii, e, params["scales"], params["rotations"], 1.0, e, rs.viewmatrix,
            rs.projmatrix, rs.tanfovx, rs.tanfovy, gc, gf, gd, params["shs"], rs.sh_degree, rs.campos, ctx.geom,
            ctx.num_rendered, ctx.binning, ctx.img, vb.scratch, vb.grads["means3D"], vb.grads["shs"], none,
            vb.grads["semantic_feature"], vb.grads["opacities"], vb.grads["scales"], vb.grads["rotations"], none,
            none, none, none, 0, False, 1.0, torch.zeros(34, device=dev))


@pytest.mark.gpu
def test_pose_recovery_on_a_small_scene():
    """Render a target at a true pose, start 1 degree and 2 % of the camera distance off, and run 100 Adam steps on an
    se3_exp delta with photometric_loss_and_grad through the autograd path.  Runs on an H100: rotation error
    1.000 -> 0.0000 to 0.028 degrees, camera-centre error 0.0700 -> 0.00024 to 0.00060; the bar (below 30 % of the
    start) leaves a wide margin."""
    from diff_gaussian_rasterization import GaussianRasterizer
    from diff_gaussian_rasterization.camera import se3_exp, settings_from_w2c
    from diff_gaussian_rasterization.image_loss import photometric_loss_and_grad

    dev = torch.device("cuda")
    sc = scenegen.make_scene(3000, 160, 120, 0, sh_degree=1, seed=5, target_radius_px=8.0)
    cam = sc.cameras[0]
    W, H = cam.image_width, cam.image_height
    d = scenegen.to_torch(sc, dev)
    w2c_true = torch.tensor(cam.viewmatrix, device=dev).t().contiguous()

    def render(w2c):
        rs = settings_from_w2c(w2c, cam.tanfovx, cam.tanfovy, H, W, d["bg"], sh_degree=sc.sh_degree)
        m2 = torch.zeros_like(d["means3D"])
        return GaussianRasterizer(rs)(means3D=d["means3D"], means2D=m2, opacities=d["opacities"], shs=d["shs"],
                                      scales=d["scales"], rotations=d["rotations"])[0]

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
    opt = torch.optim.Adam([xi], lr=2e-3)
    a0, t0 = errors(w2c0)
    for _ in range(100):
        opt.zero_grad()
        color = render(se3_exp(xi) @ w2c0)
        loss, g = photometric_loss_and_grad(color, target)
        color.backward(g)
        opt.step()
    a1, t1 = errors((se3_exp(xi) @ w2c0).detach())
    print(f"pose recovery: rotation {a0:.3f} -> {a1:.4f} deg, translation {t0:.4f} -> {t1:.5f}")
    assert a1 < 0.3 * a0 and t1 < 0.3 * t0
