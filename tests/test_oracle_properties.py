"""Properties of the CPU oracle that do not need the reference: they guard the checker itself
(culling, skip semantics, feature-width independence, and a finite-difference check of its backward)."""
import copy

import numpy as np
import pytest

import oracle
import parity
import scenegen


@pytest.fixture(scope="module")
def tiny():
    sc = scenegen.make_config("tiny")
    return sc, sc.cameras[0]


def test_behind_camera_is_culled_with_zero_gradients(tiny):
    sc, cam = tiny
    sc = copy.copy(sc)
    sc.means3D = sc.means3D.copy()
    sc.means3D[:50] = cam.campos * 2.0  # behind the camera (it looks at the origin)
    grads = scenegen.upstream_grads(cam.image_height, cam.image_width, sc.C)
    o = parity.run_oracle(sc, cam, grads=grads, threads=1)
    assert (o["radii"][:50] == 0).all()
    for k in ("means3D", "scales", "rotations", "opacities", "sh", "semantic_feature", "means2D"):
        assert np.abs(o["grads"][k][:50]).max() == 0, k


def test_zero_and_subthreshold_opacity_contribute_nothing(tiny):
    sc, cam = tiny
    base = parity.run_oracle(sc, cam, threads=1)
    sc2 = copy.copy(sc)
    sc2.opacities = sc.opacities.copy()
    drop = np.arange(sc.P) % 3 == 0
    sc2.opacities[drop] = 1.0 / 300.0
    a = parity.run_oracle(sc2, cam, threads=1)
    sc3 = copy.copy(sc)  # same cloud with those Gaussians removed altogether
    keep = ~drop
    for f in ("means3D", "scales", "rotations", "opacities", "shs", "features"):
        setattr(sc3, f, getattr(sc, f)[keep])
    b = parity.run_oracle(sc3, cam, threads=1)
    for k in ("color", "feature_map", "depth", "final_T"):
        assert np.array_equal(a[k], b[k]), k
    assert not np.array_equal(a["color"], base["color"])


def test_colour_depth_and_indices_do_not_depend_on_feature_width(tiny):
    sc, cam = tiny
    a = parity.run_oracle(sc, cam, threads=1)
    sc0 = copy.copy(sc)
    sc0.features = np.zeros((sc.P, 1, 0), np.float32)
    b = parity.run_oracle(sc0, cam, threads=1)
    for k in ("color", "depth", "final_T", "n_contrib", "point_list", "ranges", "radii"):
        assert np.array_equal(a[k], b[k]), k


def test_n_contrib_is_index_of_last_blended_and_T_matches(tiny):
    sc, cam = tiny
    o = parity.run_oracle(sc, cam, threads=1)
    f = o["fwd"]
    W = cam.image_width
    gx = (W + 15) // 16
    for (py, px) in [(3, 5), (20, 40), (55, 79), (31, 17)]:
        r0, r1 = f["ranges"][(py // 16) * gx + px // 16]
        T, last = 1.0, 0
        for i in range(int(r0), int(r1)):
            g = f["point_list"][i]
            dx, dy = f["means2D"][g] - np.array([px, py], np.float32)
            a, b, c, op = f["conic_opacity"][g]
            power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
            if power > 0:
                continue
            alpha = min(0.99, op * np.exp(power))
            if alpha < 1 / 255:
                continue
            if T * (1 - alpha) < 1e-4:
                break
            T *= 1 - alpha
            last = i - int(r0) + 1
        assert abs(T - o["final_T"][py, px]) < 1e-5
        assert last == o["n_contrib"][py, px]


def test_backward_against_finite_differences():
    """Central differences on a 40-Gaussian scene for the loss L = <color, gc> + <depth, gd> (+ <feat, gf> for the
    feature input).  Reference quirks kept: the feature loss does not reach geometry (backward.cu:575 disabled), and
    the rotation gradient omits the normalisation Jacobian, so those are checked on the matching sub-losses only."""
    sc = scenegen.make_scene(P=40, W=48, H=32, C=4, sh_degree=2, seed=77, target_radius_px=7.0)
    cam = sc.cameras[0]
    sc.opacities[:] = np.clip(sc.opacities, 0.3, 0.9)
    gc, gf, gd = scenegen.upstream_grads(32, 48, 4, seed=5)

    def loss(s, with_feat):
        f = oracle.forward(s, cam)
        v = float((f["color"].astype(np.float64) * gc).sum() + (f["depth"].astype(np.float64) * gd).sum())
        if with_feat:
            v += float((f["feature_map"].astype(np.float64) * gf).sum())
        return v

    oracle.set_threads(1)
    f0 = oracle.forward(sc, cam)
    g_geo = oracle.backward(sc, cam, f0, gc, np.zeros_like(gf), gd)
    g_all = oracle.backward(sc, cam, f0, gc, gf, gd)
    rng = np.random.Generator(np.random.PCG64(3))

    def fd(field, idx, eps, with_feat):
        sp, sm = copy.copy(sc), copy.copy(sc)
        ap, am = getattr(sc, field).copy(), getattr(sc, field).copy()
        ap[idx] += eps
        am[idx] -= eps
        setattr(sp, field, ap)
        setattr(sm, field, am)
        return (loss(sp, with_feat) - loss(sm, with_feat)) / (2 * eps)

    checks = [("means3D", "means3D", 2e-4, g_geo), ("scales", "scales", 1e-5, g_geo),
              ("opacities", "opacities", 1e-3, g_geo), ("shs", "sh", 1e-2, g_geo)]
    for field, gname, eps, g in checks:
        arr = getattr(sc, field)
        num, ana = [], []
        for _ in range(12):
            idx = tuple(rng.integers(0, s) for s in arr.shape)
            if f0["radii"][idx[0]] == 0:
                continue
            num.append(fd(field, idx, eps, False))
            ana.append(float(g[gname][idx]))
        num, ana = np.array(num), np.array(ana)
        scale = max(np.abs(ana).max(), 1e-3)
        assert np.abs(num - ana).max() <= 0.03 * scale + 2e-3, (field, num, ana)
    # features: exact linear dependence
    num, ana = [], []
    for _ in range(10):
        idx = (int(rng.integers(0, sc.P)), 0, int(rng.integers(0, 4)))
        num.append(fd("features", idx, 1e-2, True))
        ana.append(float(g_all["semantic_feature"][idx]))
    assert np.allclose(num, ana, rtol=2e-3, atol=2e-4)
    # the feature loss moves nothing but the features (reference quirk D.1)
    for k in ("means3D", "scales", "rotations", "opacities", "sh"):
        assert np.array_equal(g_geo[k], g_all[k]), k


# ------------------------------------------------------------------------------------------- projection backward
# The oracle is the only comparator for cameras inside the cloud, needles, focal_x != focal_y and scale_modifier != 1.
# These tests pin its covariance-projection backward (oracle_preprocess_backward fed nothing but dL/dconic) to central
# differences of a float64 restatement of the forward projection.
def _rot64(q):
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]  # not renormalised, as in the forward
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                     np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                     np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def _cov3d64(scale, q, mod):
    R = _rot64(q)
    return R @ ((mod * scale)[:, :, None] ** 2 * np.swapaxes(R, -1, -2))


def _view64(mean, cam):
    vm = cam.viewmatrix.astype(np.float64)
    return mean @ vm[:3, :3] + vm[3, :3]


def _limits(cam):
    return 1.3 * np.float64(np.float32(cam.tanfovx)), 1.3 * np.float64(np.float32(cam.tanfovy))


def _clamp64(t, cam):
    """The position J is evaluated at: x/z and y/z clamped to 1.3 tan_fov (reference forward.cu:82-85)."""
    lx, ly = _limits(cam)
    return np.stack([np.clip(t[:, 0] / t[:, 2], -lx, lx) * t[:, 2], np.clip(t[:, 1] / t[:, 2], -ly, ly) * t[:, 2],
                     t[:, 2]], -1)


def _conic_at64(tc, cov3d, cam):
    """(A, B, C) of the inverse of J W cov3d W^T J^T + 0.3 I with J evaluated at view-space position tc."""
    fx = cam.image_width / (2 * np.float64(cam.tanfovx))
    fy = cam.image_height / (2 * np.float64(cam.tanfovy))
    Rw = cam.viewmatrix.astype(np.float64)[:3, :3].T
    tx, ty, tz = tc[:, 0], tc[:, 1], tc[:, 2]
    z = np.zeros_like(tz)
    J = np.stack([np.stack([fx / tz, z, -fx * tx / tz ** 2], -1), np.stack([z, fy / tz, -fy * ty / tz ** 2], -1)], -2)
    T = J @ Rw
    c2 = T @ cov3d @ np.swapaxes(T, -1, -2)
    a, b, c = c2[:, 0, 0] + 0.3, c2[:, 0, 1], c2[:, 1, 1] + 0.3
    det = a * c - b * b
    return np.stack([c / det, -b / det, a / det], -1)


def _conic64(mean, scale, q, mod, cam):
    return _conic_at64(_clamp64(_view64(mean, cam), cam), _cov3d64(scale, q, mod), cam)


def _conic_backward(sc, cam, f, dL_dconic, mod):
    """oracle_preprocess_backward with dL/dconic as the only upstream gradient (no SH, mean2D or depth terms)."""
    import ctypes

    P, F, p = sc.P, oracle._f32, oracle._p
    z3, z1 = np.zeros((P, 3), np.float32), np.zeros(P, np.float32)
    g = dict(means3D=np.zeros((P, 3), np.float32), cov3D=np.zeros((P, 6), np.float32),
             scales=np.zeros((P, 3), np.float32), rotations=np.zeros((P, 4), np.float32))
    oracle.lib().oracle_preprocess_backward(
        P, 0, 0, p(F(sc.means3D)), p(f["radii"]), p(None), p(f["clamped"]), p(F(sc.scales)), p(F(sc.rotations)),
        ctypes.c_float(mod), p(F(f["cov3D"])), p(F(cam.viewmatrix).reshape(-1)), p(F(cam.projmatrix).reshape(-1)),
        p(F(cam.campos)), cam.image_width, cam.image_height, ctypes.c_float(cam.tanfovx), ctypes.c_float(cam.tanfovy),
        p(z3), p(F(dL_dconic)), p(z3), p(z1), p(g["means3D"]), p(g["cov3D"]), p(None), p(g["scales"]),
        p(g["rotations"]))
    return g


@pytest.fixture(scope="module")
def projection_case():
    """Needles seen from inside the cloud through a camera with focal_y = focal_x / 1.15, scale_modifier 1.7: about
    a third of the visible Gaussians sit in each clamp branch."""
    import test_gpu_regimes as regimes

    sc = regimes.needles(regimes.inside(0, P=600, W=64, H=48, seed=46, target_radius_px=15.0))
    cam = regimes.anisotropic(sc.cameras[0], 1.15)
    mod = 1.7
    oracle.set_threads(1)
    f = oracle.forward(sc, cam, scale_modifier=mod, render=False)
    vis = f["radii"] > 0
    rng = np.random.Generator(np.random.PCG64(9))
    g4 = rng.standard_normal((sc.P, 4)).astype(np.float32)
    # the loss whose gradient the backward forms: conic B is the off-diagonal of a symmetric matrix, counted twice
    w = np.stack([g4[:, 0], 2 * g4[:, 1], g4[:, 3]], -1).astype(np.float64)
    t = _view64(sc.means3D.astype(np.float64), cam)
    lx, ly = _limits(cam)
    rx, ry = np.abs(t[:, 0] / t[:, 2]) / lx, np.abs(t[:, 1] / t[:, 2]) / ly
    away = vis & (np.abs(rx - 1) > 0.02) & (np.abs(ry - 1) > 0.02)  # central differences stay on one side
    return dict(sc=sc, cam=cam, mod=mod, f=f, vis=vis, w=w, g=_conic_backward(sc, cam, f, g4, mod), t=t, rx=rx,
                ry=ry, free=away & (rx < 1) & (ry < 1), clamped=away & ((rx > 1) | (ry > 1)))


def _fd(fn, x, h, w):
    """Central differences of sum(w * fn(x)) per row, every row perturbed at once (rows are independent)."""
    out = np.zeros(x.shape)
    for k in range(x.shape[1]):
        xp, xm = x.copy(), x.copy()
        xp[:, k] += h
        xm[:, k] -= h
        out[:, k] = ((fn(xp) - fn(xm)) * w).sum(-1) / (2 * h)
    return out


def _rel(a, b):
    return np.linalg.norm(a - b, axis=1) / (np.linalg.norm(b, axis=1) + 1e-30)


def _assert_close(a, b, sel, what):
    e = _rel(a, b)[sel]
    assert sel.sum() > 50 and np.percentile(e, 95) < 2e-3 and e.max() < 0.1, (what, np.percentile(e, 95), e.max())


def test_float64_projection_restates_the_oracle_forward(projection_case):
    """The restatement used below reproduces the oracle's conics, clamped Gaussians included: the forward evaluates
    J at the clamped position."""
    c = projection_case
    sc = c["sc"]
    m = _conic64(sc.means3D.astype(np.float64), sc.scales.astype(np.float64), sc.rotations.astype(np.float64),
                 c["mod"], c["cam"])
    co = c["f"]["conic_opacity"][:, :3].astype(np.float64)
    e = np.abs(co - m).max(1) / np.abs(m).max(1)
    for sel in (c["free"], c["clamped"]):
        assert sel.sum() > 50 and np.median(e[sel]) < 1e-5 and e[sel].max() < 1e-2


def test_projection_backward_against_finite_differences_outside_the_clamp(projection_case):
    """fx != fy and scale_modifier != 1, Gaussians whose centre projects inside 1.3 tan_fov on both axes: dL/dmean and
    dL/drotation are the true gradients.  dL/dscale is formed with respect to s = scale_modifier * scale (the
    reference's computeCov3D backward builds M from s and never applies the chain-rule factor), so central
    differences in `scale` are scale_modifier times the returned value."""
    c = projection_case
    sc, cam, mod, w, g = c["sc"], c["cam"], c["mod"], c["w"], c["g"]
    m, s, q = sc.means3D.astype(np.float64), sc.scales.astype(np.float64), sc.rotations.astype(np.float64)
    h = 1e-6 * float(np.abs(c["t"][c["vis"], 2]).min())
    dm = _fd(lambda x: _conic64(x, s, q, mod, cam), m, h, w)
    ds = _fd(lambda x: _conic64(m, x, q, mod, cam), s, 1e-7 * float(s.max()), w)
    dq = _fd(lambda x: _conic64(m, s, x, mod, cam), q, 1e-7, w)
    _assert_close(g["means3D"], dm, c["free"], "means3D")
    _assert_close(g["rotations"], dq, c["vis"], "rotations")
    _assert_close(mod * g["scales"], ds, c["vis"], "scales")
    assert np.median(_rel(g["scales"], ds)[c["vis"]]) > 0.3  # the returned value itself is off by the factor


def test_projection_backward_clamp_branch_is_the_reference_quirk(projection_case):
    """Centre beyond 1.3 tan_fov on an axis: the forward evaluates J at the clamped position (so it does not move with
    the centre along that axis), and the backward zeroes that axis's term (x_grad_mul / y_grad_mul) and takes the
    depth derivative with the clamped coordinate held fixed, although the clamped coordinate is 1.3 tan_fov * depth.
    That is the reference's behaviour and the kernels must reproduce it, so it is asserted here, not corrected:
    view-space gradient = (mul_x dL/dtx_c, mul_y dL/dty_c, dL/dtz |tx_c, ty_c fixed), rotated to world space."""
    c = projection_case
    sc, cam, mod, w, g, t = c["sc"], c["cam"], c["mod"], c["w"], c["g"], c["t"]
    m, s, q = sc.means3D.astype(np.float64), sc.scales.astype(np.float64), sc.rotations.astype(np.float64)
    h = 1e-6 * float(np.abs(t[c["vis"], 2]).min())
    cov = _cov3d64(s, q, mod)
    dtc = _fd(lambda x: _conic_at64(x, cov, cam), _clamp64(t, cam), h, w)
    mul = np.stack([(c["rx"] <= 1), (c["ry"] <= 1), np.ones(sc.P, bool)], -1)
    Rw = cam.viewmatrix.astype(np.float64)[:3, :3].T
    quirk = (mul * dtc) @ Rw
    _assert_close(g["means3D"], quirk, c["clamped"], "means3D (clamp branch)")
    # ... which is not the gradient of the forward: differentiating through the clamp disagrees
    dm = _fd(lambda x: _conic64(x, s, q, mod, cam), m, h, w)
    assert np.median(_rel(g["means3D"], dm)[c["clamped"]]) > 0.05
    # along a clamped axis the forward is flat, so the zeroed term agrees with the true derivative there
    cx = c["clamped"] & (c["rx"] > 1)
    assert cx.sum() > 20
    along_x = (dm @ Rw.T)[cx, 0]
    assert np.abs(along_x).max() <= 1e-4 * np.abs(dm[cx]).max()
    assert np.abs((g["means3D"].astype(np.float64) @ Rw.T)[cx, 0]).max() <= 1e-4 * np.abs(g["means3D"][cx]).max()
