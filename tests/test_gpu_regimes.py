"""Rasterizer regimes the default scenes never reach (-m gpu), against the CPU oracle and, where a build for the
feature width exists, the unmodified reference extension.

scenegen.make_scene always puts the camera on a ring of radius 3.5 around a [-1,1]^3 cloud of mildly anisotropic
Gaussians, with focal_x == focal_y.  The scenes here reach what that never does:
  inside          the camera inside the cloud: Gaussians behind the camera, just past the 0.2 near plane, and centres
                  off-screen (beyond 1.3 tan_fov) whose footprints still cover the image: the clamped-Jacobian branch
                  of the projection and its zeroed gradient terms (preprocess.cu: project_cov, x_grad_mul/y_grad_mul)
  needles         one axis scaled by 1e-4..1e-3 and one by 8..20: ill-conditioned conics, footprints of hundreds of
                  tiles, the never-cull branch of alpha_extent
  inside_wide     the same camera among wide isotropic splats: the clamp branch with well-conditioned conics
  needles_inside  both at once
  plane           a planar cloud facing an axis-aligned camera: every depth bit-identical, so the order within a tile
                  comes from the stability of the sort alone
and the rasterizer options the other tests fix: focal_x != focal_y, scale_modifier != 1, prefiltered, and feature
inputs that are contiguous but not 16-byte aligned.

The builders draw from their own seeded streams and leave scenegen's untouched (golden fixtures and bench.py depend
on them bit for bit).  The CPU tests of the footprint cull and of the oracle import them from here."""
import math

import numpy as np
import pytest

import parity
import scenegen

pytestmark = pytest.mark.gpu

NEAR = 0.2  # the rasterizer's near plane (preprocess.cu: depth <= 0.2 culls)


# ------------------------------------------------------------------------------------------- scene / camera builders
def camera(W, H, eye, tanx, tany, target=(0.0, 0.0, 0.0), up=(0.0, 1.0, 0.0), znear=0.01, zfar=100.0):
    """scenegen.make_camera with the two tangents set independently (focal_x = W / 2 tanx, focal_y = H / 2 tany)."""
    W2C = scenegen._look_at(np.asarray(eye, np.float64), np.asarray(target, np.float64), np.asarray(up, np.float64))
    P = np.zeros((4, 4))
    P[0, 0] = 1.0 / tanx
    P[1, 1] = 1.0 / tany
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    view = W2C.T.astype(np.float32)
    proj = (W2C.T @ P.T).astype(np.float32)
    campos = np.linalg.inv(view.astype(np.float64))[3, :3].astype(np.float32)
    return scenegen.Camera(W, H, float(np.float32(tanx)), float(np.float32(tany)), view, proj, campos)


def anisotropic(cam, factor):
    """The same pose with tan_fovy scaled by `factor` (focal_y / focal_x = 1 / factor)."""
    return camera(cam.image_width, cam.image_height, cam.campos.astype(np.float64), cam.tanfovx,
                  cam.tanfovy * factor)


def inside(C, P=20000, W=160, H=112, sh_degree=2, views=1, seed=41, target_radius_px=6.0):
    """Camera inside the cloud: ~30 % of it behind the near plane, some Gaussians visible at 0.2 < z < 0.3."""
    return scenegen.make_scene(P=P, W=W, H=H, C=C, sh_degree=sh_degree, views=views, seed=seed, ring_radius=0.6,
                               target_radius_px=target_radius_px)


def needles(sc, seed=7):
    """Per Gaussian one axis scaled by 1e-4..1e-3 and another by 8..20 (log-uniform), in place."""
    rng = np.random.Generator(np.random.PCG64(seed))
    P = sc.P
    ax = rng.permuted(np.tile(np.arange(3), (P, 1)), axis=1)[:, :2]
    thin = np.exp(rng.uniform(math.log(1e-4), math.log(1e-3), P))
    long = np.exp(rng.uniform(math.log(8.0), math.log(20.0), P))
    s = sc.scales.astype(np.float64)
    s[np.arange(P), ax[:, 0]] *= thin
    s[np.arange(P), ax[:, 1]] *= long
    sc.scales = s.astype(np.float32)
    return sc


def plane(C, P=3000, W=128, H=96, sh_degree=1, seed=43):
    """A planar cloud (z = 0 exactly) facing a camera on the -z axis with axis-aligned view axes: every view-space
    depth is 0*x + 0*y + 1*0 + 3.5, bit-identical for all Gaussians."""
    sc = scenegen.make_scene(P=P, W=W, H=H, C=C, sh_degree=sh_degree, seed=seed, target_radius_px=5.0)
    sc.means3D = sc.means3D.copy()
    sc.means3D[:, 2] = 0.0
    tanx = math.tan(math.radians(60.0) / 2)
    sc.cameras = [camera(W, H, (0.0, 0.0, -3.5), tanx, tanx * H / W)]
    return sc


def make(name, C):
    """Regime scene by name -> (scene, camera)."""
    if name == "inside":
        sc = inside(C)
    elif name == "inside_wide":
        sc = inside(C, P=12000, seed=47, target_radius_px=40.0)
    elif name == "needles":
        sc = needles(scenegen.make_scene(P=3000, W=160, H=112, C=C, sh_degree=2, seed=42, target_radius_px=24.0))
    elif name == "needles_inside":
        sc = needles(inside(C, P=8000, seed=44, target_radius_px=15.0))
    elif name == "plane":
        sc = plane(C)
    else:
        raise KeyError(name)
    return sc, sc.cameras[0]


def view_space(sc, cam):
    """float64 view-space positions t = W2C * mean of every Gaussian."""
    vm = cam.viewmatrix.astype(np.float64)
    return sc.means3D.astype(np.float64) @ vm[:3, :3] + vm[3, :3]


def regime_counts(sc, cam, radii):
    """Visible Gaussians in the clamped-x / clamped-y branch of the projection and just past the near plane."""
    t = view_space(sc, cam)
    vis = radii > 0
    with np.errstate(all="ignore"):
        cx = vis & (np.abs(t[:, 0] / t[:, 2]) > 1.3 * cam.tanfovx)
        cy = vis & (np.abs(t[:, 1] / t[:, 2]) > 1.3 * cam.tanfovy)
    near = vis & (t[:, 2] < 0.3)
    return dict(visible=int(vis.sum()), clamp_x=int(cx.sum()), clamp_y=int(cy.sum()), near=int(near.sum()),
                behind=int((t[:, 2] <= NEAR).sum()))


def _grads(cam, C, seed=1234):
    return scenegen.upstream_grads(cam.image_height, cam.image_width, C, seed=seed)


# Needles: the gradients through the 2-D covariance are compared for conics with an eigenvalue ratio up to this; above
# it they differ between two runs of the same build (see parity.tie_aware_compare).
NEEDLE_COND_MAX = 100.0


def _check_all(sc, cam, label, **opts):
    """Forward + backward with fresh N(0,1) upstream gradients against the CPU oracle and, where available, the
    reference build; indices exact, floats at the parity bar (tie-aware against the oracle)."""
    from oracle import ref_wrapper as rw

    if label.startswith("needles"):
        opts["cond_max"] = NEEDLE_COND_MAX
    grads = _grads(cam, sc.C)
    ours = parity.tie_aware_compare(sc, cam, label, grads=grads, vs_ref=False, **opts)
    if rw.available(sc.C):
        parity.tie_aware_compare(sc, cam, label, grads=grads, vs_ref=True, ours=ours, **opts)
    return ours


# ------------------------------------------------------------------------------------------- regimes x feature widths
CASES = [("inside", 0), ("inside", 16), ("inside", 200), ("inside", 512), ("inside_wide", 3), ("inside_wide", 128),
         ("needles", 3), ("needles", 128),
         ("needles_inside", 0), ("needles_inside", 3), ("needles_inside", 16), ("needles_inside", 128),
         ("needles_inside", 200), ("needles_inside", 512), ("plane", 3), ("plane", 16), ("plane", 128), ("plane", 512)]


@pytest.mark.parametrize("name,C", CASES)
def test_regime_vs_oracle_and_structure(name, C):
    sc, cam = make(name, C)
    ours = _check_all(sc, cam, f"{name} C={C}")
    n_eq = parity.check_structure(ours, cam, sc.P)
    cnt = regime_counts(sc, cam, ours["radii"])
    print(f"[{name} C={C}] {cnt} equal-depth neighbours={n_eq} "
          f"never-cull={int((ours['rec'][ours['radii'] > 0, 2] > 1e30).sum())} max radius={int(ours['radii'].max())}")
    # the scene reaches the regime it is named for
    if name in ("inside", "inside_wide", "needles_inside"):
        assert cnt["near"] > 0 and cnt["behind"] > 0, cnt
    if name in ("inside_wide", "needles_inside"):
        assert cnt["clamp_x"] > 100 and cnt["clamp_y"] > 100, cnt
    if name.startswith("needles"):
        assert (ours["rec"][ours["radii"] > 0, 2] > 1e30).any()  # alpha_extent's never-cull branch
        assert int(ours["radii"].max()) > 200
    if name == "plane":
        assert n_eq > 1000 and np.unique(ours["rec"][ours["radii"] > 0, 11]).size == 1


# ------------------------------------------------------------------------------------------- rasterizer options
@pytest.mark.parametrize("factor", [1.15, 1 / 1.15])
@pytest.mark.parametrize("name", ["inside_wide", "needles_inside"])
def test_anisotropic_focal(name, factor):
    """focal_x != focal_y in both directions: a swapped focal or clamp limit anywhere in preprocess shows here."""
    sc, cam = make(name, 16)
    cam = anisotropic(cam, factor)
    assert abs(cam.tanfovy / cam.tanfovx - factor * cam.image_height / cam.image_width) < 1e-6
    ours = _check_all(sc, cam, f"{name} fy/fx={1 / factor:.3f}")
    cnt = regime_counts(sc, cam, ours["radii"])
    assert cnt["clamp_x"] > 100 and cnt["clamp_y"] > 100, cnt


@pytest.mark.parametrize("mod", [0.6, 1.7])
@pytest.mark.parametrize("name", ["inside_wide", "needles"])
def test_scale_modifier(name, mod):
    """scale_modifier reaches the covariance of the forward and the s = mod * scale of the backward."""
    sc, cam = make(name, 16)
    ours = _check_all(sc, cam, f"{name} scale_modifier={mod}", scale_modifier=mod)
    base = parity.run_ours(sc, cam)
    assert not np.array_equal(ours["radii"], base["radii"])  # the modifier did change the footprints


def test_prefiltered_is_bit_identical_on_a_cloud_in_front_of_the_near_plane():
    """prefiltered=True only removes the near-plane cull.  With prefiltered set, a Gaussian behind the near plane is a
    caller error that stops the kernel, so the cloud is checked to lie in front of it on the host BEFORE the call."""
    sc = scenegen.make_scene(P=4000, W=160, H=112, C=16, sh_degree=2, seed=45)
    cam = sc.cameras[0]
    assert view_space(sc, cam)[:, 2].min() > NEAR + 0.5
    grads = _grads(cam, sc.C)
    a = parity.run_ours(sc, cam, grads=grads, prefiltered=False)
    b = parity.run_ours(sc, cam, grads=grads, prefiltered=True)
    for k in ("color", "feature_map", "depth", "final_T", "radii", "n_contrib", "point_list", "ranges", "rec"):
        assert np.array_equal(a[k], b[k]), k
    for k in a["grads"]:
        r = parity.float_mismatch(b["grads"][k], a["grads"][k], atol_rel=parity.GRAD_ATOL_REL)[0]
        assert r <= 1.0, (k, r)
    from oracle import ref_wrapper as rw

    if rw.available(sc.C):
        parity.tie_aware_compare(sc, cam, "prefiltered", grads=grads, vs_ref=True, ours=b, prefiltered=True)


# ------------------------------------------------------------------------------------------- misaligned features
def _offset_copy(x):
    """A contiguous copy of `x` that starts one float past a 16-byte boundary."""
    import torch

    buf = torch.empty(x.numel() + 1, device=x.device, dtype=x.dtype)
    y = buf[1:].view(x.shape)
    y.copy_(x)
    assert y.is_contiguous() and y.data_ptr() % 16 != 0 and torch.equal(y, x)
    return y


@pytest.mark.parametrize("C", [4, 16, 128, 256, 512, 4096])
def test_misaligned_features_and_feature_gradients(C):
    """semantic_feature and dL/dfeature_map given as contiguous views at a 1-float storage offset with C % 4 == 0:
    the forward composite (use_bulk, composite_fwd.cu) and the feature backward (vec, feature_bwd.cu) test the
    pointer's alignment before any 128-bit access and fall back to scalar loads.  The forward must be bit-identical
    to the aligned call and the gradients agree within the parity bar."""
    import torch
    from diff_gaussian_rasterization import _C

    sc, cam = make("inside_wide", C)
    assert cam.image_width % 4 == 0  # the aligned call takes the 128-bit image-row loads of the backward
    t = scenegen.to_torch(sc, "cuda")
    rs = parity.settings(sc, cam, "cuda")
    gc, gf, gd = [torch.from_numpy(g).cuda() for g in _grads(cam, C)]
    e = torch.Tensor([])

    def run(sf, gfm):
        fwd = _C.rasterize_gaussians(rs["bg"], t["means3D"], e, sf, t["opacities"], t["scales"], t["rotations"],
                                     rs["scale_modifier"], e, rs["viewmatrix"], rs["projmatrix"], rs["tanfovx"],
                                     rs["tanfovy"], rs["image_height"], rs["image_width"], t["shs"], rs["sh_degree"],
                                     rs["campos"], rs["prefiltered"], False)
        R, color, feat, depth, radii, geom, binning, img = fwd
        bwd = _C.rasterize_gaussians_backward(rs["bg"], t["means3D"], radii, e, sf, t["scales"], t["rotations"],
                                              rs["scale_modifier"], e, rs["viewmatrix"], rs["projmatrix"],
                                              rs["tanfovx"], rs["tanfovy"], gc, gfm, gd, t["shs"], rs["sh_degree"],
                                              rs["campos"], geom, R, binning, img, False)
        return [x.clone() for x in (color, feat, depth, radii)], [x.clone() for x in bwd]

    sf_mis, gf_mis = _offset_copy(t["semantic_feature"]), _offset_copy(gf)
    assert t["semantic_feature"].data_ptr() % 16 == 0 and gf.data_ptr() % 16 == 0
    (fa, ga), (fm, gm) = run(t["semantic_feature"], gf), run(sf_mis, gf_mis)
    for k, x, y in zip(("color", "feature_map", "depth", "radii"), fa, fm):
        assert torch.equal(x, y), k
    names = ("means2D", "colors_precomp", "semantic_feature", "opacities", "means3D", "cov3D_precomp", "sh",
             "scales", "rotations")
    assert float(ga[2].abs().max()) > 0
    for k, x, y in zip(names, ga, gm):
        r = parity.float_mismatch(y.cpu().numpy(), x.cpu().numpy(), atol_rel=parity.GRAD_ATOL_REL)[0]
        assert r <= 1.0, (k, r)
