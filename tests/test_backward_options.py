"""The general backward (f3dgs_backward_alpha_invdepth, f3dgs_backward_accum_alpha_invdepth) with its options on
together -- antialiasing, the feature term of dL/dalpha (float32 or float16 rows), a float32 or scaled float16 map
gradient, the camera gradient, the opacity and inverse-depth planes, the assigning or accumulating entry -- against one
float64 model.

Model, per view rendered by the planes forward in the same mode, over its own records (op_eff under antialiasing),
blended pairs and blend weights:
  * composite: blend_weights.composite_model with d = c.Gc + z Gd + gI / z [+ f.Gf] and bg_dot = bg.Gc - gA
    (test_alpha_invdepth.planes_model), f the rows the backward reads and Gf the map as the composite scales it;
    dL/dcolor, dL/dfeature and dL/dz through the blend-weight identities (dL/dz with its -w gI / z^2 term);
  * preprocess: the native composite intermediates pushed through camera_grad_model.preprocess_chain, or with
    antialiasing through test_antialiasing.model_gradients, whose opacity gradient is rho g with g = dL/dop_eff of the
    composite (read from the same call with antialiasing off, on the same buffers);
  * camera: camera_grad_model.terms plus the antialiasing term, with test_antialiasing's bar;
  * accumulating entry: dL_dopacity as above, dL_dmean2D_out the composite's dL/dmean2D, grad_accum += |dL/dmean2D.xy|
    of the full model, denom += (radii > 0), dL/dfeature, and the camera on the assigning call's intermediates.  Its
    other preprocess outputs are checked on the block scene below, bitwise against the assigning entry's: its own
    composite intermediates stay in its scratch.
The matrix: antialiasing x feature term (none, float32, float16 rows) x map gradient (float32, float16 at scale 1e-3)
x camera x entry, 96 cells on `small`, and the all-on corners on harder scenes, under three upstream gradients.
On test_camera_grad._block_scene every per-Gaussian value is reduced with one add, so there the options are checked
bitwise against each other, and the Python surfaces against the C entries.  CPU: negative controls on the oracle view,
one term of the model removed at a time.
"""
import ctypes
import functools
import itertools

import numpy as np
import pytest
import torch

import blend_weights as bw
import camera_grad_model as cgm
from test_alpha_invdepth import _backward_planes, _plane_grads, dz_check, planes_model
from test_antialiasing import MIN_RATIO, model_gradients
from test_geometry_grads import NEEDLE_COND_MAX, View, _report, _scene, _upstreams, preprocess_check

S16 = 1e-3  # the float16 map's scale
FEATS = ("none", "f32", "f16")
MAPS = ("f32", "f16")
AA_BAR = 1e-4  # test_antialiasing's relative bar on the preprocess outputs


def _t(a, dev="cpu"):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_backward_scratch_bytes.restype = ctypes.c_size_t
    return L


# ------------------------------------------------------------------------------------------------------------ the model
def rho_opacity(ref_g, bar_g, rho, cond):
    """(ref, bar) of dL_dopacity = rho g under antialiasing: the composite's bar scaled by rho, plus rho's own float32
    error (test_antialiasing's 64 u (1 + cond) relative bar on op_eff) on |g|, and the product's rounding."""
    ref = rho * ref_g
    return ref, rho * bar_g + (64 * bw.U * (1.0 + cond) + bw.U) * ref.abs()


def rho_model(sc, cam, idx, mod=1.0, cov=None):
    """Per Gaussian (all P, 1 outside idx): rho = op_eff / opacity in float64, the conditioning of det0 that its float32
    value carries (infinite within a factor 4 of the clamp, where float32 may land on either side), and the needle flag
    of the dilated 2-D covariance."""
    from test_antialiasing import _f64, aa_quantities

    P = sc.P
    cv = _f64(cov)[idx] if cov is not None else cgm.cov3d_from_scale_rot(_f64(sc.scales)[idx], _f64(sc.rotations)[idx],
                                                                         mod)
    _, _, op_eff, _, _, (a0, b0, c0) = aa_quantities(
        _f64(sc.means3D)[idx], cv, _f64(sc.opacities)[idx], _f64(cam.viewmatrix).reshape(16),
        _f64(cam.projmatrix).reshape(16), _f64(cam.campos), cam.image_width, cam.image_height, cam.tanfovx,
        cam.tanfovy, 0, colors=torch.zeros(len(idx), 3, dtype=torch.float64))
    det0 = a0 * c0 - b0 * b0
    det = (a0 + 0.3) * (c0 + 0.3) - b0 * b0
    cond = (a0.abs() * c0.abs() + b0 * b0) / det0.abs().clamp_min(1e-300)
    cond = torch.where(det0 / det < 4 * MIN_RATIO, torch.full_like(cond, float("inf")), cond)
    a_, c_ = a0 + 0.3, c0 + 0.3
    mid, dd = 0.5 * (a_ + c_), torch.sqrt(0.25 * (a_ - c_) ** 2 + b0 * b0)
    out = dict(rho=torch.ones(P, dtype=torch.float64), cond=torch.zeros(P, dtype=torch.float64),
               needle=torch.zeros(P, dtype=torch.bool))
    out["rho"][idx] = op_eff / _f64(sc.opacities)[idx].reshape(-1)
    out["cond"][idx] = cond
    out["needle"][idx] = (mid + dd) / (mid - dd) > NEEDLE_COND_MAX
    return out


def camera_reference(v, mids, m=None):
    """(ref, bar) of dL_dcamera: camera_grad_model.terms on the composite intermediates mids (mean2D, conic, color, dz),
    and with antialiasing the model_gradients result m, whose extra term (rho's) is weighted as test_antialiasing does."""
    sc, cam = v.sc, v.cam
    cov = v.cov.cpu().double() if v.cov.numel() else cgm.cov3d_from_scale_rot(_t(sc.scales).double(),
                                                                             _t(sc.rotations).double(), v.mod)
    t = cgm.terms(sc.means3D, cov, v.vm.cpu(), v.pm.cpu(), v.cp.cpu(), [mids[k].cpu() for k in
                                                                        ("mean2D", "conic", "color", "dz")],
                  v.W, v.H, cam.tanfovx, cam.tanfovy, v.D, shs=v.shs.cpu() if v.M else None,
                  colors=v.cols.cpu() if v.cols.numel() else None, visible=v.visible)
    ref, scale = cgm.camera_vector(t), cgm.camera_scale(t)
    if m is not None:
        well = m["eig_ratio"] <= NEEDLE_COND_MAX
        kmax = float(m["kappa"].clamp_min(1.0)[well].max()) if bool(well.any()) else 1.0
        scale = scale + (m["camera"] - ref).abs() * kmax
        ref = m["camera"]
    return ref, 1e-5 * scale + 1e-7 * float(cgm.camera_scale(t, needles=False).max())


def aa_preprocess_check(v, m, ours, accum=False):
    """The antialiased preprocess outputs (not dL_dopacity) against model_gradients' m with test_antialiasing's bar,
    needles skipped; dL/dsh, which rho does not reach, against preprocess_chain."""
    well = m["eig_ratio"] <= NEEDLE_COND_MAX
    k = m["kappa"].clamp_min(1.0)
    out = {}
    for key in [x for x in v.outputs(ours, accum) if x in m and x != "sh"]:
        n = ours[key].cpu().double().reshape(v.P, -1)
        r = m[key]
        floor = 1e-6 * float(r[well].abs().max()) + 1e-12 if bool(well.any()) else 1e-12
        bar = AA_BAR * k[:, None] * r.abs().sum(1, keepdim=True) + floor
        ratio = ((n - r).abs() / bar)[well]
        out[f"dL_d{key}"] = float(ratio.max()) if ratio.numel() else 0.0
    return out


class Reference:
    """The composite model of one view under one set of upstream gradients, plane gradients, feature rows and map."""

    def __init__(self, v, ups, ga, gi, sf, gmap, map_scale):
        dev = v.pairs.pix.device
        HW = v.W * v.H
        self.Gc = _t(ups[0]).reshape(3, HW).t().to(dev)
        self.Gd, self.GA, self.GI = (_t(x).reshape(HW).to(dev) for x in (ups[2], ga, gi))
        # the map as the composite reads it: float32, or fl(scale * float(h))
        self.Gf = ((gmap.float() * map_scale) if map_scale is not None else gmap).reshape(v.C, HW).t().to(dev)
        F = sf.reshape(v.P, v.C).float().to(dev) if sf is not None else None
        self.rec = v.base["rec"]
        self.ref6, self.bar6 = planes_model(v.pairs, v.w, self.rec, v.P, v.bg, self.Gc, self.Gd, self.GA, self.GI,
                                            F=F, Gf=self.Gf if F is not None else None)
        self.Wt = bw.Weights(v.pairs, v.w, v.P)

    def composite(self, o, rho=None, opacity=True):
        """Worst ratios of the composite's outputs in o (an assigning entry's); rho: antialiased dL_dopacity."""
        assert bool((o["mean2D"][:, 2] == 0).all()) and bool((o["conic"][:, 2] == 0).all())
        g6 = bw.geom6(o["mean2D"], o["conic"], o["opacity"]).double().to(self.ref6.device)
        r = bw._ratio((g6 - self.ref6).abs(), self.bar6).max(0).values
        worst = {k: float(x) for k, x in zip(("dL_dmean2D.x", "dL_dmean2D.y", "dL_dconic.a", "dL_dconic.b",
                                              "dL_dconic.c"), r)}
        if opacity:
            worst["dL_dopacity"] = self.opacity(o["opacity"], rho)
        P = self.ref6.shape[0]
        worst["dL_dcolor"] = self.Wt.per_gaussian(o["color"].reshape(P, 3), self.Gc)
        worst["dL_dz"] = dz_check(self.Wt, self.rec, o["dz"], self.Gd, self.GI)
        return worst

    def opacity(self, ours, rho=None):
        ref, bar = self.ref6[:, 5].cpu(), self.bar6[:, 5].cpu()
        ours = ours.reshape(-1).cpu().double()
        if rho is None:
            return float(bw._ratio((ours - ref).abs(), bar).max())
        ref, bar = rho_opacity(ref, bar, rho["rho"], rho["cond"])
        r = bw._ratio((ours - ref).abs(), bar)[~rho["needle"]]
        return float(r.max()) if r.numel() else 0.0

    def features(self, feat):
        P = self.ref6.shape[0]
        return self.Wt.per_gaussian(feat.reshape(P, -1), self.Gf) if self.Gf.shape[1] else 0.0

    def accumulated(self, o, rho=None):
        """The accumulating entry's own outputs, accumulated into zeros: dL_dopacity, dL_dmean2D_out (every term of
        the composite's dL/dmean2D), grad_accum (|dL/dmean2D.xy| of the full model: the model's bars and the sqrt's
        and the add's rounding) and denom."""
        ref, bar = self.ref6.cpu(), self.bar6.cpu()
        m2 = o["mean2D"].cpu().double()
        assert bool((m2[:, 2] == 0).all())
        worst = {"dL_dopacity": self.opacity(o["opacity"], rho),
                 "dL_dmean2D_out": float(bw._ratio((m2[:, :2] - ref[:, :2]).abs(), bar[:, :2]).max())}
        n = ref[:, :2].norm(dim=1)
        gbar = bar[:, :2].sum(1) + 2 * bw.U * n
        worst["grad_accum"] = float(bw._ratio((o["grad_accum"].cpu().double().reshape(-1) - n).abs(), gbar).max())
        return worst


def _inputs(v, ups, feat, mp):
    """(feature rows or None, map gradient tensor, map scale or None) of one cell"""
    dev = torch.device("cuda")
    sf = None if feat == "none" else (v.feats if feat == "f32" else v.feats.half())
    gf = _t(ups[1], dev)
    return (sf, gf, None) if mp == "f32" else (sf, (gf / S16).half(), S16)


def _zeros_accum(v, camera):
    z = lambda *s: torch.zeros(*s, device="cuda")  # noqa: E731
    o = dict(opacity=z(v.P), feat=z(v.P, v.C), means3D=z(v.P, 3), sh=z(v.P, max(v.M, 1), 3), scales=z(v.P, 3),
             rotations=z(v.P, 4), mean2D=z(v.P, 3), grad_accum=z(v.P), denom=z(v.P), colors=z(v.P, 3),
             cov3D=z(v.P, 6))
    if camera:
        o["camera"] = z(35)
    return o


def check_view(lib, v, label, cells, ups_all):
    """Every cell (feat, map, camera, entry) of `cells` on the View v under each upstream gradient -> worst ratio per
    tensor over them (each cell's own are printed and asserted)."""
    aa = v.antialiasing
    vis = v.visible
    idx = vis.nonzero().flatten()
    rho = rho_model(v.sc, v.cam, idx, v.mod, v.cov.cpu() if v.cov.numel() else None) if aa else None
    worst_all = {}
    for i, (ulabel, ups) in enumerate(ups_all):
        ga, gi = _plane_grads(v.H, v.W, 90 + i, dynamic=ulabel == "dynamic range")
        for (feat, mp), group in itertools.groupby(cells, key=lambda c: c[:2]):
            sf, gmap, scale = _inputs(v, ups, feat, mp)
            R = Reference(v, ups, ga, gi, sf, gmap, scale)
            call = functools.partial(_backward_planes, lib, v, (ups[0], gmap, ups[2]), ga, gi, sf=sf, aa=int(aa),
                                     map_scale=scale)
            g_eff = None
            for _, _, camera, entry in group:
                tag = f"{label} aa={int(aa)} feat={feat} map={mp} camera={int(camera)} {entry} {ulabel}"
                if entry == "assign":
                    o = call(camera=camera)
                    worst = R.composite(o, rho)
                    worst["dL_dfeature"] = R.features(o["feat"])
                    mids = {k: o[k] for k in ("mean2D", "conic", "color", "dz")}
                    if aa:
                        if g_eff is None:  # dL/dop_eff: the composite's opacity output with antialiasing off
                            g_eff = call(aa=0)["opacity"]
                            worst["dL_dop_eff"] = R.opacity(g_eff)
                        m = model_gradients(v.sc, v.cam, [mids["mean2D"].cpu(), mids["conic"].cpu(), g_eff.cpu(),
                                                          mids["color"].cpu(), mids["dz"].cpu()], idx, mod=v.mod,
                                            cov=v.cov.cpu() if v.cov.numel() else None,
                                            colors=v.cols.cpu() if v.cols.numel() else None)
                        worst.update(aa_preprocess_check(v, m, o))
                        if v.M:
                            ch = v.chain(o)
                            worst.update(preprocess_check({k: ch[k] for k in ("sh", "mag_sh", "eig_ratio")},
                                                          {"sh": o["sh"]}, vis))
                    else:
                        m = None
                        worst.update(preprocess_check(v.chain(o), v.outputs(o), vis))
                    if camera:
                        cref, cbar = camera_reference(v, mids, m)
                        worst["dL_dcamera"] = float(((o["camera"].cpu().double() - cref).abs() / cbar).max())
                    last_assign = (mids, m)
                else:
                    o = call(camera=camera, accum=_zeros_accum(v, camera))
                    worst = R.accumulated(o, rho)
                    worst["dL_dfeature"] = R.features(o["feat"])
                    assert torch.equal(o["denom"].cpu(), vis.float()), tag
                    if camera:  # on the assigning call's intermediates (cells sort assign before accum)
                        cref, cbar = camera_reference(v, *last_assign)
                        worst["dL_dcamera"] = float(((o["camera"].cpu().double() - cref).abs() / cbar).max())
                _report(tag, worst)
                for k, x in worst.items():
                    worst_all[k] = max(worst_all.get(k, 0.0), x)
    return worst_all


def _groups(cells):
    """cells grouped by (feat, map), each group's assigning cells first: the accumulating entry's camera check reads the
    assigning call's intermediates"""
    return sorted(cells, key=lambda c: (c[0], c[1], c[3] == "accum", c[2]))


ALL_CELLS = _groups(itertools.product(FEATS, MAPS, (False, True), ("assign", "accum")))


# -------------------------------------------------------------------------------------------- CPU: negative controls
def test_negative_controls_flag_each_dropped_term():
    """On the oracle view, the float64 model with exactly one term removed exceeds the full model's bar for at least one
    Gaussian: the feature dot, gA, gI / z, -w gI / z^2 in dL/dz, rho in dL_dopacity, rho's conic term, and the gI term
    of the camera gradient."""
    from test_blend_weights import _oracle_view

    sc, cam, f, pairs, w = _oracle_view("small")
    rec = _t(bw.oracle_records(f))
    H, W, P, C = cam.image_height, cam.image_width, sc.P, sc.C
    gc, gf, gd = bw.upstream(H, W, C, 5)
    ga, gi = _plane_grads(H, W, 6)
    Gc, Gd, GA, GI = _t(gc).reshape(3, -1).t(), _t(gd).reshape(-1), _t(ga).reshape(-1), _t(gi).reshape(-1)
    Gf = _t(gf).reshape(C, -1).t()
    F = _t(sc.features).reshape(P, C)
    bg = torch.tensor(sc.bg)
    ref, bar = planes_model(pairs, w, rec, P, bg, Gc, Gd, GA, GI, F=F, Gf=Gf)
    ratios = {}

    def flagged(label, x, r, b):
        ratios[label] = float(bw._ratio((x - r).abs(), b).max())

    flagged("feature dot", planes_model(pairs, w, rec, P, bg, Gc, Gd, GA, GI)[0], ref, bar)
    flagged("gA", planes_model(pairs, w, rec, P, bg, Gc, Gd, torch.zeros_like(GA), GI, F=F, Gf=Gf)[0], ref, bar)
    flagged("gI / z", planes_model(pairs, w, rec, P, bg, Gc, Gd, GA, torch.zeros_like(GI), F=F, Gf=Gf)[0], ref, bar)
    Wt = bw.Weights(pairs, w, P)
    rz, _, _ = Wt.terms(Gd.reshape(-1, 1))
    ratios["-w gI / z^2 in dL/dz"] = dz_check(Wt, rec, rz.float().reshape(-1), Gd, GI)
    # the composite's intermediates of the full model, in float64
    r2, _, _ = Wt.terms(GI.reshape(-1, 1))
    z = rec[:, 11].double().reshape(-1, 1)
    iz2 = torch.where(z > 0, 1.0 / (z * z), torch.zeros_like(z))
    dz = (rz - r2 * iz2).reshape(-1)
    color, _, _ = Wt.terms(Gc)
    zero = torch.zeros(P, dtype=torch.float64)
    mean2D = torch.stack([ref[:, 0], ref[:, 1], zero], 1)
    conic = torch.stack([ref[:, 2], ref[:, 3], zero, ref[:, 4]], 1)
    g = ref[:, 5]
    vis = torch.as_tensor(f["radii"] > 0)
    idx = vis.nonzero().flatten()
    # rho in dL_dopacity: g itself against rho g
    rho = rho_model(sc, cam, idx)
    r_op, b_op = rho_opacity(g, bar[:, 5], rho["rho"], rho["cond"])
    ratios["rho in dL_dopacity"] = float(bw._ratio((g - r_op).abs(), b_op)[~rho["needle"]].max())
    # rho's conic term: the model with g = 0 in op_eff's gradient leaves only the terms that do not pass through rho
    m = model_gradients(sc, cam, [mean2D, conic, g, color, dz], idx)
    m0 = model_gradients(sc, cam, [mean2D, conic, zero, color, dz], idx)
    well = m["eig_ratio"] <= NEEDLE_COND_MAX
    k = m["kappa"].clamp_min(1.0)
    r_conic = 0.0
    for key in ("means3D", "scales", "rotations"):
        floor = 1e-6 * float(m[key][well].abs().max()) + 1e-12
        b = AA_BAR * k[:, None] * m[key].abs().sum(1, keepdim=True) + floor
        r_conic = max(r_conic, float(((m0[key] - m[key]).abs() / b)[well].max()))
    ratios["rho's conic term"] = r_conic
    # the gI term of the camera gradient: dL/dz without it, through camera_grad_model.terms
    cov = cgm.cov3d_from_scale_rot(_t(sc.scales).double(), _t(sc.rotations).double())
    vm, pm, cp = (torch.as_tensor(a).double() for a in (cam.viewmatrix, cam.projmatrix, cam.campos))

    def cam_terms(dz_):
        return cgm.terms(sc.means3D, cov, vm, pm, cp, [mean2D, conic, color, dz_], W, H, cam.tanfovx, cam.tanfovy,
                         sc.sh_degree, shs=sc.shs, visible=vis)

    t = cam_terms(dz)
    cbar = 1e-5 * cgm.camera_scale(t) + 1e-7 * float(cgm.camera_scale(t, needles=False).max())
    ratios["gI term of the camera gradient"] = float(((cgm.camera_vector(cam_terms(rz.reshape(-1)))
                                                       - cgm.camera_vector(t)).abs() / cbar).max())
    print("[negative controls] " + ", ".join(f"{k}={v:.3g}" for k, v in ratios.items()))
    for label, r in ratios.items():
        assert r > 1.0, (label, r)


# -------------------------------------------------------------------------------------------- GPU: against the model
@functools.lru_cache(maxsize=2)
def _options_view(name, aa):
    """The View of a scene for this file: the planes forward with antialiasing aa"""
    kw = {}
    C = 8
    if name == "inside fx!=fy":
        from test_feature_geometry import _identity_scene
        from test_blend_weights import BG

        sc, cam = _identity_scene("fx_ne_fy")
        sc.bg = BG.copy()
        kw = dict(mod=1.3)
    elif name == "precomputed":
        sc, cam, kw = _scene("cov3D_precomp")
        kw["cols"] = torch.rand(sc.P, 3, generator=torch.Generator().manual_seed(8))
    elif name == "C=200":
        sc, cam, kw = _scene("small")
        C = 200
    else:
        sc, cam, kw = _scene(name)
    return View(sc, cam, C=C, planes=True, antialiasing=aa, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("aa", [False, True])
def test_every_cell_on_small(lib, aa):
    """The 48 cells of one antialiasing mode on `small` at C = 8, under the three upstream gradients."""
    v = _options_view("small", aa)
    worst = check_view(lib, v, "small", _groups(ALL_CELLS), _upstreams(v.H, v.W, v.C, 71))
    print(f"[small aa={int(aa)}] worst over the cells: " + ", ".join(f"{k}={x:.3g}" for k, x in worst.items()))


HARD = ["needles", "inside fx!=fy", "layers129", "C=200", "precomputed", "deg0", "deg3"]
CORNERS = _groups([(feat, "f16", True, e) for feat in ("f16", "none") for e in ("assign", "accum")])


@pytest.mark.gpu
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("name", HARD)
def test_all_on_corners_on_hard_scenes(lib, name, aa):
    """Every option on (float16 rows, float16 map, camera, both entries), and the same without the feature term."""
    v = _options_view(name, aa)
    worst = check_view(lib, v, name, CORNERS, _upstreams(v.H, v.W, v.C, 81))
    print(f"[{name} aa={int(aa)}] worst over the cells: " + ", ".join(f"{k}={x:.3g}" for k, x in worst.items()))


# ------------------------------------------------------------------------------------ GPU: exact identities, block scene
def _block_view(aa):
    from test_alpha_invdepth import _block

    sc, cam = _block()
    return View(sc, cam, planes=True, antialiasing=aa, weights=False)


ACCUM_KEYS = ("opacity", "feat", "means3D", "sh", "scales", "rotations", "mean2D", "camera")


@pytest.mark.gpu
@pytest.mark.parametrize("aa", [False, True])
def test_exact_identities_on_the_block_scene(lib, aa):
    """Every cell: accumulating into zeros gives the assigning entry's bits; into a nonzero prior fl(prior + the single
    view); the camera leaves every other output unchanged; float16 rows give the bits of their float32 upcast, and a
    float16 map h at scale s those of the float32 map fl(s float(h))."""
    v = _block_view(aa)
    dev = torch.device("cuda")
    ups = bw.upstream(v.H, v.W, v.C, 13)
    ga, gi = _plane_grads(v.H, v.W, 14)
    gf = _t(ups[1], dev)
    h = (gf / S16).half()
    rows = dict(none=None, f32=v.feats, f16=v.feats.half(), f16up=v.feats.half().float())
    maps = dict(f32=(gf, None), f16=(h, S16), f16up=(h.float() * S16, None))
    gen = torch.Generator().manual_seed(15)
    cache = {}

    def run(feat, mp, camera, entry, prior=None):
        key = (feat, mp, camera, entry, prior is not None)
        if key not in cache:
            gmap, scale = maps[mp]
            acc = None
            if entry == "accum":
                acc = _zeros_accum(v, camera) if prior is None else {k: x.clone() for k, x in prior.items()}
            cache[key] = _backward_planes(lib, v, (ups[0], gmap, ups[2]), ga, gi, sf=rows[feat], aa=int(aa),
                                          map_scale=scale, camera=camera, accum=acc)
        return cache[key]

    def same(a, b, keys, label):
        for k in keys:
            assert torch.equal(a[k], b[k]), (label, k)

    assign_keys = ("mean2D", "conic", "opacity", "color", "feat", "means3D", "cov3D", "sh", "scales", "rotations", "dz")
    accum_keys = ("opacity", "feat", "means3D", "sh", "scales", "rotations", "mean2D", "grad_accum", "denom")
    for feat, mp, camera in itertools.product(FEATS, MAPS, (False, True)):
        a = run(feat, mp, camera, "assign")
        z = run(feat, mp, camera, "accum")
        label = (aa, feat, mp, camera)
        same(a, z, [k for k in ACCUM_KEYS if camera or k != "camera"], label + ("accum into zeros",))
        assert bool(a["opacity"].abs().sum() > 0)
        # a nonzero prior: every output is fl(prior + the single view)
        prior = {k: torch.randn(x.shape, generator=gen).to(dev) for k, x in z.items()}
        prior["denom"] = torch.randint(0, 5, z["denom"].shape, generator=gen).float().to(dev)
        prior["grad_accum"] = prior["grad_accum"].abs()
        p = run(feat, mp, camera, "accum", prior)
        # dL_dopacity is added in more than one step: without antialiasing, by the geometry walk (its value is the
        # call's without the feature term) and again by the feature term's kernels, two roundings; with it, the
        # preprocess adds rho g to the prior in one FMA, one rounding of the exact product
        steps = dict(opacity=1 if aa else (2 if feat != "none" else 0))
        for k in z:  # dL_dmean2D_out is the view's own, assigned
            want = z[k] if k == "mean2D" else prior[k] + z[k]
            if steps.get(k, 0) and not torch.equal(p[k], want):
                x, y = prior[k].double(), z[k].double()
                walk = run("none", mp, camera, "accum")[k].double() if steps[k] == 2 else torch.zeros_like(y)
                bar = steps[k] * bw.U * ((x + y).abs() + x.abs() + y.abs() + walk.abs())
                assert bool(((p[k].double() - (x + y)).abs() <= bar).all()), label + ("prior", k, steps[k])
            else:
                assert torch.equal(p[k], want), label + ("prior", k)
        if camera:
            same(a, run(feat, mp, False, "assign"), assign_keys, label + ("camera",))
            same(z, run(feat, mp, False, "accum"), accum_keys, label + ("camera, accum",))
            assert bool(a["camera"].abs().sum() > 0)
        for entry in ("assign", "accum"):
            keys = [k for k in (assign_keys if entry == "assign" else accum_keys + ("camera",)) if camera or
                    k != "camera"]
            o = run(feat, mp, camera, entry)
            if feat == "f16":
                same(o, run("f16up", mp, camera, entry), keys, label + (entry, "float16 rows"))
            if mp == "f16":
                same(o, run(feat, "f16up", camera, entry), keys, label + (entry, "float16 map"))
    # the options change what they should: the feature term moves dL_dopacity, the float16 map is not the float32 one
    assert not torch.equal(run("f32", "f32", False, "assign")["opacity"], run("none", "f32", False, "assign")["opacity"])
    assert not torch.equal(run("none", "f16", False, "assign")["feat"], run("none", "f32", False, "assign")["feat"])


# ---------------------------------------------------------------------------- GPU: the Python surfaces, block scene
@pytest.mark.gpu
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("half_rows", [False, True])
def test_view_batch_is_the_c_entry(lib, aa, half_rows):
    """ViewBatch.backward for every combination of camera, feature_geometry, a ScaledGrad or float32 g_feature and
    g_alpha / g_invdepth (both, one, none): bitwise the direct accumulating C call into zeros (with a plane gradient it
    does not get set to zero, which gives the call without the planes' bits)."""
    from diff_gaussian_rasterization.feature_head import ScaledGrad
    from diff_gaussian_rasterization.parallel import ViewBatch
    from test_alpha_invdepth import _settings

    v = _block_view(aa)
    dev = torch.device("cuda")
    sf = v.feats.half() if half_rows else v.feats
    params = dict(means3D=v.d["means3D"], scales=v.d["scales"], rotations=v.d["rotations"],
                  opacities=v.d["opacities"], shs=v.d["shs"], semantic_feature=sf)
    rs = _settings(v.sc, v.cam)
    gc, gf, gd = (_t(u, dev) for u in bw.upstream(v.H, v.W, v.C, 21))
    ga, gi = (_t(x, dev) for x in _plane_grads(v.H, v.W, 22))
    zero = torch.zeros_like(ga)
    h = (gf / S16).half()
    for camera, fg, scaled, planes in itertools.product((False, True), (False, True), (False, True),
                                                        ("both", "alpha", "invdepth", "none")):
        label = (aa, half_rows, camera, fg, scaled, planes)
        vb = ViewBatch(params)
        *_, ctx = vb.forward_alpha_invdepth(rs, antialiasing=aa)
        assert ctx.antialiasing == aa
        kw = dict(g_alpha=ga if planes in ("both", "alpha") else None,
                  g_invdepth=gi if planes in ("both", "invdepth") else None)
        cg = vb.backward(ctx, gc, ScaledGrad(h, S16) if scaled else gf, gd, camera=camera, feature_geometry=fg, **kw)
        pa, pi = (x if x is not None else zero for x in (kw["g_alpha"], kw["g_invdepth"]))
        o = _backward_planes(lib, v, (gc, h if scaled else gf, gd), pa, pi, sf=sf if fg else None, aa=int(aa),
                             map_scale=S16 if scaled else None, camera=camera, accum=_zeros_accum(v, camera))
        for key, k in (("opacities", "opacity"), ("semantic_feature", "feat"), ("means3D", "means3D"),
                       ("shs", "sh"), ("scales", "scales"), ("rotations", "rotations")):
            assert torch.equal(vb.grads[key].reshape(o[k].shape), o[k]), label + (key,)
        assert torch.equal(vb.grad_accum, o["grad_accum"]) and torch.equal(vb.denom, o["denom"]), label
        if camera:
            got = torch.cat([cg.viewmatrix.reshape(-1), cg.projmatrix.reshape(-1), cg.campos])
            assert torch.equal(got, o["camera"]), label
        else:
            assert cg is None
