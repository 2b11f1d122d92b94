"""The composite against its own blend weights W[g, p] = alpha_gp * T_gp (see blend_weights.py for the extraction, the
float64 model and the bars).

parity's bars scale their absolute floor with the largest entry of the whole tensor, so a Gaussian whose gradient is small
can be entirely wrong under them: a lost or doubled (Gaussian, pixel) term in a tile or block list.  Most of the
composite is linear in W, and each linear output is checked here per pixel and per Gaussian, with a bar made of that
entry's own terms:
    colour   color[:, p] = sum_g w_gp c_g + T_final_p bg          depth   depth_p = sum_g w_gp z_g
    T        1 - sum_g w_gp = T_final_p                           map     F[:, p] = sum_g w_gp f_g
    dL/dcolor_g, dL/dz_g, dL/dfeature_g = sum_p w_gp dL/d(pixel, depth, map)_p
    lift     weight_sum_g = sum_p w_gp,  feature_sum_g = sum_p w_gp map[:, p]
The nonlinear gradients (means2D, conic, opacity and what flows from them) stay under parity's bars.

CPU (`-m "not gpu"`): the checker on the CPU oracle, and negative controls: perturbations of the oracle's outputs that
parity's bar passes and this checker flags.
GPU: W is bitwise the same at every feature width; every weight of every scene passes the float64 model; every identity
holds for float32 and float16 maps and features, through the torch binding, the C ABI, ViewBatch and the lift.  The worst
ratio |err| / bar of every tensor is printed.
"""
import copy
import functools
import os

import numpy as np
import pytest
import torch

import blend_weights as bw
import parity
import scenegen

BG = np.array([0.3, 0.6, 0.9], np.float32)  # a non-zero background: the colour identity carries T_final * bg


def _t(a, dev="cpu"):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _report(label, worst):
    print(f"[{label}] worst |err|/bar: " + ", ".join(f"{k}={v:.3g}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v <= 1.0, (label, k, v)


def _model(label, pairs, w, rec, final_T):
    rep = bw.check_model(pairs, w, rec, final_T)
    counts = {k: v for k, v in rep.items() if k.startswith(("bad_", "n_", "ambiguous"))}
    print(f"[{label}] model: weight={rep['weight']:.3g} final_T={rep['final_T']:.3g} {counts}")
    assert rep["ok"], (label, {k: v for k, v in rep.items() if k != "rho"})
    assert rep["n_blended"] > 0
    return rep


def _forward_identities(Wt, label, color, depth, final_T, bg, rec, fmap=None, feats=None):
    HW = Wt.HW
    T = final_T.reshape(HW, 1).double()
    bg = bg.double().reshape(1, 3)
    worst = dict(color=Wt.per_pixel(color.reshape(3, HW).t(), rec[:, 8:11], T * bg, T * bg.abs()),
                 depth=Wt.per_pixel(depth.reshape(1, HW).t(), rec[:, 11:12]),
                 T=Wt.per_pixel(1 - T, torch.ones_like(rec[:, :1]), torch.zeros_like(T), T))
    if fmap is not None:
        C = fmap.shape[0]
        key = "feature_map_f16" if fmap.dtype == torch.float16 else "feature_map"
        worst[key] = Wt.per_pixel(fmap.reshape(C, HW).t(), feats.reshape(-1, C))
    _report(label, worst)


def test_half_rounding_covers_every_float16_rounding():
    """blend_weights.half_rounding: x is within it of x.half(), for normals, subnormals and both sides of powers of two,
    and it is no wider than the half spacing."""
    rng = np.random.default_rng(0)
    mags = 2.0 ** rng.uniform(-27, 15, 200000)
    x = torch.from_numpy(np.concatenate([mags, -mags, 2.0 ** np.arange(-24, 15), 2.0 ** np.arange(-24, 15) * 0.99999,
                                         [0.0, 2.0 ** -26, -2.0 ** -26]]).astype(np.float32))
    y = x.half().double()
    x = x.double()
    h = bw.half_rounding(y, x)
    assert bool(((x - y).abs() <= h).all())
    assert bool((h <= torch.clamp(y.abs(), min=2.0 ** -14) * 2.0 ** -11).all())


# ============================================================================================== CPU: the checker checked
@functools.lru_cache(maxsize=None)
def _oracle_view(name):
    import oracle

    oracle.set_threads(os.cpu_count())
    sc = scenegen.make_config(name)
    sc.bg = BG.copy()
    cam = sc.cameras[0]
    W, H = cam.image_width, cam.image_height
    f = oracle.forward(sc, cam)
    pairs = bw.Pairs(_t(f["point_list"].astype(np.int64)), _t(f["ranges"].astype(np.int64)),
                     _t(f["n_contrib"].astype(np.int64)), W, H)

    def render(g0, C):
        one = copy.copy(sc)
        one.features = np.zeros((sc.P, 1, C), np.float32)
        one.features[g0:g0 + C, 0, :] = np.eye(C, dtype=np.float32)
        return _t(oracle.forward(one, cam)["feature_map"].reshape(C, -1))

    w = bw.extract(pairs, sc.P, render, 1000)
    return sc, cam, f, pairs, w


def _oracle_grads(sc, cam, f, ups):
    import oracle

    return oracle.backward(sc, cam, f, *ups)


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_checker_passes_on_the_oracle(name):
    sc, cam, f, pairs, w = _oracle_view(name)
    H, W, P, C = cam.image_height, cam.image_width, sc.P, sc.C
    rec = _t(bw.oracle_records(f))
    _model(f"oracle {name}", pairs, w, rec, _t(f["final_T"]))
    Wt = bw.Weights(pairs, w, P)
    _forward_identities(Wt, f"oracle {name} forward", _t(f["color"]), _t(f["depth"]), _t(f["final_T"]), _t(sc.bg),
                        rec.double(), _t(f["feature_map"]), _t(sc.features))
    for label, ups in (("upstream_grads", scenegen.upstream_grads(H, W, C)), ("N(0,1)", bw.upstream(H, W, C, 5)),
                       ("dynamic range", bw.upstream(H, W, C, 6, dynamic=True))):
        g = _oracle_grads(sc, cam, f, ups)
        gc, gf, gd = (_t(u.reshape(u.shape[0], -1)).t() for u in ups)
        _report(f"oracle {name} backward {label}",
                dict(dL_dcolors=Wt.per_gaussian(_t(g["colors"]), gc),
                     dL_dsemantic_feature=Wt.per_gaussian(_t(g["semantic_feature"].reshape(P, C)), gf),
                     dL_dz=Wt.per_gaussian(_t(g["dz"].reshape(P, 1)), gd)))


def test_negative_controls_pass_the_parity_bar_and_fail_the_checker():
    """Perturbations of the oracle's feature gradient for a Gaussian whose whole gradient row lies under parity's floor
    (5e-5 of the largest entry of the tensor), and of one blend weight early in its pixel's list.  parity's bar passes
    every one; this checker flags every one."""
    sc, cam, f, pairs, w = _oracle_view("small")
    H, W, P, C = cam.image_height, cam.image_width, sc.P, sc.C
    ups = scenegen.upstream_grads(H, W, C)
    g = _oracle_grads(sc, cam, f, ups)
    ours = g["semantic_feature"].reshape(P, C).astype(np.float64)
    G = _t(ups[1].reshape(C, -1)).t()
    Wt = bw.Weights(pairs, w, P)

    def ratio(x):
        return Wt.per_gaussian(_t(x), G)

    def parity_passes(x):
        return parity.float_mismatch(x, ours, parity.RTOL, parity.GRAD_ATOL_REL)[0] <= 1.0

    base = ratio(ours)
    assert base <= 1.0
    rowmax = np.abs(ours).max(1)
    under = np.nonzero((rowmax < parity.GRAD_ATOL_REL * np.abs(ours).max()) & (rowmax > 0))[0]
    assert under.size > 50  # the gap: whole rows the floor hides
    gq = int(under[under.size // 2])
    sel = (pairs.gid[pairs.widx] == gq) & (w > 0)
    pix = pairs.pix[pairs.widx][sel]
    terms = (w[sel].double()[:, None] * G[pix]).numpy()  # [pixels, C]: w * dL/dF of each pixel gq blends
    med = int(np.argsort(np.abs(terms).sum(1))[pix.numel() // 2])
    p0 = int(pix[med])
    bx, by = (p0 % W) // 8 * 8, (p0 // W) // 4 * 4  # the 8x4 pixel block of that pixel
    block = ((pix % W) // 8 * 8 == bx) & ((pix // W) // 4 * 4 == by)
    controls = {"(a) one (g, p) term dropped": -terms[med], "(b) one block list entry counted twice":
                terms[block.numpy()].sum(0), "(c) the whole row zeroed": -ours[gq]}
    flagged = {}
    for label, d in controls.items():
        x = ours.copy()
        x[gq] += d
        assert parity_passes(x), label
        flagged[label] = ratio(x)
    print(f"[negative controls, Gaussian {gq}, {pix.numel()} pixels] unperturbed {base:.3g}; perturbed: "
          + ", ".join(f"{k}={v:.3g}" for k, v in flagged.items()))
    for label, r in flagged.items():
        assert r > 1.0, (label, r)
    # (d) one weight scaled by 1 + 1e-4: the float64 model flags it.  The weight is early in its pixel's list, where the
    # model's bar (its position term) is far below 1e-4; the same change of the feature map passes parity's bar.
    rec = _t(bw.oracle_records(f))
    rep = bw.check_model(pairs, w, rec, _t(f["final_T"]))
    assert rep["ok"]
    pos = pairs.pos[pairs.widx]
    cand = torch.nonzero((w > 0) & (pos < 100) & (rep["rho"] < 1e-5)).reshape(-1)
    assert cand.numel() > 0
    i = int(cand[torch.argmax(w[cand])])
    w2 = w.clone()
    w2[i] = w[i] * np.float32(1 + 1e-4)
    rep2 = bw.check_model(pairs, w2, rec, _t(f["final_T"]))
    gi, pi = int(pairs.gid[pairs.widx][i]), int(pairs.pix[pairs.widx][i])
    fmap = f["feature_map"].reshape(C, -1).astype(np.float64)
    fmap2 = fmap.copy()
    fmap2[:, pi] += (float(w2[i]) - float(w[i])) * sc.features[gi, 0].astype(np.float64)
    assert parity.float_mismatch(fmap2, fmap, parity.RTOL, parity.ATOL_REL)[0] <= 1.0
    print(f"[negative control (d): weight at list position {int(pos[i])}, model bar {float(rep['rho'][i]):.3g}] "
          f"model ratio {rep2['weight']:.3g}")
    assert not rep2["ok"] and rep2["weight"] > 1.0


# ============================================================================================== GPU
def _forward(t, rs, sf):
    from diff_gaussian_rasterization import _C

    e = torch.Tensor([])
    R, color, feat, depth, radii, geom, binning, img = _C.rasterize_gaussians(
        rs["bg"], t["means3D"], e, sf, t["opacities"], t["scales"], t["rotations"], rs["scale_modifier"], e,
        rs["viewmatrix"], rs["projmatrix"], rs["tanfovx"], rs["tanfovy"], rs["image_height"], rs["image_width"],
        t["shs"], rs["sh_degree"], rs["campos"], rs["prefiltered"], False)
    pl, ranges, n_contrib, final_T, rec = _C.debug_views(geom, binning, img, t["means3D"].shape[0], rs["image_width"],
                                                         rs["image_height"], R)
    return dict(R=R, color=color, feature_map=feat, depth=depth, radii=radii, geom=geom, binning=binning, img=img,
                point_list=pl, ranges=ranges, n_contrib=n_contrib, final_T=final_T, rec=rec)


class DeviceView:
    """One view of a scene on the device: the forward of the scene's own features, its pairs and the extracted W."""

    def __init__(self, sc, cam, group):
        self.sc, self.cam = sc, cam
        self.t = scenegen.to_torch(sc, "cuda")
        self.rs = parity.settings(sc, cam, "cuda")
        self.P, self.W, self.H = sc.P, cam.image_width, cam.image_height
        self.base = _forward(self.t, self.rs, self.t["semantic_feature"])
        b = self.base
        self.pairs = bw.Pairs(b["point_list"], b["ranges"], b["n_contrib"], self.W, self.H)
        self.w = self.weights(group)
        self.Wt = bw.Weights(self.pairs, self.w, self.P)

    def forward(self, sf):
        """A forward with other features: the same geometry, so the same walk."""
        r = _forward(self.t, self.rs, sf)
        for k in ("color", "n_contrib", "final_T", "point_list"):
            assert torch.equal(r[k], self.base[k]), k
        return r

    def weights(self, group):
        def render(g0, C):
            sf = torch.zeros(self.P, 1, C, device="cuda")
            sf[g0:g0 + C, 0, :] = torch.eye(C, device="cuda")
            return self.forward(sf)["feature_map"].reshape(C, -1)

        return bw.extract(self.pairs, self.P, render, group)


# scene builders: the ones the suite already uses to reach the composite's edges
def _layers(n, W, H, **kw):
    from test_producer_prefetch import _layers as layers

    return layers(n, W, H, 16, **kw)


def _halves(W, H, radius):
    from test_fwd_feature_halves import _scene

    sc = _scene(W, H, 16, radius)
    return sc, sc.cameras[0]


def _regime(name):
    from test_gpu_regimes import make

    return make(name, 16)


def _cfg(name):
    sc = scenegen.make_config(name)
    return sc, sc.cameras[0]


def _made(**kw):
    sc = scenegen.make_scene(**kw)
    return sc, sc.cameras[0]


SCENES = {
    "tiny": lambda: _cfg("tiny"), "small": lambda: _cfg("small"), "small128": lambda: _cfg("small128"),
    "small200": lambda: _cfg("small200"),
    **{f"layers{n}": functools.partial(_layers, n, 96, 64) for n in (1, 31, 32, 33, 127, 128, 129)},
    "checkerboard": lambda: _layers(70, 128, 64, skip=lambda tx, ty: (tx + ty) % 2 == 1),
    "opaque": lambda: _layers(200, 96, 64, opaque=True),
    "one_tile": lambda: _layers(150, 16, 16), "few_tiles": lambda: _layers(150, 40, 24),
    **{f"halves{W}x{H}": functools.partial(_halves, W, H, r) for W, H, r in
       [(96, 61, 6.0), (96, 62, 6.0), (96, 63, 1.5), (92, 45, 6.0), (97, 38, 1.5)]},
    "inside": lambda: _regime("inside"), "needles": lambda: _regime("needles"), "plane": lambda: _regime("plane"),
    # test_gpu_parity.test_huge_splats_cover_many_tiles
    "huge": functools.partial(_made, P=300, W=320, H=240, C=16, sh_degree=1, seed=6, target_radius_px=120.0),
    # past the oracle's comfortable size, extracted in groups of 4096 Gaussians
    "medium": functools.partial(_made, P=40000, W=320, H=240, C=16, sh_degree=2, seed=61),
}
GROUP = {"medium": 4096}


@functools.lru_cache(maxsize=4)
def _view(name):
    sc, cam = SCENES[name]()
    sc.bg = BG.copy()
    return DeviceView(sc, cam, GROUP.get(name, 512))


def _feats(P, C, seed, dtype=torch.float32):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(P, 1, C, device="cuda", generator=g).to(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "layers129", "halves97x38", "needles"])
def test_weights_are_bitwise_the_same_at_every_feature_width(name):
    """The alpha warps do not depend on the feature width, the kernel instantiation or the channel chunk: W read through
    32, 64, 128, 129 and 513 channels is one W."""
    v = _view(name)
    for C in (32, 64, 128, 129, 513):
        assert torch.equal(v.weights(C).view(torch.int32), v.w.view(torch.int32)), C


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SCENES))
def test_weights_match_the_float64_model(name):
    v = _view(name)
    _model(f"{name} V={int((v.base['radii'] > 0).sum())} R={v.base['R']}", v.pairs, v.w, v.base["rec"],
           v.base["final_T"])


# (scene, feature width) for the identities: every width the composite instantiates or chunks differently
IDENTITY_CASES = [("tiny", 3), ("small", 1), ("small", 16), ("small", 4096), ("small128", 128), ("small200", 200),
                  ("layers1", 16), ("layers31", 33), ("layers32", 32), ("layers33", 33), ("layers127", 64),
                  ("layers128", 128), ("layers129", 129), ("checkerboard", 64), ("opaque", 32), ("one_tile", 1),
                  ("few_tiles", 3), ("halves96x61", 33), ("halves96x62", 64), ("halves96x63", 129),
                  ("halves92x45", 1), ("halves97x38", 513), ("inside", 16), ("needles", 128), ("plane", 3),
                  ("huge", 32), ("medium", 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,C", IDENTITY_CASES)
def test_forward_identities_per_pixel(name, C):
    v = _view(name)
    rec = v.base["rec"].double()
    for dt in (torch.float32, torch.float16):
        f = _feats(v.P, C, seed=C, dtype=dt)
        r = v.forward(f)
        assert r["feature_map"].dtype == dt
        _forward_identities(v.Wt, f"{name} C={C} {dt}", r["color"], r["depth"], r["final_T"], v.rs["bg"], rec,
                            r["feature_map"], f.float())


@pytest.mark.gpu
@pytest.mark.parametrize("name,C", IDENTITY_CASES)
def test_backward_identities_per_gaussian(name, C):
    from diff_gaussian_rasterization import _C

    v = _view(name)
    t, rs, P, H, W = v.t, v.rs, v.P, v.H, v.W
    sf = _feats(P, C, seed=C + 1)
    r = v.forward(sf)
    e = torch.Tensor([])
    for label, ups in (("upstream_grads", scenegen.upstream_grads(H, W, C)), ("N(0,1)", bw.upstream(H, W, C, 7)),
                       ("dynamic range", bw.upstream(H, W, C, 8, dynamic=True))):
        gc, gf, gd = (_t(u, "cuda") for u in ups)
        g = _C.rasterize_gaussians_backward(rs["bg"], t["means3D"], r["radii"], e, sf, t["scales"], t["rotations"],
                                            rs["scale_modifier"], e, rs["viewmatrix"], rs["projmatrix"], rs["tanfovx"],
                                            rs["tanfovy"], gc, gf, gd, t["shs"], rs["sh_degree"], rs["campos"],
                                            r["geom"], r["R"], r["binning"], r["img"], False)
        _report(f"{name} C={C} backward {label}",
                dict(dL_dcolors=v.Wt.per_gaussian(g[1], gc.reshape(3, -1).t()),
                     dL_dsemantic_feature=v.Wt.per_gaussian(g[2].reshape(P, C), gf.reshape(C, -1).t())))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "needles", "layers129", "opaque"])
def test_depth_gradient_through_the_c_abi(built, name):
    """f3dgs_backward returns dL/dz, the composite's per-Gaussian depth gradient, as a scratch output."""
    import ctypes

    import test_cabi_gpu as cabi

    v = _view(name)
    sc, cam = v.sc, v.cam
    P, C, W, H, M = sc.P, sc.C, v.W, v.H, sc.shs.shape[1]
    rt = cabi._cudart()
    lib = ctypes.CDLL(built)
    lib.f3dgs_last_error.restype = ctypes.c_char_p
    d = cabi.Dev(rt)
    try:
        means, scales, rots = d.put(sc.means3D), d.put(sc.scales), d.put(sc.rotations)
        opac, shs, feats = d.put(sc.opacities), d.put(sc.shs), d.put(sc.features.reshape(P, C))
        bg, vm, pm, cp = d.put(sc.bg), d.put(cam.viewmatrix), d.put(cam.projmatrix), d.put(cam.campos)
        out_color, out_feat, out_depth, radii = d.alloc(3 * H * W * 4), d.alloc(C * H * W * 4), d.alloc(H * W * 4), \
            d.alloc(P * 4)
        bufs = {}

        def mk(key):
            def cb(_ctx, nbytes):
                bufs[key] = d.alloc(nbytes)
                return bufs[key].value

            return cabi.ALLOC(cb)

        cbs = [mk("geom"), mk("bin"), mk("img")]
        null, f = ctypes.c_void_p(0), ctypes.c_float
        R = lib.f3dgs_forward(cbs[0], null, cbs[1], null, cbs[2], null, P, sc.sh_degree, M, C, bg, W, H, means, shs,
                              null, feats, opac, scales, f(1.0), rots, null, vm, pm, cp, f(cam.tanfovx),
                              f(cam.tanfovy), 0, out_color, out_feat, out_depth, radii, 0, null)
        assert R == v.base["R"], lib.f3dgs_last_error()
        L = cabi.Layout()
        assert lib.f3dgs_get_layout(P, W, H, R, ctypes.byref(L)) == 0
        n_contrib = d.get(ctypes.c_void_p(bufs["img"].value + L.img_n_contrib), (H, W), np.int32)
        assert np.array_equal(n_contrib, v.base["n_contrib"].cpu().numpy())
        worst = {}
        for label, ups in (("N(0,1)", bw.upstream(H, W, C, 9)), ("dynamic range", bw.upstream(H, W, C, 10, True))):
            dgc, dgf, dgd = (d.put(u) for u in ups)
            g = {k: d.zeros(s) for k, s in dict(mean2D=(P, 3), conic=(P, 4), opacity=(P,), color=(P, 3),
                                                 feat=(P, C), mean3D=(P, 3), cov3D=(P, 6), sh=(P, M, 3),
                                                 scale=(P, 3), rot=(P, 4), dz=(P,)).items()}
            rc = lib.f3dgs_backward(P, sc.sh_degree, M, R, C, bg, W, H, means, shs, null, feats, scales, f(1.0), rots,
                                    null, vm, pm, cp, f(cam.tanfovx), f(cam.tanfovy), radii, bufs["geom"],
                                    bufs["bin"], bufs["img"], dgc, dgf, dgd, g["mean2D"], g["conic"], g["opacity"],
                                    g["color"], g["feat"], g["mean3D"], g["cov3D"], g["sh"], g["scale"], g["rot"],
                                    g["dz"], 0, null)
            assert rc == 0, lib.f3dgs_last_error()
            assert rt.cudaDeviceSynchronize() == 0
            dz = _t(d.get(g["dz"], (P, 1)), "cuda")
            worst[f"dL_dz {label}"] = v.Wt.per_gaussian(dz, _t(ups[2].reshape(-1, 1), "cuda"))
        _report(f"{name} C ABI", worst)
    finally:
        d.free()


@pytest.mark.gpu
@pytest.mark.parametrize("C", [16, 129])
@pytest.mark.parametrize("half", [False, True], ids=["float32 map", "float16 map + scale"])
def test_view_batch_feature_gradient_is_the_sum_of_the_views(C, half):
    """ViewBatch.backward over two views adds both views' dL/dfeature into one buffer: sum_v sum_p w_v dL/dF_v.  A float16
    map gradient stands for __fmul_rn(scale, h), which the reference applies exactly as the kernel does."""
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    from diff_gaussian_rasterization.feature_head import ScaledGrad
    from diff_gaussian_rasterization.parallel import ViewBatch

    sc = scenegen.make_config("small", views=2)
    sc.bg = BG.copy()
    sc.features = np.random.default_rng(C).standard_normal((sc.P, 1, C)).astype(np.float32)
    views = [DeviceView(sc, cam, 512) for cam in sc.cameras]
    t = views[0].t
    vb = ViewBatch({k: t[k] for k in ("means3D", "scales", "rotations", "opacities", "shs", "semantic_feature")})
    vb.zero_()
    P, H, W = sc.P, views[0].H, views[0].W
    scale = np.float32(3.0e-5)
    terms, m = None, torch.zeros(P, dtype=torch.float64, device="cuda")
    for i, v in enumerate(views):
        gc, gf, gd = (_t(u, "cuda") for u in bw.upstream(H, W, C, 20 + i, dynamic=i == 1))
        if half:  # the float16 map holds dL/dF / scale
            h = gf.half()
            g_feat, G = ScaledGrad(h, float(scale)), h.float() * torch.tensor(scale, device="cuda")
        else:
            g_feat, G = gf, gf
        _, _, _, _, ctx = vb.forward(GaussianRasterizationSettings(**v.rs))
        vb.backward(ctx, gc, g_feat, gd, last=i == len(views) - 1)
        tv = v.Wt.terms(G.reshape(C, -1).t())
        terms = tv if terms is None else tuple(a + b for a, b in zip(terms, tv))
        m += v.Wt.m
    r = bw.gaussian_ratio(vb.grads["semantic_feature"].reshape(P, C), terms, m)
    _report(f"ViewBatch two views C={C} {'float16 map + scale' if half else 'float32 map'}", {"dL_dsemantic_feature": r})


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [torch.float32, torch.float16], ids=["float32", "float16"])
@pytest.mark.parametrize("name,C", [("small", 16), ("needles", 129), ("layers129", 33), ("opaque", 1),
                                    ("halves97x38", 513), ("medium", 64)])
def test_lift_identities_per_gaussian(name, C, dt):
    from diff_gaussian_rasterization import _C

    v = _view(name)
    b, P, H, W = v.base, v.P, v.H, v.W
    g = torch.Generator(device="cuda").manual_seed(C)
    fmap = (torch.randn(C, H, W, device="cuda", generator=g)
            * 10.0 ** torch.empty(1, H, W, device="cuda").uniform_(-6, 0, generator=g)).to(dt)
    fs, ws = torch.zeros(P, C, device="cuda"), torch.zeros(P, device="cuda")
    _C.lift_features_accum(b["geom"], b["R"], b["binning"], b["img"], fmap, fs, ws)
    _report(f"{name} C={C} lift {dt}",
            dict(weight_sum=v.Wt.per_gaussian(ws.reshape(P, 1), torch.ones(H * W, 1, device="cuda")),
                 feature_sum=v.Wt.per_gaussian(fs, fmap.float().reshape(C, -1).t())))
