"""Shared parity harness: run one view through (a) this repo's CUDA path via the public Python API,
(b) the reference CUDA extension (oracle/_ref) or (c) the CPU oracle, and compare.

Tolerances (BASELINE.json north_star): bit-exact on tile/key indexing (radii, num_rendered,
point_list, ranges, n_contrib); float tensors within 1e-4 relative, implemented elementwise as
    images:     |a-b| <= 1e-4*|b| + 1e-5*max|b|
    gradients:  |a-b| <= 1e-4*|b| + 5e-5*max|b|
The absolute floor keeps near-cancelling entries from dominating: every gradient entry is a sum of thousands of
signed fp32 terms; the reference adds them with order-nondeterministic atomics (its own run-to-run spread is
~1e-6 of max|b|), we add them in a different (hierarchical) order.  Worst case over the test-suite so far:
1.4e-5 of max|b| (grad_scales with a non-zero background), i.e. 7x inside the 1e-4 bound.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "feature-3dgs_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import scenegen  # noqa: E402

RTOL = 1e-4
ATOL_REL = 1e-5
GRAD_ATOL_REL = 5e-5

INT_KEYS = ("radii", "num_rendered", "point_list", "ranges", "n_contrib")
FWD_FLOAT_KEYS = ("color", "feature_map", "depth", "final_T")
GRAD_KEYS = ("means3D", "means2D", "sh", "semantic_feature", "opacities", "scales", "rotations")


def _np(t):
    return t.detach().cpu().numpy()


def settings(scene, cam, device, debug=False, scale_modifier=1.0, prefiltered=False):
    """scenegen.settings_kwargs with the two rasterizer options it fixes made explicit."""
    rs = scenegen.settings_kwargs(scene, cam, device, debug=debug)
    rs.update(scale_modifier=float(scale_modifier), prefiltered=bool(prefiltered))
    return rs


def run_ours(scene, cam, device="cuda", grads=None, debug=False, colors_precomp=None, cov3D_precomp=None,
             scale_modifier=1.0, prefiltered=False):
    import torch
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer, _C

    t = scenegen.to_torch(scene, device, requires_grad=grads is not None)
    rs = GaussianRasterizationSettings(**settings(scene, cam, device, debug, scale_modifier, prefiltered))
    means2D = torch.zeros_like(t["means3D"], requires_grad=grads is not None)
    kw = dict(means3D=t["means3D"], means2D=means2D, opacities=t["opacities"],
              semantic_feature=t["semantic_feature"] if scene.C > 0 else None)
    if colors_precomp is None:
        kw["shs"] = t["shs"]
    else:
        kw["colors_precomp"] = torch.from_numpy(colors_precomp).to(device).requires_grad_(grads is not None)
    if cov3D_precomp is None:
        kw.update(scales=t["scales"], rotations=t["rotations"])
    else:
        kw["cov3D_precomp"] = torch.from_numpy(cov3D_precomp).to(device).requires_grad_(grads is not None)
    # direct _C call first to expose the internal buffers (same kernels as the autograd path)
    e = torch.Tensor([])
    sf = t["semantic_feature"] if scene.C > 0 else torch.empty(0, device=device)
    raw = _C.rasterize_gaussians(
        rs.bg, t["means3D"].detach(), e if colors_precomp is None else kw["colors_precomp"].detach(), sf.detach(),
        t["opacities"].detach(), e if cov3D_precomp is not None else t["scales"].detach(),
        e if cov3D_precomp is not None else t["rotations"].detach(), rs.scale_modifier,
        e if cov3D_precomp is None else kw["cov3D_precomp"].detach(), rs.viewmatrix, rs.projmatrix, rs.tanfovx,
        rs.tanfovy, rs.image_height, rs.image_width, e if colors_precomp is not None else t["shs"].detach(),
        rs.sh_degree, rs.campos, rs.prefiltered, rs.debug)
    R, color, feat, depth, radii, geom, binning, img = raw
    pl, ranges, ncontrib, final_T, rec = _C.debug_views(geom, binning, img, scene.P, cam.image_width,
                                                         cam.image_height, R)
    out = dict(num_rendered=np.int64(R), color=_np(color), feature_map=_np(feat), depth=_np(depth),
               radii=_np(radii), point_list=_np(pl).astype(np.int64), ranges=_np(ranges).astype(np.int64),
               n_contrib=_np(ncontrib).astype(np.int64), final_T=_np(final_T), rec=_np(rec))
    if grads is not None:
        color, feat, radii2, depth = GaussianRasterizer(rs)(**kw)
        gc, gf, gd = [torch.from_numpy(g).to(device) for g in grads]
        outs, gos = [color, depth], [gc, gd]
        if scene.C > 0:
            outs.append(feat)
            gos.append(gf)
        torch.autograd.backward(outs, gos)
        g = dict(means3D=_np(t["means3D"].grad), means2D=_np(means2D.grad), opacities=_np(t["opacities"].grad))
        if colors_precomp is None:
            g["sh"] = _np(t["shs"].grad)
        else:
            g["colors_precomp"] = _np(kw["colors_precomp"].grad)
        if cov3D_precomp is None:
            g["scales"], g["rotations"] = _np(t["scales"].grad), _np(t["rotations"].grad)
        else:
            g["cov3D_precomp"] = _np(kw["cov3D_precomp"].grad)
        if scene.C > 0:
            g["semantic_feature"] = _np(t["semantic_feature"].grad)
        out["grads"] = g
        out["color_autograd"] = _np(color)
    return out


def run_ref(scene, cam, device="cuda", grads=None, scale_modifier=1.0, prefiltered=False):
    """Reference CUDA extension (oracle/_ref) on the same inputs."""
    import torch
    from oracle import ref_wrapper as rw

    C = scene.C
    t = scenegen.to_torch(scene, device, requires_grad=grads is not None)
    rs = settings(scene, cam, device, scale_modifier=scale_modifier, prefiltered=prefiltered)
    mod = rw.load(C)
    e = torch.Tensor([])
    sf = t["semantic_feature"] if C > 0 else torch.zeros(scene.P, 1, 1, device=device)
    raw = mod.rasterize_gaussians(rs["bg"], t["means3D"].detach(), e, sf.detach(), t["opacities"].detach(),
                                  t["scales"].detach(), t["rotations"].detach(), rs["scale_modifier"], e,
                                  rs["viewmatrix"], rs["projmatrix"], rs["tanfovx"], rs["tanfovy"],
                                  rs["image_height"], rs["image_width"], t["shs"].detach(), rs["sh_degree"],
                                  rs["campos"], rs["prefiltered"], False)
    R, color, feat, depth, radii, geom, binning, img = raw
    final_T, ncontrib, ranges = rw.parse_image_buffer(img, cam.image_width, cam.image_height)
    pl = rw.parse_binning_buffer(binning, R)
    out = dict(num_rendered=np.int64(R), color=_np(color), feature_map=_np(feat)[:C], depth=_np(depth),
               radii=_np(radii), point_list=_np(pl).astype(np.int64), ranges=_np(ranges).astype(np.int64),
               n_contrib=_np(ncontrib).astype(np.int64), final_T=_np(final_T))
    out["geom"] = {k: _np(v) for k, v in rw.parse_geom_buffer(geom, scene.P, C).items()}
    if grads is not None:
        means2D = torch.zeros_like(t["means3D"], requires_grad=True)
        rr = rw.RefRasterizer(rs, C)
        color, feat, _, depth = rr(means3D=t["means3D"], means2D=means2D, opacities=t["opacities"], shs=t["shs"],
                                   semantic_feature=t["semantic_feature"] if C > 0 else None, scales=t["scales"],
                                   rotations=t["rotations"])
        gc, gf, gd = [torch.from_numpy(g).to(device) for g in grads]
        outs, gos = [color, depth], [gc, gd]
        if C > 0:
            outs.append(feat)
            gos.append(gf)
        torch.autograd.backward(outs, gos)
        g = dict(means3D=_np(t["means3D"].grad), means2D=_np(means2D.grad), opacities=_np(t["opacities"].grad),
                 sh=_np(t["shs"].grad), scales=_np(t["scales"].grad), rotations=_np(t["rotations"].grad))
        if C > 0:
            g["semantic_feature"] = _np(t["semantic_feature"].grad)
        out["grads"] = g
    return out


def run_oracle(scene, cam, grads=None, threads=None, **kw):
    import oracle

    if threads:
        oracle.set_threads(threads)
    f = oracle.forward(scene, cam, **kw)
    out = dict(num_rendered=np.int64(f["num_rendered"]), color=f["color"], feature_map=f["feature_map"],
               depth=f["depth"], radii=f["radii"], point_list=f["point_list"].astype(np.int64),
               ranges=f["ranges"].astype(np.int64), n_contrib=f["n_contrib"].astype(np.int64),
               final_T=f["final_T"], fwd=f)
    if grads is not None:
        g = oracle.backward(scene, cam, f, *grads, **{k: v for k, v in kw.items() if k != "render"})
        out["grads"] = dict(means3D=g["means3D"], means2D=g["means2D"], opacities=g["opacities"], sh=g["sh"],
                            scales=g["scales"], rotations=g["rotations"], semantic_feature=g["semantic_feature"],
                            colors_precomp=g["colors"], cov3D_precomp=g["cov3D"])
    return out


def golden_pair(g, key, ours):
    """(ours, stored) for array `key` of a golden file.  Large arrays are stored as every n-th element of the flattened
    array (`<key>_stride` = n, keeping the files small); `ours` is sampled the same way."""
    if key + "_stride" in g.files:
        return np.asarray(ours).reshape(-1)[:: int(g[key + "_stride"])], g[key]
    return ours, g[key]


def float_mismatch(a, b, rtol=RTOL, atol_rel=ATOL_REL):
    """-> (max violation ratio, max abs err, scale).  ratio <= 1 means within tolerance."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    if a.shape != b.shape:
        return float("inf"), float("inf"), 0.0
    if a.size == 0:
        return 0.0, 0.0, 0.0
    scale = float(np.max(np.abs(b)))
    err = np.abs(a - b)
    tol = rtol * np.abs(b) + atol_rel * scale + 1e-30
    bad = ~np.isfinite(a) | ~np.isfinite(b)
    ratio = float(np.max(np.where(bad, np.inf, err / tol)))
    return ratio, float(np.max(np.where(bad, np.inf, err))), scale


def compare(ours, ref, int_keys=INT_KEYS, float_keys=FWD_FLOAT_KEYS, grad_keys=GRAD_KEYS, rtol=RTOL,
            atol_rel=ATOL_REL, tie_tolerant=False):
    """-> dict report; report['ok'] is the overall verdict.

    tie_tolerant (CPU-oracle comparisons only): libm's expf differs from CUDA's by <= 2 ulp, so a pixel whose
    alpha or T lands within an ulp of the 1/255 or 1e-4 threshold can blend one Gaussian more or less.  Up to
    max(2, 1e-4 * pixels) such n_contrib mismatches are accepted; those pixels are masked out of the image
    comparison and, if any occurred, the gradient tolerance is widened 50x (a single flipped blend shows up in a
    few Gaussians' gradients).  The comparison against the reference CUDA build never uses this."""
    rep, ok = {}, True
    tie_mask, ties = None, 0
    for k in int_keys:
        a, b = np.asarray(ours[k]), np.asarray(ref[k])
        same = a.shape == b.shape and bool(np.array_equal(a, b))
        n_bad = int(np.sum(a != b)) if a.shape == b.shape else -1
        rep[k] = dict(exact=same, mismatches=n_bad, size=int(b.size))
        if k == "n_contrib" and tie_tolerant and not same and 0 < n_bad <= max(2, int(1e-4 * b.size)):
            tie_mask, ties = (a != b), n_bad
            rep[k]["accepted_ties"] = n_bad
            continue
        ok &= same
    for k in float_keys:
        a, b = np.asarray(ours[k]), np.asarray(ref[k])
        if tie_mask is not None and a.shape == b.shape and a.shape[-2:] == tie_mask.shape:
            a = np.where(tie_mask, b, a)
        r, e, s = float_mismatch(a, b, rtol, atol_rel)
        rep[k] = dict(ratio=r, max_abs_err=e, scale=s, bit_exact=bool(np.array_equal(ours[k], ref[k])))
        ok &= r <= 1.0
    if "grads" in ours and "grads" in ref:
        widen = 50.0 if ties else 1.0
        for k in grad_keys:
            if k in ours["grads"] and k in ref["grads"]:
                r, e, s = float_mismatch(ours["grads"][k], ref["grads"][k], rtol * widen, GRAD_ATOL_REL * widen)
                rep["grad_" + k] = dict(ratio=r, max_abs_err=e, scale=s)
                ok &= r <= 1.0
    rep["ok"] = bool(ok)
    return rep


def format_report(rep):
    lines = []
    for k, v in rep.items():
        if k == "ok":
            continue
        if "exact" in v:
            t = f" (accepted threshold ties: {v['accepted_ties']})" if "accepted_ties" in v else ""
            lines.append(f"  {k:22s} exact={v['exact']} mismatches={v['mismatches']}/{v['size']}{t}")
        else:
            extra = f" bit_exact={v['bit_exact']}" if "bit_exact" in v else ""
            lines.append(f"  {k:22s} viol={v['ratio']:.3g} max_abs_err={v['max_abs_err']:.3g} scale={v['scale']:.3g}{extra}")
    lines.append(f"  OK={rep['ok']}")
    return "\n".join(lines)


COV_GRAD_KEYS = ("means3D", "scales", "rotations")  # reach the parameters through the 2-D covariance


def conic_condition(rec):
    """Eigenvalue ratio of each Gaussian's 2-D conic (SplatRec columns 4..6 = conic a, b, c)."""
    with np.errstate(all="ignore"):  # rows of culled Gaussians are never written
        a, b, c = (rec[:, i].astype(np.float64) for i in (4, 5, 6))
        mid, d = 0.5 * (a + c), np.sqrt(0.25 * (a - c) ** 2 + b * b)
        return (mid + d) / (mid - d)


def tie_aware_compare(sc, cam, label, grads=None, vs_ref=None, ours=None, scale_modifier=1.0, prefiltered=False,
                      cond_max=None):
    """One view, compared on the device; prints the worst violation ratio (|a-b| / tolerance, <= 1 passes) of every
    float tensor and the number of n_contrib threshold ties, so the margin is on record in the test log.  -> ours.

    Against the unmodified reference build (oracle/_ref, where a reference checkout was there to build it; the default
    when one exists for sc.C): indices and colour / depth / final_T bit-identical, feature map and gradients within the
    parity bar.  Against the CPU oracle (oracle/: the reference algorithm restated in C, pinned to the reference's
    outputs by test_oracle_golden.py) with compare()'s threshold-tie rule: libm's expf differs from CUDA's by <= 2 ulp,
    so up to max(2, 1e-4 * pixels) pixels may differ in n_contrib; those are masked out of the images and widen the
    gradient bar 50x.  Every blend weight then carries those ulps, so the feature map's relative bar applies to the sum
    of its terms' magnitudes (the oracle's map of |features|) rather than to the possibly cancelled sum.

    cond_max: the gradients that pass through the 2-D covariance (COV_GRAD_KEYS) are compared only for Gaussians whose
    conic eigenvalue ratio is <= cond_max.  For a needle the conic -> covariance backward cancels terms of size ~ratio
    against each other, so the summation order of dL/dconic (float atomics, different on every run of the same build)
    moves those gradients by far more than the bar; the other gradients are compared for every Gaussian."""
    import copy

    import torch
    from oracle import ref_wrapper as rw

    opts = dict(scale_modifier=scale_modifier, prefiltered=prefiltered)
    if ours is None:
        ours = run_ours(sc, cam, grads=grads, **opts)
    if vs_ref is None:
        vs_ref = rw.available(sc.C)
    ref = (run_ref(sc, cam, grads=grads, **opts) if vs_ref else
           run_oracle(sc, cam, grads=grads, threads=os.cpu_count(), scale_modifier=scale_modifier))
    for k in ("radii", "point_list", "ranges"):
        assert np.array_equal(np.asarray(ours[k]).astype(np.int64), np.asarray(ref[k]).astype(np.int64)), k
    assert int(ours["num_rendered"]) == int(ref["num_rendered"])
    ties = np.asarray(ours["n_contrib"]).astype(np.int64) != np.asarray(ref["n_contrib"]).astype(np.int64)
    n_ties = int(ties.sum())
    if vs_ref:
        assert n_ties == 0
        for k in ("color", "depth", "final_T"):
            assert np.array_equal(ours[k], ref[k]), k
    else:
        assert n_ties <= max(2, int(1e-4 * ties.size)), n_ties
    keep = torch.from_numpy(~ties).cuda()
    extra = []  # image pixels outside the bar with n_contrib unchanged (oracle only)

    def viol(a, b, atol, widen=1.0, mask=None, mag=None):
        a = torch.from_numpy(np.ascontiguousarray(a)).cuda().double()
        b = torch.from_numpy(np.ascontiguousarray(b)).cuda().double()
        if a.numel() == 0:
            return 0.0
        if mask is not None:
            a = torch.where(mask, a, b)
        m = b.abs() if mag is None else torch.from_numpy(np.ascontiguousarray(mag)).cuda().double()
        tol = widen * (RTOL * m + atol * b.abs().max()) + 1e-30
        r = (a - b).abs() / tol
        if not vs_ref and r.dim() >= 2 and r.shape[-2:] == keep.shape:
            # a blend flipped at the threshold before the pixel's last contributor leaves n_contrib unchanged: such
            # pixels count against the same tie budget and must stay within the 50x bar of a tie
            px = r.reshape(-1, *r.shape[-2:]).amax(0)
            extra.append(px > 1.0)
            assert float(px.max()) <= 50.0, float(px.max())
            r = torch.where(px > 1.0, 0.0, px)
        return float(r.max())

    worst = {}
    if not vs_ref:
        for k in ("color", "depth", "final_T"):
            worst[k] = viol(ours[k], ref[k], ATOL_REL, mask=keep)
    if sc.C:
        mag = None
        if not vs_ref:
            sc_abs = copy.copy(sc)
            sc_abs.features = np.abs(sc.features)
            mag = run_oracle(sc_abs, cam, threads=os.cpu_count(), scale_modifier=scale_modifier)["feature_map"]
        worst["feature_map"] = viol(ours["feature_map"], ref["feature_map"], ATOL_REL, mask=keep, mag=mag)
    n_ill = 0
    if grads is not None:
        well = np.ones(sc.P, bool)
        if cond_max is not None:
            well = (ours["radii"] == 0) | (conic_condition(ours["rec"]) <= cond_max)
            n_ill = int((~well).sum())
        for k in GRAD_KEYS:
            if k in ours["grads"]:
                a, b = ours["grads"][k], ref["grads"][k]
                if k in COV_GRAD_KEYS:
                    a, b = a[well], b[well]
                worst["grad_" + k] = viol(a, b, GRAD_ATOL_REL, widen=50.0 if n_ties else 1.0)
    if extra:
        flipped = torch.stack(extra).any(0) & keep
        n_ties += int(flipped.sum())
        assert n_ties <= max(2, int(1e-4 * ties.size)), n_ties
    print(f"[{label} vs {'reference build' if vs_ref else 'CPU oracle'}] V={int((ours['radii'] > 0).sum())} "
          f"R={int(ours['num_rendered'])} n_contrib ties={n_ties} "
          + (f"cov-path grads skipped for {n_ill} conics with eigenvalue ratio > {cond_max:g}; " if n_ill else "")
          + "worst viol per tensor: "
          + ", ".join(f"{k}={v:.3g}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v <= 1.0, (k, v)
    return ours


def check_structure(ours, cam, P):
    """Size-independent properties of one view's binning and composite: ranges partition [0, R) in tile order, each
    tile's list is depth sorted with ties broken by Gaussian index (a stable sort), every visible Gaussian is listed,
    n_contrib never exceeds the tile's list length and final_T lies in (0, 1]."""
    R = int(ours["num_rendered"])
    ranges, pl = ours["ranges"], ours["point_list"]
    nz = ranges[(ranges[:, 1] - ranges[:, 0]) > 0]
    assert nz[0, 0] == 0 and nz[-1, 1] == R and np.array_equal(nz[1:, 0], nz[:-1, 1])
    depth = ours["rec"][:, 11]
    d = depth[pl]
    same_tile = np.ones(R - 1, bool)
    same_tile[nz[:-1, 1] - 1] = False
    assert (np.diff(d)[same_tile] >= 0).all()
    ties = same_tile & (np.diff(d) == 0)
    assert (np.diff(pl)[ties] > 0).all()
    counts = np.bincount(pl, minlength=P)
    assert ((counts > 0) == (ours["radii"] > 0)).all()
    gx = (cam.image_width + 15) // 16
    ty, tx = np.divmod(np.arange(cam.image_height * cam.image_width), cam.image_width)
    tile = (ty // 16) * gx + (tx // 16)
    lens = (ranges[:, 1] - ranges[:, 0])[tile].reshape(cam.image_height, cam.image_width)
    assert (ours["n_contrib"] <= lens).all()
    assert (ours["final_T"] > 0).all() and (ours["final_T"] <= 1).all()
    return int(ties.sum())
