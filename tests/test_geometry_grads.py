"""The default backward's geometric gradients per Gaussian, against float64 models.

parity's bars have a floor at 5e-5 of the largest entry of the whole tensor, so a Gaussian whose gradient is small can
be wrong under them: a lost term, a wrong sign on a small term or a wrong coefficient.  Here every gradient output of
the default backward is compared per Gaussian, with a bar made of that Gaussian's own terms:
  * the composite (dL/dmean2D, dL/dconic, dL/dopacity) against blend_weights.composite_model over the composite's own
    records and blended pairs, with the colour, depth and background terms of dL/dalpha; dL/dcolor and dL/dz against
    the blend-weight identities (blend_weights.Weights);
  * the backward preprocess (dL/dmeans3D, dL/dscales, dL/drotations, dL/dsh and dL/dcov3D, the last whether cov3D is
    precomputed or formed from scales and rotations) against camera_grad_model.preprocess_chain, float64 autograd
    pushed from the backward's OWN composite intermediates, so that the preprocess is checked apart from the
    composite.  Its bar is the kernel's expression
    evaluated on magnitudes, weighted by the conic's conditioning on the covariance path (see preprocess_chain);
  * the forward's splat records (screen mean, conic, colour, depth) against camera_grad_model.screen_quantities.
The only per-Gaussian exclusion is the needle rule (conic eigenvalue ratio > 100) on the outputs through the 2-D
covariance.  The forward's clamp of each colour channel is checked against the float64 colour: only within its bar
may the record's decision differ from the model's sign.  Exact checks: rows of culled Gaussians are 0; the third entries
of dL/dmean2D and dL/dconic, which are not gradients, are 0; SH coefficients above the active degree are 0 (unchanged when
accumulating); a colour channel the forward clamped has 0 in every coefficient; a mean outside the Jacobian's 1.3 tan_fov
limit passes no gradient through the clamped coordinate.

SH rows are staged through shared memory in both preprocess kernels, with 16-byte loads when M * 3 % 4 == 0 and the
pointer is 16-byte aligned and one float at a time otherwise: M = 1, 4, 9 and 16 at every active degree, and shs and
dL_dsh one float off a 16-byte boundary, run both.

CPU (`-m "not gpu"`): the checkers on the CPU oracle, and negative controls that parity's bar passes and these flag.
GPU: f3dgs_backward on the blend-weight and antialiasing scenes with three upstream gradients, the SH layouts, the
misaligned pointers, f3dgs_backward_accum over three views, the torch binding and ViewBatch.backward.  The worst ratio
|err| / bar of every scene and tensor is printed.
"""
import ctypes
import functools

import numpy as np
import pytest
import torch

import blend_weights as bw
import camera_grad_model as cgm
import parity
import scenegen

NEEDLE_COND_MAX = 100.0
COV_PATH = ("scales", "rotations", "cov3D")  # outputs that pass through the 2-D covariance only


def _t(a, dev="cpu"):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _report(label, worst):
    print(f"[{label}] worst |err|/bar: " + ", ".join(f"{k}={v:.3g}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v <= 1.0, (label, k, v)


def _upstreams(H, W, C, seed):
    """The three upstream gradients: scenegen's, N(0, 1), and N(0, 1) with a dynamic range of 1e6 across pixels."""
    return (("upstream_grads", scenegen.upstream_grads(H, W, C, seed)), ("N(0,1)", bw.upstream(H, W, C, seed + 1)),
            ("dynamic range", bw.upstream(H, W, C, seed + 2, dynamic=True)))


# ---------------------------------------------------------------------------------------------------------- checkers
def composite_check(pairs, w, rec, P, bg, gc, gd, ours):
    """ours: dict mean2D [P,3], conic [P,4], opacity [P], color [P,3], dz [P].  gc [3,H,W], gd [1,H,W] float32.
    -> dict of worst ratios, and the model's (ref, bar) of the six geometric values."""
    HW = pairs.HW
    Gc = gc.reshape(3, HW).t().to(pairs.pix.device)
    Gd = gd.reshape(HW).to(pairs.pix.device)
    bgp = (Gc.double() * bg.double().to(Gc.device))
    ref, bar = bw.composite_model(pairs, w, rec, P, bw.colour_depth_dots(rec, Gc, Gd), 4,
                                  (bgp.sum(1), bgp.abs().sum(1)))
    # the screen mean's third entry and the conic's third are not gradients of anything: they stay 0
    assert bool((ours["mean2D"][:, 2] == 0).all()) and bool((ours["conic"][:, 2] == 0).all())
    Wt = bw.Weights(pairs, w, P)
    g6 = bw.geom6(ours["mean2D"], ours["conic"], ours["opacity"]).double().to(ref.device)
    r = bw._ratio((g6 - ref).abs(), bar).max(0).values
    worst = {k: float(v) for k, v in zip(("dL_dmean2D.x", "dL_dmean2D.y", "dL_dconic.a", "dL_dconic.b", "dL_dconic.c",
                                          "dL_dopacity"), r)}
    worst["dL_dcolor"] = Wt.per_gaussian(ours["color"].reshape(P, 3), Gc)
    worst["dL_dz"] = Wt.per_gaussian(ours["dz"].reshape(P, 1), Gd.reshape(HW, 1))
    return worst, ref, bar


def preprocess_check(m, ours, visible, skip_needles=True):
    """ours: dict of the preprocess outputs (keys of the chain m).  -> worst ratio per output.  Needles skip the
    covariance-path outputs; their dL/dmeans3D carries the covariance share at its whole magnitude."""
    well = m["eig_ratio"] <= NEEDLE_COND_MAX
    vis = torch.as_tensor(visible).cpu().bool().reshape(-1)
    out = {}
    for k in ("means3D", "scales", "rotations", "cov3D", "sh"):
        if k not in m:
            continue
        P = m[k].shape[0]
        o = ours[k].detach().cpu().double().reshape(m[k].shape)
        bar = cgm.K_PRE * bw.U * m["mag_" + k]
        if k == "means3D":
            bar = bar + torch.where(well, torch.zeros_like(well, dtype=torch.float64), torch.ones_like(
                well, dtype=torch.float64))[:, None] * m["cov_share_means3D"].abs()
        r = bw._ratio((o - m[k]).abs(), bar).reshape(P, -1).max(1).values
        rows = vis & (well if (skip_needles and k in COV_PATH) else torch.ones_like(well))
        out[f"dL_d{k}"] = float(r[rows].max()) if bool(rows.any()) else 0.0
    return out


def exact_checks(ours, visible, D, M, clamped):
    """Rows of culled Gaussians are 0; SH coefficients above D are 0; a clamped channel has 0 in every coefficient."""
    vis = torch.as_tensor(visible).cpu().bool().reshape(-1)
    for k, v in ours.items():
        v = v.detach().cpu().reshape(vis.numel(), -1)
        assert bool((v[~vis] == 0).all()), ("culled row not zero", k)
    if "sh" in ours and M:
        sh = ours["sh"].detach().cpu().reshape(-1, M, 3)
        nb = (D + 1) ** 2
        assert bool((sh[:, nb:] == 0).all()), "SH coefficients above the active degree"
        cl = torch.as_tensor(clamped).cpu().bool().reshape(-1, 3) & vis[:, None]
        assert bool((sh.permute(0, 2, 1)[cl] == 0).all()), "clamped channel with a nonzero SH gradient"
        return int(cl.sum())
    return 0


# ---------------------------------------------------------------------------------------------------- CPU: oracle
def _oracle_intermediates(g):
    return dict(mean2D=_t(g["means2D"]), conic=_t(g["conic"]), opacity=_t(g["opacities"]), color=_t(g["colors"]),
                dz=_t(g["dz"]))


def _oracle_chain(sc, cam, f, g):
    W, H = cam.image_width, cam.image_height
    return cgm.preprocess_chain(sc.means3D, cam.viewmatrix, cam.projmatrix, cam.campos, W, H, cam.tanfovx,
                                cam.tanfovy, [g["means2D"], g["conic"], g["colors"], g["dz"]], f["radii"] > 0,
                                deg=sc.sh_degree, shs=sc.shs, clamped=f["clamped"], scales=sc.scales,
                                rotations=sc.rotations)


def _oracle_outputs(g):
    return dict(means3D=_t(g["means3D"]), scales=_t(g["scales"]), rotations=_t(g["rotations"]), cov3D=_t(g["cov3D"]),
                sh=_t(g["sh"]))


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_checkers_pass_on_the_oracle(name):
    import oracle
    from test_blend_weights import _oracle_view

    sc, cam, f, pairs, w = _oracle_view(name)
    H, W, P, C = cam.image_height, cam.image_width, sc.P, sc.C
    rec = _t(bw.oracle_records(f))
    for label, ups in _upstreams(H, W, C, 31):
        g = oracle.backward(sc, cam, f, *ups)
        worst, _, _ = composite_check(pairs, w, rec, P, _t(sc.bg), _t(ups[0]), _t(ups[2]), _oracle_intermediates(g))
        m = _oracle_chain(sc, cam, f, g)
        worst.update(preprocess_check(m, _oracle_outputs(g), f["radii"] > 0))
        n_clamped = exact_checks(_oracle_outputs(g), f["radii"] > 0, sc.sh_degree, sc.shs.shape[1], f["clamped"])
        assert n_clamped > 0
        _report(f"oracle {name} {label}", worst)


def test_negative_controls_pass_the_parity_bar_and_fail_the_checkers():
    """Perturbations of the oracle's gradients on `small` that parity's bar passes and these checkers flag: the
    background term dropped at one pixel of one Gaussian; the depth term of one pair dropped; one small dL/dsh
    coefficient (below 1e-3 of the tensor's largest) off by 1 %; one Gaussian's dL/drot scaled by 1 + 1e-3."""
    import oracle
    from test_blend_weights import _oracle_view

    sc, cam, f, pairs, w = _oracle_view("small")
    H, W, P, C = cam.image_height, cam.image_width, sc.P, sc.C
    ups = bw.upstream(H, W, C, 41)
    g = oracle.backward(sc, cam, f, *ups)
    rec = _t(bw.oracle_records(f))
    gc, gd = _t(ups[0]), _t(ups[2])
    mids = _oracle_intermediates(g)
    worst, ref, bar = composite_check(pairs, w, rec, P, _t(sc.bg), gc, gd, mids)
    assert max(worst.values()) <= 1.0
    ours6 = bw.geom6(mids["mean2D"], mids["conic"], mids["opacity"]).double()

    def composite_flags(d6):
        """parity passes the perturbed tensors, and the model's bar flags them."""
        x = ours6 + d6
        for j, (src, col) in enumerate((("mean2D", 0), ("mean2D", 1), ("conic", 0), ("conic", 1), ("conic", 3),
                                        ("opacity", None))):
            base = mids[src].double().numpy()
            pert = base.copy()
            if col is None:
                pert = x[:, j].numpy().reshape(base.shape).astype(np.float32)
            else:
                pert[:, col] = x[:, j].numpy()
            assert parity.float_mismatch(pert, base, parity.RTOL, parity.GRAD_ATOL_REL)[0] <= 1.0, j
        return float(bw._ratio((x - ref).abs(), bar).max())

    # the terms of one pair, from the model itself: L with and without the term
    sel = pairs.widx[w > 0]
    pix, gid = pairs.pix[sel], pairs.gid[sel]
    Gc = gc.reshape(3, -1).t()
    Gd = gd.reshape(-1)
    bgp = Gc.double() * _t(sc.bg).double()
    base_dfn = bw.colour_depth_dots(rec, Gc, Gd)
    bg_terms = (bgp.sum(1), bgp.abs().sum(1))
    # a Gaussian whose whole composite row lies under parity's floor in every tensor
    rowmax = ours6.abs().max(1).values
    floor = 0.5 * parity.GRAD_ATOL_REL * ours6.abs().max(0).values
    under = torch.nonzero((ours6.abs() < floor).all(1) & (rowmax > 0)).reshape(-1)
    assert under.numel() > 10
    gq = int(under[under.numel() // 2])
    on = torch.nonzero(gid == gq).reshape(-1)
    assert on.numel() > 0
    z = rec[:, 11].double()
    k = on[torch.argmax((z[gid[on]] * Gd.double()[pix[on]]).abs())]

    def no_depth(gi, px):
        d, dabs = base_dfn(gi, px)
        d = d.clone()
        d[k] -= z[gi[k]] * Gd.double()[px[k]]
        return d, dabs

    ref_nd, _ = bw.composite_model(pairs, w, rec, P, no_depth, 4, bg_terms)
    # background at one pixel of Gaussian gq: the model without that pixel's background term minus the model with it
    p0 = int(pix[on[torch.argmax(bgp.sum(1)[pix[on]].abs())]])
    bgd = bg_terms[0].clone()
    bgd[p0] = 0.0
    ref_nb, _ = bw.composite_model(pairs, w, rec, P, base_dfn, 4, (bgd, bg_terms[1]))
    d_depth = torch.zeros_like(ours6)
    d_depth[gq] = (ref_nd - ref)[gq]
    d_bg = torch.zeros_like(ours6)
    d_bg[gq] = (ref_nb - ref)[gq]  # only Gaussian gq's share of that pixel's term is dropped
    flagged = {"(a) background term dropped at one pixel": composite_flags(d_bg),
               "(b) depth term of one pair dropped": composite_flags(d_depth)}
    # preprocess controls
    m = _oracle_chain(sc, cam, f, g)
    outs = _oracle_outputs(g)
    assert max(preprocess_check(m, outs, f["radii"] > 0).values()) <= 1.0
    sh = g["sh"].copy()
    cand = np.argwhere((np.abs(sh) < 1e-3 * np.abs(sh).max()) & (np.abs(sh) > 1e-5 * np.abs(sh).max()))
    gi, ki, ci = (int(x) for x in cand[len(cand) // 2])
    sh[gi, ki, ci] *= np.float32(1.01)
    assert parity.float_mismatch(sh, g["sh"], parity.RTOL, parity.GRAD_ATOL_REL)[0] <= 1.0
    flagged["(c) small dL/dsh coefficient off by 1 %"] = preprocess_check(m, dict(outs, sh=_t(sh)),
                                                                          f["radii"] > 0)["dL_dsh"]
    rot = g["rotations"].copy()
    rmax = np.abs(rot).max(1)
    well = (m["eig_ratio"] <= NEEDLE_COND_MAX).numpy() & (f["radii"] > 0)
    ri = int(np.argsort(np.where(well, rmax, np.inf))[int(well.sum()) // 2])
    rot[ri] *= np.float32(1 + 1e-3)
    assert parity.float_mismatch(rot, g["rotations"], parity.RTOL, parity.GRAD_ATOL_REL)[0] <= 1.0
    flagged["(d) one dL/drot row scaled by 1 + 1e-3"] = preprocess_check(m, dict(outs, rotations=_t(rot)),
                                                                         f["radii"] > 0)["dL_drotations"]
    print(f"[negative controls, Gaussian {gq}] " + ", ".join(f"{k}={v:.3g}" for k, v in flagged.items()))
    for label, r in flagged.items():
        assert r > 1.0, (label, r)


# ----------------------------------------------------------------------------------------------------------- GPU
def _ptr(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None and t.numel() else 0)


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_backward_scratch_bytes.restype = ctypes.c_size_t
    return L


class View:
    """One view on the device with the rasterizer's options: its forward, the pairs, the extracted W and what the
    backward entries need.  shs / cov / cols / mod: the SH rows (default the scene's), precomputed covariances or
    colours, and the scale modifier.  C: the feature width.  planes: render with the forward that also writes the
    opacity and inverse-depth planes (rasterize_gaussians_alpha_invdepth), with antialiased opacities when
    antialiasing (the records then hold op_eff)."""

    def __init__(self, sc, cam, shs=None, D=None, cov=None, cols=None, mod=1.0, group=512, weights=True, C=8,
                 planes=False, antialiasing=False):
        assert planes or not antialiasing
        dev = torch.device("cuda")
        self.sc, self.cam, self.mod = sc, cam, mod
        self.P, self.W, self.H = sc.P, cam.image_width, cam.image_height
        self.d = scenegen.to_torch(sc, dev)
        e = torch.empty(0, device=dev)
        self.shs = e if cols is not None else (self.d["shs"] if shs is None else shs)
        self.M = self.shs.shape[1] if self.shs.numel() else 0
        self.D = sc.sh_degree if D is None else D
        self.cov = e if cov is None else cov.float().to(dev).contiguous()
        self.cols = e if cols is None else cols.float().to(dev).contiguous()
        self.scales, self.rots = (e, e) if cov is not None else (self.d["scales"], self.d["rotations"])
        self.vm, self.pm, self.cp = (torch.tensor(a, device=dev).contiguous() for a in (cam.viewmatrix,
                                                                                      cam.projmatrix, cam.campos))
        self.bg = torch.tensor(sc.bg, device=dev)
        self.C, self.planes, self.antialiasing = C, planes, antialiasing
        self.feats = torch.randn(self.P, 1, self.C, generator=torch.Generator().manual_seed(3)).to(dev)
        self.base = self.forward(self.feats)
        b = self.base
        self.R = b["R"]
        if weights:
            self.pairs = bw.Pairs(b["point_list"], b["ranges"], b["n_contrib"], self.W, self.H)
            self.w = bw.extract(self.pairs, self.P, self._onehot, group)

    def forward(self, sf):
        from diff_gaussian_rasterization import _C

        args = (self.bg, self.d["means3D"], self.cols, sf, self.d["opacities"], self.scales, self.rots, self.mod,
                self.cov, self.vm, self.pm, self.cam.tanfovx, self.cam.tanfovy, self.H, self.W, self.shs, self.D,
                self.cp, False, False)
        planes = {}
        if self.planes:
            R, color, fmap, depth, alpha, invdepth, radii, geom, binning, img = _C.rasterize_gaussians_alpha_invdepth(
                *args, antialiasing=self.antialiasing)
            planes = dict(alpha=alpha, invdepth=invdepth)
        else:
            R, color, fmap, depth, radii, geom, binning, img = _C.rasterize_gaussians(*args)
        pl, ranges, n_contrib, final_T, rec = _C.debug_views(geom, binning, img, self.P, self.W, self.H, R)
        return dict(R=R, color=color, fmap=fmap, depth=depth, radii=radii, geom=geom, binning=binning, img=img,
                    point_list=pl, ranges=ranges, n_contrib=n_contrib, final_T=final_T, rec=rec, **planes)

    def _onehot(self, g0, C):
        sf = torch.zeros(self.P, 1, C, device="cuda")
        sf[g0:g0 + C, 0, :] = torch.eye(C, device="cuda")
        r = self.forward(sf)
        for k in ("color", "n_contrib", "final_T", "point_list"):
            assert torch.equal(r[k], self.base[k]), k
        return r["fmap"].reshape(C, -1)

    @property
    def visible(self):
        return (self.base["radii"] > 0).cpu()

    @functools.cached_property
    def colour_model(self):
        """(visible indices, the unclamped SH colour [n,3] in float64, its bar [n,3]).  The kernel's float32 sum is
        within (terms + 16) u of the magnitude of its terms: the terms' monomials and products and the normalised
        direction's few u each, and one rounding per addition."""
        idx = self.visible.nonzero().flatten()
        f = lambda a: torch.as_tensor(np.asarray(a)).double()  # noqa: E731
        p, cp, shs = f(self.sc.means3D)[idx], f(self.cam.campos), self.shs.cpu().double()[idx]
        dvec = p - cp
        dn = dvec / dvec.norm(dim=1, keepdim=True)
        basis = cgm.sh_basis_abs(self.D, dn.abs())
        mag = (basis[:, :, None] * shs[:, :basis.shape[1]].abs()).sum(1) + 0.5
        return idx, cgm.sh_color(self.D, shs, dn), (basis.shape[1] + 16) * bw.U * mag

    @property
    def clamped(self):
        """The channels the forward clamps, decided by the float64 model: a negative colour beyond its bar; within the
        bar, where float32 may land on either side of 0, the kernel's own decision (the record's colour is 0)."""
        out = torch.zeros(self.P, 3, dtype=torch.bool)
        if not self.M:
            return out
        idx, col, bar = self.colour_model
        rec0 = (self.base["rec"][:, 8:11] == 0).cpu()[idx]
        out[idx] = (col < -bar) | ((col.abs() <= bar) & rec0)
        return out

    def head(self):
        return [self.P, self.D, self.M, self.R, self.C, _ptr(self.bg), self.W, self.H, _ptr(self.d["means3D"]),
                _ptr(self.shs), _ptr(self.cols)]

    def cam_args(self):
        return [_ptr(self.vm), _ptr(self.pm), _ptr(self.cp), ctypes.c_float(self.cam.tanfovx),
                ctypes.c_float(self.cam.tanfovy), _ptr(self.base["radii"]), _ptr(self.base["geom"]),
                _ptr(self.base["binning"]), _ptr(self.base["img"])]

    def backward(self, lib, ups, dsh=None):
        """f3dgs_backward -> dict of every output.  dsh: the dL_dsh buffer to write (default a fresh aligned one)."""
        dev = torch.device("cuda")
        gc, gf, gd = (_t(u, dev) for u in ups)
        P, M = self.P, self.M
        z = lambda *s: torch.zeros(*s, device=dev)  # noqa: E731
        o = dict(mean2D=z(P, 3), conic=z(P, 4), opacity=z(P), color=z(P, 3), feat=z(P, self.C), means3D=z(P, 3),
                 cov3D=z(P, 6), sh=z(P, M, 3) if dsh is None else dsh, scales=z(P, 3), rotations=z(P, 4), dz=z(P))
        sr = self.scales.numel() > 0
        null = ctypes.c_void_p(0)
        args = self.head() + [_ptr(self.feats), _ptr(self.scales), ctypes.c_float(self.mod), _ptr(self.rots),
                              _ptr(self.cov)] + self.cam_args() + [
            _ptr(gc), _ptr(gf), _ptr(gd), _ptr(o["mean2D"]), _ptr(o["conic"]), _ptr(o["opacity"]), _ptr(o["color"]),
            _ptr(o["feat"]), _ptr(o["means3D"]), _ptr(o["cov3D"]), _ptr(o["sh"]) if M else null,
            _ptr(o["scales"]) if sr else null, _ptr(o["rotations"]) if sr else null, _ptr(o["dz"]), 0,
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)]
        rc = lib.f3dgs_backward(*args)
        assert rc == 0, lib.f3dgs_last_error()
        torch.cuda.synchronize()
        return o

    def accum(self, lib, ups, o):
        """f3dgs_backward_accum into the buffers of o (opacity, feat, means3D, sh, scales, rotations, mean2D,
        grad_accum, denom; colors / cov3D when precomputed)."""
        dev = torch.device("cuda")
        gc, gf, gd = (_t(u, dev) for u in ups)
        scratch = torch.empty(lib.f3dgs_backward_scratch_bytes(self.P), dtype=torch.uint8, device=dev)
        null = ctypes.c_void_p(0)
        sr = self.scales.numel() > 0
        args = self.head() + [_ptr(self.scales), ctypes.c_float(self.mod), _ptr(self.rots), _ptr(self.cov)] + \
            self.cam_args() + [
            _ptr(gc), _ptr(gf), _ptr(gd), _ptr(scratch), _ptr(o["opacity"]),
            _ptr(o["colors"]) if self.cols.numel() else null, _ptr(o["feat"]), _ptr(o["means3D"]),
            _ptr(o["cov3D"]) if self.cov.numel() else null, _ptr(o["sh"]) if self.M else null,
            _ptr(o["scales"]) if sr else null, _ptr(o["rotations"]) if sr else null, _ptr(o["mean2D"]),
            _ptr(o["grad_accum"]), _ptr(o["denom"]), null, 0, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)]
        rc = lib.f3dgs_backward_accum(*args)
        assert rc == 0, lib.f3dgs_last_error()
        torch.cuda.synchronize()

    def chain(self, mids, clamp_grad=False):
        """preprocess_chain on intermediates mids (mean2D, conic, color, dz)."""
        sc, cam = self.sc, self.cam
        prec_cov = self.cov.numel() > 0
        return cgm.preprocess_chain(
            sc.means3D, cam.viewmatrix, cam.projmatrix, cam.campos, self.W, self.H, cam.tanfovx, cam.tanfovy,
            [mids[k] for k in ("mean2D", "conic", "color", "dz")], self.visible, deg=self.D,
            shs=self.shs.cpu() if self.M else None, clamped=self.clamped if self.M else None,
            colors=self.cols.cpu() if self.cols.numel() else None, scales=None if prec_cov else sc.scales,
            rotations=None if prec_cov else sc.rotations, mod=self.mod, cov3D=self.cov.cpu() if prec_cov else None,
            clamp_grad=clamp_grad)

    def outputs(self, o, accum=False):
        """The preprocess outputs of a backward's dict, keyed as the chain's.  f3dgs_backward writes dL/dcov3D on the
        scale / rotation path too; the accumulating entry only when cov3D is precomputed.  A precomputed colour's
        gradient is the composite's dL/dcolor, which composite_check compares with the blend weights."""
        keys = ["means3D"] + ([] if self.cov.numel() else ["scales", "rotations"]) + \
            (["cov3D"] if self.cov.numel() or not accum else []) + ([] if self.cols.numel() else ["sh"])
        return {k: o[k] for k in keys}


def _records_check(v):
    """The forward's splat records (screen mean, conic, colour, depth) against screen_quantities in float64."""
    sc, cam = v.sc, v.cam
    vis = v.visible
    idx = vis.nonzero().flatten()
    f = lambda a: torch.as_tensor(np.asarray(a)).double()  # noqa: E731
    p = f(sc.means3D)[idx]
    if v.cov.numel():
        cv = v.cov.cpu().double()[idx]
    else:
        cv = cgm.cov3d_from_scale_rot(f(sc.scales)[idx], f(sc.rotations)[idx], v.mod)
    vm, pm, cp = f(cam.viewmatrix).reshape(16), f(cam.projmatrix).reshape(16), f(cam.campos)
    cols = v.cols.cpu().double()[idx] if v.cols.numel() else None
    shs = v.shs.cpu().double()[idx] if v.M else None
    ndc, (A, B, C), col, depth = cgm.screen_quantities(p, cv, vm, pm, cp, v.W, v.H, cam.tanfovx, cam.tanfovy, v.D,
                                                       shs=shs, colors=cols)
    rec = v.base["rec"].cpu().double()[idx]
    ph = torch.cat([p, torch.ones(len(idx), 1, dtype=torch.float64)], 1)
    hw = ph @ pm[3::4]
    cw = (ph.abs() @ pm[3::4].abs()) / hw.abs()
    ix = ((ndc + 1.0) * torch.tensor([v.W, v.H], dtype=torch.float64) - 1.0) * 0.5
    # the mean: hx / hw rounded in 2 dot products (4 u each, relative to their magnitudes, with hw's cancellation cw),
    # the reciprocal and product (2 u), then ndc2pix (3 u on its terms)
    habs = torch.stack([ph.abs() @ pm[0::4].abs(), ph.abs() @ pm[1::4].abs()], 1) / hw.abs()[:, None]
    wh = torch.tensor([v.W, v.H], dtype=torch.float64)
    bar_mean = 16 * bw.U * (habs * (1 + cw[:, None]) * 0.5 * wh + ix.abs() + 0.5 * wh)
    m = v.chain(dict(mean2D=torch.zeros(v.P, 3), conic=torch.zeros(v.P, 4), color=torch.zeros(v.P, 3),
                     dz=torch.zeros(v.P)))
    kap = m["kappa_eff"][idx]
    well = m["eig_ratio"][idx] <= NEEDLE_COND_MAX
    con = torch.stack([A, B, C], 1)
    # the conic: the 2-D covariance to a few u of its magnitudes, then the inverse through det's cancellation
    bar_con = cgm.K_PRE * bw.U * kap[:, None] * (con.abs().sum(1, keepdim=True))
    # colour: View.colour_model's bar.  The clamp decision against the model: a channel the record holds at 0 must not
    # be positive beyond the bar, one it holds positive not negative beyond it
    bad_clamps = 0
    if v.M:
        _, raw, bar_col = v.colour_model
        rec0 = rec[:, 8:11] == 0
        bad_clamps = int((rec0 & (raw > bar_col)).sum() + (~rec0 & (raw < -bar_col)).sum())
        print(f"[records] clamped channels {int(rec0.sum())}, clamp decisions against the model: {bad_clamps} wrong")
    else:
        bar_col = torch.zeros_like(col)
    # depth: one dot product of four terms
    bar_depth = 4 * bw.U * (ph.abs() @ vm[2::4].abs())

    def ratio(x, ref, bar, rows=None):
        r = bw._ratio((x - ref).abs(), bar).reshape(len(idx), -1).max(1).values
        r = r if rows is None else r[rows]
        return float(r.max()) if r.numel() else 0.0

    assert bad_clamps == 0
    return {"rec.mean": ratio(rec[:, 0:2], ix, bar_mean),
            "rec.conic": ratio(rec[:, 4:7], con, bar_con, well),
            "rec.colour": ratio(rec[:, 8:11], col, bar_col),
            "rec.depth": ratio(rec[:, 11], depth, bar_depth)}


def _scene(name):
    from test_blend_weights import BG, SCENES

    if name in SCENES:
        sc, cam = SCENES[name]()
        kw = {}
    else:
        scenes = _aa_scenes()
        base = {"fx!=fy": "fx!=fy", "cov3D_precomp": "fx!=fy", "colors_precomp": "fx!=fy"}.get(name, name)
        sc, cam = scenes[base]
        kw = {}
        if name == "fx!=fy":
            kw = dict(mod=1.3)
        if name == "cov3D_precomp":
            kw = dict(cov=cgm.cov3d_from_scale_rot(torch.as_tensor(sc.scales).double(),
                                                   torch.as_tensor(sc.rotations).double()))
        if name == "colors_precomp":
            kw = dict(cols=torch.rand(sc.P, 3, generator=torch.Generator().manual_seed(8)))
    sc.bg = BG.copy()
    return sc, cam, kw


@functools.lru_cache(maxsize=1)
def _aa_scenes():
    from test_antialiasing import _scenes

    return _scenes()


@functools.lru_cache(maxsize=2)
def _view(name):
    sc, cam, kw = _scene(name)
    return View(sc, cam, group=4096 if name == "medium" else 512, **kw)


SCENE_NAMES = ["small", "inside", "needles", "plane", "layers129", "opaque", "huge", "medium", "deg0", "deg1", "deg2",
               "deg3", "fx!=fy", "cov3D_precomp", "colors_precomp"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCENE_NAMES)
def test_default_backward_matches_the_models(lib, name):
    v = _view(name)
    worst = _records_check(v)
    _report(f"{name} records", worst)
    n_clamped = n_outside = 0
    for label, ups in _upstreams(v.H, v.W, v.C, 51):
        o = v.backward(lib, ups)
        worst, _, _ = composite_check(v.pairs, v.w, v.base["rec"], v.P, v.bg, _t(ups[0]), _t(ups[2]), o)
        m = v.chain(o)
        worst.update(preprocess_check(m, v.outputs(o), v.visible))
        n_clamped += exact_checks({k: o[k] for k in ("mean2D", "conic", "opacity", "color", "dz", "means3D")}
                                  | v.outputs(o), v.visible, v.D, v.M, v.clamped)
        out = m["outside"] > 0
        if bool(out.any()):
            # the clamped coordinate passes no gradient: the model that lets it pass differs by more than the bar
            n_outside = int(out.sum())
            m2 = v.chain(o, clamp_grad=True)
            r2 = preprocess_check(m2, v.outputs(o), v.visible)["dL_dmeans3D"]
            print(f"[{name} {label}] {n_outside} means outside 1.3 tan_fov; dL/dmeans3D against a model whose clamp "
                  f"passes the gradient: {r2:.3g}")
            if name == "fx!=fy":
                assert r2 > 1.0
        _report(f"{name} V={int(v.visible.sum())} needles={int((v.visible & (m['eig_ratio'] > NEEDLE_COND_MAX)).sum())}"
                f" {label}", worst)
    print(f"[{name}] clamped channels checked: {n_clamped}")
    if name in ("small", "deg3"):
        assert n_clamped > 0
    if name == "fx!=fy":
        assert n_outside > 0


# (M, D): every active degree of each stored width; M * 3 % 4 != 0 for M = 1 and 9 (the scalar staging path)
SH_LAYOUTS = [(1, 0), (4, 0), (4, 1), (9, 0), (9, 1), (9, 2), (16, 0), (16, 1), (16, 2), (16, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("M,D", SH_LAYOUTS)
def test_sh_layouts(lib, M, D):
    """shs[:, :M] at active degree D: the preprocess chain per Gaussian, coefficients above D exactly 0, and unchanged
    when accumulated into a buffer that holds other values."""
    sc, cam, _ = _scene("deg3")
    shs = torch.from_numpy(np.ascontiguousarray(sc.shs[:, :M])).cuda()
    v = View(sc, cam, shs=shs, D=D, weights=False)
    scalar = (M * 3) % 4 != 0 or v.shs.data_ptr() % 16 != 0
    print(f"[M={M} D={D}] SH staging: {'scalar' if scalar else 'float4'} path")
    assert scalar == (M in (1, 9))
    _report(f"M={M} D={D} records", _records_check(v))
    for label, ups in _upstreams(v.H, v.W, v.C, 61)[1:]:
        o = v.backward(lib, ups)
        _report(f"M={M} D={D} {label}", preprocess_check(v.chain(o), v.outputs(o), v.visible))
        exact_checks(v.outputs(o), v.visible, D, M, v.clamped)
    # accumulation: coefficients above D and rows of culled Gaussians keep what the buffer held
    dev = torch.device("cuda")
    P = v.P
    held = torch.randn(P, M, 3, generator=torch.Generator().manual_seed(M + D)).to(dev)
    o = {k: torch.zeros(P, n, device=dev) for k, n in (("opacity", 1), ("feat", v.C), ("means3D", 3), ("scales", 3),
                                                        ("rotations", 4), ("mean2D", 3), ("grad_accum", 1),
                                                        ("denom", 1))}
    o["sh"] = held.clone()
    v.accum(lib, _upstreams(v.H, v.W, v.C, 61)[1][1], o)
    nb = (D + 1) ** 2
    assert torch.equal(o["sh"][:, nb:], held[:, nb:])
    assert torch.equal(o["sh"][~v.visible.cuda()], held[~v.visible.cuda()])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["blocks", "deg3", "small"])
def test_misaligned_sh_pointers(lib, name):
    """shs one float past a 16-byte boundary in the forward and the backward, and dL_dsh written there: the forward is
    bitwise the aligned one; on the view whose intermediates are bitwise reproducible (test_camera_grad._block_scene)
    dL/dsh is bitwise the aligned call's, elsewhere within the model's bar."""
    from test_camera_grad import _block_scene
    from test_gpu_regimes import _offset_copy

    if name == "blocks":
        sc, cam = _block_scene()
        sc.bg = np.array([0.3, 0.6, 0.9], np.float32)
    else:
        sc, cam, _ = _scene(name)
    a = View(sc, cam, weights=False)
    shs_mis = _offset_copy(a.shs)
    b = View(sc, cam, shs=shs_mis, weights=False)
    assert b.shs.data_ptr() % 16 != 0
    for k in ("color", "depth", "radii", "final_T", "n_contrib", "point_list", "rec"):
        assert torch.equal(a.base[k], b.base[k]), k
    ups = bw.upstream(a.H, a.W, a.C, 71)
    oa = a.backward(lib, ups)
    dsh = _offset_copy(torch.zeros_like(oa["sh"]))
    assert dsh.data_ptr() % 16 != 0
    print(f"[{name}] misaligned shs {b.shs.data_ptr() % 16} and dL_dsh {dsh.data_ptr() % 16} bytes off 16: scalar path")
    ob = b.backward(lib, ups, dsh=dsh)
    if name == "blocks":
        for k in ("mean2D", "conic", "color", "dz", "opacity"):
            assert torch.equal(oa[k], ob[k]), k
        assert torch.equal(oa["sh"], ob["sh"])
        assert bool(ob["sh"].abs().sum() > 0)
    _report(f"{name} misaligned", preprocess_check(b.chain(ob), b.outputs(ob), b.visible))


def _model_of_view(v, ups):
    """The models of one view with the composite's float64 values as intermediates -> (ref dict, bar dict) of the
    outputs of the accumulating entry: opacity, mean2D and the preprocess's.  The preprocess part's bar is the chain's
    own plus the chain pushed through the composite's bars (it is linear in the intermediates)."""
    P = v.P
    gc, gd = _t(ups[0]), _t(ups[2])
    HW = v.pairs.HW
    Gc = gc.reshape(3, HW).t().cuda()
    Gd = gd.reshape(HW, 1).cuda()
    bgp = Gc.double() * v.bg.double()
    ref6, bar6 = bw.composite_model(v.pairs, v.w, v.base["rec"], P, bw.colour_depth_dots(v.base["rec"], Gc, Gd[:, 0]),
                                    4, (bgp.sum(1), bgp.abs().sum(1)))
    Wt = bw.Weights(v.pairs, v.w, P)
    rc, ac, anc = Wt.terms(Gc)
    rz, az, anz = Wt.terms(Gd)
    bar_c = bw.K * bw.U * (anc + Wt.m[:, None] * ac)
    bar_z = bw.K * bw.U * (anz + Wt.m[:, None] * az)
    ref6, bar6 = ref6.cpu(), bar6.cpu()

    def mids(x6, c, z):
        return dict(mean2D=torch.stack([x6[:, 0], x6[:, 1], torch.zeros(P, dtype=torch.float64)], 1),
                    conic=torch.stack([x6[:, 2], x6[:, 3], torch.zeros(P, dtype=torch.float64), x6[:, 4]], 1),
                    color=c.cpu(), dz=z.cpu().reshape(-1))

    m = v.chain(mids(ref6, rc, rz))
    mb = v.chain(mids(bar6, bar_c, bar_z))  # magnitudes of the chain on the composite's bars
    ref = {k: m[k] for k in v.outputs({"means3D": 0, "scales": 0, "rotations": 0, "sh": 0, "cov3D": 0}, accum=True)}
    bar = {k: cgm.K_PRE * bw.U * m["mag_" + k] + mb["mag_" + k] for k in ref}
    ref["opacity"], bar["opacity"] = ref6[:, 5:6], bar6[:, 5:6]
    ref["mean2D"], bar["mean2D"] = ref6[:, 0:2], bar6[:, 0:2]
    return ref, bar, m


@pytest.mark.gpu
def test_accumulating_entry_and_view_batch_over_three_views(lib):
    """f3dgs_backward_accum over three views into one zeroed buffer, and ViewBatch.backward over the same views: the sum
    of the per-view models within the sum of their bars plus the accumulation's rounding; dL_dmean2D_out against the
    last view's model; grad_accum against the sum of the model's |dL/dmean2D.xy| and denom the visible count."""
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    from diff_gaussian_rasterization.parallel import ViewBatch

    sc = scenegen.make_config("small", views=3)
    sc.bg = np.array([0.3, 0.6, 0.9], np.float32)
    views = [View(sc, cam) for cam in sc.cameras]
    P, dev = sc.P, torch.device("cuda")
    o = {k: torch.zeros(P, n, device=dev) for k, n in (("opacity", 1), ("feat", 8), ("means3D", 3), ("scales", 3),
                                                        ("rotations", 4), ("mean2D", 3), ("grad_accum", 1),
                                                        ("denom", 1))}
    o["sh"] = torch.zeros(P, sc.shs.shape[1], 3, device=dev)
    ref, bar, gsum, gbar, cnt = None, None, 0, 0, 0
    all_ups = []
    for i, v in enumerate(views):
        ups = bw.upstream(v.H, v.W, v.C, 80 + i, dynamic=i == 2)
        all_ups.append(ups)
        v.accum(lib, ups, o)
        r, b, m = _model_of_view(v, ups)
        ref = r if ref is None else {k: ref[k] + r[k] for k in r}
        bar = b if bar is None else {k: bar[k] + b[k] for k in b}
        bar = {k: bar[k] + 2 * bw.U * ref[k].abs() for k in bar}  # one rounding of the running sum per view
        # dL_dmean2D_out receives the last view's screen-space gradient (it is assigned, not accumulated)
        ref["mean2D"], bar["mean2D"] = r["mean2D"], b["mean2D"]
        n = r["mean2D"].norm(dim=1)
        gsum = gsum + n
        gbar = gbar + b["mean2D"].sum(1) + 2 * bw.U * gsum  # sqrt and the running sum: one rounding each
        cnt = cnt + v.visible.double()
    names = {"opacity": "opacity", "mean2D": "mean2D", "means3D": "means3D", "scales": "scales",
             "rotations": "rotations", "sh": "sh"}
    worst = {}
    for k, key in names.items():
        x = o[key].cpu().double().reshape(ref[k].shape[0], -1)[:, :ref[k].reshape(P, -1).shape[1]]
        worst[f"dL_d{k}"] = float(bw._ratio((x - ref[k].reshape(P, -1)).abs(), bar[k].reshape(P, -1)).max())
    worst["grad_accum"] = float(bw._ratio((o["grad_accum"].cpu().double().reshape(-1) - gsum).abs(), gbar).max())
    assert torch.equal(o["denom"].cpu().double().reshape(-1), cnt)
    _report("f3dgs_backward_accum, three views", worst)
    # ViewBatch.backward over the same views
    t = views[0].d
    vb = ViewBatch({k: t[k] for k in ("means3D", "scales", "rotations", "opacities", "shs", "semantic_feature")},
                   densify_stats=False)
    vb.zero_()
    for i, (v, ups) in enumerate(zip(views, all_ups)):
        rs = GaussianRasterizationSettings(**parity.settings(sc, v.cam, "cuda"))
        _, _, _, _, ctx = vb.forward(rs)
        gc, gd = _t(ups[0], dev), _t(ups[2], dev)
        vb.backward(ctx, gc, torch.zeros(t["semantic_feature"].shape[-1], v.H, v.W, device=dev), gd, last=i == 2)
    torch.cuda.synchronize()
    worst = {}
    for k, key in (("opacity", "opacities"), ("means3D", "means3D"), ("scales", "scales"), ("rotations", "rotations"),
                   ("sh", "shs")):
        x = vb.grads[key].cpu().double().reshape(P, -1)
        worst[f"dL_d{k}"] = float(bw._ratio((x - ref[k].reshape(P, -1)).abs(), bar[k].reshape(P, -1)).max())
    _report("ViewBatch.backward, three views", worst)


@pytest.mark.gpu
def test_torch_binding(lib):
    """_C.rasterize_gaussians_backward on one view against the models (its dL/dmeans2D, dL/dopacity and the
    preprocess's outputs)."""
    from diff_gaussian_rasterization import _C

    v = _view("small")
    ups = bw.upstream(v.H, v.W, v.C, 91)
    gc, gf, gd = (_t(u, "cuda") for u in ups)
    e = torch.Tensor([])
    rs = parity.settings(v.sc, v.cam, "cuda")
    g = _C.rasterize_gaussians_backward(v.bg, v.d["means3D"], v.base["radii"], e, v.feats, v.d["scales"],
                                        v.d["rotations"], 1.0, e, rs["viewmatrix"], rs["projmatrix"], rs["tanfovx"],
                                        rs["tanfovy"], gc, gf, gd, v.d["shs"], v.D, rs["campos"], v.base["geom"], v.R,
                                        v.base["binning"], v.base["img"], False)
    ref, bar, _ = _model_of_view(v, ups)
    got = dict(mean2D=g[0][:, :2], opacity=g[3], means3D=g[4], sh=g[6], scales=g[7], rotations=g[8])
    worst = {}
    for k, x in got.items():
        x = x.cpu().double().reshape(v.P, -1)
        worst[f"dL_d{k}"] = float(bw._ratio((x - ref[k].reshape(v.P, -1)).abs(), bar[k].reshape(v.P, -1)).max())
    _report("rasterize_gaussians_backward small", worst)
