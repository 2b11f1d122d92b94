"""The backward's opt-in modes at the benchmark's own views, in tile windows.

test_benchmark_scale.py checks the default forward and backward per pixel and per Gaussian at bench.py's sizes.  The
opt-in variants of the same kernels -- the feature term of dL/dalpha (the feature walk over the backward's per-block
lists), the opacity and inverse-depth planes, antialiasing, float16 feature rows and the scaled float16 map gradient,
the camera gradient, and the lift and score walks -- are checked per entry elsewhere only on small scenes, whose tile
lists, per-block lists and grids are a few hundred times smaller.  Here, on bench.py's scene "c3" (1M Gaussians,
1920x1080, C = 128) in the 4x4-tile windows of test_benchmark_scale.BenchView:
  1. the general backward (f3dgs_backward_alpha_invdepth and its accumulating entry) with the camera gradient on, under
     the planes forward with antialiasing off and on, cameras 0 and 7: the feature term with float32 rows and map
     (assigning), with float16 rows and a float16 map at scale S16 (both entries), and without it (both entries), under
     bench.py's upstream gradients and a static and a dynamic-range set of plane gradients.  Per contained Gaussian:
     the six geometric values against test_alpha_invdepth.planes_model (dL/dopacity as rho g under antialiasing),
     dL/dcolor, dL/dfeature and dL/dz against the blend-weight identities, the accumulating entry's dL_dmean2D_out and
     grad_accum, and denom exactly.  The backward preprocess on test_benchmark_scale's four sets of Gaussians;
  2. the camera gradient against camera_grad_model.terms over every visible Gaussian (in chunks), on the kernel's own
     composite intermediates, with the antialiasing term under antialiasing; and at "c5" (5M Gaussians, 3840x2160),
     where the second-level sum over 128-Gaussian block partials takes ~150 trips per thread instead of the one that
     every small scene gives.  Each entry's bar is printed with the needles' share of it;
  3. the lift and score walks on camera 0 against the same blend weights: pixel_count exactly, weight_sum, max_weight,
     and the lifted feature sums of a 128-channel map;
  4. "c4" (C = 256, two channel chunks): the float32 and float16 cells of 1 on two windows, camera on;
  5. AbsGS through bench.py's step: ViewBatch(absgrad=True) with camera, feature geometry and the planes over c3's 8
     views, mean2D_abs per contained Gaussian of each view's longest-list window against ref_absgrad.abs_mean2d_model,
     and the 8-view step against the sum of the one-view runs;
  6. bench.py's e2e feature loss at its own size: feature_l1_loss_and_grad and resize_bilinear on (C, 1080, 1920) ->
     (C, 480, 853), C = 128 and 256, against a float64 bilinear resize that is F.interpolate's.
Negative controls: one pair's feature term dropped, one lifted (Gaussian, pixel) term dropped and one pair's AbsGS |t|
replaced by its signed t each pass parity's bar and are flagged here; one blended pixel counted for the wrong Gaussian,
which leaves the total count unchanged, fails the exact pixel_count check.
Every 128-Gaussian camera block partial lost or counted twice is flagged (parity's bar flags these too at c3); one
Gaussian's camera terms lost are not: at c3 the 12 needles carry most of some entries' bar.  Every GPU test
prints its wall time and peak device memory and holds the peak under 30 GB (test_benchmark_scale._budget).

CPU (`-m "not gpu"`): the planes model, the AbsGS model and the score and lift identities on windowed Pairs equal their
whole-image values on the contained Gaussians of the oracle views.
"""
import functools
import time
import types

import numpy as np
import pytest
import torch

import blend_weights as bw
import camera_grad_model as cgm
import parity
import ref_absgrad
import scenegen
from test_alpha_invdepth import _backward_planes, _plane_grads, planes_dfn, planes_model
from test_antialiasing import model_gradients
from test_backward_options import AA_BAR, S16, Reference, _inputs, _mask, _zeros_accum, rho_model
from test_benchmark_scale import _VIEWS, _bench_view, _budget, _lib, _oracle_windows, _subset  # noqa: F401
from test_blend_weights import _oracle_view
from test_geometry_grads import NEEDLE_COND_MAX, View, preprocess_check


def _t(a, dev="cpu"):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


class Ratios:
    """Worst |err| / bar per check over a test: each label's values are printed, and the test fails at its end if any
    exceeds 1, so that one run reports every check."""

    def __init__(self):
        self.worst, self.bad = {}, []

    def add(self, label, worst):
        print(f"[{label}] worst |err|/bar: " + ", ".join(f"{k}={v:.3g}" for k, v in worst.items()))
        for k, v in worst.items():
            self.worst[k] = max(self.worst.get(k, 0.0), v)
            if not v <= 1.0:
                self.bad.append((label, k, v))

    def done(self, label):
        print(f"[{label}] largest |err|/bar per check: " + ", ".join(f"{k}={v:.3g}" for k, v in self.worst.items()))
        assert not self.bad, self.bad


# ============================================================================================== CPU: windows checked
@pytest.mark.parametrize("name", ["tiny", "small"])
def test_windowed_option_models_are_the_whole_image_models(name):
    """On each window's contained Gaussians: planes_model with the feature term (six values and their bars), the AbsGS
    model of the colour / planes walk and of the feature walk, and the score and lift identities (pixel counts, weight
    sums and feature sums of a map) equal their whole-image values."""
    sc, cam, f, whole, w = _oracle_view(name)
    W, H, P, C = cam.image_width, cam.image_height, sc.P, sc.C
    HW = W * H
    pl, rg = _t(f["point_list"].astype(np.int64)), _t(f["ranges"].astype(np.int64))
    rec = _t(bw.oracle_records(f))
    gc, gf, gd = bw.upstream(H, W, C, 5)
    ga, gi = _plane_grads(H, W, 6)
    Gc, Gd, GA, GI = _t(gc).reshape(3, -1).t(), _t(gd).reshape(-1), _t(ga).reshape(-1), _t(gi).reshape(-1)
    Gf = _t(gf).reshape(C, -1).t()
    F = _t(sc.features).reshape(P, C)
    bg = torch.tensor(sc.bg)
    bgp = Gc.double() * bg.double()
    bg_dot = (bgp.sum(1) - GA.double(), bgp.abs().sum(1) + GA.double().abs())
    ref_all, bar_all = planes_model(whole, w, rec, P, bg, Gc, Gd, GA, GI, F=F, Gf=Gf)
    dfn = ref_absgrad.planes_dfn(rec, Gc, Gd, GI)
    fdn = ref_absgrad.feature_dfn(F, Gf.t())
    abs_all = ref_absgrad.abs_mean2d_model(whole, w, rec, P, dfn, bg_dot)
    absf_all = ref_absgrad.abs_mean2d_model(whole, w, rec, P, fdn)
    Wt_all = bw.Weights(whole, w, P)
    ones = torch.ones(HW, 1, dtype=torch.float64)
    for tiles in _oracle_windows(W, H):
        win = bw.Pairs(pl, rg, _t(f["n_contrib"].astype(np.int64)), W, H, tiles=tiles)
        ww = w[torch.isin(whole.pix[whole.widx], win.pixels)]
        cont = bw.contained(pl, rg, P, tiles)
        assert int(cont.sum()) > 0
        ref, bar = planes_model(win, ww, rec, P, bg, Gc, Gd, GA, GI, F=F, Gf=Gf)
        # T is a difference of one running sum over all pairs: equal to the whole image's within float64 rounding
        assert float(bw._ratio((ref - ref_all).abs(), bar_all)[cont].max()) < 1e-6
        assert float(bw._ratio((bar - bar_all).abs(), bar_all)[cont].max()) < 1e-6
        for a, b in ((ref_absgrad.abs_mean2d_model(win, ww, rec, P, dfn, bg_dot), abs_all),
                     (ref_absgrad.abs_mean2d_model(win, ww, rec, P, fdn), absf_all)):
            assert float(bw._ratio((a - b).abs(), bar_all[:, :2])[cont].max()) < 1e-6
        Wt = bw.Weights(win, ww, P)
        assert torch.equal(Wt.m[cont], Wt_all.m[cont])  # the score's pixel count
        for G in (ones, Gf):  # the lift's weight_sum and feature_sum
            for a, b in zip(Wt.terms(G), Wt_all.terms(G)):
                assert torch.equal(a[cont], b[cont])
    # the chunked pair products are the one-shot ones
    gid, pix = whole.gid[whole.widx], whole.pix[whole.widx]
    old = bw.PAIR_CHUNK
    try:
        one = bw.pair_dots(F, Gf, gid, pix)
        bw.PAIR_CHUNK = 3 * C + 1
        for a, b in zip(bw.pair_dots(F, Gf, gid, pix), one):
            assert torch.equal(a, b)
        assert torch.equal(fdn(gid, pix)[0], one[0])
        assert torch.equal(planes_dfn(rec, Gc, Gd, GI, F, Gf)(gid, pix)[0],
                           planes_dfn(rec, Gc, Gd, GI)(gid, pix)[0] + one[0])
    finally:
        bw.PAIR_CHUNK = old


# ============================================================================================== GPU
def _view(name, cam, n_windows, **kw):
    """test_benchmark_scale's BenchView of (config, camera, options), the only one held: bench-sized views take GBs."""
    key = (name, cam) + tuple(sorted(kw.items()))
    for k in [k for k in _VIEWS if k != key]:
        del _VIEWS[k]
    torch.cuda.empty_cache()
    return _bench_view(name, cam, n_windows, **kw)


def _win_view(v, win):
    """The attributes test_backward_options.Reference reads from a View, over one window's pairs and weights"""
    return types.SimpleNamespace(pairs=win["pairs"], w=win["w"], P=v.P, C=v.C, W=v.W, H=v.H, bg=v.bg, base=v.base)


def _mids(o):
    return {k: o[k] for k in ("mean2D", "conic", "color", "dz")}


def _f64(a):
    return torch.as_tensor(np.asarray(a) if not isinstance(a, torch.Tensor) else a.cpu()).double()


def camera_whole_view(v, mids, g_eff=None, chunk=1 << 18, rows=None):
    """test_backward_options.camera_reference over every visible Gaussian of the View v, in chunks of Gaussians: the
    reference, its bar and its scale are sums over Gaussians, kmax (the antialiasing term's weight) a max.  mids: the
    composite intermediates; g_eff: dL/dop_eff under antialiasing.  -> dict(ref, bar [35], needle [35]: the needles'
    share of the bar, n_needles, blocks [ceil(P / 128), 35]: the reference's terms summed per 128-Gaussian block of the
    backward preprocess, scale [35] (the bar's scale before the floor), and with rows (Gaussian ids) terms: their own
    [n, 35] terms in the order of rows_seen)."""
    sc, cam = v.sc, v.cam
    idx_all = v.visible.nonzero().flatten()
    cov = cgm.cov3d_from_scale_rot(_f64(sc.scales), _f64(sc.rotations), v.mod)
    means = _f64(sc.means3D)
    vm, pm, cp = v.vm.cpu(), v.pm.cpu(), v.cp.cpu()
    shs = v.shs.cpu() if v.M else None
    g = [mids[k].cpu() for k in ("mean2D", "conic", "color", "dz")]
    z = lambda: torch.zeros(35, dtype=torch.float64)  # noqa: E731
    ref, scale, well, m_cam = z(), z(), z(), z()
    blocks = torch.zeros((v.P + 127) // 128, 35, dtype=torch.float64)
    kmax, n_needles = 1.0, 0
    own, seen = [], []
    for s in range(0, idx_all.numel(), chunk):
        idx = idx_all[s:s + chunk]
        t = cgm.terms(means[idx], cov[idx], vm, pm, cp, [x[idx] for x in g], v.W, v.H, cam.tanfovx, cam.tanfovy, v.D,
                      shs=None if shs is None else shs[idx])
        ref += cgm.camera_vector(t)
        scale += cgm.camera_scale(t)
        well += cgm.camera_scale(t, needles=False)
        n_needles += int((t["eig_ratio"] > NEEDLE_COND_MAX).sum())
        per = torch.cat([t["vm"], t["pm"], t["campos"]], 1)
        blocks.index_add_(0, idx // 128, per)
        if rows is not None:
            hit = torch.isin(idx, rows)
            own.append(per[hit])
            seen.append(idx[hit])
        del t
        if g_eff is not None:
            m = model_gradients(sc, cam, [g[0], g[1], g_eff.cpu(), g[2], g[3]], idx, mod=v.mod)
            m_cam += m["camera"]
            ok = m["eig_ratio"][idx] <= NEEDLE_COND_MAX
            if bool(ok.any()):
                kmax = max(kmax, float(m["kappa"][idx].clamp_min(1.0)[ok].max()))
            del m
    needles = scale - well  # the needles' conic share, counted at |term| / 1e-5
    if g_eff is not None:
        scale = scale + (m_cam - ref).abs() * kmax
        ref = m_cam
    bar = 1e-5 * scale + 1e-7 * float(well.max())
    out = dict(ref=ref, bar=bar, needle=1e-5 * needles / bar, n_needles=n_needles, blocks=blocks, scale=scale)
    if rows is not None:
        out["terms"], out["rows_seen"] = torch.cat(own), torch.cat(seen)
    return out


def _camera_ratio(ours, cr):
    return float(((ours.cpu().double() - cr["ref"]).abs() / cr["bar"]).max())


def _preprocess_sets(bv):
    """test_benchmark_scale's check-4 sets: the windows' contained Gaussians, the 2000 largest radii, every visible
    Gaussian whose screen mean is outside the image, and a seeded 50k sample of the visible ones."""
    v, P = bv.v, bv.P
    vis = v.base["radii"] > 0
    radii = torch.where(vis, v.base["radii"], torch.zeros_like(v.base["radii"]))
    mean = v.base["rec"][:, 0:2]
    outside = vis & ((mean[:, 0] < 0) | (mean[:, 0] >= bv.W) | (mean[:, 1] < 0) | (mean[:, 1] >= bv.H))
    g = torch.Generator(device="cuda").manual_seed(5)
    vis_idx = vis.nonzero().flatten()
    contained = torch.zeros(P, dtype=torch.bool, device="cuda")
    for win in bv.windows.values():
        contained |= win["contained"]
    return {"contained": contained.nonzero().flatten(), "largest radii": torch.topk(radii, 2000).indices,
            "mean outside the image": outside.nonzero().flatten(),
            "sample": vis_idx[torch.randperm(vis_idx.numel(), device="cuda", generator=g)[:50000]]}


def _preprocess(bv, o, g_eff, label, R):
    """The preprocess outputs of the assigning call o on the four sets: preprocess_chain without antialiasing,
    model_gradients (test_antialiasing's bar, needles skipped) and the chain's dL/dsh with it."""
    v, P = bv.v, bv.P
    sets = _preprocess_sets(bv)
    idx = torch.unique(torch.cat(list(sets.values())))
    s = _subset(v, idx)
    ch = s.chain({k: x[idx] for k, x in _mids(o).items()})
    outs = {k: x[idx] for k, x in v.outputs(o).items()}
    pos = torch.searchsorted(idx, torch.arange(P, device="cuda")).clamp(max=idx.numel() - 1)
    if g_eff is not None:
        ic = idx.cpu()
        m = model_gradients(v.sc, v.cam, [o["mean2D"].cpu(), o["conic"].cpu(), g_eff.cpu(), o["color"].cpu(),
                                          o["dz"].cpu()], ic, mod=v.mod)
        m = {k: (x[ic] if x.dim() and x.shape[0] == P else x) for k, x in m.items()}
    for name, members in sets.items():
        mask = torch.zeros(idx.numel(), dtype=torch.bool)
        mask[pos[members].cpu()] = True
        tag = f"{label} preprocess {name} ({members.numel()}, needles {int((mask & (ch['eig_ratio'] > NEEDLE_COND_MAX)).sum())})"
        if g_eff is None:
            R.add(tag, preprocess_check(ch, outs, mask))
            continue
        # test_backward_options.aa_preprocess_check on the set's rows
        well = (m["eig_ratio"] <= NEEDLE_COND_MAX) & mask
        k = m["kappa"].clamp_min(1.0)
        worst = {}
        for key in [x for x in outs if x in m and x != "sh"]:
            n = outs[key].cpu().double().reshape(idx.numel(), -1)
            r = m[key]
            floor = 1e-6 * float(r[well].abs().max()) + 1e-12 if bool(well.any()) else 1e-12
            bar = AA_BAR * k[:, None] * r.abs().sum(1, keepdim=True) + floor
            ratio = ((n - r).abs() / bar)[well]
            worst[f"dL_d{key}"] = float(ratio.max()) if ratio.numel() else 0.0
        worst.update(preprocess_check({k: ch[k] for k in ("sh", "mag_sh", "eig_ratio")}, {"sh": outs["sh"]}, mask))
        R.add(tag, worst)


# (feature rows, map, entries): the feature term with float32 rows and map, with float16 rows and a float16 map, and
# without it.  Each group also runs its assigning call: the camera check of the accumulating entry reads its
# intermediates.
CELLS = (("f32", "f32", ("assign",)), ("f16", "f16", ("assign", "accum")), ("none", "f32", ("assign", "accum")))


def check_options(bv, label, R, cells=CELLS, plane_sets=(False, True), camera=True, preprocess=True):
    """Item 1 (and 2 with camera) on BenchView bv -> the outputs of the first cell's assigning call, its g_eff, and the
    inputs (ups, ga, gi) it ran on."""
    v, P, C = bv.v, bv.P, bv.sc.C
    aa = v.antialiasing
    lib = _lib()
    ups = scenegen.upstream_grads(bv.H, bv.W, C, seed=99)
    vis = v.base["radii"] > 0
    cont = torch.zeros(P, dtype=torch.bool, device="cuda")
    for win in bv.windows.values():
        cont |= win["contained"]
    t0 = time.time()
    rho = rho_model(bv.sc, bv.cam, cont.nonzero().flatten().cpu(), v.mod) if aa else None
    if aa:
        print(f"[{label}] rho of {int(cont.sum())} contained Gaussians: {time.time() - t0:.1f} s")
    first = None
    for dyn in plane_sets:
        ga, gi = _plane_grads(bv.H, bv.W, 90 + int(dyn), dynamic=dyn)
        ulabel = "dynamic planes" if dyn else "static planes"
        for feat, mp, entries in cells:
            sf, gmap, scale = _inputs(v, ups, feat, mp)
            call = functools.partial(_backward_planes, lib, v, (ups[0], gmap, ups[2]), ga, gi, sf=sf, aa=int(aa),
                                     map_scale=scale)
            outs = {"assign": call(camera=camera)}
            if "accum" in entries:
                outs["accum"] = call(camera=camera, accum=_zeros_accum(v, camera))
                assert torch.equal(outs["accum"]["denom"], vis.float()), (label, feat, mp)
            g_eff = call(aa=0)["opacity"] if aa else None
            if first is None:
                first = (outs["assign"], g_eff, (ups, ga, gi))
            tag = f"{label} feat={feat} map={mp} {ulabel}"
            for name, win in bv.windows.items():
                ref = Reference(_win_view(v, win), ups, ga, gi, sf, gmap, scale)
                rows = win["contained"]
                for entry in entries:
                    o = outs[entry]
                    if entry == "assign":
                        worst = ref.composite(o, rho, rows=rows)
                        if aa:
                            worst["dL_dop_eff"] = ref.opacity(g_eff, rows=rows)
                    else:
                        worst = ref.accumulated(o, rho, rows=rows)
                    worst["dL_dfeature"] = ref.features(o["feat"], rows)
                    R.add(f"{tag} {entry} {name} ({int(rows.sum())} contained)", worst)
                del ref
            if camera:
                t0 = time.time()
                cr = camera_whole_view(v, _mids(outs["assign"]), g_eff)
                worst = {f"dL_dcamera {e}": _camera_ratio(outs[e]["camera"], cr) for e in outs}
                print(f"[{tag}] camera over {int(vis.sum())} visible Gaussians ({cr['n_needles']} needles) in "
                      f"{time.time() - t0:.1f} s; needles' share of the bar: max {float(cr['needle'].max()):.3g}, "
                      f"median {float(cr['needle'].median()):.3g}")
                R.add(tag + " camera", worst)
            if preprocess and first[0] is outs["assign"]:
                _preprocess(bv, outs["assign"], g_eff, tag, R)
            del outs
    return first


@pytest.mark.gpu
@pytest.mark.parametrize("cam,aa", [(7, True), (7, False), (0, True), (0, False)])
def test_c3_options_per_gaussian(built, cam, aa):
    """Items 1 and 2 at c3: every cell on seven windows, the camera gradient over the whole view."""
    bv = _view("c3", cam, 7, planes=True, antialiasing=aa)
    R = Ratios()
    check_options(bv, f"c3 cam {cam} aa={int(aa)}", R)
    R.done(f"c3 cam {cam} aa={int(aa)}")


@pytest.mark.gpu
def test_c3_negative_controls_options(built):
    """At c3 camera 0 (antialiasing off), perturbations that parity's bar passes and these checks flag:
    the camera gradient with any one 128-Gaussian block partial dropped or counted twice (the float64 reference's own
    terms of the block; parity's bar flags these too), and dL/dopacity with one pair's feature term dropped for a contained Gaussian of the
    longest-list window."""
    bv = _view("c3", 0, 7, planes=True, antialiasing=False)
    v, P, C = bv.v, bv.P, bv.sc.C
    lib = _lib()
    ups = scenegen.upstream_grads(bv.H, bv.W, C, seed=99)
    ga, gi = _plane_grads(bv.H, bv.W, 90)
    sf, gmap, scale = _inputs(v, ups, "f32", "f32")
    o = _backward_planes(lib, v, (ups[0], gmap, ups[2]), ga, gi, sf=sf, map_scale=scale, camera=True)
    flagged = {}
    # the camera: a 128-Gaussian block partial dropped or counted twice.  Parity's bar on the 35 floats itself flags
    # the loss of most blocks at c3, so each block's partial is reported against both bars, and the control is the
    # finest such error: one contained Gaussian of the longest-list window (one thread's terms) dropped or counted
    # twice, the one the bar flags most among those parity's bar passes
    win = bv.windows["longest list"]
    cidx = win["contained"].nonzero().flatten().cpu()
    cr = camera_whole_view(v, _mids(o), rows=cidx)
    ours = o["camera"].cpu().double()
    assert _camera_ratio(ours, cr) <= 1.0

    def passes_parity(x):
        return parity.float_mismatch(x.float().numpy(), ours.float().numpy(), parity.RTOL, parity.GRAD_ATOL_REL)[0] <= 1

    nz = (cr["blocks"].abs().sum(1) > 0).nonzero().flatten()
    per_block = (cr["blocks"][nz].abs() / cr["bar"]).max(1).values
    by_parity = [not passes_parity(ours - cr["blocks"][int(c)]) for c in nz]
    print(f"[c3 controls] camera: one of the {nz.numel()} block partials with visible Gaussians dropped is flagged "
          f"by this bar for {float((per_block > 1).double().mean()):.4f} of them (median ratio "
          f"{float(per_block.median()):.3g}), by parity's bar for {sum(by_parity) / nz.numel():.4f}")
    # every block partial lost or counted twice is flagged; one Gaussian's terms are below this bar at c3 (the needles
    # carry most of some entries' bar), so single-Gaussian losses are only reported
    flagged["camera, the least flagged block partial dropped or counted twice"] = float(per_block.min())
    cand = [i for i in range(cidx.numel()) if passes_parity(ours - cr["terms"][i])]
    print(f"[c3 controls] camera: of the {cidx.numel()} contained Gaussians of the window, {len(cand)} have terms whose "
          f"loss parity passes; this bar flags {sum(float((cr['terms'][j].abs() / cr['bar']).max()) > 1 for j in cand)}"
          f" of them")
    # the feature term of one pair of a contained Gaussian whose dL/dopacity is under parity's floor
    pairs, w = win["pairs"], win["w"]
    rec = v.base["rec"]
    HW = bv.W * bv.H
    Gc, Gd = _t(ups[0], "cuda").reshape(3, HW).t(), _t(ups[2], "cuda").reshape(HW)
    GA, GI = _t(ga, "cuda").reshape(HW), _t(gi, "cuda").reshape(HW)
    Gf = gmap.reshape(C, HW).t()
    F = sf.reshape(P, C)
    ref, bar = planes_model(pairs, w, rec, P, v.bg, Gc, Gd, GA, GI, F=F, Gf=Gf)
    op = o["opacity"].double()
    floor = parity.GRAD_ATOL_REL * float(op.abs().max())
    under = (win["contained"] & (op.abs() < floor) & (op.abs() > 0)).nonzero().flatten()
    assert under.numel() > 0
    g0 = int(under[under.numel() // 2])
    on = (pairs.gid[pairs.widx] == g0) & (w > 0)
    gid0, pix0 = pairs.gid[pairs.widx][on], pairs.pix[pairs.widx][on]
    p0 = int(pix0[torch.argmax(bw.pair_dots(F, Gf, gid0, pix0)[1])])
    full, nof = planes_dfn(rec, Gc, Gd, GI, F, Gf), planes_dfn(rec, Gc, Gd, GI)

    def dropped(gid, pix):
        d, dabs = full(gid, pix)
        hit = (gid == g0) & (pix == p0)
        return torch.where(hit, nof(gid, pix)[0], d), dabs

    bgp = Gc.double() * v.bg.double()
    ref2, _ = bw.composite_model(pairs, w, rec, P, dropped, 6 + C,
                                 (bgp.sum(1) - GA.double(), bgp.abs().sum(1) + GA.double().abs()))
    x = op.clone()
    x[g0] += ref2[g0, 5] - ref[g0, 5]
    assert parity.float_mismatch(x.cpu().numpy(), op.cpu().numpy(), parity.RTOL, parity.GRAD_ATOL_REL)[0] <= 1.0
    assert float(bw._ratio((op[g0] - ref[g0, 5]).abs(), bar[g0, 5])) <= 1.0
    flagged["dL_dopacity, one pair's feature term dropped"] = float(bw._ratio((x[g0] - ref[g0, 5]).abs(), bar[g0, 5]))
    print(f"[c3 negative controls: Gaussian {g0} at pixel {p0}] flag ratios: "
          + ", ".join(f"{k}={r:.3g}" for k, r in flagged.items()))
    for lab, r in flagged.items():
        assert r > 1.0, (lab, r)


@pytest.mark.gpu
def test_c3_scores_and_lift(built):
    """Item 3 on camera 0, default forward, seven windows: gaussian_scores_accum's pixel_count exactly the blended
    pairs of every contained Gaussian, its weight_sum and max_weight within test_gaussian_scores' bars;
    lift_features_accum of bench.py's 128-channel map within the per-Gaussian identity bars.  Negative controls: one
    pixel counted for the wrong Gaussian, one lifted (Gaussian, pixel) term dropped."""
    from diff_gaussian_rasterization import _C
    from test_gaussian_scores import _scores

    bv = _view("c3", 0, 7)
    v, P, C, W, H = bv.v, bv.P, bv.sc.C, bv.W, bv.H
    b = v.base
    ws, mw, pc = _scores(b, P, W, H)
    G = _t(scenegen.upstream_grads(H, W, C, seed=99)[1], "cuda")
    fs, wl = torch.zeros(P, C, device="cuda"), torch.zeros(P, device="cuda")
    _C.lift_features_accum(b["geom"], b["R"], b["binning"], b["img"], G, fs, wl)
    Gp = G.reshape(C, -1).t()
    ones = torch.ones(W * H, 1, device="cuda")
    R = Ratios()
    for name, win in bv.windows.items():
        Wt, rows, pairs, w = win["Wt"], win["contained"], win["pairs"], win["w"]
        assert torch.equal(pc[rows], Wt.m[rows].long()), name
        blended = w > 0
        idx = pairs.widx[blended]
        g, n = pairs.gid[idx], pairs.n[pairs.pix[idx]].double()
        wb = w[blended].double()
        ref = torch.zeros(P, dtype=torch.float64, device="cuda").scatter_reduce_(0, g, wb, "amax")
        bar = torch.zeros(P, dtype=torch.float64, device="cuda").scatter_reduce_(0, g, bw.K * bw.U * (2 * n + 4) * wb,
                                                                                 "amax")
        R.add(f"c3 scores and lift {name} ({int(rows.sum())} contained, pixel_count exact, "
              f"{int(Wt.m[rows].max())} pixels at most)",
              {"weight_sum": Wt.per_gaussian(ws.reshape(P, 1), ones, rows),
               "max_weight": float(bw._ratio((mw.double() - ref).abs(), bar)[rows].max()),
               "lift weight_sum": Wt.per_gaussian(wl.reshape(P, 1), ones, rows),
               "lift feature_sum": Wt.per_gaussian(fs, Gp, rows)})
    R.done("c3 scores and lift")
    # controls on the longest-list window: a contained Gaussian with the lifted row under parity's floor
    win = bv.windows["longest list"]
    Wt, rows, pairs, w = win["Wt"], win["contained"], win["pairs"], win["w"]
    # one blended pixel counted for the wrong Gaussian: the total, which test_gaussian_scores checks, is unchanged
    cidx = rows.nonzero().flatten()
    gs, gs2 = int(cidx[cidx.numel() // 2]), int(cidx[cidx.numel() // 2 + 1])
    x = pc.clone()
    x[gs] += 1
    x[gs2] -= 1
    assert int(x.sum()) == int(pc.sum())
    assert not torch.equal(x[rows], Wt.m[rows].long())  # the exact per-Gaussian check sees it
    flagged = {}
    fsd = fs.double()
    floor = parity.GRAD_ATOL_REL * float(fsd.abs().max())
    under = (rows & (fsd.abs().max(1).values < floor) & (fsd.abs().max(1).values > 0)).nonzero().flatten()
    assert under.numel() > 0
    gq = int(under[under.numel() // 2])
    on = (pairs.gid[pairs.widx] == gq) & (w > 0)
    pix = pairs.pix[pairs.widx][on]
    terms = w[on].double()[:, None] * Gp[pix].double()
    med = int(torch.argsort(terms.abs().sum(1))[pix.numel() // 2])
    y = fsd.clone()
    y[gq] -= terms[med]
    assert parity.float_mismatch(y.cpu().numpy(), fsd.cpu().numpy(), parity.RTOL, parity.GRAD_ATOL_REL)[0] <= 1.0
    one = torch.zeros(P, dtype=torch.bool, device="cuda")
    one[gq] = True
    flagged["lift, one (g, p) term dropped"] = Wt.per_gaussian(y, Gp, one)
    print(f"[c3 score / lift negative controls: Gaussians {gs}, {gq}] flag ratios: "
          + ", ".join(f"{k}={r:.3g}" for k, r in flagged.items()))
    for lab, r in flagged.items():
        assert r > 1.0, (lab, r)


@pytest.mark.gpu
def test_c4_two_channel_chunks_options(built):
    """Item 4: c4 (C = 256), antialiasing off, two windows: the float32 and the float16 cells of item 1 (the float16 one
    through both entries), with the camera gradient over the whole view."""
    bv = _view("c4", 0, 2, planes=True)
    R = Ratios()
    check_options(bv, "c4", R, cells=(("f32", "f32", ("assign",)), ("f16", "f16", ("assign", "accum"))),
                  preprocess=False)
    R.done("c4")


@pytest.mark.gpu
def test_c5_camera_gradient(built):
    """Item 2 at c5 (5M Gaussians, 3840x2160, 39063 block partials): the default forward and the general backward with
    zero plane gradients and the camera gradient, against the float64 reference over every visible Gaussian."""
    _VIEWS.clear()  # frees the held view
    torch.cuda.empty_cache()
    sc = scenegen.make_config("c5", views=1)
    cam = sc.cameras[0]
    v = View(sc, cam, C=sc.C, weights=False)
    del v.base["fmap"], v.base["point_list"]
    ups = scenegen.upstream_grads(v.H, v.W, sc.C, seed=99)
    z = np.zeros((1, v.H, v.W), np.float32)
    o = _backward_planes(_lib(), v, ups, z, z, camera=True)
    del ups
    t0 = time.time()
    cr = camera_whole_view(v, _mids(o))
    print(f"[c5] camera over {int(v.visible.sum())} visible Gaussians ({cr['n_needles']} needles) in "
          f"{time.time() - t0:.1f} s; needles' share of the bar: max {float(cr['needle'].max()):.3g}, median "
          f"{float(cr['needle'].median()):.3g}")
    R = Ratios()
    R.add("c5 camera", {"dL_dcamera": _camera_ratio(o["camera"], cr)})
    R.done("c5")


# ------------------------------------------------------------------------------ the e2e feature loss at bench.py's size
def _taps(n_in, n_out, r32=True, dev="cuda"):
    """The bilinear taps of align_corners=True along one axis -> (i0, i1, l0, l1) with l0, l1 float64.  r32: as the
    kernel forms them (feature_head.cu src_of: r = (in - 1) / (out - 1) and s = r o in float32, l0 = 1 - l1 in float32);
    else in float64, as F.interpolate does."""
    o = torch.arange(n_out, device=dev)
    if r32:
        r = float(np.float32(n_in - 1) / np.float32(n_out - 1)) if n_out > 1 else 0.0
        s = torch.tensor(r, dtype=torch.float32, device=dev) * o.float()
    else:
        s = o.double() * ((n_in - 1) / (n_out - 1) if n_out > 1 else 0.0)
    i0 = s.floor().long()
    i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
    l1 = s - i0.to(s.dtype)
    l0 = 1 - l1
    return i0, i1, l0.double(), l1.double()


def _bilinear64(x, Hg, Wg, r32=True):
    """[C, Hg, Wg] float64 bilinear resize of x [C, H, W] (any float type) with _taps' coordinates."""
    C, H, W = x.shape
    y0, y1, ly0, ly1 = _taps(H, Hg, r32, x.device)
    x0, x1, lx0, lx1 = _taps(W, Wg, r32, x.device)
    out = torch.empty(C, Hg, Wg, dtype=torch.float64, device=x.device)
    for c in range(C):  # one channel at a time: a float64 copy of the whole map is 2 GB at C = 128
        xc = x[c].double()
        rows = xc[:, x0] * lx0 + xc[:, x1] * lx1
        out[c] = rows[y0] * ly0[:, None] + rows[y1] * ly1[:, None]
    return out


def _bilinear64_t(d, H, W):
    """The transpose of _bilinear64 (kernel's coordinates) applied to d [C, Hg, Wg] -> [C, H, W] float64."""
    C, Hg, Wg = d.shape
    y0, y1, ly0, ly1 = _taps(H, Hg, True, d.device)
    x0, x1, lx0, lx1 = _taps(W, Wg, True, d.device)
    out = torch.empty(C, H, W, dtype=torch.float64, device=d.device)
    for c in range(C):
        dc = d[c].double()
        rows = torch.zeros(H, Wg, dtype=torch.float64, device=d.device)
        rows.index_add_(0, y0, dc * ly0[:, None]).index_add_(0, y1, dc * ly1[:, None])
        oc = torch.zeros(H, W, dtype=torch.float64, device=d.device)
        oc.index_add_(1, x0, rows * lx0).index_add_(1, x1, rows * lx1)
        out[c] = oc
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("C", [128, 256])
def test_feature_l1_at_bench_size(built, C):
    """bench.py's e2e feature loss, feature_l1_loss_and_grad on a (C, 1080, 1920) map against its (C, 480, 853) teacher
    (C = 128: c3, C = 256: c4), against float64:
      * resize_bilinear per element within 4 u of the magnitude of its four weighted taps (u, the float32 unit
        roundoff: two products and sums per axis), on the kernel's float32 coordinates; those coordinates within
        2 u s of F.interpolate's, and the float64 resize on them is F.interpolate's on float64 coordinates;
      * the loss: the per-element errors plus the float32 sums' (each lane's running sum, 8 shuffle levels and one
        atomic per CTA: u (n_lane + 8 + CTAs) sum |d|) and the final scaling's;
      * the sign gradient exact wherever |interp - gt| exceeds the element's resize bar;
      * the resize backward (the gather transpose) per element within 4 u of the magnitude of its weighted terms (one tap
        per axis at this ratio, two at most)."""
    import torch.nn.functional as Fn
    from diff_gaussian_rasterization import feature_head as fh

    H, W = 1080, 1920
    Hg, Wg = max(int(round(H / 2.25)), 1), max(int(round(W / 2.25)), 1)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(C, H, W, device="cuda", generator=g)
    gt = torch.rand(C, Hg, Wg, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    u = bw.U
    # the coordinates and the float64 model against F.interpolate
    for n_in, n_out in ((H, Hg), (W, Wg)):
        a, b = _taps(n_in, n_out), _taps(n_in, n_out, r32=False)
        s32, s64 = a[0].double() + a[3], b[0].double() + b[3]
        assert bool(((s32 - s64).abs() <= 2 * u * s64).all())
    xs = x[:2, :64, :96]
    assert torch.allclose(_bilinear64(xs, 27, 43, r32=False),
                          Fn.interpolate(xs.double()[None], (27, 43), mode="bilinear", align_corners=True)[0],
                          rtol=1e-12, atol=1e-12)
    ref = _bilinear64(x, Hg, Wg)
    mag = _bilinear64(x.abs(), Hg, Wg)
    bar = 4 * u * mag
    got = fh.resize_bilinear(x, (Hg, Wg))
    worst = {"resize_bilinear": float(bw._ratio((got.double() - ref).abs(), bar).max())}
    del got
    loss, grad = fh.feature_l1_loss_and_grad(x, gt, 1.0)
    n = C * Hg * Wg
    d = ref - gt.double()
    ad = float(d.abs().sum())
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    warps_per_cta = 8
    ctas = min((C * Hg + warps_per_cta - 1) // warps_per_cta, sms * 8)
    n_lane = -(-Wg // 32) * -(-(C * Hg) // (ctas * warps_per_cta))
    lbar = (float(bar.sum()) + u * (n_lane + 8 + ctas + 1) * ad) / n + 2 * u * ad / n
    worst["loss"] = abs(float(loss) - ad / n) / lbar
    # the sign map the backward reads: sign(interp - gt) exactly where the element is farther from gt than its bar
    sign, _ = fh._C().feature_resize_fwd(x, gt, Hg, Wg, 1.0)
    sure = d.abs() > bar + u * gt.double().abs()
    wrong = int((sign.double()[sure] != torch.sign(d[sure])).sum())
    print(f"[feature L1 C={C}] {n} elements, {int((~sure).sum())} within their bar of gt")
    assert wrong == 0, wrong
    assert bool((sign.abs() <= 1).all())
    del d, ref, mag, bar, sure
    # the backward: the kernel's own signs through the float64 transpose, a few channels at a time
    scale = np.float32(1.0 / n)
    dout = sign * float(scale)
    del sign
    rb = 0.0
    for c in range(0, C, 16):
        gref = _bilinear64_t(dout[c:c + 16], H, W)
        gmag = _bilinear64_t(dout[c:c + 16].abs(), H, W)
        rb = max(rb, float(bw._ratio((grad[c:c + 16].double() - gref).abs(), 4 * u * gmag).max()))
        del gref, gmag
    worst["resize backward"] = rb
    R = Ratios()
    R.add(f"feature L1 C={C} ({C}, {H}, {W}) -> ({Hg}, {Wg})", worst)
    R.done(f"feature L1 C={C}")


# ------------------------------------------------------------------------------------- AbsGS through bench.py's step
@pytest.mark.gpu
def test_c3_absgrad_view_batch(built):
    """ViewBatch(absgrad=True) with camera, feature_geometry and the planes forward over c3's 8 views, under bench.py's
    upstream gradients and plane gradients:
      * per view, on the contained Gaussians of its longest-list window: mean2D_abs against ref_absgrad.abs_mean2d_model,
        the colour / planes walk (with its background and gA terms) plus the feature walk's |terms|, within the sum of
        the two walks' composite_model bars on dL/dmean2D (no tensor-wide floor);
      * the 8-view step against the 8 one-view runs: denom exactly; grad_accum_abs, each view's norm of sums of
        non-negative terms (at most n_v = 2 (8 instances + 1) float adds onto the buffer per view and walk, in an order the
        run does not fix, so within 2 u n_v of it on either component), within 2 u (2 sum_v n_v + 10) (1 + 1e-3) of the
        one-view sum; dL/dfeature within test_benchmark_scale's step bar.
    Negative control: one pair's |t| replaced by its signed t, for a contained Gaussian under parity's floor."""
    from diff_gaussian_rasterization import GaussianRasterizationSettings, _C
    from diff_gaussian_rasterization.parallel import ViewBatch
    from test_benchmark_scale import BenchView, _scene

    _VIEWS.clear()
    torch.cuda.empty_cache()
    sc = _scene("c3")
    P, C = sc.P, sc.C
    t = scenegen.to_torch(sc, "cuda")
    params = {k: t[k] for k in ("means3D", "scales", "rotations", "opacities", "shs", "semantic_feature")}
    cam0 = sc.cameras[0]
    H, W = cam0.image_height, cam0.image_width
    HW = H * W
    gc, gf, gd = (_t(u, "cuda") for u in scenegen.upstream_grads(H, W, C, seed=99))
    ga, gi = (_t(a, "cuda") for a in _plane_grads(H, W, 90))
    rss = [GaussianRasterizationSettings(**parity.settings(sc, cam, "cuda")) for cam in sc.cameras]
    kw = dict(camera=True, feature_geometry=True, g_alpha=ga, g_invdepth=gi)
    vb = ViewBatch(params, absgrad=True)
    vb.zero_()
    for i, rs in enumerate(rss):
        *_, ctx = vb.forward_alpha_invdepth(rs)
        vb.backward(ctx, gc, gf, gd, last=i == len(rss) - 1, **kw)
    step_feat, step_denom = vb.grads["semantic_feature"].reshape(P, C).clone(), vb.denom.clone()
    step_abs = vb.grad_accum_abs.clone()
    z = lambda *s: torch.zeros(*s, dtype=torch.float64, device="cuda")  # noqa: E731
    xsum, asum, abs_sum, N, Na = z(P, C), z(P, C), z(P), z(P), z(P)
    count = torch.zeros(P, device="cuda")
    Gc, Gd = gc.reshape(3, HW).t(), gd.reshape(HW)
    GA = ga.reshape(HW).double()
    F = params["semantic_feature"].reshape(P, C)
    R = Ratios()
    control = None
    for vi, (cam, rs) in enumerate(zip(sc.cameras, rss)):
        runs = {}
        for G in (gf, gf.abs()):
            vb.zero_()
            *_, radii, _, _, _, ctx = vb.forward_alpha_invdepth(rs)
            vb.backward(ctx, gc, G, gd, last=True, **kw)
            runs[G is gf] = (vb.grads["semantic_feature"].reshape(P, C).double(), vb.mean2D_abs.clone(),
                             vb.grad_accum_abs.double())
        xsum += runs[True][0]
        asum += runs[False][0]
        abs_sum += runs[True][2]
        ours = runs[True][1]
        count += (radii > 0).float()
        pl, _, n_contrib, _, _ = _C.debug_views(ctx.geom, ctx.binning, ctx.img, P, W, H, ctx.num_rendered)
        inst = torch.bincount(pl.long(), minlength=P).double()
        N += 8 * inst + 1
        Na += 2 * (8 * inst + 1)
        # the view's longest-list window, from its own planes forward
        bv = BenchView(sc, cam, 1, planes=True)
        v = bv.v
        assert torch.equal(v.base["n_contrib"], n_contrib) and torch.equal(v.base["point_list"], pl)
        win = bv.windows["longest list"]
        pairs, w, rows, rec = win["pairs"], win["w"], win["contained"], v.base["rec"]
        bgp = Gc.double() * v.bg.double()
        bg_dot = (bgp.sum(1) - GA, bgp.abs().sum(1) + GA.abs())
        dfn = ref_absgrad.planes_dfn(rec, Gc, Gd, gi.reshape(HW))
        fd = ref_absgrad.feature_dfn(F, gf.reshape(C, HW))
        ref, t_pairs, t_gid = ref_absgrad.abs_mean2d_model(pairs, w, rec, P, dfn, bg_dot, signed=True)
        ref = ref + ref_absgrad.abs_mean2d_model(pairs, w, rec, P, fd)
        bar = (bw.composite_model(pairs, w, rec, P, dfn, 5, bg_dot)[1] +
               bw.composite_model(pairs, w, rec, P, fd, C)[1])[:, :2]
        got = ours[:, :2].double()
        R.add(f"c3 view {vi} AbsGS mean2D_abs ({int(rows.sum())} contained)",
              {"mean2D_abs": float(bw._ratio((got - ref).abs(), bar)[rows].max())})
        assert bool((ours[:, 2] == 0).all()) and bool((ours[radii == 0] == 0).all())
        if vi == 0:  # the control: one pair's |t_x| replaced by t_x, on a contained Gaussian under parity's floor
            floor = parity.GRAD_ATOL_REL * float(got[:, 0].abs().max())
            under = (rows & (got[:, 0] < floor) & (got[:, 0] > 0)).nonzero().flatten()
            # each such Gaussian's most negative t_x flipped: the share the bar flags, and the control on the one it
            # flags most (the bar is composite_model's, made for signed sums: loose for a sum of |t|)
            neg = torch.isin(t_gid, under) & (t_pairs[:, 0] < 0)
            assert bool(neg.any())
            tmin = torch.zeros(P, dtype=torch.float64, device="cuda").scatter_reduce_(0, t_gid[neg], t_pairs[neg, 0],
                                                                                      "amin")
            cand = torch.unique(t_gid[neg])
            flip = bw._ratio((got[cand, 0] - 2 * tmin[cand].abs() - ref[cand, 0]).abs(), bar[cand, 0])
            g0 = int(cand[torch.argmax(flip)])
            x = got.clone()
            x[g0, 0] -= 2 * tmin[g0].abs()
            assert parity.float_mismatch(x.cpu().numpy(), got.cpu().numpy(), parity.RTOL, parity.GRAD_ATOL_REL)[0] <= 1
            control = (g0, float(bw._ratio((x[g0, 0] - ref[g0, 0]).abs(), bar[g0, 0])),
                       float((flip > 1).double().mean()), cand.numel())
        del bv, v, win, pairs, w, ref, bar, t_pairs, t_gid, runs
        torch.cuda.empty_cache()
    assert torch.equal(step_denom, count)
    worst = {"grad_accum_abs": float(bw._ratio((step_abs.double() - abs_sum).abs(),
                                               2 * bw.U * (2 * Na + 10) * (1 + 1e-3) * abs_sum).max()),
             "dL_dfeature": float(bw._ratio((step_feat.double() - xsum).abs(),
                                            2 * bw.U * N[:, None] * (1 + 1e-3) * asum).max())}
    R.add("c3 8-view AbsGS step (denom exact)", worst)
    print(f"[c3 AbsGS negative control: Gaussian {control[0]}] one pair's |t| replaced by t: flag ratio "
          f"{control[1]:.3g}; of the {control[3]} contained Gaussians under parity's floor, the flip of the most "
          f"negative term is flagged for {control[2]:.3f}")
    R.done("c3 AbsGS")
    assert control[1] > 1.0
