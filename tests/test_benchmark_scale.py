"""The composite per pixel and per Gaussian at the benchmark's own views, in tile windows.

The per-entry checks of test_blend_weights.py and test_geometry_grads.py run on small scenes.  At bench.py's sizes
(scenegen "c3": 1M Gaussians, 1920x1080, C = 128) the tile lists run to ~1000 entries, thousands of CTAs share the
persistent tile counter, the backward's per-block lists hold ~25M entries, "c4" splits C = 256 into two channel chunks,
"c5" (5M Gaussians, 3840x2160) sorts on 47-bit keys, and 1080 = 67 * 16 + 8 leaves a bottom tile row 8 px tall.  A whole
image of (pixel, list entry) pairs is ~0.8 billion pairs there, so every check here runs in windows of 4x4 tiles
(blend_weights.Pairs(tiles=)), with the weights of the Gaussians in their lists read back by one-hot renders
(blend_weights.extract_ids):
  1. every walked weight of every window pixel, the walk's end and final_T against the float64 model (check_model);
  2. the per-pixel forward identities at the window pixels: colour (with T bg), depth, 1 - T, the C-channel map of the
     scene's own features;
  3. per Gaussian contained in a window (every instance in its tiles, so every blended pixel in it): dL/dcolor, dL/dz
     and dL/dfeature against the blend-weight identities, dL/dmean2D, dL/dconic and dL/dopacity against
     composite_model, through f3dgs_backward (the autograd API's backward) and through ViewBatch.backward
     (f3dgs_backward_accum, bench.py's `value` path: its dL/dfeature, dL/dopacity and dL/dmean2D), at bg = 0 and at
     test_blend_weights.BG (the background terms of dL/dalpha);
  4. the backward preprocess per Gaussian against camera_grad_model.preprocess_chain fed from the kernel's own
     composite intermediates, and the splat records, on the contained Gaussians, the 2000 largest radii, every visible
     Gaussian whose screen mean is outside the image (the Jacobian clamp's side) and a seeded 50k sample.  The needle
     rule of test_geometry_grads (no bar on the covariance-path outputs of conics with eigenvalue ratio > 100) applies;
  5. bench.py's 8-view ViewBatch step against the 8 one-view results: denom exactly, dL/dfeature per element.
Windows are data-driven: the longest list, the most pixels stopped by T < 1e-4, the image centre, the bottom tile row
at mid-width and at the bottom-right corner, and two seeded random tiles.  Each check prints its worst |err| / bar.
Negative controls show parity's bar passing perturbations at c3 that these checks flag.  Every GPU test resets the
allocator's peak, prints its wall time and peak, and holds the peak under 30 GB.

CPU (`-m "not gpu"`): windowed Pairs, extract_ids, the windowed checkers and containment against the whole-image ones
on the oracle.
"""
import copy
import functools
import time

import numpy as np
import pytest
import torch

import blend_weights as bw
import parity
import scenegen
from test_blend_weights import BG, _forward_identities, _model, _oracle_view, _report
from test_geometry_grads import NEEDLE_COND_MAX, View, _records_check, preprocess_check

PEAK_BYTES = 30 << 30
WIN = 4  # window side in tiles


def _t(a, dev="cpu"):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.fixture(autouse=True)
def _budget(request):
    """Wall time and peak device memory of every test; the peak stays under PEAK_BYTES."""
    gpu = "gpu" in request.keywords and torch.cuda.is_available()
    if gpu:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    if gpu:
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated()
        print(f"[{request.node.name}] wall {time.time() - t0:.1f} s, peak {peak / 2**30:.2f} GB")
        assert peak < PEAK_BYTES, peak


def window_tiles(tx, ty, gx, gy):
    """The WIN x WIN tiles around tile (tx, ty) (from one before it), clipped to the gx x gy grid -> tile ids."""
    x0 = min(max(tx - 1, 0), max(gx - WIN, 0))
    y0 = min(max(ty - 1, 0), max(gy - WIN, 0))
    xs, ys = np.arange(x0, min(x0 + WIN, gx)), np.arange(y0, min(y0 + WIN, gy))
    return torch.from_numpy((ys[:, None] * gx + xs[None, :]).reshape(-1)).long()


# ============================================================================================== CPU: windows checked
def _oracle_windows(W, H):
    gx, gy = (W + 15) // 16, (H + 15) // 16
    return [window_tiles(1, 1, gx, gy), window_tiles(gx - 1, gy - 1, gx, gy)]


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_windowed_pairs_are_the_whole_image_rows(name):
    sc, cam, f, whole, w = _oracle_view(name)
    W, H, P = cam.image_width, cam.image_height, sc.P
    args = (_t(f["point_list"].astype(np.int64)), _t(f["ranges"].astype(np.int64)), _t(f["n_contrib"].astype(np.int64)))
    for tiles in _oracle_windows(W, H):
        win = bw.Pairs(*args, W, H, tiles=tiles)
        px = torch.arange(W * H)
        tile = (px // W // 16) * ((W + 15) // 16) + px % W // 16
        assert torch.equal(win.pixels, px[torch.isin(tile, tiles)])
        rows = torch.isin(whole.pix, win.pixels)
        for k in ("pix", "pos", "gid", "walked"):
            assert torch.equal(getattr(win, k), getattr(whole, k)[rows]), k
        assert torch.equal(win.pix[win.first], win.pix) and bool((win.pos[win.first] == 1).all())
        assert torch.equal(win.wgid, whole.gid[rows & whole.walked])
        assert win.HW == W * H and torch.equal(win.n, whole.n)


def _oracle_render(sc, cam):
    import oracle

    def render(sf):
        one = copy.copy(sc)
        one.features = sf.numpy().reshape(sc.P, 1, -1).astype(np.float32)
        return _t(oracle.forward(one, cam)["feature_map"].reshape(sf.shape[1], -1))

    return render


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_extract_ids_is_extract_on_the_same_gaussians(name):
    sc, cam, f, whole, w = _oracle_view(name)
    W, H, P = cam.image_width, cam.image_height, sc.P
    args = (_t(f["point_list"].astype(np.int64)), _t(f["ranges"].astype(np.int64)), _t(f["n_contrib"].astype(np.int64)))
    render = _oracle_render(sc, cam)
    tiles = _oracle_windows(W, H)[0]
    win = bw.Pairs(*args, W, H, tiles=tiles)
    sel = torch.isin(whole.pix[whole.widx], win.pixels)  # the whole image's walked pairs at the window's pixels
    gids = torch.unique(win.wgid)
    wi = bw.extract_ids(win, P, render, gids[torch.randperm(gids.numel(), generator=torch.Generator().manual_seed(1))],
                        64)
    assert torch.equal(wi.view(torch.int32), w[sel].view(torch.int32))
    # a subset of the Gaussians: theirs as extract reads them, 0 for the others
    sub = gids[::3]
    ws = bw.extract_ids(win, P, render, sub, 32)
    keep = torch.isin(win.wgid, sub)
    assert torch.equal(ws[keep].view(torch.int32), w[sel][keep].view(torch.int32)) and bool((ws[~keep] == 0).all())


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_windowed_checkers_are_the_whole_image_checkers(name):
    """check_model's per-pair bar (to float64 rounding), the per-pixel identities and the per-Gaussian terms of
    contained Gaussians (bit for bit) on a window are the whole image's on the same entries."""
    import oracle

    sc, cam, f, whole, w = _oracle_view(name)
    W, H, P, C = cam.image_width, cam.image_height, sc.P, sc.C
    pl, rg = _t(f["point_list"].astype(np.int64)), _t(f["ranges"].astype(np.int64))
    rec, fT = _t(bw.oracle_records(f)), _t(f["final_T"])
    rep_all = bw.check_model(whole, w, rec, fT)
    Wt_all = bw.Weights(whole, w, P)
    G = _t(scenegen.upstream_grads(H, W, C)[1].reshape(C, -1)).t()
    terms_all = Wt_all.terms(G)
    feats = _t(sc.features.reshape(P, C)).double()
    for tiles in _oracle_windows(W, H):
        win = bw.Pairs(pl, rg, _t(f["n_contrib"].astype(np.int64)), W, H, tiles=tiles)
        sel = torch.isin(whole.pix[whole.widx], win.pixels)
        ww = w[sel]
        rep = bw.check_model(win, ww, rec, fT)
        assert rep["ok"] and rep_all["ok"]
        # the segmented sums are differences of one running sum over all pairs: equal to its float64 rounding
        assert torch.allclose(rep["rho"], rep_all["rho"][sel], rtol=1e-9, atol=0.0)
        assert rep["weight"] <= rep_all["weight"] and rep["final_T"] <= rep_all["final_T"]
        Wt = bw.Weights(win, ww, P)
        fmap = _t(f["feature_map"].reshape(C, -1)).t()
        assert torch.equal(torch.sparse.mm(Wt.Wt, feats), torch.sparse.mm(Wt_all.Wt, feats)[win.pixels])
        assert Wt.per_pixel(fmap, feats) <= Wt_all.per_pixel(fmap, feats)
        cont = bw.contained(pl, rg, P, tiles)
        assert int(cont.sum()) > 0
        # a contained Gaussian blends only window pixels
        wp, wg = whole.pix[whole.widx][w > 0], whole.gid[whole.widx][w > 0]
        assert bool(torch.isin(wp[cont[wg]], win.pixels).all())
        terms = Wt.terms(G)
        for a, b in zip(terms, terms_all):
            assert torch.equal(a[cont], b[cont])
        assert torch.equal(Wt.m[cont], Wt_all.m[cont])
        ours = _t(oracle.backward(sc, cam, f, *scenegen.upstream_grads(H, W, C))["semantic_feature"].reshape(P, C))
        assert Wt.per_gaussian(ours, G, cont) == bw.gaussian_ratio(ours, terms_all, Wt_all.m, cont) <= 1.0


def test_containment_on_a_hand_made_list():
    """3 x 2 tiles, window {0, 1, 3}: g0 (tiles 0, 1, 3) is contained; g1 (tiles 1, 2) has one instance outside; g2 lies
    only outside; g3 has no instance; tile 4 is empty."""
    pl = torch.tensor([0, 1, 0, 1, 1, 2, 0, 2])
    ranges = torch.tensor([[0, 2], [2, 4], [4, 6], [6, 7], [7, 7], [7, 8]])  # tiles 0 .. 5 of a 3 x 2 grid
    assert bw.contained(pl, ranges, 4, torch.tensor([0, 1, 3])).tolist() == [True, False, False, False]
    assert bw.contained(pl, ranges, 4, torch.tensor([5, 3, 2, 1, 0])).tolist() == [True, True, True, False]
    assert bw.contained(pl, ranges, 4, torch.tensor([1, 2, 3, 4, 5])).tolist() == [False, False, True, False]


# ============================================================================================== GPU
class BenchView:
    """One camera of a bench scene on the device: test_geometry_grads.View rendering the scene's own features (its
    forward is bench.py's: _C.rasterize_gaussians; with planes, rasterize_gaussians_alpha_invdepth, antialiased when
    antialiasing), the data-driven windows, and per window the pairs, the weights of the Gaussians in its lists and the
    contained Gaussians."""

    def __init__(self, sc, cam, n_windows, group=128, backward=True, planes=False, antialiasing=False):
        v = View(sc, cam, C=sc.C, weights=False, planes=planes, antialiasing=antialiasing)
        v.feats = v.d["semantic_feature"]
        v.base = v.forward(v.feats)
        if not backward:  # the forward's buffers are for the backward only; the extraction renders hold their own
            for k in ("geom", "binning", "img"):
                del v.base[k]
        self.v, self.sc, self.cam, self.P, self.W, self.H = v, sc, cam, sc.P, v.W, v.H
        b = v.base
        gx, gy = (self.W + 15) // 16, (self.H + 15) // 16
        L = (b["ranges"][:, 1] - b["ranges"][:, 0]).long()
        px = torch.arange(self.W * self.H, device="cuda")
        tile = (px // self.W // 16) * gx + px % self.W // 16
        n = b["n_contrib"].reshape(-1).long()
        # stopped by T: the walk ended before the list's end on a pixel whose T is below 1e-4 / (1 - 0.99)
        stopped = (n < L[tile]) & (b["final_T"].reshape(-1) < 1e-2)
        n_stop = torch.zeros(gx * gy, dtype=torch.long, device="cuda").index_add_(0, tile, stopped.long())
        rng = np.random.default_rng(7)
        anchors = {"longest list": int(L.argmax()), "most T stops": int(n_stop.argmax()),
                   "centre": (self.H // 2 // 16) * gx + self.W // 2 // 16,
                   "bottom row mid-width": (gy - 1) * gx + gx // 2,
                   # the corner itself may hold no Gaussian: the bottom row's rightmost tile with a list
                   "bottom-right corner": (gy - 1) * gx + int((L[(gy - 1) * gx:] > 0).nonzero().max()),
                   "random 0": int(rng.integers(gx * gy)), "random 1": int(rng.integers(gx * gy))}
        self.windows = {}
        for name, a in list(anchors.items())[:n_windows]:
            tiles = window_tiles(a % gx, a // gx, gx, gy).cuda()
            pairs = bw.Pairs(b["point_list"], b["ranges"], b["n_contrib"], self.W, self.H, tiles=tiles)
            w = bw.extract_ids(pairs, self.P, self._render, torch.unique(pairs.wgid), group)
            cont = bw.contained(b["point_list"], b["ranges"], self.P, tiles)
            lens = L[tiles]
            print(f"[{name}: tile {a}, tiles {tiles.min().item()}..{tiles.max().item()}] list lengths "
                  f"{lens.min().item()}..{lens.max().item()} (mean {lens.double().mean().item():.0f}), "
                  f"{pairs.pix.numel()} pairs, {pairs.widx.numel()} walked, {int(cont.sum())} contained Gaussians")
            # the scene thins out towards the image's corners: there a window holds fewer whole Gaussians
            assert int(cont.sum()) >= (10 if name == "bottom-right corner" else 100), name
            self.windows[name] = dict(tiles=tiles, pairs=pairs, w=w, contained=cont, Wt=bw.Weights(pairs, w, self.P))
        assert int(L.max()) == int(L[self.windows["longest list"]["tiles"]].max())

    def _render(self, sf):
        r = self.v.forward(sf.reshape(self.P, 1, -1))
        for k in ("color", "n_contrib", "final_T", "point_list"):
            assert torch.equal(r[k], self.v.base[k]), k
        return r["fmap"].reshape(sf.shape[1], -1)

    def with_bg(self, bg):
        """Render with another background: the same walk, so the same pairs and weights."""
        v = self.v
        v.bg = torch.tensor(np.asarray(bg, np.float32), device="cuda")
        r = v.forward(v.feats)
        vis = v.base["radii"] > 0
        for k in ("n_contrib", "final_T", "point_list", "ranges"):
            assert torch.equal(r[k], v.base[k]), k
        # the records the composite reads: visible rows, without the two padding floats
        used = [0, 1] + list(range(4, 12))
        assert torch.equal(r["rec"][vis][:, used], v.base["rec"][vis][:, used])
        v.base = r
        return r


@functools.lru_cache(maxsize=1)
def _scene(name):
    return scenegen.make_config(name, views=8 if name == "c3" else 1)


_VIEWS = {}


def _bench_view(name, cam, n_windows, **kw):
    """One BenchView per (config, camera, options), built once; another config frees the previous one's."""
    key = (name, cam) + tuple(sorted(kw.items()))
    if key not in _VIEWS:
        for k in [k for k in _VIEWS if k[0] != name]:
            del _VIEWS[k]
        sc = _scene(name)
        _VIEWS[key] = BenchView(sc, sc.cameras[cam], n_windows, **kw)
    return _VIEWS[key]


def _checks_forward(bv, label):
    v = bv.v
    rec = v.base["rec"].double()
    for name, win in bv.windows.items():
        _model(f"{label} {name}", win["pairs"], win["w"], v.base["rec"], v.base["final_T"])
        _forward_identities(win["Wt"], f"{label} {name} forward", v.base["color"], v.base["depth"], v.base["final_T"],
                            v.bg, rec, v.base["fmap"], v.feats.reshape(bv.P, -1))


def _composite_ratios(win, rec, P, bg, gc, gd, got):
    """Worst ratio of got (mean2D [P,>=2], conic [P,4] or None, opacity [P]) over the window's contained Gaussians
    against composite_model, at background bg."""
    pairs, w, rows = win["pairs"], win["w"], win["contained"]
    Gc = gc.reshape(3, -1).t()
    bgp = Gc.double() * bg.double()
    ref, bar = bw.composite_model(pairs, w, rec, P, bw.colour_depth_dots(rec, Gc, gd.reshape(-1)), 4,
                                  (bgp.sum(1), bgp.abs().sum(1)))
    names = ["dL_dmean2D.x", "dL_dmean2D.y", "dL_dconic.a", "dL_dconic.b", "dL_dconic.c", "dL_dopacity"]
    cols = [0, 1, 5] if got["conic"] is None else list(range(6))
    conic = got["conic"] if got["conic"] is not None else torch.zeros(P, 4, device=rec.device)
    g6 = bw.geom6(got["mean2D"], conic, got["opacity"]).double()
    r = bw._ratio((g6 - ref).abs(), bar)[rows].max(0).values
    return {names[j]: float(r[j]) for j in cols}, ref, bar


def _checks_backward(bv, label, bgs=(None, BG), view_batch=True):
    """Check 3 at each background -> the f3dgs_backward outputs at the first."""
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    from diff_gaussian_rasterization.parallel import ViewBatch

    v, P, C = bv.v, bv.P, bv.sc.C
    lib = _lib()
    ups = scenegen.upstream_grads(bv.H, bv.W, C, seed=99)
    gc, gf, gd = (_t(u, "cuda") for u in ups)
    first = None
    for bg in bgs:
        bgv = np.zeros(3, np.float32) if bg is None else bg
        bv.with_bg(bgv)
        rec, bgt = v.base["rec"], v.bg
        o = v.backward(lib, ups)
        if first is None:
            first = o
        vb = ViewBatch({k: v.d[k] for k in ("means3D", "scales", "rotations", "opacities", "shs", "semantic_feature")})
        rs = parity.settings(bv.sc, bv.cam, "cuda")
        rs["bg"] = bgt
        vb.zero_()
        _, _, _, _, ctx = vb.forward(GaussianRasterizationSettings(**rs))
        m2d = torch.zeros(P, 3, device="cuda")
        vb.backward(ctx, gc, gf, gd, means2D_out=m2d, last=True)
        torch.cuda.synchronize()
        for name, win in bv.windows.items():
            Wt, rows = win["Wt"], win["contained"]
            worst, _, _ = _composite_ratios(win, rec, P, bgt, gc, gd, o)
            worst["dL_dcolor"] = Wt.per_gaussian(o["color"], gc.reshape(3, -1).t(), rows)
            worst["dL_dz"] = Wt.per_gaussian(o["dz"].reshape(P, 1), gd.reshape(-1, 1), rows)
            worst["dL_dfeature"] = Wt.per_gaussian(o["feat"], gf.reshape(C, -1).t(), rows)
            _report(f"{label} {name} bg={bgv.tolist()} f3dgs_backward", worst)
            if view_batch:
                worst, _, _ = _composite_ratios(win, rec, P, bgt, gc, gd, dict(
                    mean2D=m2d, conic=None, opacity=vb.grads["opacities"].reshape(-1)))
                worst["dL_dfeature"] = Wt.per_gaussian(vb.grads["semantic_feature"].reshape(P, C),
                                                       gf.reshape(C, -1).t(), rows)
                _report(f"{label} {name} bg={bgv.tolist()} ViewBatch.backward", worst)
        del vb
    bv.with_bg(np.zeros(3, np.float32))
    return first, ups


@functools.lru_cache(maxsize=1)
def _lib():
    import ctypes
    import os

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = ctypes.CDLL(os.path.join(root, "feature-3dgs_b200", "libf3dgs_b200.so"))
    lib.f3dgs_last_error.restype = ctypes.c_char_p
    lib.f3dgs_backward_scratch_bytes.restype = ctypes.c_size_t
    return lib


@pytest.mark.gpu
@pytest.mark.parametrize("cam", [0, 7])
def test_c3_weights_and_forward_identities(built, cam):
    bv = _bench_view("c3", cam, 7)
    _checks_forward(bv, f"c3 cam {cam}")


@pytest.mark.gpu
@pytest.mark.parametrize("cam", [0, 7])
def test_c3_backward_per_gaussian(built, cam):
    bv = _bench_view("c3", cam, 7)
    _checks_backward(bv, f"c3 cam {cam}")


def _subset(v, idx):
    """The Gaussians idx of View v as a View of their own (the chain and the records are per Gaussian)."""
    s = object.__new__(View)
    sc = copy.copy(v.sc)
    ii = idx.cpu().numpy()
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        setattr(sc, k, getattr(v.sc, k)[ii])
    s.sc, s.cam, s.mod, s.P, s.W, s.H = sc, v.cam, v.mod, len(ii), v.W, v.H
    s.shs, s.M, s.D, s.cov, s.cols = v.shs[idx], v.M, v.D, v.cov, v.cols
    s.base = {"rec": v.base["rec"][idx], "radii": v.base["radii"][idx]}
    return s


@pytest.mark.gpu
def test_c3_backward_preprocess_per_gaussian(built):
    """Check 4 on camera 0: the preprocess chain and the records on the four sets, each reported apart."""
    bv = _bench_view("c3", 0, 7)
    v, P = bv.v, bv.P
    o = v.backward(_lib(), scenegen.upstream_grads(bv.H, bv.W, bv.sc.C, seed=99))
    vis = (v.base["radii"] > 0)
    radii = torch.where(vis, v.base["radii"], torch.zeros_like(v.base["radii"]))
    mean = v.base["rec"][:, 0:2]
    outside = vis & ((mean[:, 0] < 0) | (mean[:, 0] >= bv.W) | (mean[:, 1] < 0) | (mean[:, 1] >= bv.H))
    g = torch.Generator(device="cuda").manual_seed(5)
    vis_idx = vis.nonzero().flatten()
    contained = torch.zeros(P, dtype=torch.bool, device="cuda")
    for win in bv.windows.values():
        contained |= win["contained"]
    sets = {"contained": contained.nonzero().flatten(), "largest radii": torch.topk(radii, 2000).indices,
            "mean outside the image": outside.nonzero().flatten(),
            "sample": vis_idx[torch.randperm(vis_idx.numel(), device="cuda", generator=g)[:50000]]}
    idx = torch.unique(torch.cat(list(sets.values())))
    t0 = time.time()
    s = _subset(v, idx)
    mids = {k: o[k][idx] for k in ("mean2D", "conic", "color", "dz")}
    m = s.chain(mids)
    rec_r = _records_check(s)
    print(f"[c3 preprocess] {idx.numel()} Gaussians ({', '.join(f'{k} {x.numel()}' for k, x in sets.items())}), "
          f"{int(m['outside'].gt(0).sum())} beyond the Jacobian's clamp; float64 chain {time.time() - t0:.1f} s")
    _report("c3 records, all sets", rec_r)
    outs = {k: x[idx] for k, x in v.outputs(o).items()}
    pos = torch.searchsorted(idx, torch.arange(P, device="cuda")).clamp(max=idx.numel() - 1)
    for name, members in sets.items():
        mask = torch.zeros(idx.numel(), dtype=torch.bool)
        mask[pos[members].cpu()] = True
        worst = preprocess_check(m, outs, mask)
        _report(f"c3 preprocess {name} ({members.numel()}, needles "
                f"{int((mask & (m['eig_ratio'] > NEEDLE_COND_MAX)).sum())})", worst)


@pytest.mark.gpu
def test_c3_view_batch_step_is_the_sum_of_the_views(built):
    """bench.py's step: vb.zero_(), 8 x forward / backward (last= on the final view) against each view alone.

    denom counts the views in which a Gaussian is visible: exactly the sum of the one-view counts.  dL/dfeature of
    Gaussian g, channel c: every view adds its terms t (one reduced row per list entry of g, at most 8 per tile, 8x4-pixel
    blocks, plus one) with float adds onto the buffer, in an order the run does not fix.  To first order any such sum
    of n terms onto a buffer holding a is within u n (|a| + sum |t|) of exact, and the one-view result x_v within
    u n_v sum_v |t|; so with N = sum_v n_v (n_v = 8 instances of g in view v + 1) and A_v = sum_v |t| <= sum_p w_gp |G_p|,
    which the same backward with |dL/dfeature_map| returns (every term non-negative: within u n_v of it):
        |step - sum_v x_v| <= 2 u N (1 + 1e-3) sum_v A_v.
    No tensor-wide floor: the bar is each element's own."""
    from diff_gaussian_rasterization import GaussianRasterizationSettings, _C
    from diff_gaussian_rasterization.parallel import ViewBatch

    sc = _scene("c3")
    P, C = sc.P, sc.C
    t = scenegen.to_torch(sc, "cuda")
    vb = ViewBatch({k: t[k] for k in ("means3D", "scales", "rotations", "opacities", "shs", "semantic_feature")})
    cam0 = sc.cameras[0]
    gc, gf, gd = (_t(u, "cuda") for u in scenegen.upstream_grads(cam0.image_height, cam0.image_width, C, seed=99))
    rss = [GaussianRasterizationSettings(**parity.settings(sc, cam, "cuda")) for cam in sc.cameras]
    vb.zero_()
    for i, rs in enumerate(rss):
        _, _, _, _, ctx = vb.forward(rs)
        vb.backward(ctx, gc, gf, gd, last=i == len(rss) - 1)
    step_feat, step_denom = vb.grads["semantic_feature"].reshape(P, C).clone(), vb.denom.clone()
    xsum = torch.zeros(P, C, dtype=torch.float64, device="cuda")
    asum = torch.zeros(P, C, dtype=torch.float64, device="cuda")
    N = torch.zeros(P, dtype=torch.float64, device="cuda")
    count = torch.zeros(P, device="cuda")
    for rs in rss:
        for G, acc in ((gf, xsum), (gf.abs(), asum)):
            vb.zero_()
            _, _, radii, _, ctx = vb.forward(rs)
            vb.backward(ctx, gc, G, gd, last=True)
            acc += vb.grads["semantic_feature"].reshape(P, C).double()
        count += (radii > 0).float()
        pl = _C.debug_views(ctx.geom, ctx.binning, ctx.img, P, rs.image_width, rs.image_height, ctx.num_rendered)[0]
        N += 8 * torch.bincount(pl.long(), minlength=P).double() + 1
    assert torch.equal(step_denom, count)
    bar = 2 * bw.U * N[:, None] * (1 + 1e-3) * asum
    r = float(bw._ratio((step_feat.double() - xsum).abs(), bar).max())
    print(f"[c3 8-view step] denom exact over {int((count > 0).sum())} Gaussians; "
          f"mean list entries per Gaussian {float(N.mean()):.1f}")
    _report("c3 8-view ViewBatch step", {"dL_dfeature": r})


@pytest.mark.gpu
def test_c3_negative_controls(built):
    """Perturbations of the GPU's dL/dfeature and dL/dopacity at c3 (camera 0, the longest-list window) that parity's bar
    passes and the per-Gaussian checks flag: (a) one (g, p) term dropped, (b) one 8x4-block list entry counted twice,
    (c) a row under parity's floor zeroed; and (d) one early weight scaled by 1 + 1e-4, which the model flags."""
    bv = _bench_view("c3", 0, 7)
    v, P, C, W = bv.v, bv.P, bv.sc.C, bv.W
    o, ups = _checks_backward(bv, "c3 cam 0 (controls)", bgs=(None,), view_batch=False)
    gc, gf, gd = (_t(u, "cuda") for u in ups)
    win = bv.windows["longest list"]
    pairs, w, Wt, cont = win["pairs"], win["w"], win["Wt"], win["contained"]
    rec = v.base["rec"]
    G = gf.reshape(C, -1).t()
    feat = o["feat"].double()
    fnp = feat.cpu().numpy()
    op = o["opacity"].double().reshape(-1)
    opnp = op.cpu().numpy()
    floor_f = parity.GRAD_ATOL_REL * float(feat.abs().max())
    under = cont & (feat.abs().max(1).values < floor_f) & (feat.abs().max(1).values > 0)
    all_cont = torch.zeros(P, dtype=torch.bool, device="cuda")
    for x in bv.windows.values():
        all_cont |= x["contained"]
    all_under = all_cont & (feat.abs().max(1).values < floor_f)
    print(f"[c3 controls] contained Gaussians with the whole dL/dfeature row under parity's floor: "
          f"{int(all_under.sum())} of {int(all_cont.sum())}")
    assert int(under.sum()) > 0
    under_idx = under.nonzero().flatten()
    gq = int(under_idx[under_idx.numel() // 2])
    on = (pairs.gid[pairs.widx] == gq) & (w > 0)
    pix = pairs.pix[pairs.widx][on]
    terms = w[on].double()[:, None] * G[pix].double()
    med = int(torch.argsort(terms.abs().sum(1))[pix.numel() // 2])
    p0 = int(pix[med])
    bx, by = (p0 % W) // 8, (p0 // W) // 4
    block = ((pix % W) // 8 == bx) & ((pix // W) // 4 == by)
    one = torch.zeros(P, dtype=torch.bool, device="cuda")
    one[gq] = True
    flagged = {}
    for lab, d in {"(a) one (g, p) term dropped": -terms[med], "(b) one block list entry counted twice":
                   terms[block].sum(0), "(c) the whole row zeroed": -feat[gq]}.items():
        x = fnp.copy()
        x[gq] += d.cpu().numpy()
        assert parity.float_mismatch(x, fnp, parity.RTOL, parity.GRAD_ATOL_REL)[0] <= 1.0, lab
        flagged["dL_dfeature " + lab] = Wt.per_gaussian(_t(x, "cuda"), G, one)
    # dL/dopacity: a contained Gaussian's row under the floor; pixel p0's term and its block's terms from the model
    # without them (L with the pixels' colour, depth and background terms removed)
    floor_o = parity.GRAD_ATOL_REL * float(op.abs().max())
    under_o = (cont & (op.abs() < floor_o) & (op.abs() > 0)).nonzero().flatten()
    assert under_o.numel() > 0
    go = int(under_o[under_o.numel() // 2])
    on = (pairs.gid[pairs.widx] == go) & (w > 0)
    pix_o = pairs.pix[pairs.widx][on]
    q0 = int(pix_o[pix_o.numel() // 2])
    blk = (((pairs.pix % W) // 8 == (q0 % W) // 8) & ((pairs.pix // W) // 4 == (q0 // W) // 4))
    blk_pix = torch.unique(pairs.pix[blk])
    Gc = gc.reshape(3, -1).t()
    bgp = Gc.double() * v.bg.double()
    base_dfn = bw.colour_depth_dots(rec, Gc, gd.reshape(-1))
    ref, bar = bw.composite_model(pairs, w, rec, P, base_dfn, 4, (bgp.sum(1), bgp.abs().sum(1)))

    def without(pixels):
        drop = torch.zeros(pairs.HW, dtype=torch.bool, device="cuda")
        drop[pixels] = True

        def dfn(gid, px):
            d, dabs = base_dfn(gid, px)
            return torch.where(drop[px], torch.zeros_like(d), d), dabs

        bgd = torch.where(drop, torch.zeros_like(bgp[:, 0]), bgp.sum(1))
        return bw.composite_model(pairs, w, rec, P, dfn, 4, (bgd, bgp.abs().sum(1)))[0][go, 5] - ref[go, 5]

    for lab, d in {"(a) one (g, p) term dropped": without(torch.tensor([q0], device="cuda")),
                   "(b) one block list entry counted twice": -without(blk_pix),
                   "(c) the whole row zeroed": -op[go]}.items():
        x = opnp.copy()
        x[go] += float(d)
        assert parity.float_mismatch(x, opnp, parity.RTOL, parity.GRAD_ATOL_REL)[0] <= 1.0, lab
        flagged["dL_dopacity " + lab] = float(bw._ratio((_t(x, "cuda")[go] - ref[go, 5]).abs(), bar[go, 5]))
    # (d) one weight early in its list scaled by 1 + 1e-4
    rep = bw.check_model(pairs, w, rec, v.base["final_T"])
    assert rep["ok"]
    pos = pairs.pos[pairs.widx]
    cand = torch.nonzero((w > 0) & (pos < 100) & (rep["rho"] < 1e-5)).reshape(-1)
    i = int(cand[torch.argmax(w[cand])])
    w2 = w.clone()
    w2[i] = w[i] * np.float32(1 + 1e-4)
    rep2 = bw.check_model(pairs, w2, rec, v.base["final_T"])
    gi, pi = int(pairs.gid[pairs.widx][i]), int(pairs.pix[pairs.widx][i])
    fmap = v.base["fmap"].reshape(C, -1).double()
    fm2 = fmap[:, pi] + (float(w2[i]) - float(w[i])) * v.feats.reshape(P, C)[gi].double()
    # parity's bar on the map: only column pi changes, so its ratio there against the map's scale decides
    tol = parity.RTOL * fmap[:, pi].abs() + parity.ATOL_REL * float(fmap.abs().max())
    assert float(((fm2 - fmap[:, pi]).abs() / tol).max()) <= 1.0
    flagged[f"weight at list position {int(pos[i])} x (1 + 1e-4)"] = rep2["weight"]
    print(f"[c3 negative controls: Gaussians {gq} (dL/dfeature) and {go} (dL/dopacity)] "
          + ", ".join(f"{k}={x:.3g}" for k, x in flagged.items()))
    for lab, r in flagged.items():
        assert r > 1.0, (lab, r)


@pytest.mark.gpu
def test_c4_two_channel_chunks(built):
    """c4 (C = 256: two 128-channel chunks in the forward and in the feature backward): checks 1-3 on two windows."""
    bv = _bench_view("c4", 0, 2)
    _checks_forward(bv, "c4")
    _checks_backward(bv, "c4")


@pytest.mark.gpu
def test_c5_forward(built):
    """c5 (5M Gaussians, 3840x2160, 47-bit sort keys): checks 1-2 on three windows, extracted 64 Gaussians a render
    (c5's own feature width: a 4K map of 64 channels is 2.1 GB)."""
    bv = _bench_view("c5", 0, 3, group=64, backward=False)
    _checks_forward(bv, "c5")
