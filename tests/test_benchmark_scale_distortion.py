"""The depth distortion loss at the benchmark's own view, in tile windows.

test_distortion.py checks the distortion forward and backward per pixel and per Gaussian on small scenes, whose tile lists
hold tens of entries.  On bench.py's scene "c3" (1M Gaussians, 1920x1080, C = 128) the lists run to ~1000 entries, so
the float32 error of the unwound T in A_i - Abar_i and of the walk's running register E = 2 Dbar - D_tot grows with
the list length that the bars of test_distortion scale with.  Here, on cameras 0 and 7 in the seven 4x4-tile windows of
test_benchmark_scale.BenchView:
  1. f3dgs_forward_distortion with NaN-prefilled outputs: colour, feature map, depth and radii bitwise those of bench.py's
     forward, every pixel of the plane written, and the plane at every window pixel against test_distortion's float64
     model on the extracted weights, within its derived bar;
  2. f3dgs_backward_distortion under bench.py's upstream gradients and a N(0, 1) and a dynamic-range distortion gradient:
     per contained Gaussian the six geometric values against test_distortion.backward_model, dL/dz against its sum over
     pixels and dL/dcolor against the blend-weight identity; and ViewBatch.backward(..., g_distortion=)'s dL_dmean2D and
     dL/dopacity (f3dgs_backward_accum_distortion, bench.py's path) against the same model.
Negative controls in the longest-list window: the plane with the largest single pair's term removed from one pixel, and
the backward models without the later pairs' Abar term and of 2DGS's squared form, are each outside the bars.
Every GPU test prints its wall time and peak device memory and holds the peak under 30 GB
(test_benchmark_scale._budget).
"""
import numpy as np
import pytest
import torch

import blend_weights as bw
import parity
import scenegen
from test_benchmark_scale import _VIEWS, _bench_view, _budget, _lib  # noqa: F401
from test_distortion import (_ctypes_backward, _dist_grad, _forward_ctypes, backward_model, blended, distortion_model,
                             prefix_sums)
from test_geometry_grads import _report


def _t(a, dev="cpu"):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.mark.gpu
@pytest.mark.parametrize("cam", [0, 7])
def test_c3_distortion_forward_per_pixel(built, cam):
    bv = _bench_view("c3", cam, 7)
    v = bv.v
    bv.with_bg(bv.sc.bg)  # the scene's background, which _forward_ctypes renders with
    new = _forward_ctypes(_lib(), bv.sc, bv.cam, v.feats, False)
    assert new["R"] == v.base["R"]
    for k in ("color", "fmap", "depth", "radii"):
        assert torch.equal(new[k], v.base[k]), k
    dist = new["distortion"].reshape(-1).double()
    del new
    assert not bool(dist.isnan().any()) and bool((dist >= 0).all())
    assert bool((dist[v.base["n_contrib"].reshape(-1) == 0] == 0).all())
    for name, win in bv.windows.items():
        pairs = win["pairs"]
        L, bar = distortion_model(pairs, win["w"], v.base["rec"])
        px = pairs.pixels
        r = float(bw._ratio((dist[px] - L[px]).abs(), bar[px]).max())
        print(f"[c3 cam {cam} {name}] distortion worst |err|/bar {r:.3g}, max L {float(L[px].max()):.3g}, "
              f"longest walk {int(pairs.n[px].max())}")
        assert r <= 1.0 and bool((L[px] > 0).any()), name
        if name == "longest list":  # negative control: one pair's term dropped from the plane
            pix, _, wv, z, first = blended(pairs, win["w"], v.base["rec"])
            A, D, _, _ = prefix_sums(wv, z, pix, first, pairs.HW)
            term = 2 * wv * (z * A - D)
            k = int(term.argmax())
            bad = dist.clone()
            bad[pix[k]] -= term[k]
            rb = float(bw._ratio((bad[px] - L[px]).abs(), bar[px]).max())
            print(f"[c3 cam {cam} {name}] one pair's term dropped: worst |err|/bar {rb:.3g}")
            assert rb > 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("cam", [0, 7])
def test_c3_distortion_backward_per_gaussian(built, cam):
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    from diff_gaussian_rasterization.parallel import ViewBatch

    bv = _bench_view("c3", cam, 7)
    v, P, C, H, W = bv.v, bv.P, bv.sc.C, bv.H, bv.W
    lib = _lib()
    ups = scenegen.upstream_grads(H, W, C, seed=99)
    ug = [_t(u, "cuda") for u in ups]
    gc, gf, gd = ug
    Gc, Gd = gc.reshape(3, -1).t(), gd.reshape(-1)
    z = lambda *s: torch.zeros(*s, device="cuda")  # noqa: E731
    for label, dyn in (("N(0,1)", False), ("dynamic range", True)):
        g = _t(_dist_grad(H, W, 70 + cam, dynamic=dyn), "cuda")
        o = dict(mean2D=z(P, 3), conic=z(P, 4), opacity=z(P), color=z(P, 3), feat=z(P, C), means3D=z(P, 3),
                 cov3D=z(P, 6), sh=z(P, v.M, 3), scales=z(P, 3), rotations=z(P, 4), dz=z(P))
        _ctypes_backward(lib, v, ug, g, o)
        del o["feat"], o["sh"], o["cov3D"], o["means3D"], o["scales"], o["rotations"]
        vb = ViewBatch({k: v.d[k] for k in ("means3D", "scales", "rotations", "opacities", "shs", "semantic_feature")})
        rs = parity.settings(bv.sc, bv.cam, "cuda")
        rs["bg"] = v.bg
        vb.zero_()
        *_, ctx = vb.forward_distortion(GaussianRasterizationSettings(**rs))
        m2d = z(P, 3)
        vb.backward(ctx, gc, gf, gd, means2D_out=m2d, g_distortion=g)
        torch.cuda.synchronize()
        vb_opacity = vb.grads["opacities"].reshape(-1).clone()
        del vb, ctx
        for name, win in bv.windows.items():
            pairs, w, rows, Wt = win["pairs"], win["w"], win["contained"], win["Wt"]
            ref, bar, dz, m = backward_model(pairs, w, v.base["rec"], P, v.bg, Gc, Gd, g)
            names = ["dL_dmean2D.x", "dL_dmean2D.y", "dL_dconic.a", "dL_dconic.b", "dL_dconic.c", "dL_dopacity"]
            g6 = bw.geom6(o["mean2D"], o["conic"], o["opacity"]).double()
            r = bw._ratio((g6 - ref).abs(), bar)[rows].max(0).values
            worst = {k: float(x) for k, x in zip(names, r)}
            worst["dL_dz"] = bw.gaussian_ratio(o["dz"].reshape(P, 1), dz, m, rows)
            worst["dL_dcolor"] = Wt.per_gaussian(o["color"], Gc, rows)
            _report(f"c3 cam {cam} {name} distortion {label} f3dgs_backward_distortion", worst)
            g6 = bw.geom6(m2d, torch.zeros(P, 4, device="cuda"), vb_opacity).double()
            r = bw._ratio((g6 - ref).abs(), bar)[rows].max(0).values
            _report(f"c3 cam {cam} {name} distortion {label} ViewBatch.backward",
                    {names[j]: float(r[j]) for j in (0, 1, 5)})
            if name == "longest list" and label == "N(0,1)":  # negative controls: the ablated models
                g6 = bw.geom6(o["mean2D"], o["conic"], o["opacity"]).double()
                for form in ("no_abar", "squared"):
                    x, _, _, _ = backward_model(pairs, w, v.base["rec"], P, v.bg, Gc, Gd, g, form)
                    rx = float(bw._ratio((g6 - x).abs(), bar)[rows].max())
                    print(f"[c3 cam {cam} {name}] {form} model: worst |err|/bar {rx:.3g}")
                    assert rx > 1.0, form
