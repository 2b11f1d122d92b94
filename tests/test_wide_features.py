"""Wide feature vectors (-m gpu): C from 512 (LSeg without --speedup) up to F3DGS_MAX_FEATURE_DIM = 4096.

The composite kernels split C into chunks of 128 channels: the forward runs one work item per (tile, chunk) and repeats
the alpha pass for every chunk (composite_fwd.cu), the feature backward runs one item per (tile, chunk, 8x4 block) over
the same per-block instance lists (feature_bwd.cu).  Two properties follow from the arithmetic and are checked here at
widths of 4 to 32 chunks, on a small scene and on config 3's cloud and camera:
  * channel chunks are independent.  Every (pixel, channel) of the feature map is the same fma(f, alpha*T, acc) sequence
    in list order whatever the width (a pixel that did not blend adds nothing, composite_fwd.cu), so the C-wide map is
    bitwise the concatenation of the maps rendered from 128-channel slices of the same features.  dL/dfeature is the
    concatenation of the slices' gradients up to the order of its float atomics.
  * the features change nothing else.  dL/dfeature never feeds dL/dalpha (feature_bwd.cu), so colour, depth, final_T,
    n_contrib, the tile lists and radii are bitwise those of a C = 0 render, and the geometric gradients agree within the
    parity bar (their atomics may reorder).
Config 2's cloud and camera at C = 512 are also compared with the CPU oracle, forward and backward.

Every scene gets its width here: scenegen.CONFIGS stays as it is (its seeds follow the order of its entries)."""
import numpy as np
import pytest
import torch

import parity
import scenegen

pytestmark = pytest.mark.gpu

CHUNK = 128  # channels per work item of the composite kernels
GEOM_GRADS = ("means2D", "opacities", "means3D", "sh", "scales", "rotations")


def _render(t, rs, sf, gc, gf, gd):
    """One forward + backward through the torch binding; everything stays on the device."""
    from diff_gaussian_rasterization import _C

    e = torch.Tensor([])
    R, color, feat, depth, radii, geom, binning, img = _C.rasterize_gaussians(
        rs["bg"], t["means3D"], e, sf, t["opacities"], t["scales"], t["rotations"], rs["scale_modifier"], e,
        rs["viewmatrix"], rs["projmatrix"], rs["tanfovx"], rs["tanfovy"], rs["image_height"], rs["image_width"],
        t["shs"], rs["sh_degree"], rs["campos"], rs["prefiltered"], False)
    pl, ranges, n_contrib, final_T, _ = _C.debug_views(geom, binning, img, t["means3D"].shape[0], rs["image_width"],
                                                       rs["image_height"], R)
    g = _C.rasterize_gaussians_backward(
        rs["bg"], t["means3D"], radii, e, sf, t["scales"], t["rotations"], rs["scale_modifier"], e, rs["viewmatrix"],
        rs["projmatrix"], rs["tanfovx"], rs["tanfovy"], gc, gf, gd, t["shs"], rs["sh_degree"], rs["campos"], geom, R,
        binning, img, False)
    names = ("means2D", "colors_precomp", "semantic_feature", "opacities", "means3D", "cov3D_precomp", "sh", "scales",
             "rotations")
    return dict(color=color, feature_map=feat, depth=depth, radii=radii, point_list=pl, ranges=ranges,
                n_contrib=n_contrib, final_T=final_T, grads=dict(zip(names, g)))


def _viol(a, b):
    """Worst |a - b| over the gradient tolerance of the parity bar (<= 1 passes), on the device."""
    a, b = a.double(), b.double()
    if b.numel() == 0:
        return 0.0
    tol = parity.RTOL * b.abs() + parity.GRAD_ATOL_REL * b.abs().max() + 1e-30
    return float(((a - b).abs() / tol).max())


def _scene(name):
    if name == "small":
        return scenegen.make_scene(P=1500, W=96, H=64, C=0, sh_degree=1, seed=7)
    sc = scenegen.make_config(name)
    sc.features = np.zeros((sc.P, 1, 0), np.float32)  # the width is given below
    return sc


@pytest.mark.parametrize("name,C", [("small", 512), ("small", 513), ("small", 4096), ("c3", 512)])
def test_channel_chunks_are_independent(name, C):
    sc = _scene(name)
    cam = sc.cameras[0]
    H, W = cam.image_height, cam.image_width
    t = scenegen.to_torch(sc, "cuda")
    rs = parity.settings(sc, cam, "cuda")
    gen = torch.Generator(device="cuda").manual_seed(C)
    # one C-wide array; the slices below are views of it (a narrower draw would hold other numbers)
    feats = torch.randn(sc.P, 1, C, device="cuda", generator=gen)
    gc, gf, gd = (torch.randn(n, H, W, device="cuda", generator=gen) for n in (3, C, 1))

    full = _render(t, rs, feats, gc, gf, gd)
    assert full["feature_map"].shape == (C, H, W) and float(full["feature_map"].abs().max()) > 0
    assert float(full["grads"]["semantic_feature"].abs().max()) > 0

    bare = _render(t, rs, torch.empty(0, device="cuda"), gc, torch.empty(0, H, W, device="cuda"), gd)
    for k in ("color", "depth", "final_T", "n_contrib", "point_list", "ranges", "radii"):
        assert torch.equal(full[k], bare[k]), k
    worst = {k: _viol(full["grads"][k], bare["grads"][k]) for k in GEOM_GRADS}
    print(f"[{name} C={C}] R={full['point_list'].numel()} geometric gradients vs C=0, worst viol: "
          + ", ".join(f"{k}={v:.3g}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v <= 1.0, (k, v)
    del bare

    worst_f = 0.0
    for c0 in range(0, C, CHUNK):
        c1 = min(C, c0 + CHUNK)
        part = _render(t, rs, feats[..., c0:c1].contiguous(), gc, gf[c0:c1], gd)
        assert torch.equal(full["feature_map"][c0:c1], part["feature_map"]), (c0, c1)
        v = _viol(full["grads"]["semantic_feature"][..., c0:c1], part["grads"]["semantic_feature"])
        worst_f = max(worst_f, v)
        assert v <= 0.5, (c0, c1, v)
    print(f"[{name} C={C}] dL/dfeature vs the 128-channel slices, worst viol {worst_f:.3g}")


def test_c2_cloud_at_C512_vs_oracle():
    """300k Gaussians at 800x800 with 512 channels, forward and backward against the CPU oracle."""
    sc = scenegen.make_config("c2")
    C = 512
    sc.features = np.random.Generator(np.random.PCG64(C)).standard_normal((sc.P, 1, C), dtype=np.float32)
    cam = sc.cameras[0]
    grads = scenegen.upstream_grads(cam.image_height, cam.image_width, C)
    parity.tie_aware_compare(sc, cam, "c2 C=512", grads=grads)
