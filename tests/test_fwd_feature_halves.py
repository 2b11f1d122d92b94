"""The forward composite's feature warps split each 8x4 pixel block into two 8x2 halves (-m gpu).

Warp h of a block's pair accumulates rows 2h and 2h+1 only, walks only the instances that blended a pixel in those rows,
and stores only its two rows (csrc/composite_fwd.cu).  These tests render images whose last block row is cut by the
image border in every way (H % 4 = 1: the lower half and one upper row outside; 2: the lower half outside; 3: one lower
row outside), widths off the 8- and 4-pixel store paths, and feature widths around the 32 / 64 / 128-channel kernels
and the 128-channel chunks (bulk copies for C % 4 == 0, scalar row loads otherwise), and check:
  * float32: colour, depth, final_T, the feature map and the tile lists against the CPU oracle, with the parity bar;
  * float16: the map is bitwise the float32 render of the upcast features followed by .half(), and everything else is
    bitwise the float32 render's.
Small splats (target radius 1.5 px) give many entries that blend in one half of a block only.
"""
import pytest
import torch

import parity
import scenegen

pytestmark = pytest.mark.gpu

WIDTHS = [1, 3, 32, 33, 64, 65, 128, 129, 200]
# (W, H, target splat radius in pixels)
IMAGES = [(96, 61, 6.0), (96, 62, 6.0), (96, 63, 1.5), (92, 45, 6.0), (97, 38, 1.5)]


def _scene(W, H, C, radius):
    return scenegen.make_scene(P=1500, W=W, H=H, C=C, sh_degree=1, seed=W * 1000 + H * 10 + C,
                               target_radius_px=radius)


@pytest.mark.parametrize("W,H,radius", IMAGES)
@pytest.mark.parametrize("C", WIDTHS)
def test_feature_map_matches_the_oracle(C, W, H, radius):
    sc = _scene(W, H, C, radius)
    cam = sc.cameras[0]
    ours = parity.run_ours(sc, cam, device="cuda")
    orc = parity.run_oracle(sc, cam, threads=1)
    rep = parity.compare(ours, orc, tie_tolerant=True)
    print(f"[W={W} H={H} C={C}]\n" + parity.format_report(rep))
    assert ours["feature_map"].shape == (C, H, W)
    assert float(abs(orc["feature_map"]).max()) > 0
    assert rep["ok"]


def _render(t, rs, sf):
    from diff_gaussian_rasterization import _C

    e = torch.Tensor([])
    R, color, feat, depth, radii, geom, binning, img = _C.rasterize_gaussians(
        rs["bg"], t["means3D"], e, sf, t["opacities"], t["scales"], t["rotations"], rs["scale_modifier"], e,
        rs["viewmatrix"], rs["projmatrix"], rs["tanfovx"], rs["tanfovy"], rs["image_height"], rs["image_width"],
        t["shs"], rs["sh_degree"], rs["campos"], rs["prefiltered"], False)
    pl, ranges, n_contrib, final_T, _ = _C.debug_views(geom, binning, img, t["means3D"].shape[0], rs["image_width"],
                                                       rs["image_height"], R)
    return dict(num_rendered=R, color=color, feature_map=feat, depth=depth, radii=radii, point_list=pl,
                ranges=ranges, n_contrib=n_contrib, final_T=final_T)


def _bits(x):
    return x.view(torch.int16) if x.dtype == torch.float16 else x.view(torch.int32) if x.dtype == torch.float32 else x


@pytest.mark.parametrize("W,H,radius", IMAGES)
@pytest.mark.parametrize("C", WIDTHS)
def test_half_feature_map_is_the_float_map_rounded(C, W, H, radius):
    sc = _scene(W, H, C, radius)
    t = scenegen.to_torch(sc, "cuda")
    rs = parity.settings(sc, sc.cameras[0], "cuda")
    sf16 = t["semantic_feature"].half()
    r16 = _render(t, rs, sf16)
    r32 = _render(t, rs, sf16.float())
    assert r16["feature_map"].dtype == torch.float16 and r16["feature_map"].shape == (C, H, W)
    assert float(r32["feature_map"].abs().max()) > 0
    assert torch.equal(_bits(r16["feature_map"]), _bits(r32["feature_map"].half()))
    assert r16["num_rendered"] == r32["num_rendered"]
    for k in ("color", "depth", "radii", "final_T", "n_contrib", "point_list", "ranges"):
        assert torch.equal(_bits(r16[k]), _bits(r32[k])), k
