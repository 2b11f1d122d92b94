"""Loader + autograd wrapper for oracle/_ref: the UNMODIFIED reference CUDA rasterizer (sm_90a build).

TEST / BENCH INFRASTRUCTURE ONLY (needs a GPU; the modules are built in the CPU container by
oracle/build_ref.py and are loaded on the GPU machine).

The reference fixes the feature width at compile time, so `load(C)` picks the module built for
that width (C = 0 is served by the C = 1 build with an all-zero feature column: colour, depth and
all integer outputs are independent of the features).  `RefRasterizer` re-states the ~60 lines of
argument shuffling of the reference's Python autograd function
(diff_gaussian_rasterization/__init__.py:46-172) around the reference's own `_C` functions, so that
"reference" numbers and parity targets come from the reference's kernels, untouched.
"""
import importlib.util
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_REF = os.path.join(_HERE, "_ref")
_mods = {}


def available(C: int) -> bool:
    return os.path.exists(os.path.join(_REF, f"ref_rast_C{max(C, 1)}.so"))


def load(C: int):
    C = max(C, 1)
    if C not in _mods:
        name = f"ref_rast_C{C}"
        path = os.path.join(_REF, name + ".so")
        if not os.path.exists(path):
            raise FileNotFoundError(f"{path} missing: run `python oracle/build_ref.py {C}` in the build container")
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        _mods[C] = mod
    return _mods[C]


class _RefFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mod, means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                cov3Ds_precomp, rs):
        out = mod.rasterize_gaussians(
            rs["bg"], means3D, colors_precomp, semantic_feature, opacities, scales, rotations, rs["scale_modifier"],
            cov3Ds_precomp, rs["viewmatrix"], rs["projmatrix"], rs["tanfovx"], rs["tanfovy"], rs["image_height"],
            rs["image_width"], sh, rs["sh_degree"], rs["campos"], rs["prefiltered"], rs["debug"])
        num_rendered, color, feature_map, depth, radii, geom, binning, img = out
        ctx.mod, ctx.rs, ctx.num_rendered = mod, rs, num_rendered
        ctx.save_for_backward(colors_precomp, semantic_feature, means3D, scales, rotations, cov3Ds_precomp, radii, sh,
                              geom, binning, img)
        ctx.mark_non_differentiable(radii)
        return color, feature_map, radii, depth

    @staticmethod
    def backward(ctx, g_color, g_feature, _g_radii, g_depth):
        rs = ctx.rs
        (colors_precomp, semantic_feature, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geom, binning,
         img) = ctx.saved_tensors
        (g_means2D, g_colors, g_sem, g_opac, g_means3D, g_cov3D, g_sh, g_scales, g_rot) = \
            ctx.mod.rasterize_gaussians_backward(
                rs["bg"], means3D, radii, colors_precomp, semantic_feature, scales, rotations, rs["scale_modifier"],
                cov3Ds_precomp, rs["viewmatrix"], rs["projmatrix"], rs["tanfovx"], rs["tanfovy"], g_color, g_feature,
                g_depth, sh, rs["sh_degree"], rs["campos"], geom, ctx.num_rendered, binning, img, rs["debug"])
        return (None, g_means3D, g_means2D, g_sh, g_colors, g_sem, g_opac, g_scales, g_rot, g_cov3D, None)


class RefRasterizer:
    """Callable with the same keyword surface as GaussianRasterizer.forward."""

    def __init__(self, raster_settings: dict, C: int):
        self.rs = dict(raster_settings)
        self.C = C
        self.mod = load(C)

    def __call__(self, means3D, means2D, opacities, shs=None, semantic_feature=None, colors_precomp=None, scales=None,
                 rotations=None, cov3D_precomp=None):
        e = torch.Tensor([])
        if self.C == 0:  # C=1 build, zero feature column
            semantic_feature = torch.zeros(means3D.shape[0], 1, 1, device=means3D.device)
        color, feat, radii, depth = _RefFn.apply(
            self.mod, means3D, means2D, e if shs is None else shs, e if colors_precomp is None else colors_precomp,
            semantic_feature, opacities, e if scales is None else scales, e if rotations is None else rotations,
            e if cov3D_precomp is None else cov3D_precomp, self.rs)
        if self.C == 0:
            feat = feat[:0]
        return color, feat, radii, depth


# ---- reference buffer layout (rasterizer_impl.cu:154-194, 128-byte aligned bump allocation) ----------
def _bump(fields, base=0):
    """fields: list of (name, count, elem_bytes) -> dict name -> (offset, count)."""
    off, out = base, {}
    for name, count, esz in fields:
        off = (off + 127) // 128 * 128
        out[name] = (off, count)
        off += count * esz
    return out


def parse_image_buffer(img: torch.Tensor, W: int, H: int):
    """-> final_T [H,W] f32, n_contrib [H,W] i32, ranges [tiles,2] i32   (ImageState, :172-179)"""
    N = W * H
    lay = _bump([("accum_alpha", N, 4), ("n_contrib", N, 4), ("ranges", N, 8)])
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    base = img.data_ptr() % 128
    assert base == 0
    fT = img[lay["accum_alpha"][0]: lay["accum_alpha"][0] + 4 * N].view(torch.float32).view(H, W)
    nc = img[lay["n_contrib"][0]: lay["n_contrib"][0] + 4 * N].view(torch.int32).view(H, W)
    rg = img[lay["ranges"][0]: lay["ranges"][0] + 8 * tiles].view(torch.int32).view(tiles, 2)
    return fT.clone(), nc.clone(), rg.clone()


def parse_binning_buffer(binning: torch.Tensor, R: int):
    """-> point_list [R] i32 (sorted Gaussian ids)   (BinningState, :181-194)"""
    lay = _bump([("point_list", R, 4)])
    assert binning.data_ptr() % 128 == 0
    return binning[lay["point_list"][0]: lay["point_list"][0] + 4 * R].view(torch.int32).clone()


def parse_geom_buffer(geom: torch.Tensor, P: int, C: int):
    """-> dict(depths, means2D, conic_opacity, rgb)   (GeometryState, :154-170)"""
    C = max(C, 1)
    lay = _bump([("depths", P, 4), ("clamped", 3 * P, 1), ("internal_radii", P, 4), ("means2D", P, 8),
                 ("cov3D", 6 * P, 4), ("conic_opacity", P, 16), ("rgb", 3 * P, 4), ("semantic", P * C, 4)])
    assert geom.data_ptr() % 128 == 0

    def f(name, n, shape):
        o = lay[name][0]
        return geom[o: o + 4 * n].view(torch.float32).view(*shape).clone()

    return dict(depths=f("depths", P, (P,)), means2D=f("means2D", 2 * P, (P, 2)),
                conic_opacity=f("conic_opacity", 4 * P, (P, 4)), rgb=f("rgb", 3 * P, (P, 3)),
                cov3D=f("cov3D", 6 * P, (P, 6)))
