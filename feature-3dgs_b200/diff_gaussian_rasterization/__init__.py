"""Drop-in `diff_gaussian_rasterization` on the H100-native rasterizer (libf3dgs_b200.so).

Public surface = the reference extension's
(submodules/diff-gaussian-rasterization-feature/diff_gaussian_rasterization/__init__.py):

  GaussianRasterizationSettings   NamedTuple, same fields/order            (reference :174-186)
  GaussianRasterizer              nn.Module with .forward / .markVisible   (reference :188-238)
  rasterize_gaussians             functional entry                         (reference :21-44)
  _RasterizeGaussians             torch.autograd.Function                  (reference :46-172)

so the reference's gaussian_renderer/__init__.py and train.py import and call it unchanged:
`GaussianRasterizer(raster_settings=...)(means3D=..., means2D=..., shs=..., colors_precomp=...,
semantic_feature=..., opacities=..., scales=..., rotations=..., cov3D_precomp=...)`
returns `(color[3,H,W], feature_map[C,H,W], radii[P] int32, depth[1,H,W])`.

Behavioural notes
  * feature width C is taken from `semantic_feature.shape[-1]` at run time (the reference needs a
    rebuild per width, config.h:16); `semantic_feature=None` renders RGB + depth only (C = 0).
  * the feature map has the dtype of `semantic_feature`: float32 or float16 (the reference is float32 only).  A float16
    map is bitwise the float32 map of `semantic_feature.float()` rounded by `.half()`, without a float32 map ever
    being made; colour, depth and radii are bitwise the float32 render's.  A float16 map's gradient goes to the native
    backward as it is (upcast exactly as it is loaded, no float32 copy); dL/dsemantic_feature is accumulated in float32
    and returned in `semantic_feature`'s dtype.  To train a float16 feature field use GaussianState(feature_dtype=
    torch.float16) with ViewBatch and feature_head's `*_and_grad(..., grad_dtype=torch.float16)`: their ScaledGrad
    carries the float32 scale that keeps the L1 gradient (~1e-8) from underflowing in float16, which autograd cannot.
  * `debug=True` keeps the reference semantics: arguments are snapshotted to CPU first and dumped
    to snapshot_fw.dump / snapshot_bw.dump if the native call raises (reference :89-97,:147-155);
    natively it synchronises and checks after every stage.
  * there is deliberately no CPU or pure-PyTorch fallback: importing this package without the
    compiled extension raises ImportError with build instructions.
"""
from typing import NamedTuple

import torch
import torch.nn as nn

try:
    from . import _C
except ImportError as exc:  # pragma: no cover - exercised only on a broken install
    raise ImportError(
        "diff_gaussian_rasterization._C (f3dgs_b200) is not built. Run "
        "`python feature-3dgs_b200/build.py` (needs nvcc, targets sm_90a). "
        "There is no CPU fallback. Original error: %s" % (exc,)
    ) from exc

__all__ = [
    "GaussianRasterizationSettings",
    "GaussianRasterizer",
    "rasterize_gaussians",
]


def cpu_deep_copy_tuple(input_tuple):
    """Snapshot every tensor of an argument tuple on the CPU (reference :17-19)."""
    return tuple(a.cpu().clone() if isinstance(a, torch.Tensor) else a for a in input_tuple)


def _call_native(fn, args, debug, dump_name, what):
    if not debug:
        return fn(*args)
    snapshot = cpu_deep_copy_tuple(args)  # before anything can be corrupted
    try:
        return fn(*args)
    except Exception:
        torch.save(snapshot, dump_name)
        print("\nAn error occured in %s. Please forward %s for debugging." % (what, dump_name))
        raise


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


class _RasterizeGaussians(torch.autograd.Function):
    """Autograd bridge; argument and gradient order identical to the reference (:46-172)."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                cov3Ds_precomp, raster_settings):
        rs = raster_settings
        if semantic_feature is None:
            semantic_feature = torch.empty(0, device=means3D.device, dtype=means3D.dtype)
        args = (rs.bg, means3D, colors_precomp, semantic_feature, opacities, scales, rotations, rs.scale_modifier,
                cov3Ds_precomp, rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height,
                rs.image_width, sh, rs.sh_degree, rs.campos, rs.prefiltered, rs.debug)
        (num_rendered, color, feature_map, depth, radii, geomBuffer, binningBuffer, imgBuffer) = _call_native(
            _C.rasterize_gaussians, args, rs.debug, "snapshot_fw.dump", "forward")
        ctx.raster_settings = rs
        ctx.num_rendered = num_rendered
        ctx.save_for_backward(colors_precomp, semantic_feature, means3D, scales, rotations, cov3Ds_precomp, radii,
                              sh, geomBuffer, binningBuffer, imgBuffer)
        ctx.mark_non_differentiable(radii)
        return color, feature_map, radii, depth

    @staticmethod
    def backward(ctx, grad_out_color, grad_out_feature, _grad_radii, grad_depth):
        rs = ctx.raster_settings
        (colors_precomp, semantic_feature, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer,
         binningBuffer, imgBuffer) = ctx.saved_tensors
        # autograd hands None/undefined for outputs that did not take part in the loss
        if grad_out_color is None:
            grad_out_color = torch.zeros(3, rs.image_height, rs.image_width, device=means3D.device)
        if grad_depth is None:
            grad_depth = torch.zeros(1, rs.image_height, rs.image_width, device=means3D.device)
        if grad_out_feature is None:
            C = semantic_feature.shape[-1] if semantic_feature.numel() else 0
            grad_out_feature = torch.zeros(C, rs.image_height, rs.image_width, device=means3D.device)
        args = (rs.bg, means3D, radii, colors_precomp, semantic_feature, scales, rotations, rs.scale_modifier,
                cov3Ds_precomp, rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, grad_out_color,
                grad_out_feature, grad_depth, sh, rs.sh_degree, rs.campos, geomBuffer, ctx.num_rendered,
                binningBuffer, imgBuffer, rs.debug)
        (grad_means2D, grad_colors_precomp, grad_semantic_feature, grad_opacities, grad_means3D,
         grad_cov3Ds_precomp, grad_sh, grad_scales, grad_rotations) = _call_native(
            _C.rasterize_gaussians_backward, args, rs.debug, "snapshot_bw.dump", "backward")
        if not ctx.needs_input_grad[4]:
            grad_semantic_feature = None
        else:
            grad_semantic_feature = grad_semantic_feature.to(semantic_feature.dtype)
        return (grad_means3D, grad_means2D, grad_sh, grad_colors_precomp, grad_semantic_feature, grad_opacities,
                grad_scales, grad_rotations, grad_cov3Ds_precomp, None)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                        cov3Ds_precomp, raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales,
                                     rotations, cov3Ds_precomp, raster_settings)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        """Boolean mask of points in front of the near plane (reference :193-202)."""
        with torch.no_grad():
            rs = self.raster_settings
            return _C.mark_visible(positions, rs.viewmatrix, rs.projmatrix)

    def forward(self, means3D, means2D, opacities, shs=None, semantic_feature=None, colors_precomp=None,
                scales=None, rotations=None, cov3D_precomp=None):
        rs = self.raster_settings
        if (shs is None) == (colors_precomp is None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        empty = torch.Tensor([])  # absent optional = empty CPU tensor, as in the reference
        if shs is None:
            shs = empty
        if colors_precomp is None:
            colors_precomp = empty
        if scales is None:
            scales = empty
        if rotations is None:
            rotations = empty
        if cov3D_precomp is None:
            cov3D_precomp = empty
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, semantic_feature, opacities, scales,
                                   rotations, cov3D_precomp, rs)
