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
  * camera gradients (pose refinement, localisation, tracking): when grad mode is on and `raster_settings.viewmatrix`,
    `.projmatrix` or `.campos` requires grad, `rasterize_gaussians` goes through `_RasterizeGaussiansCamera`, which
    also returns dL/dviewmatrix, dL/dprojmatrix and dL/dcampos (f3dgs_backward_cam); otherwise the call and its graph
    are `_RasterizeGaussians`'s.  `camera.settings_from_w2c` builds differentiable settings from a world-to-camera pose.
  * feature gradients into geometry (opt-in): `GaussianRasterizer(raster_settings, feature_geometry=True)`, or
    `rasterize_gaussians_feature_geometry` with `rasterize_gaussians`'s arguments, lets a loss on the feature map move
    opacities, means, scales, rotations and the camera too (f3dgs_backward_feature_geometry).  By default the feature
    map feeds dL/dsemantic_feature only, as in the reference (SURVEY D.1).
  * antialiased rendering (opt-in): `AntialiasedGaussianRasterizer(raster_settings)` multiplies each opacity by
    sqrt(det(S) / det(S + 0.3 I)), S the 2-D covariance before the rasterizer's 0.3 px^2 dilation, so that a dilated
    sub-pixel Gaussian keeps the integral of the undilated one (f3dgs_forward_antialiased / f3dgs_backward_antialiased).
    Renders at a resolution other than the training one (lower-resolution feature targets, lifting at a teacher's
    resolution) then stay consistent.  By default the opacity is used as it is, as in the reference.
  * opacity and inverse-depth maps (opt-in): `AlphaInvDepthGaussianRasterizer(raster_settings, feature_geometry=False,
    antialiasing=False)`, or `rasterize_gaussians_alpha_invdepth`, also returns alpha = 1 - T_final (accumulated
    opacity) and invdepth = sum_i w_i / z_i, both [1,H,W] float32 and differentiable (f3dgs_forward_alpha_invdepth /
    f3dgs_backward_alpha_invdepth): mask losses, RGBA cut-outs, expected depth depth / alpha and inverse-depth
    supervision.  Colour, feature map, depth, radii and their gradients are those of the rasterizer without the maps.
  * sparse Adam (opt-in): `SparseGaussianAdam(params, lr, eps)` with `.step(visibility, N)` is the upstream
    rasterizer's optimizer of that name: it updates only the Gaussians marked visible (f3dgs_adam_step_masked), without
    bias correction, and leaves the others' parameters and moments untouched.
  * 3D smoothing filter (opt-in, Mip-Splatting): `compute_3d_filter(means3D, train_settings)` gives every Gaussian a
    world-space filter size from the highest sampling rate any training camera has at it, and
    `apply_3d_filter(opacities, scales, filter_3D)` returns the filtered opacities and scales to render with, with a
    native backward (f3dgs_filter3d_*).  Renders closer than or at a higher resolution than the training views then
    show no Gaussians smaller than the training views could sample.  `GaussianState.compute_3d_filter` turns it on for
    training.  By default the opacities and scales are used as they are, as in the reference.
  * compaction (opt-in): `GaussianScores(means3D, opacities, scales, rotations)` accumulates each Gaussian's blend-weight
    sum, largest blend weight and blended-pixel count over views (f3dgs_gaussian_scores_accum), and
    `GaussianState.prune(keep)` / `prune_by_importance(scores, ratio)` remove rows with the Adam state carried along
    (f3dgs_prune_plan + f3dgs_densify_apply).
  * absolute-gradient densification (opt-in, AbsGS): `AbsGradGaussianRasterizer(raster_settings, feature_geometry=False,
    antialiasing=False)` takes AbsGS's `screenspace_points_abs` as `forward(..., means2D_abs=...)`, a [P,3] tensor that
    requires grad, and gives it the view's per-Gaussian sums over pixels of |x| and |y| of each pixel's dL/dmean2D term
    as its `.grad` (f3dgs_backward_absgrad).  A large Gaussian over fine texture, whose per-pixel terms cancel in
    dL/dmean2D, keeps a large statistic there, so AbsGS's split rule splits it.  The render and every other gradient
    are GaussianRasterizer's (AntialiasedGaussianRasterizer's with antialiasing).  `ViewBatch(absgrad=True)` and
    `GaussianState(absgrad=True)` accumulate the statistic natively, and `densify_and_prune(abs_grad=...)` applies
    the split rule.
  * depth distortion loss (opt-in; Mip-NeRF 360's term as 2DGS and gsplat's `distloss` use it, in its L1 form on view
    depth): `DistortionGaussianRasterizer(raster_settings, feature_geometry=False, antialiasing=False)`, or
    `rasterize_gaussians_distortion`, also returns, per pixel p over the pairs i it blends in blend order,
        distortion_p = sum_i sum_j w_i w_j |z_i - z_j| = 2 sum_i w_i (z_i A_i - D_i),
        A_i = sum_{j<i} w_j = 1 - T_i,   D_i = sum_{j<i} w_j z_j,
    with w_i = alpha_i T_i and z_i the view depth the depth plane blends ([1,H,W] float32, differentiable;
    f3dgs_forward_distortion / f3dgs_backward_distortion).  Each tile list is sorted by depth, so the prefix sums equal
    the pairwise sum.  The loss pulls each pixel's blend weights together along the ray, which removes semi-transparent
    floaters.  Its weight, and any normalisation by scene scale, is the caller's.  At ties in z the backward orders the
    tied pairs by blend order.  Colour, feature map, depth, radii and their gradients are those of the rasterizer
    without it.  `ViewBatch.forward_distortion` and `ViewBatch.backward(..., g_distortion=)` do the same without
    autograd.
  * vector-quantised feature fields (LightGaussian, CompGS): `kmeans(x, K)` fits a codebook [K,D] and int32 codes on the
    GPU (a TF32 tensor-core assignment with the argmin fused into the GEMM, float64 segment means), `decode(codebook,
    code)` gathers the rows back (float32 or float16), and `CodePlan(code, K)` gives the codebook gradient of the
    gather.  `GaussianState.quantize_features(K)` trains the codebook in place of per-Gaussian features, and io.save_ply
    stores it with one ushort code per Gaussian.
  * neighbour graphs of Gaussians: `knn_graph(points, k)` is the exact k-NN graph (f3dgs_knn_graph, int32 indices and
    squared distances, ties to the lower index).  Over it, `feature_tv_loss(features, graph, weight)` is the total
    variation of the feature field (Gaussian Grouping's 3-D neighbour term, in L1), `fill_features(features, weight,
    graph)` gives rows no view blended their neighbours' weighted mean, and `outlier_mask(graph, std_ratio)` is
    statistical outlier removal.  `GaussianState.add_feature_tv_grads` and `remove_outliers` use them in training.
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

from .filter3d import apply_3d_filter, compute_3d_filter  # noqa: E402
from .codebook import CodePlan, decode, kmeans  # noqa: E402
from .scores import GaussianScores  # noqa: E402
from .neighbors import (KnnGraph, feature_tv_loss, feature_tv_loss_and_grad, fill_features, knn_graph,  # noqa: E402
                        outlier_mask)

__all__ = [
    "GaussianRasterizationSettings",
    "GaussianRasterizer",
    "rasterize_gaussians",
    "rasterize_gaussians_feature_geometry",
    "AntialiasedGaussianRasterizer",
    "rasterize_gaussians_alpha_invdepth",
    "AlphaInvDepthGaussianRasterizer",
    "rasterize_gaussians_distortion",
    "DistortionGaussianRasterizer",
    "SparseGaussianAdam",
    "compute_3d_filter",
    "apply_3d_filter",
    "GaussianScores",
    "AbsGradGaussianRasterizer",
    "kmeans",
    "decode",
    "CodePlan",
    "KnnGraph",
    "knn_graph",
    "feature_tv_loss",
    "feature_tv_loss_and_grad",
    "fill_features",
    "outlier_mask",
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
                cov3Ds_precomp, raster_settings, antialiasing=False):
        fn = _C.rasterize_gaussians_antialiased if antialiasing else _C.rasterize_gaussians
        color, feature_map, depth, radii = _native_forward(ctx, fn, means3D, sh, colors_precomp, semantic_feature,
                                                           opacities, scales, rotations, cov3Ds_precomp,
                                                           raster_settings, antialiasing)
        return color, feature_map, radii, depth

    @staticmethod
    def backward(ctx, grad_out_color, grad_out_feature, _grad_radii, grad_depth):
        fn = _antialiased_backward(False, False) if ctx.antialiasing else _C.rasterize_gaussians_backward
        grads = _native_backward(ctx, fn, grad_out_color, grad_out_feature, grad_depth)
        return grads[:9] + (None, None)


def _native_forward(ctx, fn, means3D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                    cov3Ds_precomp, rs, antialiasing, save_depth=False):
    """The native forward `fn` with the reference forward's positional arguments; saves on ctx what _native_backward
    reads (save_depth: and the depth plane, last) -> fn's results between num_rendered and the three buffers, radii
    last"""
    if semantic_feature is None:
        semantic_feature = torch.empty(0, device=means3D.device, dtype=means3D.dtype)
    args = (rs.bg, means3D, colors_precomp, semantic_feature, opacities, scales, rotations, rs.scale_modifier,
            cov3Ds_precomp, rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height,
            rs.image_width, sh, rs.sh_degree, rs.campos, rs.prefiltered, rs.debug)
    (num_rendered, *outs, geomBuffer, binningBuffer, imgBuffer) = _call_native(
        fn, args, rs.debug, "snapshot_fw.dump", "forward")
    radii = outs[-1]
    ctx.raster_settings = rs
    ctx.antialiasing = antialiasing
    ctx.num_rendered = num_rendered
    ctx.save_for_backward(colors_precomp, semantic_feature, means3D, scales, rotations, cov3Ds_precomp, radii,
                          sh, geomBuffer, binningBuffer, imgBuffer, *((outs[2],) if save_depth else ()))
    ctx.mark_non_differentiable(radii)
    return outs


def _native_backward(ctx, fn, grad_out_color, grad_out_feature, grad_depth):
    """The native backward `fn` of a forward saved by _RasterizeGaussians.forward -> the autograd gradients of
    (means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations, cov3Ds_precomp), followed by
    whatever else `fn` returns."""
    rs = ctx.raster_settings
    (colors_precomp, semantic_feature, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer,
     binningBuffer, imgBuffer) = ctx.saved_tensors[:11]
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
     grad_cov3Ds_precomp, grad_sh, grad_scales, grad_rotations, *rest) = _call_native(
        fn, args, rs.debug, "snapshot_bw.dump", "backward")
    if not ctx.needs_input_grad[4]:
        grad_semantic_feature = None
    else:
        grad_semantic_feature = grad_semantic_feature.to(semantic_feature.dtype)
    return (grad_means3D, grad_means2D, grad_sh, grad_colors_precomp, grad_semantic_feature, grad_opacities,
            grad_scales, grad_rotations, grad_cov3Ds_precomp, *rest)


class _RasterizeGaussiansCamera(torch.autograd.Function):
    """_RasterizeGaussians with the camera as autograd inputs: viewmatrix, projmatrix and campos (the tensors of
    raster_settings, passed explicitly) also get gradients, from the native backward (f3dgs_backward_cam).  Intrinsics
    (tanfovx/y) are floats and get none."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                cov3Ds_precomp, viewmatrix, projmatrix, campos, raster_settings, antialiasing=False):
        rs = raster_settings._replace(viewmatrix=viewmatrix, projmatrix=projmatrix, campos=campos)
        ctx.camera_shapes = (viewmatrix.shape, projmatrix.shape, campos.shape)
        return _RasterizeGaussians.forward(ctx, means3D, means2D, sh, colors_precomp, semantic_feature, opacities,
                                           scales, rotations, cov3Ds_precomp, rs, antialiasing)

    @staticmethod
    def backward(ctx, grad_out_color, grad_out_feature, _grad_radii, grad_depth):
        fn = _antialiased_backward(True, False) if ctx.antialiasing else _C.rasterize_gaussians_backward_camera
        grads = _native_backward(ctx, fn, grad_out_color, grad_out_feature, grad_depth)
        cam = tuple(g.reshape(shape) for g, shape in zip(grads[9:], ctx.camera_shapes))
        return grads[:9] + cam + (None, None)


def _antialiased_backward(camera, feature_geometry):
    """rasterize_gaussians_backward_antialiased with the reference backward's positional arguments; the feature term
    reads the forward's semantic_feature (the fifth argument)"""
    return lambda *args: _C.rasterize_gaussians_backward_antialiased(
        *args, camera=camera, semantic_feature=args[4] if feature_geometry else None)


def _feature_geometry_backward(ctx, camera):
    """rasterize_gaussians_backward_feature_geometry (or its antialiased counterpart, for an antialiased forward) with
    the reference backward's positional arguments"""
    if ctx.antialiasing:
        return _antialiased_backward(camera, True)
    return lambda *args: _C.rasterize_gaussians_backward_feature_geometry(*args, camera)


class _RasterizeGaussiansFeatureGeometry(_RasterizeGaussians):
    """_RasterizeGaussians whose backward also carries the feature map's gradient into the geometry: the feature term
    of dL/dalpha (f3dgs_backward_feature_geometry), which reads semantic_feature."""

    @staticmethod
    def backward(ctx, grad_out_color, grad_out_feature, _grad_radii, grad_depth):
        grads = _native_backward(ctx, _feature_geometry_backward(ctx, False), grad_out_color, grad_out_feature,
                                 grad_depth)
        return grads[:9] + (None, None)


class _RasterizeGaussiansCameraFeatureGeometry(_RasterizeGaussiansCamera):
    """_RasterizeGaussiansCamera with the feature term of dL/dalpha, so that the camera gets it too."""

    @staticmethod
    def backward(ctx, grad_out_color, grad_out_feature, _grad_radii, grad_depth):
        grads = _native_backward(ctx, _feature_geometry_backward(ctx, True), grad_out_color, grad_out_feature,
                                 grad_depth)
        cam = tuple(g.reshape(shape) for g, shape in zip(grads[9:], ctx.camera_shapes))
        return grads[:9] + cam + (None, None)


class _RasterizeGaussiansAlphaInvDepth(torch.autograd.Function):
    """The render with the opacity and inverse-depth planes (f3dgs_forward_alpha_invdepth / f3dgs_backward_alpha_invdepth)
    in every mode: the camera tensors are always inputs and get gradients when they require grad; feature_geometry
    adds the feature term of dL/dalpha; antialiasing renders with the antialiased opacities."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                cov3Ds_precomp, viewmatrix, projmatrix, campos, raster_settings, feature_geometry, antialiasing):
        rs = raster_settings._replace(viewmatrix=viewmatrix, projmatrix=projmatrix, campos=campos)
        ctx.camera_shapes = (viewmatrix.shape, projmatrix.shape, campos.shape)
        ctx.feature_geometry = feature_geometry
        fn = lambda *args: _C.rasterize_gaussians_alpha_invdepth(*args, antialiasing=antialiasing)  # noqa: E731
        color, feature_map, depth, alpha, invdepth, radii = _native_forward(
            ctx, fn, means3D, sh, colors_precomp, semantic_feature, opacities, scales, rotations, cov3Ds_precomp, rs,
            antialiasing)
        return color, feature_map, radii, depth, alpha, invdepth

    @staticmethod
    def backward(ctx, grad_out_color, grad_out_feature, _grad_radii, grad_depth, grad_alpha, grad_invdepth):
        rs = ctx.raster_settings
        camera = any(ctx.needs_input_grad[9:12])
        planes = tuple(torch.zeros(1, rs.image_height, rs.image_width, device=rs.bg.device) if g is None else g
                       for g in (grad_alpha, grad_invdepth))
        fn = lambda *args: _C.rasterize_gaussians_backward_alpha_invdepth(  # noqa: E731
            *args, *planes, camera=camera, semantic_feature=args[4] if ctx.feature_geometry else None,
            antialiasing=ctx.antialiasing)
        grads = _native_backward(ctx, fn, grad_out_color, grad_out_feature, grad_depth)
        cam = tuple(None if g is None else g.reshape(shape) for g, shape in zip(grads[9:], ctx.camera_shapes))
        return grads[:9] + cam + (None, None, None)


def _rasterize_alpha_invdepth(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                              cov3Ds_precomp, rs, feature_geometry, antialiasing=False):
    return _RasterizeGaussiansAlphaInvDepth.apply(means3D, means2D, sh, colors_precomp, semantic_feature, opacities,
                                                  scales, rotations, cov3Ds_precomp, rs.viewmatrix, rs.projmatrix,
                                                  rs.campos, rs, feature_geometry, antialiasing)


class _RasterizeGaussiansDistortion(torch.autograd.Function):
    """The render with the depth distortion plane (f3dgs_forward_distortion / f3dgs_backward_distortion) in every mode:
    the camera tensors are always inputs and get gradients when they require grad; feature_geometry adds the feature
    term of dL/dalpha; antialiasing renders with the antialiased opacities.  The depth plane is saved: the backward
    reads it."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                cov3Ds_precomp, viewmatrix, projmatrix, campos, raster_settings, feature_geometry, antialiasing):
        rs = raster_settings._replace(viewmatrix=viewmatrix, projmatrix=projmatrix, campos=campos)
        ctx.camera_shapes = (viewmatrix.shape, projmatrix.shape, campos.shape)
        ctx.feature_geometry = feature_geometry
        fn = lambda *args: _C.rasterize_gaussians_distortion(*args, antialiasing=antialiasing)  # noqa: E731
        color, feature_map, depth, distortion, radii = _native_forward(
            ctx, fn, means3D, sh, colors_precomp, semantic_feature, opacities, scales, rotations, cov3Ds_precomp, rs,
            antialiasing, save_depth=True)
        return color, feature_map, radii, depth, distortion

    @staticmethod
    def backward(ctx, grad_out_color, grad_out_feature, _grad_radii, grad_depth, grad_distortion):
        rs = ctx.raster_settings
        camera = any(ctx.needs_input_grad[9:12])
        depth = ctx.saved_tensors[11]
        if grad_distortion is None:
            grad_distortion = torch.zeros(1, rs.image_height, rs.image_width, device=rs.bg.device)
        fn = lambda *args: _C.rasterize_gaussians_backward_distortion(  # noqa: E731
            *args, depth, grad_distortion, camera=camera, semantic_feature=args[4] if ctx.feature_geometry else None,
            antialiasing=ctx.antialiasing)
        grads = _native_backward(ctx, fn, grad_out_color, grad_out_feature, grad_depth)
        cam = tuple(None if g is None else g.reshape(shape) for g, shape in zip(grads[9:], ctx.camera_shapes))
        return grads[:9] + cam + (None, None, None)


def _rasterize_distortion(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                          cov3Ds_precomp, rs, feature_geometry, antialiasing=False):
    return _RasterizeGaussiansDistortion.apply(means3D, means2D, sh, colors_precomp, semantic_feature, opacities,
                                               scales, rotations, cov3Ds_precomp, rs.viewmatrix, rs.projmatrix,
                                               rs.campos, rs, feature_geometry, antialiasing)


class _RasterizeGaussiansAbsGrad(torch.autograd.Function):
    """The default or antialiased render whose backward also gives means2D_abs AbsGS's statistic, the view's sums over
    pixels of |x| and |y| of each pixel's dL/dmean2D term (f3dgs_backward_absgrad), in every mode: the camera tensors
    are always inputs and get gradients when they require grad; feature_geometry adds the feature term of dL/dalpha
    (and its walk's own absolute terms); antialiasing renders with the antialiased opacities."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                cov3Ds_precomp, means2D_abs, viewmatrix, projmatrix, campos, raster_settings, feature_geometry,
                antialiasing):
        rs = raster_settings._replace(viewmatrix=viewmatrix, projmatrix=projmatrix, campos=campos)
        ctx.camera_shapes = (viewmatrix.shape, projmatrix.shape, campos.shape)
        ctx.feature_geometry = feature_geometry
        fn = _C.rasterize_gaussians_antialiased if antialiasing else _C.rasterize_gaussians
        color, feature_map, depth, radii = _native_forward(ctx, fn, means3D, sh, colors_precomp, semantic_feature,
                                                           opacities, scales, rotations, cov3Ds_precomp, rs,
                                                           antialiasing)
        return color, feature_map, radii, depth

    @staticmethod
    def backward(ctx, grad_out_color, grad_out_feature, _grad_radii, grad_depth):
        camera = any(ctx.needs_input_grad[10:13])
        fn = lambda *args: _C.rasterize_gaussians_backward_absgrad(  # noqa: E731
            *args, camera=camera, semantic_feature=args[4] if ctx.feature_geometry else None,
            antialiasing=ctx.antialiasing)
        grads = _native_backward(ctx, fn, grad_out_color, grad_out_feature, grad_depth)
        cam = tuple(None if g is None else g.reshape(shape) for g, shape in zip(grads[9:12], ctx.camera_shapes))
        return grads[:9] + (grads[12],) + cam + (None, None, None)


def _rasterize_absgrad(means3D, means2D, means2D_abs, sh, colors_precomp, semantic_feature, opacities, scales,
                       rotations, cov3Ds_precomp, rs, feature_geometry, antialiasing=False):
    # means2D_abs after the reference's nine inputs: _native_backward reads semantic_feature's needs_input_grad at 4
    return _RasterizeGaussiansAbsGrad.apply(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales,
                                            rotations, cov3Ds_precomp, means2D_abs, rs.viewmatrix, rs.projmatrix,
                                            rs.campos, rs, feature_geometry, antialiasing)


def _camera_requires_grad(rs):
    return any(isinstance(t, torch.Tensor) and t.requires_grad for t in (rs.viewmatrix, rs.projmatrix, rs.campos))


def _rasterize(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations, cov3Ds_precomp,
               rs, feature_geometry, antialiasing=False):
    if torch.is_grad_enabled() and _camera_requires_grad(rs):
        fn = _RasterizeGaussiansCameraFeatureGeometry if feature_geometry else _RasterizeGaussiansCamera
        return fn.apply(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                        cov3Ds_precomp, rs.viewmatrix, rs.projmatrix, rs.campos, rs, antialiasing)
    fn = _RasterizeGaussiansFeatureGeometry if feature_geometry else _RasterizeGaussians
    return fn.apply(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                    cov3Ds_precomp, rs, antialiasing)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                        cov3Ds_precomp, raster_settings):
    return _rasterize(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                      cov3Ds_precomp, raster_settings, False)


def rasterize_gaussians_feature_geometry(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales,
                                         rotations, cov3Ds_precomp, raster_settings):
    """rasterize_gaussians whose backward also feeds the feature map's gradient into dL/dalpha, and so into the
    opacities, means, scales, rotations (or cov3Ds_precomp) and a camera that requires grad.  The render and every
    other gradient are rasterize_gaussians'."""
    return _rasterize(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales, rotations,
                      cov3Ds_precomp, raster_settings, True)


def rasterize_gaussians_alpha_invdepth(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales,
                                       rotations, cov3Ds_precomp, raster_settings, feature_geometry=False,
                                       antialiasing=False):
    """rasterize_gaussians (feature_geometry=True: rasterize_gaussians_feature_geometry; antialiasing=True: the
    antialiased render) that also returns the opacity plane alpha = 1 - T_final and the inverse-depth plane
    invdepth = sum_i w_i / z_i, [1,H,W] float32 each, and differentiates them ->
    (color, feature_map, radii, depth, alpha, invdepth).  Everything else, gradients included, is bitwise that of the
    call without the planes."""
    return _rasterize_alpha_invdepth(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales,
                                     rotations, cov3Ds_precomp, raster_settings, feature_geometry, antialiasing)


def rasterize_gaussians_distortion(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales,
                                   rotations, cov3Ds_precomp, raster_settings, feature_geometry=False,
                                   antialiasing=False):
    """rasterize_gaussians (feature_geometry=True: rasterize_gaussians_feature_geometry; antialiasing=True: the
    antialiased render) that also returns the depth distortion plane sum_ij w_i w_j |z_i - z_j| ([1,H,W] float32, see
    the module docstring) and differentiates it -> (color, feature_map, radii, depth, distortion).  Everything else,
    gradients included, is bitwise that of the call without it."""
    return _rasterize_distortion(means3D, means2D, sh, colors_precomp, semantic_feature, opacities, scales,
                                 rotations, cov3Ds_precomp, raster_settings, feature_geometry, antialiasing)


class GaussianRasterizer(nn.Module):
    """The reference's rasterizer module.  feature_geometry=True: the backward also feeds the feature map's gradient
    into the geometry (rasterize_gaussians_feature_geometry)."""

    antialiasing = False  # AntialiasedGaussianRasterizer
    _render = staticmethod(_rasterize)  # AlphaInvDepthGaussianRasterizer

    def __init__(self, raster_settings, feature_geometry=False):
        super().__init__()
        self.raster_settings = raster_settings
        self.feature_geometry = feature_geometry

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
        return self._render(means3D, means2D, shs, colors_precomp, semantic_feature, opacities, scales, rotations,
                            cov3D_precomp, rs, self.feature_geometry, self.antialiasing)


class AntialiasedGaussianRasterizer(GaussianRasterizer):
    """GaussianRasterizer with antialiased opacities: each opacity is scaled by sqrt(det(S) / det(S + 0.3 I)), S the
    2-D covariance before the 0.3 px^2 dilation, so that the dilation conserves a Gaussian's integral (see the module
    docstring).  The render and every gradient are those of the antialiased model; the arguments are
    GaussianRasterizer's."""

    antialiasing = True


class AlphaInvDepthGaussianRasterizer(GaussianRasterizer):
    """GaussianRasterizer whose forward also returns the opacity and inverse-depth planes:
    (color, feature_map, radii, depth, alpha, invdepth), alpha = 1 - T_final and invdepth = sum_i w_i / z_i, [1,H,W]
    float32 each, both differentiable (rasterize_gaussians_alpha_invdepth).  antialiasing=True renders with
    AntialiasedGaussianRasterizer's opacities."""

    _render = staticmethod(_rasterize_alpha_invdepth)

    def __init__(self, raster_settings, feature_geometry=False, antialiasing=False):
        super().__init__(raster_settings, feature_geometry)
        self.antialiasing = antialiasing


class DistortionGaussianRasterizer(GaussianRasterizer):
    """GaussianRasterizer whose forward also returns the depth distortion plane:
    (color, feature_map, radii, depth, distortion), distortion = sum_ij w_i w_j |z_i - z_j| per pixel, [1,H,W] float32
    and differentiable (rasterize_gaussians_distortion).  antialiasing=True renders with AntialiasedGaussianRasterizer's
    opacities."""

    _render = staticmethod(_rasterize_distortion)

    def __init__(self, raster_settings, feature_geometry=False, antialiasing=False):
        super().__init__(raster_settings, feature_geometry)
        self.antialiasing = antialiasing


class AbsGradGaussianRasterizer(GaussianRasterizer):
    """GaussianRasterizer for AbsGS (Ye et al., ACM MM 2024): forward(..., means2D_abs=screenspace_points_abs) takes a
    second [P,3] screen-space tensor that requires grad, and the backward gives it the view's per-Gaussian sums over
    pixels of |x| and |y| of each pixel's dL/dmean2D term (third column 0), the statistic of AbsGS's split rule.  The
    render and every other gradient are GaussianRasterizer's (AntialiasedGaussianRasterizer's with antialiasing=True);
    with feature_geometry the feature walk's terms are summed on their own and added (see f3dgs_backward_absgrad).
    Without means2D_abs the call is GaussianRasterizer's."""

    def __init__(self, raster_settings, feature_geometry=False, antialiasing=False):
        super().__init__(raster_settings, feature_geometry)
        self.antialiasing = antialiasing
        self._means2D_abs = None

    def forward(self, means3D, means2D, opacities, shs=None, semantic_feature=None, colors_precomp=None,
                scales=None, rotations=None, cov3D_precomp=None, means2D_abs=None):
        self._means2D_abs = means2D_abs  # read by _render, which GaussianRasterizer.forward calls
        try:
            return super().forward(means3D, means2D, opacities, shs, semantic_feature, colors_precomp, scales,
                                   rotations, cov3D_precomp)
        finally:
            self._means2D_abs = None

    def _render(self, means3D, means2D, *args):
        if self._means2D_abs is None:
            return _rasterize(means3D, means2D, *args)
        return _rasterize_absgrad(means3D, means2D, self._means2D_abs, *args)


class SparseGaussianAdam(torch.optim.Adam):
    """Sparse Adam for the autograd path (GaussianRasterizer on raw parameters): the upstream 3DGS rasterizer's
    SparseGaussianAdam, called the same way,

        optimizer = SparseGaussianAdam(param_groups, lr=0.0, eps=1e-15)
        ...
        optimizer.step(visibility=radii > 0, N=P)

    Each group holds one parameter of N rows (any trailing shape).  step() updates only the rows marked in
    `visibility` (bool or uint8 [N], on the parameter's device), with betas 0.9 and 0.999 and no bias correction:
    m = 0.9 m + 0.1 g, v = 0.999 v + 0.001 g^2, p -= lr m / (sqrt(v) + eps), in one native pass per group
    (f3dgs_adam_step_masked, step 0).  The other rows keep parameter and moments bitwise.  Groups whose parameter has
    no gradient are skipped.  The moments live in torch Adam's state keys (exp_avg, exp_avg_sq, and step, which stays
    0), so code that edits optimizer.state[param] directly, as the reference's densification does, keeps working."""

    def __init__(self, params, lr, eps):
        super().__init__(params=params, lr=lr, eps=eps)

    @torch.no_grad()
    def step(self, visibility, N):
        if visibility.numel() != N:
            raise ValueError(f"visibility has {visibility.numel()} elements, expected N = {N}")
        for group in self.param_groups:
            if len(group["params"]) != 1:
                raise ValueError("SparseGaussianAdam takes one parameter per group")
            param = group["params"][0]
            if param.grad is None:
                continue
            state = self.state[param]
            if len(state) == 0:
                state["step"] = torch.tensor(0.0, dtype=torch.float32)
                state["exp_avg"] = torch.zeros_like(param, memory_format=torch.preserve_format)
                state["exp_avg_sq"] = torch.zeros_like(param, memory_format=torch.preserve_format)
            _C.adam_step(0, param, param.grad, state["exp_avg"], state["exp_avg_sq"], 1, float(group["lr"]), 0.9, 0.999,
                         float(group["eps"]), 0, None, visibility)
