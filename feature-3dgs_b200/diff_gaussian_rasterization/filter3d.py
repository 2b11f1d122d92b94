"""Mip-Splatting's 3D smoothing filter (Yu et al., CVPR 2024; the official scene/gaussian_model.py compute_3D_filter,
get_opacity_with_3D_filter, get_scaling_with_3D_filter) on csrc/filter3d.cu.

Each Gaussian gets a world-space filter size from the highest sampling rate any training camera has at it.  Rendering
with the filtered opacity and scales keeps every Gaussian at least as large as the training views could sample, so
zooming in, rendering closer than any training camera or at a higher resolution shows no needles or erosion, in the
colour and in the feature map.  With a renderer written for the reference:

    filter_3D = compute_3d_filter(means3D, train_settings)     # every 100 iterations, and after densification
    opacity, scales = apply_3d_filter(opacities, scales, filter_3D)
    GaussianRasterizer(raster_settings=rs)(..., opacities=opacity, scales=scales, ...)

GaussianState.compute_3d_filter turns the filter on for the autograd-free training path (trainer.py).
"""
from typing import Sequence, Tuple

import torch

from . import _C


def camera_tensors(cameras: Sequence) -> Tuple[torch.Tensor, torch.Tensor]:
    """GaussianRasterizationSettings of the training cameras -> (viewmatrices [V,16], intrinsics [V,4]) float32 on the
    viewmatrices' device; intrinsics = (fx, fy, W, H), fx = W / (2 tanfovx) and fy = H / (2 tanfovy) from the settings'
    Python floats, rounded to float32 once (the official Camera's focal_x / focal_y)."""
    cameras = list(cameras)
    if not cameras:
        raise ValueError("compute_3d_filter needs at least one camera")
    vms = torch.stack([c.viewmatrix.detach().reshape(16) for c in cameras]).float().contiguous()
    intr = torch.tensor([[c.image_width / (2 * c.tanfovx), c.image_height / (2 * c.tanfovy), c.image_width,
                          c.image_height] for c in cameras], dtype=torch.float32).to(vms.device)
    return vms, intr


def compute_from_tensors(means3D: torch.Tensor, viewmatrices: torch.Tensor, intrinsics: torch.Tensor) -> torch.Tensor:
    """compute_3d_filter on camera_tensors' output -> [P,1] float32.  One host read, of the seen count."""
    filter_3D, n_seen = _C.filter3d_compute(means3D.detach(), viewmatrices, intrinsics)
    if means3D.shape[0] == 0 or int(n_seen) == 0:
        raise ValueError("compute_3d_filter: no Gaussian is seen by any camera")
    return filter_3D


def compute_3d_filter(means3D: torch.Tensor, cameras: Sequence) -> torch.Tensor:
    """The official compute_3D_filter: cameras is a sequence of GaussianRasterizationSettings (the training views) ->
    filter_3D [P,1] float32, the official shape.  A Gaussian that a camera sees (view-space depth z > 0.2 and its
    projection within 15 % of the image beyond every edge) takes the smallest such depth over the cameras; one that no
    camera sees takes the largest of those.  filter = depth / focal * sqrt(0.2), focal the largest fx of all cameras.
    Native (f3dgs_filter3d_compute), bitwise deterministic and independent of the camera order.  Raises ValueError when
    no Gaussian is seen by any camera (the official code fails there too)."""
    return compute_from_tensors(means3D, *camera_tensors(cameras))


class _Apply3DFilter(torch.autograd.Function):
    @staticmethod
    def forward(ctx, opacities, scales, filter_3D):
        o, s = _C.filter3d_apply(opacities, scales, filter_3D)
        ctx.save_for_backward(opacities, scales, filter_3D)
        return o.view_as(opacities), s

    @staticmethod
    def backward(ctx, grad_opacities, grad_scales):
        opacities, scales, filter_3D = ctx.saved_tensors
        if grad_opacities is None:
            grad_opacities = torch.zeros_like(opacities)
        if grad_scales is None:
            grad_scales = torch.zeros_like(scales)
        go, gs = _C.filter3d_apply_backward(opacities, scales, filter_3D, grad_opacities, grad_scales)
        return go.view_as(opacities), gs, None


def apply_3d_filter(opacities: torch.Tensor, scales: torch.Tensor, filter_3D: torch.Tensor):
    """The official get_opacity_with_3D_filter and get_scaling_with_3D_filter on activated opacities [P,1] and scales
    [P,3] -> (opacities * sqrt(det1 / det2), sqrt(scales^2 + filter_3D^2)), det1 = prod scales^2 and
    det2 = prod (scales^2 + filter_3D^2): bitwise the official float32 torch formula.  Differentiable in opacities and
    scales with a native backward (f3dgs_filter3d_apply / _apply_backward); the filter gets no gradient."""
    return _Apply3DFilter.apply(opacities, scales, filter_3D.detach())
