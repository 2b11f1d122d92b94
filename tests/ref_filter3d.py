"""Mip-Splatting's 3D filter restated in PyTorch: the official scene/gaussian_model.py compute_3D_filter,
get_opacity_with_3D_filter, get_scaling_with_3D_filter and reset_opacity, in this project's camera terms.  For camera v,
vm is its 16-float viewmatrix (world_view_transform = W2C^T, the layout the rasterizer takes), so the official
`xyz @ R + T` is `xyz @ vm[:3,:3] + vm[3,:3]`; fx = W / (2 tanfovx) and fy = H / (2 tanfovy) are Python floats (the
official Camera's focal_x / focal_y), passed here already rounded to float32 as the native path takes them.

The float32 functions are the official code as written (a per-camera loop of about 15 tensor kernels); `*64` evaluate
the same definitions in float64, for the gradient checks."""
import math

import torch


def compute_3d_filter(xyz, viewmatrices, intrinsics):
    """xyz [P,3] float32, viewmatrices [V,16], intrinsics [V,4] = (fx, fy, W, H) -> filter_3D [P,1] float32."""
    distance = torch.ones((xyz.shape[0]), device=xyz.device) * 100000.0
    valid_points = torch.zeros((xyz.shape[0]), device=xyz.device, dtype=torch.bool)
    focal_length = 0.0
    for vm, (fx, fy, W, H) in zip(viewmatrices.reshape(-1, 4, 4), intrinsics.tolist()):
        R, T = vm[:3, :3], vm[3, :3]
        xyz_cam = xyz @ R + T[None, :]
        valid_depth = xyz_cam[:, 2] > 0.2
        x, y, z = xyz_cam[:, 0], xyz_cam[:, 1], xyz_cam[:, 2]
        z = torch.clamp(z, min=0.001)
        x = x / z * fx + W / 2.0
        y = y / z * fy + H / 2.0
        in_screen = torch.logical_and(torch.logical_and(x >= -0.15 * W, x <= W * 1.15),
                                      torch.logical_and(y >= -0.15 * H, y <= 1.15 * H))
        valid = torch.logical_and(valid_depth, in_screen)
        distance[valid] = torch.min(distance[valid], z[valid])
        valid_points = torch.logical_or(valid_points, valid)
        if focal_length < fx:
            focal_length = fx
    distance[~valid_points] = distance[valid_points].max()
    filter_3D = distance / focal_length * (0.2 ** 0.5)
    return filter_3D[..., None]


def margins(xyz, viewmatrices, intrinsics):
    """For each Gaussian, the smallest relative distance, over the cameras, of its float64 projection to a screen margin
    or of its depth to the 0.2 threshold: where it is tiny the float32 rounding of the camera transform may decide
    `valid` either way."""
    x64 = xyz.double()
    rel = torch.full((xyz.shape[0],), math.inf, dtype=torch.float64, device=xyz.device)
    for vm, (fx, fy, W, H) in zip(viewmatrices.double().reshape(-1, 4, 4), intrinsics.tolist()):
        c = x64 @ vm[:3, :3] + vm[3, :3]
        z = c[:, 2].clamp(min=0.001)
        px, py = c[:, 0] / z * fx + W / 2.0, c[:, 1] / z * fy + H / 2.0
        for v, edge, scale in ((c[:, 2], 0.2, 0.2), (px, -0.15 * W, W), (px, 1.15 * W, W), (py, -0.15 * H, H),
                               (py, 1.15 * H, H)):
            rel = torch.minimum(rel, (v - edge).abs() / scale)
    return rel


def opacity_with_3d_filter(opacity, scales, filter_3D):
    """get_opacity_with_3D_filter on activated opacity [P,1] and scales [P,3]"""
    scales_square = torch.square(scales)
    det1 = scales_square.prod(dim=1)
    scales_after_square = scales_square + torch.square(filter_3D)
    det2 = scales_after_square.prod(dim=1)
    coef = torch.sqrt(det1 / det2)
    return opacity * coef[..., None]


def scaling_with_3d_filter(scales, filter_3D):
    """get_scaling_with_3D_filter"""
    scales = torch.square(scales) + torch.square(filter_3D)
    return torch.sqrt(scales)


def reset_opacity(raw_opacity, raw_scaling, filter_3D, ceiling=0.01):
    """reset_opacity: the new raw opacity [P,1]"""
    scales = torch.exp(raw_scaling)
    current_opacity_with_filter = opacity_with_3d_filter(torch.sigmoid(raw_opacity), scales, filter_3D)
    opacities_new = torch.min(current_opacity_with_filter, torch.ones_like(current_opacity_with_filter) * ceiling)
    scales_square = torch.square(scales)
    det1 = scales_square.prod(dim=1)
    scales_after_square = scales_square + torch.square(filter_3D)
    det2 = scales_after_square.prod(dim=1)
    coef = torch.sqrt(det1 / det2)
    opacities_new = opacities_new / coef[..., None]
    return torch.log(opacities_new / (1 - opacities_new))


def apply64(opacity, scales, filter_3D):
    """(o_f, s_f) in float64, differentiable in opacity and scales"""
    o, s, f = opacity.double(), scales.double(), filter_3D.double()
    return opacity_with_3d_filter(o, s, f), scaling_with_3d_filter(s, f)
