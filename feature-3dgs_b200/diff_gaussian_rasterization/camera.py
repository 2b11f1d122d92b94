"""Differentiable camera glue for pose refinement, localisation and tracking (plain torch, no native code).

    xi = torch.zeros(6, device="cuda", requires_grad=True)          # pose delta (rho, phi)
    rs = settings_from_w2c(se3_exp(xi) @ w2c0, tanfovx, tanfovy, H, W, bg)
    color, feat, radii, depth = rasterize_gaussians(..., raster_settings=rs)   # routes to the camera-aware backward
    loss(color).backward()                                             # xi.grad

`settings_from_w2c` builds the settings as the reference's `Camera` (scene/cameras.py) and `getProjectionMatrix`
(utils/graphics_utils.py) do, with differentiable ops: for a float32 world-to-camera matrix the three tensors are
bitwise the reference's.
"""
import torch

from . import GaussianRasterizationSettings

__all__ = ["projection_matrix", "settings_from_w2c", "se3_exp"]


def projection_matrix(tanfovx: float, tanfovy: float, znear: float = 0.01, zfar: float = 100.0, device=None):
    """The reference getProjectionMatrix (row-major [4,4] float32) for tan(fov/2) = tanfovx, tanfovy."""
    top = tanfovy * znear
    bottom = -top
    right = tanfovx * znear
    left = -right
    P = torch.zeros(4, 4, device=device)
    z_sign = 1.0
    P[0, 0] = 2.0 * znear / (right - left)
    P[1, 1] = 2.0 * znear / (top - bottom)
    P[0, 2] = (right + left) / (right - left)
    P[1, 2] = (top + bottom) / (top - bottom)
    P[3, 2] = z_sign
    P[2, 2] = z_sign * zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def settings_from_w2c(w2c: torch.Tensor, tanfovx: float, tanfovy: float, image_height: int, image_width: int,
                      bg: torch.Tensor, znear: float = 0.01, zfar: float = 100.0, scale_modifier: float = 1.0,
                      sh_degree: int = 0, prefiltered: bool = False, debug: bool = False):
    """GaussianRasterizationSettings of the world-to-camera matrix `w2c` [4,4] (column-vector convention, the
    reference's getWorld2View2), differentiable in `w2c`:
        viewmatrix = w2c^T, projmatrix = viewmatrix @ proj^T, campos = viewmatrix.inverse()[3, :3] (the camera centre).
    """
    world_view = w2c.transpose(0, 1)
    proj = projection_matrix(tanfovx, tanfovy, znear, zfar, device=w2c.device).transpose(0, 1)
    full_proj = world_view.unsqueeze(0).bmm(proj.unsqueeze(0)).squeeze(0)
    campos = world_view.inverse()[3, :3]
    return GaussianRasterizationSettings(
        image_height=int(image_height), image_width=int(image_width), tanfovx=tanfovx, tanfovy=tanfovy, bg=bg,
        scale_modifier=scale_modifier, viewmatrix=world_view, projmatrix=full_proj, sh_degree=sh_degree,
        campos=campos, prefiltered=prefiltered, debug=debug)


def _hat(v: torch.Tensor) -> torch.Tensor:
    z = torch.zeros((), dtype=v.dtype, device=v.device)
    return torch.stack([torch.stack([z, -v[2], v[1]]), torch.stack([v[2], z, -v[0]]),
                        torch.stack([-v[1], v[0], z])])


def se3_exp(xi: torch.Tensor) -> torch.Tensor:
    """exp of the twist xi = (rho[3], phi[3]) -> [4,4] rigid transform [[R, V rho], [0, 1]] (R = exp(hat(phi)),
    Rodrigues), differentiable at xi = 0 as well (Taylor branch for small angles).  Left-multiply a world-to-camera
    matrix with it to move the camera in its own frame: w2c = se3_exp(xi) @ w2c0."""
    rho, phi = xi[:3], xi[3:6]
    th2 = (phi * phi).sum()
    small = th2 < 1e-8
    th2s = torch.where(small, torch.ones_like(th2), th2)  # keeps the unused branch finite (and its gradient)
    th = th2s.sqrt()
    A = torch.where(small, 1.0 - th2 / 6.0, th.sin() / th)                        # sin t / t
    B = torch.where(small, 0.5 - th2 / 24.0, (1.0 - th.cos()) / th2s)             # (1 - cos t) / t^2
    C = torch.where(small, 1.0 / 6.0 - th2 / 120.0, (th - th.sin()) / (th2s * th))  # (t - sin t) / t^3
    K = _hat(phi)
    K2 = K @ K
    eye = torch.eye(3, dtype=xi.dtype, device=xi.device)
    R = eye + A * K + B * K2
    V = eye + B * K + C * K2
    top = torch.cat([R, (V @ rho).unsqueeze(1)], dim=1)
    bottom = torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=xi.dtype, device=xi.device)
    return torch.cat([top, bottom], dim=0)

