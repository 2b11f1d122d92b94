"""Float64 torch restatement of what the composite reads for each Gaussian -- NDC mean, conic, colour and view depth --
as a function of (means3D, cov3D, shs or colours, viewmatrix, projmatrix, campos), for the camera gradient.

It follows the native backward's conventions (csrc/preprocess.cu, preprocess_bwd_kernel):
  * a clamped view-space coordinate of the EWA Jacobian is a constant (detached);
  * the screen mean is h_r / (h_w + 1e-7);
  * the conic's gradient divides by det^2 + 1e-7;
  * clamped colour channels pass no gradient.
Contracted with the composite's per-Gaussian gradients (dL_dmean2D per NDC unit, dL_dconic [P,4] with the off-diagonal
entry counted twice, dL_dcolor, dL_dz) it is a scalar whose gradients are the backward preprocess's.  The camera tensors
are given one copy per Gaussian, so `terms` returns each Gaussian's own contribution: their sum is the camera gradient
and the sum of their magnitudes scales its error bar.
"""
import torch

SH_C0 = 0.28209479177387814
SH_C1 = 0.4886025119029199
SH_C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
SH_C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
         1.445305721320277, -0.5900435899266435]


class _Conic(torch.autograd.Function):
    """(a, b, c) -> (c, -b, a) / det with the backward's 1 / (det^2 + 1e-7)."""

    @staticmethod
    def forward(ctx, a, b, c):
        ctx.save_for_backward(a, b, c)
        det = a * c - b * b
        return c / det, -b / det, a / det

    @staticmethod
    def backward(ctx, gx, gy, gz):
        a, b, c = ctx.saved_tensors
        denom = a * c - b * b
        d2 = 1.0 / (denom * denom + 1e-7)
        ga = d2 * (-c * c * gx + b * c * gy + (denom - a * c) * gz)
        gc = d2 * (-a * a * gz + a * b * gy + (denom - a * c) * gx)
        gb = d2 * (2 * b * c * gx - (denom + 2 * b * b) * gy + 2 * a * b * gz)
        return ga, gb, gc


def sh_color(deg, sh, d):
    x, y, z = d[:, 0:1], d[:, 1:2], d[:, 2:3]
    r = SH_C0 * sh[:, 0]
    if deg > 0:
        r = r - SH_C1 * y * sh[:, 1] + SH_C1 * z * sh[:, 2] - SH_C1 * x * sh[:, 3]
        if deg > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            r = (r + SH_C2[0] * xy * sh[:, 4] + SH_C2[1] * yz * sh[:, 5] + SH_C2[2] * (2 * zz - xx - yy) * sh[:, 6]
                 + SH_C2[3] * xz * sh[:, 7] + SH_C2[4] * (xx - yy) * sh[:, 8])
            if deg > 2:
                r = (r + SH_C3[0] * y * (3 * xx - yy) * sh[:, 9] + SH_C3[1] * xy * z * sh[:, 10]
                     + SH_C3[2] * y * (4 * zz - xx - yy) * sh[:, 11]
                     + SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[:, 12]
                     + SH_C3[4] * x * (4 * zz - xx - yy) * sh[:, 13] + SH_C3[5] * z * (xx - yy) * sh[:, 14]
                     + SH_C3[6] * x * (xx - 3 * yy) * sh[:, 15])
    return r + 0.5


def screen_quantities(means3D, cov3D, vm, pm, campos, W, H, tanfovx, tanfovy, deg=0, shs=None, colors=None,
                      vm_depth=None):
    """Per-Gaussian (ndc [P,2], conic (A, B, C) each [P], colour [P,3], depth [P]).  vm, pm: [P,16] or [16]; campos:
    [P,3] or [3], in the kernels' layout (m[4k + r] is row r, column k).  vm_depth (default vm): the viewmatrix the
    depth is read from, so that the depth's share of dL/dviewmatrix can be told from the conic's."""
    P = means3D.shape[0]
    vm = vm.expand(P, 16) if vm.dim() == 1 else vm
    vm_depth = vm if vm_depth is None else vm_depth
    pm = pm.expand(P, 16) if pm.dim() == 1 else pm
    campos = campos.expand(P, 3) if campos.dim() == 1 else campos
    p = torch.cat([means3D, torch.ones_like(means3D[:, :1])], 1)

    def row(m, r):
        return (m[:, r::4] * p).sum(1)

    hx, hy, hw = row(pm, 0), row(pm, 1), row(pm, 3)
    p_w = 1.0 / (hw + 1e-7)
    ndc = torch.stack([hx * p_w, hy * p_w], 1)
    tx, ty, tz = row(vm, 0), row(vm, 1), row(vm, 2)
    fx, fy = W / (2.0 * tanfovx), H / (2.0 * tanfovy)
    limx, limy = 1.3 * tanfovx, 1.3 * tanfovy
    rx, ry = tx / tz, ty / tz
    cx = (rx < -limx) | (rx > limx)
    cy = (ry < -limy) | (ry > limy)
    tx = torch.where(cx, (rx.clamp(-limx, limx) * tz).detach(), tx)
    ty = torch.where(cy, (ry.clamp(-limy, limy) * tz).detach(), ty)
    zero = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, zero, -fx * tx / (tz * tz)], 1),
                     torch.stack([zero, fy / tz, -fy * ty / (tz * tz)], 1)], 1)  # [P, 2, 3]
    Wr = torch.stack([vm[:, 0:3], vm[:, 4:7], vm[:, 8:11]], 1)  # Wr[:, k, r] = vm[4k + r]: row r of the rotation, col k
    T = J @ Wr.transpose(1, 2)  # [P, 2, 3]: T[a, k] = sum_r J[a, r] vm[4k + r]
    c = cov3D
    V = torch.stack([torch.stack([c[:, 0], c[:, 1], c[:, 2]], 1), torch.stack([c[:, 1], c[:, 3], c[:, 4]], 1),
                     torch.stack([c[:, 2], c[:, 4], c[:, 5]], 1)], 1)
    S = T @ V @ T.transpose(1, 2)
    A, B, C = _Conic.apply(S[:, 0, 0] + 0.3, S[:, 0, 1], S[:, 1, 1] + 0.3)
    if colors is None:
        d = means3D - campos
        d = d / d.norm(dim=1, keepdim=True)
        colors = sh_color(deg, shs, d).clamp_min(0.0)
    depth = row(vm_depth, 2)
    return ndc, (A, B, C), colors, depth


def contract(q, dL_dmean2D, dL_dconic, dL_dcolor, dL_dz):
    ndc, (A, B, C), colors, depth = q
    return ((ndc * dL_dmean2D[:, :2]).sum() + (A * dL_dconic[:, 0] + 2 * B * dL_dconic[:, 1] + C * dL_dconic[:, 3]).sum()
            + (colors * dL_dcolor).sum() + (depth * dL_dz).sum())


def terms(means3D, cov3D, vm, pm, campos, grads, W, H, tanfovx, tanfovy, deg=0, shs=None, colors=None,
          visible=None):
    """Float64 gradients of the contracted loss: dict(means3D [P,3], cov3D [P,6], vm [P,16], pm [P,16], campos [P,3])
    per Gaussian, over the `visible` rows only (rows outside it are 0).  grads = (dL_dmean2D, dL_dconic, dL_dcolor,
    dL_dz).  vm = vm_cov + vm_depth: the share through the EWA projection (t and W of T = W J) and the depth's.  Also
    kappa and eig_ratio, the conditioning and eigenvalue ratio of each 2-D covariance."""
    f = lambda a: torch.as_tensor(a).double()  # noqa: E731
    P = means3D.shape[0]
    vis = torch.ones(P, dtype=torch.bool) if visible is None else torch.as_tensor(visible).bool()
    idx = vis.nonzero().flatten()
    n = idx.numel()
    m = f(means3D)[idx].clone().requires_grad_()
    cv = f(cov3D)[idx].clone().requires_grad_()
    vmP = f(vm).reshape(16).expand(n, 16).clone().requires_grad_()
    vmD = f(vm).reshape(16).expand(n, 16).clone().requires_grad_()
    pmP = f(pm).reshape(16).expand(n, 16).clone().requires_grad_()
    cpP = f(campos).reshape(3).expand(n, 3).clone().requires_grad_()
    q = screen_quantities(m, cv, vmP, pmP, cpP, W, H, tanfovx, tanfovy, deg,
                          shs=None if shs is None else f(shs)[idx], colors=None if colors is None else f(colors)[idx],
                          vm_depth=vmD)
    g = [f(x).reshape(P, -1)[idx] for x in grads]
    L = contract(q, g[0], g[1], g[2], g[3].reshape(-1))
    gm, gc, gv, gvd, gp, gcp = torch.autograd.grad(L, [m, cv, vmP, vmD, pmP, cpP], allow_unused=True)
    A, B, C = (x.detach() for x in q[1])
    mid, d = 0.5 * (A + C), torch.sqrt(0.25 * (A - C) ** 2 + B * B)
    out = {"kappa": torch.zeros(P, dtype=torch.float64), "eig_ratio": torch.zeros(P, dtype=torch.float64)}
    out["kappa"][idx] = (A * C + B * B) / (A * C - B * B)
    out["eig_ratio"][idx] = (mid + d) / (mid - d)
    for k, v, w in (("means3D", gm, 3), ("cov3D", gc, 6), ("vm_cov", gv, 16), ("vm_depth", gvd, 16), ("pm", gp, 16),
                    ("campos", gcp, 3)):
        full = torch.zeros(P, w, dtype=torch.float64)
        if v is not None:
            full[idx] = v
        out[k] = full
    out["vm"] = out["vm_cov"] + out["vm_depth"]
    return out


def camera_vector(t):
    """The 35-float layout of the native camera gradient from per-Gaussian terms (summed over Gaussians)."""
    return torch.cat([t["vm"].sum(0), t["pm"].sum(0), t["campos"].sum(0)])


def camera_scale(t, rel=1e-5, cond_max=100.0, needles=True):
    """Per entry of the camera gradient, the sum over Gaussians of its terms' magnitudes, the scale of the float32
    rounding error for a bar rel * scale.  Only the share through the EWA projection (vm_cov) passes through the
    backward's conic gradient, which evaluates det = ac - b^2 in float32, so its relative error grows with the
    conditioning kappa: that share is weighted by kappa.  For a Gaussian whose conic eigenvalue ratio exceeds cond_max
    (a needle) the float32 chain cancels terms of size ~ratio against each other and a float64 model does not bound
    it -- parity.tie_aware_compare skips the gradients through the 2-D covariance there -- so that share counts with
    its whole magnitude (|term| / rel) when `needles`, and not at all otherwise (the well-conditioned scale, for a
    floor).  The depth, projmatrix and campos terms never pass through the conic and count once, needles included."""
    well = t["eig_ratio"] <= cond_max
    k = torch.where(well, t["kappa"].clamp_min(1.0), torch.full_like(t["kappa"], 1.0 / rel if needles else 0.0))
    vm = (t["vm_cov"].abs() * k[:, None] + t["vm_depth"].abs()).sum(0)
    return torch.cat([vm, t["pm"].abs().sum(0), t["campos"].abs().sum(0)])
