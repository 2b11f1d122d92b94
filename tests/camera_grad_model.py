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
import numpy as np
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


def sh_basis_abs(deg, d):
    """The SH basis of sh_color with every constant and every sign taken positive, at d >= 0 ([P, 3]): the magnitude of
    the products the kernel forms for each coefficient's gradient, and (differentiated by d) for the view-direction
    gradient.  -> [P, (deg + 1)^2]."""
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    out = [torch.full_like(x, SH_C0)]
    if deg > 0:
        out += [SH_C1 * y, SH_C1 * z, SH_C1 * x]
    if deg > 1:
        c = [abs(v) for v in SH_C2]
        out += [c[0] * x * y, c[1] * y * z, c[2] * (2 * z * z + x * x + y * y), c[3] * x * z, c[4] * (x * x + y * y)]
    if deg > 2:
        c = [abs(v) for v in SH_C3]
        xx, yy, zz = x * x, y * y, z * z
        out += [c[0] * y * (3 * xx + yy), c[1] * x * y * z, c[2] * y * (4 * zz + xx + yy),
                c[3] * z * (2 * zz + 3 * xx + 3 * yy), c[4] * x * (4 * zz + xx + yy), c[5] * z * (xx + yy),
                c[6] * x * (xx + 3 * yy)]
    return torch.stack(out, 1)


def cov3d_from_scale_rot(scales, rotations, mod=1.0):
    """Float64 torch twin of the forward's computeCov3D ([P,6] upper triangle), differentiable.  Rc[:, i] is column i of
    the forward's GLM rotation; GLM's M = S R has M[c][r] = s[r] Rc[c][r], and Sigma = M^T M has
    Sigma[i][j] = sum_k s_k^2 Rc[i][k] Rc[j][k]."""
    s = scales * mod
    r, x, y, z = rotations.unbind(1)
    Rc = torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                      torch.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                      torch.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], 1)
    M = Rc * s[:, None, :]
    S = M @ M.transpose(1, 2)
    return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1)


def screen_quantities(means3D, cov3D, vm, pm, campos, W, H, tanfovx, tanfovy, deg=0, shs=None, colors=None,
                      vm_depth=None, clamp_grad=False):
    """Per-Gaussian (ndc [P,2], conic (A, B, C) each [P], colour [P,3], depth [P]).  vm, pm: [P,16] or [16]; campos:
    [P,3] or [3], in the kernels' layout (m[4k + r] is row r, column k).  vm_depth (default vm): the viewmatrix the
    depth is read from, so that the depth's share of dL/dviewmatrix can be told from the conic's.  clamp_grad: let the
    clamped view-space coordinate of the Jacobian pass its gradient (not what the kernels do: a negative control)."""
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
    keep = (lambda x: x) if clamp_grad else (lambda x: x.detach())
    tx = torch.where(cx, keep(rx.clamp(-limx, limx) * tz), tx)
    ty = torch.where(cy, keep(ry.clamp(-limy, limy) * tz), ty)
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


K_PRE = 32  # preprocess bar constant (see preprocess_chain)


def _f64(a):
    return (a.detach().cpu() if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a))).double()


def preprocess_chain(means3D, vm, pm, campos, W, H, tanfovx, tanfovy, grads, visible, deg=0, shs=None, clamped=None,
                     colors=None, scales=None, rotations=None, mod=1.0, cov3D=None, clamp_grad=False):
    """The backward preprocess in float64 from the composite's own per-Gaussian gradients, with a per-entry bar.

    grads = (dL_dmean2D [P,3], dL_dconic [P,4], dL_dcolor [P,3], dL_dz [P]) as the backward returns them; visible: the
    rows the preprocess runs on; clamped [P,3]: the colour channels the forward clamped (they pass no gradient).  The
    covariance comes from (scales * mod, rotations) or the precomputed cov3D, the colour from shs [P,M,3] at degree deg
    or the precomputed colors.  (A precomputed colour's gradient is the composite's dL/dcolor itself, which the
    preprocess does not touch: the chain has nothing of its own to say about it.)  The model is torch autograd of contract() through screen_quantities, on
    camera_grad_model's conventions.  -> dict of float64 [P, ...] (0 outside visible): means3D, cov3D (the leaf when
    precomputed, else the covariance formed from scales and rotations), scales and rotations unless cov3D is
    precomputed, and sh unless the colours are; for each the same key with "mag_" (below); kappa and eig_ratio of the conic,
    and kappa_eff, the factor the conic gradients' bar carries (below); cov_share_means3D, the part of dL/dmeans3D that
    passes through the 2-D covariance; outside, whether the mean is outside the Jacobian's 1.3 tan_fov limit.
    clamp_grad: see screen_quantities.

    Bar.  mag_X is the kernel's own expression for X (csrc/preprocess.cu, preprocess_bwd_kernel) evaluated with every
    operand replaced by its magnitude and every subtraction by an addition, in float64: to first order the kernel's
    float32 result is within (number of roundings on the longest path) u mag_X of the exact value of its expression,
    and the model is that value.  Two operands carry an error larger than their roundings: det = ac - b^2, whose
    cancellation (ac + b^2) / (ac - b^2) measures, with a, b, c at the magnitudes of the products that form them (the
    2-D covariance |T| |V| |T|^T, where |V| of a covariance formed from scales and rotations is the magnitude of its
    own float32 sum, sum_k s_k^2 |R_ik R_jk|); and the recomputed view depth t_z, whose cancellation its abs-evaluation
    over its value measures.  The conic gradients dL/d(a, b, c), and everything that flows from them, carry the product
    of the two, and use the same magnitudes of a, b and c.  The longest paths
    round about 20 times: the conic backward (4), dL/dcov3D (3) and the recomputed T = W J (4), then to the mean through
    dL/dT, dL/dJ, dL/dt and the view rotation (8), or to the rotation through dL/dM, dL/dM^T and the quaternion terms
    (7) with the recomputed rotation matrix (3).  So bar = K_PRE u mag_X with K_PRE = 32, which leaves room for the
    second-order terms; FMA contraction only removes roundings.  The SH coefficient gradients are single products of a
    basis value (at most ~12 u from the normalised direction and its monomials) and the colour gradient, within it."""
    P = int(np.asarray(_f64(means3D)).shape[0])
    vis = _f64(visible).bool().reshape(-1)
    idx = vis.nonzero().flatten()
    n = idx.numel()
    vm16, pm16, cp = _f64(vm).reshape(16), _f64(pm).reshape(16), _f64(campos).reshape(3)
    g = [_f64(x).reshape(P, -1)[idx] for x in grads]
    p = _f64(means3D)[idx].clone().requires_grad_()
    leaves = {"means3D": p}
    if cov3D is None:
        s = (_f64(scales)[idx] * mod).clone().requires_grad_()
        r = _f64(rotations)[idx].clone().requires_grad_()
        cv = cov3d_from_scale_rot(s, r)
        leaves.update(scales=s, rotations=r, cov3D=cv)  # dL/dcov3D, which the kernel also writes on this path
    else:
        cv = _f64(cov3D)[idx].clone().requires_grad_()
        leaves["cov3D"] = cv
    keep = ~_f64(clamped).bool().reshape(P, 3)[idx] if clamped is not None else torch.ones(n, 3, dtype=torch.bool)
    if colors is None:
        sh = _f64(shs)[idx].clone().requires_grad_()
        leaves["sh"] = sh
        dvec = p - cp
        col = sh_color(deg, sh, dvec / dvec.norm(dim=1, keepdim=True)) * keep.double()
    else:
        col = _f64(colors)[idx]
    q = screen_quantities(p, cv, vm16, pm16, cp, W, H, tanfovx, tanfovy, colors=col, clamp_grad=clamp_grad)
    out_g = torch.autograd.grad(contract(q, g[0], g[1], g[2], g[3].reshape(-1)), list(leaves.values()),
                                retain_graph=True)
    ndc, (A, B, C), _, _ = q
    zero = torch.zeros_like(g[0])
    cov_share = torch.autograd.grad(contract((ndc, (A, B, C), col, q[3]), zero, g[1], zero[:, :3] * 0,
                                             zero[:, 0]), [p], allow_unused=True)[0]
    out = {}

    def full(key, v):
        t = torch.zeros((P,) + tuple(v.shape[1:]), dtype=torch.float64)
        t[idx] = v
        out[key] = t

    for k, v in zip(leaves, out_g):
        full(k, v)
    full("cov_share_means3D", cov_share if cov_share is not None else torch.zeros(n, 3, dtype=torch.float64))
    A, B, C = (x.detach() for x in (A, B, C))
    mid, dd = 0.5 * (A + C), torch.sqrt(0.25 * (A - C) ** 2 + B * B)
    full("kappa", (A * C + B * B) / (A * C - B * B))
    full("eig_ratio", (mid + dd) / (mid - dd))

    # ---------------------------------------------------------------- magnitudes of the kernel's expressions
    with torch.no_grad():
        p = p.detach()
        cv = cv.detach()
        ph = torch.cat([p, torch.ones(n, 1, dtype=torch.float64)], 1)
        vma, pma = vm16.abs(), pm16.abs()

        def row(m, r):
            return ph @ m[r::4]

        def row_abs(m, r):
            return ph.abs() @ m[r::4].abs()

        tx, ty, tz = row(vm16, 0), row(vm16, 1), row(vm16, 2)
        cond_t = row_abs(vm16, 2) / tz.abs()
        fx, fy = W / (2.0 * tanfovx), H / (2.0 * tanfovy)
        limx, limy = 1.3 * tanfovx, 1.3 * tanfovy
        xmul = ((tx / tz).abs() <= limx).double()
        ymul = ((ty / tz).abs() <= limy).double()
        txc, tyc = (tx / tz).clamp(-limx, limx) * tz, (ty / tz).clamp(-limy, limy) * tz
        itz = 1.0 / tz.abs()
        J00, J02, J11, J12 = fx * itz, fx * txc.abs() * itz ** 2, fy * itz, fy * tyc.abs() * itz ** 2
        A0 = torch.stack([J00 * vma[4 * k] + J02 * vma[4 * k + 2] for k in range(3)], 1)  # |T[0, k]|
        A1 = torch.stack([J11 * vma[4 * k + 1] + J12 * vma[4 * k + 2] for k in range(3)], 1)  # |T[1, k]|
        V = torch.stack([torch.stack([cv[:, 0], cv[:, 1], cv[:, 2]], 1), torch.stack([cv[:, 1], cv[:, 3], cv[:, 4]], 1),
                         torch.stack([cv[:, 2], cv[:, 4], cv[:, 5]], 1)], 1)
        if cov3D is None:
            # the covariance the forward formed in float32: each entry within a few u of sum_k s_k^2 |R_ik R_jk|
            sa, (qr, qx, qy, qz) = s.detach().abs(), r.detach().abs().unbind(1)
            Ra = torch.stack([torch.stack([1 + 2 * (qy * qy + qz * qz), 2 * (qx * qy + qr * qz), 2 * (qx * qz + qr * qy)], -1),
                              torch.stack([2 * (qx * qy + qr * qz), 1 + 2 * (qx * qx + qz * qz), 2 * (qy * qz + qr * qx)], -1),
                              torch.stack([2 * (qx * qz + qr * qy), 2 * (qy * qz + qr * qx), 1 + 2 * (qx * qx + qy * qy)], -1)],
                             1)  # |R[c][r]|, the kernel's column-major R
            Va = torch.einsum("nik,nk,njk->nij", Ra, sa * sa, Ra)
        else:
            Va = V.abs()
        # sum_j |T[a, j]| |V[j, k]| of the values (TV0, TV1) and of the magnitudes the covariance is formed from
        TV0, TV1 = (A0[:, :, None] * V.abs()).sum(1), (A1[:, :, None] * V.abs()).sum(1)
        TW0, TW1 = (A0[:, :, None] * Va).sum(1) * cond_t[:, None], (A1[:, :, None] * Va).sum(1) * cond_t[:, None]
        # the recomputed 2-D covariance, and the magnitudes of its float32 errors (per u; t_z's through T)
        a, b, c = 1.0 / (A * C - B * B) * C, -B / (A * C - B * B), A / (A * C - B * B)
        aA, bA, cA = (TW0 * A0).sum(1) * cond_t + 0.3, (TW0 * A1).sum(1) * cond_t, (TW1 * A1).sum(1) * cond_t + 0.3
        ab_, bc_, ac_ = (a * b).abs(), (b * c).abs(), a * c
        # first-order error of a product x y: |x| err(y) + err(x) |y|
        m_ac, m_ab, m_bc, m_bb = c * aA + a * cA, a * bA + b.abs() * aA, c * bA + b.abs() * cA, 2 * b.abs() * bA
        den = ac_ - b * b
        den_m = m_ac + m_bb + ac_ + b * b  # its inputs' errors and its own two roundings
        kap = den_m / den
        full("kappa_eff", kap)
        full("outside", ((1 - xmul) + (1 - ymul)).clamp(max=1.0))
        D2 = 1.0 / (den * den)  # relative error 2 kap
        Lx, Ly, Lz = g[1][:, 0].abs(), g[1][:, 1].abs(), g[1][:, 3].abs()
        # each numerator's value magnitude (n) and error magnitude (e): dL/dx = D2 n with error D2 (2 kap n + e)
        n_a = c * c * Lx + 2 * bc_ * Ly + b * b * Lz
        n_c = a * a * Lz + 2 * ab_ * Ly + b * b * Lx
        n_b = 2 * (bc_ * Lx + (den.abs() + 2 * b * b) * Ly + ab_ * Lz)
        e_a = 2 * c * cA * Lx + 2 * m_bc * Ly + (den_m + m_ac) * Lz
        e_c = 2 * a * aA * Lz + 2 * m_ab * Ly + (den_m + m_ac) * Lx
        e_b = 2 * (m_bc * Lx + (den_m + 2 * m_bb) * Ly + m_ab * Lz)
        da_v, dc_v, db_v = D2 * n_a, D2 * n_c, D2 * n_b
        da, dc, db = D2 * (2 * kap * n_a + e_a), D2 * (2 * kap * n_c + e_c), D2 * (2 * kap * n_b + e_b)
        dcov = torch.stack([A0[:, 0] ** 2 * da + A0[:, 0] * A1[:, 0] * db + A1[:, 0] ** 2 * dc,
                            2 * A0[:, 0] * A0[:, 1] * da + (A0[:, 0] * A1[:, 1] + A0[:, 1] * A1[:, 0]) * db
                            + 2 * A1[:, 0] * A1[:, 1] * dc,
                            2 * A0[:, 0] * A0[:, 2] * da + (A0[:, 0] * A1[:, 2] + A0[:, 2] * A1[:, 0]) * db
                            + 2 * A1[:, 0] * A1[:, 2] * dc,
                            A0[:, 1] ** 2 * da + A0[:, 1] * A1[:, 1] * db + A1[:, 1] ** 2 * dc,
                            2 * A0[:, 2] * A0[:, 1] * da + (A0[:, 1] * A1[:, 2] + A0[:, 2] * A1[:, 1]) * db
                            + 2 * A1[:, 1] * A1[:, 2] * dc,
                            A0[:, 2] ** 2 * da + A0[:, 2] * A1[:, 2] * db + A1[:, 2] ** 2 * dc], 1)
        dT0 = 2 * (TV0 * da[:, None] + TW0 * da_v[:, None]) + TV1 * db[:, None] + TW1 * db_v[:, None]
        dT1 = 2 * (TV1 * dc[:, None] + TW1 * dc_v[:, None]) + TV0 * db[:, None] + TW0 * db_v[:, None]
        dJ00 = sum(vma[4 * k] * dT0[:, k] for k in range(3))
        dJ02 = sum(vma[4 * k + 2] * dT0[:, k] for k in range(3))
        dJ11 = sum(vma[4 * k + 1] * dT1[:, k] for k in range(3))
        dJ12 = sum(vma[4 * k + 2] * dT1[:, k] for k in range(3))
        dtx = xmul * fx * itz ** 2 * dJ02
        dty = ymul * fy * itz ** 2 * dJ12
        dtz = (fx * itz ** 2 * dJ00 + fy * itz ** 2 * dJ11 + 2 * fx * txc.abs() * itz ** 3 * dJ02
               + 2 * fy * tyc.abs() * itz ** 3 * dJ12)
        mean = torch.stack([vma[4 * k] * dtx + vma[4 * k + 1] * dty + vma[4 * k + 2] * dtz for k in range(3)], 1)
        # the screen mean and the depth
        hw = row(pm16, 3)
        mw = 1.0 / (hw + 1e-7).abs()
        cw = row_abs(pm16, 3) / hw.abs()
        mul1, mul2 = row_abs(pm16, 0) * mw * mw, row_abs(pm16, 1) * mw * mw
        d2x, d2y, dz = g[0][:, 0].abs(), g[0][:, 1].abs(), g[3].reshape(-1).abs()
        mean += torch.stack([cw * ((pma[4 * k] * mw + pma[4 * k + 3] * mul1) * d2x
                                   + (pma[4 * k + 1] * mw + pma[4 * k + 3] * mul2) * d2y) + dz * vma[4 * k + 2]
                             for k in range(3)], 1)
        if colors is None:
            dvec = p - cp
            ln = dvec.norm(dim=1)
            dR = g[2].abs() * keep.double()
            with torch.enable_grad():
                da_ = (dvec.abs() / ln[:, None]).requires_grad_()
                basis = sh_basis_abs(deg, da_)
                nb = basis.shape[1]
                e = (basis[:, :, None] * sh.detach()[:, :nb].abs() * dR[:, None, :]).sum()
                ddm = torch.autograd.grad(e, da_)[0] if deg > 0 else torch.zeros(n, 3, dtype=torch.float64)
            dsh = torch.zeros_like(sh.detach())
            dsh[:, :nb] = basis.detach()[:, :, None] * dR[:, None, :]
            full("mag_sh", dsh)
            v = dvec.abs()
            s2 = ln * ln
            mean += torch.stack([((s2 + v[:, k] ** 2) * ddm[:, k] + sum(v[:, j] * v[:, k] * ddm[:, j]
                                                                        for j in range(3) if j != k)) / ln ** 3
                                 for k in range(3)], 1)
        full("mag_means3D", mean)
        if cov3D is None:
            Mm = sa[:, None, :] * Ra  # M[c][r] = s[r] R[c][r]
            h = 0.5
            Sm = torch.stack([torch.stack([dcov[:, 0], h * dcov[:, 1], h * dcov[:, 2]], 1),
                              torch.stack([h * dcov[:, 1], dcov[:, 3], h * dcov[:, 4]], 1),
                              torch.stack([h * dcov[:, 2], h * dcov[:, 4], dcov[:, 5]], 1)], 1)
            dM = 2 * torch.einsum("nkr,nck->ncr", Mm, Sm)  # dM[c][r] = 2 sum_k M[k][r] S[c][k]
            full("mag_scales", torch.einsum("nck,nck->nk", Ra, dM))  # sum_c R[c][k] dM^T[k][c], dM^T[k][c] = dM[c][k]
            dMt = dM.transpose(1, 2) * sa[:, :, None]  # dMt[k][r] = dM[r][k] s[k]
            t = lambda i, j: dMt[:, i, j]  # noqa: E731
            full("mag_rotations", torch.stack([
                2 * qz * (t(0, 1) + t(1, 0)) + 2 * qy * (t(2, 0) + t(0, 2)) + 2 * qx * (t(1, 2) + t(2, 1)),
                2 * qy * (t(1, 0) + t(0, 1)) + 2 * qz * (t(2, 0) + t(0, 2)) + 2 * qr * (t(1, 2) + t(2, 1))
                + 4 * qx * (t(2, 2) + t(1, 1)),
                2 * qx * (t(1, 0) + t(0, 1)) + 2 * qr * (t(2, 0) + t(0, 2)) + 2 * qz * (t(1, 2) + t(2, 1))
                + 4 * qy * (t(2, 2) + t(0, 0)),
                2 * qr * (t(0, 1) + t(1, 0)) + 2 * qx * (t(2, 0) + t(0, 2)) + 2 * qy * (t(1, 2) + t(2, 1))
                + 4 * qz * (t(1, 1) + t(0, 0))], 1))
        full("mag_cov3D", dcov)
    return out
