"""PyTorch restatement of 3DGS-MCMC's densification (Kheradmand et al., "3D Gaussian Splatting as Markov Chain Monte
Carlo", NeurIPS 2024): the official code's relocate_gs, add_new_gs (with _sample_alives, _update_params and
replace_tensors_to_optimizer), the position noise of its train.py and its two regularisers, on a trainer.GaussianState.
It is the yardstick of tests/test_mcmc.py and tools/time_mcmc.py.

One part is not the official code: its compute_relocation CUDA kernel (float32, powf) is replaced by the float64 model
`relocation64`, whose result is rounded to float once, raw fields included.  That is the rule csrc/mcmc.cu implements."""
import decimal
import math

import torch

N_MAX = 51  # gsplat's n_max: a source and its copies count as at most 51 Gaussians
F32_EPS = torch.finfo(torch.float32).eps


# ---------------------------------------------------------------------------------------------------- float64 models
def relocation64(o, N):
    """o' = 1 - (1 - o)^(1/N) and o / D(o', N) in float64, D(x, N) = sum_{j=1..N} C(N,j) (-1)^(j-1) x^j / sqrt(j).
    o: float64 tensor, N: int64 tensor of the same shape (>= 1, not clamped here).  The sum runs j = 1..N with the
    binomials by the recurrence C(N,j) = C(N,j-1) (N-j+1) / j, as csrc/mcmc.cu sums it."""
    op = -torch.expm1(torch.log1p(-o) / N)
    Nd = N.double()
    c, p, D = torch.ones_like(o), torch.ones_like(o), torch.zeros_like(o)
    for j in range(1, int(N.max()) + 1 if N.numel() else 1):
        live = N >= j
        c = torch.where(live, c * (Nd - j + 1) / j, c)
        p = torch.where(live, p * op, p)
        t = c * p / math.sqrt(j)
        D = torch.where(live, D + t if j & 1 else D - t, D)
    return op, o / D


def D_double_loop(x, N):
    """The official kernel's form of D, sum_{i=1..N} sum_{k=0..i-1} C(i-1,k) (-1)^k x^(k+1) / sqrt(k+1), evaluated
    with 60 significant digits (x a Python float, N an int): the check that the closed form above is the same sum."""
    with decimal.localcontext() as ctx:
        ctx.prec = 60
        X = decimal.Decimal(x)
        roots = [decimal.Decimal(k + 1).sqrt() for k in range(N)]
        D = sum(math.comb(i - 1, k) * (-1) ** k * X ** (k + 1) / roots[k] for i in range(1, N + 1) for k in range(i))
        return float(D)


def raw_opacity64(op, min_opacity):
    """logit of o' clamped to [min_opacity, 1 - FLT_EPSILON] (both as float32), rounded to float32 once"""
    x = op.clamp(min=float(torch.tensor(min_opacity, dtype=torch.float32)), max=1.0 - F32_EPS)
    return torch.log(x / (1.0 - x)).float()


def compute_relocation(opacity_old, scale_old, N, min_opacity):
    """The official _update_params' compute_relocation + clamp + inverse activations, as the float64 model: float32
    activated opacity [n] and scales [n,3], N [n] (clamped to 51 here) -> raw opacity [n,1] and raw scaling [n,3]."""
    op, ratio = relocation64(opacity_old.double(), N.clamp(max=N_MAX))
    raw_s = torch.log(scale_old.double() * ratio[:, None]).float()
    return raw_opacity64(op, min_opacity)[:, None], raw_s


def noise_step64(st, eps, scale):
    """The position step of inject_noise in float64 from the state's float32 activations: [P,3]."""
    r = st.raw
    o = torch.sigmoid(r["opacity"]).double().squeeze(-1)
    g = 1.0 / (1.0 + torch.exp(-100.0 * ((1.0 - o) - 0.995)))
    q = r["rotation"].double()
    q = q / torch.sqrt((q * q).sum(1, keepdim=True))
    R = build_rotation(q)
    s2 = torch.exp(r["scaling"]).double() ** 2
    v = eps.double() * (g * float(scale))[:, None]
    t = s2 * torch.einsum("pkc,pk->pc", R, v)  # diag(s^2) R^T v
    return torch.einsum("pck,pk->pc", R, t)


# ---------------------------------------------------------------------------------------------------- the official code
def build_rotation(q):
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.zeros((q.size(0), 3, 3), device=q.device, dtype=q.dtype)
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 0, 1] = 2 * (x * y - w * z); R[:, 0, 2] = 2 * (x * z + w * y)
    R[:, 1, 0] = 2 * (x * y + w * z); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 1, 2] = 2 * (y * z - w * x)
    R[:, 2, 0] = 2 * (x * z - w * y); R[:, 2, 1] = 2 * (y * z + w * x); R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def _sample_alives(probs, num, generator, alive_indices=None):
    probs = probs / (probs.sum() + F32_EPS)
    sampled_idxs = torch.multinomial(probs, num, replacement=True, generator=generator)
    if alive_indices is not None:
        sampled_idxs = alive_indices[sampled_idxs]
    ratio = torch.bincount(sampled_idxs).unsqueeze(-1)
    return sampled_idxs, ratio


def _update_params(st, idxs, ratio, min_opacity):
    raw_o, raw_s = compute_relocation(torch.sigmoid(st.raw["opacity"])[idxs, 0], torch.exp(st.raw["scaling"])[idxs],
                                      ratio[idxs, 0] + 1, min_opacity)
    new = {k: v[idxs] for k, v in st.raw.items()}
    new["opacity"], new["scaling"] = raw_o, raw_s
    return new


def _replace_tensors_to_optimizer(st, inds):
    for k in st.raw:
        st.exp_avg[k][inds] = 0
        st.exp_avg_sq[k][inds] = 0


def relocate_gs(st, min_opacity=0.005, generator=None, info=None):
    """-> n_relocated.  info (a dict) receives dead_indices and reinit_idx (the draws' sources)."""
    dead_mask = (torch.sigmoid(st.raw["opacity"]) <= min_opacity).squeeze(-1)
    if dead_mask.sum() == 0:
        return 0
    alive_mask = ~dead_mask
    dead_indices = dead_mask.nonzero(as_tuple=True)[0]
    alive_indices = alive_mask.nonzero(as_tuple=True)[0]
    if alive_indices.shape[0] <= 0:
        return 0
    probs = torch.sigmoid(st.raw["opacity"])[alive_indices, 0]
    reinit_idx, ratio = _sample_alives(probs, dead_indices.shape[0], generator, alive_indices)
    new = _update_params(st, reinit_idx, ratio, min_opacity)
    for k in st.raw:
        st.raw[k][dead_indices] = new[k]
    st.raw["opacity"][reinit_idx] = st.raw["opacity"][dead_indices]
    st.raw["scaling"][reinit_idx] = st.raw["scaling"][dead_indices]
    _replace_tensors_to_optimizer(st, reinit_idx)
    if info is not None:
        info["dead_indices"], info["reinit_idx"] = dead_indices, reinit_idx
    return int(dead_indices.shape[0])


def add_new_gs(st, cap_max, min_opacity=0.005, generator=None, info=None):
    """-> n_added.  info (a dict) receives add_idx (the draws' sources)."""
    current_num_points = st.P
    target_num = min(cap_max, int(1.05 * current_num_points))
    num_gs = max(0, target_num - current_num_points)
    if num_gs <= 0:
        return 0
    probs = torch.sigmoid(st.raw["opacity"]).squeeze(-1)
    add_idx, ratio = _sample_alives(probs, num_gs, generator)
    new = _update_params(st, add_idx, ratio, min_opacity)
    st.raw["opacity"][add_idx] = new["opacity"]
    st.raw["scaling"][add_idx] = new["scaling"]
    for k in st.raw:  # densification_postfix: new rows start with zero moments
        st.raw[k] = torch.cat((st.raw[k], new[k]), dim=0).contiguous()
        st.exp_avg[k] = torch.cat((st.exp_avg[k], torch.zeros_like(new[k])), dim=0).contiguous()
        st.exp_avg_sq[k] = torch.cat((st.exp_avg_sq[k], torch.zeros_like(new[k])), dim=0).contiguous()
    _replace_tensors_to_optimizer(st, add_idx)
    st._reset_derived(keep_optimizer_state=True)
    if info is not None:
        info["add_idx"] = add_idx
    return num_gs


def relocate_and_add(st, cap_max, min_opacity=0.005, generator=None, info=None):
    """The official train.py's densification step: relocate_gs(dead_mask = opacity <= min_opacity), add_new_gs."""
    return (relocate_gs(st, min_opacity, generator, info), add_new_gs(st, cap_max, min_opacity, generator, info))


def inject_noise(st, xyz_lr, noise_lr=5e5, generator=None):
    """The official train.py's noise, in float32 tensor code (randn_like replaced by a draw from `generator`)."""
    r = st.raw
    s = torch.exp(r["scaling"])
    q = torch.nn.functional.normalize(r["rotation"])
    L = build_rotation(q) * s[:, None, :]  # build_scaling_rotation: R @ diag(s)
    actual_covariance = L @ L.transpose(1, 2)

    def op_sigmoid(x, k=100, x0=0.995):
        return 1 / (1 + torch.exp(-k * (x - x0)))

    eps = torch.randn((st.P, 3), generator=generator, device=r["xyz"].device)
    noise = eps * op_sigmoid(1 - torch.sigmoid(r["opacity"])) * noise_lr * xyz_lr
    noise = torch.bmm(actual_covariance, noise.unsqueeze(-1)).squeeze(-1)
    r["xyz"].add_(noise)
    return eps


def regularizer_grads(st, opacity_reg, scale_reg):
    """d/d(activated) of opacity_reg * |opacity|.mean() + scale_reg * |scales|.mean(), by autograd."""
    o = torch.sigmoid(st.raw["opacity"]).requires_grad_()
    s = torch.exp(st.raw["scaling"]).requires_grad_()
    (opacity_reg * torch.abs(o).mean() + scale_reg * torch.abs(s).mean()).backward()
    return o.grad, s.grad
