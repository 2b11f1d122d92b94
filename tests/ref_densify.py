"""PyTorch restatement of the reference's adaptive density control (scene/gaussian_model.py:350-434 densify_and_prune,
:231-234 reset_opacity, train.py:131 max_radii2D), on a trainer.GaussianState.  This is the tensor code the trainer
ran before its densification moved to csrc/densify.cu; it is the yardstick of tests/test_densify.py and of
tools/time_densify.py.  `build_rotation` is written as the reference writes it (utils/general_utils.py:78-100)."""
from typing import Dict

import torch


def inverse_sigmoid(x):
    return torch.log(x / (1 - x))


def build_rotation(r):
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    R = torch.zeros((q.size(0), 3, 3), device=r.device)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 0, 1] = 2 * (x * y - w * z); R[:, 0, 2] = 2 * (x * z + w * y)
    R[:, 1, 0] = 2 * (x * y + w * z); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 1, 2] = 2 * (y * z - w * x)
    R[:, 2, 0] = 2 * (x * z - w * y); R[:, 2, 1] = 2 * (y * z + w * x); R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def _select(st, mask):
    for d in (st.raw, st.exp_avg, st.exp_avg_sq):
        for k in d:
            d[k] = d[k][mask].contiguous()


def _append(st, new: Dict[str, torch.Tensor]):
    for k in st.raw:
        st.raw[k] = torch.cat((st.raw[k], new[k]), dim=0).contiguous()
        st.exp_avg[k] = torch.cat((st.exp_avg[k], torch.zeros_like(new[k])), dim=0).contiguous()
        st.exp_avg_sq[k] = torch.cat((st.exp_avg_sq[k], torch.zeros_like(new[k])), dim=0).contiguous()


def densify_and_prune(st, max_grad, min_opacity, extent, max_screen_size, grad_accum=None, denom=None, generator=None,
                      info=None):
    """GaussianState.densify_and_prune as tensor code.  `info` (a dict) receives, for the tolerance of the split
    children's xyz: the split parents' xyz `parent_xyz` [2 Ns, 3] and the offsets R (z * std) `rsz` [2 Ns, 3] in virtual
    child order, and `child_keep` [2 Ns] (which children survive the prune)."""
    vb = st.batch()
    grad_accum = vb.grad_accum if grad_accum is None else grad_accum
    denom = vb.denom if denom is None else denom
    grads = grad_accum / denom
    grads[grads.isnan()] = 0.0
    scaling = torch.exp(st.raw["scaling"])
    # ---- clone small Gaussians with a large screen-space gradient
    sel = (grads >= max_grad) & (scaling.max(dim=1).values <= st.percent_dense * extent)
    n0 = st.P
    _append(st, {k: v[sel] for k, v in st.raw.items()})
    # ---- split large ones (the clones appended above take part with zero gradient, as in the reference :384-386)
    padded = torch.zeros(st.P, device=grads.device)
    padded[:n0] = grads
    scaling = torch.exp(st.raw["scaling"])
    sel = (padded >= max_grad) & (scaling.max(dim=1).values > st.percent_dense * extent)
    N = 2
    stds = scaling[sel].repeat(N, 1)
    samples = torch.normal(mean=torch.zeros_like(stds), std=stds, generator=generator)
    rots = build_rotation(st.raw["rotation"][sel]).repeat(N, 1, 1)
    new = {k: v[sel].repeat(N, *([1] * (v.dim() - 1))) for k, v in st.raw.items()}
    new["xyz"] = torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + st.raw["xyz"][sel].repeat(N, 1)
    new["scaling"] = torch.log(scaling[sel].repeat(N, 1) / (0.8 * N))
    if info is not None:
        info["parent_xyz"] = st.raw["xyz"][sel].repeat(N, 1)
        info["rsz"] = new["xyz"] - info["parent_xyz"]
    n_before_split = st.P
    _append(st, new)
    keep = torch.ones(st.P, dtype=torch.bool, device=grads.device)
    keep[:n_before_split] = ~sel
    # ---- prune: transparent, or too large on screen / in the world
    opacity = torch.sigmoid(st.raw["opacity"]).squeeze(-1)
    prune = opacity < min_opacity
    if max_screen_size:
        mr = torch.zeros(st.P, device=grads.device)  # densification_postfix resets max_radii2D (:376)
        big_ws = torch.exp(st.raw["scaling"]).max(dim=1).values > 0.1 * extent
        prune = prune | (mr > max_screen_size) | big_ws
    if info is not None:
        info["child_keep"] = (keep & ~prune)[n_before_split:]
    _select(st, keep & ~prune)
    steps = dict(st.steps)
    m, v = st.exp_avg, st.exp_avg_sq
    st._reset_derived()
    st.exp_avg, st.exp_avg_sq, st.steps = m, v, steps
    return st.P


def reset_opacity(st):
    o = torch.sigmoid(st.raw["opacity"])
    st.raw["opacity"] = inverse_sigmoid(torch.min(o, torch.ones_like(o) * 0.01)).contiguous()
    st.exp_avg["opacity"].zero_()
    st.exp_avg_sq["opacity"].zero_()


def update_max_radii(max_radii2D, radii):
    vis = radii > 0
    max_radii2D[vis] = torch.max(max_radii2D[vis], radii[vis].float())
    return max_radii2D
