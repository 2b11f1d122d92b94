"""Yardsticks of AbsGS's densification statistic (Ye et al., ACM MM 2024) for tests/test_absgrad.py.

  abs_mean2d_model   the composite's loss of blend_weights.composite_model, built with one leaf per blended (Gaussian,
                     pixel) pair for the 2-D mean, so that torch autograd gives each pixel's term t_ip of dL/dmean2D_i;
                     their absolute values summed per Gaussian are the statistic dL_dmean2D_abs in float64.
  absgs_masks        AbsGS's clone / split rule on the statistics, as the paper describes it:
                       g = grad_accum / denom, ga = grad_accum_abs / denom (NaN -> 0), smax = max exp(scaling)
                       clone  g  >= max_grad && smax <= dense_scale   (the 3DGS rule, unchanged)
                       split  ga >= abs_grad && smax >  dense_scale   (AbsGS's split on the absolute statistic)
  densify_and_prune  ref_densify.densify_and_prune with that split rule: the PyTorch restatement that
                     GaussianState.densify_and_prune(abs_grad=...) must equal bitwise.
"""
import torch

import blend_weights as bw
from ref_densify import _append, _select, build_rotation


def abs_mean2d_model(pairs, w, rec, P, dfn, bg_dot=None, signed=False):
    """[P, 2] float64: per Gaussian, sum over its blended pairs of |t_x| and |t_y|, t the pair's term of dL/dmean2D in
    the composite's units (0.5 W, 0.5 H), for composite_model's loss with the same dfn and bg_dot.  signed: also the
    pairs' own t [n, 2] and their Gaussians [n], in the order of the blended pairs."""
    W, H, HW = pairs.W, pairs.H, pairs.HW
    sel = pairs.widx[w > 0]
    pix, gid = pairs.pix[sel], pairs.gid[sel]
    d, _ = dfn(gid, pix)
    _, counts = torch.unique_consecutive(pix, return_counts=True)
    first = torch.repeat_interleave(torch.cumsum(counts, 0) - counts, counts)
    rec = rec.to(pix.device).double()
    mean = rec[gid, 0:2].clone().requires_grad_()  # one leaf per pair
    dx = mean[:, 0] - (pix % W).double()
    dy = mean[:, 1] - (pix // W).double()
    a, b, c = rec[gid, 4], rec[gid, 5], rec[gid, 6]
    G = torch.exp(-0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy)
    av = rec[gid, 7] * G
    alpha = av - (av - bw.ALPHA_MAX).clamp(min=0.0).detach()
    logf = torch.log1p(-alpha)
    T = torch.exp(bw._seg_excl_cumsum(logf, first))
    L = (alpha * T * d).sum()
    if bg_dot is not None:
        bgd = bg_dot[0].to(pix.device).double().reshape(-1)
        T_fin = torch.exp(torch.zeros(HW, dtype=torch.float64, device=pix.device).index_add(0, pix, logf))
        L = L + (T_fin * bgd).sum()
    (gm,) = torch.autograd.grad(L, [mean])
    t = torch.stack([gm[:, 0] * 0.5 * W, gm[:, 1] * 0.5 * H], 1)
    out = torch.zeros(P, 2, dtype=torch.float64, device=pix.device).index_add_(0, gid, t.abs())
    return (out, t, gid) if signed else out


def planes_dfn(rec, Gc, Gd, gI):
    """dfn of the backward with the inverse-depth plane: d = c_g . Gc_p + z_g Gd_p + gI_p / z_g (I_p = sum_i w_i / z_i
    is one more blended value per pair), and its products' magnitudes."""
    c, z = rec[:, 8:11].double(), rec[:, 11].double()
    Gc, Gd, gI = Gc.double(), Gd.double().reshape(-1), gI.double().reshape(-1)

    def dfn(gid, pix):
        cg, t, i = c[gid] * Gc[pix], z[gid] * Gd[pix], gI[pix] / z[gid]
        return cg.sum(1) + t + i, cg.abs().sum(1) + t.abs() + i.abs()

    return dfn


def feature_dfn(feats, Gf):
    """dfn of the feature walk: d = f_g . Gf_p (feats [P, C], Gf [C, HW])."""
    def dfn(gid, pix):
        if gid.numel() * Gf.shape[0] <= bw.PAIR_CHUNK:
            t = feats.double()[gid] * Gf.double()[:, pix].t()
            return t.sum(1), t.abs().sum(1)
        return bw.pair_dots(feats, Gf.t(), gid, pix)  # bench-sized windows: over chunks of pairs

    return dfn


def absgs_masks(grad_accum, grad_accum_abs, denom, scaling, max_grad, abs_grad, dense_scale):
    """(clone, split) bool masks of AbsGS's rule (module docstring); scaling is exp(raw scaling) [P, 3]."""
    grads = grad_accum / denom
    grads[grads.isnan()] = 0.0
    grads_abs = grad_accum_abs / denom
    grads_abs[grads_abs.isnan()] = 0.0
    smax = scaling.max(dim=1).values
    return (grads >= max_grad) & (smax <= dense_scale), (grads_abs >= abs_grad) & (smax > dense_scale)


def densify_and_prune(st, max_grad, abs_grad, min_opacity, extent, max_screen_size, grad_accum, grad_accum_abs, denom,
                      generator=None, info=None):
    """ref_densify.densify_and_prune with AbsGS's split rule: split when grad_accum_abs / denom >= abs_grad (the clones
    appended first take part with zero statistic, as in the reference).  `info` as there."""
    scaling = torch.exp(st.raw["scaling"])
    clone, _ = absgs_masks(grad_accum, grad_accum_abs, denom, scaling, max_grad, abs_grad, st.percent_dense * extent)
    n0 = st.P
    _append(st, {k: v[clone] for k, v in st.raw.items()})
    grads_abs = grad_accum_abs / denom
    grads_abs[grads_abs.isnan()] = 0.0
    padded = torch.zeros(st.P, device=grads_abs.device)
    padded[:n0] = grads_abs
    scaling = torch.exp(st.raw["scaling"])
    sel = (padded >= abs_grad) & (scaling.max(dim=1).values > st.percent_dense * extent)
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
    keep = torch.ones(st.P, dtype=torch.bool, device=grads_abs.device)
    keep[:n_before_split] = ~sel
    opacity = torch.sigmoid(st.raw["opacity"]).squeeze(-1)
    prune = opacity < min_opacity
    if max_screen_size:
        mr = torch.zeros(st.P, device=grads_abs.device)
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
