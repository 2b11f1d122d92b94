"""Parameter state, activation prologue, fused optimizer and densification on the rasterizer's own buffers
(SURVEY.md section 8 f2 / f3; reference scene/gaussian_model.py).

`GaussianState` keeps the RAW parameters the reference's GaussianModel optimises (`_xyz, _features_dc, _features_rest,
_opacity, _scaling, _rotation, _semantic_feature`, :47-58) as plain CUDA tensors, and

  from_point_cloud()    create_from_pcd (:133-160): a fresh state from a point cloud, initial scales from the native
                        exact 3-NN distance (f3dgs_knn_mean_dist, the reference's simple_knn distCUDA2);
  activate()            raw -> the activated tensors the rasterizer consumes (:98-121) in ONE kernel (f3dgs_activate), once
                        per optimizer step instead of four elementwise kernels + a concat per view;
  batch()               a ViewBatch (parallel.py) over the activated tensors: forward / in-kernel accumulated backward of
                        the step's views, densification statistics (:436-438) folded into the same flat buffer, one
                        all-reduce;
  step(lrs)             Adam (:163-190: lr per group, eps 1e-15) fused with the activations' Jacobians
                        (f3dgs_adam_step): consumes the all-reduced gradients w.r.t. the ACTIVATED tensors straight from the
                        flat buffer and updates the raw parameters in place -- no autograd graph anywhere;
  densify_and_prune()   clone / split / prune (:350-434) with the optimizer state carried along, as in the reference
                        (host-side tensor logic: the reference's is Python too).
"""
import math
from typing import Dict, Optional

import numpy as np
import torch

from .parallel import ViewBatch

KIND = dict(xyz=0, semantic_feature=0, opacity=1, scaling=2, rotation=3, f_dc=4, f_rest=5)  # F3DGS_PARAM_*
GRAD_OF = dict(xyz="means3D", f_dc="shs", f_rest="shs", opacity="opacities", scaling="scales", rotation="rotations",
               semantic_feature="semantic_feature")


def inverse_sigmoid(x):
    return torch.log(x / (1 - x))


def build_rotation(r):
    """utils/general_utils.py:78-100: rotation matrices of (normalised) quaternions (w, x, y, z)."""
    q = r / r.norm(dim=1, keepdim=True)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.zeros((q.shape[0], 3, 3), device=r.device)
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 0, 1] = 2 * (x * y - w * z); R[:, 0, 2] = 2 * (x * z + w * y)
    R[:, 1, 0] = 2 * (x * y + w * z); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 1, 2] = 2 * (y * z - w * x)
    R[:, 2, 0] = 2 * (x * z - w * y); R[:, 2, 1] = 2 * (y * z + w * x); R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


class GaussianState:
    NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "semantic_feature")

    def __init__(self, xyz, features_dc, features_rest, opacity, scaling, rotation, semantic_feature,
                 betas=(0.9, 0.999), eps=1e-15, percent_dense=0.01):
        self.raw: Dict[str, torch.Tensor] = dict(
            xyz=xyz.contiguous(), f_dc=features_dc.contiguous(), f_rest=features_rest.contiguous(),
            opacity=opacity.contiguous(), scaling=scaling.contiguous(), rotation=rotation.contiguous(),
            semantic_feature=semantic_feature.contiguous())
        for k, v in self.raw.items():
            if not v.is_cuda or v.dtype != torch.float32:
                raise RuntimeError(f"{k} must be a float32 CUDA tensor (this build has no CPU path)")
        self.betas, self.eps, self.percent_dense = betas, eps, percent_dense
        self._reset_derived()

    @classmethod
    def from_point_cloud(cls, points, colors, semantic_feature_size: int, speedup: bool = False, max_sh_degree: int = 3,
                         device="cuda", **kwargs):
        """scene/gaussian_model.py:133-160 (create_from_pcd): a fresh state from a point cloud.

        points [P,3] and colors [P,3] (RGB in [0,1]) are arrays or tensors of any float dtype; both are converted to
        float32 first, as the reference does.  The initial scale of each Gaussian is log(sqrt(mean squared distance to its
        three nearest neighbours)), isotropic, from the native distCUDA2 (csrc/knn.cu).  Every other field is computed
        with the reference's own tensor operations, so it is bitwise what create_from_pcd builds.  With `speedup` the
        feature width is int(semantic_feature_size / 4), as there.  Raises ValueError on mismatched shapes or a
        non-finite coordinate."""
        from . import _C

        def as_f32(a):
            t = a if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a))
            return t.float().to(device)

        xyz, rgb = as_f32(points), as_f32(colors)
        if xyz.dim() != 2 or xyz.shape[1] != 3 or rgb.shape != xyz.shape:
            raise ValueError(f"points and colors must both be [P,3], got {tuple(xyz.shape)} and {tuple(rgb.shape)}")
        if not bool(torch.isfinite(xyz).all()):
            raise ValueError("points contain a non-finite coordinate")
        P = xyz.shape[0]
        fused_color = (rgb - 0.5) / 0.28209479177387814  # utils/sh_utils.py RGB2SH
        features = torch.zeros((P, 3, (max_sh_degree + 1) ** 2), dtype=torch.float32, device=device)
        features[:, :3, 0] = fused_color
        if speedup:
            semantic_feature_size = int(semantic_feature_size / 4)
        semantic_feature = torch.zeros(P, semantic_feature_size, 1, dtype=torch.float32, device=device)
        dist2 = torch.clamp_min(_C.knn_mean_dist(xyz), 0.0000001)
        scales = torch.log(torch.sqrt(dist2))[..., None].repeat(1, 3)
        rots = torch.zeros((P, 4), device=device)
        rots[:, 0] = 1
        opacities = inverse_sigmoid(0.1 * torch.ones((P, 1), dtype=torch.float, device=device))
        return cls(xyz, features[:, :, 0:1].transpose(1, 2).contiguous(), features[:, :, 1:].transpose(1, 2).contiguous(),
                   opacities, scales, rots, semantic_feature.transpose(1, 2).contiguous(), **kwargs)

    # ---------------------------------------------------------------------------------------------- buffers
    @property
    def P(self):
        return self.raw["xyz"].shape[0]

    @property
    def M(self):
        return 1 + self.raw["f_rest"].shape[1]

    def _reset_derived(self):
        dev, P = self.raw["xyz"].device, self.P
        self.exp_avg = {k: torch.zeros_like(v) for k, v in self.raw.items()}
        self.exp_avg_sq = {k: torch.zeros_like(v) for k, v in self.raw.items()}
        self.steps = {k: 0 for k in self.raw}
        self.max_radii2D = torch.zeros(P, device=dev)
        self.act = dict(means3D=self.raw["xyz"], opacities=torch.empty(P, 1, device=dev), scales=torch.empty(P, 3, device=dev),
                        rotations=torch.empty(P, 4, device=dev), shs=torch.empty(P, self.M, 3, device=dev),
                        semantic_feature=self.raw["semantic_feature"])
        self._batch: Optional[ViewBatch] = None

    def activate(self):
        from . import _C

        a, r = self.act, self.raw
        _C.activate(r["opacity"], r["scaling"], r["rotation"], r["f_dc"], r["f_rest"], a["opacities"], a["scales"],
                    a["rotations"], a["shs"])
        return a

    def batch(self) -> ViewBatch:
        if self._batch is None:
            self._batch = ViewBatch(self.act, densify_stats=True)
        return self._batch

    # ---------------------------------------------------------------------------------------------- optimizer
    def step(self, lrs: Dict[str, float], grads: Optional[Dict[str, torch.Tensor]] = None):
        """One Adam step of every group.  `grads`: gradients w.r.t. the activated tensors (default: the ViewBatch's)."""
        from . import _C

        g = grads if grads is not None else self.batch().grads
        for name in self.NAMES:
            p = self.raw[name]
            if p.numel() == 0:
                continue
            self.steps[name] += 1
            _C.adam_step(KIND[name], p, g[GRAD_OF[name]], self.exp_avg[name], self.exp_avg_sq[name], self.M, lrs[name],
                         self.betas[0], self.betas[1], self.eps, self.steps[name])

    # ---------------------------------------------------------------------------------------------- densification
    def update_max_radii(self, radii):
        vis = radii > 0
        self.max_radii2D[vis] = torch.max(self.max_radii2D[vis], radii[vis].float())  # train.py:131

    def _select(self, mask):
        for d in (self.raw, self.exp_avg, self.exp_avg_sq):
            for k in d:
                d[k] = d[k][mask].contiguous()

    def _append(self, new: Dict[str, torch.Tensor]):
        for k in self.raw:
            self.raw[k] = torch.cat((self.raw[k], new[k]), dim=0).contiguous()
            self.exp_avg[k] = torch.cat((self.exp_avg[k], torch.zeros_like(new[k])), dim=0).contiguous()
            self.exp_avg_sq[k] = torch.cat((self.exp_avg_sq[k], torch.zeros_like(new[k])), dim=0).contiguous()

    def densify_and_prune(self, max_grad, min_opacity, extent, max_screen_size, grad_accum=None, denom=None, generator=None):
        """scene/gaussian_model.py:420-434 (clone :407-418, split :381-405, prune :316-330)."""
        vb = self.batch()
        grad_accum = vb.grad_accum if grad_accum is None else grad_accum
        denom = vb.denom if denom is None else denom
        grads = grad_accum / denom
        grads[grads.isnan()] = 0.0
        max_radii = self.max_radii2D
        scaling = torch.exp(self.raw["scaling"])
        # ---- clone small Gaussians with a large screen-space gradient
        sel = (grads >= max_grad) & (scaling.max(dim=1).values <= self.percent_dense * extent)
        n0 = self.P
        self._append({k: v[sel] for k, v in self.raw.items()})
        # ---- split large ones (the clones appended above take part with zero gradient, as in the reference :384-386)
        padded = torch.zeros(self.P, device=grads.device)
        padded[:n0] = grads
        scaling = torch.exp(self.raw["scaling"])
        sel = (padded >= max_grad) & (scaling.max(dim=1).values > self.percent_dense * extent)
        N = 2
        stds = scaling[sel].repeat(N, 1)
        samples = torch.normal(mean=torch.zeros_like(stds), std=stds, generator=generator)
        rots = build_rotation(self.raw["rotation"][sel]).repeat(N, 1, 1)
        new = {k: v[sel].repeat(N, *([1] * (v.dim() - 1))) for k, v in self.raw.items()}
        new["xyz"] = torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + self.raw["xyz"][sel].repeat(N, 1)
        new["scaling"] = torch.log(scaling[sel].repeat(N, 1) / (0.8 * N))
        n_before_split = self.P
        self._append(new)
        keep = torch.ones(self.P, dtype=torch.bool, device=grads.device)
        keep[:n_before_split] = ~sel
        # ---- prune: transparent, or too large on screen / in the world
        opacity = torch.sigmoid(self.raw["opacity"]).squeeze(-1)
        prune = opacity < min_opacity
        if max_screen_size:
            mr = torch.zeros(self.P, device=grads.device)  # densification_postfix resets max_radii2D (:376)
            big_ws = torch.exp(self.raw["scaling"]).max(dim=1).values > 0.1 * extent
            prune = prune | (mr > max_screen_size) | big_ws
        del max_radii
        self._select(keep & ~prune)
        steps = dict(self.steps)
        m, v = self.exp_avg, self.exp_avg_sq
        self._reset_derived()
        self.exp_avg, self.exp_avg_sq, self.steps = m, v, steps
        return self.P

    def reset_opacity(self):
        """scene/gaussian_model.py:231-234: clamp opacity to <= 0.01 and clear its optimizer state."""
        o = torch.sigmoid(self.raw["opacity"])
        self.raw["opacity"] = inverse_sigmoid(torch.min(o, torch.ones_like(o) * 0.01)).contiguous()
        self.exp_avg["opacity"].zero_()
        self.exp_avg_sq["opacity"].zero_()


def expon_lr(step, lr_init, lr_final, lr_delay_steps=0, lr_delay_mult=1.0, max_steps=1000000):
    """utils/general_utils.py:40-76 (get_expon_lr_func): the position learning-rate schedule."""
    if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
        return 0.0
    if lr_delay_steps > 0:
        delay_rate = lr_delay_mult + (1 - lr_delay_mult) * math.sin(0.5 * math.pi * min(max(step / lr_delay_steps, 0), 1))
    else:
        delay_rate = 1.0
    t = min(max(step / max_steps, 0), 1)
    return delay_rate * math.exp(math.log(lr_init) * (1 - t) + math.log(lr_final) * t)
