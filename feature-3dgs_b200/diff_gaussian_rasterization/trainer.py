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
                        step(lrs, visible=vb.visible()) is the sparse Adam step on the Gaussians the step's views saw;
  densify_and_prune()   clone / split / prune (:350-434) with the optimizer state carried along, in two native calls
                        (f3dgs_densify_plan / f3dgs_densify_apply) with one host read in between;
  reset_opacity()       :231-234 in one kernel (f3dgs_reset_opacity).

Float16 feature fields: with feature_dtype=torch.float16 the rasterizer reads a float16 working copy
act["semantic_feature"] of the float32 master raw["semantic_feature"], so every view renders a float16 map and the feature
loss hands back a float16 gradient (feature_head `*_and_grad(..., grad_dtype=torch.float16)`).  The master, its Adam
moments and the accumulated gradient stay float32; the copy is made by one cast at construction and after
densify_and_prune, and step() refreshes it in the Adam pass itself (f3dgs_adam_step_f16out).
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


class GaussianState:
    NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "semantic_feature")

    def __init__(self, xyz, features_dc, features_rest, opacity, scaling, rotation, semantic_feature,
                 betas=(0.9, 0.999), eps=1e-15, percent_dense=0.01, feature_dtype=torch.float32):
        self.raw: Dict[str, torch.Tensor] = dict(
            xyz=xyz.contiguous(), f_dc=features_dc.contiguous(), f_rest=features_rest.contiguous(),
            opacity=opacity.contiguous(), scaling=scaling.contiguous(), rotation=rotation.contiguous(),
            semantic_feature=semantic_feature.contiguous())
        for k, v in self.raw.items():
            if not v.is_cuda or v.dtype != torch.float32:
                raise RuntimeError(f"{k} must be a float32 CUDA tensor (this build has no CPU path)")
        if feature_dtype not in (torch.float32, torch.float16):
            raise ValueError(f"feature_dtype must be torch.float32 or torch.float16, got {feature_dtype}")
        self.betas, self.eps, self.percent_dense = betas, eps, percent_dense
        self.feature_dtype = feature_dtype
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
        non-finite coordinate.  kwargs (feature_dtype among them) go to the constructor."""
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

    def _reset_derived(self, keep_optimizer_state=False):
        dev, P = self.raw["xyz"].device, self.P
        self.act = self._batch = None  # the old buffers are released before the new ones are allocated
        if not keep_optimizer_state:
            self.exp_avg = {k: torch.zeros_like(v) for k, v in self.raw.items()}
            self.exp_avg_sq = {k: torch.zeros_like(v) for k, v in self.raw.items()}
            self.steps = {k: 0 for k in self.raw}
        self.max_radii2D = torch.zeros(P, device=dev)
        sf = self.raw["semantic_feature"]
        self.act = dict(means3D=self.raw["xyz"], opacities=torch.empty(P, 1, device=dev), scales=torch.empty(P, 3, device=dev),
                        rotations=torch.empty(P, 4, device=dev), shs=torch.empty(P, self.M, 3, device=dev),
                        semantic_feature=sf if self.feature_dtype == torch.float32 else sf.to(self.feature_dtype))
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
    def step(self, lrs: Dict[str, float], grads: Optional[Dict[str, torch.Tensor]] = None,
             visible: Optional[torch.Tensor] = None):
        """One Adam step of every group.  `grads`: gradients w.r.t. the activated tensors (default: the ViewBatch's).

        visible: None for the dense step, or a bool [P] CUDA mask (ViewBatch.visible() after all_reduce()) for the sparse
        Adam step (f3dgs_adam_step_masked): only the marked Gaussians' raw parameters, moments and float16 feature copy
        change, bitwise as in the dense step; the others stay exactly as they are, so momentum no longer moves Gaussians
        that no view of the step saw.  Bias correction still uses each group's step count, which advances every step."""
        from . import _C

        g = grads if grads is not None else self.batch().grads
        for name in self.NAMES:
            p = self.raw[name]
            if p.numel() == 0:
                continue
            self.steps[name] += 1
            # a float16 working copy of the features is rewritten in the same pass
            half = name == "semantic_feature" and self.feature_dtype == torch.float16
            copy = self.act["semantic_feature"] if half else None
            _C.adam_step(KIND[name], p, g[GRAD_OF[name]], self.exp_avg[name], self.exp_avg_sq[name], self.M, lrs[name],
                         self.betas[0], self.betas[1], self.eps, self.steps[name], copy, visible)

    # ---------------------------------------------------------------------------------------------- densification
    def update_max_radii(self, radii):
        """train.py:131, without a host sync: max_radii2D = max(max_radii2D, radii) where radii > 0."""
        self.max_radii2D = torch.where(radii > 0, torch.maximum(self.max_radii2D, radii.float()), self.max_radii2D)

    def densify_and_prune(self, max_grad, min_opacity, extent, max_screen_size, grad_accum=None, denom=None, generator=None):
        """scene/gaussian_model.py:420-434 (clone :407-418, split :381-405, prune :316-330); returns the new P.

        With g = grad_accum / denom (0 where that is NaN) and smax the largest of exp(scaling), a Gaussian is cloned when
        g >= max_grad and smax <= percent_dense * extent, and split in two when g >= max_grad and smax is larger.  The
        new rows are the order-preserving compaction of [originals | clones | split copy 0 | split copy 1] without the
        split originals and without every row that is pruned: sigmoid(opacity) < min_opacity, or, when max_screen_size
        is truthy, max(exp(scaling)) > 0.1 * extent on the row's own scaling.  As in the reference, max_radii2D is reset
        before that test (densification_postfix), so its screen-size part never prunes anything.  The thresholds are
        rounded to float32 once, as torch compares a float32 tensor with a Python scalar.

        A split child copies its parent except scaling = log(exp(scaling) / 1.6) and xyz = R(rotation) (z * exp(scaling))
        + xyz, with z = torch.randn((2 Ns, 3), generator=generator) over all Ns split Gaussians (rows [0, Ns) copy 0).
        Kept rows keep their Adam moments, new rows start at zero; `steps` is unchanged.  Every output is bitwise what the
        reference's tensor code computes, except the split children's xyz, which agree within float rounding (the
        reference's torch.bmm has no defined summation order).

        Two native calls (csrc/densify.cu) and ONE host sync, the read of the four output counts that size the new
        tensors and the normal draw.  Deterministic: identical state, statistics and generator state give bitwise-
        identical output, so data-parallel replicas that densify from the same all-reduced statistics with the same seed
        stay identical."""
        from . import _C

        if grad_accum is None or denom is None:
            vb = self.batch()
            grad_accum = vb.grad_accum if grad_accum is None else grad_accum
            denom = vb.denom if denom is None else denom
            del vb
        r = self.raw
        scratch, counts = _C.densify_plan(grad_accum, denom, r["opacity"], r["scaling"], max_grad,
                                          self.percent_dense * extent, min_opacity,
                                          0.1 * extent if max_screen_size else math.inf)
        del grad_accum, denom
        A, B, Cc, Ns = counts.tolist()
        normals = torch.randn((2 * Ns, 3), generator=generator, device=r["xyz"].device)
        Pn = A + B + 2 * Cc
        groups = (self.raw, self.exp_avg, self.exp_avg_sq)
        new = [{k: torch.empty((Pn,) + r[k].shape[1:], device=r[k].device) for k in self.NAMES} for _ in groups]
        _C.densify_apply(scratch, [A, B, Cc, Ns], normals, [g[k] for g in groups for k in self.NAMES],
                         [g[k] for g in new for k in self.NAMES])
        del r, groups, scratch, normals
        self.raw, self.exp_avg, self.exp_avg_sq = new
        del new
        self._reset_derived(keep_optimizer_state=True)
        return self.P

    def reset_opacity(self):
        """scene/gaussian_model.py:231-234: clamp opacity to <= 0.01 and clear its optimizer state, in place."""
        from . import _C

        _C.reset_opacity(self.raw["opacity"], self.exp_avg["opacity"], self.exp_avg_sq["opacity"])


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
