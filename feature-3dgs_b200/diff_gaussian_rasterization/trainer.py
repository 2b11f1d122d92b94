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
                        (f3dgs_densify_plan / f3dgs_densify_apply) with one host read in between; with absgrad=True
                        the batch also accumulates AbsGS's statistic and densify_and_prune(abs_grad=...) splits on it;
  reset_opacity()       :231-234 in one kernel (f3dgs_reset_opacity);
  relocate_and_add()    3DGS-MCMC's fixed-budget densification (relocate_gs + add_new_gs) with the optimizer state
                        carried along (f3dgs_mcmc_plan / _relocate / _add), one host read; inject_noise() and
                        add_regularizer_grads() its per-step position noise and regulariser gradients;
  compute_3d_filter()   Mip-Splatting's 3D smoothing filter (opt-in, f3dgs_filter3d_*): once on, activate() hands the
                        rasterizer the filtered opacity and scales, step() takes the filter's backward first,
                        densification recomputes it, reset_opacity() resets the filtered opacity, and baked_raw()
                        gives the parameters with the filter folded in, for export;
  prune(keep)           removes the rows a mask drops, with the optimizer state carried along (f3dgs_prune_plan /
                        f3dgs_densify_apply), one host read; prune_by_importance() drops the lowest blend-weight
                        scores (scores.GaussianScores), LightGaussian's rule;
  quantize_features()   LightGaussian's / CompGS's vector quantisation of the feature field (codebook.kmeans): the state
                        then trains a codebook [K,C] in place of per-Gaussian features, activate() decodes codebook[code]
                        for the rasterizer and step() takes the codebook gradient of that gather; dequantize() returns
                        to per-Gaussian features;
  neighbor_graph(k)     the exact k-NN graph of the means (neighbors.knn_graph), cached until the rows change;
                        add_feature_tv_grads() adds the gradient of the feature field's total variation over it, and
                        remove_outliers() prunes statistical outliers.

Float16 feature fields: with feature_dtype=torch.float16 the rasterizer reads a float16 working copy
act["semantic_feature"] of the float32 master raw["semantic_feature"], so every view renders a float16 map and the feature
loss hands back a float16 gradient (feature_head `*_and_grad(..., grad_dtype=torch.float16)`).  The master, its Adam
moments and the accumulated gradient stay float32; the copy is made by one cast at construction and after
densify_and_prune, relocate_and_add writes the relocated rows' copies in its own pass, and step() refreshes it in the
Adam pass itself (f3dgs_adam_step_f16out).
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
                 betas=(0.9, 0.999), eps=1e-15, percent_dense=0.01, feature_dtype=torch.float32, absgrad=False):
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
        self.absgrad = absgrad  # the batch also accumulates AbsGS's statistic (ViewBatch(absgrad=True))
        self.filter_3d: Optional[torch.Tensor] = None  # [P,1] while the 3D filter is on
        self._filter_cameras = None
        # quantised features (quantize_features): codebook [K,C] with its own Adam state, code [P] int32 and its plan
        self.codebook: Optional[torch.Tensor] = None
        self.code: Optional[torch.Tensor] = None
        self._code_plan = None
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
        non-finite coordinate.  kwargs (feature_dtype and absgrad among them) go to the constructor."""
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
        if self.code is not None:  # the decoded field, rewritten by every activate()
            sf = self._decode_features()
        self.act = dict(means3D=self.raw["xyz"], opacities=torch.empty(P, 1, device=dev), scales=torch.empty(P, 3, device=dev),
                        rotations=torch.empty(P, 4, device=dev), shs=torch.empty(P, self.M, 3, device=dev),
                        semantic_feature=sf if sf.dtype == self.feature_dtype else sf.to(self.feature_dtype))
        self._batch: Optional[ViewBatch] = None
        self._graph = None  # neighbor_graph()'s cache: the rows it was built on are gone or reordered
        self._unfiltered = None  # the unfiltered opacity [P,1] and scales [P,3] while the 3D filter is on

    def activate(self):
        """The activated tensors the rasterizer reads (self.act), from the raw parameters.  With the 3D filter on,
        act["opacities"] and act["scales"] hold the filtered values (apply_3d_filter) and the unfiltered ones are kept
        for step().  With quantised features, act["semantic_feature"] is rewritten with codebook[code]."""
        from . import _C

        a, r = self.act, self.raw
        if self.code is not None:
            self._decode_features(a["semantic_feature"])
        if self.filter_3d is None:
            _C.activate(r["opacity"], r["scaling"], r["rotation"], r["f_dc"], r["f_rest"], a["opacities"], a["scales"],
                        a["rotations"], a["shs"])
            return a
        o, s = self._unfiltered
        _C.activate(r["opacity"], r["scaling"], r["rotation"], r["f_dc"], r["f_rest"], o, s, a["rotations"], a["shs"])
        _C.filter3d_apply(o, s, self.filter_3d, a["opacities"], a["scales"])
        return a

    def batch(self) -> ViewBatch:
        if self._batch is None:
            self._batch = ViewBatch(self.act, densify_stats=True, absgrad=self.absgrad)
        return self._batch

    # ---------------------------------------------------------------------------------------------- optimizer
    def step(self, lrs: Dict[str, float], grads: Optional[Dict[str, torch.Tensor]] = None,
             visible: Optional[torch.Tensor] = None):
        """One Adam step of every group.  `grads`: gradients w.r.t. the activated tensors (default: the ViewBatch's).

        visible: None for the dense step, or a bool [P] CUDA mask (ViewBatch.visible() after all_reduce()) for the sparse
        Adam step (f3dgs_adam_step_masked): only the marked Gaussians' raw parameters, moments and float16 feature copy
        change, bitwise as in the dense step; the others stay exactly as they are, so momentum no longer moves Gaussians
        that no view of the step saw.  Bias correction still uses each group's step count, which advances every step.

        With quantised features the codebook takes a dense step (a code is shared by rows in and out of view) from the
        exact gradient of the gather, the per-code sum of grads["semantic_feature"] (CodePlan.grad), with its own
        moments and step count.

        With the 3D filter on, `grads` holds the gradients w.r.t. the filtered opacity and scales; they are turned into
        those w.r.t. the unfiltered ones of the last activate(), in place (f3dgs_filter3d_apply_backward), first."""
        from . import _C

        g = grads if grads is not None else self.batch().grads
        if self.filter_3d is not None:
            o, s = self._unfiltered
            _C.filter3d_apply_backward(o, s, self.filter_3d, g["opacities"], g["scales"], g["opacities"], g["scales"])
        if self.code is not None:
            self.codebook_steps += 1
            _C.adam_step(KIND["semantic_feature"], self.codebook, self._code_plan.grad(g["semantic_feature"]),
                         self.codebook_exp_avg, self.codebook_exp_avg_sq, self.M, lrs["semantic_feature"], self.betas[0],
                         self.betas[1], self.eps, self.codebook_steps, None, None)
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

    def densify_and_prune(self, max_grad, min_opacity, extent, max_screen_size, grad_accum=None, denom=None, generator=None,
                          abs_grad=None, grad_accum_abs=None):
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

        abs_grad (AbsGS's split rule, Ye et al., ACM MM 2024): with ga = grad_accum_abs / denom (0 where NaN), a
        Gaussian is split when ga >= abs_grad and smax > percent_dense * extent; cloning and pruning are unchanged.
        grad_accum_abs defaults to the batch's (GaussianState(absgrad=True)); ValueError when abs_grad is given and
        there is none.  With abs_grad=None the statistic is not read and the result is that of the call without it.
        gsplat's variant, the abs statistic for both decisions, needs no option:
        densify_and_prune(0.0008, ..., grad_accum=vb.grad_accum_abs).

        Two native calls (csrc/densify.cu) and ONE host sync, the read of the four output counts that size the new
        tensors and the normal draw.  Deterministic: identical state, statistics and generator state give bitwise-
        identical output, so data-parallel replicas that densify from the same all-reduced statistics with the same seed
        stay identical."""
        from . import _C

        self._refuse_quantized("densify_and_prune")
        if grad_accum is None or denom is None or (abs_grad is not None and grad_accum_abs is None):
            vb = self.batch()
            grad_accum = vb.grad_accum if grad_accum is None else grad_accum
            denom = vb.denom if denom is None else denom
            if abs_grad is not None and grad_accum_abs is None:
                grad_accum_abs = vb.grad_accum_abs
            del vb
        if abs_grad is None:
            grad_accum_abs = None
        elif grad_accum_abs is None:
            raise ValueError("densify_and_prune: abs_grad needs AbsGS's statistic: pass grad_accum_abs, or build the "
                             "state with absgrad=True")
        r = self.raw
        scratch, counts = _C.densify_plan(grad_accum, denom, r["opacity"], r["scaling"], max_grad,
                                          self.percent_dense * extent, min_opacity,
                                          0.1 * extent if max_screen_size else math.inf, grad_accum_abs,
                                          0.0 if abs_grad is None else abs_grad)
        del grad_accum, denom, grad_accum_abs
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
        if self.filter_3d is not None:
            self.compute_3d_filter()
        return self.P

    def prune(self, keep: torch.Tensor) -> int:
        """Keep the rows where `keep` (a bool or uint8 CUDA tensor [P], any nonzero byte keeps) is set; returns the new P.

        Every raw field and its exp_avg and exp_avg_sq become bitwise t[keep], in order; `steps` is unchanged, the
        float16 feature copy is bitwise raw.half() and max_radii2D is compacted with the rows, as the reference's
        prune_points does.  With quantised features the codes are compacted the same way (the codebook is unchanged)
        and their plan rebuilt, without another host read.  The ViewBatch is rebuilt, and the 3D filter, when on, is
        recomputed for the new means (its own host read).  Per-row statistics the caller keeps (densification statistics, scores) are the caller's to
        index with `keep`.

        Two native calls (csrc/densify.cu: the mask plan, then densify_apply's compaction) and ONE host read, the
        number of rows kept, which sizes the new tensors."""
        from . import _C

        P = self.P
        dev = self.raw["xyz"].device
        if not isinstance(keep, torch.Tensor) or keep.dtype not in (torch.bool, torch.uint8) or keep.shape != (P,):
            raise ValueError(f"prune: keep must be a bool or uint8 tensor [{P}], got "
                             f"{getattr(keep, 'dtype', type(keep))} {tuple(getattr(keep, 'shape', ()))}")
        if keep.device != dev:
            raise ValueError(f"prune: keep must be on {dev}, got {keep.device}")
        keep = keep if keep.dtype == torch.bool else keep != 0
        scratch, counts = _C.prune_plan(keep)
        # max_radii2D's new position: the rank among the kept rows, slot A for the dropped ones
        rank = torch.cumsum(keep, 0, dtype=torch.int64) - 1
        A = int(counts[0])
        slot = torch.where(keep, rank, A)
        radii = torch.empty(A + 1, device=dev).scatter_(0, slot, self.max_radii2D)[:A]
        if self.code is not None:
            self.code = torch.empty(A + 1, dtype=torch.int32, device=dev).scatter_(0, slot, self.code)[:A].contiguous()
            self._code_plan = None
        del rank, slot
        groups = (self.raw, self.exp_avg, self.exp_avg_sq)
        r = self.raw
        new = [{k: torch.empty((A,) + r[k].shape[1:], device=dev) for k in self.NAMES} for _ in groups]
        _C.densify_apply(scratch, [A, 0, 0, 0], torch.empty(0, device=dev), [g[k] for g in groups for k in self.NAMES],
                         [g[k] for g in new for k in self.NAMES])
        del r, groups, scratch
        self.raw, self.exp_avg, self.exp_avg_sq = new
        del new
        if self.code is not None:
            from .codebook import CodePlan

            self._code_plan = CodePlan(self.code, self.codebook.shape[0])
        self._reset_derived(keep_optimizer_state=True)
        self.max_radii2D = radii
        if self.filter_3d is not None:
            self.compute_3d_filter()
        return self.P

    def prune_by_importance(self, scores, prune_ratio: float, volume_power: float = 0.1) -> int:
        """LightGaussian's global-significance pruning: remove exactly n = int(prune_ratio * P) rows, those with the
        smallest v = scores.weight_sum * V ** volume_power, V the product of the three activated scales (the filtered
        ones with the 3D filter on).  Ties go to the lower index first (a stable sort).  LightGaussian also divides V by
        a reference volume; a constant factor does not change the ranking, so it is left out.  `scores` is a
        scores.GaussianScores of this state's Gaussians (all_reduce'd first when data-parallel).  Returns the new P; one
        host read, prune's.

        RadSplat's rule needs no method: state.prune(scores.max_weight >= tau).  Mini-Splatting's importance is
        volume_power=0."""
        P = self.P
        if not 0.0 <= prune_ratio <= 1.0:
            raise ValueError(f"prune_by_importance: prune_ratio must be in [0, 1], got {prune_ratio}")
        w = scores.weight_sum
        if w.shape != (P,):
            raise ValueError(f"prune_by_importance: the scores are of {w.shape[0]} Gaussians, the state has {P}")
        n = int(prune_ratio * P)
        v = w * self.activate()["scales"].prod(dim=1) ** volume_power
        keep = torch.ones(P, dtype=torch.bool, device=w.device)
        keep[torch.sort(v, stable=True).indices[:n]] = False
        return self.prune(keep)

    def reset_opacity(self):
        """scene/gaussian_model.py:231-234: clamp opacity to <= 0.01 and clear its optimizer state, in place.  With the
        3D filter on, Mip-Splatting's reset: the filtered opacity is clamped and the raw opacity set to match it
        (f3dgs_reset_opacity_filter3d)."""
        from . import _C

        r = self.raw
        if self.filter_3d is not None:
            _C.reset_opacity_filter3d(r["opacity"], r["scaling"], self.filter_3d, self.exp_avg["opacity"],
                                      self.exp_avg_sq["opacity"])
            return
        _C.reset_opacity(r["opacity"], self.exp_avg["opacity"], self.exp_avg_sq["opacity"])

    # ---------------------------------------------------------------------------------------------- quantised features
    def quantize_features(self, K: int, iters: int = 10, weights: Optional[torch.Tensor] = None, generator=None):
        """Replace the per-Gaussian features by a k-means codebook [K,C] and one code per Gaussian (LightGaussian's and
        CompGS's vector quantisation; codebook.kmeans on raw["semantic_feature"], `iters` rounds, seeded by
        `generator`).  weights=scores.weight_sum (scores.GaussianScores) weights each Gaussian by how much it renders.

        Afterwards self.codebook [K,C] is trained with its own exp_avg, exp_avg_sq and step count, self.code [P] int32
        stays fixed, and raw["semantic_feature"] with its two moments is released (kept as [P,1,0]).  activate() decodes
        codebook[code] into act["semantic_feature"] (float16 with feature_dtype=torch.float16, half_rn of the float32
        codebook), so ViewBatch, the rasterizer and the feature losses are unchanged; step() trains the codebook (see
        step()).  prune() carries the codes; densify_and_prune and relocate_and_add raise ValueError, as they would need a
        code for every new row.  dequantize() goes back.

        Returns the bytes held for the feature field before and after (dict before=, after=): the per-row features,
        their moments and working copy before; the codebook, its moments, the codes, their plan and the decoded field
        after.  ValueError when already quantised, without features (C == 0), or from kmeans (K > P, bad weights)."""
        from .codebook import CodePlan, kmeans

        if self.code is not None:
            raise ValueError("quantize_features: the features are already quantised")
        P, sf = self.P, self.raw["semantic_feature"]
        C = sf.shape[-1]
        if C == 0:
            raise ValueError("quantize_features: the state has no features (C == 0)")
        before = self._feature_bytes()
        codebook, code = kmeans(sf.reshape(P, C), K, iters=iters, weights=weights, generator=generator)
        self.codebook, self.code, self._code_plan = codebook, code, CodePlan(code, K)
        self.codebook_exp_avg, self.codebook_exp_avg_sq = torch.zeros_like(codebook), torch.zeros_like(codebook)
        self.codebook_steps = 0
        del sf
        for group in (self.raw, self.exp_avg, self.exp_avg_sq):
            group["semantic_feature"] = torch.empty(P, 1, 0, device=codebook.device)
        radii = self.max_radii2D
        self._reset_derived(keep_optimizer_state=True)
        self.max_radii2D = radii
        return dict(before=before, after=self._feature_bytes())

    def dequantize(self):
        """Back to per-Gaussian features: raw["semantic_feature"] = codebook[code] as [P,1,C] float32, with zero Adam
        moments and step count; the codebook, its state and the codes are dropped."""
        if self.code is None:
            raise ValueError("dequantize: the features are not quantised")
        from .codebook import decode

        P = self.P
        sf = decode(self.codebook, self.code).reshape(P, 1, -1)
        self.raw["semantic_feature"] = sf
        self.exp_avg["semantic_feature"] = torch.zeros_like(sf)
        self.exp_avg_sq["semantic_feature"] = torch.zeros_like(sf)
        self.steps["semantic_feature"] = 0
        self.codebook = self.code = self._code_plan = None
        self.codebook_exp_avg = self.codebook_exp_avg_sq = None
        radii = self.max_radii2D
        self._reset_derived(keep_optimizer_state=True)
        self.max_radii2D = radii

    def _decode_features(self, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """codebook[code] as [P,1,C] of feature_dtype, written into `out` when given"""
        from .codebook import decode

        P, C = self.P, self.codebook.shape[1]
        return decode(self.codebook, self.code, self.feature_dtype, out=out).view(P, 1, C)

    def _feature_bytes(self) -> int:
        """bytes of the distinct tensors that hold the feature field and its optimizer state"""
        ts = [self.raw["semantic_feature"], self.exp_avg["semantic_feature"], self.exp_avg_sq["semantic_feature"],
              self.act["semantic_feature"]]
        if self.code is not None:
            ts += [self.codebook, self.codebook_exp_avg, self.codebook_exp_avg_sq, self.code, self._code_plan.scratch]
        seen = {t.data_ptr(): t.numel() * t.element_size() for t in ts if t.numel()}
        return sum(seen.values())

    def _refuse_quantized(self, what: str):
        if self.code is not None:
            raise ValueError(f"{what}: not available while the features are quantised (new rows would need codes); "
                             "call dequantize() first")

    # ---------------------------------------------------------------------------------------------- 3D filter
    def compute_3d_filter(self, cameras=None):
        """Mip-Splatting's compute_3D_filter (filter3d.compute_3d_filter) on the current means: cameras is a sequence of
        GaussianRasterizationSettings, the training views.  It turns the 3D filter on; the camera tensors are kept, so
        that a call without cameras recomputes from the same views (Mip-Splatting recomputes every 100 iterations, and
        densify_and_prune / relocate_and_add recompute it for the new cloud themselves).  One host read.  Raises
        ValueError when no Gaussian is seen (or, without cameras, when the filter has never been computed)."""
        from .filter3d import camera_tensors, compute_from_tensors

        if cameras is not None:
            self._filter_cameras = camera_tensors(cameras)
        elif self._filter_cameras is None:
            raise ValueError("compute_3d_filter: no cameras given and none kept from an earlier call")
        self.filter_3d = compute_from_tensors(self.raw["xyz"], *self._filter_cameras)
        dev, P = self.raw["xyz"].device, self.P
        if self._unfiltered is None or self._unfiltered[0].shape[0] != P:
            self._unfiltered = (torch.empty(P, 1, device=dev), torch.empty(P, 3, device=dev))
        return self.filter_3d

    def baked_raw(self) -> Dict[str, torch.Tensor]:
        """The raw parameters with the 3D filter folded in, Mip-Splatting's save_fused_ply: opacity =
        inverse_sigmoid(filtered opacity) and scaling = log(filtered scales); the other fields are self.raw's.  A model
        saved from it (io.save_ply) renders correctly in any 3DGS renderer without the filter.  With the filter off,
        the raw parameters as they are."""
        from . import _C

        if self.filter_3d is None:
            return dict(self.raw)
        r, P, dev, e = self.raw, self.P, self.raw["xyz"].device, torch.empty(0, device=self.raw["xyz"].device)
        o, s = torch.empty(P, 1, device=dev), torch.empty(P, 3, device=dev)
        _C.activate(r["opacity"], r["scaling"], e, e, e, o, s, e, e)
        o, s = _C.filter3d_apply(o, s, self.filter_3d)
        return dict(r, opacity=inverse_sigmoid(o), scaling=torch.log(s))

    # ---------------------------------------------------------------------------------------------- 3DGS-MCMC
    def relocate_and_add(self, cap_max: int, min_opacity: float = 0.005, generator=None):
        """Fixed-budget densification of 3DGS-MCMC (Kheradmand et al., NeurIPS 2024): the official code's relocate_gs
        followed by add_new_gs; returns (n_relocated, n_added).  Use it in place of densify_and_prune: the cloud grows by
        at most 5 % per call and never past cap_max, so the memory of a run is set by cap_max.

        Relocation: the Gaussians with sigmoid(opacity) <= min_opacity (dead) are moved onto alive ones, drawn with
        torch.multinomial(alive opacity / (sum + float32 eps), n_dead, replacement=True, generator=generator).  Addition:
        n = min(cap_max, int(1.05 P)) - P new rows, drawn the same way over all P opacities, are appended.  A source
        drawn c times and its copies all take the opacity and scale of the relocation rule (csrc/mcmc.cu: N = min(c + 1,
        51) copies render like the original did) and zero Adam moments; a dead row keeps its moments, as in the
        reference.  No draw is made where the reference returns early (nothing dead, nothing alive, no room), so the
        generator advances exactly as the reference's does.  `steps` is unchanged; the float16 feature copy stays
        bitwise raw.half().

        Native calls (f3dgs_mcmc_plan, _relocate, _add) and ONE host read, the number of dead rows, besides what
        torch.multinomial itself does.  Deterministic for equal state and generator state: the draws are made with
        torch's deterministic algorithms enabled (see _multinomial), so data-parallel replicas stay identical."""
        from . import _C

        self._refuse_quantized("relocate_and_add")
        P, r = self.P, self.raw
        if P == 0:
            return 0, 0
        eps = torch.finfo(torch.float32).eps
        groups = [g[k] for g in (self.raw, self.exp_avg, self.exp_avg_sq) for k in self.NAMES]
        scratch, n_dead, index, alive_opacity = _C.mcmc_plan(r["opacity"], min_opacity)
        n_dead = int(n_dead)
        n_relocated = 0
        if 0 < n_dead < P:
            probs = alive_opacity[:P - n_dead]
            draws = _multinomial(probs / (probs.sum() + eps), n_dead, generator)
            half = self.feature_dtype == torch.float16 and self.act["semantic_feature"].numel() > 0
            _C.mcmc_relocate(scratch, index[:n_dead], index[n_dead:][draws], min_opacity, groups,
                             self.act["semantic_feature"] if half else None)
            n_relocated = n_dead
            self._graph = None  # the relocated rows moved (and _reset_derived is not reached without additions)
        del index, alive_opacity
        n_added = min(cap_max, int(1.05 * P)) - P
        if n_added <= 0:
            if n_relocated and self.filter_3d is not None:
                self.compute_3d_filter()
            return n_relocated, 0
        probs = torch.empty(P, 1, device=r["opacity"].device)
        e = torch.empty(0, device=probs.device)
        _C.activate(r["opacity"], e, e, e, e, probs, e, e, e)  # torch.sigmoid, bitwise
        probs = probs.squeeze(-1)
        src = _multinomial(probs / (probs.sum() + eps), n_added, generator).int()
        del probs
        Pn = P + n_added
        new = [{k: torch.empty((Pn,) + r[k].shape[1:], device=r[k].device) for k in self.NAMES} for _ in range(3)]
        _C.mcmc_add(scratch, src, min_opacity, groups, [g[k] for g in new for k in self.NAMES])
        del r, groups, scratch, src
        self.raw, self.exp_avg, self.exp_avg_sq = new
        del new
        self._reset_derived(keep_optimizer_state=True)
        if self.filter_3d is not None:
            self.compute_3d_filter()
        return n_relocated, n_added

    def inject_noise(self, xyz_lr: float, noise_lr: float = 5e5, generator=None):
        """3DGS-MCMC's position noise, after every optimizer step: xyz += R diag(s^2) R^T (eps * g * noise_lr * xyz_lr)
        with eps = torch.randn((P, 3), generator=generator), s = exp(scaling), R the rotation, and the gate
        g = 1 / (1 + exp(-100 ((1 - opacity) - 0.995))), so only nearly transparent Gaussians move.  One kernel
        (f3dgs_mcmc_inject_noise), in place, without host sync."""
        from . import _C

        r = self.raw
        eps = torch.randn((self.P, 3), generator=generator, device=r["xyz"].device)
        _C.mcmc_inject_noise(r["xyz"], r["opacity"], r["scaling"], r["rotation"], eps, noise_lr * xyz_lr)

    def add_regularizer_grads(self, opacity_reg: float, scale_reg: float, grads: Optional[Dict[str, torch.Tensor]] = None):
        """3DGS-MCMC's regularisers opacity_reg * mean(|opacity|) + scale_reg * mean(|scales|) on the activated tensors:
        adds their gradients, opacity_reg / P to every opacity gradient and scale_reg / (3 P) to every scale gradient
        (the activations are positive, so d|x|/dx = 1), to `grads` (default: the ViewBatch's).  Call it once per step,
        after vb.all_reduce() and before step().  The reference adds both terms to the loss of every rendered view, so
        a step over V views matches it with opacity_reg and scale_reg multiplied by V.  Raises ValueError while the 3D
        filter is on: the terms are defined on the unfiltered tensors, but the gradients then belong to filtered ones."""
        if self.filter_3d is not None:
            raise ValueError("add_regularizer_grads: not defined with the 3D filter on (the gradients are those of the "
                             "filtered opacity and scales)")
        g = grads if grads is not None else self.batch().grads
        P = self.P
        if P == 0:
            return
        g["opacities"].add_(opacity_reg / P)
        g["scales"].add_(scale_reg / (3 * P))

    # ---------------------------------------------------------------------------------------------- neighbour graph
    def neighbor_graph(self, k: int, rebuild: bool = False):
        """The exact k-NN graph of raw["xyz"] (neighbors.knn_graph, one host read for its finiteness check), cached.
        Densification, prune, relocate_and_add and quantisation drop the cache; while the means move under step() it is
        the caller's choice when to pass rebuild=True (or call again with another k)."""
        from .neighbors import knn_graph

        if rebuild or self._graph is None or self._graph.k != k:
            self._graph = knn_graph(self.raw["xyz"], k)
        return self._graph

    def add_feature_tv_grads(self, weight: float, k: int = 8, grads: Optional[Dict[str, torch.Tensor]] = None):
        """Adds the gradient of the feature field's total variation over the k-NN graph, weight / (|E| C) * sum over
        edges (i, j) of ||f_i - f_j||_1 (neighbors.feature_tv_loss_and_grad) on the float32 master raw["semantic_feature"],
        to grads["semantic_feature"] (default: the ViewBatch's).  Gaussian Grouping's 3-D neighbour term, in L1: it pulls
        the features of Gaussians that the 2-D loss barely reaches (inside objects, occluded, nearly transparent)
        towards their neighbours'.  Call it once per step after vb.all_reduce() and before step().  Returns the loss (a
        CUDA scalar; no host read besides the graph's).  Raises ValueError while the features are quantised."""
        from .neighbors import feature_tv_loss_and_grad

        if self.code is not None:
            raise ValueError("add_feature_tv_grads: not available while the features are quantised; call dequantize() "
                             "first")
        g = grads if grads is not None else self.batch().grads
        sf = self.raw["semantic_feature"]
        return feature_tv_loss_and_grad(sf, self.neighbor_graph(k), weight, g["semantic_feature"])

    def remove_outliers(self, k: int = 16, std_ratio: float = 2.0) -> int:
        """Statistical outlier removal (neighbors.outlier_mask over the k-NN graph of the means): prune(mask), with the
        optimizer state carried along as prune() does.  Returns the new P."""
        from .neighbors import outlier_mask

        return self.prune(outlier_mask(self.neighbor_graph(k), std_ratio))


def _multinomial(probs, n, generator):
    """torch.multinomial(probs, n, replacement=True, generator=generator), bitwise reproducible: on CUDA its prefix sum
    over the probabilities is only deterministic with torch's deterministic algorithms on, so they are on for this call
    (and the caller's setting is restored).  The draws and the generator's advance are those of the plain call."""
    on, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        return torch.multinomial(probs, n, replacement=True, generator=generator)
    finally:
        torch.use_deterministic_algorithms(on, warn_only=warn_only)


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
