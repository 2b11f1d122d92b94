"""Per-Gaussian blend-weight scores over views, the statistics compaction methods prune a trained scene by
(csrc/composite_bwd.cu's score mode, f3dgs_gaussian_scores_accum):

    weight_sum[i]   = sum_{v,p} w_ivp        LightGaussian's global significance (before its volume factor),
                                             Mini-Splatting's importance
    max_weight[i]   = max_{v,p} w_ivp        RadSplat's score
    pixel_count[i]  = #{(v, p) blended}      LightGaussian's hit count

with w_ivp = alpha * T, Gaussian i's blend weight at pixel p of view v, and the pairs counted exactly those the forward
composited.  A Gaussian with pixel_count 0 adds nothing to any pixel, but it may still end one: the composite stops, as
the reference's does, at the first pair that would take T below 1e-4, without blending it.  Pruning it lets the next
Gaussians blend there, so renders change only at pixels whose T_final was below 0.01.  Usage:

    scores = GaussianScores(means3D, opacities, scales, rotations)     # or GaussianScores.from_state(state)
    for rs in train_settings:
        scores.add(rs)
    scores.all_reduce()                  # data-parallel: each rank scored a share of the views
    state.prune_by_importance(scores, 0.6)        # or state.prune(scores.max_weight >= tau), ...

Pruning itself is GaussianState.prune / prune_by_importance (trainer.py).  There is no autograd and no CPU path.
"""
import torch

from .feature_head import _C, _weights_forward


class GaussianScores:
    """Accumulates weight_sum [P] float32, max_weight [P] float32 and pixel_count [P] int64 over views.

    Each `add` is the forward FeatureLift.add makes (C = 0, zero colors_precomp, so no SH work) and one score walk: the
    backward's geometry walk over the forward's buffers without instance lists, feature kernel or upstream gradient.
    It allocates nothing beyond the forward's buffers and makes no host sync beyond the forward's own read of R.
    antialiasing=True scores the antialiased model (AntialiasedGaussianRasterizer's opacities).  pixel_count and
    max_weight are exact and do not depend on the order of the views; weight_sum is a float sum."""

    def __init__(self, means3D, opacities, scales=None, rotations=None, cov3D_precomp=None, antialiasing: bool = False):
        if (scales is None or rotations is None) == (cov3D_precomp is None):
            raise ValueError("GaussianScores: provide exactly one of (scales, rotations) / cov3D_precomp")
        if not means3D.is_cuda:
            raise ValueError("GaussianScores: means3D must be a CUDA tensor (there is no CPU path)")
        dev = means3D.device
        self.P = int(means3D.shape[0])
        self.antialiasing = bool(antialiasing)
        e = torch.empty(0, device=dev)
        self._geom = dict(means3D=means3D.detach(), opacities=opacities.detach(),
                          scales=e if scales is None else scales.detach(),
                          rotations=e if rotations is None else rotations.detach(),
                          cov3D=e if cov3D_precomp is None else cov3D_precomp.detach())
        self._colors = torch.zeros(self.P, 3, device=dev)
        self._empty = e
        self.weight_sum = torch.zeros(self.P, device=dev)
        self.max_weight = torch.zeros(self.P, device=dev)
        self.pixel_count = torch.zeros(self.P, dtype=torch.int64, device=dev)

    @classmethod
    def from_state(cls, state, antialiasing: bool = False):
        """Scores of a trainer.GaussianState's Gaussians as they render: its activated tensors, the filtered opacity
        and scales when the 3D filter is on."""
        act = state.activate()
        return cls(act["means3D"], act["opacities"], act["scales"], act["rotations"], antialiasing=antialiasing)

    def add(self, raster_settings):
        """Accumulate one view, rendered at (raster_settings.image_height, raster_settings.image_width)."""
        if self.P == 0:
            return
        rs = raster_settings
        H, W = rs.image_height, rs.image_width
        with torch.no_grad():
            R, geom, binning, img = _weights_forward(self._geom, self._colors, self._empty, self.antialiasing, rs, H, W)
            _C().gaussian_scores_accum(geom, R, binning, img, W, H, self.weight_sum, self.max_weight, self.pixel_count)

    def all_reduce(self, group=None):
        """Combine the ranks' scores in place (torch.distributed): weight_sum and pixel_count by SUM, max_weight by MAX.
        Every rank then holds the scores of all views and prunes identically."""
        import torch.distributed as dist

        dist.all_reduce(self.weight_sum, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(self.pixel_count, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(self.max_weight, op=dist.ReduceOp.MAX, group=group)
