"""Neighbour graphs of Gaussians on the GPU (csrc/knn.cu, csrc/neighbors.cu; include/f3dgs_b200.h f3dgs_knn_graph,
f3dgs_knn_reverse, f3dgs_feature_tv_accum, f3dgs_feature_fill).

  knn_graph(points, k)        the exact k-NN graph of a cloud: idx [P,k] int32 and dist2 [P,k] float32, rows ascending by
                              (dist2, index), the point itself excluded by index, (-1, +inf) past P - 1 neighbours;
  feature_tv_loss(f, g, w)    total variation of a feature field over the graph's edges, an autograd function:
                              w / (|E| C) * sum_{(i,j) in E} sum_c |f_ic - f_jc| (Gaussian Grouping's 3-D neighbour term
                              in L1: it flattens features inside an object and keeps the jump at its boundary);
  feature_tv_loss_and_grad    the same loss with its gradient ADDED to a caller's buffer, for the native training loop;
  fill_features(f, w, g)      rows whose weight is <= min_weight take the weighted mean of their neighbours' rows
                              (FeatureLift.result()'s Gaussians that no view blended);
  outlier_mask(g, r)          statistical outlier removal: keep rows whose mean neighbour distance is <= mean + r std.
"""
import math
from typing import Optional, Tuple

import torch


class KnnGraph:
    """The exact k-NN graph of P points: idx [P,k] int32, dist2 [P,k] float32 (input row order), order [P] int32 (the
    Morton order of the search, a permutation in which rows close in space are close in memory; the loss walks its rows
    in it) and, built on first use, the reverse lists (reverse(): CSR offsets [P+1] and sources [P k], the rows that list
    each point, ascending, -1 past offsets[P])."""

    def __init__(self, idx: torch.Tensor, dist2: torch.Tensor, order: torch.Tensor):
        self.idx, self.dist2, self.order = idx, dist2, order
        self._reverse: Optional[Tuple[torch.Tensor, torch.Tensor]] = None

    @property
    def P(self) -> int:
        return self.idx.shape[0]

    @property
    def k(self) -> int:
        return self.idx.shape[1]

    @property
    def n_edges(self) -> int:
        """|E|, the number of valid entries of idx: every point has min(k, P - 1) neighbours"""
        return self.P * min(self.k, max(self.P - 1, 0))

    def reverse(self) -> Tuple[torch.Tensor, torch.Tensor]:
        from . import _C

        if self._reverse is None:
            self._reverse = _C.knn_reverse(self.idx)
        return self._reverse


def knn_graph(points: torch.Tensor, k: int) -> KnnGraph:
    """The exact k-NN graph of points [P,3] (a float32 CUDA tensor), 1 <= k <= 32.  ValueError on a non-finite
    coordinate (one host read) or k out of range."""
    from . import _C

    if not isinstance(points, torch.Tensor) or points.dim() != 2 or points.shape[1] != 3 or not points.is_cuda:
        raise ValueError(f"points must be a CUDA tensor [P,3], got {tuple(getattr(points, 'shape', ()))}")
    if not 1 <= k <= 32:
        raise ValueError(f"k must be in [1, 32], got {k}")
    points = points.float()
    if not bool(torch.isfinite(points).all()):
        raise ValueError("points contain a non-finite coordinate")
    return KnnGraph(*_C.knn_graph(points, int(k)))


def _rows(features: torch.Tensor, graph: KnnGraph) -> torch.Tensor:
    if features.dtype != torch.float32 or not features.is_cuda or features.shape[0] != graph.P:
        raise ValueError(f"features must be a float32 CUDA tensor with {graph.P} rows, got {features.dtype} "
                         f"{tuple(features.shape)} on {features.device}")
    return features.reshape(graph.P, -1)


def feature_tv_loss_and_grad(features: torch.Tensor, graph: KnnGraph, weight: float, grad: torch.Tensor) -> torch.Tensor:
    """Total variation of features [P, ...] (float32, P rows of C values) over the graph's valid edges E:

        L = weight / (|E| C) * sum_{(i,j) in E} sum_c |f_ic - f_jc|

    Returns L as a float32 CUDA scalar (summed in float64, in a fixed order) and ADDS dL/df to grad (a contiguous
    float32 tensor of P C elements), bitwise grad + float(n) * s with s = float32(weight / (|E| C)) and n the integer
    count sum_{j in N(i)} sign(f_i - f_j) - sum_{i' in R(i)} sign(f_i' - f_i), sign(0) = 0.  No host read; the reverse
    lists are built on the first call for the graph."""
    from . import _C

    f = _rows(features, graph)
    if graph.P == 0 or f.shape[1] == 0:
        return torch.zeros((), device=features.device)
    offsets, sources = graph.reverse()
    loss = _C.feature_tv_accum(f, graph.idx, offsets, sources, graph.order, float(weight), graph.n_edges, grad)
    return loss.float()


class _FeatureTV(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, graph, weight):
        g = torch.zeros(features.shape, dtype=torch.float32, device=features.device)
        loss = feature_tv_loss_and_grad(features.detach(), graph, weight, g)
        ctx.save_for_backward(g)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        (g,) = ctx.saved_tensors
        return g * dloss, None, None


def feature_tv_loss(features: torch.Tensor, graph: KnnGraph, weight: float = 1.0) -> torch.Tensor:
    """feature_tv_loss_and_grad as an autograd function of features: the gradient is formed in the forward pass and
    scaled by the incoming gradient in the backward."""
    return _FeatureTV.apply(features, graph, weight)


def fill_features(features: torch.Tensor, weight: torch.Tensor, graph: KnnGraph, min_weight: float = 0.0) -> torch.Tensor:
    """A new tensor of features' shape: every row i with weight[i] <= min_weight that has neighbours j with weight[j] >
    min_weight becomes sum_j w_j f_j / sum_j w_j over them (float64 sums in neighbour order, rounded once); every other
    row is copied bitwise.  Meant for FeatureLift.result(): fill_features(feats, weight_sum, graph)."""
    from . import _C

    f = _rows(features, graph)
    if weight.shape != (graph.P,) or not weight.is_cuda:
        raise ValueError(f"weight must be a CUDA tensor [{graph.P}], got {tuple(weight.shape)}")
    if math.isnan(min_weight):
        raise ValueError("min_weight must not be NaN")
    return _C.feature_fill(f, weight.float(), graph.idx, float(min_weight)).view(features.shape)


def outlier_mask(graph: KnnGraph, std_ratio: float = 2.0) -> torch.Tensor:
    """Statistical outlier removal (PCL's StatisticalOutlierRemoval, Open3D's remove_statistical_outlier; their
    neighbour conventions differ, so the masks need not agree bitwise): a bool keep-mask [P].  With d_i the mean of
    sqrt(dist2) over row i's valid neighbours, row i is kept when d_i <= mean(d) + std_ratio * std(d), std the population
    one, all in float64.  Rows without neighbours (P = 1) are kept."""
    valid = graph.idx >= 0
    n = valid.sum(1)
    d = torch.where(valid, graph.dist2.double().sqrt(), 0.0).sum(1) / n.clamp_min(1)
    has = n > 0
    dh = d[has]
    if dh.numel() == 0:
        return torch.ones(graph.P, dtype=torch.bool, device=graph.idx.device)
    mu = dh.mean()
    sd = ((dh - mu) ** 2).mean().sqrt()
    return ~has | (d <= mu + std_ratio * sd)
