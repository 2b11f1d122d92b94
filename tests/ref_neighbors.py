"""numpy / float64 restatement of the neighbour-graph features (csrc/knn.cu graph_kernel and reverse lists,
csrc/neighbors.cu, diff_gaussian_rasterization/neighbors.py): the exact k-NN graph with ties to the lower index, the
integer sign counts of the total-variation gradient and its loss, the neighbour fill and the statistical outlier mask."""
import numpy as np


def dist2_matrix(pts, rows=None):
    """float64 squared distances of the float32 points: [len(rows), P]"""
    p = np.asarray(pts, np.float32).astype(np.float64)
    q = p if rows is None else p[rows]
    return ((q[:, None, :] - p[None, :, :]) ** 2).sum(-1)


def graph(pts, k):
    """(idx [P,k] int64, dist2 [P,k] float64): row i the k nearest j != i ascending by (distance, j), (-1, inf) past
    P - 1.  Brute force, for small clouds."""
    P = len(pts)
    idx = np.full((P, k), -1, np.int64)
    d2 = np.full((P, k), np.inf)
    for s in range(0, P, 1024):
        rows = np.arange(s, min(P, s + 1024))
        d = dist2_matrix(pts, rows)
        d[np.arange(len(rows)), rows] = np.inf
        m = min(k, P - 1)
        if m <= 0:
            continue
        order = np.lexsort((np.broadcast_to(np.arange(P), d.shape), d), axis=1)[:, :m]  # by distance, then index
        idx[rows, :m] = order
        d2[rows, :m] = np.take_along_axis(d, order, 1)
    return idx, d2


def kdtree_graph(pts, k):
    """(idx, dist2 float64) from scipy's cKDTree: query k + 1 and drop the query's own index (with duplicates it need not
    come first), else the last entry.  Ties are in cKDTree's order."""
    from scipy.spatial import cKDTree

    p = np.asarray(pts, np.float32).astype(np.float64)
    P = len(p)
    m = min(k, P - 1)
    idx = np.full((P, k), -1, np.int64)
    d2 = np.full((P, k), np.inf)
    if m <= 0:
        return idx, d2
    dist, nb = cKDTree(p).query(p, k=m + 1, workers=-1)
    own = nb == np.arange(P)[:, None]
    drop = np.where(own.any(1), own.argmax(1), m)
    keep = np.ones_like(own)
    keep[np.arange(P), drop] = False
    idx[:, :m] = nb[keep].reshape(P, m)
    d2[:, :m] = dist[keep].reshape(P, m) ** 2
    return idx, d2


def reverse(idx, P):
    """(offsets [P+1], sources [P k]) of the transpose, sources ascending per row, -1 past offsets[P]"""
    rows = [[] for _ in range(P)]
    for i, r in enumerate(idx):
        for j in r:
            if 0 <= j < P:
                rows[j].append(i)
    offsets = np.zeros(P + 1, np.int64)
    offsets[1:] = np.cumsum([len(r) for r in rows])
    sources = np.full(idx.size, -1, np.int64)
    flat = [i for r in rows for i in r]
    sources[:len(flat)] = flat
    return offsets, sources


def tv_counts(f, idx):
    """n [P,C] int64: sum_{j in N(i)} sign(f_i - f_j) - sum_{i' in R(i)} sign(f_i' - f_i)"""
    f = np.asarray(f, np.float32).reshape(len(idx), -1)
    n = np.zeros(f.shape, np.int64)
    i, j = np.nonzero(idx >= 0)
    nb = idx[i, j]
    s = np.sign(f[i].astype(np.float64) - f[nb]).astype(np.int64)
    np.add.at(n, i, s)
    np.add.at(n, nb, -s)
    return n


def n_edges(idx):
    return int((idx >= 0).sum())


def tv_loss(f, idx, weight):
    """weight / (|E| C) * sum_{(i,j) in E} sum_c |f_ic - f_jc| in float64"""
    f = np.asarray(f, np.float32).reshape(len(idx), -1).astype(np.float64)
    i, j = np.nonzero(idx >= 0)
    E = len(i)
    if E == 0:
        return 0.0
    return weight / (E * f.shape[1]) * np.abs(f[i] - f[idx[i, j]]).sum()


def tv_scale(idx, C, weight):
    """s = float32(weight / (|E| C))"""
    return np.float32(weight / (n_edges(idx) * C))


def fill(f, w, idx, min_weight=0.0):
    """float64 fill: rows with w <= min_weight that have neighbours with w > min_weight take their weighted mean"""
    f = np.asarray(f, np.float32).reshape(len(idx), -1).astype(np.float64)
    out = f.copy()
    w = np.asarray(w, np.float32).astype(np.float64)
    for i in range(len(idx)):
        if not w[i] <= min_weight:
            continue
        nb = [j for j in idx[i] if j >= 0 and w[j] > min_weight]
        if nb:
            out[i] = (w[nb, None] * f[nb]).sum(0) / w[nb].sum()
    return out


def outlier_mask(idx, dist2, std_ratio=2.0):
    valid = idx >= 0
    n = valid.sum(1)
    d = np.where(valid, np.sqrt(np.where(valid, dist2, 0.0)), 0.0).sum(1) / np.maximum(n, 1)
    has = n > 0
    if not has.any():
        return np.ones(len(idx), bool)
    mu = d[has].mean()
    sd = d[has].std()
    return ~has | (d <= mu + std_ratio * sd)
