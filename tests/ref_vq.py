"""CPU restatement of csrc/vq.cu in numpy float64: brute-force distances, Lloyd's k-means, segment sums and means, and
the assignment's error bound stated in include/f3dgs_b200.h (f3dgs_vq_assign)."""
import numpy as np


def distances(x, c):
    """d[i, k] = ||x_i - c_k||^2 in float64, [P, K]"""
    x, c = np.asarray(x, np.float64), np.asarray(c, np.float64)
    return (x * x).sum(1)[:, None] - 2.0 * (x @ c.T) + (c * c).sum(1)[None, :]


def assign(x, c):
    """argmin_k d(x_i, c_k), the lowest index on ties"""
    return np.argmin(distances(x, c), axis=1).astype(np.int32)


def assign_bound(x, c):
    """[P]: the bound on d(x, c_code) - min_k d(x, c_k) of the header, per row"""
    D = np.asarray(x).shape[1]
    u = 2.0 ** -11
    g = (D + 8) * 2.0 ** -22
    nx = np.linalg.norm(np.asarray(x, np.float64), axis=1)
    cmax = np.linalg.norm(np.asarray(c, np.float64), axis=1).max()
    return (4 * (2 * u + u * u) + 4 * g * (1 + u) ** 2) * nx * cmax + 2 * g * cmax * cmax


def segment_sum(x, code, K, w=None):
    """(sum_i w_i x_i [K, D], sum_i w_i [K]) over the rows of each code, float64"""
    x = np.asarray(x, np.float64)
    w = np.ones(x.shape[0]) if w is None else np.asarray(w, np.float64)
    s = np.zeros((K, x.shape[1]))
    np.add.at(s, code, w[:, None] * x)
    sw = np.zeros(K)
    np.add.at(sw, code, w)
    return s, sw


def update(c, x, code, w=None):
    """one Lloyd update of codebook c: the float64 weighted means where the total weight is positive, else c"""
    s, sw = segment_sum(x, code, c.shape[0], w)
    out = np.asarray(c, np.float64).copy()
    nz = sw > 0
    out[nz] = s[nz] / sw[nz, None]
    return out


def lloyd(x, c0, iters, w=None):
    """`iters` rounds of assign + update from c0, then a final assign -> (codebook float64, codes)"""
    c = np.asarray(c0, np.float64)
    for _ in range(iters):
        c = update(c, x, assign(x, c), w)
    return c, assign(x, c)
