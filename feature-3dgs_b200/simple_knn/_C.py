"""`simple_knn._C.distCUDA2` on libf3dgs_b200 (f3dgs_knn_mean_dist)."""
from diff_gaussian_rasterization import _C as _native


def distCUDA2(points):
    """points: float32 CUDA tensor [P,3] -> [P] float32, the mean squared distance of each point to its three nearest
    other points (exact; FLT_MAX fills missing neighbours when P < 4, as in the reference)."""
    return _native.knn_mean_dist(points)
