"""Neighbour graphs of Gaussians: the exact k-NN graph and its reverse lists (csrc/knn.cu), the total variation of the
feature field over it and the neighbour fill (csrc/neighbors.cu), the outlier mask, neighbors.py and GaussianState's
neighbor_graph / add_feature_tv_grads / remove_outliers.

The yardstick is tests/ref_neighbors.py, a numpy / float64 restatement.  The graph's distances are within 1e-6 of the
float64 ones, relatively, and its index sets equal the restatement's except where the float64 k-th and (k+1)-th
distances are within that bound of each other (a near tie the float32 distances may order either way).  On integer
grids every distance is exact and the graph is compared bitwise, tie order included.  The gradient is compared bitwise
with grad + float(n) * s, n counted by the restatement."""
import ctypes

import numpy as np
import pytest
import torch

import ref_neighbors as ref
from test_knn_init import clustered, small_clouds

INT_MAX = 2**31 - 1
NEAR_TIE = 1e-6


# ---------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", list(small_clouds()))
@pytest.mark.parametrize("k", [1, 3, 8])
def test_restatement_matches_kdtree(name, k):
    pts = small_clouds()[name]
    idx, d2 = ref.graph(pts, k)
    kidx, kd2 = ref.kdtree_graph(pts, k)
    assert np.array_equal(np.isfinite(d2), np.isfinite(kd2))
    fin = np.isfinite(d2)
    assert np.allclose(d2[fin], kd2[fin], rtol=1e-12, atol=1e-15)
    assert np.array_equal(idx < 0, kidx < 0)
    _, d2n = ref.graph(pts, k + 1)
    for i in range(len(pts)):
        m = int((idx[i] >= 0).sum())
        if m == k and np.isfinite(d2n[i, k]) and d2n[i, k] - d2[i, k - 1] <= NEAR_TIE * d2n[i, k]:
            continue  # a tie at the k-th place: cKDTree may pick either
        assert set(idx[i, :m]) == set(kidx[i, :m]), (name, i)


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    p, i = ctypes.c_void_p, ctypes.c_int
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_launch_count.restype = ctypes.c_ulonglong
    L.f3dgs_knn_graph_scratch_bytes.restype = ctypes.c_size_t
    L.f3dgs_knn_graph_scratch_bytes.argtypes = [i, i]
    L.f3dgs_knn_graph.argtypes = [i, i, p, p, p, p, p, p]
    L.f3dgs_knn_reverse.argtypes = [i, i, p, p, p, p, p]
    L.f3dgs_feature_tv_accum.argtypes = [i, i, i, p, p, p, p, p, ctypes.c_double, ctypes.c_longlong, p, p, p]
    L.f3dgs_feature_fill.argtypes = [i, i, i, p, p, p, ctypes.c_float, p, p]
    return L


def _rejected(lib, name, call, msg):
    assert call() == -1
    err = lib.f3dgs_last_error()
    assert err.startswith(name + b": ") and msg in err, (name, err)


BAD_PK = [(-1, 8), (10, 0), (10, 33), (2**27, 32)]


def test_cabi_rejects_bad_arguments_before_touching_cuda(lib):
    n0 = lib.f3dgs_launch_count()
    P, k, C = 10, 4, 8
    pts, idx, d2, order, scr = 0x1000000, 0x2000000, 0x3000000, 0x4000000, 0x5000000
    off, src, f, g, loss, w, out = 0x6000000, 0x7000000, 0x8000000, 0x9000000, 0xa000000, 0xb000000, 0xc000000

    fn, name = lib.f3dgs_knn_graph, b"f3dgs_knn_graph"
    for s in BAD_PK:
        _rejected(lib, name, lambda: fn(*s, pts, idx, d2, order, scr, None), b"bad sizes")
    assert fn(0, k, None, None, None, None, None, None) == 0
    for j in range(5):
        a = [pts, idx, d2, order, scr]
        a[j] = None
        _rejected(lib, name, lambda: fn(P, k, *a, None), b"NULL")
    for a in ([pts, idx, idx + 8, order, scr], [pts, pts + 4, d2, order, scr], [pts, idx, d2, d2 + 16, scr],
              [pts, idx, d2, order, order - 8], [pts, scr + 256, d2, order, scr]):
        _rejected(lib, name, lambda: fn(P, k, *a, None), b"overlap")

    fn, name = lib.f3dgs_knn_reverse, b"f3dgs_knn_reverse"
    for s in BAD_PK:
        _rejected(lib, name, lambda: fn(*s, idx, off, src, scr, None), b"bad sizes")
    for j in range(4):
        a = [idx, off, src, scr]
        a[j] = None
        _rejected(lib, name, lambda: fn(P, k, *a, None), b"NULL")
    for a in ([idx, off, off + 4 * P, scr], [idx, idx + 4, src, scr], [idx, off, scr + 512, scr]):
        _rejected(lib, name, lambda: fn(P, k, *a, None), b"overlap")

    fn, name = lib.f3dgs_feature_tv_accum, b"f3dgs_feature_tv_accum"
    good = [f, idx, off, src, order, 1.0, P * k, g, loss]
    for s in [(-1, k, C), (P, 0, C), (P, 33, C), (P, k, 0), (P, k, 4097), (2**27, 32, C)]:
        _rejected(lib, name, lambda: fn(*s, *good, None), b"bad sizes")
    for ne in (-1, P * k + 1):
        a = list(good)
        a[6] = ne
        _rejected(lib, name, lambda: fn(P, k, C, *a, None), b"bad sizes")
    a = list(good)
    a[5] = float("inf")
    _rejected(lib, name, lambda: fn(P, k, C, *a, None), b"finite")
    for j in (0, 1, 2, 3, 7, 8):
        a = list(good)
        a[j] = None
        _rejected(lib, name, lambda: fn(P, k, C, *a, None), b"NULL")
    for j, v in ((7, f + 16), (7, src - 8), (8, g + 8), (8, order)):
        a = list(good)
        a[j] = v
        _rejected(lib, name, lambda: fn(P, k, C, *a, None), b"overlap")
    a = list(good)
    a[4] = None  # order may be NULL: row order; the call then gets as far as the overlap check
    a[7] = f
    _rejected(lib, name, lambda: fn(P, k, C, *a, None), b"overlap")

    fn, name = lib.f3dgs_feature_fill, b"f3dgs_feature_fill"
    for s in [(-1, k, C), (P, 0, C), (P, 33, C), (P, k, 0), (P, k, 4097)]:
        _rejected(lib, name, lambda: fn(*s, f, w, idx, 0.0, out, None), b"bad sizes")
    _rejected(lib, name, lambda: fn(P, k, C, f, w, idx, float("nan"), out, None), b"NaN")
    for j in range(4):
        a = [f, w, idx, out]
        a[j] = None
        _rejected(lib, name, lambda: fn(P, k, C, a[0], a[1], a[2], 0.0, a[3], None), b"NULL")
    for o in (f + 4, w - 4 * P * C + 4, idx + 16):
        _rejected(lib, name, lambda: fn(P, k, C, f, w, idx, 0.0, o, None), b"overlap")

    assert lib.f3dgs_knn_graph_scratch_bytes(0, 8) == 0 and lib.f3dgs_knn_graph_scratch_bytes(10, 33) == 0
    assert lib.f3dgs_launch_count() == n0


def test_python_api_rejects_bad_input_without_a_gpu(built):
    from diff_gaussian_rasterization import knn_graph

    with pytest.raises(ValueError):
        knn_graph(torch.zeros(5, 3), 4)  # a CPU tensor


# ---------------------------------------------------------------------------------------------------- GPU helpers
def _graph(pts, k):
    from diff_gaussian_rasterization import knn_graph

    return knn_graph(torch.from_numpy(np.ascontiguousarray(pts, np.float32)).cuda(), k)


def _np(g):
    return g.idx.cpu().numpy().astype(np.int64), g.dist2.cpu().numpy()


def _check_graph(pts, k, gi, gd, ridx=None, rd2=None):
    """gi / gd against the restatement (brute force, or the given one): the row order, the distances within NEAR_TIE,
    the index sets outside near ties at the k-th place, the (-1, inf) fill"""
    P = len(pts)
    if ridx is None:
        ridx, rd2 = ref.graph(pts, k + 1)
    m = min(k, P - 1) if P > 0 else 0
    assert gi.shape == (P, k) and gd.shape == (P, k) and gd.dtype == np.float32
    assert np.all(gi[:, m:] == -1) and np.all(np.isposinf(gd[:, m:]))
    if m == 0:
        return
    gi, gd = gi[:, :m], gd[:, :m]
    assert np.all((gi >= 0) & (gi < P)) and np.all(gi != np.arange(P)[:, None])
    for i in range(0, P, max(1, P // 2000)):  # distinct, ascending by (dist2, index)
        assert len(set(gi[i])) == m
    prev_d, prev_i = gd[:, :-1], gi[:, :-1]
    assert np.all((prev_d < gd[:, 1:]) | ((prev_d == gd[:, 1:]) & (prev_i < gi[:, 1:])))
    r = rd2[:, :m]
    err = np.abs(gd.astype(np.float64) - r)
    assert np.all(err <= NEAR_TIE * r + 1e-30), float((err - NEAR_TIE * r).max())
    kth = rd2[:, m - 1]
    nxt = rd2[:, m] if rd2.shape[1] > m else np.full(P, np.inf)
    clear = ~np.isfinite(nxt) | (nxt - kth > NEAR_TIE * nxt)
    a, b = np.sort(gi[clear], 1), np.sort(ridx[clear, :m], 1)
    assert np.array_equal(a, b), int(np.argmax((a != b).any(1)))


def _uniform(P, seed, a=1.3):
    return np.random.default_rng(seed).uniform(-a, a, (P, 3)).astype(np.float32)


def _clouds():
    rng = np.random.default_rng(31)
    dup = rng.uniform(-1, 1, (300, 3)).astype(np.float32)
    planar = rng.uniform(-1, 1, (3000, 3)).astype(np.float32)
    planar[:, 2] = 0.5
    t = rng.uniform(-1, 1, (3000, 1))
    return {"uniform": _uniform(5000, 1), "clustered": clustered(6000, 2),
            "duplicates": np.concatenate([dup, dup[:150], dup[:40], dup[:7]]),
            "identical": np.full((200, 3), 0.25, np.float32), "planar": planar,
            "collinear": (np.array([[0.3, -0.2, 0.9]]) * t + np.array([[1.0, 2.0, 3.0]])).astype(np.float32)}


# ---------------------------------------------------------------------------------------------------- graph
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_clouds()))
@pytest.mark.parametrize("k", [1, 4, 5, 8, 16, 17, 32])
def test_graph_is_exact(name, k):
    pts = _clouds()[name]
    _check_graph(pts, k, *_np(_graph(pts, k)))


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3, 4, 5, 40])
@pytest.mark.parametrize("k", [1, 3, 8, 32])
def test_tiny_clouds_fill_with_minus_one_and_inf(P, k):
    pts = _uniform(P, 100 + P)
    gi, gd = _np(_graph(pts, k))
    _check_graph(pts, k, gi, gd)
    assert np.all(gi[:, min(k, P - 1):] == -1)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [6, 8, 26, 32])
def test_integer_grid_is_bitwise_with_ties_to_the_lower_index(k):
    g = np.stack(np.meshgrid(*[np.arange(9, dtype=np.float32)] * 3, indexing="ij"), -1).reshape(-1, 3)
    pts = np.random.default_rng(k).permutation(np.concatenate([g, g[::7]]))  # duplicates too
    gi, gd = _np(_graph(pts, k))
    ridx, rd2 = ref.graph(pts, k)
    assert np.array_equal(gi, ridx)
    assert np.array_equal(gd, rd2.astype(np.float32))


@pytest.mark.gpu
def test_large_cloud_against_kdtree():
    pts = clustered(200000, 77)
    k = 16
    ridx, rd2 = ref.kdtree_graph(pts, k + 1)
    _check_graph(pts, k, *_np(_graph(pts, k)), ridx=ridx, rd2=rd2)


@pytest.mark.gpu
def test_reproducible_and_permutation_equivariant():
    pts = clustered(100000, 5)
    a, b = _np(_graph(pts, 16)), _np(_graph(pts, 16))
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    perm = np.random.default_rng(2).permutation(len(pts))
    pi, pd = _np(_graph(pts[perm], 16))
    assert np.array_equal(pd, a[1][perm])
    # indices: renamed by the permutation, except where equal distances let the lower-index rule choose differently
    distinct = np.all(np.diff(a[1][perm], axis=1) > 0, axis=1)
    assert np.array_equal(perm[pi[distinct]], a[0][perm][distinct])


@pytest.mark.gpu
def test_order_is_a_permutation_and_reverse_lists_are_the_transpose():
    pts = clustered(20000, 8)
    for k in (3, 16):
        g = _graph(pts, k)
        assert np.array_equal(np.sort(g.order.cpu().numpy()), np.arange(len(pts)))
        off, src = g.reverse()
        ro, rs = ref.reverse(_np(g)[0], len(pts))
        assert np.array_equal(off.cpu().numpy(), ro) and np.array_equal(src.cpu().numpy(), rs)
    g = _graph(_uniform(4, 3), 8)  # P <= k: the -1 entries are dropped
    off, src = g.reverse()
    ro, rs = ref.reverse(_np(g)[0], 4)
    assert np.array_equal(off.cpu().numpy(), ro) and np.array_equal(src.cpu().numpy(), rs) and int(off[-1]) == 12


@pytest.mark.gpu
def test_knn_graph_rejects_bad_input():
    from diff_gaussian_rasterization import knn_graph

    pts = torch.zeros(10, 3, device="cuda")
    for k in (0, 33):
        with pytest.raises(ValueError):
            knn_graph(pts, k)
    for bad in (float("nan"), float("inf")):
        p = pts.clone()
        p[3, 1] = bad
        with pytest.raises(ValueError, match="non-finite"):
            knn_graph(p, 4)


# ---------------------------------------------------------------------------------------------------- total variation
def _features(P, C, seed):
    rng = np.random.default_rng(seed)
    return (np.round(rng.normal(size=(P, C)) * 4) / 4).astype(np.float32)  # coarse values: many exact ties, sign(0)


@pytest.mark.gpu
@pytest.mark.parametrize("P,k,C", [(3000, 8, 1), (3000, 8, 3), (3000, 8, 128), (2000, 16, 512), (300, 8, 4096),
                                   (3, 8, 5), (5, 8, 128), (1000, 3, 130)])
def test_tv_gradient_is_bitwise_and_loss_within_1e6(P, k, C):
    from diff_gaussian_rasterization import feature_tv_loss_and_grad

    pts = clustered(P, P + C)
    g = _graph(pts, k)
    idx = _np(g)[0]
    f = _features(P, C, C)
    g0 = np.random.default_rng(1).normal(size=(P, C)).astype(np.float32)
    grad = torch.from_numpy(g0).cuda()
    weight = 0.37
    loss = feature_tv_loss_and_grad(torch.from_numpy(f).cuda(), g, weight, grad)
    n = ref.tv_counts(f, idx)
    s = ref.tv_scale(idx, C, weight)
    want = g0 + n.astype(np.float32) * s  # numpy float32: the product rounded, then the sum
    assert np.array_equal(grad.cpu().numpy(), want)
    rl = ref.tv_loss(f, idx, weight)
    assert abs(float(loss) - rl) <= 1e-6 * abs(rl) + 1e-30, (float(loss), rl)
    assert loss.dtype == torch.float32 and loss.is_cuda


@pytest.mark.gpu
def test_tv_autograd_and_independence_from_the_walk_order():
    from diff_gaussian_rasterization import feature_tv_loss, feature_tv_loss_and_grad
    from diff_gaussian_rasterization import _C

    pts = clustered(5000, 3)
    g = _graph(pts, 8)
    f = torch.from_numpy(_features(5000, 64, 4)).cuda()
    x = f.clone().requires_grad_(True)
    loss = feature_tv_loss(x, g, 2.0)
    (3.0 * loss).backward()
    grad = torch.zeros_like(f)
    l2 = feature_tv_loss_and_grad(f, g, 2.0, grad)
    assert torch.equal(loss.detach(), l2) and torch.equal(x.grad, grad * 3.0)
    # row order instead of the Morton walk: bitwise the same
    off, src = g.reverse()
    grad2 = torch.zeros_like(f)
    l3 = _C.feature_tv_accum(f, g.idx, off, src, None, 2.0, g.n_edges, grad2)
    assert torch.equal(grad2, grad) and float(l3) == float(
        _C.feature_tv_accum(f, g.idx, off, src, g.order, 2.0, g.n_edges, torch.zeros_like(f)))


# ---------------------------------------------------------------------------------------------------- fill and mask
def _within_one_ulp(out, want):
    w32 = want.astype(np.float32)
    return np.all(np.abs(out.astype(np.float64) - want) <= np.spacing(np.abs(w32)).astype(np.float64))


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 3, 128, 4096])
def test_fill_within_one_ulp_and_copies_the_rest(C):
    from diff_gaussian_rasterization import fill_features

    P = 2000 if C < 4096 else 300
    pts = clustered(P, C)
    g = _graph(pts, 8)
    rng = np.random.default_rng(C)
    f = rng.normal(size=(P, C)).astype(np.float32)
    w = rng.uniform(0, 2, P).astype(np.float32)
    w[rng.random(P) < 0.4] = 0.0
    w[rng.random(P) < 0.1] = 0.25  # <= min_weight below
    out = fill_features(torch.from_numpy(f).cuda(), torch.from_numpy(w).cuda(), g, min_weight=0.25).cpu().numpy()
    want = ref.fill(f, w, _np(g)[0], 0.25)
    filled = np.any(want != f.astype(np.float64), axis=1)
    assert np.array_equal(out[~filled], f[~filled])
    assert filled.sum() > 0.2 * P and _within_one_ulp(out[filled], want[filled])


@pytest.mark.gpu
def test_outlier_mask_matches_restatement_and_removes_planted_outliers():
    from diff_gaussian_rasterization import outlier_mask

    rng = np.random.default_rng(4)
    body = clustered(20000, 6, outlier_frac=0.0)
    far = rng.uniform(5, 6, (25, 3)).astype(np.float32) * rng.choice([-1, 1], (25, 3))
    pts = np.concatenate([body, far]).astype(np.float32)
    g = _graph(pts, 16)
    m = outlier_mask(g, 2.0)
    assert m.dtype == torch.bool and m.shape == (len(pts),)
    gi, gd = _np(g)
    assert np.array_equal(m.cpu().numpy(), ref.outlier_mask(gi, gd.astype(np.float64), 2.0))
    assert not m[-25:].any() and m[:-25].float().mean() > 0.9
    assert bool(outlier_mask(_graph(_uniform(1, 0), 4)).all())  # P = 1: no neighbours, kept


# ---------------------------------------------------------------------------------------------------- GaussianState
def _state(P=3000, C=16, seed=0, **kw):
    from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid

    gen = torch.Generator(device="cuda").manual_seed(seed)
    xyz = torch.from_numpy(clustered(P, seed)).cuda()
    return GaussianState(xyz, torch.rand(P, 1, 3, device="cuda", generator=gen) - 0.5, torch.zeros(P, 3, 3, device="cuda"),
                         inverse_sigmoid(torch.rand(P, 1, device="cuda", generator=gen) * 0.9 + 0.05),
                         torch.log(torch.rand(P, 3, device="cuda", generator=gen) * 0.02 + 0.001),
                         torch.nn.functional.normalize(torch.randn(P, 4, device="cuda", generator=gen), dim=1),
                         torch.randn(P, 1, C, device="cuda", generator=gen), **kw)


def _zero_grads(st):
    """zero gradients w.r.t. the activated tensors, shaped as the ViewBatch's (float32 also for float16 features)"""
    return {k: torch.zeros(v.shape, device=v.device) for k, v in st.act.items()}


LRS = dict(xyz=0.0, f_dc=0.0, f_rest=0.0, opacity=0.0, scaling=0.0, rotation=0.0, semantic_feature=0.01)


@pytest.mark.gpu
def test_graph_cache_is_dropped_when_rows_change():
    st = _state()
    g = st.neighbor_graph(8)
    assert st.neighbor_graph(8) is g and st.neighbor_graph(8, rebuild=True) is not g
    g = st.neighbor_graph(8)
    assert st.neighbor_graph(4) is not g and st.neighbor_graph(4).k == 4
    g = st.neighbor_graph(8)
    keep = torch.ones(st.P, dtype=torch.bool, device="cuda")
    keep[::5] = False
    st.prune(keep)
    assert st._graph is None and st.neighbor_graph(8).P == st.P
    st.neighbor_graph(8)
    vb = st.batch()
    vb.grad_accum.fill_(1.0)
    vb.denom.fill_(1.0)
    st.densify_and_prune(0.5, 0.0, 1.0, False, generator=torch.Generator(device="cuda").manual_seed(0))
    assert st._graph is None
    # relocate_and_add moving dead rows onto live ones but adding none (cap_max = P)
    st.raw["opacity"][:50] = -20.0
    st.neighbor_graph(8)
    n_rel, n_add = st.relocate_and_add(st.P, min_opacity=0.005, generator=torch.Generator(device="cuda").manual_seed(1))
    assert n_rel == 50 and n_add == 0 and st._graph is None
    st.neighbor_graph(8)
    st.quantize_features(8, iters=2, generator=torch.Generator().manual_seed(0))
    assert st._graph is None
    with pytest.raises(ValueError, match="quantised"):
        st.add_feature_tv_grads(0.1, grads=_zero_grads(st))


@pytest.mark.gpu
@pytest.mark.parametrize("feature_dtype", [torch.float32, torch.float16])
def test_add_feature_tv_grads_then_adam_matches_autograd_and_torch_adam(feature_dtype):
    st = _state(P=2000, C=24, seed=3, feature_dtype=feature_dtype)
    g = st.neighbor_graph(8)
    idx = g.idx.long()
    valid = idx >= 0
    rows = torch.arange(st.P, device="cuda")[:, None].expand_as(idx)[valid]
    nbrs = idx[valid]
    scale = 0.5 / (g.n_edges * 24)
    x = st.raw["semantic_feature"].clone().requires_grad_(True)
    opt = torch.optim.Adam([x], lr=LRS["semantic_feature"], betas=st.betas, eps=st.eps)
    for _ in range(3):
        # autograd at the state's features: the two Adam implementations round differently, and a pair of neighbouring
        # features rounded to either side of equality would flip a sign; torch.optim.Adam steps x with that gradient
        y = st.raw["semantic_feature"].clone().requires_grad_(True)
        grads = _zero_grads(st)
        loss = st.add_feature_tv_grads(0.5, k=8, grads=grads)
        st.step(LRS, grads)
        f = y.reshape(st.P, 24)
        want = (f[rows] - f[nbrs]).abs().sum() * scale
        want.backward()
        assert abs(float(loss) - float(want.detach())) <= 1e-5 * abs(float(want.detach()))
        # autograd sums the +-s of a row one at a time, the native count is rounded once (n * s): the two agree to far
        # less than s, so the integer counts are the same
        assert float((grads["semantic_feature"] - y.grad).abs().max()) <= 1e-3 * scale
        # the integer counts times s: autograd's rounding residue where n = 0 would make Adam (eps 1e-15) take a full step
        s32 = torch.tensor(scale, dtype=torch.float32, device="cuda")
        opt.zero_grad()
        x.grad = torch.round(y.grad / s32) * s32
        opt.step()
    assert torch.allclose(st.raw["semantic_feature"], x.detach(), rtol=1e-5, atol=1e-7)
    if feature_dtype == torch.float16:
        assert torch.equal(st.act["semantic_feature"], st.raw["semantic_feature"].half())


@pytest.mark.gpu
def test_remove_outliers_prunes_with_the_adam_state():
    st = _state(P=4000, C=8, seed=9)
    st.raw["xyz"][-10:] = torch.rand(10, 3, device="cuda") + 20.0
    for name in st.NAMES:
        st.exp_avg[name].normal_()
        st.exp_avg_sq[name].uniform_()
    from diff_gaussian_rasterization import outlier_mask

    keep = outlier_mask(st.neighbor_graph(16), 2.0)
    old = {n: (st.raw[n].clone(), st.exp_avg[n].clone(), st.exp_avg_sq[n].clone()) for n in st.NAMES}
    P = st.remove_outliers(16, 2.0)
    assert P == int(keep.sum()) and not keep[-10:].any()
    for n in st.NAMES:
        for a, b in zip((st.raw[n], st.exp_avg[n], st.exp_avg_sq[n]), old[n]):
            assert torch.equal(a, b[keep]), n


# ---------------------------------------------------------------------------------------------------- lift
@pytest.mark.gpu
def test_fill_gives_unseen_gaussians_of_a_lift_their_neighbours_weighted_mean():
    import scenegen
    from diff_gaussian_rasterization import GaussianRasterizationSettings, fill_features
    from diff_gaussian_rasterization.feature_head import FeatureLift

    sc = scenegen.make_scene(P=3000, W=150, H=100, C=8, sh_degree=1, seed=4)
    t = scenegen.to_torch(sc, "cuda")
    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, sc.cameras[0], "cuda"))
    # 300 transparent copies of visible Gaussians: no view blends them, their originals are at distance 0
    n = 300
    means = torch.cat([t["means3D"], t["means3D"][:n]])
    opac = torch.cat([t["opacities"], torch.zeros(n, 1, device="cuda")])
    scales = torch.cat([t["scales"], t["scales"][:n]])
    rots = torch.cat([t["rotations"], t["rotations"][:n]])
    lift = FeatureLift(means, opac, scales, rots, 8)
    lift.add(rs, torch.randn(8, rs.image_height, rs.image_width, device="cuda",
                             generator=torch.Generator(device="cuda").manual_seed(0)))
    feats, w = lift.result()
    assert bool((w[-n:] == 0).all()) and bool((feats[-n:] == 0).all())
    g = _graph(means.cpu().numpy(), 8)
    out = fill_features(feats, w, g)
    assert out.shape == feats.shape
    want = ref.fill(feats.cpu().numpy(), w.cpu().numpy(), _np(g)[0])
    got = out.reshape(len(w), 8).cpu().numpy()
    blank = w.cpu().numpy() <= 0
    has = np.array([(w.cpu().numpy()[j[j >= 0]] > 0).any() for j in _np(g)[0]])
    assert _within_one_ulp(got[blank & has], want[blank & has])
    assert np.array_equal(got[~(blank & has)], feats.reshape(len(w), 8).cpu().numpy()[~(blank & has)])
    assert (blank[-n:] & has[-n:]).mean() > 0.5
