"""Point-cloud initialisation: the native distCUDA2 (f3dgs_knn_mean_dist, csrc/knn.cu), the `simple_knn` drop-in,
GaussianState.from_point_cloud (the reference's create_from_pcd) and io.load_point_cloud (its fetchPly).

The yardstick is a float64 restatement on the float32 inputs: out[i] = mean of the three smallest squared distances to
the points j != i.  The native result is computed in fp32 and must be within 1e-6 of it, relatively."""
import ctypes
import os

import numpy as np
import pytest
import torch

FLT_MAX = np.finfo(np.float32).max
C0 = 0.28209479177387814


# ---------------------------------------------------------------------------------------------------- restatements
def _finish(best):
    """best [P,3] ascending float64 squared distances, +inf where a neighbour is missing -> the reference's result:
    the float64 mean when all three exist, else the fp32 sum with FLT_MAX for the missing ones (as simple-knn does)."""
    out = np.empty(best.shape[0], np.float64)
    for i, b in enumerate(best):
        if np.isfinite(b).all():
            out[i] = b.mean()
        else:
            f = np.where(np.isfinite(b), b, FLT_MAX).astype(np.float32)
            with np.errstate(over="ignore"):  # FLT_MAX + FLT_MAX = inf, as on the GPU
                out[i] = (f[0] + f[1] + f[2]) / np.float32(3)
    return out


def brute_force(pts):
    """float64 restatement over all pairs (small clouds)."""
    p = np.asarray(pts, np.float32).astype(np.float64)
    P = p.shape[0]
    best = np.full((P, 3), np.inf)
    for s in range(0, P, 2048):
        d = ((p[s:s + 2048, None, :] - p[None, :, :]) ** 2).sum(-1)
        d[np.arange(d.shape[0]), np.arange(s, s + d.shape[0])] = np.inf  # exclusion by index
        k = min(3, P - 1) if P > 1 else 0
        if k:
            part = np.sort(np.partition(d, k - 1, axis=1)[:, :k], axis=1)
            best[s:s + 2048, :k] = part
    return _finish(best)


def kdtree(pts):
    """The same quantity from scipy's cKDTree: query k = 4 and drop the query's own index (with duplicates it need not
    come first), else the fourth entry."""
    from scipy.spatial import cKDTree

    p = np.asarray(pts, np.float32).astype(np.float64)
    P = p.shape[0]
    dist, idx = cKDTree(p).query(p, k=4, workers=-1)
    own = idx == np.arange(P)[:, None]
    drop = np.where(own.any(1), own.argmax(1), 3)
    keep = np.ones_like(own)
    keep[np.arange(P), drop] = False
    best = (dist[keep].reshape(P, 3)) ** 2
    return _finish(np.sort(best, axis=1))


def clustered(P, seed, n_clusters=64, radius=0.01, outlier_frac=0.001):
    """Gaussian clusters of the given radius in [-1,1]^3, plus a fraction of far outliers at 100x the radius."""
    rng = np.random.default_rng(seed)
    centers = rng.uniform(-1, 1, (n_clusters, 3))
    n_out = int(P * outlier_frac)
    pts = centers[rng.integers(0, n_clusters, P - n_out)] + rng.normal(0, radius, (P - n_out, 3))
    d = rng.normal(size=(n_out, 3))
    far = centers[rng.integers(0, n_clusters, n_out)] + 100 * radius * d / np.linalg.norm(d, axis=1, keepdims=True)
    return rng.permutation(np.concatenate([pts, far])).astype(np.float32)


def small_clouds():
    rng = np.random.default_rng(7)
    dup = rng.uniform(-1, 1, (40, 3)).astype(np.float32)
    clouds = {f"P{P}": rng.uniform(-1, 1, (P, 3)).astype(np.float32) for P in (1, 2, 3, 4)}
    clouds["uniform300"] = rng.uniform(-1.3, 1.3, (300, 3)).astype(np.float32)
    clouds["duplicates"] = np.concatenate([dup, dup[:20], dup[:5], dup[:2]])
    clouds["identical"] = np.ones((9, 3), np.float32)
    clouds["pair_dup4"] = np.array([[0, 0, 0]] * 2 + [[1, 2, 3]] * 2, np.float32)
    return clouds


# ---------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", list(small_clouds()))
def test_restatement_matches_kdtree(name):
    pts = small_clouds()[name]
    a, b = brute_force(pts), kdtree(pts)
    fin = np.isfinite(a)
    assert np.array_equal(fin, np.isfinite(b))
    assert np.allclose(a[fin], b[fin], rtol=1e-12, atol=0)
    if len(pts) <= 2:
        assert np.isinf(a).all()
    if len(pts) == 3:
        assert np.all(a == np.float32(FLT_MAX) / np.float32(3))


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_knn_scratch_bytes.restype = ctypes.c_size_t
    L.f3dgs_knn_scratch_bytes.argtypes = [ctypes.c_int]
    L.f3dgs_knn_mean_dist.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    L.f3dgs_launch_count.restype = ctypes.c_ulonglong
    return L


def test_cabi_rejects_bad_arguments_before_touching_cuda(lib):
    f = lib.f3dgs_knn_mean_dist
    n0 = lib.f3dgs_launch_count()
    pts, out, scr = 0x100000, 0x900000, 0x2000000  # never dereferenced: every call below is rejected first
    assert f(-1, pts, out, scr, None) == -1 and b"P < 0" in lib.f3dgs_last_error()
    assert f(0, None, None, None, None) == 0  # empty cloud: nothing to do
    for args in ((None, out, scr), (pts, None, scr), (pts, out, None)):
        assert f(10, *args, None) == -1 and b"NULL" in lib.f3dgs_last_error()
    assert f(10, pts, pts + 8, scr, None) == -1 and b"overlaps" in lib.f3dgs_last_error()  # inside points [P,3]
    assert f(10, pts, pts - 16, scr, None) == -1  # out [P] runs into points
    assert f(10, pts, scr, scr, None) == -1 and b"overlaps" in lib.f3dgs_last_error()
    assert f(100000, pts, scr + 4096, scr, None) == -1  # out inside the scratch
    assert lib.f3dgs_knn_scratch_bytes(0) == 0 and lib.f3dgs_knn_scratch_bytes(-3) == 0
    assert lib.f3dgs_launch_count() == n0


def test_load_point_cloud_reads_a_colmap_points3d_ply(tmp_path):
    from diff_gaussian_rasterization import io

    rng = np.random.default_rng(3)
    P = 57
    dt = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                   ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    v = np.empty(P, dt)
    xyz, nrm = rng.normal(size=(P, 3)).astype(np.float32), rng.normal(size=(P, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (P, 3)).astype(np.uint8)
    for i, n in enumerate("xyz"):
        v[n], v["n" + n] = xyz[:, i], nrm[:, i]
    for i, n in enumerate(("red", "green", "blue")):
        v[n] = rgb[:, i]
    header = ["ply", "format binary_little_endian 1.0", f"element vertex {P}"]
    header += [f"property float {n}" for n in ("x", "y", "z", "nx", "ny", "nz")]
    header += [f"property uchar {n}" for n in ("red", "green", "blue")] + ["end_header"]
    path = tmp_path / "points3D.ply"
    path.write_bytes(("\n".join(header) + "\n").encode("ascii") + v.tobytes())
    points, colors, normals = io.load_point_cloud(str(path))
    assert points.dtype == np.float32 and np.array_equal(points, xyz)
    assert normals.dtype == np.float32 and np.array_equal(normals, nrm)
    assert colors.dtype == np.float64 and np.array_equal(colors, rgb / 255.0)


def test_simple_knn_dropin_imports_and_rejects_cpu_input(built):
    from simple_knn._C import distCUDA2

    with pytest.raises(RuntimeError, match="must be a CUDA tensor \\(this build has no CPU path\\)"):
        distCUDA2(torch.zeros(5, 3))


# ---------------------------------------------------------------------------------------------------- GPU
def _dist(pts):
    from simple_knn._C import distCUDA2

    return distCUDA2(torch.from_numpy(np.ascontiguousarray(pts)).cuda()).cpu().numpy()


def _check(out, ref):
    assert out.dtype == np.float32 and out.shape == ref.shape
    fin = np.isfinite(ref)
    assert np.array_equal(np.isfinite(out), fin)
    assert np.array_equal(out[~fin], ref[~fin].astype(np.float32))
    err = np.abs(out[fin].astype(np.float64) - ref[fin])
    assert np.all(err <= 1e-6 * ref[fin]), (err.max(), int(np.argmax(err - 1e-6 * ref[fin])))


def _uniform(P, seed=0, a=1.3):
    return np.random.default_rng(seed).uniform(-a, a, (P, 3)).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1000, 4097, 30000, 200000, 1000000])
def test_uniform_is_exact(P):
    pts = _uniform(P, seed=P)
    _check(_dist(pts), brute_force(pts) if P <= 4097 else kdtree(pts))


@pytest.mark.gpu
@pytest.mark.parametrize("P", [20000, 300000])
def test_clustered_with_outliers_is_exact(P):
    pts = clustered(P, seed=P)
    _check(_dist(pts), kdtree(pts))


@pytest.mark.gpu
def test_degenerate_clouds():
    rng = np.random.default_rng(11)
    identical = np.full((5000, 3), 0.25, np.float32)
    assert np.all(_dist(identical) == 0)
    planar = rng.uniform(-1, 1, (20000, 3)).astype(np.float32)
    planar[:, 2] = 0.5
    _check(_dist(planar), kdtree(planar))
    t = rng.uniform(-1, 1, (20000, 1))
    collinear = (np.array([[0.3, -0.2, 0.9]]) * t + np.array([[1.0, 2.0, 3.0]])).astype(np.float32)
    _check(_dist(collinear), kdtree(collinear))
    axis = np.zeros((3000, 3), np.float32)  # zero extent on two axes
    axis[:, 1] = rng.uniform(-5, 5, 3000)
    _check(_dist(axis), brute_force(axis))
    grid = np.stack(np.meshgrid(*[np.arange(12, dtype=np.float32)] * 3, indexing="ij"), -1).reshape(-1, 3)
    _check(_dist(grid), brute_force(grid))  # many exact ties


@pytest.mark.gpu
def test_three_coincident_neighbours_give_exactly_zero():
    rng = np.random.default_rng(5)
    base = rng.uniform(-1, 1, (2500, 3)).astype(np.float32)
    pts = np.concatenate([base, base[:1000], base[:1000], base[:1000]])  # the first 1000 points appear four times
    out = _dist(pts)
    quad = np.zeros(len(pts), bool)
    quad[:1000] = quad[2500:] = True
    assert np.all(out[quad] == 0)
    _check(out, kdtree(pts))


@pytest.mark.gpu
@pytest.mark.parametrize("P", [0, 1, 2, 3, 4])
def test_tiny_clouds(P):
    pts = _uniform(P, seed=40 + P)
    out = _dist(pts)
    assert out.shape == (P,)
    ref = brute_force(pts)
    _check(out, ref)
    if P in (1, 2):
        assert np.isposinf(out).all()
    if P == 3:  # (d0 + d1 + FLT_MAX) / 3 in fp32
        assert np.array_equal(out, ref.astype(np.float32))


@pytest.mark.gpu
def test_bitwise_reproducible_and_order_independent():
    pts = clustered(150000, seed=9)
    a, b = _dist(pts), _dist(pts)
    assert np.array_equal(a, b)
    perm = np.random.default_rng(1).permutation(len(pts))
    assert np.array_equal(_dist(pts[perm]), a[perm])


@pytest.mark.gpu
def test_non_contiguous_input():
    from simple_knn._C import distCUDA2

    pts = torch.from_numpy(_uniform(10000, seed=2)).cuda()
    wide = torch.zeros(10000, 5, device="cuda")
    wide[:, 1:4] = pts
    t = pts.t().contiguous().t()
    assert not wide[:, 1:4].is_contiguous() and not t.is_contiguous()
    ref = distCUDA2(pts)
    assert torch.equal(distCUDA2(wide[:, 1:4]), ref) and torch.equal(distCUDA2(t), ref)


@pytest.mark.gpu
def test_binding_rejects_bad_shapes():
    from simple_knn._C import distCUDA2

    for bad in (torch.zeros(4, 2, device="cuda"), torch.zeros(4, 3, device="cuda", dtype=torch.float64),
                torch.zeros(4, 3, 1, device="cuda")):
        with pytest.raises(RuntimeError, match="float32 tensor \\[P,3\\]"):
            distCUDA2(bad)


@pytest.mark.gpu
def test_against_reference_build():
    import ref_knn

    ref = ref_knn.load()
    if ref is None:
        pytest.skip("no reference simple-knn checkout to build")
    cases = [_uniform(P, seed=60 + P) for P in (1, 2, 3, 4, 1000)] + [_uniform(100000, seed=3), clustered(200000, 4)]
    bitwise = True
    for pts in cases:
        x = torch.from_numpy(pts).cuda()
        ours, theirs = _dist(pts), ref.distCUDA2(x).cpu().numpy()
        fin = np.isfinite(theirs)
        assert np.array_equal(np.isfinite(ours), fin)
        if len(pts) <= 3:
            assert np.array_equal(ours, theirs)
        assert np.all(np.abs(ours[fin].astype(np.float64) - theirs[fin]) <= 1e-6 * np.abs(theirs[fin]))
        bitwise &= np.array_equal(ours, theirs)
    print("bitwise equal to the reference build:", bitwise)


# ---------------------------------------------------------------------------------------------------- from_point_cloud
def create_from_pcd(points, colors, semantic_feature_size, speedup, max_sh_degree=3):
    """Restatement of the reference's create_from_pcd (scene/gaussian_model.py:133-160) with `dist2` left to the caller."""
    fused_point_cloud = torch.tensor(np.asarray(points)).float().cuda()
    fused_color = (torch.tensor(np.asarray(colors)).float().cuda() - 0.5) / C0
    features = torch.zeros((fused_color.shape[0], 3, (max_sh_degree + 1) ** 2)).float().cuda()
    features[:, :3, 0] = fused_color
    features[:, 3:, 1:] = 0.0
    if speedup:
        semantic_feature_size = int(semantic_feature_size / 4)
    semantic_feature = torch.zeros(fused_point_cloud.shape[0], semantic_feature_size, 1).float().cuda()
    rots = torch.zeros((fused_point_cloud.shape[0], 4), device="cuda")
    rots[:, 0] = 1
    x = 0.1 * torch.ones((fused_point_cloud.shape[0], 1), dtype=torch.float, device="cuda")
    opacities = torch.log(x / (1 - x))
    return dict(xyz=fused_point_cloud, f_dc=features[:, :, 0:1].transpose(1, 2).contiguous(),
                f_rest=features[:, :, 1:].transpose(1, 2).contiguous(), rotation=rots, opacity=opacities,
                semantic_feature=semantic_feature.transpose(1, 2).contiguous())


@pytest.mark.gpu
@pytest.mark.parametrize("speedup", [False, True])
def test_from_point_cloud_matches_create_from_pcd(speedup):
    from diff_gaussian_rasterization.trainer import GaussianState

    rng = np.random.default_rng(21)
    points = rng.uniform(-1.3, 1.3, (5000, 3))  # float64, as fetchPly / the synthetic init hand them over
    colors = rng.integers(0, 256, (5000, 3)) / 255.0
    st = GaussianState.from_point_cloud(points, colors, 512, speedup=speedup)
    ref = create_from_pcd(points, colors, 512, speedup)
    for k, v in ref.items():
        assert st.raw[k].shape == v.shape and st.raw[k].dtype == v.dtype, k
        assert torch.equal(st.raw[k], v), k
    assert st.raw["semantic_feature"].shape == (5000, 1, 128 if speedup else 512)
    d = kdtree(points.astype(np.float32))
    want = np.log(np.sqrt(np.maximum(d, 1e-7)))
    s = st.raw["scaling"].cpu().numpy()
    assert s.shape == (5000, 3) and np.array_equal(s[:, 0], s[:, 1]) and np.array_equal(s[:, 0], s[:, 2])
    # |d err| <= 1e-6 d  ->  |log sqrt d err| <= 5e-7, plus the fp32 rounding of log and sqrt
    assert np.all(np.abs(s[:, 0] - want) <= 6e-7 + 2.4e-7 * np.abs(want))


@pytest.mark.gpu
def test_from_point_cloud_rejects_bad_input():
    from diff_gaussian_rasterization.trainer import GaussianState

    pts = np.zeros((10, 3))
    with pytest.raises(ValueError):
        GaussianState.from_point_cloud(pts, np.zeros((9, 3)), 16)
    with pytest.raises(ValueError):
        GaussianState.from_point_cloud(np.zeros((10, 2)), np.zeros((10, 2)), 16)
    bad = pts.copy()
    bad[3, 1] = np.nan
    with pytest.raises(ValueError):
        GaussianState.from_point_cloud(bad, np.zeros((10, 3)), 16)
    bad[3, 1] = np.inf
    with pytest.raises(ValueError):
        GaussianState.from_point_cloud(bad, np.zeros((10, 3)), 16)


@pytest.mark.gpu
def test_training_from_a_point_cloud_end_to_end():
    """A state built from the `small` scene's means and SH-DC colours trains: six steps of activate -> ViewBatch ->
    photometric + feature L1 loss and gradient -> fused Adam lower the loss against targets rendered from that scene."""
    import scenegen
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    from diff_gaussian_rasterization import feature_head as fh
    from diff_gaussian_rasterization.image_loss import photometric_loss_and_grad
    from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid

    sc = scenegen.make_config("small", views=2)
    dev = "cuda"
    t = scenegen.to_torch(sc, dev)
    colors = np.clip(sc.shs[:, 0, :] * C0 + 0.5, 0.0, 1.0)  # SH2RGB of the DC term
    settings = [GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev)) for cam in sc.cameras]

    src = GaussianState(t["means3D"].clone(), t["shs"][:, :1].contiguous(), t["shs"][:, 1:].contiguous(),
                        inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                        t["rotations"].clone(), t["semantic_feature"].clone())
    src.activate()
    vb = src.batch()
    vb.zero_()
    gt_color = [vb.forward(rs)[0].clone() for rs in settings]
    gt_feat = [torch.rand(sc.C, 40, 56, device=dev, generator=torch.Generator(device=dev).manual_seed(v))
               for v in range(len(settings))]

    st = GaussianState.from_point_cloud(sc.means3D, colors, sc.C, max_sh_degree=sc.sh_degree)
    assert st.P == sc.P and st.raw["semantic_feature"].shape == (sc.P, 1, sc.C)
    lrs = dict(xyz=0.0, f_dc=0.02, f_rest=0.0, opacity=0.05, scaling=0.005, rotation=0.001, semantic_feature=0.05)
    losses = []
    for it in range(6):
        st.activate()
        vb = st.batch()
        vb.zero_()
        total = torch.zeros((), device=dev)
        for v, rs in enumerate(settings):
            color, feat, radii, depth, ctx = vb.forward(rs)
            lc, gcolor = photometric_loss_and_grad(color, gt_color[v], 0.2)
            lf, gfeat = fh.feature_l1_loss_and_grad(feat, gt_feat[v], 1.0)
            vb.backward(ctx, gcolor, gfeat, torch.zeros_like(depth), last=(v == len(settings) - 1))
            total = total + lc + lf
        vb.all_reduce()
        st.step(lrs)
        losses.append(float(total))
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
