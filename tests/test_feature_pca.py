"""PCA picture of a feature map (csrc/feature_pca.cu, feature_head.pca_fit / pca_image): render.py's
feature_visualize_saving on the device.

CPU part (`-m "not gpu"`): `pca64`, a float64 NumPy restatement of the contract, is pinned against the reference function
verbatim (scikit-learn PCA(3)) on several shapes, and the device-side float64 restatement `pca64_torch` against `pca64`;
the sign rule and the percentile rule against np.percentile; the C ABI and the Python functions reject bad arguments
before touching CUDA.

GPU part (`-m gpu`): the native path against `pca64_torch` with bars that follow from float32 rounding, u = 2^-24:
  - xh = x * (1 / max(||x||, 1e-12)), ||x||^2 summed in fp32 as 8 partial sums of C/8 terms and then 8 terms, a sqrt, a
    reciprocal and a product: |xh - xh64| <= rx |xh64|, rx = (C/8 + 12) u.
  - mean: tiles of 32 samples summed in fp32, the rest in fp64, rounded to fp32: |dmu| <= (rx + 34 u) mean|xh| + u |mu|.
  - centred sample a = fma(x, inv, -mu): |da| <= rx |xh| + |dmu| + u |a|.
  - cov: fp32 FMA sums over blocks of 2048 samples (a block sum carries at most 2049 u of sum |a_i a_j|), fp64 beyond:
    |dcov| <= (M + M^T + 2050 u |A| |A|^T) / (n - 1), M = |dA| |A|^T, elementwise.
  - components: Davis-Kahan, with e = ||dcov||_F (plus 1e-12 ||cov|| for the fp64 eigensolver) and gap_k the distance of
    lambda_k to its neighbours: ||c_k - c64_k|| <= 2 e / (gap_k - e) + 2 u (rounding to fp32); a component whose gap does
    not exceed 4 e is not unique at this precision and is not compared (nor its image channel).
  - t = c_k . a_p summed as 8 partial sums and 8 terms: |dt| <= ||dc_k|| ||a_p|| + sum |c_k| |da_p| + (C/8 + 10) u sum |c_k| |a_p|.
  - lo, hi: an order statistic moves by at most max |dt| over the samples; interpolation and rounding add 4 u max(|lo|, |hi|).
  - image: v = (t - lo) / (hi - lo) with the errors above, |dv| <= (|dt| + |dlo|) / w + |t - lo| (|dlo| + |dhi|) / w^2 + 2 u,
    w = hi - lo - |dlo| - |dhi| (clamping is 1-Lipschitz).
Exact properties: float16 x gives bitwise the result of x.float(); only the pixels p % 3 == 0 enter the fit; [C,N] is
bitwise the rows of [C,H,W]; two calls are bitwise identical; no buffer of C x n floats is allocated.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

U = 2.0 ** -24


def _sign_rule(comps):
    """scikit-learn's svd_flip(u_based_decision=False): each row's first entry of largest |value| is positive."""
    idx = np.argmax(np.abs(comps), axis=1)
    return comps * np.sign(comps[np.arange(comps.shape[0]), idx])[:, None]


def _percentile_linear(v, q):
    """np.percentile(v, q) with the linear method, written out: h = (m - 1) q / 100, v_j + (h - j)(v_{j+1} - v_j)."""
    s = np.sort(np.asarray(v, np.float64).ravel())
    h = (s.size - 1) * q / 100.0
    j = int(np.floor(h))
    j1 = min(j + 1, s.size - 1)
    return s[j] + (h - j) * (s[j1] - s[j])


def pca64(x):
    """float64 restatement of the contract: x [C,H,W] or [C,N] -> dict(mean, cov, lam (descending), components [3,C],
    lo, hi, image [...,3])."""
    x = np.asarray(x, np.float64)
    C = x.shape[0]
    X = x.reshape(C, -1)
    xh = X / np.maximum(np.sqrt((X * X).sum(0)), 1e-12)
    S = xh[:, ::3]
    n = S.shape[1]
    mu = S.mean(1)
    A = S - mu[:, None]
    cov = A @ A.T / (n - 1)
    lam, V = np.linalg.eigh(cov)
    comps = _sign_rule(V[:, ::-1][:, :3].T.copy())
    lo, hi = np.percentile(comps @ A, [1, 99])
    with np.errstate(divide="ignore", invalid="ignore"):
        img = np.clip((comps @ (xh - mu[:, None]) - lo) / (hi - lo), 0.0, 1.0)
    return dict(mean=mu, cov=cov, lam=lam[::-1].copy(), components=comps, lo=lo, hi=hi,
                image=img.T.reshape(x.shape[1:] + (3,)))


def pca64_torch(x):
    """pca64 on torch float64 tensors of any device (the GPU tests run it next to the kernels); also returns the
    normalised map xh [C,N] and the centred samples A [C,n] the bars are computed from."""
    C = x.shape[0]
    X = x.reshape(C, -1).double()
    xh = X / X.norm(dim=0).clamp_min(1e-12)
    S = xh[:, ::3]
    n = S.shape[1]
    mu = S.mean(1)
    A = S - mu[:, None]
    cov = A @ A.t() / (n - 1)
    lam, V = torch.linalg.eigh(cov)
    comps = V.flip(1)[:, :3].t()
    first = comps.abs().argmax(dim=1, keepdim=True)
    comps = comps * torch.sign(comps.gather(1, first))
    t = comps @ A
    lo, hi = torch.quantile(t.flatten().cpu(), torch.tensor([0.01, 0.99], dtype=torch.float64)).tolist()
    img = ((comps @ (xh - mu[:, None]) - lo) / (hi - lo)).clamp(0, 1)
    return dict(mean=mu, cov=cov, lam=lam.flip(0), components=comps, lo=lo, hi=hi,
                image=img.t().reshape(tuple(x.shape[1:]) + (3,)), xh=xh, A=A)


def reference_visualize(feature):
    """render.py's feature_visualize_saving as written (SURVEY section 3.2), on CPU float32 tensors."""
    import sklearn.decomposition

    C = feature.shape[0]
    fmap = F.normalize(feature[None], dim=1)
    f_samples = fmap.permute(0, 2, 3, 1).reshape(-1, C)[::3].numpy()
    pca = sklearn.decomposition.PCA(3)
    transformed = pca.fit_transform(f_samples)
    mean, comps = torch.tensor(f_samples.mean(0)), torch.tensor(pca.components_)
    q1, q99 = np.percentile(transformed, [1, 99])
    vis = ((fmap.permute(0, 2, 3, 1).reshape(-1, C) - mean) @ comps.T - q1) / (q99 - q1)
    return vis.clamp(0, 1).reshape(feature.shape[1], feature.shape[2], 3), mean.numpy(), pca.components_, (q1, q99)


def synthetic(C, H, W, seed, offset=8.0, noise=0.05):
    """A rank-3 signal with scales 3 / 2 / 1.2 along random orthonormal directions, isotropic noise and a large common
    offset along a random unit vector: a clearly separated top-3 spectrum, and centring that matters.  float32 [C,H,W]."""
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((C, 3)))
    o = rng.standard_normal(C)
    o /= np.linalg.norm(o)
    z = rng.standard_normal((3, H * W)) * np.array([3.0, 2.0, 1.2])[:, None]
    x = offset * o[:, None] + Q @ z + noise * rng.standard_normal((C, H * W))
    return x.reshape(C, H, W).astype(np.float32)


def _clear_components(lam, err):
    """Indices k < 3 whose eigenvalue is separated from its neighbours by more than 4 err."""
    out = []
    for k in range(3):
        gaps = [lam[k - 1] - lam[k]] if k > 0 else []
        if k + 1 < len(lam):
            gaps.append(lam[k] - lam[k + 1])
        if min(gaps) > 4 * err:
            out.append(k)
    return out


SHAPES_CPU = [(16, 1, 7), (3, 3, 5), (64, 90, 161), (8, 7, 13), (32, 1, 100)]  # (C, H, W): n = 3 and N % 3 != 0


@pytest.mark.parametrize("C,H,W", SHAPES_CPU)
def test_restatement_matches_reference_function(C, H, W):
    pytest.importorskip("sklearn")
    x = synthetic(C, H, W, seed=C + H)
    vis, mean, comps, (q1, q99) = reference_visualize(torch.from_numpy(x))
    r = pca64(x)
    keep = _clear_components(r["lam"], 1e-6 * r["lam"][0])
    assert keep[:2] == [0, 1] or len(keep) == 3, keep
    assert np.abs(r["mean"] - mean).max() < 1e-6
    for k in keep:
        assert np.abs(r["components"][k] - comps[k]).max() < 1e-4, k
    if len(keep) == 3:  # lo / hi mix all three components
        assert abs(r["lo"] - q1) < 1e-5 and abs(r["hi"] - q99) < 1e-5
        assert np.abs(r["image"] - vis.numpy()).max() < 1e-4


@pytest.mark.parametrize("C,H,W", SHAPES_CPU[:3])
def test_torch_restatement_matches_numpy(C, H, W):
    x = synthetic(C, H, W, seed=7)
    a, b = pca64(x), pca64_torch(torch.from_numpy(x))
    keep = _clear_components(a["lam"], 1e-9 * a["lam"][0])
    for key in ("mean", "cov", "lam"):
        assert np.allclose(a[key], b[key].numpy(), rtol=0, atol=1e-12), key
    for k in keep:
        assert np.allclose(a["components"][k], b["components"][k].numpy(), rtol=0, atol=1e-10)
    if len(keep) == 3:
        assert abs(a["lo"] - b["lo"]) < 1e-12 and abs(a["hi"] - b["hi"]) < 1e-12
        assert np.allclose(a["image"], b["image"].numpy(), rtol=0, atol=1e-10)


def test_sign_rule_and_percentile_rule():
    c = np.array([[0.1, -0.7, 0.7, 0.0], [0.5, 0.2, -0.5, 0.1], [-0.2, 0.3, 0.1, -0.9]])
    s = _sign_rule(c)
    assert s[0].tolist() == (-c[0]).tolist()    # -0.7 comes first among the |0.7| ties
    assert s[1].tolist() == c[1].tolist()       # 0.5 first
    assert s[2].tolist() == (-c[2]).tolist()
    rng = np.random.default_rng(3)
    for m in (9, 10, 101, 1000, 3001):
        v = rng.standard_normal(m).astype(np.float32)
        for q in (1, 99):
            assert abs(_percentile_linear(v, q) - np.percentile(v.astype(np.float64), q)) < 1e-12


# ---- C ABI argument validation (no CUDA call is made for rejected arguments)
@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_feature_pca_scratch_bytes.restype = ctypes.c_size_t
    L.f3dgs_feature_pca_scratch_bytes.argtypes = [ctypes.c_int, ctypes.c_int]
    for h in ("", "_f16x"):
        getattr(L, "f3dgs_feature_pca_moments" + h).argtypes = [ctypes.c_int] * 2 + [ctypes.c_void_p] * 5
        getattr(L, "f3dgs_feature_pca_range" + h).argtypes = [ctypes.c_int] * 2 + [ctypes.c_void_p] * 6
        getattr(L, "f3dgs_feature_pca_image" + h).argtypes = [ctypes.c_int] * 2 + [ctypes.c_void_p] * 6
    return L


def test_abi_rejects_bad_arguments_before_touching_cuda(lib):
    x, sc, mu, cov, cp, rg, img = (k << 32 for k in range(1, 8))  # never dereferenced: validation fails first
    C, N = 16, 1000

    def call(fn, half, *args):
        return getattr(lib, "f3dgs_feature_pca_" + fn + ("_f16x" if half else ""))(*args, None)

    def bad(msg, fn, *args, half=False):
        assert call(fn, half, *args) == -1, (fn, args)
        assert msg in lib.f3dgs_last_error(), (fn, args, lib.f3dgs_last_error())

    for c, n in ((2, N), (1025, N), (C, 6), (C, -1), (0, 0)):
        assert lib.f3dgs_feature_pca_scratch_bytes(c, n) == 0
        for half in (False, True):
            bad(b"bad sizes", "moments", c, n, x, sc, mu, cov, half=half)
            bad(b"bad sizes", "range", c, n, x, mu, cp, sc, rg, half=half)
            bad(b"bad sizes", "image", c, n, x, mu, cp, rg, img, half=half)
    for half in (False, True):
        es = 2 if half else 4
        for i in range(4):
            a = [x, sc, mu, cov]
            a[i] = None
            bad(b"NULL pointer", "moments", C, N, *a, half=half)
        for i in range(5):
            a = [x, mu, cp, sc, rg]
            a[i] = None
            bad(b"NULL pointer", "range", C, N, *a, half=half)
            a = [x, mu, cp, rg, img]
            a[i] = None
            bad(b"NULL pointer", "image", C, N, *a, half=half)
        last_x = x + es * C * N - 4
        bad(b"must not overlap", "moments", C, N, x, last_x, mu, cov, half=half)       # scratch starts in x
        bad(b"must not overlap", "moments", C, N, x, sc, last_x, cov, half=half)       # mean in x
        bad(b"must not overlap", "moments", C, N, x, sc, mu, sc + 8, half=half)        # cov in scratch
        bad(b"must not overlap", "moments", C, N, x, sc, mu, mu + 4 * C - 8, half=half)  # cov's start is mean's end
        bad(b"overlaps an input", "range", C, N, x, mu, cp, sc, last_x, half=half)
        bad(b"overlaps an input", "range", C, N, x, mu, cp, sc, cp + 4 * 3 * C - 4, half=half)
        bad(b"overlaps an input", "range", C, N, x, mu, cp, mu + 4, rg, half=half)     # scratch on mean
        bad(b"overlaps an input", "image", C, N, x, mu, cp, rg, last_x, half=half)
        bad(b"overlaps an input", "image", C, N, x, mu, cp, rg, rg - 12 * N + 4, half=half)  # image ends in range
        bad(b"overlaps an input", "image", C, N, x, mu, cp, rg, mu - 12 * N + 4, half=half)


def test_python_functions_reject_bad_arguments():
    from diff_gaussian_rasterization import feature_head as fh

    cases = [(torch.randn(16, 4, 5, 2), "C,H,W"), (torch.randn(16), "C,H,W"), (torch.randn(16, 8, 8).double(), "float32"),
             (torch.randn(2, 8, 8), "3 <= C"), (torch.randn(1025, 2, 4), "3 <= C"), (torch.randn(16, 2, 3), "samples"),
             (torch.randn(16, 6), "samples"), (torch.randn(16, 8, 8), "CUDA"), (torch.randn(16, 8, 8).half(), "CUDA")]
    for x, msg in cases:
        for f in (fh.pca_fit, fh.pca_image):
            with pytest.raises(ValueError, match=msg):
                f(x)
    fit = fh.FeaturePCA(torch.zeros(8), torch.zeros(3, 8), torch.tensor(0.0), torch.tensor(1.0))
    with pytest.raises(ValueError, match="channels"):
        fh.pca_image(torch.randn(16, 8, 8), fit)


# =================================================================================================== GPU
def _native(x):
    from diff_gaussian_rasterization import feature_head as fh
    from diff_gaussian_rasterization import _C

    mean, cov = _C.feature_pca_moments(x)
    fit = fh.pca_fit(x)
    return dict(mean=mean, cov=cov, fit=fit, image=fh.pca_image(x, fit))


def _bars(r, C):
    """Per-quantity bars of the module docstring, from the float64 restatement r (pca64_torch on the device)."""
    xh, A = r["xh"], r["A"]
    n = A.shape[1]
    rx = (C / 8 + 12) * U
    bmu = (rx + 34 * U) * xh[:, ::3].abs().mean(1) + U * r["mean"].abs()
    dA = rx * xh[:, ::3].abs() + bmu[:, None] + U * A.abs()
    M = dA @ A.abs().t()
    dcov = (M + M.t() + 2050 * U * (A.abs() @ A.abs().t())) / (n - 1)
    err = float(dcov.norm()) + 1e-12 * float(r["cov"].norm())
    lam = r["lam"].tolist()
    keep = _clear_components(lam, err)
    dc = torch.zeros(3, dtype=torch.float64, device=A.device)
    for k in keep:
        gaps = ([lam[k - 1] - lam[k]] if k > 0 else []) + ([lam[k] - lam[k + 1]] if k + 1 < len(lam) else [])
        dc[k] = 2 * err / (min(gaps) - err) + 2 * U
    a_all = xh - r["mean"][:, None]
    da_all = rx * xh.abs() + bmu[:, None] + U * a_all.abs()
    ca = r["components"].abs()
    dt = dc[:, None] * a_all.norm(dim=0)[None] + ca @ da_all + (C / 8 + 10) * U * (ca @ a_all.abs())  # [3, N]
    dlh = float(dt[:, ::3][keep].max()) + 4 * U * max(abs(r["lo"]), abs(r["hi"]))
    return dict(dcov=dcov, dmu=bmu, dc=dc, keep=keep, dt=dt, dlh=dlh)


def _image_bar(t64, lo, hi, dt, dlh):
    w = hi - lo - 2 * dlh
    assert w > 0
    return (dt + dlh) / w + (t64 - lo).abs() * 2 * dlh / w ** 2 + 2 * U


def _check_against_pca64(x):
    C = x.shape[0]
    r = pca64_torch(x.float())
    b = _bars(r, C)
    got = _native(x)
    assert bool(((got["mean"].double() - r["mean"]).abs() <= b["dmu"]).all())
    assert bool(((got["cov"] - r["cov"]).abs() <= b["dcov"]).all())
    assert torch.equal(got["cov"], got["cov"].t())
    fit = got["fit"]
    for k in b["keep"]:
        assert float((fit.components[k].double() - r["components"][k]).norm()) <= float(b["dc"][k]), k
    if len(b["keep"]) < 3:  # lo / hi and every image channel depend on all three components
        return b["keep"]
    assert abs(float(fit.lo) - r["lo"]) <= b["dlh"] and abs(float(fit.hi) - r["hi"]) <= b["dlh"]
    t64 = r["components"] @ (r["xh"] - r["mean"][:, None])
    bar = _image_bar(t64, r["lo"], r["hi"], b["dt"], b["dlh"]).t().reshape(r["image"].shape)
    assert bool(((got["image"].double() - r["image"]).abs() <= bar).all())
    return b["keep"]


GPU_SHAPES = [(1, 7), (7, 13), (37, 61), (540, 960)]


@pytest.mark.gpu
@pytest.mark.parametrize("C", [3, 16, 128, 512])
@pytest.mark.parametrize("H,W", GPU_SHAPES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_parity_with_float64(C, H, W, dtype):
    x = torch.from_numpy(synthetic(C, H, W, seed=C * 7 + H)).cuda().to(dtype)
    keep = _check_against_pca64(x)
    if H * W >= 37 * 61 and C > 3:
        assert keep == [0, 1, 2]


@pytest.mark.gpu
@pytest.mark.parametrize("C", [16, 512])
def test_half_input_is_bitwise_its_float_upcast(C):
    xh = torch.from_numpy(synthetic(C, 91, 67, seed=5)).cuda().half()
    a, b = _native(xh), _native(xh.float())
    for k in ("mean", "cov", "image"):
        assert torch.equal(a[k], b[k]), k
    for u, v in zip(a["fit"], b["fit"]):
        assert torch.equal(u, v)


@pytest.mark.gpu
def test_only_every_third_pixel_enters_the_fit():
    x = torch.from_numpy(synthetic(64, 45, 77, seed=9)).cuda()
    y = x.clone().view(64, -1)
    off = torch.arange(y.shape[1], device="cuda") % 3 != 0
    y[:, off] = torch.randn(64, int(off.sum()), device="cuda") * 5
    y = y.view_as(x)
    a, b = _native(x), _native(y)
    assert torch.equal(a["mean"], b["mean"]) and torch.equal(a["cov"], b["cov"])
    for u, v in zip(a["fit"], b["fit"]):
        assert torch.equal(u, v)
    ia, ib = a["image"].view(-1, 3), b["image"].view(-1, 3)
    assert torch.equal(ia[~off], ib[~off])
    assert bool((ia[off] != ib[off]).any(dim=1).float().mean() > 0.9)


@pytest.mark.gpu
def test_zero_pixels_follow_the_eps_rule():
    x = torch.from_numpy(synthetic(32, 40, 50, seed=10)).cuda()
    x.view(32, -1)[:, [0, 5, 300, 1999]] = 0.0  # samples 0 and 300, and two other pixels
    _check_against_pca64(x)
    fit = _native(x)["fit"]
    img = _native(x)["image"].view(-1, 3)
    t0 = -(fit.components @ fit.mean)  # a zero pixel normalises to 0
    ref = ((t0 - fit.lo) / (fit.hi - fit.lo)).clamp(0, 1)
    for p in (0, 5, 300, 1999):
        assert torch.allclose(img[p], ref, rtol=0, atol=1e-5)


@pytest.mark.gpu
def test_fit_applied_to_another_map():
    from diff_gaussian_rasterization import feature_head as fh

    C = 128
    x = torch.from_numpy(synthetic(C, 120, 160, seed=11)).cuda()
    y = torch.from_numpy(synthetic(C, 90, 70, seed=12)).cuda()
    fit = fh.pca_fit(x)
    img = fh.pca_image(y, fit)
    Y = y.view(C, -1).double()
    yh = Y / Y.norm(dim=0).clamp_min(1e-12)
    c64, m64 = fit.components.double(), fit.mean.double()
    t = c64 @ (yh - m64[:, None])
    lo, hi = float(fit.lo), float(fit.hi)
    ref = ((t - lo) / (hi - lo)).clamp(0, 1).t().reshape(90, 70, 3)
    rx = (C / 8 + 12) * U
    ya = yh - m64[:, None]
    dt = c64.abs() @ (rx * yh.abs() + U * ya.abs()) + (C / 8 + 10) * U * (c64.abs() @ ya.abs())
    bar = (dt / (hi - lo) + 2 * U).t().reshape(90, 70, 3)
    assert bool(((img.double() - ref).abs() <= bar).all())


@pytest.mark.gpu
def test_flat_map_is_bitwise_the_rows_of_the_image_map_and_reproducible():
    from diff_gaussian_rasterization import feature_head as fh

    x = torch.from_numpy(synthetic(128, 101, 203, seed=13)).cuda()
    a, b = fh.pca_fit(x), fh.pca_fit(x.view(128, -1))
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    ia, ib = fh.pca_image(x, a), fh.pca_image(x.view(128, -1), b)
    assert ia.shape == (101, 203, 3) and ib.shape == (101 * 203, 3)
    assert torch.equal(ia.view(-1, 3), ib)
    again = _native(x)
    first = _native(x)
    for k in ("mean", "cov", "image"):
        assert torch.equal(first[k], again[k])
    for u, v in zip(first["fit"], again["fit"]):
        assert torch.equal(u, v)


@pytest.mark.gpu
def test_peak_memory_has_no_sample_matrix(lib):
    from diff_gaussian_rasterization import feature_head as fh

    C, H, W = 512, 540, 960
    x = torch.from_numpy(synthetic(C, H, W, seed=14)).cuda()
    n = (H * W + 2) // 3
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    img = fh.pca_image(x)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    scratch = lib.f3dgs_feature_pca_scratch_bytes(C, H * W)
    budget = scratch + img.numel() * 4 + 2 * C * C * 8 + (2 << 20)
    assert growth <= budget < C * n * 4, (growth, budget)


@pytest.mark.gpu
def test_against_scikit_learn_at_full_size():
    pytest.importorskip("sklearn")
    from diff_gaussian_rasterization import feature_head as fh

    x = torch.from_numpy(synthetic(512, 1080, 1920, seed=15))
    vis, mean, comps, (q1, q99) = reference_visualize(x)
    fit = fh.pca_fit(x.cuda())
    img = fh.pca_image(x.cuda(), fit).cpu()
    # scikit-learn's float32 covariance carries errors that grow with n (691 200 samples), so the bar is looser
    assert np.abs(fit.mean.cpu().numpy() - mean).max() < 1e-5
    assert np.abs(fit.components.cpu().numpy() - comps).max() < 1e-3
    assert abs(float(fit.lo) - q1) < 1e-3 and abs(float(fit.hi) - q99) < 1e-3
    assert float((img - vis).abs().max()) < 2e-3
