"""Text queries of a feature field (csrc/feature_query.cu, feature_head.query): LSeg's segmentation head (decode, cosine
similarity with normalised text embeddings, argmax) and render_edit's softmax selection score of positive prompts.

CPU part (`-m "not gpu"`): a float64 NumPy restatement of the contract is pinned against the PyTorch float64
composition (conv2d, normalize, matmul, softmax, argmax); the C ABI and the Python function reject bad arguments before
touching CUDA.  GPU part (`-m gpu`): the TF32 kernel against the restatement with per-element bars that follow from
rounding both products' operands to TF32 (2^-11 relative each, the decoder's DECODE_REL for y), labels wherever the
float64 top-two margin exceeds twice the bar; exact cases (prob = 1, ties, zero and NaN columns, float16 x); bitwise
reproducibility; peak memory without any D x N buffer; the per-Gaussian selection path.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

DECODE_REL = 1.2e-3  # test_feature_decoder.py: |y - y64| <= DECODE_REL (|W| |x| + |b|) + 1e-6


def query64(x, W, b, T, scale=1.0, positive=None):
    """float64 restatement: x [C,N], W [D,C] or None, b [D] or None, T [K,D] -> (labels [N], prob [N] or None,
    logits [K,N])."""
    y = np.asarray(x, np.float64)
    if W is not None:
        y = W.astype(np.float64) @ y + (0.0 if b is None else b.astype(np.float64)[:, None])
    yh = y / np.maximum(np.sqrt((y * y).sum(0)), 1e-12)
    T = T.astype(np.float64)
    th = T / np.maximum(np.sqrt((T * T).sum(1)), 1e-12)[:, None]
    lg = scale * (th @ yh)
    prob = None
    if positive is not None:
        e = np.exp(lg - lg.max(0))
        prob = e[list(positive)].sum(0) / e.sum(0)
    return np.argmax(lg, axis=0), prob, lg


def _torch64(x, W, b, T, scale, positive):
    y = torch.from_numpy(x.astype(np.float64))
    if W is not None:
        bt = None if b is None else torch.from_numpy(b.astype(np.float64))
        y = F.conv2d(y[None, :, :, None], torch.from_numpy(W.astype(np.float64))[:, :, None, None], bt)[0, :, :, 0]
    lg = scale * (F.normalize(torch.from_numpy(T.astype(np.float64)), dim=1) @ F.normalize(y, dim=0))
    prob = None if positive is None else lg.softmax(0)[list(positive)].sum(0).numpy()
    return lg.argmax(0).numpy(), prob, lg.numpy()


def _np_case(C, D, K, N, decoder, bias, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((C if decoder else D, N)).astype(np.float32)
    W = (rng.standard_normal((D, C)) / np.sqrt(C)).astype(np.float32) if decoder else None
    b = (0.1 * rng.standard_normal(D)).astype(np.float32) if bias else None
    T = rng.standard_normal((K, D)).astype(np.float32)
    return x, W, b, T


@pytest.mark.parametrize("C,D,decoder,bias", [(5, 7, True, True), (5, 7, True, False), (8, 32, True, True),
                                              (8, 32, True, False), (16, 16, False, False), (1, 1, False, False)])
@pytest.mark.parametrize("K", [1, 3, 12])
def test_restatement_matches_pytorch_float64(C, D, decoder, bias, K):
    x, W, b, T = _np_case(C, D, K, 57, decoder, bias, 1)
    if K >= 3:
        T[2] = T[0]            # duplicate text rows: ties go to the lower index
    if K == 12:
        T[5] = 0.0             # a zero text row: cosine 0 with everything
    x[:, 3] = 0.0              # a zero feature column (decoded to b, or to 0 without a bias)
    pos = list(range(0, K, 2))
    lab, prob, lg = query64(x, W, b, T, 2.5, pos)
    rl, rp, rg = _torch64(x, W, b, T, 2.5, pos)
    assert np.allclose(lg, rg, rtol=1e-12, atol=1e-12)
    assert np.allclose(prob, rp, rtol=1e-12, atol=1e-12)
    assert np.array_equal(lab, rl)
    if K >= 3:
        assert not np.any(lab == 2)
    if b is None:
        assert lg[:, 3].tolist() == [0.0] * K and lab[3] == 0
    if K == 1:
        assert np.all(prob == 1.0) and np.all(lab == 0)


# ---- C ABI argument validation (no CUDA call is made for rejected arguments)
@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    sig = [ctypes.c_int] * 4 + [ctypes.c_void_p] * 4 + [ctypes.c_float] + [ctypes.c_void_p] * 5
    L.f3dgs_feature_query.argtypes = sig
    L.f3dgs_feature_query_f16x.argtypes = sig
    return L


def test_query_rejects_bad_arguments_before_touching_cuda(lib):
    W, b, x, T, pos, lab, pr, lg = (k << 24 for k in range(1, 9))  # never dereferenced: validation fails first
    C, D, K, N = 16, 64, 10, 100

    def q(C=C, D=D, K=K, N=N, w=W, bias=b, xx=x, t=T, s=1.0, p=pos, labels=lab, prob=pr, logits=lg, half=False):
        f = lib.f3dgs_feature_query_f16x if half else lib.f3dgs_feature_query
        return f(C, D, K, N, w, bias, xx, t, s, p, labels, prob, logits, None)

    def bad(msg, **kw):
        assert q(**kw) == -1, kw
        assert msg in lib.f3dgs_last_error(), (kw, lib.f3dgs_last_error())

    for kw in (dict(K=0), dict(K=257), dict(D=0), dict(D=4097), dict(C=0), dict(C=257), dict(N=-1),
               dict(C=4097, D=4097, w=None, bias=None)):
        bad(b"bad sizes", **kw)
    bad(b"needs a decoder weight", w=None, bias=None)                 # D != C without a decoder
    bad(b"bias without weight", C=64, w=None)
    bad(b"NULL pointer", xx=None)
    bad(b"NULL pointer", t=None)
    bad(b"no output requested", labels=None, prob=None, logits=None)
    bad(b"positive", p=None)                                         # prob without a positive set
    for s in (float("inf"), float("-inf"), float("nan")):
        bad(b"not finite", s=s)
    for half in (False, True):
        esize = 2 if half else 4
        bad(b"overlaps an input", labels=x, half=half)
        bad(b"overlaps an input", logits=x + esize * C * N - 4, half=half)   # the last element of x
        bad(b"overlaps an input", prob=W + 4 * D * C - 4, half=half)
        bad(b"overlaps an input", prob=b, half=half)
        bad(b"overlaps an input", logits=T + 4 * K * D - 1, half=half)
        bad(b"overlaps an input", labels=pos + K - 1, half=half)
        bad(b"overlaps an input", logits=x - 4 * K * N + 4, half=half)       # logits' last element is x's first
        bad(b"outputs overlap", prob=lab + 8 * N - 4, half=half)
        bad(b"outputs overlap", logits=pr + 4 * N - 4, half=half)
        bad(b"outputs overlap", logits=lab, half=half)


def test_python_query_rejects_bad_positive_and_cpu_tensors():
    from diff_gaussian_rasterization import feature_head as fh

    x, text = torch.randn(4, 6, 5), torch.randn(3, 4)
    for p in ([3], [-1], [0, 7]):
        with pytest.raises(ValueError, match="out of range"):
            fh.query(x, text, positive=p)
    with pytest.raises(ValueError, match="CUDA"):
        fh.query(x, text, positive=[0, 2])
    with pytest.raises(ValueError, match="CUDA"):
        fh.query(x, text)


# =================================================================================================== GPU
def _query(x, T, W=None, b=None, scale=1.0, positive=None, labels=True, prob=None, logits=True):
    from diff_gaussian_rasterization import _C

    e = torch.empty(0, device=x.device)
    mask = torch.empty(0, dtype=torch.uint8, device=x.device)
    if positive is not None:
        mask = torch.zeros(T.shape[0], dtype=torch.uint8, device=x.device)
        mask[list(positive)] = 1
    want_prob = positive is not None if prob is None else prob
    return _C.feature_query(x, T, e if W is None else W, e if b is None else b, scale, mask, labels, want_prob, logits)


def _dev_case(C, D, K, N, decoder, bias, seed):
    """Clustered columns: x = (prototype of a random prompt) + noise, text = decoded prototypes + noise, so that most
    columns have a clear winner (at D >= 16) and the label checks cover most of them."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    Cx = C if decoder else D
    P = torch.randn(Cx, K, device="cuda", generator=g)
    lab = torch.randint(0, K, (N,), device="cuda", generator=g)
    x = (P[:, lab] + 0.3 * torch.randn(Cx, N, device="cuda", generator=g)).contiguous()
    W = torch.randn(D, C, device="cuda", generator=g) / C ** 0.5 if decoder else None
    b = 0.1 * torch.randn(D, device="cuda", generator=g) if bias else None
    proto = P if W is None else W @ P + (0.0 if b is None else b[:, None])
    T = (proto.t() + 0.1 * proto.abs().mean() * torch.randn(K, D, device="cuda", generator=g)).contiguous()
    return x, W, b, T


def _ref_dev(x, W, b, T, scale, positive):
    """-> (l64 [K,N], logit bar [K,N], prob64, prob bar) in float64 on the device.
    y's bar is the decoder's; ||yh - yh64|| <= 2 ||dy|| / ||y64||; the TF32 operands of the second product add 2^-10 of
    <|yh|, |th|>, and the fp32 sums (||y||^2, ||t||^2, the product over D) at most 2 D 2^-24 of it and of |cos|."""
    y = x.double()
    ybar = torch.zeros_like(y)
    if W is not None:
        W64 = W.double()
        ybar = DECODE_REL * (W64.abs() @ y.abs()) + 1e-6
        y = W64 @ y
        if b is not None:
            y += b.double()[:, None]
            ybar += DECODE_REL * b.double().abs()[:, None]
    ny = y.norm(dim=0).clamp_min(1e-12)
    yh = y / ny
    T64 = T.double()
    th = T64 / T64.norm(dim=1, keepdim=True).clamp_min(1e-12)
    cos = th @ yh
    A = th.abs() @ yh.abs()
    D = T.shape[1]
    bar = abs(scale) * (2 * ybar.norm(dim=0) / ny + (2.0 ** -10 + 2.4e-7 * D) * (A + cos.abs()) + 1e-6)
    l64 = scale * cos
    p64 = pbar = None
    if positive is not None:
        sm = torch.softmax(l64, 0)
        p64 = sm[list(positive)].sum(0)
        beta = bar.max(0).values
        pbar = p64 * (1 - p64) * torch.expm1(2 * beta) + 1e-6 + 1.2e-7 * T.shape[0]
    return l64, bar, p64, pbar


def _check(x, W, b, T, scale, positive):
    """Kernel against float64 with the bars above -> (columns whose label is decided by the margin rule, N)."""
    lab, prob, lg = _query(x, T, W, b, scale, positive)
    l64, bar, p64, pbar = _ref_dev(x.float(), W, b, T, scale, positive)
    err = (lg.double() - l64).abs()
    assert bool((err <= bar).all()), float((err / bar).max())
    if positive is not None:
        perr = (prob.double() - p64).abs()
        assert bool((perr <= pbar).all()), float((perr / pbar).max())
    K = T.shape[0]
    if K == 1:
        assert bool((lab == 0).all())
        return lab.numel(), lab.numel()
    top = l64.topk(2, dim=0)
    clear = (top.values[0] - top.values[1]) > 2 * bar.max(0).values
    assert torch.equal(lab[clear], top.indices[0][clear])
    assert torch.equal(lab, lg.argmax(0))  # labels are the first maximal index of the kernel's own logits
    return int(clear.sum()), lab.numel()


CD = [(1, 1), (5, 7), (16, 64), (128, 512), (256, 4096)]
KS = [1, 2, 7, 128, 129, 150, 256]
NS = [1, 15, 16, 17, 4099]


@pytest.mark.gpu
@pytest.mark.parametrize("C,D", CD)
@pytest.mark.parametrize("decoder", [True, False])
@pytest.mark.parametrize("K", KS)
def test_parity_with_float64(C, D, decoder, K):
    """Every N, bias on / off (decoder) and float32 / float16 x; without a decoder x has D channels."""
    variants = [(bias, dt) for bias in ((True, False) if decoder else (False,)) for dt in (torch.float32, torch.float16)]
    clear = total = 0
    for i, N in enumerate(NS):
        for j, (bias, dt) in enumerate(variants):
            x, W, b, T = _dev_case(C, D, K, N, decoder, bias, 100 * i + j)
            x = x.to(dt)
            pos = list(range(0, K, 3))
            c, n = _check(x, W, b, T, 10.0 if j % 2 == 0 else 1.0, pos)
            clear, total = clear + c, total + n
    if D >= 16:
        assert clear >= 0.9 * total, (clear, total)


@pytest.mark.gpu
def test_full_size_view_on_a_sample():
    C, D, K, N = 128, 512, 150, 1080 * 1920
    x, W, b, T = _dev_case(C, D, K, N, True, True, 7)
    pos = [0, 3, 77, 149]
    lab, prob, lg = _query(x, T, W, b, 10.0, pos)
    g = torch.Generator(device="cuda").manual_seed(8)
    idx = torch.randperm(N, device="cuda", generator=g)[:65536]
    l64, bar, p64, pbar = _ref_dev(x[:, idx], W, b, T, 10.0, pos)
    assert bool(((lg[:, idx].double() - l64).abs() <= bar).all())
    assert bool(((prob[idx].double() - p64).abs() <= pbar).all())
    top = l64.topk(2, dim=0)
    clear = (top.values[0] - top.values[1]) > 2 * bar.max(0).values
    assert float(clear.double().mean()) > 0.9
    assert torch.equal(lab[idx][clear], top.indices[0][clear])


@pytest.mark.gpu
@pytest.mark.parametrize("decoder", [True, False])
def test_prob_is_exactly_one(decoder):
    for K in (1, 150):
        x, W, b, T = _dev_case(16, 64, K, 4099, decoder, decoder, 11)
        _, prob, _ = _query(x, T, W, b, 10.0, list(range(K)))
        assert bool((prob == 1.0).all())


@pytest.mark.gpu
def test_identical_text_rows_tie_to_the_lower_index():
    K = 200  # two chunks of prompts; the pairs sit inside a tile, across tiles and across the chunk boundary
    x, W, b, T = _dev_case(16, 64, K, 8000, True, True, 12)
    pairs = [(3, 5), (20, 190), (100, 130)]
    for lo, hi in pairs:
        T[hi] = T[lo]
    lab, _, lg = _query(x, T, W, b, 10.0)
    for lo, hi in pairs:
        assert torch.equal(lg[lo], lg[hi])
        assert not bool((lab == hi).any())
        assert int((lab == lo).sum()) > 0
    assert torch.equal(lab, lg.argmax(0))


@pytest.mark.gpu
@pytest.mark.parametrize("decoder", [True, False])
def test_zero_and_nan_columns(decoder):
    x, W, _, T = _dev_case(16, 64, 150, 4099, decoder, False, 13)
    lab0, prob0, lg0 = _query(x, T, W, None, 10.0, [1, 2])
    xz = x.clone()
    xz[:, 5] = 0.0
    xz[:, [7, 40, 4098]] = float("nan")
    lab, prob, lg = _query(xz, T, W, None, 10.0, [1, 2])
    assert bool((lg[:, 5] == 0).all()) and int(lab[5]) == 0
    for c in (7, 40, 4098):
        assert int(lab[c]) == 0 and bool(lg[:, c].isnan().all())
    keep = torch.ones(x.shape[1], dtype=torch.bool, device="cuda")
    keep[[5, 7, 40, 4098]] = False
    assert torch.equal(lab[keep], lab0[keep]) and torch.equal(prob[keep], prob0[keep])
    assert torch.equal(lg[:, keep], lg0[:, keep])


@pytest.mark.gpu
@pytest.mark.parametrize("C,D,decoder", [(16, 64, True), (256, 512, True), (512, 512, False)])
def test_half_x_is_bitwise_its_float_upcast(C, D, decoder):
    x, W, b, T = _dev_case(C, D, 150, 4099, decoder, decoder, 14)
    xh = x.half()
    a = _query(xh, T, W, b, 10.0, [0, 1])
    f = _query(xh.float(), T, W, b, 10.0, [0, 1])
    for u, v in zip(a, f):
        assert torch.equal(u, v)


@pytest.mark.gpu
@pytest.mark.parametrize("C,D,K,decoder", [(128, 512, 150, True), (256, 300, 7, True), (64, 64, 129, False)])
def test_bitwise_reproducible_and_independent_of_requested_outputs(C, D, K, decoder):
    x, W, b, T = _dev_case(C, D, K, 50000, decoder, decoder, 15)
    pos = [0, K - 1]
    full = _query(x, T, W, b, 10.0, pos)
    again = _query(x, T, W, b, 10.0, pos)
    for u, v in zip(full, again):
        assert torch.equal(u, v)
    assert torch.equal(_query(x, T, W, b, 10.0, pos, labels=False, logits=False)[1], full[1])
    assert torch.equal(_query(x, T, W, b, 10.0, None, logits=False)[0], full[0])
    assert torch.equal(_query(x, T, W, b, 10.0, None, labels=False)[2], full[2])


def _default_pool_used_high(reset):
    """High watermark of the device's default stream-ordered pool (cudaMallocAsync scratch; torch's caching allocator
    does not use it)."""
    cu = ctypes.CDLL("libcuda.so.1")
    dev, pool, v = ctypes.c_int(), ctypes.c_void_p(), ctypes.c_uint64(0)
    assert cu.cuDeviceGet(ctypes.byref(dev), torch.cuda.current_device()) == 0
    assert cu.cuDeviceGetDefaultMemPool(ctypes.byref(pool), dev) == 0
    used_mem_high = 8  # CU_MEMPOOL_ATTR_USED_MEM_HIGH
    if reset:
        assert cu.cuMemPoolSetAttribute(pool, used_mem_high, ctypes.byref(v)) == 0
    assert cu.cuMemPoolGetAttribute(pool, used_mem_high, ctypes.byref(v)) == 0
    return v.value


@pytest.mark.gpu
def test_peak_memory_has_no_decoded_map():
    C, D, K, H, Wd = 128, 512, 150, 1080, 1920
    N = H * Wd
    x, W, b, T = _dev_case(C, D, K, N, True, True, 16)
    x = x.view(C, H, Wd)
    torch.cuda.synchronize()
    _default_pool_used_high(reset=True)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    from diff_gaussian_rasterization import feature_head as fh

    lab, prob, lg = fh.query(x, T, W[:, :, None, None], b, 10.0, positive=[0, 1])
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base + _default_pool_used_high(reset=False)
    assert lab.shape == (H, Wd) and lab.dtype == torch.int64 and prob.shape == (H, Wd) and lg is None
    outputs = N * (8 + 4)
    scratch = 4 * (D * C + D) + 4 * 152 * D + 152 + 4 * 256
    budget = outputs + scratch + (4 << 20)
    assert growth <= budget < D * N * 4, (growth, budget)


@pytest.mark.gpu
def test_per_gaussian_selection_score():
    from diff_gaussian_rasterization import feature_head as fh
    from diff_gaussian_rasterization.trainer import GaussianState

    P, C, D = 200000, 128, 512
    g = torch.Generator(device="cuda").manual_seed(17)
    z = lambda *s: torch.zeros(*s, device="cuda")  # noqa: E731
    sf = torch.randn(P, 1, C, device="cuda", generator=g)
    st = GaussianState(torch.randn(P, 3, device="cuda", generator=g), z(P, 1, 3), z(P, 15, 3), z(P, 1), z(P, 3),
                       torch.nn.functional.normalize(torch.randn(P, 4, device="cuda", generator=g), dim=1), sf)
    W = torch.randn(D, C, 1, 1, device="cuda", generator=g) / C ** 0.5
    b = 0.1 * torch.randn(D, device="cuda", generator=g)
    # the "positive" prompt is the decoded feature of a few Gaussians, the other one unrelated
    T = torch.stack([(W[:, :, 0, 0] @ sf[:8, 0].mean(0) + b), torch.randn(D, device="cuda", generator=g)])
    feats = st.raw["semantic_feature"][:, 0, :].t().contiguous()
    lab, prob, lg = fh.query(feats, T, W, b, logit_scale=10.0, positive=[0], logits=True)
    assert prob.shape == (P,) and lg.shape == (2, P) and lab.shape == (P,)
    # the composition render_edit is written as: decode, normalize, cosine with the normalised text, softmax
    with torch.no_grad():
        y = F.conv2d(feats.double().t()[:, :, None, None], W.double(), b.double())[:, :, 0, 0]
        ref = torch.softmax(10.0 * F.normalize(y, dim=1) @ F.normalize(T.double(), dim=1).t(), dim=1)[:, 0]
    l64, bar, p64, pbar = _ref_dev(feats, W[:, :, 0, 0], b, T, 10.0, [0])
    assert torch.allclose(p64, ref, rtol=0, atol=1e-12)
    assert bool(((prob.double() - ref).abs() <= pbar).all())
    assert bool(((lg.double() - l64).abs() <= bar).all())


@pytest.mark.gpu
def test_binding_and_abi_on_real_memory(lib):
    from diff_gaussian_rasterization import _C

    C, D, K, N = 16, 64, 7, 1000
    x, W, b, T = _dev_case(C, D, K, N, True, True, 18)
    e, m = torch.empty(0, device="cuda"), torch.ones(K, dtype=torch.uint8, device="cuda")
    bad = [
        lambda: _C.feature_query(x.double(), T, W, b, 1.0, m, True, False, False),
        lambda: _C.feature_query(x, T[:, :63], W, b, 1.0, m, True, False, False),       # D of text vs weight
        lambda: _C.feature_query(x[:15], T, W, b, 1.0, m, True, False, False),          # C of x vs weight
        lambda: _C.feature_query(torch.randn(D, N, device="cuda"), T, e, b, 1.0, m, True, False, False),  # bias, no W
        lambda: _C.feature_query(x, T, W, b[:63], 1.0, m, True, False, False),
        lambda: _C.feature_query(x, T, W, b, 1.0, e.byte(), True, True, False),         # prob without positive
        lambda: _C.feature_query(x, T, W, b, 1.0, m[:6], True, True, False),
        lambda: _C.feature_query(x, T, W, b, 1.0, m, False, False, False),              # nothing requested
        lambda: _C.feature_query(x, T, W, b, float("nan"), m, True, False, False),
        lambda: _C.feature_query(x, T.cpu(), W, b, 1.0, m, True, False, False),
        lambda: _C.feature_query(x, T, W, b, 1.0, m.cpu(), True, True, False),
    ]
    for i, f in enumerate(bad):
        with pytest.raises(RuntimeError):
            f()
            pytest.fail(f"case {i} was accepted")
    # float16 x: the overlap check uses its 2-byte size, so labels may start right after x's last element
    ref = _query(x.half(), T, W, b, logits=False)[0]
    buf = torch.empty(C * N * 2 + N * 8, dtype=torch.uint8, device="cuda")
    buf[: C * N * 2].view(torch.float16).view(C, N).copy_(x.half())
    base, s = buf.data_ptr(), torch.cuda.current_stream().cuda_stream
    args = (C, D, K, N, W.data_ptr(), b.data_ptr(), base, T.data_ptr(), 1.0, None)
    assert lib.f3dgs_feature_query_f16x(*args, base + C * N * 2 - 8, None, None, s) == -1
    assert lib.f3dgs_feature_query_f16x(*args, base + C * N * 2, None, None, s) == 0
    torch.cuda.synchronize()
    assert torch.equal(buf[C * N * 2:].view(torch.int64), ref)
