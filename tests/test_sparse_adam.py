"""Sparse Adam: the masked optimizer step that updates only the Gaussians a step's views see (f3dgs_adam_step_masked[_f16out],
`_C.adam_step(..., visible=)`, `ViewBatch.visible()`, `GaussianState.step(..., visible=)`, `SparseGaussianAdam`).

A visible row is bitwise the dense step's row, so the dense kernel is the reference for every kind; an invisible row is
neither read nor written.  step == 0 is the upstream SparseGaussianAdam's uncorrected update, checked against a float64
restatement.  CPU part (`-m "not gpu"`): both entries reject every bad argument before any CUDA call.
"""
import ctypes

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

c_f, c_p, c_i, c_sz = ctypes.c_float, ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
IDENTITY, SIGMOID, EXP, NORMALIZE4, SH_DC, SH_REST = range(6)  # F3DGS_PARAM_*
B1, B2, EPS = 0.9, 0.999, 1e-15
RTOL, ATOL = 2e-5, 2e-6  # test_next_rows.py's fused Adam against torch


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_launch_count.restype = ctypes.c_ulonglong
    L.f3dgs_adam_step_masked.argtypes = [c_i, c_sz, c_i, c_i] + [c_p] * 5 + [c_f] * 4 + [c_i, c_p]
    L.f3dgs_adam_step_masked_f16out.argtypes = [c_i, c_sz, c_i, c_i] + [c_p] * 6 + [c_f] * 4 + [c_i, c_p]
    return L


def _rejected(lib, fn, msg, *args):
    assert fn(*args) == -1, (fn.__name__, msg)
    err = lib.f3dgs_last_error()
    assert err.startswith(fn.__name__.encode() + b": ") and msg in err, (fn.__name__, msg, err)


# ---- CPU: C ABI validation (fake addresses, never dereferenced: every call below fails validation or is a no-op)
def test_masked_adam_rejects_bad_arguments_before_touching_cuda(lib):
    launches = lib.f3dgs_launch_count()
    A = lambda k: k << 24  # noqa: E731  (distinct fake device addresses, 16 MiB apart)
    P, M = 1000, 16
    width = {IDENTITY: 24, SIGMOID: 1, EXP: 3, NORMALIZE4: 4, SH_DC: 3, SH_REST: 3 * (M - 1)}
    f, h = lib.f3dgs_adam_step_masked, lib.f3dgs_adam_step_masked_f16out

    def dense(kind=IDENTITY, n=None, P=P, M=M, ptrs=None, step=1):
        n = width[kind] * P if n is None else n
        return (kind, n, P, M, *(ptrs or [A(1), A(2), A(3), A(4), A(5)]), 1e-3, B1, B2, EPS, step, None)

    def half(n=None, P=P, ptrs=None, step=1, kind=IDENTITY):
        n = width[IDENTITY] * P if n is None else n
        return (kind, n, P, M, *(ptrs or [A(1), A(2), A(3), A(4), A(5), A(6)]), 1e-3, B1, B2, EPS, step, None)

    for kind in (6, -1):
        _rejected(lib, f, b"unknown parameter kind", kind, 24 * P, P, M, A(1), A(2), A(3), A(4), A(5), 1e-3, B1, B2, EPS,
                  1, None)
    for kind in (1, 2, 3, 4, 5, 6, -1):
        _rejected(lib, h, b"kind must be F3DGS_PARAM_IDENTITY", *half(kind=kind))
    _rejected(lib, f, b"step < 0", *dense(step=-1))
    _rejected(lib, h, b"step < 0", *half(step=-1))
    for k in range(5):
        ptrs = [A(1), A(2), A(3), A(4), A(5)]
        ptrs[k] = None
        _rejected(lib, f, b"NULL pointer", *dense(ptrs=ptrs))
    for k in range(6):
        ptrs = [A(1), A(2), A(3), A(4), A(5), A(6)]
        ptrs[k] = None
        _rejected(lib, h, b"NULL pointer", *half(ptrs=ptrs))
    for bad_P in (0, -1, 7):  # 24000 % 7 != 0
        _rejected(lib, f, b"P < 1 or n % P != 0", *dense(n=24 * P, P=bad_P))
        _rejected(lib, h, b"P < 1 or n % P != 0", *half(n=24 * P, P=bad_P))
    for kind, n in ((SIGMOID, 2 * P), (EXP, P), (EXP, 4 * P), (NORMALIZE4, 3 * P), (NORMALIZE4, 8 * P), (SH_DC, 6 * P),
                    (SH_REST, 3 * M * P)):
        _rejected(lib, f, b"n / P is not the row width of the kind", *dense(kind=kind, n=n))
    _rejected(lib, f, b"M < 1 for F3DGS_PARAM_SH_DC", *dense(kind=SH_DC, n=3 * P, M=0))
    _rejected(lib, f, b"M < 2 for F3DGS_PARAM_SH_REST", *dense(kind=SH_REST, n=3 * P, M=1))
    n = width[IDENTITY] * P
    sizes = [n * 4, n * 4, n * 4, n * 4, P]  # param, grad, exp_avg, exp_avg_sq, visible
    for k in range(5):  # param_f16 overlapping each other buffer in turn, by its last two bytes
        ptrs = [A(1), A(2), A(3), A(4), A(5), A(k + 1) + sizes[k] - 2]
        _rejected(lib, h, b"param_f16 overlaps", *half(ptrs=ptrs))
    # n == 0 is a no-op: nothing is checked but the kind, the step and M
    assert f(IDENTITY, 0, 0, 1, None, None, None, None, None, 1e-3, B1, B2, EPS, 0, None) == 0
    assert h(IDENTITY, 0, 0, 1, None, None, None, None, None, None, 1e-3, B1, B2, EPS, 0, None) == 0
    assert lib.f3dgs_launch_count() == launches


# =================================================================================================== GPU
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _group(kind, P, M=16, C=24, seed=0):
    """(param, grad_activated, exp_avg, exp_avg_sq) of one group of P Gaussians, moments nonzero"""
    g = _gen(seed)
    shape = {IDENTITY: (P, 1, C), SIGMOID: (P, 1), EXP: (P, 3), NORMALIZE4: (P, 4), SH_DC: (P, 1, 3),
             SH_REST: (P, M - 1, 3)}[kind]
    gshape = (P, M, 3) if kind in (SH_DC, SH_REST) else shape
    p = torch.randn(shape, device="cuda", generator=g)
    grad = torch.randn(gshape, device="cuda", generator=g)
    m = 0.1 * torch.randn(shape, device="cuda", generator=g)
    v = 0.01 * torch.rand(shape, device="cuda", generator=g)
    return p, grad, m, v


KINDS = [(IDENTITY, 1), (IDENTITY, 24), (IDENTITY, 512), (SIGMOID, 0), (EXP, 0), (NORMALIZE4, 0), (SH_DC, 0),
         (SH_REST, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,C", KINDS)
def test_full_mask_is_the_dense_step_bitwise(kind, C):
    from diff_gaussian_rasterization import _C

    P, M = 1001, 16
    p, grad, m, v = _group(kind, P, M, C or 24, seed=1)
    dense = [t.clone() for t in (p, m, v)]
    masked = [t.clone() for t in (p, m, v)]
    every = torch.ones(P, dtype=torch.bool, device="cuda")
    for step in (1, 2, 3):
        grad = grad * 0.5 + 0.1 * step
        _C.adam_step(kind, dense[0], grad, dense[1], dense[2], M, 1e-2, B1, B2, EPS, step)
        _C.adam_step(kind, masked[0], grad, masked[1], masked[2], M, 1e-2, B1, B2, EPS, step, None, every)
        for a, b in zip(dense, masked):
            assert torch.equal(a, b), (kind, C, step)
    assert not torch.equal(dense[0], p)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 24, 512])
def test_full_mask_f16out_is_the_dense_f16out_bitwise(C):
    from diff_gaussian_rasterization import _C

    P = 1001
    p, grad, m, v = _group(IDENTITY, P, C=C, seed=2)
    dense = [t.clone() for t in (p, m, v)] + [p.half()]
    masked = [t.clone() for t in (p, m, v)] + [p.half()]
    every = torch.ones(P, dtype=torch.uint8, device="cuda")
    for step in (1, 2, 3, 4):
        grad = grad * 0.7 - 0.05 * step
        _C.adam_step(IDENTITY, dense[0], grad, dense[1], dense[2], 1, 1e-2, B1, B2, EPS, step, dense[3])
        _C.adam_step(IDENTITY, masked[0], grad, masked[1], masked[2], 1, 1e-2, B1, B2, EPS, step, masked[3], every)
        for a, b in zip(dense, masked):
            assert torch.equal(a, b), (C, step)
        assert torch.equal(masked[3], masked[0].half())


@pytest.mark.gpu
@pytest.mark.parametrize("kind,C,f16", [k + (False,) for k in KINDS] + [(IDENTITY, C, True) for C in (1, 24, 512)])
def test_random_mask_updates_visible_rows_only_and_never_reads_the_others(kind, C, f16):
    """About 30 % of an odd P visible.  Visible rows are bitwise a dense step run on copies; invisible rows keep param,
    m, v and the float16 copy bitwise although their gradient is nonzero, and NaN in every invisible row's gradient
    reaches nothing (so those rows are not read)."""
    from diff_gaussian_rasterization import _C

    P, M = 1001, 16
    p, grad, m, v = _group(kind, P, M, C or 24, seed=3)
    vis = torch.rand(P, device="cuda", generator=_gen(4)) < 0.3
    inv = ~vis
    assert 0 < int(vis.sum()) < P
    for poison in (False, True):
        g = grad.clone()
        if poison:
            g[inv] = float("nan")
        dense = [t.clone() for t in (p, m, v)] + ([p.half()] if f16 else [])
        masked = [t.clone() for t in (p, m, v)] + ([p.half()] if f16 else [])
        for step in (1, 2):
            _C.adam_step(kind, dense[0], g, dense[1], dense[2], M, 1e-2, B1, B2, EPS, step, dense[3] if f16 else None)
            _C.adam_step(kind, masked[0], g, masked[1], masked[2], M, 1e-2, B1, B2, EPS, step,
                         masked[3] if f16 else None, vis)
        orig = [p, m, v] + ([p.half()] if f16 else [])
        for a, b, o in zip(dense, masked, orig):
            assert torch.equal(a[vis], b[vis]), (kind, C, poison)
            assert torch.equal(b[inv], o[inv]), (kind, C, poison)
            assert not torch.isnan(b).any(), (kind, C, poison)
        assert not torch.equal(masked[0][vis], p[vis])


@pytest.mark.gpu
def test_empty_masks_and_groups_are_no_ops():
    from diff_gaussian_rasterization import _C

    P = 777
    for kind, C in KINDS:
        p, grad, m, v = _group(kind, P, 16, C or 24, seed=5)
        out = [t.clone() for t in (p, m, v)]
        _C.adam_step(kind, out[0], grad, out[1], out[2], 16, 1e-2, B1, B2, EPS, 3, None,
                     torch.zeros(P, dtype=torch.bool, device="cuda"))
        for a, b in zip(out, (p, m, v)):
            assert torch.equal(a, b), kind
    # n == 0: no Gaussians, and a C = 0 feature group of P Gaussians
    e = torch.empty(0, 1, 0, device="cuda")
    _C.adam_step(IDENTITY, e, e, e.clone(), e.clone(), 1, 1e-2, B1, B2, EPS, 1, None,
                 torch.empty(0, dtype=torch.bool, device="cuda"))
    z = torch.empty(P, 1, 0, device="cuda")
    _C.adam_step(IDENTITY, z, z, z.clone(), z.clone(), 1, 1e-2, B1, B2, EPS, 1, z.half(),
                 torch.ones(P, dtype=torch.bool, device="cuda"))
    torch.cuda.synchronize()


def _upstream_update(p, g, m, v, lr, eps, vis):
    """Float64 restatement of the upstream SparseGaussianAdam's update on the rows in vis (no bias correction)."""
    p, g, m, v = (t.double().clone() for t in (p, g, m, v))
    m[vis] = 0.9 * m[vis] + 0.1 * g[vis]
    v[vis] = 0.999 * v[vis] + 0.001 * g[vis] ** 2
    p[vis] -= lr * m[vis] / (v[vis].sqrt() + eps)
    return p, m, v


def _close(a, ref):
    return torch.allclose(a.double(), ref, rtol=RTOL, atol=ATOL)


@pytest.mark.gpu
def test_step_zero_is_the_uncorrected_upstream_update():
    from diff_gaussian_rasterization import _C

    P, C = 1001, 24
    p, grad, m, v = _group(IDENTITY, P, C=C, seed=6)
    vis = torch.rand(P, device="cuda", generator=_gen(7)) < 0.5
    for lr, eps in ((1e-2, 1e-15), (1e-3, 1e-8)):
        out = [t.clone() for t in (p, m, v)]
        ref = [t.double() for t in (p, m, v)]
        for it in range(3):
            g = grad * (1 + it)
            _C.adam_step(IDENTITY, out[0], g, out[1], out[2], 1, lr, B1, B2, eps, 0, None, vis)
            ref = list(_upstream_update(*ref[:1], g, *ref[1:], lr, eps, vis))
            for a, r in zip(out, ref):
                assert _close(a, r), (lr, eps, it)
        assert torch.equal(out[0][~vis], p[~vis])


# ---- GaussianState: the native training loop with visible=vb.visible()
def _restated_step(raw, m, v, grads, lrs, steps, vis):
    """Float64 restatement of GaussianState.step(lrs, grads, visible=vis): the activations' Jacobians through torch
    autograd, then the bias-corrected Adam update on the visible rows only."""
    from diff_gaussian_rasterization.trainer import GaussianState

    r = {k: t.double().requires_grad_(True) for k, t in raw.items()}
    act = dict(means3D=r["xyz"], opacities=torch.sigmoid(r["opacity"]), scales=torch.exp(r["scaling"]),
               rotations=F.normalize(r["rotation"]), shs=torch.cat((r["f_dc"], r["f_rest"]), dim=1),
               semantic_feature=r["semantic_feature"])
    torch.autograd.backward([act[k] for k in act], [grads[k].double() for k in act])
    out = {}
    for k in GaussianState.NAMES:
        p, g, mk, vk = r[k].detach().clone(), r[k].grad, m[k].double().clone(), v[k].double().clone()
        t = steps[k]
        mk[vis] = B1 * mk[vis] + (1 - B1) * g[vis]
        vk[vis] = B2 * vk[vis] + (1 - B2) * g[vis] ** 2
        p[vis] -= lrs[k] / (1 - B1 ** t) * mk[vis] / (vk[vis].sqrt() / (1 - B2 ** t) ** 0.5 + EPS)
        out[k] = (p, mk, vk)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("feature_dtype", [torch.float32, torch.float16])
def test_gaussian_state_sparse_training(feature_dtype):
    import scenegen
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    from diff_gaussian_rasterization import feature_head as fh
    from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid

    sc = scenegen.make_scene(P=3000, W=96, H=64, C=16, sh_degree=3, views=2, seed=11)
    dev = "cuda"
    t = scenegen.to_torch(sc, dev)
    P = sc.P
    means = t["means3D"].clone()
    means[::4, 1] += 40.0  # far above the ring of cameras: outside every view
    st = GaussianState(means, t["shs"][:, :1].contiguous(), t["shs"][:, 1:].contiguous(),
                       inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                       t["rotations"].clone(), t["semantic_feature"].clone(), feature_dtype=feature_dtype)
    g = _gen(12)
    gt_color = [torch.rand(3, 64, 96, device=dev, generator=g) for _ in sc.cameras]
    gt_feat = [torch.randn(sc.C, 64, 96, device=dev, generator=g) for _ in sc.cameras]
    lrs = dict(xyz=1e-3, f_dc=5e-3, f_rest=5e-3 / 20, opacity=0.05, scaling=5e-3, rotation=1e-3, semantic_feature=0.05)
    rs = [GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev)) for cam in sc.cameras]
    seen_ever = torch.zeros(P, dtype=torch.bool, device=dev)
    first = {k: (st.raw[k].clone(), st.exp_avg[k].clone(), st.exp_avg_sq[k].clone()) for k in st.NAMES}
    losses = []

    def one_step(check):
        st.activate()
        vb = st.batch()
        vb.zero_()
        union = torch.zeros(st.P, dtype=torch.bool, device=dev)
        total = 0.0
        for i, r in enumerate(rs):
            color, feat, radii, depth, ctx = vb.forward(r)
            n = color.numel()
            total += float(((color - gt_color[i]) ** 2).mean())
            fl, gfeat = fh.feature_l1_loss_and_grad(feat.float(), gt_feat[i], 1.0)
            total += float(fl)
            vb.backward(ctx, 2.0 * (color - gt_color[i]) / n, gfeat, torch.zeros_like(depth), last=(i == len(rs) - 1))
            union |= radii > 0
        vb.all_reduce()
        vis = vb.visible()
        assert vis.dtype == torch.bool and torch.equal(vis, union)
        before = {k: (st.raw[k].clone(), st.exp_avg[k].clone(), st.exp_avg_sq[k].clone()) for k in st.NAMES}
        grads = {k: t.clone() for k, t in vb.grads.items()}
        steps = {k: st.steps[k] + 1 for k in st.NAMES}
        st.step(lrs, visible=vis)
        if check:
            ref = _restated_step({k: b[0] for k, b in before.items()}, {k: b[1] for k, b in before.items()},
                                 {k: b[2] for k, b in before.items()}, grads, lrs, steps, vis)
            for k in st.NAMES:
                for a, r_, b in zip((st.raw[k], st.exp_avg[k], st.exp_avg_sq[k]), ref[k], before[k]):
                    assert torch.equal(a[~vis], b[~vis]), k
                    assert torch.allclose(a[vis].double(), r_[vis], rtol=RTOL, atol=ATOL), k
        sf = st.raw["semantic_feature"]
        assert torch.equal(st.act["semantic_feature"], sf if feature_dtype == torch.float32 else sf.half())
        return vis, total

    for it in range(6):
        vis, loss = one_step(check=True)
        seen_ever |= vis
        losses.append(loss)
    assert losses[-1] < losses[0], losses
    never = ~seen_ever
    assert int(never.sum()) >= P // 5, int(never.sum())
    for k in st.NAMES:
        for a, b in zip((st.raw[k], st.exp_avg[k], st.exp_avg_sq[k]), first[k]):
            assert torch.equal(a[never], b[never]), k
    # densification, then more sparse steps on the new rows
    n = st.densify_and_prune(max_grad=0.0, min_opacity=0.005, extent=4.0, max_screen_size=None, generator=_gen(13))
    assert n != P and st.P == n
    for it in range(2):
        one_step(check=True)


def test_view_batch_visible_needs_the_statistics():
    from diff_gaussian_rasterization.parallel import ViewBatch

    vb = ViewBatch.__new__(ViewBatch)
    vb.denom = None
    with pytest.raises(RuntimeError, match="densify_stats"):
        vb.visible()
    vb.denom = torch.tensor([0.0, 2.0, 0.0, 1.0])
    assert vb.visible().tolist() == [False, True, False, True]


# ---- SparseGaussianAdam on the autograd path
def _prune_optimizer(optimizer, mask):
    """The reference's GaussianModel._prune_optimizer (scene/gaussian_model.py), on an optimizer's own state."""
    out = {}
    for group in optimizer.param_groups:
        stored_state = optimizer.state.get(group["params"][0], None)
        if stored_state is not None:
            stored_state["exp_avg"] = stored_state["exp_avg"][mask]
            stored_state["exp_avg_sq"] = stored_state["exp_avg_sq"][mask]
            del optimizer.state[group["params"][0]]
            group["params"][0] = nn.Parameter((group["params"][0][mask].requires_grad_(True)))
            optimizer.state[group["params"][0]] = stored_state
        else:
            group["params"][0] = nn.Parameter(group["params"][0][mask].requires_grad_(True))
        out[group["name"]] = group["params"][0]
    return out


def _cat_tensors_to_optimizer(optimizer, tensors_dict):
    """The reference's GaussianModel.cat_tensors_to_optimizer."""
    out = {}
    for group in optimizer.param_groups:
        ext = tensors_dict[group["name"]]
        stored_state = optimizer.state.get(group["params"][0], None)
        if stored_state is not None:
            stored_state["exp_avg"] = torch.cat((stored_state["exp_avg"], torch.zeros_like(ext)), dim=0)
            stored_state["exp_avg_sq"] = torch.cat((stored_state["exp_avg_sq"], torch.zeros_like(ext)), dim=0)
            del optimizer.state[group["params"][0]]
            group["params"][0] = nn.Parameter(torch.cat((group["params"][0], ext), dim=0).requires_grad_(True))
            optimizer.state[group["params"][0]] = stored_state
        else:
            group["params"][0] = nn.Parameter(torch.cat((group["params"][0], ext), dim=0).requires_grad_(True))
        out[group["name"]] = group["params"][0]
    return out


def _render_loss(params, sc, cam):
    import scenegen
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer

    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, "cuda"))
    means2D = torch.zeros_like(params["xyz"], requires_grad=True)
    color, feat, radii, depth = GaussianRasterizer(raster_settings=rs)(
        means3D=params["xyz"], means2D=means2D, shs=torch.cat((params["f_dc"], params["f_rest"]), dim=1),
        colors_precomp=None, semantic_feature=params["semantic_feature"], opacities=torch.sigmoid(params["opacity"]),
        scales=torch.exp(params["scaling"]), rotations=F.normalize(params["rotation"]), cov3D_precomp=None)
    g = _gen(21)
    loss = ((color - torch.rand(color.shape, device="cuda", generator=g)) ** 2).mean() + \
        (feat - torch.randn(feat.shape, device="cuda", generator=g)).abs().mean()
    return loss, radii


@pytest.mark.gpu
def test_sparse_gaussian_adam_on_the_autograd_path():
    import scenegen
    from diff_gaussian_rasterization import SparseGaussianAdam, __all__
    from diff_gaussian_rasterization.trainer import inverse_sigmoid

    assert "SparseGaussianAdam" in __all__
    sc = scenegen.make_scene(P=2000, W=96, H=64, C=8, sh_degree=3, views=1, seed=17)
    t = scenegen.to_torch(sc, "cuda")
    means = t["means3D"].clone()
    means[::3, 1] += 40.0  # outside the view
    raw = dict(xyz=means, f_dc=t["shs"][:, :1], f_rest=t["shs"][:, 1:],
               opacity=inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), scaling=torch.log(t["scales"]),
               rotation=t["rotations"], semantic_feature=t["semantic_feature"])
    params = {k: nn.Parameter(v.contiguous().clone().requires_grad_(True)) for k, v in raw.items()}
    lrs = dict(xyz=1.6e-4, f_dc=2.5e-3, f_rest=2.5e-3 / 20, opacity=0.025, scaling=5e-3, rotation=1e-3,
               semantic_feature=1e-3)
    frozen = nn.Parameter(torch.randn(sc.P, 2, device="cuda"))  # never gets a gradient: its group is skipped
    groups = [{"params": [params[k]], "lr": lrs[k], "name": k} for k in params]
    groups.append({"params": [frozen], "lr": 1.0, "name": "frozen"})
    opt = SparseGaussianAdam(groups, lr=0.0, eps=1e-15)
    ref = {k: (v.detach().double(), torch.zeros_like(v, dtype=torch.float64), torch.zeros_like(v, dtype=torch.float64))
           for k, v in params.items()}
    frozen0 = frozen.detach().clone()
    for it in range(3):
        opt.zero_grad(set_to_none=True)
        loss, radii = _render_loss(params, sc, sc.cameras[0])
        loss.backward()
        vis = radii > 0
        assert 0 < int(vis.sum()) < sc.P
        before = {k: v.detach().clone() for k, v in params.items()}
        opt.step(vis, sc.P)
        for k, p in params.items():
            ref[k] = _upstream_update(ref[k][0], p.grad, ref[k][1], ref[k][2], lrs[k], 1e-15, vis)
            st = opt.state[p]
            for a, r in zip((p.detach(), st["exp_avg"], st["exp_avg_sq"]), ref[k]):
                assert _close(a, r), (k, it)
            assert torch.equal(p.detach()[~vis], before[k][~vis]), (k, it)
            assert float(st["step"]) == 0.0
        assert torch.equal(frozen.detach(), frozen0) and len(opt.state[frozen]) == 0

    # the reference's densification helpers rewrite state[param]: later steps use the new tensors
    opt.param_groups.pop()  # the reference's optimizer has the Gaussians' groups only
    m_before = {k: opt.state[p]["exp_avg"].clone() for k, p in params.items()}
    keep = torch.rand(sc.P, device="cuda", generator=_gen(22)) < 0.8
    params = _prune_optimizer(opt, keep)
    n_new = 100
    ext = {k: v.detach()[:n_new].clone() for k, v in params.items()}
    params = _cat_tensors_to_optimizer(opt, ext)
    N = params["xyz"].shape[0]
    assert N == int(keep.sum()) + n_new
    state0 = {k: (p.detach().double(), opt.state[p]["exp_avg"].double(), opt.state[p]["exp_avg_sq"].double())
              for k, p in params.items()}
    for k, p in params.items():
        assert torch.equal(opt.state[p]["exp_avg"][:-n_new], m_before[k][keep])
    vis = torch.rand(N, device="cuda", generator=_gen(23)) < 0.5
    for k, p in params.items():
        p.grad = torch.randn_like(p)
    opt.step(vis, N)
    for k, p in params.items():
        r = _upstream_update(state0[k][0], p.grad, state0[k][1], state0[k][2], lrs[k], 1e-15, vis)
        st = opt.state[p]
        for a, b in zip((p.detach(), st["exp_avg"], st["exp_avg_sq"]), r):
            assert _close(a, b), k
        assert not torch.equal(p.detach()[vis], state0[k][0][vis].float()), k
    with pytest.raises(ValueError, match="visibility"):
        opt.step(vis[:-1], N)
    two = SparseGaussianAdam([{"params": [nn.Parameter(torch.zeros(4, 3, device="cuda")),
                                          nn.Parameter(torch.zeros(4, 3, device="cuda"))], "lr": 1e-3}], lr=0.0,
                             eps=1e-15)
    with pytest.raises(ValueError, match="one parameter per group"):
        two.step(torch.ones(4, dtype=torch.bool, device="cuda"), 4)
