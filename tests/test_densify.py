"""Adaptive density control on the GPU: GaussianState.densify_and_prune / reset_opacity / update_max_radii on
csrc/densify.cu (f3dgs_densify_plan, f3dgs_densify_apply, f3dgs_reset_opacity).

The yardstick is tests/ref_densify.py, the PyTorch restatement of the reference (scene/gaussian_model.py:350-434).
Every output tensor must be bitwise equal to it, except the xyz of split children: the restatement's torch.bmm has no
defined summation order, so those agree to 1e-6 of (|parent xyz| + sum_k |R[c,k] s_k z_k|) per element."""
import ctypes
import math
import warnings

import numpy as np
import pytest
import torch

import ref_densify

NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "semantic_feature")
INT_MAX = 2**31 - 1


# ---------------------------------------------------------------------------------------------------- C ABI (CPU)
class Fields(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in NAMES]


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    p, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_densify_scratch_bytes.restype = ctypes.c_size_t
    L.f3dgs_densify_scratch_bytes.argtypes = [i]
    L.f3dgs_densify_plan.argtypes = [i, p, p, p, p, f, f, f, f, p, p, p]
    L.f3dgs_densify_apply.argtypes = [i, i, i, p, p, p, p, p, p]
    L.f3dgs_reset_opacity.argtypes = [i, p, p, p, f, p]
    L.f3dgs_launch_count.restype = ctypes.c_ulonglong
    return L


def _fields(base):
    out = (Fields * 3)()
    for g in range(3):
        for j, n in enumerate(NAMES):
            setattr(out[g], n, base + (7 * g + j) * 0x1000000)
    return out


def test_cabi_rejects_bad_arguments_before_touching_cuda(lib):
    n0 = lib.f3dgs_launch_count()
    err = lib.f3dgs_last_error
    # never dereferenced: every call below is rejected first
    ga, dn, op, sc, scr, cnt = 0x1000000, 0x2000000, 0x3000000, 0x4000000, 0x80000000, 0x90000000
    plan = lib.f3dgs_densify_plan
    th = (2e-4, 0.04, 0.005, 0.4)
    assert plan(-1, ga, dn, op, sc, *th, scr, cnt, None) == -1 and b"bad sizes" in err()
    assert plan(INT_MAX // 3 + 1, ga, dn, op, sc, *th, scr, cnt, None) == -1 and b"bad sizes" in err()
    for k in range(6):
        args = [ga, dn, op, sc, scr, cnt]
        args[k] = None
        assert plan(10, *args[:4], *th, *args[4:], None) == -1 and b"NULL" in err(), k
    assert plan(0, None, None, None, None, *th, None, None, None) == -1 and b"NULL" in err()  # counts always needed
    assert plan(10, ga, dn, op, sc, *th, scr, scr + 64, None) == -1 and b"overlaps" in err()

    apply = lib.f3dgs_densify_apply
    src, dst, nrm = _fields(0x100000000), _fields(0x200000000), 0xA0000000
    good = (ctypes.c_int32 * 4)(4, 2, 3, 3)  # P = 10 -> P' = 12
    assert apply(-1, 16, 8, scr, good, nrm, src, dst, None) == -1 and b"bad sizes" in err()
    assert apply(INT_MAX // 3 + 1, 16, 8, scr, good, nrm, src, dst, None) == -1 and b"bad sizes" in err()
    assert apply(10, 0, 8, scr, good, nrm, src, dst, None) == -1 and b"bad sizes" in err()
    assert apply(10, 16, -1, scr, good, nrm, src, dst, None) == -1 and b"bad sizes" in err()
    assert apply(10, 16, 4097, scr, good, nrm, src, dst, None) == -1 and b"bad sizes" in err()
    assert apply(10, 16, 8, scr, None, nrm, src, dst, None) == -1 and b"NULL" in err()
    for bad in ((-1, 0, 0, 0), (11, 0, 0, 0), (0, 11, 0, 0), (0, 0, 3, 2), (0, 0, 0, 11)):
        c = (ctypes.c_int32 * 4)(*bad)
        assert apply(10, 16, 8, scr, c, nrm, src, dst, None) == -1 and b"counts" in err(), bad
    assert apply(10, 16, 8, scr, good, None, src, dst, None) == -1 and b"normals" in err()
    assert apply(10, 16, 8, None, good, nrm, src, dst, None) == -1 and b"scratch" in err()
    for g in range(3):
        for n in NAMES:
            for which in (src, dst):
                f = _fields(0x100000000 if which is src else 0x200000000)
                setattr(f[g], n, None)
                args = (f, dst) if which is src else (src, f)
                assert apply(10, 16, 8, scr, good, nrm, *args, None) == -1 and b"NULL" in err(), (g, n)
    # optional fields: f_rest with M == 1 and semantic_feature with C == 0 may be NULL (then the call would run: not made)
    for g in range(3):
        for n in NAMES:
            for target in (src[0].xyz + 8, scr + 16, nrm + 8, src[2].semantic_feature):
                f = _fields(0x200000000)
                setattr(f[g], n, target)
                assert apply(10, 16, 8, scr, good, nrm, src, f, None) == -1 and b"overlaps" in err(), (g, n, target)
    # a dst field that starts below a src field and runs into it (P' = 12 rows of 4 floats)
    f = _fields(0x200000000)
    f[0].rotation = src[0].xyz - 12 * 16 + 4
    assert apply(10, 16, 8, scr, good, nrm, src, f, None) == -1 and b"overlaps" in err()

    ro = lib.f3dgs_reset_opacity
    assert ro(-1, op, ga, dn, 0.01, None) == -1 and b"P < 0" in err()
    for k in range(3):
        args = [op, ga, dn]
        args[k] = None
        assert ro(10, *args, 0.01, None) == -1 and b"NULL" in err()
    assert ro(0, None, None, None, 0.01, None) == 0  # nothing to do
    assert lib.f3dgs_densify_scratch_bytes(0) == 0 and lib.f3dgs_densify_scratch_bytes(-3) == 0
    assert lib.f3dgs_launch_count() == n0


# ---------------------------------------------------------------------------------------------------- GPU helpers
PERCENT_DENSE, EXTENT, MAX_GRAD, MIN_OPACITY = 0.01, 3.7, 2e-4, 0.005  # 0.01 * 3.7 is not a float32


def _exact_exp_log(target):
    """A float32 s with exp(s) == float32(target) on the GPU, or None (for rows right at a threshold)."""
    t = torch.tensor([target], dtype=torch.float32, device="cuda")
    s0 = torch.log(t)
    cand = s0 + torch.arange(-64, 65, device="cuda", dtype=torch.float32) * torch.finfo(torch.float32).eps * s0.abs()
    cand = torch.cat([s0, cand])
    hit = cand[torch.exp(cand) == t]
    return float(hit[0]) if hit.numel() else None


def make_state(P, C, M, seed):
    """A seeded state whose statistics produce every class: clones, splits, transparent and world-size-pruned originals,
    clones and children, denom == 0 (NaN -> 0, and x / 0 = inf -> selected), and rows exactly at the thresholds."""
    from diff_gaussian_rasterization.trainer import GaussianState

    g = torch.Generator().manual_seed(seed)
    raw_scaling = torch.rand(P, 3, generator=g) * 6.0 - 6.0  # exp in [0.0025, 1]: both sides of 0.037 and 0.37
    raw_opacity = torch.randn(P, 1, generator=g) * 3.0       # about 4 % below min_opacity
    denom = torch.randint(0, 4, (P,), generator=g).float()
    grad_accum = torch.rand(P, generator=g) * denom * 4e-4
    inf_rows = torch.rand(P, generator=g) < 0.01
    grad_accum[inf_rows & (denom == 0)] = 1e-3
    if P >= 8:
        grad_accum[:4], denom[:4] = float(np.float32(MAX_GRAD)), 1.0  # g == float32(max_grad): selected
        grad_accum[4], denom[4] = 0.0, 1.0
        grad_accum[5], denom[5], raw_scaling[5], raw_opacity[5] = 1e-3, 1.0, -5.0, -8.0  # a transparent clone
        for row, thr in ((0, PERCENT_DENSE * EXTENT), (1, PERCENT_DENSE * EXTENT), (4, 0.1 * EXTENT)):
            s = _exact_exp_log(thr)
            if s is not None:
                raw_scaling[row] = torch.tensor([s, -6.0, -6.0])
    st = GaussianState(torch.randn(P, 3, generator=g).cuda(), torch.randn(P, 1, 3, generator=g).cuda(),
                       torch.randn(P, M - 1, 3, generator=g).cuda(), raw_opacity.cuda(), raw_scaling.cuda(),
                       torch.randn(P, 4, generator=g).cuda(), torch.randn(P, 1, C, generator=g).cuda(),
                       percent_dense=PERCENT_DENSE)
    for k in NAMES:
        st.exp_avg[k] = torch.randn(st.raw[k].shape, generator=g).cuda()
        st.exp_avg_sq[k] = torch.rand(st.raw[k].shape, generator=g).cuda()
    st.steps = {k: int(i) + 3 for i, k in enumerate(NAMES)}
    return st, grad_accum.cuda(), denom.cuda()


def clone_state(st):
    from diff_gaussian_rasterization.trainer import GaussianState

    c = GaussianState(*[st.raw[k].clone() for k in NAMES], percent_dense=st.percent_dense)
    c.exp_avg = {k: v.clone() for k, v in st.exp_avg.items()}
    c.exp_avg_sq = {k: v.clone() for k, v in st.exp_avg_sq.items()}
    c.steps = dict(st.steps)
    return c


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def bits(t):
    return t.contiguous().view(torch.int32)


def run_both(st, ga, dn, max_screen_size, seed=7, **kw):
    args = dict(max_grad=MAX_GRAD, min_opacity=MIN_OPACITY, extent=EXTENT, max_screen_size=max_screen_size)
    args.update(kw)
    a, b = clone_state(st), clone_state(st)
    ga_, gb_ = gen(seed), gen(seed)
    na = a.densify_and_prune(grad_accum=ga, denom=dn, generator=ga_, **args)
    info = {}
    nb = ref_densify.densify_and_prune(b, grad_accum=ga, denom=dn, generator=gb_, info=info, **args)
    return a, b, na, nb, info, ga_, gb_


def assert_matches(a, b, na, nb, info, ga_, gb_):
    assert na == nb == a.P == b.P
    kept = info["child_keep"]
    nk = int(kept.sum())
    for d in ("raw", "exp_avg", "exp_avg_sq"):
        for k in NAMES:
            x, y = getattr(a, d)[k], getattr(b, d)[k]
            assert x.shape == y.shape and x.is_contiguous(), (d, k)
            if d == "raw" and k == "xyz":
                assert torch.equal(bits(x[:na - nk]), bits(y[:nb - nk])), (d, k)
                parent, rsz = info["parent_xyz"][kept], info["rsz"][kept]
                tol = 1e-6 * (parent.abs() + rsz.norm(dim=1, keepdim=True))
                assert torch.all((x[na - nk:] - y[nb - nk:]).abs() <= tol), (x[na - nk:] - y[nb - nk:]).abs().max()
            else:
                assert torch.equal(bits(x), bits(y)), (d, k)
    assert a.steps == b.steps
    assert a.max_radii2D.shape == (na,) and not a.max_radii2D.any()
    assert a.batch().P == na
    assert torch.equal(torch.randn(8, generator=ga_, device="cuda"), torch.randn(8, generator=gb_, device="cuda"))


def classes(st, ga, dn):
    """Which of the selection / prune classes the statistics exercise (restated with torch, for coverage only)."""
    g = ga / dn
    g[g.isnan()] = 0
    smax = torch.exp(st.raw["scaling"]).max(1).values
    sel = g >= MAX_GRAD
    clone, split = sel & (smax <= PERCENT_DENSE * EXTENT), sel & (smax > PERCENT_DENSE * EXTENT)
    low = torch.sigmoid(st.raw["opacity"]).squeeze(-1) < MIN_OPACITY
    big = smax > 0.1 * EXTENT
    cbig = torch.exp(torch.log(torch.exp(st.raw["scaling"]) / 1.6)).max(1).values > 0.1 * EXTENT
    return dict(clone=clone.any(), split=split.any(), pruned_original=(~split & low).any(),
                pruned_clone=(clone & low).any(), pruned_child=(split & low).any(), world_original=(~split & big).any(),
                world_child=(split & cbig).any(), denom0=(dn == 0).any(), inf_grad=torch.isinf(g).any())


# ---------------------------------------------------------------------------------------------------- GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 16])
@pytest.mark.parametrize("C", [0, 3, 32, 128, 257, 512])
@pytest.mark.parametrize("P", [0, 1, 1000, 200_000])
def test_densify_matches_restatement(P, C, M):
    st, ga, dn = make_state(P, C, M, seed=P + 7 * C + M)
    if P >= 1000:
        cls = {k: bool(v) for k, v in classes(st, ga, dn).items()}
        assert all(cls.values()), cls
    for screen in (None, 20):
        a, b, na, nb, info, ga_, gb_ = run_both(st, ga, dn, screen)
        assert_matches(a, b, na, nb, info, ga_, gb_)
        if P >= 1000:
            assert 0 < na != P
        # determinism: the same inputs and generator state give bitwise the same output, children's xyz included
        a2 = clone_state(st)
        a2.densify_and_prune(MAX_GRAD, MIN_OPACITY, EXTENT, screen, grad_accum=ga, denom=dn, generator=gen(7))
        for d in ("raw", "exp_avg", "exp_avg_sq"):
            for k in NAMES:
                assert torch.equal(bits(getattr(a, d)[k]), bits(getattr(a2, d)[k])), (d, k)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["nothing_selected", "everything_pruned", "all_denom_zero", "max_grad_zero"])
def test_densify_edge_cases(case):
    st, ga, dn = make_state(1000, 32, 16, seed=11)
    kw = {}
    if case == "nothing_selected":
        kw["max_grad"] = 1e30
        ga = torch.where(dn == 0, 0.0, ga)  # x / 0 = inf would still be selected
    elif case == "everything_pruned":
        kw["min_opacity"] = 2.0
    elif case == "all_denom_zero":
        ga, dn = torch.zeros_like(ga), torch.zeros_like(dn)
    else:
        kw["max_grad"] = 0.0  # every Gaussian is cloned or split; clones (gradient 0) are still never split
    a, b, na, nb, info, ga_, gb_ = run_both(st, ga, dn, 20, **kw)
    assert_matches(a, b, na, nb, info, ga_, gb_)
    if case == "everything_pruned":
        assert na == 0
        # an empty state densifies (to nothing) and activates
        a.densify_and_prune(0.0, MIN_OPACITY, EXTENT, None, grad_accum=torch.zeros(0, device="cuda"),
                            denom=torch.zeros(0, device="cuda"))
        assert a.P == 0 and a.activate()["opacities"].shape == (0, 1)
    if case in ("nothing_selected", "all_denom_zero"):
        assert "parent_xyz" in info and info["parent_xyz"].shape[0] == 0


@pytest.mark.gpu
def test_densify_uses_the_viewbatch_statistics_by_default():
    st, ga, dn = make_state(1000, 8, 4, seed=5)
    ref = clone_state(st)
    vb = st.batch()
    vb.grad_accum.copy_(ga)
    vb.denom.copy_(dn)
    del vb
    n = st.densify_and_prune(MAX_GRAD, MIN_OPACITY, EXTENT, None, generator=gen(1))
    nb = ref_densify.densify_and_prune(ref, MAX_GRAD, MIN_OPACITY, EXTENT, None, grad_accum=ga, denom=dn,
                                       generator=gen(1))
    assert n == nb and torch.equal(bits(st.raw["semantic_feature"]), bits(ref.raw["semantic_feature"]))


def _count_syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    # (torch also warns once that the debug mode is a prototype; that notice is not a sync)
    return [f"{x.filename}:{x.lineno}: {x.message}" for x in w if "called a synchronizing CUDA operation" in str(x.message)]


@pytest.mark.gpu
def test_one_host_sync_and_sync_free_max_radii():
    st, ga, dn = make_state(20_000, 32, 16, seed=3)
    g = gen(2)
    syncs = _count_syncs(lambda: st.densify_and_prune(MAX_GRAD, MIN_OPACITY, EXTENT, 20, grad_accum=ga, denom=dn,
                                                      generator=g))
    assert len(syncs) == 1, syncs
    P = st.P
    gr = torch.Generator().manual_seed(4)
    for _ in range(3):
        radii = (torch.randint(-2, 30, (P,), generator=gr, dtype=torch.int32)).cuda()
        expect = ref_densify.update_max_radii(st.max_radii2D.clone(), radii)
        assert _count_syncs(lambda: st.update_max_radii(radii)) == []
        assert torch.equal(st.max_radii2D, expect)
    assert st.max_radii2D.max() > 0


def _growth(fn):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    a0 = torch.cuda.memory_allocated()
    r0 = torch.cuda.memory_stats()["requested_bytes.all.current"]
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - a0, torch.cuda.memory_stats()["requested_bytes.all.peak"] - r0


@pytest.mark.gpu
def test_peak_memory():
    """The native call holds the old and the new state side by side and nothing else of size: its requested-bytes peak
    grows by at most new state + scratch + normals + 1 MiB.  The caching allocator rounds every block up (by less than
    1 MiB for blocks above 1 MiB), so max_memory_allocated gets that much more per allocation (24 in the call)."""
    from diff_gaussian_rasterization import _C

    P, C, M = 200_000, 128, 16
    st, ga, dn = make_state(P, C, M, seed=9)
    ref = clone_state(st)
    scratch, counts = _C.densify_plan(ga, dn, st.raw["opacity"], st.raw["scaling"], MAX_GRAD, PERCENT_DENSE * EXTENT,
                                      MIN_OPACITY, 0.1 * EXTENT)
    A, B, Cc, Ns = counts.tolist()
    W = 14 + 3 * (M - 1) + C
    budget = 3 * (A + B + 2 * Cc) * W * 4 + scratch.numel() + 2 * Ns * 3 * 4 + (1 << 20)
    del scratch, counts
    alloc, req = _growth(lambda: st.densify_and_prune(MAX_GRAD, MIN_OPACITY, EXTENT, 20, grad_accum=ga, denom=dn,
                                                      generator=gen(0)))
    ref_alloc, ref_req = _growth(lambda: ref_densify.densify_and_prune(ref, MAX_GRAD, MIN_OPACITY, EXTENT, 20,
                                                                       grad_accum=ga, denom=dn, generator=gen(0)))
    state = 3 * P * W * 4
    print(f"\nP={P} C={C}: state {state / 2**20:.1f} MiB; peak growth native {alloc / 2**20:.1f} MiB "
          f"(requested {req / 2**20:.1f}, budget {budget / 2**20:.1f}), restatement {ref_alloc / 2**20:.1f} MiB "
          f"(requested {ref_req / 2**20:.1f})")
    assert st.P == ref.P == A + B + 2 * Cc
    assert req <= budget
    assert alloc <= budget + 24 * (1 << 20)


@pytest.mark.gpu
def test_reset_opacity_matches_torch_formula():
    from diff_gaussian_rasterization.trainer import GaussianState

    P = 10_000
    g = torch.Generator().manual_seed(8)
    op = torch.randn(P, 1, generator=g) * 6.0  # many already below 0.01 (raw < -4.6)
    op[:6, 0] = torch.tensor([float("inf"), float("-inf"), float("nan"), -4.59512, 0.0, -30.0])
    st = GaussianState(torch.randn(P, 3).cuda(), torch.randn(P, 1, 3).cuda(), torch.randn(P, 15, 3).cuda(), op.cuda(),
                       torch.randn(P, 3).cuda(), torch.randn(P, 4).cuda(), torch.randn(P, 1, 4).cuda())
    for k in NAMES:
        st.exp_avg[k].normal_()
        st.exp_avg_sq[k].uniform_()
    ref = clone_state(st)
    xyz_m = st.exp_avg["xyz"].clone()
    st.reset_opacity()
    ref_densify.reset_opacity(ref)
    x, y = st.raw["opacity"], ref.raw["opacity"]
    assert torch.equal(x.isnan(), y.isnan()) and bool(x[2].isnan())
    assert torch.equal(bits(torch.nan_to_num(x)), bits(torch.nan_to_num(y)))
    assert (x.squeeze(-1)[6:] < 0).all() and torch.sigmoid(x[6:]).max() <= 0.0100001
    assert not st.exp_avg["opacity"].any() and not st.exp_avg_sq["opacity"].any()
    assert torch.equal(st.exp_avg["xyz"], xyz_m)


@pytest.mark.gpu
def test_training_keeps_improving_after_densification():
    """activate -> ViewBatch over two views (fused feature loss) -> Adam, a densification from the accumulated statistics,
    then more steps on the new P: the loss keeps going down."""
    import scenegen
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    from diff_gaussian_rasterization import feature_head as fh
    from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid

    sc = scenegen.make_config("small", views=2)
    dev = "cuda"
    t = scenegen.to_torch(sc, dev)
    st = GaussianState(t["means3D"].clone(), t["shs"][:, :1].contiguous(), t["shs"][:, 1:].contiguous(),
                       inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                       t["rotations"].clone(), t["semantic_feature"].clone())
    gts = [torch.rand(sc.C, 40, 56, device=dev) for _ in sc.cameras]
    lrs = dict(xyz=0.0, f_dc=0.0, f_rest=0.0, opacity=0.0, scaling=0.0, rotation=0.0, semantic_feature=0.05)
    losses, P0 = [], st.P

    def step():
        st.activate()
        vb = st.batch()
        vb.zero_()
        total = 0.0
        for v, cam in enumerate(sc.cameras):
            rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))
            color, feat, radii, depth, ctx = vb.forward(rs)
            loss, gfeat = fh.feature_l1_loss_and_grad(feat, gts[v], 1.0)
            vb.backward(ctx, torch.zeros_like(color), gfeat, torch.zeros_like(depth), last=(v == len(sc.cameras) - 1))
            st.update_max_radii(radii)
            total += float(loss)
        vb.all_reduce()
        st.step(lrs)
        return total

    for _ in range(4):
        losses.append(step())
    g = st.batch().grad_accum / st.batch().denom
    thr = float(torch.nan_to_num(g).median())
    n = st.densify_and_prune(max_grad=thr, min_opacity=0.005, extent=4.0, max_screen_size=20, generator=gen(0))
    assert n != P0 and st.raw["semantic_feature"].shape[0] == n and st.exp_avg["xyz"].shape[0] == n
    after = [step() for _ in range(4)]
    assert losses[-1] < losses[0], losses
    assert after[-1] < after[0], after
    assert st.batch().P == n and math.isfinite(after[-1])
