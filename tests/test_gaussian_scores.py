"""Per-Gaussian blend-weight scores (f3dgs_gaussian_scores_accum, the geometry walk's score mode, scores.GaussianScores)
and pruning from a mask with the Adam state carried along (f3dgs_prune_plan + f3dgs_densify_apply,
GaussianState.prune / prune_by_importance).

The scores are checked against the forward's own blend weights W[g, p] (the one-hot extraction of blend_weights.py):
pixel_count exactly the pairs with W > 0, weight_sum within Weights.per_gaussian's bar, max_weight within the backward's
unwind bar of the largest extracted weight.  Pruning is checked bitwise against t[keep].
CPU part (`-m "not gpu"`): both C symbols reject malformed calls before any CUDA call.
"""
import ctypes
import types

import pytest
import torch

import blend_weights as bw
import parity
import scenegen

c_p, c_i = ctypes.c_void_p, ctypes.c_int
NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "semantic_feature")


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_launch_count.restype = ctypes.c_ulonglong
    L.f3dgs_gaussian_scores_accum.argtypes = [c_i] * 4 + [c_p] * 7
    L.f3dgs_prune_plan.argtypes = [c_i] + [c_p] * 4
    return L


def _rejected(lib, sym, rc, msg, kw):
    assert rc == -1, (sym, kw)
    err = lib.f3dgs_last_error()
    assert err.startswith(sym.encode() + b": ") and msg in err, (sym, kw, err)


A = lambda k: k << 28  # noqa: E731  (distinct fake device addresses, 256 MiB apart, never dereferenced)


# ---- CPU: C ABI validation
def test_scores_reject_malformed_calls_before_touching_cuda(lib):
    sym = "f3dgs_gaussian_scores_accum"
    launches = lib.f3dgs_launch_count()
    P, R, W, H = 1000, 5000, 64, 48

    def call(P=P, R=R, W=W, H=H, geom=A(1), binning=A(2), img=A(3), ws=A(4), mw=A(5), pc=A(6)):
        return lib.f3dgs_gaussian_scores_accum(P, R, W, H, geom, binning, img, ws, mw, pc, None)

    def rejected(msg, **kw):
        _rejected(lib, sym, call(**kw), msg, kw)

    for kw in (dict(P=-1), dict(R=-1), dict(W=0), dict(H=0), dict(W=-5)):
        rejected(b"bad sizes", **kw)
    for k in ("geom", "binning", "img"):
        rejected(b"missing forward buffers", **{k: None})
    for k in ("ws", "mw", "pc"):
        rejected(b"NULL pointer", **{k: None})
    rejected(b"must not overlap", mw=A(4) + P * 4 - 4)   # max_weight starts in weight_sum's last element
    rejected(b"must not overlap", ws=A(5) - P * 4 + 4)   # weight_sum ends in max_weight's first element
    rejected(b"must not overlap", pc=A(4) + 8)
    rejected(b"must not overlap", mw=A(6) + P * 8 - 4)   # max_weight inside pixel_count's last element
    rejected(b"must not overlap", pc=A(5) - P * 8 + 4)
    rejected(b"must not overlap", ws=A(5))
    # nothing to blend: nothing is launched and nothing is read
    assert call(P=0) == 0 and call(R=0) == 0 and call(P=0, geom=None, ws=None) == 0
    assert lib.f3dgs_launch_count() == launches


def test_prune_plan_rejects_malformed_calls_before_touching_cuda(lib):
    sym = "f3dgs_prune_plan"
    launches = lib.f3dgs_launch_count()
    P = 1000
    flags = ((P + 1) * 16 + 255) // 256 * 256  # the scanned flags at the front of the scratch

    def call(P=P, keep=A(1), scratch=A(2), counts=A(3)):
        return lib.f3dgs_prune_plan(P, keep, scratch, counts, None)

    def rejected(msg, **kw):
        _rejected(lib, sym, call(**kw), msg, kw)

    for kw in (dict(P=-1), dict(P=(2 ** 31 - 1) // 3 + 1)):
        rejected(b"bad sizes", **kw)
    for k in ("keep", "scratch", "counts"):
        rejected(b"NULL pointer", **{k: None})
    rejected(b"NULL pointer", P=0, counts=None)
    rejected(b"overlaps scratch", keep=A(2) + flags - 1)
    rejected(b"overlaps scratch", keep=A(2) - P + 1)
    rejected(b"overlaps scratch", counts=A(2) + 16)
    rejected(b"overlaps scratch", counts=A(2) - 12)
    assert lib.f3dgs_launch_count() == launches


# =================================================================================================== GPU
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _settings(sc, cam=None):
    from diff_gaussian_rasterization import GaussianRasterizationSettings

    return GaussianRasterizationSettings(**parity.settings(sc, cam or sc.cameras[0], "cuda"))


def _scores(b, P, W, H):
    """One view's scores from a forward's buffers b -> (weight_sum, max_weight, pixel_count)."""
    from diff_gaussian_rasterization import _C

    ws, mw = torch.zeros(P, device="cuda"), torch.zeros(P, device="cuda")
    pc = torch.zeros(P, dtype=torch.int64, device="cuda")
    _C.gaussian_scores_accum(b["geom"], b["R"], b["binning"], b["img"], W, H, ws, mw, pc)
    return ws, mw, pc


def _check_against_weights(label, v):
    """v: a test_blend_weights.DeviceView (its forward's buffers, pairs and extracted weights)."""
    P, H, W = v.P, v.H, v.W
    ws, mw, pc = _scores(v.base, P, W, H)
    blended = v.w > 0
    idx = v.pairs.widx[blended]
    g, n = v.pairs.gid[idx], v.pairs.n[v.pairs.pix[idx]].double()
    w = v.w[blended].double()
    # the count: exactly the pairs the forward composited
    assert torch.equal(pc, v.Wt.m.long()), label
    # the sum: the per-Gaussian identity's bar
    r_sum = v.Wt.per_gaussian(ws.reshape(P, 1), torch.ones(H * W, 1, device="cuda"))
    # the max: each of the walk's weights is within the unwind bar K u (2 n_p + 4) w of the forward's, so the largest
    # is within the largest of those bars of the largest extracted weight
    ref = torch.zeros(P, dtype=torch.float64, device="cuda").scatter_reduce_(0, g, w, "amax")
    bar = torch.zeros(P, dtype=torch.float64, device="cuda").scatter_reduce_(0, g, bw.K * bw.U * (2 * n + 4) * w, "amax")
    r_max = float(bw._ratio((mw.double() - ref).abs(), bar).max())
    # no blended pair (radii == 0 among them): exactly zero
    none = v.Wt.m == 0
    assert bool((v.base["radii"][v.Wt.m > 0] > 0).all())
    assert bool((ws[none] == 0).all() and (mw[none] == 0).all() and (pc[none] == 0).all()), label
    assert int(pc.sum()) == int(blended.sum()) > 0
    print(f"[{label}] blended pairs {int(blended.sum())}, Gaussians blended {int((~none).sum())} of {P}, "
          f"radii == 0: {int((v.base['radii'] == 0).sum())}; worst |err|/bar: weight_sum={r_sum:.3g} "
          f"max_weight={r_max:.3g}")
    assert r_sum <= 1.0 and r_max <= 1.0, label
    return ws, mw, pc


SCORE_SCENES = ["small", "needles", "layers129", "opaque", "halves97x38", "inside", "medium"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCORE_SCENES)
def test_scores_against_the_forwards_weights(name):
    from diff_gaussian_rasterization import _C
    from test_blend_weights import _view

    v = _view(name)
    ws, _, _ = _check_against_weights(name, v)
    # weight_sum is the lift's weight_sum on the same buffers, up to the order of the float reductions
    b, P = v.base, v.P
    fs, wl = torch.zeros(P, 1, device="cuda"), torch.zeros(P, device="cuda")
    _C.lift_features_accum(b["geom"], b["R"], b["binning"], b["img"], torch.ones(1, v.H, v.W, device="cuda"), fs, wl)
    assert torch.allclose(ws, wl, rtol=1e-5, atol=1e-7 * float(wl.max()))


def _aa_forward(t, rs, sf):
    from diff_gaussian_rasterization import _C

    e = torch.Tensor([])
    R, color, feat, depth, radii, geom, binning, img = _C.rasterize_gaussians_antialiased(
        rs["bg"], t["means3D"], e, sf, t["opacities"], t["scales"], t["rotations"], rs["scale_modifier"], e,
        rs["viewmatrix"], rs["projmatrix"], rs["tanfovx"], rs["tanfovy"], rs["image_height"], rs["image_width"],
        t["shs"], rs["sh_degree"], rs["campos"], rs["prefiltered"], False)
    pl, ranges, n_contrib, final_T, rec = _C.debug_views(geom, binning, img, t["means3D"].shape[0], rs["image_width"],
                                                         rs["image_height"], R)
    return dict(R=R, color=color, feature_map=feat, depth=depth, radii=radii, geom=geom, binning=binning, img=img,
                point_list=pl, ranges=ranges, n_contrib=n_contrib, final_T=final_T, rec=rec)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["small", "needles", "inside"])
def test_antialiased_forward_scores_the_antialiased_weights(name):
    import test_blend_weights as tbw

    class AntialiasedView(tbw.DeviceView):
        def __init__(self, sc, cam, group):
            self.sc, self.cam = sc, cam
            self.t = scenegen.to_torch(sc, "cuda")
            self.rs = parity.settings(sc, cam, "cuda")
            self.P, self.W, self.H = sc.P, cam.image_width, cam.image_height
            self.base = _aa_forward(self.t, self.rs, self.t["semantic_feature"])
            self.pairs = bw.Pairs(self.base["point_list"], self.base["ranges"], self.base["n_contrib"], self.W, self.H)
            self.w = self.weights(group)
            self.Wt = bw.Weights(self.pairs, self.w, self.P)

        def forward(self, sf):
            r = _aa_forward(self.t, self.rs, sf)
            for k in ("color", "n_contrib", "final_T", "point_list"):
                assert torch.equal(r[k], self.base[k]), k
            return r

    sc, cam = tbw.SCENES[name]()
    v = AntialiasedView(sc, cam, 512)
    ws, _, _ = _check_against_weights(f"{name} antialiased", v)
    # the antialiased model is another model: its weights are not the default forward's
    plain = tbw._view(name)
    assert not torch.equal(ws, _scores(plain.base, plain.P, plain.W, plain.H)[0])


@pytest.mark.gpu
def test_views_accumulate_with_sum_and_max_and_halves_combine_like_all_reduce():
    from diff_gaussian_rasterization import GaussianScores

    sc = scenegen.make_scene(P=6000, W=150, H=100, C=0, sh_degree=1, views=4, seed=51)
    t = scenegen.to_torch(sc, "cuda")
    views = [_settings(sc, cam) for cam in sc.cameras]

    def scored(vs):
        s = GaussianScores(t["means3D"], t["opacities"], t["scales"], t["rotations"])
        for rs in vs:
            s.add(rs)
        return s

    whole = scored(views)
    each = [scored([rs]) for rs in views]
    assert torch.equal(whole.pixel_count, sum(s.pixel_count for s in each))
    assert torch.equal(whole.max_weight, torch.stack([s.max_weight for s in each]).amax(0))
    ws = sum(s.weight_sum for s in each)
    assert torch.allclose(whole.weight_sum, ws, rtol=1e-5, atol=1e-7 * float(ws.max()))
    a, b = scored(views[:2]), scored(views[2:])
    assert torch.equal(whole.pixel_count, a.pixel_count + b.pixel_count)
    assert torch.equal(whole.max_weight, torch.maximum(a.max_weight, b.max_weight))
    assert torch.allclose(whole.weight_sum, a.weight_sum + b.weight_sum, rtol=1e-5, atol=1e-7 * float(ws.max()))
    assert int((whole.pixel_count > 0).sum()) > int((each[0].pixel_count > 0).sum())
    assert whole.pixel_count.dtype == torch.int64


# ---- pruning
def _state(P, C, M, seed, feature_dtype=torch.float32):
    from diff_gaussian_rasterization.trainer import GaussianState

    g = _gen(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)  # noqa: E731
    st = GaussianState(r(P, 3), r(P, 1, 3), r(P, M - 1, 3), r(P, 1), r(P, 3) * 0.5 - 4.0, r(P, 4), r(P, 1, C),
                       feature_dtype=feature_dtype)
    st.exp_avg = {k: torch.randn(v.shape, device="cuda", generator=g) for k, v in st.raw.items()}
    st.exp_avg_sq = {k: torch.rand(v.shape, device="cuda", generator=g) for k, v in st.raw.items()}
    st.steps = {k: 3 + i for i, k in enumerate(NAMES)}
    st.max_radii2D = torch.rand(P, device="cuda", generator=g) * 40
    return st


def _expect(st, keep):
    return dict(raw={k: st.raw[k][keep].clone() for k in NAMES}, exp_avg={k: st.exp_avg[k][keep].clone() for k in NAMES},
                exp_avg_sq={k: st.exp_avg_sq[k][keep].clone() for k in NAMES}, steps=dict(st.steps),
                max_radii2D=st.max_radii2D[keep].clone())


def _bits(t):
    return t.contiguous().view(torch.int32)


def _assert_pruned(st, e, label):
    for grp in ("raw", "exp_avg", "exp_avg_sq"):
        for k in NAMES:
            a, b = getattr(st, grp)[k], e[grp][k]
            assert a.shape == b.shape and torch.equal(_bits(a), _bits(b)), (label, grp, k)
    assert st.steps == e["steps"], label
    assert torch.equal(_bits(st.max_radii2D), _bits(e["max_radii2D"])), label
    sf = st.act["semantic_feature"]
    if st.feature_dtype == torch.float16:
        assert sf.dtype == torch.float16 and torch.equal(sf.view(torch.int16), st.raw["semantic_feature"].half().view(
            torch.int16)), label
    else:
        assert sf.data_ptr() == st.raw["semantic_feature"].data_ptr() or sf.numel() == 0, label


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 16])
@pytest.mark.parametrize("C", [0, 3, 128, 512])
@pytest.mark.parametrize("P", [0, 1, 1000, 200_000])
def test_prune_equals_the_restatement(P, C, M):
    """keep-all, keep-none and a random mask (uint8 with bytes other than 1 among them); float16 features with M = 16."""
    fd = torch.float16 if M == 16 else torch.float32
    g = _gen(P + C + M)
    masks = dict(all=torch.ones(P, dtype=torch.bool, device="cuda"), none=torch.zeros(P, dtype=torch.bool, device="cuda"),
                 random=torch.rand(P, device="cuda", generator=g) < 0.6,
                 random_u8=torch.randint(0, 3, (P,), dtype=torch.uint8, device="cuda", generator=g) * 70)
    for label, keep in masks.items():
        st = _state(P, C, M, seed=P + C + M, feature_dtype=fd)
        kb = keep if keep.dtype == torch.bool else keep != 0
        e = _expect(st, kb)
        n = st.prune(keep)
        assert n == int(kb.sum()) == st.P
        _assert_pruned(st, e, (P, C, M, label))
        assert st.act["opacities"].shape == (n, 1)


@pytest.mark.gpu
def test_prune_makes_one_host_sync():
    from test_densify import _count_syncs

    st = _state(20_000, 32, 16, seed=5)
    keep = torch.rand(20_000, device="cuda", generator=_gen(6)) < 0.5
    e = _expect(st, keep)
    syncs = _count_syncs(lambda: st.prune(keep))
    assert len(syncs) == 1, syncs
    _assert_pruned(st, e, "sync")


@pytest.mark.gpu
def test_prune_recomputes_the_3d_filter_and_rejects_bad_masks():
    from diff_gaussian_rasterization import compute_3d_filter

    sc = scenegen.make_scene(P=5000, W=150, H=100, C=8, sh_degree=1, views=3, seed=52)
    views = [_settings(sc, cam) for cam in sc.cameras]
    st = _state_of(sc)
    st.compute_3d_filter(views)
    keep = torch.rand(sc.P, device="cuda", generator=_gen(7)) < 0.7
    xyz = st.raw["xyz"][keep].clone()
    st.prune(keep)
    assert torch.equal(_bits(st.raw["xyz"]), _bits(xyz))
    assert torch.equal(_bits(st.filter_3d), _bits(compute_3d_filter(xyz, views)))
    st.activate()  # the filtered tensors of the new size
    with pytest.raises(ValueError, match="bool or uint8"):
        st.prune(torch.ones(st.P, device="cuda"))
    with pytest.raises(ValueError, match="bool or uint8"):
        st.prune(torch.ones(st.P + 1, dtype=torch.bool, device="cuda"))


@pytest.mark.gpu
@pytest.mark.parametrize("ratio,power", [(0.3, 0.1), (0.6, 0.1), (0.5, 0.0), (0.0, 0.1), (1.0, 0.1)])
def test_prune_by_importance_equals_the_restatement(ratio, power):
    P = 4000
    st = _state(P, 16, 4, seed=8)
    g = _gen(9)
    st.raw["scaling"][: P // 2] = st.raw["scaling"][0]  # equal volumes: ties in v wherever weight_sum ties
    w = torch.randint(0, 6, (P,), device="cuda", generator=g).float()  # many ties, zeros among them
    scores = types.SimpleNamespace(weight_sum=w)
    v = w * st.activate()["scales"].prod(dim=1) ** power
    drop = torch.sort(v, stable=True).indices[: int(ratio * P)]
    keep = torch.ones(P, dtype=torch.bool, device="cuda")
    keep[drop] = False
    e = _expect(st, keep)
    n = st.prune_by_importance(scores, ratio, power)
    assert n == P - int(ratio * P)
    _assert_pruned(st, e, (ratio, power))


# ---- properties
def _state_of(sc, feature_dtype=torch.float32):
    from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid

    t = scenegen.to_torch(sc, "cuda")
    return GaussianState(t["means3D"].clone(), t["shs"][:, :1].contiguous(), t["shs"][:, 1:].contiguous(),
                         inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                         t["rotations"].clone(), t["semantic_feature"].reshape(sc.P, 1, -1).clone(),
                         feature_dtype=feature_dtype)


def _render(act, rs, antialiasing=False):
    from diff_gaussian_rasterization import _C

    e = torch.Tensor([])
    out = _C.rasterize_gaussians_alpha_invdepth(
        rs.bg, act["means3D"], e, act["semantic_feature"], act["opacities"], act["scales"], act["rotations"],
        rs.scale_modifier, e, rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width,
        act["shs"], rs.sh_degree, rs.campos, rs.prefiltered, False, antialiasing=antialiasing)
    return dict(color=out[1], feature_map=out[2], depth=out[3], alpha=out[4], invdepth=out[5])


@pytest.mark.gpu
@pytest.mark.parametrize("antialiasing", [False, True])
def test_pruning_unblended_gaussians_changes_only_pixels_they_ended(antialiasing):
    """Rows no view blends add nothing to any pixel, and the compaction keeps the order of the others.  But a pair is
    also not blended when it ends the pixel: the composite stops, as the reference does, at the first pair that would
    take T (1 - alpha) below 1e-4, without blending it.  Pruning such a row lets the next ones blend there.  So every
    pixel stays bitwise identical (colour, depth, feature map, opacity and inverse-depth planes) except pixels that
    had T_final < 0.01 (T (1 - alpha) < 1e-4 with alpha <= 0.99), and there the opacity plane moves by at most T_final."""
    from diff_gaussian_rasterization import GaussianScores

    sc = scenegen.make_scene(P=20_000, W=160, H=120, C=16, sh_degree=2, views=3, seed=53)
    views = [_settings(sc, cam) for cam in sc.cameras]
    st = _state_of(sc)
    with torch.no_grad():
        st.raw["opacity"][:2000] = -7.0  # alpha < 1/255 everywhere
    scores = GaussianScores.from_state(st, antialiasing=antialiasing)
    for rs in views:
        scores.add(rs)
    keep = scores.pixel_count > 0
    assert 2000 <= int((~keep).sum()) < sc.P
    act = st.activate()
    before = [_render(act, rs, antialiasing) for rs in views]
    n = st.prune(keep)
    act = st.activate()
    changed_all = 0
    for i, rs in enumerate(views):
        after = _render(act, rs, antialiasing)
        T = 1.0 - before[i]["alpha"].double().reshape(-1)
        changed = torch.zeros_like(T, dtype=torch.bool)
        for k, x in before[i].items():
            ch = x.shape[0]
            same = _bits(after[k].float()).reshape(ch, -1) == _bits(x.float()).reshape(ch, -1)
            changed |= ~same.all(0)
        assert bool((T[changed] < 0.011).all()), (i, float(T[changed].max()))
        dA = (after["alpha"].double() - before[i]["alpha"].double()).reshape(-1).abs()
        assert bool((dA <= T + 1e-6).all()), i
        changed_all += int(changed.sum())
    print(f"[antialiasing={antialiasing}] pruned {sc.P - n} of {sc.P} (never blended); pixels changed over "
          f"{len(views)} views: {changed_all} of {len(views) * sc.cameras[0].image_width * sc.cameras[0].image_height}, "
          f"all with T_final < 0.01")


def _l1(act, views, ref):
    return sum(float((_render(act, rs)["color"] - r).abs().mean()) for rs, r in zip(views, ref)) / len(views)


@pytest.mark.gpu
def test_pruning_the_lowest_weight_sums_changes_the_renders_less_than_random():
    from diff_gaussian_rasterization import GaussianScores

    sc = scenegen.make_scene(P=30_000, W=200, H=150, C=0, sh_degree=1, views=4, seed=54)
    views = [_settings(sc, cam) for cam in sc.cameras]
    st = _state_of(sc)
    scores = GaussianScores.from_state(st)
    for rs in views:
        scores.add(rs)
    act = st.activate()
    ref = [_render(act, rs)["color"].clone() for rs in views]
    P, n = sc.P, int(0.3 * sc.P)
    lowest = torch.ones(P, dtype=torch.bool, device="cuda")
    lowest[torch.sort(scores.weight_sum, stable=True).indices[:n]] = False
    rand = torch.ones(P, dtype=torch.bool, device="cuda")
    rand[torch.randperm(P, device="cuda", generator=_gen(55))[:n]] = False
    a, b = _state_of(sc), _state_of(sc)
    a.prune(lowest)
    b.prune(rand)
    la, lb = _l1(a.activate(), views, ref), _l1(b.activate(), views, ref)
    print(f"L1 against the unpruned render, 30 % pruned: lowest weight_sum {la:.5f}, random {lb:.5f}")
    assert la < lb


@pytest.mark.gpu
@pytest.mark.parametrize("feature_dtype", [torch.float32, torch.float16], ids=["float32", "float16"])
def test_training_keeps_lowering_the_loss_after_prune_by_importance(feature_dtype):
    from diff_gaussian_rasterization import GaussianScores
    from test_feature_lift import _feature_loss

    C = 16
    sc = scenegen.make_scene(P=6000, W=128, H=96, C=C, sh_degree=1, views=4, seed=56)
    views = [_settings(sc, cam) for cam in sc.cameras]
    teacher = _state_of(sc)
    teachers = []
    for rs in views:
        fm = _render(teacher.activate(), rs)["feature_map"]
        teachers.append(fm.half() if feature_dtype == torch.float16 else fm.clone())
    grad_dtype = torch.float16 if feature_dtype == torch.float16 else None
    st = _state_of(sc, feature_dtype)
    with torch.no_grad():
        st.raw["semantic_feature"].zero_()
    st._reset_derived(keep_optimizer_state=True)
    l0 = _feature_loss(st, views, teachers, grad_dtype, train_steps=10)
    scores = GaussianScores.from_state(st)
    for rs in views:
        scores.add(rs)
    P0 = st.P
    st.prune_by_importance(scores, 0.3)
    assert st.P == P0 - int(0.3 * P0)
    l1 = _feature_loss(st, views, teachers, grad_dtype)
    l2 = _feature_loss(st, views, teachers, grad_dtype, train_steps=10)
    print(f"[{feature_dtype}] feature L1: after 10 steps {l0:.4f}, after the prune {l1:.4f}, 10 steps later {l2:.4f}")
    assert l2 < l1
