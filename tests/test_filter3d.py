"""Mip-Splatting's 3D smoothing filter on the GPU: csrc/filter3d.cu (f3dgs_filter3d_compute, _apply, _apply_backward,
f3dgs_reset_opacity_filter3d), filter3d.compute_3d_filter / apply_3d_filter and the filter in GaussianState.

The yardstick is tests/ref_filter3d.py, the official code restated in PyTorch.  The filter agrees within a few float32
ulp (the restatement's camera transform is an sgemm with its own summation order); the apply forward and the filtered
reset are bitwise the official float32 formula; the backward matches float64 autograd."""
import ctypes
import math

import numpy as np
import pytest
import torch

import ref_filter3d as ref

INT_MAX = 2**31 - 1


# ---------------------------------------------------------------------------------------------------- C ABI (CPU)
@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    p, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_launch_count.restype = ctypes.c_ulonglong
    L.f3dgs_filter3d_scratch_bytes.restype = ctypes.c_size_t
    L.f3dgs_filter3d_scratch_bytes.argtypes = [i]
    L.f3dgs_filter3d_compute.argtypes = [i, i, p, p, p, p, p, p, p]
    L.f3dgs_filter3d_apply.argtypes = [i, p, p, p, p, p, p]
    L.f3dgs_filter3d_apply_backward.argtypes = [i, p, p, p, p, p, p, p, p]
    L.f3dgs_reset_opacity_filter3d.argtypes = [i, p, p, p, p, p, f, p]
    return L


def _rejected(lib, name, call, msg):
    """call() is rejected with `name: ...msg...`, also right after another entry point failed"""
    lib.f3dgs_filter3d_apply(-1, None, None, None, None, None, None)
    assert call() == -1
    err = lib.f3dgs_last_error()
    assert err.startswith(name + b": ") and msg in err, (name, err)


def test_cabi_rejects_bad_arguments_before_touching_cuda(lib):
    n0 = lib.f3dgs_launch_count()
    # never dereferenced: every call below is rejected first
    P, V = 10, 3
    m, vm, intr, flt, ns, scr = 0x1000000, 0x2000000, 0x3000000, 0x4000000, 0x5000000, 0x6000000
    comp, name = lib.f3dgs_filter3d_compute, b"f3dgs_filter3d_compute"
    _rejected(lib, name, lambda: comp(-1, V, m, vm, intr, flt, ns, scr, None), b"bad sizes")
    _rejected(lib, name, lambda: comp(INT_MAX // 3 + 1, V, m, vm, intr, flt, ns, scr, None), b"bad sizes")
    _rejected(lib, name, lambda: comp(P, 0, m, vm, intr, flt, ns, scr, None), b"bad sizes")
    _rejected(lib, name, lambda: comp(0, 0, m, vm, intr, flt, ns, scr, None), b"bad sizes")
    _rejected(lib, name, lambda: comp(P, -2, m, vm, intr, flt, ns, scr, None), b"bad sizes")
    for k in range(6):
        a = [m, vm, intr, flt, ns, scr]
        a[k] = None
        _rejected(lib, name, lambda: comp(P, V, *a, None), b"NULL")
    # an output on an input, on another output, or on the scratch
    for a in ([m, vm, intr, m + 4, ns, scr], [m, vm, intr, flt, vm + 8, scr], [m, vm, intr, flt, ns, intr],
              [m, vm, intr, flt, flt + 36, scr], [m, vm, intr, flt, ns, ns], [m, vm, intr, flt, scr + 128, scr]):
        _rejected(lib, name, lambda: comp(P, V, *a, None), b"overlap")
    assert comp(0, V, None, None, None, None, None, None, None) == 0  # nothing to do
    assert lib.f3dgs_filter3d_scratch_bytes(0) == 0 and lib.f3dgs_filter3d_scratch_bytes(-3) == 0
    assert lib.f3dgs_filter3d_scratch_bytes(1) > 0

    o, s, f, oo, so = 0x1000000, 0x2000000, 0x3000000, 0x4000000, 0x5000000
    app, name = lib.f3dgs_filter3d_apply, b"f3dgs_filter3d_apply"
    _rejected(lib, name, lambda: app(-1, o, s, f, oo, so, None), b"bad sizes")
    _rejected(lib, name, lambda: app(INT_MAX // 3 + 1, o, s, f, oo, so, None), b"bad sizes")
    for k in range(5):
        a = [o, s, f, oo, so]
        a[k] = None
        _rejected(lib, name, lambda: app(P, *a, None), b"NULL")
    for a in ([o, s, f, o, so], [o, s, f, oo, s + 12], [o, s, f, oo, f - 4], [o, s, f, oo, oo + 36]):
        _rejected(lib, name, lambda: app(P, *a, None), b"overlap")
    assert app(0, None, None, None, None, None, None) == 0

    gof, gsf, go, gs = 0x6000000, 0x7000000, 0x8000000, 0x9000000
    bwd, name = lib.f3dgs_filter3d_apply_backward, b"f3dgs_filter3d_apply_backward"
    _rejected(lib, name, lambda: bwd(-1, o, s, f, gof, gsf, go, gs, None), b"bad sizes")
    for k in range(7):
        a = [o, s, f, gof, gsf, go, gs]
        a[k] = None
        _rejected(lib, name, lambda: bwd(P, *a, None), b"NULL")
    # in place is allowed only onto the output's own upstream gradient, at the same address
    for a in ([o, s, f, gof, gsf, gof + 4, gs], [o, s, f, gof, gsf, go, gsf + 4], [o, s, f, gof, gsf, gsf, gs],
              [o, s, f, gof, gsf, go, gof], [o, s, f, gof, gsf, o, gs], [o, s, f, gof, gsf, go, s],
              [o, s, f, gof, gsf, go, f], [o, s, f, gof, gsf, go, go + 4], [o, s, f, gof, gsf, gof, gof + 8]):
        _rejected(lib, name, lambda: bwd(P, *a, None), b"overlap")
    assert bwd(0, None, None, None, None, None, None, None, None) == 0

    ro, rs, m1, m2 = 0x1000000, 0x2000000, 0x4000000, 0x5000000
    rst, name = lib.f3dgs_reset_opacity_filter3d, b"f3dgs_reset_opacity_filter3d"
    _rejected(lib, name, lambda: rst(-1, ro, rs, f, m1, m2, 0.01, None), b"bad sizes")
    for k in range(5):
        a = [ro, rs, f, m1, m2]
        a[k] = None
        _rejected(lib, name, lambda: rst(P, a[0], a[1], a[2], a[3], a[4], 0.01, None), b"NULL")
    for a in ([ro, rs, f, ro, m2], [ro, rs, f, m1, m1 + 4], [ro, rs, f, rs + 8, m2], [ro, rs, f, m1, f],
              [f + 4, rs, f, m1, m2]):
        _rejected(lib, name, lambda: rst(P, a[0], a[1], a[2], a[3], a[4], 0.01, None), b"overlap")
    assert rst(0, None, None, None, None, None, 0.01, None) == 0
    assert lib.f3dgs_launch_count() == n0


# ---------------------------------------------------------------------------------------------------- GPU helpers
def bits(t):
    return t.contiguous().view(torch.int32)


def ulp32(x):
    x = x.abs().float()
    return (torch.nextafter(x, torch.full_like(x, float("inf"))) - x).double()


def settings(sc, cam):
    import scenegen
    from diff_gaussian_rasterization import GaussianRasterizationSettings

    return GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, "cuda"))


def cams_of(vms, intr):
    return torch.as_tensor(np.asarray(vms, np.float32)).reshape(-1, 16).cuda(), \
        torch.as_tensor(np.asarray(intr, np.float32)).reshape(-1, 4).cuda()


def native(xyz, vms, intr):
    from diff_gaussian_rasterization import _C

    f, n = _C.filter3d_compute(xyz, vms, intr)
    return f, int(n)


def check_compute(xyz, vms, intr, what, ulps=4):
    """native filter against the restatement; rows within 1e-5 relative of a margin or the depth threshold, where the
    restatement's sgemm may decide `valid` the other way, are excluded and counted"""
    f, n_seen = native(xyz, vms, intr)
    r = ref.compute_3d_filter(xyz, vms, intr)
    keep = ref.margins(xyz, vms, intr) > 1e-5
    excluded = int((~keep).sum())
    err = (f.double() - r.double()).abs().squeeze(1)
    bad = keep & ~(err <= ulps * ulp32(r.squeeze(1)))
    print(f"\n{what}: P={xyz.shape[0]} V={vms.shape[0]} seen={n_seen} excluded={excluded} "
          f"max|err|/ulp={float((err / ulp32(r.squeeze(1)))[keep].max()):.2f}")
    assert int(bad.sum()) == 0, (what, int(bad.sum()), f.squeeze(1)[bad][:5], r.squeeze(1)[bad][:5])
    assert excluded <= max(2, xyz.shape[0] // 1000), excluded
    return f, n_seen


def identity_cam(fx, fy, W, H, t=(0.0, 0.0, 0.0)):
    """camera coordinates = world coordinates + t (viewmatrix = I with translation row t)"""
    vm = np.eye(4, dtype=np.float32)
    vm[3, :3] = t
    return vm.reshape(16), [fx, fy, W, H]


# ---------------------------------------------------------------------------------------------------- compute
@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_compute_matches_the_official_loop_on_scenes(seed):
    import scenegen
    from diff_gaussian_rasterization import compute_3d_filter

    sc = scenegen.make_scene(P=20_000, W=320, H=240, C=0, views=8, seed=seed)
    # some Gaussians outside the ring of cameras: behind some of them, unseen by all
    sc.means3D[:500] *= 6.0
    xyz = torch.from_numpy(sc.means3D).cuda()
    rs = [settings(sc, c) for c in sc.cameras]
    from diff_gaussian_rasterization.filter3d import camera_tensors

    vms, intr = camera_tensors(rs)
    f, n_seen = check_compute(xyz, vms, intr, f"scene seed {seed}")
    assert 0 < n_seen < xyz.shape[0]
    # the public entry is the same call
    assert torch.equal(bits(compute_3d_filter(xyz, rs)), bits(f)) and f.shape == (xyz.shape[0], 1)
    # bitwise reproducible and independent of the camera order
    perm = torch.randperm(len(rs), generator=torch.Generator().manual_seed(seed))
    f2 = compute_3d_filter(xyz, [rs[int(i)] for i in perm])
    assert torch.equal(bits(f2), bits(f))
    assert torch.equal(bits(compute_3d_filter(xyz, rs[::-1])), bits(f))
    assert torch.equal(bits(compute_3d_filter(xyz, rs)), bits(f))


@pytest.mark.gpu
def test_compute_constructed_cases():
    W, H, fx, fy = 640.0, 480.0, 500.0, 800.0  # fx != fy, neither W / (2 tan) of the other's axis
    g = torch.Generator().manual_seed(3)
    pts = []
    # behind the camera, and nearer than 0.2 (just below, well below, at zero, negative)
    pts += [[0.0, 0.0, -1.0], [0.1, 0.1, -5.0], [0.0, 0.0, 0.2 * (1 - 1e-3)], [0.0, 0.0, 0.1], [0.0, 0.0, 0.0],
            [0.0, 0.0, 0.2 * (1 + 1e-3)]]
    # just inside and just outside each margin, at several depths
    for z in (0.5, 2.0, 7.0):
        for edge_x, edge_y in ((-0.15 * W, H / 2), (1.15 * W, H / 2), (W / 2, -0.15 * H), (W / 2, 1.15 * H)):
            for d in (-1e-3, 1e-3):
                px = edge_x + d * W * (1 if edge_x > W / 2 else -1) if edge_x != W / 2 else edge_x
                py = edge_y + d * H * (1 if edge_y > H / 2 else -1) if edge_y != H / 2 else edge_y
                pts.append([(px - W / 2) * z / fx, (py - H / 2) * z / fy, z])
    # a cloud in front
    cloud = torch.rand(2000, 3, generator=g) * torch.tensor([4.0, 4.0, 6.0]) - torch.tensor([2.0, 2.0, -0.5])
    xyz = torch.cat([torch.tensor(pts, dtype=torch.float32), cloud]).cuda()
    vm, it = identity_cam(fx, fy, W, H)
    vms, intr = cams_of([vm], [it])
    f, n = check_compute(xyz, vms, intr, "V=1, constructed", ulps=2)
    x, y, z = xyz.double().unbind(1)
    zc = z.clamp(min=0.001)
    px, py = x / zc * fx + W / 2, y / zc * fy + H / 2
    seen = (z > 0.2) & (px >= -0.15 * W) & (px <= 1.15 * W) & (py >= -0.15 * H) & (py <= 1.15 * H)
    # behind, below 0.2 and at 0 are unseen, just above 0.2 is seen; just inside each margin is seen, just outside not
    assert not bool(seen[:5].any()) and bool(seen[5])
    assert bool(seen[6:30:2].all()) and not bool(seen[7:30:2].any())
    assert n == int(seen.sum()) and 0 < n < xyz.shape[0]
    # an unseen Gaussian takes the largest filter of the seen ones
    assert bool((f[~seen] == f[seen].max()).all())
    # the filter is the depth over the largest fx of every camera, times sqrt(0.2): a second camera with a larger fx
    # that sees nothing new scales every row
    vm2, it2 = identity_cam(2 * fx, fy, W, H, t=(0.0, 0.0, -100.0))  # everything behind it
    vms2, intr2 = cams_of([vm, vm2], [it, it2])
    f2, n2 = check_compute(xyz, vms2, intr2, "V=2, larger fx unseen", ulps=2)
    assert n2 == n
    assert torch.equal(bits(f2 * 2), bits(f))


@pytest.mark.gpu
def test_compute_mixed_focal_lengths_and_aspects():
    g = np.random.default_rng(7)
    xyz = torch.from_numpy((g.uniform(-1, 1, (30_000, 3)) * [3, 3, 3]).astype(np.float32)).cuda()
    vms, intr = [], []
    for v in range(12):
        W, H = [(640, 480), (1920, 1080), (300, 700), (512, 512)][v % 4]
        fx, fy = W / (2 * math.tan(0.3 + 0.1 * v)), H / (2 * math.tan(0.2 + 0.07 * v)) * (1 + 0.3 * (v % 3))
        vm, it = identity_cam(np.float32(fx), np.float32(fy), W, H, t=(g.uniform(-1, 1), g.uniform(-1, 1), 2 + v))
        # a rotation about y, so that the viewmatrix is not diagonal
        a = 0.2 * v
        R = np.array([[math.cos(a), 0, -math.sin(a)], [0, 1, 0], [math.sin(a), 0, math.cos(a)]], np.float32)
        vm = vm.reshape(4, 4)
        vm[:3, :3] = R
        vms.append(vm.reshape(16))
        intr.append(it)
    vms, intr = cams_of(vms, intr)
    check_compute(xyz, vms, intr, "V=12, mixed fx / fy / W / H")


@pytest.mark.gpu
def test_compute_v300_ring_more_than_one_chunk():
    import scenegen
    from diff_gaussian_rasterization.filter3d import camera_tensors

    sc = scenegen.make_scene(P=20_000, W=400, H=300, C=0, views=300, seed=5)
    sc.means3D[:300] *= 8.0
    xyz = torch.from_numpy(sc.means3D).cuda()
    vms, intr = camera_tensors([settings(sc, c) for c in sc.cameras])
    f, _ = check_compute(xyz, vms, intr, "V=300 ring")
    perm = torch.randperm(300, generator=torch.Generator().manual_seed(1)).cuda()
    assert torch.equal(bits(native(xyz, vms[perm], intr[perm])[0]), bits(f))


@pytest.mark.gpu
def test_compute_raises_when_nothing_is_seen():
    from diff_gaussian_rasterization.filter3d import compute_from_tensors

    vm, it = identity_cam(500.0, 500.0, 640, 480)
    vms, intr = cams_of([vm], [it])
    xyz = torch.tensor([[0.0, 0.0, -1.0], [0.0, 0.0, 0.1], [100.0, 0.0, 1.0]], device="cuda")
    with pytest.raises(ValueError, match="no Gaussian is seen"):
        compute_from_tensors(xyz, vms, intr)
    assert native(xyz, vms, intr)[1] == 0


# ---------------------------------------------------------------------------------------------------- apply
def _apply_inputs(P=60_000, seed=0):
    g = torch.Generator().manual_seed(seed)
    s = torch.pow(10.0, torch.rand(P, 3, generator=g) * 8.0 - 6.0)  # 1e-6 .. 1e2, per axis
    o = torch.rand(P, 1, generator=g) * 0.999 + 1e-4
    kind = torch.arange(P) % 4
    f = torch.where(kind == 0, torch.zeros(P), torch.where(kind == 1, torch.full((P,), 1e-30),
                    torch.pow(10.0, torch.rand(P, generator=g) * 8.0 - 6.0) * torch.where(kind == 3, 100.0, 1.0)))
    return o.cuda(), s.cuda(), f[:, None].cuda()


@pytest.mark.gpu
def test_apply_forward_is_the_official_formula_bitwise():
    from diff_gaussian_rasterization import _C

    o, s, f = _apply_inputs()
    of, sf = _C.filter3d_apply(o, s, f)
    ro, rs = ref.opacity_with_3d_filter(o, s, f), ref.scaling_with_3d_filter(s, f)
    assert torch.equal(bits(of), bits(ro)), int((bits(of) != bits(ro)).sum())
    assert torch.equal(bits(sf), bits(rs)), int((bits(sf) != bits(rs)).sum())
    assert bool(torch.isfinite(of).all()) and bool((of <= o).all())
    # underflowed det1: coef and o_f are 0 in both
    tiny = torch.full((4, 3), 1e-14, device="cuda")
    of, _ = _C.filter3d_apply(o[:4], tiny, torch.full((4, 1), 1e-3, device="cuda"))
    assert torch.equal(of, torch.zeros_like(of))


@pytest.mark.gpu
def test_apply_backward_matches_float64_autograd_and_runs_in_place():
    from diff_gaussian_rasterization import _C

    o, s, f = _apply_inputs(seed=1)
    g = torch.Generator(device="cuda").manual_seed(2)
    gof, gsf = torch.randn(o.shape, device="cuda", generator=g), torch.randn(s.shape, device="cuda", generator=g)
    go, gs = _C.filter3d_apply_backward(o, s, f, gof, gsf)
    o64, s64 = o.double().requires_grad_(True), s.double().requires_grad_(True)
    of64, sf64 = ref.apply64(o64, s64, f)
    # the two terms of dL/ds separately, to scale the tolerance of their sum
    t1 = torch.autograd.grad(sf64, s64, gsf.double(), retain_graph=True)[0]
    ro, t2 = torch.autograd.grad(of64, (o64, s64), gof.double())
    # rows where the float32 formula itself underflows (a partial product of det1, or det1 / det2, below FLT_MIN: coef
    # is then 0 or subnormal in float32, in the official formula as here) are compared for finiteness only
    s2, tiny = s.double().square(), torch.finfo(torch.float32).tiny
    det1 = s2.prod(1)
    normal = ((s2[:, 0] * s2[:, 2] >= tiny) & (det1 >= tiny) & (det1 / (s2 + f.double().square()).prod(1) >= tiny))
    print(f"\nbackward: {int((~normal).sum())} of {normal.numel()} rows underflow in float32")
    assert int((~normal).sum()) < normal.numel() // 4
    assert bool(torch.isfinite(go).all()) and bool(torch.isfinite(gs).all())
    go, ro, gs_, t1, t2 = go[normal], ro[normal], gs[normal], t1[normal], t2[normal]
    assert torch.all((go.double() - ro).abs() <= 1e-5 * ro.abs()), float(((go.double() - ro).abs() / ro.abs()).max())
    err = (gs_.double() - (t1 + t2)).abs()
    assert torch.all(err <= 1e-5 * (t1.abs() + t2.abs()) + 1e-37), float((err / (t1.abs() + t2.abs())).max())
    go, gs = _C.filter3d_apply_backward(o, s, f, gof, gsf)
    # in place over the upstream gradients: the same bits
    a, b = gof.clone(), gsf.clone()
    ra, rb = _C.filter3d_apply_backward(o, s, f, a, b, a, b)
    assert ra.data_ptr() == a.data_ptr() and rb.data_ptr() == b.data_ptr()
    assert torch.equal(bits(a), bits(go)) and torch.equal(bits(b), bits(gs))
    # an underflowed det1 (o_f == 0) and s == 0 give no NaN
    s0 = torch.tensor([[1e-20, 1e-20, 1e-20], [0.0, 1.0, 1.0], [1e-25, 2.0, 3.0]], device="cuda")
    f0 = torch.full((3, 1), 1e-3, device="cuda")
    go0, gs0 = _C.filter3d_apply_backward(o[:3], s0, f0, gof[:3], gsf[:3])
    assert bool(torch.isfinite(go0).all()) and bool(torch.isfinite(gs0).all())


# ---------------------------------------------------------------------------------------------------- end to end
def _render(sc, cam, opac, scales, rest):
    from diff_gaussian_rasterization import GaussianRasterizer

    means2D = torch.zeros_like(rest["means3D"], requires_grad=True)
    return GaussianRasterizer(settings(sc, cam))(means3D=rest["means3D"], means2D=means2D, opacities=opac,
                                                 shs=rest["shs"], semantic_feature=rest["semantic_feature"],
                                                 scales=scales, rotations=rest["rotations"])


@pytest.mark.gpu
def test_apply_3d_filter_with_the_rasterizer_matches_the_reference_properties():
    import scenegen
    from diff_gaussian_rasterization import apply_3d_filter, compute_3d_filter

    sc = scenegen.make_config("small", views=3)
    t = scenegen.to_torch(sc, "cuda")
    rs = [settings(sc, c) for c in sc.cameras]
    f = compute_3d_filter(t["means3D"], rs) * 3.0  # large enough to change most Gaussians
    up = scenegen.upstream_grads(sc.cameras[0].image_height, sc.cameras[0].image_width, sc.C)
    up = [torch.from_numpy(u).cuda() for u in up]
    outs = []
    for native_filter in (True, False):
        o = t["opacities"].clone().requires_grad_(True)
        s = t["scales"].clone().requires_grad_(True)
        if native_filter:
            of, sf = apply_3d_filter(o, s, f)
        else:
            of, sf = ref.opacity_with_3d_filter(o, s, f), ref.scaling_with_3d_filter(s, f)
        color, feat, radii, depth = _render(sc, sc.cameras[0], of, sf, t)
        torch.autograd.backward([color, feat, depth], up)
        outs.append((color.detach(), feat.detach(), depth.detach(), o.grad, s.grad))
    for a, b in zip(outs[0][:3], outs[1][:3]):
        assert torch.equal(bits(a), bits(b))
    for a, b in zip(outs[0][3:], outs[1][3:]):
        scale = float(b.abs().max())
        assert scale > 0 and torch.allclose(a, b, rtol=1e-4, atol=1e-5 * scale), float((a - b).abs().max()) / scale


# ---------------------------------------------------------------------------------------------------- training
def _state(sc, feature_dtype=torch.float32):
    import scenegen
    from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid

    t = scenegen.to_torch(sc, "cuda")
    return GaussianState(t["means3D"].clone(), t["shs"][:, :1].contiguous(), t["shs"][:, 1:].contiguous(),
                         inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                         t["rotations"].clone(), t["semantic_feature"].clone(), feature_dtype=feature_dtype)


LRS = dict(xyz=1.6e-4, f_dc=2.5e-3, f_rest=1.25e-4, opacity=0.05, scaling=5e-3, rotation=1e-3, semantic_feature=0.05)


def _targets(sc):
    g = torch.Generator(device="cuda").manual_seed(11)
    H, W = sc.cameras[0].image_height, sc.cameras[0].image_width
    return [(torch.rand(3, H, W, device="cuda", generator=g), torch.rand(sc.C, H, W, device="cuda", generator=g))
            for _ in sc.cameras]


@pytest.mark.gpu
@pytest.mark.parametrize("sparse", [False, True], ids=["dense", "sparse"])
def test_gaussian_state_training_matches_the_torch_reference(sparse):
    """Three steps of ViewBatch forward, colour + feature L1, backward, all_reduce and step() with the filter on,
    against the reference's properties + GaussianRasterizer + torch.optim.Adam(eps=1e-15) on the raw parameters."""
    import scenegen
    import torch.nn.functional as F
    from diff_gaussian_rasterization.trainer import GaussianState

    sc = scenegen.make_config("small", views=2)
    # a corner of the cloud that no view sees: zero gradients there
    st = _state(sc)
    rs = [settings(sc, c) for c in sc.cameras]
    st.compute_3d_filter(rs)
    filt = st.filter_3d.clone()
    raw = {k: v.clone().requires_grad_(True) for k, v in st.raw.items()}
    opt = torch.optim.Adam([{"params": [raw[k]], "lr": LRS[k]} for k in GaussianState.NAMES], lr=0.0, eps=1e-15)
    tg = _targets(sc)
    for step in range(3):
        st.activate()
        vb = st.batch()
        vb.zero_()
        for v, r in enumerate(rs):
            color, feat, radii, depth, ctx = vb.forward(r)
            n_c, n_f = color.numel(), feat.numel()
            vb.backward(ctx, torch.sign(color - tg[v][0]) / n_c, torch.sign(feat - tg[v][1]) / n_f,
                        torch.zeros_like(depth), last=v == len(rs) - 1)
        vb.all_reduce()
        visible = vb.visible() if sparse else None
        st.step(LRS, visible=visible)

        opt.zero_grad()
        o = ref.opacity_with_3d_filter(torch.sigmoid(raw["opacity"]), torch.exp(raw["scaling"]), filt)
        s = ref.scaling_with_3d_filter(torch.exp(raw["scaling"]), filt)
        rest = dict(means3D=raw["xyz"], shs=torch.cat((raw["f_dc"], raw["f_rest"]), dim=1),
                    rotations=F.normalize(raw["rotation"]), semantic_feature=raw["semantic_feature"])
        loss = 0.0
        for v, cam in enumerate(sc.cameras):
            color, feat, radii, depth = _render(sc, cam, o, s, rest)
            loss = loss + (color - tg[v][0]).abs().mean() + (feat - tg[v][1]).abs().mean()
        loss.backward()
        before = {k: (raw[k].detach().clone(), {n: x.clone() for n, x in opt.state[raw[k]].items()} if opt.state else {})
                  for k in raw}
        opt.step()
        if sparse:  # the reference's sparse step: rows no view saw keep their parameters and moments
            keep = ~visible
            with torch.no_grad():
                for k in raw:
                    p0, m0 = before[k]
                    raw[k][keep] = p0[keep]
                    for n in ("exp_avg", "exp_avg_sq"):
                        if n in m0:
                            opt.state[raw[k]][n][keep] = m0[n][keep]
                        else:
                            opt.state[raw[k]][n][keep] = 0.0
        for k in GaussianState.NAMES:
            a, b = st.raw[k], raw[k].detach()
            err = (a - b).abs()
            # Adam normalises each update: rows whose gradient is at rounding level may step
            # either way, by a bounded multiple of lr
            assert float(err.max()) <= 8 * LRS[k] * (step + 1) + 1e-6, (k, step, float(err.max()))
            close = torch.isclose(a, b, rtol=1e-4, atol=1e-6)
            assert float((~close).float().mean()) <= 2e-3, (k, step, float((~close).float().mean()))


@pytest.mark.gpu
def test_filter_off_adds_nothing_and_regularizers_refuse_the_filter():
    import scenegen
    from diff_gaussian_rasterization import _C

    sc = scenegen.make_config("small", views=2)
    st = _state(sc)
    n0 = _C.launch_count()
    st.activate()
    plain = _C.launch_count() - n0
    assert st.filter_3d is None and st._unfiltered is None
    st.batch()
    st.add_regularizer_grads(0.01, 0.01)
    with pytest.raises(ValueError):
        st.compute_3d_filter()  # never computed, no cameras kept
    st.compute_3d_filter([settings(sc, c) for c in sc.cameras])
    n0 = _C.launch_count()
    st.activate()
    assert _C.launch_count() - n0 == plain + 1  # the apply kernel
    with pytest.raises(ValueError, match="3D filter"):
        st.add_regularizer_grads(0.01, 0.01)


# ---------------------------------------------------------------------------------------------------- densify, reset, export
@pytest.mark.gpu
def test_densify_and_relocate_recompute_the_filter():
    import scenegen
    from diff_gaussian_rasterization import compute_3d_filter

    sc = scenegen.make_config("small", views=2)
    st = _state(sc)
    rs = [settings(sc, c) for c in sc.cameras]
    st.compute_3d_filter(rs)
    vb = st.batch()
    vb.zero_()
    vb.grad_accum.normal_().abs_()
    vb.denom.fill_(1.0)
    P0 = st.P
    n = st.densify_and_prune(max_grad=0.5, min_opacity=0.005, extent=4.0, max_screen_size=None,
                             generator=torch.Generator(device="cuda").manual_seed(0))
    assert n != P0 and st.filter_3d.shape == (n, 1)
    assert torch.equal(bits(st.filter_3d), bits(compute_3d_filter(st.raw["xyz"], rs)))
    st.activate()
    assert st.act["opacities"].shape == (n, 1)
    st.relocate_and_add(int(n * 1.03), generator=torch.Generator(device="cuda").manual_seed(1))
    assert st.filter_3d.shape == (st.P, 1)
    assert torch.equal(bits(st.filter_3d), bits(compute_3d_filter(st.raw["xyz"], rs)))


@pytest.mark.gpu
def test_filtered_reset_opacity_is_the_official_reset():
    import scenegen

    sc = scenegen.make_config("small", views=2)
    st = _state(sc)
    st.raw["scaling"][:50] = -40.0  # det1 underflows: coef == 0
    st.compute_3d_filter([settings(sc, c) for c in sc.cameras])
    st.exp_avg["opacity"].fill_(1.0)
    st.exp_avg_sq["opacity"].fill_(1.0)
    r_op, r_sc, f = st.raw["opacity"].clone(), st.raw["scaling"].clone(), st.filter_3d
    want = ref.reset_opacity(r_op, r_sc, f)
    st.reset_opacity()
    s2 = torch.exp(r_sc).square()
    coef = torch.sqrt(s2.prod(1) / (s2 + f.square()).prod(1))
    pos = coef > 0
    assert int((~pos).sum()) == 50
    assert torch.equal(bits(st.raw["opacity"][pos]), bits(want[pos]))
    # where the official formula is 0 / 0: the unfiltered reset
    x = torch.min(torch.sigmoid(r_op[~pos]), torch.full_like(r_op[~pos], 0.01))
    assert torch.equal(bits(st.raw["opacity"][~pos]), bits(torch.log(x / (1 - x))))
    assert not bool(st.exp_avg["opacity"].any()) and not bool(st.exp_avg_sq["opacity"].any())
    # the filtered opacity is now at most 0.01
    st.activate()
    assert float(st.act["opacities"].max()) <= 0.01 * (1 + 1e-6)


@pytest.mark.gpu
def test_baked_raw_renders_like_the_filter():
    import scenegen
    from diff_gaussian_rasterization.trainer import GaussianState

    sc = scenegen.make_config("small", views=2)
    st = _state(sc)
    assert st.baked_raw()["opacity"] is st.raw["opacity"]  # filter off: the raw parameters
    st.compute_3d_filter([settings(sc, c) for c in sc.cameras])
    st.activate()
    baked = st.baked_raw()
    plain = GaussianState(*(baked[k].clone() for k in GaussianState.NAMES))
    plain.activate()
    assert torch.allclose(plain.act["opacities"], st.act["opacities"], rtol=1e-5, atol=1e-7)
    assert torch.allclose(plain.act["scales"], st.act["scales"], rtol=1e-5, atol=0)
    for cam in sc.cameras:
        r = settings(sc, cam)
        a = st.batch().forward(r)
        b = plain.batch().forward(r)
        for x, y in zip(a[:2] + a[3:4], b[:2] + b[3:4]):
            scale = float(y.abs().max())
            assert torch.allclose(x, y, rtol=1e-4, atol=1e-4 * scale), float((x - y).abs().max()) / scale
