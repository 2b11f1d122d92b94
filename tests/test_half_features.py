"""Float16 feature fields in the forward composite (csrc/composite_fwd.cu, f3dgs_forward_f16, the binding's dtype rule).

The feature map has the dtype of `semantic_feature`.  Converting float16 to float32 is exact and the kernel keeps the
float32 accumulation, so a float16 render has an exact definition: the feature map is bitwise
`render(sf16.float())[feature_map].half()`, and colour, depth, radii, final_T, n_contrib and the tile lists are bitwise
the float32 render's.  The GPU part checks exactly that over the copy paths of the kernel (bulk copies for C % 8 == 0
and 16-byte aligned rows, scalar loads otherwise) and its store paths (16-byte rows for W % 8 == 0, 8-byte groups for
W % 4 == 0, scalar stores otherwise), and that autograd through a float16 render gives float16 gradients that match the
float32 path's.  CPU part (`-m "not gpu"`): f3dgs_forward_f16 rejects bad arguments before any CUDA call.
"""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

import parity
import scenegen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEOM_GRADS = ("means3D", "means2D", "opacities", "shs", "scales", "rotations")


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_launch_count.restype = ctypes.c_ulonglong
    return L


# ---- CPU: C ABI validation (fake addresses, never dereferenced: every call below fails validation)
def test_forward_f16_rejects_bad_arguments_before_touching_cuda(lib):
    launches = lib.f3dgs_launch_count()
    CB = ctypes.CFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t)
    cb = CB(lambda ctx, n: None)
    null = ctypes.c_void_p(0)
    m3, op, bg, vm, pm, cp, col, dep, sh, sc, rot, sf, fm = (ctypes.c_void_p(k << 24) for k in range(1, 14))

    def call(P=10, C=4, W=64, H=64, D=3, allocs=True, ptrs=True, feat=True):
        a = cb if allocs else ctypes.cast(null, CB)
        p = (lambda x: x) if ptrs else (lambda x: null)
        f = (lambda x: x) if feat else (lambda x: null)
        return lib.f3dgs_forward_f16(a, null, a, null, a, null, P, D, 16, C, p(bg), W, H, p(m3), sh, null, f(sf),
                                     p(op), sc, ctypes.c_float(1.0), rot, null, p(vm), p(pm), p(cp),
                                     ctypes.c_float(0.5), ctypes.c_float(0.5), 0, p(col), f(fm), p(dep), null, 0, null)

    def rejected(msg, **kw):
        assert call(**kw) == -1, kw
        err = lib.f3dgs_last_error()
        assert err.startswith(b"f3dgs_forward_f16: ") and msg in err, (kw, err)

    rejected(b"bad sizes", P=-1)
    rejected(b"bad sizes", C=-1)
    rejected(b"bad sizes", C=4097)  # F3DGS_MAX_FEATURE_DIM + 1
    rejected(b"bad sizes", W=0)
    rejected(b"bad sizes", H=-3)
    rejected(b"bad sizes", D=4)
    rejected(b"allocator", allocs=False)
    rejected(b"NULL required pointer", ptrs=False)
    rejected(b"C > 0 needs semantic_feature and out_feature_map", feat=False)
    assert call(P=0) == 0  # empty cloud: nothing to do
    # the float32 symbol names itself too, and a failure of one does not leak into the other's message
    args = [ctypes.cast(null, CB), null] * 3 + [10, 3, 16, 4, null, 64, 64] + [null] * 6 + [
        ctypes.c_float(1.0)] + [null] * 5 + [ctypes.c_float(0.5), ctypes.c_float(0.5), 0] + [null] * 4 + [0, null]
    assert len(args) == 34
    assert lib.f3dgs_forward(*args) == -1 and lib.f3dgs_last_error().startswith(b"f3dgs_forward: ")
    rejected(b"bad sizes", P=-1)
    assert lib.f3dgs_launch_count() == launches


# =================================================================================================== GPU
def _render(t, rs, sf):
    """One forward through the torch binding, with the internal lists; everything stays on the device."""
    from diff_gaussian_rasterization import _C

    e = torch.Tensor([])
    R, color, feat, depth, radii, geom, binning, img = _C.rasterize_gaussians(
        rs["bg"], t["means3D"], e, sf, t["opacities"], t["scales"], t["rotations"], rs["scale_modifier"], e,
        rs["viewmatrix"], rs["projmatrix"], rs["tanfovx"], rs["tanfovy"], rs["image_height"], rs["image_width"],
        t["shs"], rs["sh_degree"], rs["campos"], rs["prefiltered"], False)
    out = dict(num_rendered=R, color=color, feature_map=feat, depth=depth, radii=radii)
    if t["means3D"].shape[0]:
        pl, ranges, n_contrib, final_T, _ = _C.debug_views(geom, binning, img, t["means3D"].shape[0],
                                                           rs["image_width"], rs["image_height"], R)
        out.update(point_list=pl, ranges=ranges, n_contrib=n_contrib, final_T=final_T)
    return out


def _bits(x):
    return x.view(torch.int16) if x.dtype == torch.float16 else x.view(torch.int32) if x.dtype == torch.float32 else x


def _check_half_render(t, rs, sf16):
    """render(sf16) against render(sf16.float()): the map bitwise after .half(), everything else bitwise."""
    r16 = _render(t, rs, sf16)
    r32 = _render(t, rs, sf16.float())
    C = sf16.shape[-1]
    fm = r16["feature_map"]
    assert fm.dtype == torch.float16 and fm.shape == (C, rs["image_height"], rs["image_width"])
    assert r32["feature_map"].dtype == torch.float32
    assert torch.equal(_bits(fm), _bits(r32["feature_map"].half()))
    assert r16["num_rendered"] == r32["num_rendered"]
    for k in ("color", "depth", "radii", "final_T", "n_contrib", "point_list", "ranges"):
        assert r16[k].dtype == r32[k].dtype and torch.equal(_bits(r16[k]), _bits(r32[k])), k
    return r16, r32


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _small(W=96, H=64):
    sc = scenegen.make_scene(P=1500, W=W, H=H, C=0, sh_degree=1, seed=7)  # test_wide_features.py's small scene
    return sc, scenegen.to_torch(sc, "cuda"), parity.settings(sc, sc.cameras[0], "cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 3, 13, 32, 64, 128, 129, 512, 516, 4096])
def test_half_render_is_the_float_render_rounded(C):
    sc, t, rs = _small()
    sf16 = torch.randn(sc.P, 1, C, device="cuda", generator=_gen(C)).half()
    r16, _ = _check_half_render(t, rs, sf16)
    assert float(r16["feature_map"].float().abs().max()) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("W,H", [(94, 50), (100, 37), (97, 61), (40, 17)])
@pytest.mark.parametrize("C", [8, 64, 128, 256])
def test_half_render_at_image_widths_off_the_vector_stores(W, H, C):
    """W % 8 != 0 (no 16-byte rows), W % 4 != 0 (no 8-byte groups either) and a partial last tile row."""
    sc, t, rs = _small(W, H)
    sf16 = torch.randn(sc.P, 1, C, device="cuda", generator=_gen(W * C)).half()
    _check_half_render(t, rs, sf16)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [8, 128, 512])
def test_half_render_of_features_at_an_odd_offset(C):
    """Features one element into their storage: the rows are not 16-byte aligned, so no bulk copies."""
    sc, t, rs = _small()
    base = torch.randn(sc.P * C + 1, device="cuda", generator=_gen(C + 1)).half()
    sf16 = base[1:].view(sc.P, 1, C)
    assert sf16.is_contiguous() and sf16.data_ptr() % 16 != 0
    _check_half_render(t, rs, sf16)


@pytest.mark.gpu
@pytest.mark.parametrize("name,C", [("c2", 16), ("c3", 128), ("c3", 512)])
def test_half_render_on_config_clouds(name, C):
    sc = scenegen.make_config(name)
    sc.features = np.zeros((sc.P, 1, 0), np.float32)  # the width is given below
    t = scenegen.to_torch(sc, "cuda")
    rs = parity.settings(sc, sc.cameras[0], "cuda")
    sf16 = torch.randn(sc.P, 1, C, device="cuda", generator=_gen(C)).half()
    r16, r32 = _check_half_render(t, rs, sf16)
    print(f"[{name} C={C}] R={r16['num_rendered']}")


@pytest.mark.gpu
def test_half_render_of_an_empty_cloud():
    sc, t, rs = _small()
    empty = {k: v[:0] for k, v in t.items() if k != "bg"}
    for C in (0, 16):
        r = _render(empty, rs, torch.empty(0, 1, C, device="cuda", dtype=torch.float16))
        assert r["num_rendered"] == 0
        assert r["feature_map"].dtype == torch.float16 and r["feature_map"].shape == (C, 64, 96)
        assert not r["feature_map"].any() and not r["color"].any()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.bfloat16])
def test_binding_rejects_other_feature_dtypes(dtype):
    sc, t, rs = _small()
    sf = torch.randn(sc.P, 1, 8, device="cuda").to(dtype)
    with pytest.raises(RuntimeError, match="semantic_feature must be float32 or float16"):
        _render(t, rs, sf)


def _autograd(sc, sf, gc, gf, gd):
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer

    t = scenegen.to_torch(sc, "cuda", requires_grad=True)
    means2D = torch.zeros_like(t["means3D"], requires_grad=True)
    rs = GaussianRasterizationSettings(**parity.settings(sc, sc.cameras[0], "cuda"))
    color, feat, radii, depth = GaussianRasterizer(rs)(
        means3D=t["means3D"], means2D=means2D, opacities=t["opacities"], shs=t["shs"], semantic_feature=sf,
        scales=t["scales"], rotations=t["rotations"])
    torch.autograd.backward([color, feat, depth], [gc, gf.to(feat.dtype), gd])
    g = {k: t[k].grad for k in ("means3D", "opacities", "shs", "scales", "rotations")}
    g["means2D"] = means2D.grad
    return feat, g


def _viol(a, b, extra=None):
    """Worst |a - b| over the gradient tolerance of the parity bar (+ `extra`), <= 1 passes."""
    a, b = a.double(), b.double()
    tol = parity.RTOL * b.abs() + parity.GRAD_ATOL_REL * b.abs().max() + 1e-30
    if extra is not None:
        tol = tol + extra
    return float(((a - b).abs() / tol).max())


def _half_ulp(x):
    """Half a float16 ulp at |x| (subnormal spacing below 2^-14)."""
    e = torch.floor(torch.log2(x.double().abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 11)


@pytest.mark.gpu
@pytest.mark.parametrize("name,C", [("small", 16), ("small128", 128), ("small200", 200)])
def test_autograd_through_a_half_render(name, C):
    sc = scenegen.make_config(name)
    cam = sc.cameras[0]
    H, W = cam.image_height, cam.image_width
    g = _gen(C)
    sf16 = torch.randn(sc.P, 1, C, device="cuda", generator=g).half().requires_grad_(True)
    sf32 = sf16.detach().float().requires_grad_(True)
    gc, gd = torch.randn(3, H, W, device="cuda", generator=g), torch.randn(1, H, W, device="cuda", generator=g)
    gf16 = torch.randn(C, H, W, device="cuda", generator=g).half()  # the same upstream gradient for both paths

    fm16, g16 = _autograd(sc, sf16, gc, gf16, gd)
    fm32, g32 = _autograd(sc, sf32, gc, gf16.float(), gd)
    assert fm16.dtype == torch.float16 and torch.equal(_bits(fm16.detach()), _bits(fm32.detach().half()))
    assert sf16.grad.dtype == torch.float16 and sf16.grad.shape == sf16.shape
    assert float(sf32.grad.abs().max()) > 0
    v = _viol(sf16.grad.float(), sf32.grad, extra=_half_ulp(sf16.grad.float()))
    worst = {k: _viol(g16[k], g32[k]) for k in GEOM_GRADS}
    print(f"[{name} C={C}] dL/dfeature viol {v:.3g}; geometric: " + ", ".join(f"{k}={x:.3g}" for k, x in worst.items()))
    assert v <= 1.0
    for k, x in worst.items():
        assert g16[k].dtype == torch.float32 and x <= 1.0, (k, x)


@pytest.mark.gpu
def test_half_render_makes_no_float32_map():
    """A float16 render at C = 512 grows peak memory by less than one float32 [C,H,W] map."""
    C, W, H = 512, 960, 544
    sc = scenegen.make_scene(P=20000, W=W, H=H, C=0, sh_degree=1, seed=11)
    t = scenegen.to_torch(sc, "cuda")
    rs = parity.settings(sc, sc.cameras[0], "cuda")
    sf16 = torch.randn(sc.P, 1, C, device="cuda", generator=_gen(5)).half()
    _render(t, rs, sf16)  # warm-up: module load, scratch sizes
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    r = _render(t, rs, sf16)
    torch.cuda.synchronize()
    grew = torch.cuda.max_memory_allocated() - base
    map32 = C * H * W * 4
    print(f"peak growth {grew / 2**20:.1f} MiB, float16 map {map32 / 2**21:.1f} MiB, "
          f"float32 map {map32 / 2**20:.1f} MiB")
    assert r["feature_map"].dtype == torch.float16
    assert grew < map32


@pytest.mark.gpu
def test_rendered_half_map_feeds_pca_query_and_io(tmp_path):
    from diff_gaussian_rasterization import feature_head as fh

    spec = importlib.util.spec_from_file_location(
        "f3dgs_io_half_render", os.path.join(ROOT, "feature-3dgs_b200", "diff_gaussian_rasterization", "io.py"))
    io = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(io)

    C = 16
    sc, t, rs = _small()
    sf16 = torch.randn(sc.P, 1, C, device="cuda", generator=_gen(3)).half()
    fm = _render(t, rs, sf16)["feature_map"]
    assert fm.dtype == torch.float16 and fm.is_contiguous()

    img16, img32 = fh.pca_image(fm), fh.pca_image(fm.float())
    assert img16.shape == (64, 96, 3) and torch.equal(img16, img32)

    text = torch.randn(5, C, device="cuda", generator=_gen(4))
    lab16, prob16, _ = fh.query(fm, text, positive=[0, 2])
    lab32, prob32, _ = fh.query(fm.float(), text, positive=[0, 2])
    assert torch.equal(lab16, lab32) and torch.equal(prob16, prob32)

    path = str(tmp_path / io.fmap_filename("00000", C, 64, 96))
    io.save_feature_map(path, fm)
    back = io.load_feature_map(path, dtype=None)
    assert back.dtype == torch.float16 and torch.equal(_bits(back), _bits(fm.cpu()))
