"""Float16 teacher maps in the fused feature losses, and float16 decoded maps (csrc/feature_head.cu, csrc/feature_decoder.cu,
the _f16gt / _f16 symbols of include/f3dgs_b200.h, diff_gaussian_rasterization/feature_head.py and io.py).

Converting float16 to float32 is exact, so every float16 path has an exact definition: the float32 path applied to
gt.float(), or for the decode, decode(...).half().  The GPU part checks exactly that, bitwise, and that no float32 copy of the
teacher map is made.  CPU part (`-m "not gpu"`): the C ABI rejects bad arguments before any CUDA call, and the feature-map
loader keeps the stored float16 on request.
"""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.next_rows import resize_bilinear_ac, resize_bilinear_ac_bwd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DECODE_REL = 1.2e-3  # the TF32 decode bar of test_feature_decoder.py
# test_next_rows.py SHAPES plus the LSeg --speedup sizes (map 1080x1920, teacher 480x853) and LSeg's full width (C = 512)
RESIZE_SHAPES = [((5, 37, 53), (21, 30)), ((3, 16, 16), (16, 16)), ((4, 20, 31), (45, 64)), ((2, 9, 7), (1, 1)),
                 ((6, 54, 96), (24, 43)), ((128, 1080, 1920), (480, 853)), ((512, 270, 480), (120, 160))]
DECODER_SHAPES = [(1, 1, 1), (5, 7, 1000), (16, 64, 4099), (128, 512, 409440), (256, 33, 777)]  # test_feature_decoder.py


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_launch_count.restype = ctypes.c_ulonglong
    L.f3dgs_feature_resize_fwd_f16gt.argtypes = [ctypes.c_int] * 5 + [ctypes.c_void_p] * 2 + [ctypes.c_float] + \
        [ctypes.c_void_p] * 3
    L.f3dgs_decoder_l1_f16gt.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 4 + [ctypes.c_float] + [ctypes.c_void_p] * 5
    L.f3dgs_decoder_forward_f16.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 5
    return L


@pytest.fixture(scope="module")
def io_module():
    path = os.path.join(ROOT, "feature-3dgs_b200", "diff_gaussian_rasterization", "io.py")
    spec = importlib.util.spec_from_file_location("f3dgs_io_half", path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


# ---- CPU: C ABI validation (fake addresses, never dereferenced: every call below fails validation)
def test_f16_symbols_reject_bad_arguments_before_touching_cuda(lib):
    launches = lib.f3dgs_launch_count()
    fm, gt, out, ls, W, b, x, dx, dW, db = (k << 24 for k in range(1, 11))

    def rz(C=2, H=4, Wd=5, Hg=3, Wg=3, f=fm, g=gt, o=out):
        return lib.f3dgs_feature_resize_fwd_f16gt(C, H, Wd, Hg, Wg, f, g, 0.5, o, ls, None)

    assert rz(C=-1) == -1 and b"bad sizes" in lib.f3dgs_last_error()
    assert rz(H=0) == -1 and rz(Wd=0) == -1 and rz(Hg=0) == -1 and rz(Wg=-2) == -1
    for kw in ("f", "o", "g"):  # gt is required: resizing without a target is the float32 symbol's job
        assert rz(**{kw: None}) == -1 and b"NULL pointer" in lib.f3dgs_last_error(), kw
    n = 2 * 3 * 3  # C * Hg * Wg elements: out has 4 n bytes, gt 2 n bytes, feature_map 4 * 2 * 4 * 5 bytes
    assert rz(o=gt) == -1 and b"overlaps" in lib.f3dgs_last_error()
    assert rz(o=gt + 2 * n - 2) == -1          # out's first element over gt's last
    assert rz(o=gt - 4 * n + 2) == -1          # out's last bytes over gt's first element
    assert rz(o=fm) == -1 and rz(o=fm + 4 * 40 - 4) == -1 and rz(o=fm - 4 * n + 4) == -1

    def l1(Cin=16, Cout=64, N=100, w=W, bias=b, xx=x, g=gt, s=ls, d=dx, dw=dW, dbb=db):
        return lib.f3dgs_decoder_l1_f16gt(Cin, Cout, N, w, bias, xx, g, 0.5, s, d, dw, dbb, None)

    assert l1(Cin=0) == -1 and b"bad sizes" in lib.f3dgs_last_error()
    assert l1(Cin=257) == -1 and l1(Cout=0) == -1 and l1(Cout=4097) == -1 and l1(N=0) == -1 and l1(N=-5) == -1
    for kw in ("w", "xx", "g", "s", "d", "dw"):
        assert l1(**{kw: None}) == -1 and b"NULL pointer" in lib.f3dgs_last_error(), kw
    assert l1(dbb=None) == -1 and b"dL_dbias goes with bias" in lib.f3dgs_last_error()
    assert l1(bias=None) == -1
    assert l1(d=x) == -1 and b"overlaps" in lib.f3dgs_last_error()
    assert l1(d=gt) == -1 and l1(d=W) == -1 and l1(d=dW) == -1 and l1(d=b) == -1 and l1(d=db) == -1
    assert l1(d=gt + 2 * 64 * 100 - 2) == -1   # dL_dx's first element over gt's last (2-byte) element
    assert l1(d=gt - 4 * 16 * 100 + 2) == -1   # dL_dx's last element over gt's first

    def fwd(Cin=8, Cout=8, N=10, w=W, bias=b, xx=x, y=out):
        return lib.f3dgs_decoder_forward_f16(Cin, Cout, N, w, bias, xx, y, None)

    assert fwd(Cin=300) == -1 and b"bad sizes" in lib.f3dgs_last_error()
    assert fwd(Cout=0) == -1 and fwd(N=0) == -1
    for kw in ("w", "xx", "y"):
        assert fwd(**{kw: None}) == -1 and b"NULL pointer" in lib.f3dgs_last_error(), kw
    assert fwd(y=x) == -1 and b"overlaps" in lib.f3dgs_last_error()
    assert fwd(y=W + 4) == -1 and fwd(y=b) == -1
    assert fwd(y=x - 2 * 8 * 10 + 2) == -1     # y's last (2-byte) element over x's first
    assert fwd(y=x + 4 * 8 * 10 - 4) == -1     # y's first element over x's last
    assert lib.f3dgs_launch_count() == launches


def test_load_feature_map_keeps_float16_on_request(tmp_path, io_module):
    fm = torch.from_numpy(np.random.default_rng(3).normal(size=(12, 9, 11)).astype(np.float32))
    path = str(tmp_path / io_module.fmap_filename("00007", 12, 9, 11))
    io_module.save_feature_map(path, fm)
    stored = torch.load(path)
    kept = io_module.load_feature_map(path, dtype=None)
    assert kept.dtype == torch.float16 and torch.equal(kept.view(torch.int16), stored.view(torch.int16))
    default = io_module.load_feature_map(path)
    assert default.dtype == torch.float32 and torch.equal(default, stored.float())
    assert torch.equal(io_module.load_feature_map(path, dtype=torch.float32), default)


# =================================================================================================== GPU
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,size", RESIZE_SHAPES)
def test_resize_l1_with_half_target_equals_upcast_target(shape, size):
    from diff_gaussian_rasterization import _C
    from diff_gaussian_rasterization import feature_head as fh

    g = _gen(1)
    fm = torch.randn(shape, device="cuda", generator=g)
    g16 = torch.randn((shape[0],) + size, device="cuda", generator=g).half()
    g16.view(-1)[::5] = fh.resize_bilinear(fm, size).half().view(-1)[::5]  # some residuals near zero
    g32 = g16.float()
    gs = 0.7 / g16.numel()
    out16, ls16 = _C.feature_resize_fwd(fm, g16, size[0], size[1], gs)
    out32, ls32 = _C.feature_resize_fwd(fm, g32, size[0], size[1], gs)
    assert out16.dtype == torch.float32 and torch.equal(out16, out32)
    # the cross-block sum of |d| uses float atomics: its order varies between calls
    assert abs(float(ls16[0]) - float(ls32[0])) <= 1e-6 * abs(float(ls32[0]))
    l16, grad16 = fh.feature_l1_loss_and_grad(fm, g16, 0.7)
    l32, grad32 = fh.feature_l1_loss_and_grad(fm, g32, 0.7)
    assert l16.dtype == torch.float32 and grad16.dtype == torch.float32 and torch.equal(grad16, grad32)
    assert abs(float(l16) - float(l32)) <= 1e-6 * abs(float(l32))


def _decoder_case(Cin, Cout, N, bias, seed):
    g = _gen(seed)
    x = torch.randn(Cin, N, device="cuda", generator=g)
    W = torch.randn(Cout, Cin, device="cuda", generator=g) / Cin ** 0.5
    b = 0.1 * torch.randn(Cout, device="cuda", generator=g) if bias else None
    return x, W, b, g


def _l1(x, gt, W, b, gs):
    from diff_gaussian_rasterization import _C

    dW = torch.zeros_like(W)
    db = torch.zeros_like(b) if b is not None else torch.empty(0, device="cuda")
    ls, dx = _C.decoder_l1(x, gt, W, b if b is not None else torch.empty(0, device="cuda"), gs, dW, db)
    return ls, dx, dW, db


@pytest.mark.gpu
@pytest.mark.parametrize("Cin,Cout,N", DECODER_SHAPES)
@pytest.mark.parametrize("bias", [True, False])
def test_decoder_loss_with_half_target_is_bitwise_the_upcast_one(Cin, Cout, N, bias):
    from diff_gaussian_rasterization import _C

    x, W, b, g = _decoder_case(Cin, Cout, N, bias, 2)
    y = _C.decoder_forward(x, W, b if bias else torch.empty(0, device="cuda"))
    g16 = (y + 0.3 * torch.randn(y.shape, device="cuda", generator=g)).half()
    g16.view(-1)[::7] = y.view(-1)[::7].half()
    gs = 0.7 / (Cout * N)
    r16, r32 = _l1(x, g16, W, b, gs), _l1(x, g16.float(), W, b, gs)
    for a, c in zip(r16, r32):
        assert a.dtype == torch.float32 and torch.equal(a, c)


@pytest.mark.gpu
@pytest.mark.parametrize("Cin,Cout,N", DECODER_SHAPES + [(256, 512, 40000)])
@pytest.mark.parametrize("bias", [True, False])
def test_decode_to_half_is_bitwise_the_rounded_float32_map(Cin, Cout, N, bias):
    from diff_gaussian_rasterization import _C

    x, W, b, _ = _decoder_case(Cin, Cout, N, bias, 3)
    # rows scaled past the float16 range (65504: +-inf after rounding) and into its subnormals
    scale = torch.ones(Cout, 1, device="cuda")
    scale[1::4], scale[2::4] = 3e5, 1e-6
    W = (W * scale).contiguous()
    bb = b * scale[:, 0] if bias else torch.empty(0, device="cuda")
    y16 = _C.decoder_forward(x, W, bb, torch.float16)
    ref = _C.decoder_forward(x, W, bb).half()
    assert y16.dtype == torch.float16 and y16.shape == (Cout, N)
    assert torch.equal(y16.view(torch.int16), ref.view(torch.int16))
    if Cout > 1 and N > 100:
        assert bool(torch.isinf(y16).any()) and bool(((y16 != 0) & (y16.abs() < 6.1e-5)).any())
    # the default output dtype stays float32
    assert _C.decoder_forward(x, W, bb).dtype == torch.float32


@pytest.mark.gpu
def test_half_overlap_checks_use_the_half_size(lib):
    """Buffers placed back to back with the float16 one's 2-byte elements: accepted, and the results are right."""
    from diff_gaussian_rasterization import _C

    Cin, Cout, N = 8, 12, 50
    x, W, b, g = _decoder_case(Cin, Cout, N, True, 4)
    buf = torch.zeros(Cout * N // 2 + Cin * N, device="cuda")  # [gt16 | dL_dx] and then [y16 | ...]
    g16 = torch.randn(Cout, N, device="cuda", generator=g).half()
    buf.view(torch.float16)[: Cout * N].copy_(g16.view(-1))
    gt_ptr, dx_ptr = buf.data_ptr(), buf.data_ptr() + 2 * Cout * N
    ls, dW, db = torch.zeros(1, device="cuda"), torch.zeros_like(W), torch.zeros_like(b)
    stream = torch.cuda.current_stream().cuda_stream
    assert lib.f3dgs_decoder_l1_f16gt(Cin, Cout, N, W.data_ptr(), b.data_ptr(), x.data_ptr(), gt_ptr, 0.5, ls.data_ptr(),
                                      dx_ptr, dW.data_ptr(), db.data_ptr(), stream) == 0, lib.f3dgs_last_error()
    r = _l1(x, g16, W, b, 0.5)
    assert torch.equal(ls, r[0]) and torch.equal(buf[Cout * N // 2:].view(Cin, N), r[1])
    assert torch.equal(dW, r[2]) and torch.equal(db, r[3])
    # y16 directly in front of x
    xb = torch.empty(Cout * N // 2 + Cin * N, device="cuda")
    xb[Cout * N // 2:].copy_(x.view(-1))
    assert lib.f3dgs_decoder_forward_f16(Cin, Cout, N, W.data_ptr(), b.data_ptr(), xb.data_ptr() + 2 * Cout * N,
                                         xb.data_ptr(), stream) == 0, lib.f3dgs_last_error()
    y16 = xb.view(torch.float16)[: Cout * N].view(Cout, N)
    assert torch.equal(y16, _C.decoder_forward(x, W, b).half())


@pytest.mark.gpu
@pytest.mark.parametrize("bias", [True, False])
def test_autograd_drop_ins_with_half_target(bias):
    from diff_gaussian_rasterization import feature_head as fh

    Cin, Cout, hw, ghw = 16, 64, (37, 53), (20, 30)
    g = _gen(5)
    fm = torch.randn(Cin, *hw, device="cuda", generator=g)
    W = (torch.randn(Cout, Cin, 1, 1, device="cuda", generator=g) / Cin ** 0.5)
    b = 0.1 * torch.randn(Cout, device="cuda", generator=g) if bias else None
    g16 = torch.randn(Cout, *ghw, device="cuda", generator=g).half()
    w = 0.9

    def run(gt):
        fm_g, W_g = fm.clone().requires_grad_(True), W.clone().requires_grad_(True)
        b_g = None if b is None else b.clone().requires_grad_(True)
        loss = fh.decoded_feature_l1_loss(fm_g, gt, W_g, b_g, w)
        (2.0 * loss).backward()
        return loss.detach(), fm_g.grad, W_g.grad, None if b is None else b_g.grad

    got, want = run(g16), run(g16.float())
    for a, c in zip(got, want):
        assert (a is None and c is None) or (a.dtype == torch.float32 and torch.equal(a, c))

    # against PyTorch float64 l1_loss(decoder(F.interpolate(fm)), gt16), the bars of test_feature_decoder.py
    x64 = fm.double().requires_grad_(True)
    W64 = W.double().requires_grad_(True)
    b64 = None if b is None else b.double().requires_grad_(True)
    r = F.interpolate(x64[None], size=ghw, mode="bilinear", align_corners=True)
    y64 = F.conv2d(r, W64, b64)[0]
    loss64 = F.l1_loss(y64, g16.double()) * w  # PyTorch's promotion of the float16 target: exact
    loss64.backward()
    rr = resize_bilinear_ac(fm.cpu().numpy(), *ghw).astype(np.float64).reshape(Cin, -1)
    Wn = W.cpu().numpy()[:, :, 0, 0].astype(np.float64)
    A = np.abs(Wn) @ np.abs(rr) + (0.0 if b is None else np.abs(b.cpu().numpy().astype(np.float64))[:, None])
    bar = DECODE_REL * A + 1e-6
    d64 = (y64.detach().reshape(Cout, -1) - g16.double().reshape(Cout, -1)).cpu().numpy()
    s, flip = np.sign(d64), (np.abs(d64) <= bar).astype(np.float64)
    gs = w / d64.size
    loss, dfm, dW = float(got[0]), got[1].cpu().numpy(), got[2].cpu().numpy()[:, :, 0, 0] / 2.0
    loss_ref = float(loss64.detach())
    assert abs(loss - loss_ref) <= gs * bar.sum() + 1e-5 * loss_ref
    dres_bar = (DECODE_REL * np.abs(Wn.T) @ np.abs(s) + 2 * np.abs(Wn.T) @ flip) * gs + 1e-9
    dfm_bar = resize_bilinear_ac_bwd(dres_bar.reshape(Cin, *ghw), *hw).astype(np.float64) + 1e-9
    assert np.all(np.abs(dfm / 2.0 - x64.grad.cpu().numpy()) <= dfm_bar)
    dW_bar = gs * (1.5e-3 * np.abs(s) @ np.abs(rr).T + 2 * flip @ np.abs(rr).T) + 1e-12
    assert np.all(np.abs(dW - W64.grad.cpu().numpy()[:, :, 0, 0]) <= dW_bar)
    if bias:
        assert np.all(np.abs(got[3].cpu().numpy() / 2.0 - b64.grad.cpu().numpy()) <= gs * (1e-6 * d64.shape[1] +
                                                                                           2 * flip.sum(1)))

    # the resize-L1 drop-in: same gradient as with the upcast target, and PyTorch float64 within test_next_rows.py's bars
    gr16 = torch.randn(Cin, *ghw, device="cuda", generator=g).half()
    grads, losses = [], []
    for gt in (gr16, gr16.float()):
        fm_g = fm.clone().requires_grad_(True)
        loss = fh.feature_l1_loss(fm_g, gt, 0.7)
        loss.backward()
        grads.append(fm_g.grad)
        losses.append(float(loss.detach()))
    assert torch.equal(grads[0], grads[1]) and abs(losses[0] - losses[1]) <= 1e-6 * abs(losses[1])
    x64 = fm.double().requires_grad_(True)
    ref = F.l1_loss(F.interpolate(x64[None], size=ghw, mode="bilinear", align_corners=True)[0], gr16.double()) * 0.7
    ref.backward()
    ref = float(ref.detach())
    assert abs(losses[0] - ref) <= 2e-5 * abs(ref) + 1e-7
    assert torch.allclose(grads[0].double(), x64.grad, rtol=1e-4, atol=1e-7)


@pytest.mark.gpu
def test_half_target_makes_no_float32_copy():
    from diff_gaussian_rasterization import feature_head as fh

    Cin, Cout, hw, ghw = 16, 512, (270, 480), (240, 427)
    g = _gen(6)
    fm = torch.randn(Cin, *hw, device="cuda", generator=g)
    W = torch.randn(Cout, Cin, 1, 1, device="cuda", generator=g) / Cin ** 0.5
    b = 0.1 * torch.randn(Cout, device="cuda", generator=g)
    dW, db = torch.zeros_like(W), torch.zeros_like(b)
    g16 = torch.randn(Cout, *ghw, device="cuda", generator=g).half()
    gr16 = torch.randn(Cin, *ghw, device="cuda", generator=g).half()
    n_map, n_res = Cin * hw[0] * hw[1] * 4, Cin * ghw[0] * ghw[1] * 4
    # the loss scalars, and a cached block reused whole (the caching allocator leaves remainders below 1 MiB unsplit)
    slack = 4 << 20
    assert n_res > slack  # so a float32 copy of either teacher map cannot hide in the slack

    def rise(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        m0 = torch.cuda.memory_allocated()
        out = fn()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - m0, out

    # decoder path: the resized map, dL/d(resized map) and dL/dfeature_map are its float32 outputs
    bound = 2 * n_res + n_map + slack
    r, _ = rise(lambda: fh.decoded_feature_l1_loss_and_grad(fm, g16, W, b, 1.0, dW, db))
    assert r <= bound, (r, bound)
    # resize-L1: the sign map and dL/dfeature_map
    bound = n_res + n_map + slack
    r, _ = rise(lambda: fh.feature_l1_loss_and_grad(fm, gr16, 1.0))
    assert r <= bound, (r, bound)


@pytest.mark.gpu
def test_rejects_other_target_dtypes_devices_and_shapes():
    from diff_gaussian_rasterization import _C
    from diff_gaussian_rasterization import feature_head as fh

    x, W, b, g = _decoder_case(8, 12, 50, True, 7)
    dW, db = torch.zeros_like(W), torch.zeros_like(b)
    gt = torch.randn(12, 50, device="cuda", generator=g)
    fm = torch.randn(3, 9, 11, device="cuda", generator=g)
    fm8 = torch.randn(8, 9, 11, device="cuda", generator=g)  # the decoder's Cin
    gr = torch.randn(3, 5, 6, device="cuda", generator=g)
    gd = torch.randn(12, 5, 6, device="cuda", generator=g)
    bad = [
        lambda: _C.decoder_l1(x, gt.bfloat16(), W, b, 1.0, dW, db),
        lambda: _C.decoder_l1(x, gt.double(), W, b, 1.0, dW, db),
        lambda: _C.decoder_l1(x, gt.half().cpu(), W, b, 1.0, dW, db),
        lambda: _C.decoder_l1(x, gt[:, :49].contiguous().half(), W, b, 1.0, dW, db),
        lambda: _C.decoder_l1(x, gt[:11].half(), W, b, 1.0, dW, db),
        lambda: _C.feature_resize_fwd(fm, gr.bfloat16(), 5, 6, 1.0),
        lambda: _C.feature_resize_fwd(fm, gr.double(), 5, 6, 1.0),
        lambda: _C.feature_resize_fwd(fm, gr.half().cpu(), 5, 6, 1.0),
        lambda: _C.feature_resize_fwd(fm, gr.half(), 5, 7, 1.0),
        lambda: _C.feature_resize_fwd(fm, gr[:2].half(), 5, 6, 1.0),
        lambda: fh.feature_l1_loss_and_grad(fm, gr.bfloat16()),
        lambda: fh.decoded_feature_l1_loss_and_grad(fm8, gd.bfloat16(), W, b),
        lambda: fh.decoded_feature_l1_loss_and_grad(fm8, gd.double(), W, b),
        lambda: fh.decoded_feature_l1_loss_and_grad(fm8, gd.half().cpu(), W, b),
        lambda: _C.decoder_forward(x, W, b, torch.bfloat16),
        lambda: _C.decoder_forward(x, W, b, torch.float64),
        lambda: fh.decode(x, W, b, dtype=torch.int16),
    ]
    for i, f in enumerate(bad):
        with pytest.raises(RuntimeError):
            f()
            pytest.fail(f"case {i} was accepted")


@pytest.mark.gpu
def test_training_step_with_decoder_learns_from_half_teacher_maps():
    """The --speedup ViewBatch loop of test_feature_decoder.py::test_training_step_with_decoder_learns with the teacher maps
    stored as float16 (decode(..., dtype=torch.float16), as render.py saves them).  In the first iteration every view's
    loss, g_feature and decoder gradients are bitwise those of the upcast maps; over six steps the loss falls."""
    import scenegen
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid
    from diff_gaussian_rasterization import feature_head as fh

    sc = scenegen.make_config("small", views=2)
    dev = "cuda"
    t = scenegen.to_torch(sc, dev)
    C, Cout = sc.C, 4 * sc.C
    g = _gen(0)

    def state(feat):
        return GaussianState(t["means3D"].clone(), t["shs"][:, :1].contiguous(), t["shs"][:, 1:].contiguous(),
                             inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                             t["rotations"].clone(), feat)

    def render(st):
        st.activate()
        vb = st.batch()
        vb.zero_()
        for cam in sc.cameras:
            rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))
            color, feat, radii, depth, ctx = vb.forward(rs)
            yield vb, color, feat, depth, ctx

    W_true = torch.randn(Cout, C, 1, 1, device=dev, generator=g) / C ** 0.5
    b_true = 0.1 * torch.randn(Cout, device=dev, generator=g)
    gts = []
    for _, _, feat, _, _ in render(state(t["semantic_feature"].clone())):
        gsz = (feat.shape[1] // 2, feat.shape[2] // 2)
        gts.append(fh.decode(fh.resize_bilinear(feat, gsz), W_true, b_true, dtype=torch.float16))
    assert all(gt.dtype == torch.float16 for gt in gts)
    sf = t["semantic_feature"]
    st = state((sf + 0.3 * sf.abs().mean() * torch.randn(sf.shape, device=dev, generator=g)).contiguous())
    conv = torch.nn.Conv2d(C, Cout, kernel_size=1).to(dev)
    with torch.no_grad():
        conv.weight.copy_(W_true + 0.3 * torch.randn(W_true.shape, device=dev, generator=g) / C ** 0.5)
    opt = torch.optim.Adam(conv.parameters(), lr=1e-2)
    lrs = dict(xyz=0.0, f_dc=0.0, f_rest=0.0, opacity=0.0, scaling=0.0, rotation=0.0, semantic_feature=0.02)
    losses = []
    for it in range(6):
        opt.zero_grad(set_to_none=False)
        conv.weight.grad = torch.zeros_like(conv.weight) if conv.weight.grad is None else conv.weight.grad
        conv.bias.grad = torch.zeros_like(conv.bias) if conv.bias.grad is None else conv.bias.grad
        total = torch.zeros((), device=dev)
        for v, (vb, color, feat, depth, ctx) in enumerate(render(st)):
            if it == 0:
                both = [fh.decoded_feature_l1_loss_and_grad(feat, gt, conv.weight, conv.bias, 1.0)
                        for gt in (gts[v], gts[v].float())]
                for a, c in zip(*both):
                    assert torch.equal(a, c), v
            loss, gfeat, _, _ = fh.decoded_feature_l1_loss_and_grad(feat, gts[v], conv.weight, conv.bias, 1.0,
                                                                    conv.weight.grad, conv.bias.grad)
            if it == 0:
                assert torch.equal(loss, both[0][0]) and torch.equal(gfeat, both[0][1])
            vb.backward(ctx, torch.zeros_like(color), gfeat, torch.zeros_like(depth), last=(v == len(sc.cameras) - 1))
            total = total + loss
        vb.all_reduce()
        st.step(lrs)
        opt.step()
        losses.append(float(total))
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
