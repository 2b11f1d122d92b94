"""Feature decoder of the --speedup mode (csrc/feature_decoder.cu, diff_gaussian_rasterization/feature_head.py): the
reference's 1x1 `CNN_decoder` (models/networks.py:107-119) after the bilinear resize, and its L1 loss (train.py:100-104).

CPU part (`-m "not gpu"`): a float64 restatement (y = W x + b and the closed-form dx, dW, db, composed with the oracle's
resize and its transpose) is pinned against PyTorch float64 autograd of the reference formula; the C ABI rejects bad
arguments before touching CUDA.  GPU part (`-m gpu`): the TF32 kernels against float64 with per-element bars that follow
from rounding both operands to TF32 (2^-11 relative each), sign flips allowed only where the float64 residual is inside
the decode bar; bitwise self-consistency, accumulation and reproducibility; the Python API; a ViewBatch training loop.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.next_rows import resize_bilinear_ac, resize_bilinear_ac_bwd

DECODE_REL = 1.2e-3


def decoded_l1(fm, gt, W, b, w):
    """float64 restatement: -> (loss, dL/dfm, dL/dW, dL/db, y) for
    loss = w * mean|W resize(fm) + b - gt|, resize = F.interpolate(bilinear, align_corners=True)."""
    Cin, H, Wd = fm.shape
    Cout, Hg, Wg = gt.shape
    r = resize_bilinear_ac(fm, Hg, Wg).astype(np.float64).reshape(Cin, -1)
    y = W.astype(np.float64) @ r + (0.0 if b is None else b.astype(np.float64)[:, None])
    s = np.sign(y - gt.reshape(Cout, -1).astype(np.float64))
    gs = w / s.size
    loss = gs * np.abs(y - gt.reshape(Cout, -1)).sum()
    dres = gs * (W.astype(np.float64).T @ s)
    dfm = resize_bilinear_ac_bwd(dres.reshape(Cin, Hg, Wg), H, Wd)
    return loss, dfm, gs * (s @ r.T), None if b is None else gs * s.sum(1), y.reshape(Cout, Hg, Wg)


def _torch_reference(fm, gt, W, b, w):
    x = torch.from_numpy(fm.astype(np.float64)).requires_grad_(True)
    Wt = torch.from_numpy(W.astype(np.float64)).requires_grad_(True)
    bt = None if b is None else torch.from_numpy(b.astype(np.float64)).requires_grad_(True)
    r = F.interpolate(x[None], size=gt.shape[1:], mode="bilinear", align_corners=True)
    y = F.conv2d(r, Wt[:, :, None, None], bt)[0]
    loss = F.l1_loss(y, torch.from_numpy(gt.astype(np.float64))) * w
    loss.backward()
    return float(loss.detach()), x.grad.numpy(), Wt.grad.numpy(), None if b is None else bt.grad.numpy(), y.detach().numpy()


def _inputs(Cin, Cout, hw, ghw, bias, seed):
    rng = np.random.default_rng(seed)
    fm = rng.standard_normal((Cin,) + hw).astype(np.float32)
    W = (rng.standard_normal((Cout, Cin)) / np.sqrt(Cin)).astype(np.float32)
    b = (0.1 * rng.standard_normal(Cout)).astype(np.float32) if bias else None
    gt = rng.standard_normal((Cout,) + ghw).astype(np.float32)
    return fm, W, b, gt


@pytest.mark.parametrize("Cin,Cout", [(1, 1), (5, 7), (16, 64)])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("same", [False, True])
def test_restatement_matches_pytorch_float64_autograd(Cin, Cout, bias, same):
    fm, W, b, gt = _inputs(Cin, Cout, (13, 17), (6, 9), bias, 1)
    w = 0.7
    if same:  # gt == y: each side's own decoded map, so every residual is exactly zero
        loss, dfm, dW, db, _ = decoded_l1(fm, decoded_l1(fm, gt, W, b, w)[4].astype(np.float64), W, b, w)
        ref = _torch_reference(fm, _torch_reference(fm, gt, W, b, w)[4], W, b, w)
        assert loss == 0.0 and ref[0] == 0.0
    else:
        loss, dfm, dW, db, _ = decoded_l1(fm, gt, W, b, w)
        ref = _torch_reference(fm, gt, W, b, w)
    # the oracle's resize runs in float32 (as the kernel does), PyTorch's float64 one differs in the 7th digit
    assert abs(loss - ref[0]) <= 1e-6 * max(abs(ref[0]), 1e-30)
    for got, want in ((dfm, ref[1]), (dW, ref[2])) + (((db, ref[3]),) if bias else ()):
        assert np.allclose(got, want, rtol=1e-6, atol=1e-6 * max(np.abs(want).max(), 1e-30)), np.abs(got - want).max()


# ---- C ABI argument validation (no CUDA call is made for rejected arguments)
@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_decoder_l1.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 4 + [ctypes.c_float] + [ctypes.c_void_p] * 5
    L.f3dgs_decoder_forward.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 5
    return L


def test_decoder_rejects_bad_arguments_before_touching_cuda(lib):
    W, b, x, gt, ls, dx, dW, db = (k << 24 for k in range(1, 9))  # never dereferenced: validation fails first

    def l1(Cin=16, Cout=64, N=100, w=W, bias=b, xx=x, g=gt, s=ls, d=dx, dw=dW, dbb=db):
        return lib.f3dgs_decoder_l1(Cin, Cout, N, w, bias, xx, g, 0.5, s, d, dw, dbb, None)

    assert l1(Cin=0) == -1 and b"bad sizes" in lib.f3dgs_last_error()
    assert l1(Cin=257) == -1 and b"bad sizes" in lib.f3dgs_last_error()
    assert l1(Cout=0) == -1 and l1(Cout=4097) == -1 and l1(N=0) == -1 and l1(N=-5) == -1 and l1(Cin=-1) == -1
    for kw in ("w", "xx", "g", "s", "d", "dw"):
        assert l1(**{kw: None}) == -1 and b"NULL pointer" in lib.f3dgs_last_error(), kw
    assert l1(dbb=None) == -1 and b"NULL pointer" in lib.f3dgs_last_error()  # a bias needs its gradient
    assert l1(bias=None) == -1                                              # and the other way round
    assert l1(d=x) == -1 and b"overlaps" in lib.f3dgs_last_error()
    assert l1(d=x + 4 * 16 * 100 - 4) == -1                                 # the last element of x
    assert l1(d=gt) == -1 and l1(d=W) == -1 and l1(d=dW) == -1
    assert l1(d=x - 4 * 16 * 100 + 4) == -1                                 # dL_dx's last element is x's first
    fwd = lib.f3dgs_decoder_forward
    assert fwd(300, 8, 10, W, b, x, dx, None) == -1 and b"bad sizes" in lib.f3dgs_last_error()
    assert fwd(8, 8, 10, None, b, x, dx, None) == -1 and b"NULL pointer" in lib.f3dgs_last_error()
    assert fwd(8, 8, 10, W, b, x, None, None) == -1
    assert fwd(8, 8, 10, W, b, x, x, None) == -1 and b"overlaps" in lib.f3dgs_last_error()
    assert fwd(8, 8, 10, W, b, x, W + 4, None) == -1


# =================================================================================================== GPU
def _dev_case(Cin, Cout, N, bias, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(Cin, N, device="cuda", generator=g)
    W = torch.randn(Cout, Cin, device="cuda", generator=g) / Cin ** 0.5
    b = 0.1 * torch.randn(Cout, device="cuda", generator=g) if bias else None
    return x, W, b


def _ref64(x, W, b):
    """-> (y64, decode bar) in float64 on the device."""
    x64, W64 = x.double(), W.double()
    y = W64 @ x64
    A = W64.abs() @ x64.abs()
    if b is not None:
        y += b.double()[:, None]
        A += b.double().abs()[:, None]
    return y, DECODE_REL * A + 1e-6


def _l1(x, W, b, gt, gs):
    from diff_gaussian_rasterization import _C

    dW = torch.zeros_like(W)
    db = torch.zeros_like(b) if b is not None else torch.empty(0, device="cuda")
    ls, dx = _C.decoder_l1(x, gt, W, b if b is not None else torch.empty(0, device="cuda"), gs, dW, db)
    return ls, dx, dW, (db if b is not None else None)


def _check_loss_mode(x, W, b, gt, gs, y64, bar):
    """TF32 bars for the loss mode; a sign may differ from float64 only where |y64 - gt| <= the decode bar."""
    ls, dx, dW, db = _l1(x, W, b, gt, gs)
    d64 = y64 - gt.double()
    s = torch.sign(d64)
    flip = (d64.abs() <= bar).double()
    ref_ls = float(d64.abs().sum())
    assert abs(float(ls[0]) - ref_ls) <= float(bar.sum()) + 1e-5 * ref_ls, (float(ls[0]), ref_ls)
    W64, x64, ags = W.double(), x.double(), abs(gs)
    dx_bar = DECODE_REL * ags * (W64.abs().T @ s.abs()) + 1e-9 + 2 * ags * (W64.abs().T @ flip)
    err = (dx.double() - gs * (W64.T @ s)).abs()
    assert bool((err <= dx_bar).all()), float((err / dx_bar).max())
    dW_bar = 1.5e-3 * ags * (s.abs() @ x64.abs().T) + 2 * ags * (flip @ x64.abs().T)
    err = (dW.double() - gs * (s @ x64.T)).abs()
    assert bool((err <= dW_bar + 1e-30).all()), float((err / (dW_bar + 1e-30)).max())
    if b is not None:
        db_bar = 1e-6 * ags * x.shape[1] + 2 * ags * flip.sum(1)
        err = (db.double() - gs * s.sum(1)).abs()
        assert bool((err <= db_bar).all()), float((err / db_bar).max())
    return ls, dx, dW, db


SHAPES = [(1, 1, 1), (5, 7, 1000), (16, 64, 4099), (128, 512, 409440), (256, 33, 777)]


@pytest.mark.gpu
@pytest.mark.parametrize("Cin,Cout,N", SHAPES)
@pytest.mark.parametrize("bias", [True, False])
def test_decode_matches_float64(Cin, Cout, N, bias):
    from diff_gaussian_rasterization import _C

    x, W, b = _dev_case(Cin, Cout, N, bias, 1)
    y = _C.decoder_forward(x, W, b if bias else torch.empty(0, device="cuda"))
    y64, bar = _ref64(x, W, b)
    assert y.shape == (Cout, N)
    err = (y.double() - y64).abs()
    assert bool((err <= bar).all()), float((err / bar).max())


@pytest.mark.gpu
@pytest.mark.parametrize("Cin,Cout,N", SHAPES + [(64, 256, 20000), (200, 4096, 300)])
@pytest.mark.parametrize("bias", [True, False])
def test_loss_mode_with_unambiguous_signs(Cin, Cout, N, bias):
    x, W, b = _dev_case(Cin, Cout, N, bias, 2)
    y64, bar = _ref64(x, W, b)
    g = torch.Generator(device="cuda").manual_seed(3)
    sigma = torch.where(torch.rand(y64.shape, device="cuda", generator=g) < 0.5, -1.0, 1.0).double()
    gt = (y64 + sigma * (4 * bar + torch.rand(y64.shape, device="cuda", generator=g).double())).float()
    gs = 0.7 / (Cout * N)
    _check_loss_mode(x, W, b, gt, gs, y64, bar)


@pytest.mark.gpu
@pytest.mark.parametrize("Cin,Cout,N", [(5, 7, 1000), (16, 64, 4099), (128, 512, 409440), (256, 33, 777)])
def test_loss_mode_random_targets(Cin, Cout, N):
    x, W, b = _dev_case(Cin, Cout, N, True, 4)
    y64, bar = _ref64(x, W, b)
    g = torch.Generator(device="cuda").manual_seed(5)
    gt = y64.float() + 0.3 * torch.randn(y64.shape, device="cuda", generator=g)
    gt.view(-1)[::7] = y64.view(-1)[::7].float()  # some residuals within rounding of zero
    _check_loss_mode(x, W, b, gt, -1.3 / (Cout * N), y64, bar)


@pytest.mark.gpu
@pytest.mark.parametrize("Cin,Cout,N", [(5, 7, 1000), (128, 512, 40000), (256, 33, 777)])
def test_self_consistency_accumulation_and_reproducibility(Cin, Cout, N):
    from diff_gaussian_rasterization import _C

    x, W, b = _dev_case(Cin, Cout, N, True, 6)
    y = _C.decoder_forward(x, W, b)
    dW0 = torch.randn_like(W)
    db0 = torch.randn_like(b)
    dW, db = dW0.clone(), db0.clone()
    ls, dx = _C.decoder_l1(x, y, W, b, 1.0 / (Cout * N), dW, db)
    assert float(ls[0]) == 0.0 and bool((dx == 0).all())
    assert torch.equal(dW, dW0) and torch.equal(db, db0)

    gt = y + 0.1 * torch.randn_like(y)
    outs = []
    for _ in range(2):
        dW, db = torch.zeros_like(W), torch.zeros_like(b)
        ls, dx = _C.decoder_l1(x, gt, W, b, 1.0 / (Cout * N), dW, db)
        dW2, db2 = dW.clone(), db.clone()
        ls2, dx2 = _C.decoder_l1(x, gt, W, b, 1.0 / (Cout * N), dW2, db2)
        assert torch.equal(ls, ls2) and torch.equal(dx, dx2)
        assert torch.equal(dW2, 2 * dW) and torch.equal(db2, 2 * db)
        outs.append((ls, dx, dW, db))
    for a, c in zip(*outs):
        assert torch.equal(a, c)


@pytest.mark.gpu
@pytest.mark.parametrize("bias", [True, False])
def test_python_api_end_to_end_matches_float64(bias):
    from diff_gaussian_rasterization import feature_head as fh

    Cin, Cout, hw, ghw = 16, 64, (37, 53), (20, 30)
    fm, W, b, gt = _inputs(Cin, Cout, hw, ghw, bias, 7)
    w = 0.9
    loss64, dfm64, dW64, db64, y64 = decoded_l1(fm, gt, W, b, w)
    r = resize_bilinear_ac(fm, *ghw).astype(np.float64).reshape(Cin, -1)
    A = np.abs(W.astype(np.float64)) @ np.abs(r) + (0.0 if b is None else np.abs(b.astype(np.float64))[:, None])
    bar = DECODE_REL * A + 1e-6
    d64 = y64.reshape(Cout, -1) - gt.reshape(Cout, -1)
    s, flip = np.sign(d64), (np.abs(d64) <= bar).astype(np.float64)
    gs = w / d64.size
    cu = lambda a: None if a is None else torch.from_numpy(a).cuda()  # noqa: E731
    fm_t, gt_t, W_t, b_t = cu(fm), cu(gt), cu(W), cu(b)
    loss, dfm, dW, db = fh.decoded_feature_l1_loss_and_grad(fm_t, gt_t, W_t[:, :, None, None], b_t, w)
    assert dW.shape == (Cout, Cin, 1, 1) and (db is None) == (not bias) and dfm.shape == fm.shape
    assert abs(float(loss) - loss64) <= gs * bar.sum() + 1e-5 * loss64
    dres_bar = (DECODE_REL * np.abs(W.T) @ np.abs(s) + 2 * np.abs(W.T) @ flip) * gs + 1e-9
    dfm_bar = resize_bilinear_ac_bwd(dres_bar.reshape(Cin, *ghw), *hw).astype(np.float64) + 1e-9
    assert np.all(np.abs(dfm.cpu().numpy() - dfm64) <= dfm_bar)
    dW_bar = gs * (1.5e-3 * np.abs(s) @ np.abs(r).T + 2 * flip @ np.abs(r).T) + 1e-12
    assert np.all(np.abs(dW.cpu().numpy()[:, :, 0, 0] - dW64) <= dW_bar)
    if bias:
        assert np.all(np.abs(db.cpu().numpy() - db64) <= gs * (1e-6 * d64.shape[1] + 2 * flip.sum(1)))

    # the decode hook and the autograd drop-in give the same numbers as the graph-free path
    y = fh.decode(fh.resize_bilinear(fm_t, ghw), W_t[:, :, None, None], b_t)
    assert np.all(np.abs(y.cpu().numpy().reshape(Cout, -1) - y64.reshape(Cout, -1)) <= bar)
    fm_g = fm_t.clone().requires_grad_(True)
    W_g = W_t[:, :, None, None].clone().requires_grad_(True)
    b_g = None if b_t is None else b_t.clone().requires_grad_(True)
    l2 = fh.decoded_feature_l1_loss(fm_g, gt_t, W_g, b_g, w)
    (2.0 * l2).backward()
    assert torch.equal(l2.detach(), loss)
    assert torch.equal(fm_g.grad, 2.0 * dfm) and torch.equal(W_g.grad, 2.0 * dW)
    if bias:
        assert torch.equal(b_g.grad, 2.0 * db)


@pytest.mark.gpu
def test_binding_rejects_mismatched_inputs():
    from diff_gaussian_rasterization import _C

    x, W, b = _dev_case(8, 12, 50, True, 8)
    gt = torch.randn(12, 50, device="cuda")
    dW, db = torch.zeros_like(W), torch.zeros_like(b)
    bad = [
        lambda: _C.decoder_l1(x, torch.randn(12, 51, device="cuda"), W, b, 1.0, dW, db),  # N
        lambda: _C.decoder_l1(x[:7], gt, W, b, 1.0, dW, db),                              # Cin
        lambda: _C.decoder_l1(x, gt[:11], W, b, 1.0, dW, db),                             # Cout of gt
        lambda: _C.decoder_l1(x, gt, W, b[:11], 1.0, dW, db),                             # Cout of bias
        lambda: _C.decoder_l1(x, gt, W, b, 1.0, dW[:11], db),                             # Cout of dweight
        lambda: _C.decoder_l1(x, gt, W, b, 1.0, dW, db[:11]),                             # Cout of dbias
        lambda: _C.decoder_l1(x.cpu(), gt.cpu(), W.cpu(), b.cpu(), 1.0, dW.cpu(), db.cpu()),
        lambda: _C.decoder_l1(x, gt.cpu(), W, b, 1.0, dW, db),
        lambda: _C.decoder_l1(x.double(), gt, W, b, 1.0, dW, db),
        lambda: _C.decoder_l1(x, gt, W.double(), b, 1.0, dW, db),
        lambda: _C.decoder_l1(x, gt, W, b, 1.0, dW.double(), db),
        lambda: _C.decoder_forward(x[:7], W, b),
        lambda: _C.decoder_forward(x.cpu(), W.cpu(), b.cpu()),
        lambda: _C.decoder_forward(x.half(), W, b),
        lambda: _C.decoder_forward(torch.randn(300, 4, device="cuda"), torch.randn(5, 300, device="cuda"), b[:5]),
    ]
    for i, f in enumerate(bad):
        with pytest.raises(RuntimeError):
            f()
            pytest.fail(f"case {i} was accepted")


@pytest.mark.gpu
def test_training_step_with_decoder_learns():
    """The loop of test_training_step_end_to_end_and_densify in --speedup form: teacher maps are a fixed random 1x1
    decoder (Cout = 4 C) of the maps rendered from the unperturbed scene at half resolution; the run starts from perturbed
    semantic features and another random decoder, and both learn (fused Adam on the features, torch.optim.Adam on W, b)."""
    import scenegen
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    from diff_gaussian_rasterization import feature_head as fh
    from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid

    sc = scenegen.make_config("small", views=2)
    dev = "cuda"
    t = scenegen.to_torch(sc, dev)
    C, Cout = sc.C, 4 * sc.C
    g = torch.Generator(device=dev).manual_seed(0)

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
        gts.append(fh.decode(fh.resize_bilinear(feat, gsz), W_true, b_true))
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
            loss, gfeat, _, _ = fh.decoded_feature_l1_loss_and_grad(feat, gts[v], conv.weight, conv.bias, 1.0,
                                                                    conv.weight.grad, conv.bias.grad)
            vb.backward(ctx, torch.zeros_like(color), gfeat, torch.zeros_like(depth), last=(v == len(sc.cameras) - 1))
            total = total + loss
        vb.all_reduce()
        st.step(lrs)
        opt.step()
        losses.append(float(total))
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
