"""Fused L1 + D-SSIM photometric loss (csrc/image_loss.cu, diff_gaussian_rasterization/image_loss.py), the colour term of
the reference training step (train.py; utils/loss_utils.py l1_loss + ssim(window_size=11, size_average=True)).

CPU part (`-m "not gpu"`): a float64 numpy restatement with a separable zero-padded blur and the closed-form gradient is
pinned against PyTorch float64 autograd of the reference formula (11x11 window, F.conv2d(padding=5, groups=C)); the C ABI
rejects bad arguments before touching CUDA.  GPU part (`-m gpu`): the kernel against that float64 restatement, bitwise
reproducibility, the `ssim` drop-in, and a reference-loss training loop.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

C1, C2 = 0.01 ** 2, 0.03 ** 2
SHAPES = [(3, 37, 53), (3, 5, 7), (1, 1, 1), (2, 3, 20, 31)]
GPU_SHAPES = SHAPES + [(3, 1080, 1920), (3, 17, 23), (4, 64, 64), (2, 3, 40, 50)]


def _gauss():
    g = np.exp(-((np.arange(11) - 5.0) ** 2) / 4.5)
    return g / g.sum()


def _blur(a):
    """Separable 11-tap Gaussian blur over the last two axes, zero padding (= F.conv2d(padding=5) per plane)."""
    w = _gauss()
    p = np.pad(a, [(0, 0)] * (a.ndim - 2) + [(5, 5), (0, 0)])
    a = sum(w[t] * p[..., t:t + a.shape[-2], :] for t in range(11))
    p = np.pad(a, [(0, 0)] * (a.ndim - 1) + [(5, 5)])
    return sum(w[t] * p[..., t:t + a.shape[-1]] for t in range(11))


def photometric(x, gt, lam):
    """float64 restatement: -> (loss, dL/dx, sum|x - gt|, sum ssim_map) for
    loss = (1 - lam) * mean|x - gt| + lam * (1 - mean(ssim_map))."""
    x, y = x.astype(np.float64), gt.astype(np.float64)
    mx, my, mxx, myy, mxy = _blur(x), _blur(y), _blur(x * x), _blur(y * y), _blur(x * y)
    A1, A2 = 2 * mx * my + C1, 2 * (mxy - mx * my) + C2
    B1, B2 = mx * mx + my * my + C1, (mxx - mx * mx) + (myy - my * my) + C2
    S = A1 * A2 / (B1 * B2)
    d_mx = S * (2 * my / A1 - 2 * my / A2 - 2 * mx / B1 + 2 * mx / B2)
    gS = _blur(d_mx) + 2 * x * _blur(-S / B2) + y * _blur(2 * S / A2)
    n = x.size
    l1, ssum = np.abs(x - y).sum(), S.sum()
    loss = (1 - lam) * l1 / n + lam * (1 - ssum / n)
    return loss, (1 - lam) / n * np.sign(x - y) - lam / n * gS, l1, ssum


def _torch_reference(x, gt, lam):
    """The reference's l1_loss + ssim (utils/loss_utils.py) in float64 on the CPU, gradient by autograd."""
    g = torch.from_numpy(_gauss())
    ch = x.shape[-3]
    win = (g[:, None] @ g[None, :]).expand(ch, 1, 11, 11).contiguous()
    xt = torch.from_numpy(x.astype(np.float64)).requires_grad_(True)
    yt = torch.from_numpy(gt.astype(np.float64))
    conv = lambda a: F.conv2d(a, win, padding=5, groups=ch)  # noqa: E731
    mu1, mu2 = conv(xt), conv(yt)
    s11, s22, s12 = conv(xt * xt) - mu1 ** 2, conv(yt * yt) - mu2 ** 2, conv(xt * yt) - mu1 * mu2
    ssim_map = ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 ** 2 + mu2 ** 2 + C1) * (s11 + s22 + C2))
    loss = (1 - lam) * torch.abs(xt - yt).mean() + lam * (1 - ssim_map.mean())
    loss.backward()
    return float(loss.detach()), xt.grad.numpy()


def _pair(shape, seed, noise=0.1):
    rng = np.random.default_rng(seed)
    x = rng.random(shape).astype(np.float32)
    gt = np.clip(x + noise * rng.standard_normal(shape), 0.0, 1.0).astype(np.float32)
    return x, gt


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("lam", [0.0, 0.2, 1.0])
@pytest.mark.parametrize("same", [False, True])
def test_restatement_matches_pytorch_float64_autograd(shape, lam, same):
    x, gt = _pair(shape, 1)
    if same:
        gt = x.copy()
    loss, grad, _, _ = photometric(x, gt, lam)
    ref_loss, ref_grad = _torch_reference(x, gt, lam)
    assert abs(loss - ref_loss) <= 1e-12 * max(abs(ref_loss), 1.0)
    assert np.allclose(grad, ref_grad, rtol=1e-9, atol=1e-10 / x.size)  # gradient entries are O(1 / N)


# ---- C ABI argument validation (no CUDA call is made for rejected arguments)
@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_image_loss.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 2 + [ctypes.c_float] * 2 + [ctypes.c_void_p] * 3
    return L


def test_image_loss_rejects_bad_arguments_before_touching_cuda(lib):
    img, gt, sums, grad = 0x10000, 0x20000, 0x30000, 0x40000  # never dereferenced: validation fails first

    def call(planes=3, H=8, W=8, image=img, target=gt, s=sums, g=grad):
        return lib.f3dgs_image_loss(planes, H, W, image, target, 0.8, -0.2, s, g, None)

    assert call(planes=-1) == -1 and b"bad sizes" in lib.f3dgs_last_error()
    assert call(H=0) == -1 and call(W=0) == -1 and call(H=-3) == -1 and call(W=-1) == -1
    assert call(planes=70000) == -1 and b"grid" in lib.f3dgs_last_error()
    assert call(H=16 * 65535 + 1) == -1
    for kw in ("image", "target", "s"):
        assert call(**{kw: None}) == -1 and b"NULL pointer" in lib.f3dgs_last_error(), kw
    assert call(g=img) == -1 and b"overlaps" in lib.f3dgs_last_error()
    assert call(g=gt) == -1
    assert call(g=img + 4 * 3 * 8 * 8 - 4) == -1  # the last element of image
    assert call(planes=0) == 0 and lib.f3dgs_last_error() == b""  # nothing to do
    assert call(planes=0, image=None, target=None, s=None, g=None) == 0


# =================================================================================================== GPU
def _loss_bars(loss, grad, ref_loss, ref_grad):
    assert abs(float(loss) - ref_loss) <= 2e-5 * abs(ref_loss), (float(loss), ref_loss)
    g = grad.cpu().numpy().astype(np.float64)
    err = np.abs(g - ref_grad)
    bar = 1e-4 * np.abs(ref_grad) + 1e-5 * np.abs(ref_grad).max()
    assert np.all(err <= bar), (err.max(), float((err / bar).max()))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", GPU_SHAPES)
def test_kernel_matches_float64_reference(shape):
    from diff_gaussian_rasterization.image_loss import photometric_loss_and_grad

    x, gt = _pair(shape, 2)
    lams = (0.0, 0.2, 1.0) if x.size < 100000 else (0.2,)
    for lam in lams:
        ref_loss, ref_grad, _, _ = photometric(x, gt, lam)
        loss, grad = photometric_loss_and_grad(torch.from_numpy(x).cuda(), torch.from_numpy(gt).cuda(), lam)
        assert grad.shape == x.shape and loss.shape == ()
        _loss_bars(loss, grad, ref_loss, ref_grad)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 37, 53), (2, 3, 40, 50), (3, 1080, 1920)])
def test_identical_images_give_zero_loss_and_gradient(shape):
    from diff_gaussian_rasterization.image_loss import photometric_loss_and_grad

    x = torch.from_numpy(_pair(shape, 3)[0]).cuda()
    lam, n = 0.2, x.numel()
    loss, grad = photometric_loss_and_grad(x, x.clone(), lam)
    assert abs(float(loss)) <= 1e-6
    assert float(grad.abs().max()) <= 1e-4 * lam / n


@pytest.mark.gpu
def test_bitwise_reproducible_and_value_only_sums():
    from diff_gaussian_rasterization import _C

    x, gt = (torch.from_numpy(a).cuda() for a in _pair((3, 270, 480), 4))
    s1, g1 = _C.image_loss(x, gt, 0.8 / x.numel(), -0.2 / x.numel(), True)
    s2, g2 = _C.image_loss(x, gt, 0.8 / x.numel(), -0.2 / x.numel(), True)
    s3, g3 = _C.image_loss(x, gt, 0.8 / x.numel(), -0.2 / x.numel(), False)
    assert torch.equal(s1, s2) and torch.equal(g1, g2)
    assert torch.equal(s1, s3) and g3.numel() == 0
    _, _, l1, ssum = photometric(x.cpu().numpy(), gt.cpu().numpy(), 0.2)
    assert abs(float(s1[0]) - l1) <= 2e-5 * l1 and abs(float(s1[1]) - ssum) <= 2e-5 * ssum


@pytest.mark.gpu
def test_binding_rejects_mismatched_inputs():
    from diff_gaussian_rasterization import _C
    from diff_gaussian_rasterization.image_loss import ssim

    x = torch.rand(3, 8, 8, device="cuda")
    with pytest.raises(RuntimeError):
        _C.image_loss(x, torch.rand(3, 8, 9, device="cuda"), 1.0, 1.0, True)
    with pytest.raises(RuntimeError):
        _C.image_loss(x.cpu(), x.cpu(), 1.0, 1.0, True)
    with pytest.raises(RuntimeError):
        _C.image_loss(x.double(), x.double(), 1.0, 1.0, True)
    with pytest.raises(ValueError):
        ssim(x, x, window_size=7)
    with pytest.raises(ValueError):
        ssim(x, x, size_average=False)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 37, 53), (2, 3, 40, 50), (3, 270, 480)])
def test_ssim_drop_in_value_and_gradient(shape):
    from diff_gaussian_rasterization.image_loss import ssim

    x, gt = _pair(shape, 5)
    ref_loss, ref_grad, _, _ = photometric(x, gt, 1.0)  # 1 - mean(ssim_map)
    xt = torch.from_numpy(x).cuda().requires_grad_(True)
    gtt = torch.from_numpy(gt).cuda()
    s = ssim(xt, gtt)
    (1.0 - s).backward()
    _loss_bars(1.0 - s.detach(), xt.grad, ref_loss, ref_grad)
    with torch.no_grad():
        s_ng = ssim(xt, gtt)
    assert torch.equal(s_ng, s.detach())
    assert torch.equal(ssim(xt.detach(), gtt), s.detach())


@pytest.mark.gpu
def test_training_step_with_reference_photometric_loss():
    """The loop of test_training_step_end_to_end_and_densify with the reference's colour loss: targets rendered from the
    unperturbed scene, a perturbed f_dc as the starting point, dL/dcolor from photometric_loss_and_grad, Adam on f_dc only;
    the summed loss must decrease."""
    import scenegen
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    from diff_gaussian_rasterization.image_loss import photometric_loss_and_grad
    from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid

    sc = scenegen.make_config("small", views=2)
    dev = "cuda"
    t = scenegen.to_torch(sc, dev)

    def state(f_dc):
        return GaussianState(t["means3D"].clone(), f_dc, t["shs"][:, 1:].contiguous(),
                             inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                             t["rotations"].clone(), t["semantic_feature"].clone())

    def render(st):
        st.activate()
        vb = st.batch()
        vb.zero_()
        for cam in sc.cameras:
            rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))
            color, feat, radii, depth, ctx = vb.forward(rs)
            yield vb, cam, color, feat, depth, ctx

    f_dc = t["shs"][:, :1].contiguous()
    gts = [color.clone() for _, _, color, _, _, _ in render(state(f_dc.clone()))]
    g = torch.Generator(device=dev).manual_seed(0)
    st = state((f_dc + 0.3 * torch.randn(f_dc.shape, device=dev, generator=g)).contiguous())
    lrs = dict(xyz=0.0, f_dc=0.02, f_rest=0.0, opacity=0.0, scaling=0.0, rotation=0.0, semantic_feature=0.0)
    losses = []
    for it in range(6):
        total = torch.zeros((), device=dev)
        for v, (vb, cam, color, feat, depth, ctx) in enumerate(render(st)):
            loss, gcolor = photometric_loss_and_grad(color, gts[v], 0.2)
            vb.backward(ctx, gcolor, torch.zeros_like(feat), torch.zeros_like(depth), last=(v == len(sc.cameras) - 1))
            total = total + loss
        vb.all_reduce()
        st.step(lrs)
        losses.append(float(total))
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
