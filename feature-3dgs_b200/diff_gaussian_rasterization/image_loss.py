"""Photometric loss of the reference training step (train.py, utils/loss_utils.py):

    loss = (1 - lambda_dssim) * l1_loss(image, gt) + lambda_dssim * (1 - ssim(image, gt))     # lambda_dssim = 0.2

on one CUDA kernel of libf3dgs_b200 (csrc/image_loss.cu) that returns sum |image - gt|, the sum of the SSIM map (11-tap
Gaussian window, sigma 1.5, zero padding) and dL/dimage in a single pass.  There is no CPU path (the extension raises on
CPU tensors).
"""
import torch


def _C():
    from . import _C as ext  # deferred: keeps this module importable for documentation tools without the extension

    return ext


def photometric_loss_and_grad(image: torch.Tensor, gt: torch.Tensor, lambda_dssim: float = 0.2):
    """-> (loss, dL/dimage) for loss = (1 - lambda_dssim) * mean|image - gt| + lambda_dssim * (1 - ssim(image, gt)),
    no autograd graph: dL/dimage is the `g_color` a ViewBatch loop passes to `vb.backward`.  image, gt: [C,H,W] or
    [B,C,H,W] float32 CUDA tensors of the same shape.  The loss stays on the device (no host sync)."""
    lam = float(lambda_dssim)
    n = max(image.numel(), 1)
    sums, grad = _C().image_loss(image, gt, (1.0 - lam) / n, -lam / n, True)
    return sums[0] * ((1.0 - lam) / n) + lam * (1.0 - sums[1] / n), grad


class _SSIM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img1, img2):
        n = max(img1.numel(), 1)
        sums, grad = _C().image_loss(img1, img2, 0.0, 1.0 / n, True)
        ctx.save_for_backward(grad)
        return sums[1] / n

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return grad * g, None


def ssim(img1: torch.Tensor, img2: torch.Tensor, window_size: int = 11, size_average: bool = True) -> torch.Tensor:
    """Autograd-aware drop-in for the reference's `utils.loss_utils.ssim(img1, img2)`: the mean SSIM over all planes and
    pixels.  Only img1 (the rendered image) receives a gradient; img2 is the constant target."""
    if window_size != 11 or not size_average:
        raise ValueError("only ssim(window_size=11, size_average=True), the reference training loss, is implemented")
    if not (torch.is_grad_enabled() and img1.requires_grad):
        sums, _ = _C().image_loss(img1.detach(), img2.detach(), 0.0, 0.0, False)
        return sums[1] / max(img1.numel(), 1)
    if img2.requires_grad:
        raise ValueError("ssim: img2 is the target and receives no gradient; pass img2.detach()")
    return _SSIM.apply(img1, img2)
