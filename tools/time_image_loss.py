"""Per-call time of the reference's photometric loss with its gradient, two ways, in one process:

  (a) PyTorch: l1_loss + the ssim formula of utils/loss_utils.py (five depthwise 11x11 F.conv2d) under autograd, then
      .backward(); default backend settings (cuDNN, TF32 allowed).  The window is built once on the device, which
      favours (a): the reference rebuilds it and copies it to the GPU on every call.
  (b) image_loss.photometric_loss_and_grad (csrc/image_loss.cu): one fused kernel + a tiny reduction.

Both are warmed up, then timed with CUDA events in alternating rounds (ROUNDS x ITERS calls each).  The algorithmic
traffic is 2 reads + 1 write of planes*H*W fp32; achieved GB/s is that over the per-call time, against the H100 SXM
data-sheet HBM3 bandwidth of 3.35 TB/s.  Development tool, not product code:
    python tools/time_image_loss.py
"""
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "feature-3dgs_b200"))
from diff_gaussian_rasterization.image_loss import photometric_loss_and_grad  # noqa: E402

LAMBDA = 0.2
SHAPES = [(3, 1080, 1920), (3, 2160, 3840)]
ROUNDS, ITERS, WARMUP = 8, 100, 20  # a fused round is ~25 ms at 3x1080x1920: long enough to ride out host noise
PEAK_GBS = 3350.0


def window(channels, dev):
    g = torch.exp(-((torch.arange(11, dtype=torch.float64) - 5) ** 2) / 4.5)
    g = (g / g.sum()).float()
    return (g[:, None] @ g[None, :]).expand(channels, 1, 11, 11).contiguous().to(dev)


def reference_step(x, gt, win):
    """utils/loss_utils.py l1_loss + ssim, as train.py combines them; returns (loss, dL/dx)."""
    x.grad = None
    ch = x.shape[-3]
    mu1, mu2 = F.conv2d(x, win, padding=5, groups=ch), F.conv2d(gt, win, padding=5, groups=ch)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    s1 = F.conv2d(x * x, win, padding=5, groups=ch) - mu1_sq
    s2 = F.conv2d(gt * gt, win, padding=5, groups=ch) - mu2_sq
    s12 = F.conv2d(x * gt, win, padding=5, groups=ch) - mu1_mu2
    ssim_map = ((2 * mu1_mu2 + 0.01 ** 2) * (2 * s12 + 0.03 ** 2)) / ((mu1_sq + mu2_sq + 0.01 ** 2) * (s1 + s2 + 0.03 ** 2))
    loss = (1.0 - LAMBDA) * torch.abs(x - gt).mean() + LAMBDA * (1.0 - ssim_map.mean())
    loss.backward()
    return loss.detach(), x.grad


def fused_step(x, gt, _win):
    return photometric_loss_and_grad(x, gt, LAMBDA)


def time_calls(fn, args, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn(*args)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv"], capture_output=True, text=True)
    print(q.stdout.strip() or q.stderr.strip())
    print("torch", torch.__version__, " cudnn.allow_tf32 =", torch.backends.cudnn.allow_tf32)
    gen = torch.Generator(device="cuda").manual_seed(0)
    for shape in SHAPES:
        planes, H, W = shape
        x = torch.rand(shape, device="cuda", generator=gen)
        gt = (x + 0.1 * torch.randn(shape, device="cuda", generator=gen)).clamp(0, 1)
        xa = x.clone().requires_grad_(True)
        win = window(planes, x.device)
        la, ga = reference_step(xa, gt, win)
        lb, gb = fused_step(x, gt, win)
        rel = float((ga - gb).abs().max() / ga.abs().max())
        print(f"{planes}x{H}x{W}: loss (a) {float(la):.7f} (b) {float(lb):.7f}; max|g_a - g_b| / max|g_a| = {rel:.2e}")
        for fn, a in ((reference_step, (xa, gt, win)), (fused_step, (x, gt, win))):
            time_calls(fn, a, WARMUP)
        ta, tb = [], []
        for _ in range(ROUNDS):
            ta.append(time_calls(reference_step, (xa, gt, win), ITERS))
            tb.append(time_calls(fused_step, (x, gt, win), ITERS))
        nbytes = 3 * planes * H * W * 4
        for name, ts in (("(a) pytorch", ta), ("(b) fused  ", tb)):
            ts = sorted(ts)
            med = ts[len(ts) // 2]
            gbs = nbytes / (med * 1e-3) / 1e9
            print(f"  {name} {med:8.3f} ms/call (median of {ROUNDS} rounds x {ITERS}; min {ts[0]:.3f}, max {ts[-1]:.3f})"
                  f"  {nbytes / 1e6:.1f} MB algorithmic -> {gbs:7.1f} GB/s = {100 * gbs / PEAK_GBS:5.1f}% of 3.35 TB/s")
        print(f"  speed-up (a)/(b): {sorted(ta)[ROUNDS // 2] / sorted(tb)[ROUNDS // 2]:.1f}x")


if __name__ == "__main__":
    main()
