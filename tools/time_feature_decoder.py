"""Per-call time of the --speedup feature loss with its gradients, two ways, in one process:

  (a) PyTorch: F.interpolate(bilinear, align_corners=True) + nn.Conv2d(Cin, Cout, 1) + l1_loss under autograd, then
      .backward() into the feature map, the weight and the bias; default backend settings (cuDNN, TF32 allowed).
  (b) feature_head.decoded_feature_l1_loss_and_grad: resize kernel -> fused decoder + L1 kernels
      (csrc/feature_decoder.cu) -> gather resize backward.

Feature map 1080x1920 -> teacher 480x853, (Cin, Cout) = (128, 512) (LSeg) and (64, 256) (SAM).  Both are warmed up, then
timed with CUDA events in alternating rounds (ROUNDS x ITERS calls each).  Algorithmic bytes of (b): read the map, write
and read the resized map, read the teacher map, write dL/d(resized) and read it back, write dL/dmap; FLOPs: the three
products 3 x 2 Cout Cin N.  Rates are printed against the H100 SXM data-sheet 3.35 TB/s and 495 TFLOP/s dense TF32.
Development tool, not product code:
    python tools/time_feature_decoder.py
"""
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "feature-3dgs_b200"))
from diff_gaussian_rasterization.feature_head import decoded_feature_l1_loss_and_grad  # noqa: E402

HW, GHW = (1080, 1920), (480, 853)
SHAPES = [("LSeg", 128, 512), ("SAM", 64, 256)]
ROUNDS, ITERS, WARMUP = 6, 20, 5
PEAK_GBS, PEAK_TFLOPS = 3350.0, 495.0


def reference_step(fm, gt, conv):
    fm.grad = None
    conv.zero_grad(set_to_none=True)
    r = F.interpolate(fm[None], size=gt.shape[1:], mode="bilinear", align_corners=True)[0]
    loss = F.l1_loss(conv(r[None])[0], gt)
    loss.backward()
    return loss.detach(), fm.grad, conv.weight.grad, conv.bias.grad


def fused_step(fm, gt, conv):
    return decoded_feature_l1_loss_and_grad(fm, gt, conv.weight, conv.bias, 1.0)


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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                       text=True)
    print(q.stdout.strip() or q.stderr.strip())
    print("torch", torch.__version__, " cudnn.allow_tf32 =", torch.backends.cudnn.allow_tf32)
    gen = torch.Generator(device="cuda").manual_seed(0)
    for name, cin, cout in SHAPES:
        fm = torch.randn(cin, *HW, device="cuda", generator=gen)
        gt = torch.randn(cout, *GHW, device="cuda", generator=gen)
        conv = torch.nn.Conv2d(cin, cout, kernel_size=1).cuda()
        fa = fm.clone().requires_grad_(True)
        la, ga, wa, ba = reference_step(fa, gt, conv)
        wa, ba = wa.clone(), ba.clone()
        lb, gb, wb, bb = fused_step(fm, gt, conv)
        rel = lambda u, v: float((u - v.view_as(u)).abs().max() / u.abs().max())  # noqa: E731
        print(f"{name} Cin={cin} Cout={cout} {HW[0]}x{HW[1]} -> {GHW[0]}x{GHW[1]}: loss (a) {float(la):.7f} "
              f"(b) {float(lb):.7f}; max|diff|/max|(a)|: dmap {rel(ga, gb):.2e}, dW {rel(wa, wb):.2e}, db {rel(ba, bb):.2e}")
        for fn, a in ((reference_step, (fa, gt, conv)), (fused_step, (fm, gt, conv))):
            time_calls(fn, a, WARMUP)
        ta, tb = [], []
        for _ in range(ROUNDS):
            ta.append(time_calls(reference_step, (fa, gt, conv), ITERS))
            tb.append(time_calls(fused_step, (fm, gt, conv), ITERS))
        n, nm = GHW[0] * GHW[1], HW[0] * HW[1]
        nbytes = 4 * (2 * cin * nm + 4 * cin * n + cout * n)
        flops = 3 * 2 * cout * cin * n
        for label, ts in (("(a) pytorch", ta), ("(b) fused  ", tb)):
            ts = sorted(ts)
            med = ts[len(ts) // 2]
            gbs, tfl = nbytes / (med * 1e-3) / 1e9, flops / (med * 1e-3) / 1e12
            print(f"  {label} {med:8.3f} ms/call (median of {ROUNDS} rounds x {ITERS}; min {ts[0]:.3f}, max {ts[-1]:.3f})"
                  f"  {nbytes / 1e6:.0f} MB -> {gbs:7.1f} GB/s = {100 * gbs / PEAK_GBS:5.1f}% of 3.35 TB/s;"
                  f"  {flops / 1e9:.1f} GFLOP -> {tfl:6.1f} TFLOP/s = {100 * tfl / PEAK_TFLOPS:5.1f}% of 495")
        print(f"  speed-up (a)/(b): {sorted(ta)[ROUNDS // 2] / sorted(tb)[ROUNDS // 2]:.2f}x")
        del fa, ga, fm, gt
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
