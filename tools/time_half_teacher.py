"""Per-call time of the feature losses with a float16 teacher map (the data format's dtype), two ways, in one process:

  (a) what a caller does without float16 support: gt16.float() and then the float32 path;
  (b) the float16-native path: the same call with gt16 itself (the kernels upcast each element at its load).

and of writing a float16 decoded map: (a) feature_head.decode(...).half() against (b) decode(..., dtype=torch.float16).

Shapes: the LSeg --speedup loss (Cin 128 -> Cout 512, map 1080x1920, teacher 480x853,
decoded_feature_l1_loss_and_grad), the resize-L1 loss without a decoder (C = 512, same sizes, feature_l1_loss_and_grad),
and the decode at 1080x1920 (128 -> 512).  The two arms of each row are checked bitwise equal (the resize-L1 loss to
1e-6 relative: its cross-block sum uses float atomics), warmed up, then timed with CUDA events in alternating rounds
(ROUNDS x ITERS calls each).  The card's name and power limit are read in the same run.  Development tool:
    python tools/time_half_teacher.py
"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "feature-3dgs_b200"))
from diff_gaussian_rasterization import feature_head as fh  # noqa: E402

HW, GHW = (1080, 1920), (480, 853)
CIN, COUT = 128, 512
ROUNDS, ITERS, WARMUP = 6, 10, 3


def time_calls(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def compare(label, arm_a, arm_b, gt_mb):
    for fn in (arm_a, arm_b):
        for _ in range(WARMUP):
            fn()
    ta, tb = [], []
    for _ in range(ROUNDS):
        ta.append(time_calls(arm_a, ITERS))
        tb.append(time_calls(arm_b, ITERS))
    ta, tb = sorted(ta), sorted(tb)
    print(f"{label}")
    for name, ts in (("(a) upcast / cast  ", ta), ("(b) float16-native ", tb)):
        print(f"  {name} {ts[ROUNDS // 2]:8.3f} ms/call (median of {ROUNDS} rounds x {ITERS}; min {ts[0]:.3f}, "
              f"max {ts[-1]:.3f})")
    print(f"  (a)/(b) {ta[ROUNDS // 2] / tb[ROUNDS // 2]:.3f}x;  float16 map {gt_mb:.0f} MB, its float32 copy "
          f"{2 * gt_mb:.0f} MB")


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                       text=True)
    print(q.stdout.strip() or q.stderr.strip())
    print("torch", torch.__version__)
    gen = torch.Generator(device="cuda").manual_seed(0)
    n = GHW[0] * GHW[1]

    # --speedup: resize -> fused 1x1 decoder + L1 -> resize backward
    fm = torch.randn(CIN, *HW, device="cuda", generator=gen)
    W = torch.randn(COUT, CIN, 1, 1, device="cuda", generator=gen) / CIN ** 0.5
    b = 0.1 * torch.randn(COUT, device="cuda", generator=gen)
    gt16 = torch.randn(COUT, *GHW, device="cuda", generator=gen).half()
    dW, db = torch.zeros_like(W), torch.zeros_like(b)
    arm_a = lambda: fh.decoded_feature_l1_loss_and_grad(fm, gt16.float(), W, b, 1.0, dW, db)  # noqa: E731
    arm_b = lambda: fh.decoded_feature_l1_loss_and_grad(fm, gt16, W, b, 1.0, dW, db)  # noqa: E731
    ra = fh.decoded_feature_l1_loss_and_grad(fm, gt16.float(), W, b)
    rb = fh.decoded_feature_l1_loss_and_grad(fm, gt16, W, b)
    same = all(torch.equal(u, v) for u, v in zip(ra, rb))
    compare(f"LSeg --speedup loss {CIN}->{COUT}, {HW[0]}x{HW[1]} -> {GHW[0]}x{GHW[1]} (loss, dmap, dW, db bitwise "
            f"equal: {same})", arm_a, arm_b, COUT * n * 2 / 1e6)
    del ra, rb, arm_a, arm_b, gt16

    # decode of the rendered map at full resolution, written as float16
    y_a, y_b = fh.decode(fm, W, b).half(), fh.decode(fm, W, b, dtype=torch.float16)
    same = torch.equal(y_a.view(torch.int16), y_b.view(torch.int16))
    del y_a, y_b
    compare(f"decode {CIN}->{COUT} at {HW[0]}x{HW[1]} to float16 (bitwise equal: {same})",
            lambda: fh.decode(fm, W, b).half(), lambda: fh.decode(fm, W, b, dtype=torch.float16),
            COUT * HW[0] * HW[1] * 2 / 1e6)
    del fm, W, b, dW, db
    torch.cuda.empty_cache()

    # resize-L1 without a decoder, C = COUT
    fm = torch.randn(COUT, *HW, device="cuda", generator=gen)
    gt16 = torch.randn(COUT, *GHW, device="cuda", generator=gen).half()
    la, ga = fh.feature_l1_loss_and_grad(fm, gt16.float())
    lb, gb = fh.feature_l1_loss_and_grad(fm, gt16)
    same = torch.equal(ga, gb) and abs(float(la) - float(lb)) <= 1e-6 * abs(float(la))
    del la, ga, lb, gb
    compare(f"resize-L1 loss C={COUT}, {HW[0]}x{HW[1]} -> {GHW[0]}x{GHW[1]} (dmap bitwise and loss to 1e-6 equal: "
            f"{same})", lambda: fh.feature_l1_loss_and_grad(fm, gt16.float()), lambda: fh.feature_l1_loss_and_grad(fm, gt16),
            COUT * n * 2 / 1e6)


if __name__ == "__main__":
    main()
