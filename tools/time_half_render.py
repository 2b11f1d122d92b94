"""Forward time and peak memory of rendering a feature field to float16, two ways, in one process:

  (a) what a caller does without float16 rendering: a float32 render, then feature_map.half();
  (b) a float16 render: semantic_feature cast to float16 once (outside the timed loop), the map written as float16.

Config 3's cloud and camera (1 M Gaussians, 1920x1080) at C = 128, 512 and 2048, forward only, through the public
GaussianRasterizer under torch.no_grad().  The two arms of each row are first checked bitwise equal
(render(sf16.float()).half() against render(sf16)), warmed up, then timed with CUDA events in alternating rounds
(ROUNDS x ITERS calls each); the peak memory of one call of each arm is measured above what is allocated before it
(features and scene included in neither).  The card's name and power limit are read in the same run.  Development tool:
    python tools/time_half_render.py [C ...]
"""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "feature-3dgs_b200")):
    sys.path.insert(0, p)
import scenegen  # noqa: E402
from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer  # noqa: E402

WIDTHS = (128, 512, 2048)
ROUNDS, ITERS, WARMUP = 5, 4, 2


def time_calls(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def peak_bytes(fn):
    """Peak allocation of one call above what is allocated before it (its result is dropped after)."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del out
    return peak


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    print(q.stdout.strip() or f"nvidia-smi unavailable: {q.stderr.strip()}")
    print(f"torch {torch.__version__}, device {torch.cuda.get_device_name()}")
    widths = [int(a) for a in sys.argv[1:]] or list(WIDTHS)

    sc = scenegen.make_config("c3")
    sc.features = np.zeros((sc.P, 1, 0), np.float32)  # the width is given per row
    cam = sc.cameras[0]
    H, W = cam.image_height, cam.image_width
    t = scenegen.to_torch(sc, "cuda")
    rast = GaussianRasterizer(GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, "cuda")))
    means2D = torch.zeros_like(t["means3D"])

    def render(sf):
        return rast(means3D=t["means3D"], means2D=means2D, opacities=t["opacities"], shs=t["shs"], semantic_feature=sf,
                    scales=t["scales"], rotations=t["rotations"])

    rows = []
    with torch.no_grad():
        for C in widths:
            sf16 = torch.randn(sc.P, 1, C, device="cuda", generator=torch.Generator("cuda").manual_seed(C)).half()
            sf32 = sf16.float()
            arm_a = lambda: render(sf32)[1].half()  # noqa: E731
            arm_b = lambda: render(sf16)[1]  # noqa: E731
            fa, fb = arm_a(), arm_b()
            same = fa.dtype == fb.dtype == torch.float16 and torch.equal(fa.view(torch.int16), fb.view(torch.int16))
            del fa, fb
            for fn in (arm_a, arm_b):
                for _ in range(WARMUP):
                    fn()
            pa, pb = peak_bytes(arm_a), peak_bytes(arm_b)
            ta, tb = [], []
            for _ in range(ROUNDS):
                ta.append(time_calls(arm_a, ITERS))
                tb.append(time_calls(arm_b, ITERS))
            ta, tb = sorted(ta), sorted(tb)
            rows.append((C, ta, tb, pa, pb, same))
            del sf16, sf32
            torch.cuda.empty_cache()

    map16 = lambda C: C * H * W * 2 / 2**30  # noqa: E731
    print(f"\nconfig 3 cloud (P = {sc.P}), {W}x{H}, forward only; median of {ROUNDS} rounds x {ITERS} calls "
          f"(min-max); peak = one call above what is allocated before it")
    print(f"{'C':>5} | {'(a) f32 render + .half() ms':>28} | {'(b) f16 render ms':>22} | {'(a)/(b)':>7} | "
          f"{'peak (a) GiB':>12} | {'peak (b) GiB':>12} | {'f16 map GiB':>11} | bitwise")
    for C, ta, tb, pa, pb, same in rows:
        print(f"{C:>5} | {ta[ROUNDS // 2]:10.3f} ({ta[0]:.3f}-{ta[-1]:.3f}) | {tb[ROUNDS // 2]:9.3f} "
              f"({tb[0]:.3f}-{tb[-1]:.3f}) | {ta[ROUNDS // 2] / tb[ROUNDS // 2]:6.3f}x | {pa / 2**30:12.2f} | "
              f"{pb / 2**30:12.2f} | {map16(C):11.2f} | {'equal' if same else 'DIFFERENT'}")
    if not all(r[-1] for r in rows):
        sys.exit("the two arms disagree")


if __name__ == "__main__":
    main()
