"""Training step time and peak memory with float32 and float16 feature fields, in one process.

The workload is bench.py's `step_e2e_batch` loop with the optimizer step added: ViewBatch forward, the colour / depth
loss through autograd on the two small maps, the fused L1 feature loss against a teacher at 1/2.25 resolution
(feature_l1_loss_and_grad), the accumulating backward and the fused Adam step of every group (GaussianState.step).
Config 3's cloud and camera (1 M Gaussians, 1920x1080) at C = 128 and 512; per width, the float32 arm and the float16 arm
(GaussianState(feature_dtype=torch.float16): float16 map, ScaledGrad map gradient, Adam refreshing the float16 copy) are
warmed up, then timed with CUDA events in alternating rounds (ROUNDS x ITERS steps each).  Peak memory is that of one
step above what is allocated before it (state and teacher included in neither).  The card's name and power limit are
read in the same run.  Development tool:
    python tools/time_half_training.py [C ...]
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
from diff_gaussian_rasterization import GaussianRasterizationSettings  # noqa: E402
from diff_gaussian_rasterization import feature_head as fh  # noqa: E402
from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid  # noqa: E402

WIDTHS = (128, 512)
ROUNDS, ITERS, WARMUP = 5, 4, 3
LRS = dict(xyz=1.6e-5, f_dc=2.5e-3, f_rest=1.25e-4, opacity=0.05, scaling=5e-3, rotation=1e-3, semantic_feature=1e-3)


def time_calls(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def peak_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def make_arm(sc, t, C, dtype, rs, gc, gd, gt):
    M = (sc.sh_degree + 1) ** 2
    shs = t["shs"][:, :M]
    sf = torch.randn(sc.P, 1, C, device="cuda", generator=torch.Generator("cuda").manual_seed(C)) * 0.1
    state = GaussianState(t["means3D"].clone(), shs[:, :1].clone(), shs[:, 1:].clone(),
                          inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                          t["rotations"].clone(), sf, feature_dtype=dtype)
    grad_dtype = torch.float16 if dtype == torch.float16 else None
    state.activate()
    vb = state.batch()

    def step():
        vb.zero_()
        color, feat, radii, depth, ctx = vb.forward(rs)
        outs = [color.requires_grad_(), depth.requires_grad_()]
        ((outs[0] * gc).sum() + (outs[1] * gd).sum()).backward()
        _, gfeat = fh.feature_l1_loss_and_grad(feat, gt, 1.0, grad_dtype=grad_dtype)
        vb.backward(ctx, color.grad, gfeat, depth.grad, last=True)
        vb.all_reduce()
        state.step(LRS)
        state.activate()

    return state, step


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
    Hg, Wg = max(round(H / 2.25), 1), max(round(W / 2.25), 1)
    t = scenegen.to_torch(sc, "cuda")
    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, "cuda"))
    gc, gf, gd = [torch.from_numpy(g).cuda() for g in scenegen.upstream_grads(H, W, 0, seed=99)]
    del gf

    rows = []
    for C in widths:
        gt = torch.rand(C, Hg, Wg, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
        arms = {}
        for dt in (torch.float32, torch.float16):
            arms[dt] = make_arm(sc, t, C, dt, rs, gc, gd, gt)
            for _ in range(WARMUP):
                arms[dt][1]()
        peaks = {dt: peak_bytes(arms[dt][1]) for dt in arms}
        times = {dt: [] for dt in arms}
        for _ in range(ROUNDS):
            for dt in arms:
                times[dt].append(time_calls(arms[dt][1], ITERS))
        rows.append((C, {dt: sorted(v) for dt, v in times.items()}, peaks))
        del arms, gt
        torch.cuda.empty_cache()

    print(f"\nconfig 3 cloud (P = {sc.P}), {W}x{H}, teacher {Wg}x{Hg}; one view per step: forward, colour loss, "
          f"feature L1 loss, backward, Adam; median of {ROUNDS} rounds x {ITERS} steps (min-max); peak = one step "
          f"above what is allocated before it")
    print(f"{'C':>5} | {'float32 ms/view':>22} | {'float16 ms/view':>22} | {'f32/f16':>7} | {'peak f32 GiB':>12} | "
          f"{'peak f16 GiB':>12}")
    f32, f16 = torch.float32, torch.float16
    for C, tm, pk in rows:
        a, b = tm[f32], tm[f16]
        print(f"{C:>5} | {a[ROUNDS // 2]:9.3f} ({a[0]:.3f}-{a[-1]:.3f}) | {b[ROUNDS // 2]:9.3f} ({b[0]:.3f}-{b[-1]:.3f}) "
              f"| {a[ROUNDS // 2] / b[ROUNDS // 2]:6.3f}x | {pk[f32] / 2**30:12.2f} | {pk[f16] / 2**30:12.2f}")


if __name__ == "__main__":
    main()
