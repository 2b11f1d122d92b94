"""Cost of the depth distortion loss, in one process, at config 3's cloud and camera (1 M Gaussians, SH degree 3,
1920x1080, scenegen seed 3) with C = 0 and C = 128: the forward and backward composite stages (the library's per-stage
events) and a forward plus `ViewBatch.backward` per view (CUDA events around each round, per-stage profiling off), with
the distortion (`ViewBatch.forward_distortion`, nonzero g_distortion) and without it (`ViewBatch.forward`),
alternating, medians over ROUNDS rounds of ITERS views per arm.

The card's name and power limit are printed by the same run.  Development tool:
    python tools/time_distortion.py
"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "feature-3dgs_b200"))
import scenegen  # noqa: E402
from diff_gaussian_rasterization import GaussianRasterizationSettings, _C  # noqa: E402
from diff_gaussian_rasterization.parallel import ViewBatch  # noqa: E402

ROUNDS, ITERS = 7, 5
STAGE_COMPOSITE_FWD, STAGE_COMPOSITE_BWD = 5, 6  # F3DGS_STAGE_*, include/f3dgs_b200.h


def median(x):
    x = sorted(x)
    return x[len(x) // 2]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def run(C, dev):
    sc = scenegen.make_scene(P=1_000_000, W=1920, H=1080, C=max(C, 1), sh_degree=3, views=1, seed=3)
    cam = sc.cameras[0]
    d = scenegen.to_torch(sc, dev)
    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))
    keys = ("means3D", "scales", "rotations", "opacities", "shs") + (("semantic_feature",) if C else ())
    vb = ViewBatch({k: d[k] for k in keys})
    H, W = cam.image_height, cam.image_width
    gc, gf, gd = (torch.from_numpy(a).to(dev) for a in scenegen.upstream_grads(H, W, max(C, 1)))
    g = torch.Generator().manual_seed(1)
    gD = torch.randn(1, H, W, generator=g).to(dev) * 1e-6

    def step(dist):
        if dist:
            *_, ctx = vb.forward_distortion(rs)
            vb.backward(ctx, gc, gf if C else None, gd, g_distortion=gD)
        else:
            *_, ctx = vb.forward(rs)
            vb.backward(ctx, gc, gf if C else None, gd)

    for dist in (False, True):  # warm-up
        step(dist)
    torch.cuda.synchronize()
    arms = (False, True)
    t = {a: [] for a in arms}
    for _ in range(ROUNDS):
        for a in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(ITERS):
                step(a)
            e1.record()
            torch.cuda.synchronize()
            t[a].append(e0.elapsed_time(e1) / ITERS)
    fwd, bwd = {a: [] for a in arms}, {a: [] for a in arms}
    for _ in range(ROUNDS):
        for a in arms:
            _C.profile_enable(True)
            _C.profile_read()
            for _ in range(ITERS):
                step(a)
            torch.cuda.synchronize()
            ms, cnt = _C.profile_read()
            _C.profile_enable(False)
            fwd[a].append(ms[STAGE_COMPOSITE_FWD] / max(cnt[STAGE_COMPOSITE_FWD], 1))
            bwd[a].append(ms[STAGE_COMPOSITE_BWD] / max(cnt[STAGE_COMPOSITE_BWD], 1))
    for a in arms:
        print(f"C={C} distortion={a}: composite forward {median(fwd[a]):.3f} ms, composite backward {median(bwd[a]):.3f} ms "
              f"(profiled rounds); forward + ViewBatch.backward {median(t[a]):.3f} ms per view (median of "
              f"{ROUNDS}x{ITERS}, per-round ms: {', '.join(f'{x:.3f}' for x in t[a])})")
    del vb
    torch.cuda.empty_cache()


def main():
    if not torch.cuda.is_available():
        sys.exit("time_distortion.py needs a CUDA device")
    dev = torch.device("cuda")
    print("card:", card())
    for C in (0, 128):
        run(C, dev)


if __name__ == "__main__":
    main()
