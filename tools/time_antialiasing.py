"""Cost of antialiased rendering, in one process, at config 3's cloud and camera (1 M Gaussians, SH degree 3, 1920x1080,
scenegen seed 3) with C = 128: a forward (`ViewBatch.forward`) plus `ViewBatch.backward` per view, with and without
antialiasing, alternating, median over ROUNDS rounds of ITERS views per arm (CUDA events around each round, per-stage
profiling off), and then, in separate alternating rounds with the library's per-stage events on, the preprocess forward
and backward stages, the only kernels the option changes.

The card's name and power limit are printed by the same run.  Development tool:
    python tools/time_antialiasing.py
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
STAGE_PREPROCESS_FWD, STAGE_PREPROCESS_BWD = 0, 7  # F3DGS_STAGE_*, include/f3dgs_b200.h


def median(x):
    x = sorted(x)
    return x[len(x) // 2]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def main():
    if not torch.cuda.is_available():
        sys.exit("time_antialiasing.py needs a CUDA device")
    dev = torch.device("cuda")
    print("card:", card())
    C = 128
    sc = scenegen.make_scene(P=1_000_000, W=1920, H=1080, C=C, sh_degree=3, views=1, seed=3)
    cam = sc.cameras[0]
    d = scenegen.to_torch(sc, dev)
    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))
    vb = ViewBatch({k: d[k] for k in ("means3D", "scales", "rotations", "opacities", "shs", "semantic_feature")})
    gc, gf, gd = (torch.from_numpy(a).to(dev) for a in scenegen.upstream_grads(cam.image_height, cam.image_width, C))

    def step(aa):
        color, feat, radii, depth, ctx = vb.forward(rs, antialiasing=aa)
        vb.backward(ctx, gc, gf, gd)

    for aa in (False, True):  # warm-up
        step(aa)
    torch.cuda.synchronize()
    t = {False: [], True: []}
    for _ in range(ROUNDS):
        for aa in (False, True):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(ITERS):
                step(aa)
            e1.record()
            torch.cuda.synchronize()
            t[aa].append(e0.elapsed_time(e1) / ITERS)
    stages = {False: [0.0, 0.0, 0], True: [0.0, 0.0, 0]}
    for _ in range(ROUNDS):
        for aa in (False, True):
            _C.profile_enable(True)
            _C.profile_read()
            for _ in range(ITERS):
                step(aa)
            torch.cuda.synchronize()
            ms, cnt = _C.profile_read()
            _C.profile_enable(False)
            stages[aa][0] += ms[STAGE_PREPROCESS_FWD]
            stages[aa][1] += ms[STAGE_PREPROCESS_BWD]
            stages[aa][2] += cnt[STAGE_PREPROCESS_FWD]
    for aa in (False, True):
        n = max(stages[aa][2], 1)
        print(f"antialiasing={aa}: forward + ViewBatch.backward {median(t[aa]):.3f} ms per view (median of "
              f"{ROUNDS}x{ITERS}, per-round ms: {', '.join(f'{x:.3f}' for x in t[aa])}); preprocess forward "
              f"{stages[aa][0] / n:.3f} ms, preprocess backward {stages[aa][1] / n:.3f} ms (profiled rounds, mean)")


if __name__ == "__main__":
    main()
