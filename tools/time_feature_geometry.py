"""Cost of the feature term of dL/dalpha (f3dgs_backward_feature_geometry), in one process, at config 3's cloud and
camera (1 M Gaussians, SH degree 3, 1920x1080, scenegen seed 3) with C = 128 and C = 512:

  (a) the backward composite stage (profile stage COMPOSITE_BWD of f3dgs_profile_*: the geometry walk, feature_bwd and,
      with the term, the pair dot products and the re-walk) with and without the feature term, alternating, median over
      ROUNDS rounds of ITERS backwards per arm;
  (b) the feature term's two kernels alone, feature_dot_kernel and composite_bwd_kernel<FEAT>, from a torch.profiler run
      of its own (mean device time per call).

The card's name and power limit are printed by the same run.  Development tool:
    python tools/time_feature_geometry.py
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

ROUNDS, ITERS = 7, 5
STAGE_COMPOSITE_BWD = 6  # F3DGS_STAGE_COMPOSITE_BWD, include/f3dgs_b200.h


def median(x):
    x = sorted(x)
    return x[len(x) // 2]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def composite_ms(fn):
    """Mean time of the backward composite stage over the calls inside fn (the library's per-stage CUDA events)."""
    _C.profile_enable(True)
    _C.profile_read()
    fn()
    torch.cuda.synchronize()
    ms, cnt = _C.profile_read()
    _C.profile_enable(False)
    return ms[STAGE_COMPOSITE_BWD] / max(cnt[STAGE_COMPOSITE_BWD], 1)


def main():
    if not torch.cuda.is_available():
        sys.exit("time_feature_geometry.py needs a CUDA device")
    dev = torch.device("cuda")
    print("card:", card())
    for C in (128, 512):
        sc = scenegen.make_scene(P=1_000_000, W=1920, H=1080, C=C, sh_degree=3, views=1, seed=3)
        cam = sc.cameras[0]
        d = scenegen.to_torch(sc, dev)
        rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))
        e = torch.Tensor([])
        R, color, fmap, depth, radii, geom, binning, img = _C.rasterize_gaussians(
            rs.bg, d["means3D"], e, d["semantic_feature"], d["opacities"], d["scales"], d["rotations"], 1.0, e,
            rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, cam.image_height, cam.image_width, d["shs"],
            rs.sh_degree, rs.campos, False, False)
        gc, gf, gd = (torch.from_numpy(a).to(dev) for a in
                      scenegen.upstream_grads(cam.image_height, cam.image_width, C))
        args = (rs.bg, d["means3D"], radii, e, d["semantic_feature"], d["scales"], d["rotations"], 1.0, e,
                rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, gc, gf, gd, d["shs"], rs.sh_degree, rs.campos,
                geom, R, binning, img, False)
        arms = {
            False: lambda: _C.rasterize_gaussians_backward(*args),
            True: lambda: _C.rasterize_gaussians_backward_feature_geometry(*args, False),
        }
        for fn in arms.values():  # warm-up
            fn()
        torch.cuda.synchronize()
        t = {False: [], True: []}
        for _ in range(ROUNDS):
            for flag, fn in arms.items():
                t[flag].append(composite_ms(lambda: [fn() for _ in range(ITERS)]))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(ITERS):
                arms[True]()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            tag = ("pair dot products" if "feature_dot_kernel" in ev.key else
                   "re-walk" if "composite_bwd_kernel" in ev.key and ("BwdMode)3" in ev.key or "FEAT" in ev.key) else
                   None)
            if tag:
                kern[tag] = kern.get(tag, 0.0) + ev.device_time_total / 1e3 / ITERS
        print(f"C = {C}: backward composite {median(t[False]):.3f} ms without the feature term, "
              f"{median(t[True]):.3f} ms with it (medians of {ROUNDS}x{ITERS}); "
              + ", ".join(f"{k} {v:.3f} ms" for k, v in kern.items()) + " (profiler, mean per call)")
        del d, geom, binning, img, fmap


if __name__ == "__main__":
    main()
