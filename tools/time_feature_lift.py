"""Time per view and peak memory of lifting a teacher feature map onto Gaussians, two ways, in one process:

  (a) lift         feature_head.FeatureLift.add: a forward at C = 0 with zero colors_precomp, then the native lift
                   (the backward composite's lift mode + the feature kernel over its lists);
  (b) composition  the same forward, then the full rasterize_gaussians_backward with dL/dfeature_map = the teacher map,
                   dL/dcolor = the planes (1, 0, 0) and dL/ddepth = 0: dL_dsemantic_feature is the lift's numerator and
                   dL_dcolors[:, 0] its denominator.

Config 3's cloud and camera (scenegen "c3", 1 M Gaussians) rendered at the teacher's resolution 480x853, at C = 512 with
a float16 teacher map (a saved LSeg map) and C = 128 float32.  Each arm is warmed up, then the arms alternate for ROUNDS
rounds of ITERS views each, timed with CUDA events (median per view).  Also printed: the C = 0 forward on its own (its
share of a lift), the peak memory growth per arm (torch.cuda.max_memory_allocated: torch's allocator only; both arms
also take the instance lists, 8 R x 136 bytes, from the CUDA default pool, printed separately), the largest relative
difference between the arms' sums, and the card's name and power limit, read in the same run.  Development tool:
    python tools/time_feature_lift.py
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
from diff_gaussian_rasterization.feature_head import FeatureLift  # noqa: E402

ROUNDS, ITERS = 5, 4
HG, WG = 480, 853
CASES = [(512, torch.float16), (128, torch.float32)]


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2**20


def median(x):
    x = sorted(x)
    return x[len(x) // 2]


def main():
    if not torch.cuda.is_available():
        sys.exit("time_feature_lift.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    print(q.stdout.strip() or f"nvidia-smi unavailable: {q.stderr.strip()}")
    print(f"torch {torch.__version__}, device {torch.cuda.get_device_name()}")

    sc = scenegen.make_config("c3_C0")
    t = scenegen.to_torch(sc, "cuda")
    P = sc.P
    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, sc.cameras[0], "cuda"))
    rs = rs._replace(image_height=HG, image_width=WG)
    e = torch.empty(0, device="cuda")
    colors = torch.zeros(P, 3, device="cuda")
    gc = torch.zeros(3, HG, WG, device="cuda")
    gc[0] = 1.0
    gd = torch.zeros(1, HG, WG, device="cuda")

    def forward():
        return _C.rasterize_gaussians(rs.bg, t["means3D"], colors, e, t["opacities"], t["scales"], t["rotations"], 1.0,
                                      e, rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, HG, WG, e, rs.sh_degree,
                                      rs.campos, False, False)

    for C, dtype in CASES:
        fmap = torch.randn(C, HG, WG, device="cuda", generator=torch.Generator(device="cuda").manual_seed(C)).to(dtype)
        lift = FeatureLift(t["means3D"], t["opacities"], t["scales"], t["rotations"], C)
        sf_shape = torch.empty(P, 1, C, device="cuda")
        out = {}

        def arm_lift():
            lift.flat.zero_()
            lift.add(rs, fmap)

        def arm_composition():
            R, _, _, _, radii, geom, binning, img = forward()
            g = _C.rasterize_gaussians_backward(rs.bg, t["means3D"], radii, colors, sf_shape, t["scales"],
                                                t["rotations"], 1.0, e, rs.viewmatrix, rs.projmatrix, rs.tanfovx,
                                                rs.tanfovy, gc, fmap, gd, e, rs.sh_degree, rs.campos, geom, R, binning,
                                                img, False)
            out["comp"] = (g[2].reshape(P, C), g[1][:, 0])

        arms = {"lift": arm_lift, "composition": arm_composition, "C = 0 forward": forward}
        for fn in arms.values():  # warm-up
            fn()
        times = {k: [] for k in arms}
        for _ in range(ROUNDS):
            for k, fn in arms.items():
                for _ in range(ITERS):
                    times[k].append(timed(fn))
        peaks = {k: peak(fn) for k, fn in arms.items()}

        arm_lift()
        arm_composition()
        fs, ws = lift.feature_sum[:, 0], lift.weight_sum
        cf, cw = out["comp"]
        rel = lambda a, b: float(((a.double() - b.double()).abs().max() / b.double().abs().max()))  # noqa: E731
        R = forward()[0]
        seen = int((ws > 0).sum())
        print(f"\nC = {C} {str(dtype).replace('torch.', '')} teacher {HG}x{WG}, P = {P}, R = {R}, "
              f"Gaussians with weight > 0: {seen}")
        print(f"  instance lists in both arms (CUDA pool, not in the peaks below): {8 * R * 136 / 2**20:.1f} MiB")
        for k in arms:
            print(f"  {k:14s} {median(times[k]):8.3f} ms/view (median of {len(times[k])}), "
                  f"peak memory growth {peaks[k]:8.1f} MiB")
        ml, mc, mf = (median(times[k]) for k in arms)
        print(f"  composition / lift: {mc / ml:.2f}x; C = 0 forward share of a lift: {100 * mf / ml:.1f} %")
        print(f"  largest difference between the arms, relative to max|.|: feature_sum {rel(fs, cf):.3g}, "
              f"weight_sum {rel(ws, cw):.3g}")


if __name__ == "__main__":
    main()
