"""Cost of the camera gradient, in one process:

  (a) the backward preprocess alone (profile stage PREPROCESS_BWD of f3dgs_profile_*) and the whole
      ViewBatch.backward, at config 3's cloud and camera (scenegen "c3_C32": 1 M Gaussians, SH degree 3, C = 32,
      1920x1080), with camera=False and camera=True, alternating;
  (b) one pose-refinement iteration at config 3's cloud, C = 0, 1920x1080: settings_from_w2c(se3_exp(xi) @ w2c0),
      forward, photometric_loss_and_grad, backward through _RasterizeGaussiansCamera, one Adam step on xi.

CUDA events, median over ROUNDS rounds of ITERS calls per arm.  The card's name and power limit are printed by the
same run.  Development tool:
    python tools/time_camera_grad.py
"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "feature-3dgs_b200"))
import scenegen  # noqa: E402
from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer, _C  # noqa: E402
from diff_gaussian_rasterization.camera import se3_exp, settings_from_w2c  # noqa: E402
from diff_gaussian_rasterization.image_loss import photometric_loss_and_grad  # noqa: E402
from diff_gaussian_rasterization.parallel import ViewBatch  # noqa: E402

ROUNDS, ITERS = 7, 5
STAGE_PREPROCESS_BWD = 7  # F3DGS_STAGE_PREPROCESS_BWD, include/f3dgs_b200.h


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def median(x):
    x = sorted(x)
    return x[len(x) // 2]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def preprocess_ms(fn):
    """Mean time of the backward preprocess stage (kernel + camera reduction) over the calls inside fn (the
    library's per-stage CUDA events)."""
    _C.profile_enable(True)
    _C.profile_read()
    fn()
    torch.cuda.synchronize()
    ms, cnt = _C.profile_read()
    _C.profile_enable(False)
    return ms[STAGE_PREPROCESS_BWD] / max(cnt[STAGE_PREPROCESS_BWD], 1)


def main():
    if not torch.cuda.is_available():
        sys.exit("time_camera_grad.py needs a CUDA device")
    dev = torch.device("cuda")
    print("card:", card())

    # (a) ViewBatch.backward with and without the camera gradient
    sc = scenegen.make_config("c3_C32")
    cam = sc.cameras[0]
    d = scenegen.to_torch(sc, dev)
    params = {k: d[k] for k in ("means3D", "scales", "rotations", "opacities", "shs", "semantic_feature")}
    vb = ViewBatch(params)
    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))
    color, feat, radii, depth, ctx = vb.forward(rs)
    gc, gf, gd = (torch.from_numpy(a).to(dev) for a in
                  scenegen.upstream_grads(cam.image_height, cam.image_width, sc.features.shape[-1]))
    arms = {False: [], True: []}
    pre = {False: [], True: []}
    for flag in (False, True):  # warm-up
        vb.backward(ctx, gc, gf, gd, camera=flag)
    torch.cuda.synchronize()
    for _ in range(ROUNDS):
        for flag in (False, True):
            arms[flag].append(timed(lambda: [vb.backward(ctx, gc, gf, gd, camera=flag) for _ in range(ITERS)]) / ITERS)
            pre[flag].append(preprocess_ms(lambda: [vb.backward(ctx, gc, gf, gd, camera=flag) for _ in range(ITERS)]))
    for flag in (False, True):
        print(f"camera={flag}: ViewBatch.backward {median(arms[flag]):.3f} ms/view, backward preprocess "
              f"{median(pre[flag]):.4f} ms (medians of {ROUNDS}x{ITERS})")

    # (b) one pose-refinement iteration, C = 0
    sc0 = scenegen.make_config("c3_C0")
    cam0 = sc0.cameras[0]
    d0 = scenegen.to_torch(sc0, dev)
    W, H = cam0.image_width, cam0.image_height
    w2c0 = torch.tensor(cam0.viewmatrix, device=dev).t().contiguous()
    with torch.no_grad():
        rs0 = settings_from_w2c(w2c0, cam0.tanfovx, cam0.tanfovy, H, W, d0["bg"], sh_degree=sc0.sh_degree)
        target = GaussianRasterizer(rs0)(means3D=d0["means3D"], means2D=torch.zeros_like(d0["means3D"]),
                                         opacities=d0["opacities"], shs=d0["shs"], scales=d0["scales"],
                                         rotations=d0["rotations"])[0]
    xi = torch.zeros(6, device=dev, requires_grad=True)
    opt = torch.optim.Adam([xi], lr=1e-3)

    def step():
        opt.zero_grad()
        rs_ = settings_from_w2c(se3_exp(xi) @ w2c0, cam0.tanfovx, cam0.tanfovy, H, W, d0["bg"],
                                sh_degree=sc0.sh_degree)
        color_ = GaussianRasterizer(rs_)(means3D=d0["means3D"], means2D=torch.zeros_like(d0["means3D"]),
                                         opacities=d0["opacities"], shs=d0["shs"], scales=d0["scales"],
                                         rotations=d0["rotations"])[0]
        _, g = photometric_loss_and_grad(color_, target)
        color_.backward(g)
        opt.step()

    for _ in range(3):
        step()
    its = [timed(lambda: [step() for _ in range(ITERS)]) / ITERS for _ in range(ROUNDS)]
    print(f"pose-refinement iteration (c3 cloud, C = 0, {W}x{H}): {median(its):.3f} ms (median of {ROUNDS}x{ITERS})")


if __name__ == "__main__":
    main()
