"""Cost of the sparse Adam step against the dense one, in one process, at config 3's cloud and camera (1 M Gaussians, SH
degree 3, 1920x1080, scenegen seed 3), C = 128 and C = 512, float32 and float16 feature fields:

  * the visible fraction under config 3's camera (radii > 0, `ViewBatch.visible()`);
  * the seven-group `GaussianState.step` dense against masked, with that mask and with random masks of 10 %, 50 % and
    100 % of the Gaussians;
  * at C = 128, one whole training step per view (activate, zero, forward, colour loss, feature L1 loss against a
    853x480 teacher, backward, step), dense against masked (`visible=vb.visible()`);
  * `activate()` and `ViewBatch.zero_()` on their own (both still touch every Gaussian).

Arms alternate within each round; each round is timed with CUDA events, and medians over ROUNDS rounds of ITERS calls
are printed.  The card's name and power limit are printed by the same run.  Development tool:
    python tools/time_sparse_adam.py
"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "feature-3dgs_b200"))
import scenegen  # noqa: E402
from diff_gaussian_rasterization import GaussianRasterizationSettings  # noqa: E402
from diff_gaussian_rasterization import feature_head as fh  # noqa: E402
from diff_gaussian_rasterization.image_loss import photometric_loss_and_grad  # noqa: E402
from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid  # noqa: E402

ROUNDS, ITERS = 7, 5
LRS = dict(xyz=1.6e-6, f_dc=2.5e-5, f_rest=1.25e-6, opacity=5e-4, scaling=5e-5, rotation=1e-5, semantic_feature=1e-5)
TEACHER = (480, 853)


def median(x):
    x = sorted(x)
    return x[len(x) // 2]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def timed(arms):
    """arms: {name: callable} -> {name: [ms per call, one per round]}, the arms alternating within each round"""
    for f in arms.values():  # warm-up
        f()
    torch.cuda.synchronize()
    t = {a: [] for a in arms}
    for _ in range(ROUNDS):
        for a, f in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(ITERS):
                f()
            e1.record()
            torch.cuda.synchronize()
            t[a].append(e0.elapsed_time(e1) / ITERS)
    return t


def report(what, t):
    for a, x in t.items():
        print(f"  {what} {a}: {median(x):.3f} ms (per-round: {', '.join(f'{v:.3f}' for v in x)})")


def run(C, dtype, dev):
    sc = scenegen.make_scene(P=1_000_000, W=1920, H=1080, C=C, sh_degree=3, views=1, seed=3)
    cam = sc.cameras[0]
    d = scenegen.to_torch(sc, dev)
    st = GaussianState(d["means3D"], d["shs"][:, :1].contiguous(), d["shs"][:, 1:].contiguous(),
                       inverse_sigmoid(d["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(d["scales"]), d["rotations"],
                       d["semantic_feature"], feature_dtype=dtype)
    del d
    P = st.P
    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))
    H, W = cam.image_height, cam.image_width
    g = torch.Generator(device=dev).manual_seed(1)
    gt_color = torch.rand(3, H, W, device=dev, generator=g)
    gt_feat = torch.randn(C, *TEACHER, device=dev, generator=g)
    half = dtype == torch.float16

    def view(visible):
        """one training step of one view; visible: use the step's mask"""
        st.activate()
        vb = st.batch()
        vb.zero_()
        color, feat, radii, depth, ctx = vb.forward(rs)
        _, g_color = photometric_loss_and_grad(color, gt_color)
        _, g_feat = fh.feature_l1_loss_and_grad(feat, gt_feat, 1.0, grad_dtype=torch.float16 if half else None)
        vb.backward(ctx, g_color, g_feat, torch.zeros_like(depth), last=True)
        vb.all_reduce()
        st.step(LRS, visible=vb.visible() if visible else None)

    view(False)  # leaves the batch's gradients and statistics of one view in place
    vb = st.batch()
    cam_mask = vb.visible()
    frac = float(cam_mask.float().mean())
    print(f"C={C} {str(dtype).replace('torch.', '')}: visible fraction under config 3's camera {frac:.4f} "
          f"({int(cam_mask.sum())} of {P})")
    masks = {"camera": cam_mask}
    for pct in (10, 50, 100):
        masks[f"random {pct}%"] = torch.rand(P, device=dev, generator=g) < pct / 100
    arms = {"dense": lambda: st.step(LRS)}
    for name, m in masks.items():
        arms[f"masked ({name})"] = lambda m=m: st.step(LRS, visible=m)
    report("GaussianState.step", timed(arms))
    report("prologue", timed({"activate()": st.activate, "ViewBatch.zero_()": vb.zero_}))
    if C == 128:
        report("training step per view", timed({"dense": lambda: view(False), "masked": lambda: view(True)}))
    del st, vb, masks, arms
    torch.cuda.empty_cache()


def main():
    if not torch.cuda.is_available():
        sys.exit("time_sparse_adam.py needs a CUDA device")
    dev = torch.device("cuda")
    print("card:", card())
    for C in (128, 512):
        for dtype in (torch.float32, torch.float16):
            run(C, dtype, dev)


if __name__ == "__main__":
    main()
