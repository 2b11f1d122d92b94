"""Time of Mip-Splatting's 3D smoothing filter:

  (a) compute: filter3d.compute_3d_filter's native path (f3dgs_filter3d_compute, two kernels, one host read of the seen
      count) against the PyTorch restatement of the official compute_3D_filter (tests/ref_filter3d.py: a loop over the
      cameras of about 15 tensor kernels each), alternating over ROUNDS rounds after one warm-up call each, host clock
      around calls that end in torch.cuda.synchronize();
  (b) apply forward + backward (f3dgs_filter3d_apply + f3dgs_filter3d_apply_backward in place), CUDA events over ITERS
      back-to-back pairs;
  (c) one whole GaussianState training step (activate, ViewBatch forward and backward of STEP_VIEWS views with fixed
      upstream gradients, step) with and without the filter, alternating, host clock around synchronised steps,
      reported per view.

Workloads: config 3's cloud (P = 1 M, C = 128, 1920x1080) with V = 64 ring cameras (config 4's view count) and
V = 300.  Bytes are computed from shapes: the compute reads 12 B per Gaussian and 80 B per camera per block and writes 4,
its second pass reads and writes 4; the apply reads 20 and writes 16 B per Gaussian, the backward reads 36 and writes
16.  Camera tests per second = P V / compute time.  The card's name and power limit are printed by the same run.
Development tool:
    python tools/time_filter3d.py
"""
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "feature-3dgs_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import ref_filter3d  # noqa: E402
import scenegen  # noqa: E402
from diff_gaussian_rasterization import GaussianRasterizationSettings, _C  # noqa: E402
from diff_gaussian_rasterization.filter3d import camera_tensors, compute_from_tensors  # noqa: E402
from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid  # noqa: E402

ROUNDS, ITERS, STEP_VIEWS, STEP_ROUNDS = 5, 50, 4, 5
LRS = dict(xyz=1.6e-4, f_dc=2.5e-3, f_rest=1.25e-4, opacity=0.05, scaling=5e-3, rotation=1e-3, semantic_feature=0.05)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else f"{torch.cuda.get_device_name()} (nvidia-smi failed)"


def bench_compute(xyz, vms, intr):
    P, V = xyz.shape[0], vms.shape[0]
    nat = lambda: compute_from_tensors(xyz, vms, intr)  # noqa: E731
    rst = lambda: ref_filter3d.compute_3d_filter(xyz, vms, intr)  # noqa: E731
    a, b = nat(), rst()
    ulp = (torch.nextafter(b, torch.full_like(b, float("inf"))) - b).double()
    far = int(((a.double() - b.double()).abs() > 4 * ulp).sum())
    tn, tr = [], []
    for _ in range(ROUNDS):
        tn.append(timed(nat)[0])
        tr.append(timed(rst)[0])
    mn, mr = min(tn), min(tr)
    gb = (16 * P + 8 * P + 80 * V * ((P + 255) // 256)) / 1e9
    print(f"compute V={V:3d}: native {mn:8.3f} ms (median {sorted(tn)[len(tn) // 2]:.3f}), restatement {mr:8.2f} ms "
          f"(median {sorted(tr)[len(tr) // 2]:.2f}) -> {mr / mn:.0f}x; native {gb / (mn / 1e3):.1f} GB/s, "
          f"{P * V / (mn / 1e3) / 1e9:.1f} G camera tests/s; rows beyond 4 ulp of the restatement: {far} of {P}")


def bench_apply(P):
    g = torch.Generator(device="cuda").manual_seed(0)
    o = torch.rand(P, 1, device="cuda", generator=g)
    s = torch.rand(P, 3, device="cuda", generator=g) * 0.1
    f = torch.rand(P, 1, device="cuda", generator=g) * 0.01
    oo, so = torch.empty_like(o), torch.empty_like(s)
    go, gs = torch.randn(P, 1, device="cuda", generator=g), torch.randn(P, 3, device="cuda", generator=g)

    def pair():
        _C.filter3d_apply(o, s, f, oo, so)
        _C.filter3d_apply_backward(o, s, f, go, gs, go, gs)

    for _ in range(3):
        pair()
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    e0.record()
    for _ in range(ITERS):
        _C.filter3d_apply(o, s, f, oo, so)
    e1.record()
    for _ in range(ITERS):
        _C.filter3d_apply_backward(o, s, f, go, gs, go, gs)
    e2.record()
    torch.cuda.synchronize()
    tf, tb = e0.elapsed_time(e1) / ITERS, e1.elapsed_time(e2) / ITERS
    print(f"apply P={P}: forward {tf * 1e3:.1f} us ({36 * P / tf / 1e6:.0f} GB/s), backward {tb * 1e3:.1f} us "
          f"({52 * P / tb / 1e6:.0f} GB/s), per step {(tf + tb) * 1e3:.1f} us")


def bench_step(sc, rs):
    t = scenegen.to_torch(sc, "cuda")

    def state():
        return GaussianState(t["means3D"].clone(), t["shs"][:, :1].contiguous(), t["shs"][:, 1:].contiguous(),
                             inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                             t["rotations"].clone(), t["semantic_feature"].clone())

    plain, filt = state(), state()
    filt.compute_3d_filter(rs)
    views = rs[:STEP_VIEWS]
    H, W = views[0].image_height, views[0].image_width
    g = torch.Generator(device="cuda").manual_seed(1)
    gc = torch.randn(3, H, W, device="cuda", generator=g) * 1e-6
    gf = torch.randn(sc.C, H, W, device="cuda", generator=g) * 1e-8
    gd = torch.zeros(1, H, W, device="cuda")

    def step(st):
        st.activate()
        vb = st.batch()
        vb.zero_()
        for i, r in enumerate(views):
            _, _, _, _, ctx = vb.forward(r)
            vb.backward(ctx, gc, gf, gd, last=i == len(views) - 1)
        vb.all_reduce()
        st.step(LRS)

    step(plain)
    step(filt)
    tp, tf = [], []
    for _ in range(STEP_ROUNDS):
        tp.append(timed(lambda: step(plain))[0] / len(views))
        tf.append(timed(lambda: step(filt))[0] / len(views))
    mp, mf = sorted(tp)[len(tp) // 2], sorted(tf)[len(tf) // 2]
    print(f"training step per view (P={sc.P}, C={sc.C}, {W}x{H}, {len(views)} views per step), median: without the "
          f"filter {mp:.2f} ms, with it {mf:.2f} ms ({(mf - mp) / mp * 100:+.1f} %)")


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    print("card:", card())
    cfg = dict(scenegen.CONFIGS["c3"])
    for V in (64, 300):
        cfg["views"] = V
        sc = scenegen.make_scene(seed=3, **cfg)
        rs = [GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, c, "cuda")) for c in sc.cameras]
        xyz = torch.from_numpy(sc.means3D).cuda()
        vms, intr = camera_tensors(rs)
        bench_compute(xyz, vms, intr)
        if V == 64:
            bench_apply(sc.P)
            bench_step(sc, rs)
        del sc, rs, xyz, vms, intr
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
