"""Per-call time and peak memory of render.py's PCA picture of a feature map, three ways, in one process:

  (a) the reference's feature_visualize_saving as written: F.normalize on the device, every 3rd pixel copied to the host,
      scikit-learn PCA(3), np.percentile, the projection back on the device, the image copied to the host (skipped, with a
      message, where scikit-learn is missing);
  (b) the same algorithm as PyTorch ops on the device: F.normalize, strided sample, matmul with TF32 off, eigh (cuSOLVER),
      quantile;
  (c) feature_head.pca_image(x): the native moments, eigh of the C x C covariance, range and image calls.

Settings: 1080x1920 at C = 512 float32 (a decoded LSeg map), the same map in float16 (a saved map) and C = 128 float32.
The maps are synthetic: a rank-3 signal, noise and a large common offset.  Arms (b) and (c) are timed with CUDA events,
(a) with the host clock around a synchronised call, in alternating rounds (median of ROUNDS rounds); every arm is warmed
up first.  Also printed: the native stages on their own (moments, eigh of the float64 covariance on the host with LAPACK
and on the device with cuSOLVER, range, image), the image pass's achieved bandwidth against the H100 SXM data-sheet
3.35 TB/s (bytes = the map once + the [N,3] image), the peak memory growth per arm (torch.cuda.max_memory_allocated), and
the largest image difference between the arms.  Development tool, not product code:
    python tools/time_feature_pca.py
"""
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "feature-3dgs_b200"))
from diff_gaussian_rasterization import _C  # noqa: E402
from diff_gaussian_rasterization import feature_head as fh  # noqa: E402

ROUNDS, ITERS = 3, 3
PEAK_GBS = 3350.0
SETTINGS = [("1080x1920, C = 512, float32", 512, torch.float32), ("1080x1920, C = 512, float16", 512, torch.float16),
            ("1080x1920, C = 128, float32", 128, torch.float32)]
H, W = 1080, 1920


def reference(feature):
    import sklearn.decomposition

    C = feature.shape[0]
    fmap = F.normalize(feature[None].float(), dim=1)
    f_samples = fmap.permute(0, 2, 3, 1).reshape(-1, C)[::3].cpu().numpy()
    pca = sklearn.decomposition.PCA(3)
    transformed = pca.fit_transform(f_samples)
    mean, comps = torch.tensor(f_samples.mean(0)).cuda(), torch.tensor(pca.components_).cuda()
    q1, q99 = np.percentile(transformed, [1, 99])
    vis = ((fmap.permute(0, 2, 3, 1).reshape(-1, C) - mean) @ comps.T - q1) / (q99 - q1)
    return vis.clamp(0, 1).reshape(feature.shape[1], feature.shape[2], 3).cpu()


def torch_gpu(feature):
    C = feature.shape[0]
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    fmap = F.normalize(feature.float().reshape(C, -1), dim=0)
    S = fmap[:, ::3]
    mean = S.mean(1)
    A = S - mean[:, None]
    cov = (A @ A.t()) / (A.shape[1] - 1)
    _, vec = torch.linalg.eigh(cov)
    comps = vec.flip(1)[:, :3].t()
    first = comps.abs().argmax(dim=1, keepdim=True)
    comps = comps * torch.sign(comps.gather(1, first))
    q = torch.quantile((comps @ A).flatten(), torch.tensor([0.01, 0.99], device=feature.device))
    vis = ((comps @ (fmap - mean[:, None]) - q[0]) / (q[1] - q[0])).clamp(0, 1)
    torch.backends.cuda.matmul.allow_tf32 = prev
    return vis.t().reshape(feature.shape[1], feature.shape[2], 3)


def native(feature):
    return fh.pca_image(feature)


def synthetic(C, dtype, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    Q, _ = torch.linalg.qr(torch.randn(C, 3, device="cuda", generator=g))
    o = torch.nn.functional.normalize(torch.randn(C, device="cuda", generator=g), dim=0)
    z = torch.randn(3, H * W, device="cuda", generator=g) * torch.tensor([3.0, 2.0, 1.2], device="cuda")[:, None]
    x = 8.0 * o[:, None] + Q @ z
    x += 0.05 * torch.randn(C, H * W, device="cuda", generator=g)
    return x.view(C, H, W).to(dtype)


def gpu_ms(fn, *args, n=ITERS):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn(*args)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def host_ms(fn, *args):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn(*args)
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def peak(fn, *args):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn(*args)
    torch.cuda.synchronize()
    return out, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def med(v):
    return sorted(v)[len(v) // 2]


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                       text=True)
    print(q.stdout.strip() or q.stderr.strip())
    try:
        import sklearn

        have_sk = True
        print("torch", torch.__version__, " scikit-learn", sklearn.__version__, " host threads", torch.get_num_threads())
    except ImportError:
        have_sk = False
        print("arm (a) skipped: scikit-learn is not installed on this machine")
    for name, C, dt in SETTINGS:
        x = synthetic(C, dt)
        N, esize = H * W, x.element_size()
        arms = [("(b) pytorch gpu", torch_gpu), ("(c) native     ", native)]
        if have_sk:
            arms.insert(0, ("(a) reference  ", reference))
        outs, mems, times = {}, {}, {a: [] for a, _ in arms}
        for a, fn in arms:
            outs[a], mems[a] = peak(fn, x)
        for a, fn in arms:  # warm-up beyond the peak-memory call
            fn(x)
        for _ in range(ROUNDS):
            for a, fn in arms:
                times[a].append(host_ms(fn, x) if a.startswith("(a)") else gpu_ms(fn, x))
        img_c = outs["(c) native     "].float().cpu()
        print(f"{name}: N = {N}, n = {(N + 2) // 3} samples, map {C * N * esize / 1e9:.2f} GB")
        for a, _ in arms:
            ts = times[a]
            diff = "" if a.startswith("(c)") else f"  max|image - (c)| {float((outs[a].float().cpu() - img_c).abs().max()):.2e}"
            print(f"  {a} {med(ts):10.2f} ms/call (median of {ROUNDS}; min {min(ts):.2f}, max {max(ts):.2f})  "
                  f"peak device memory growth {mems[a]:8.1f} MiB{diff}")
        # native stages on their own
        mean, cov = _C.feature_pca_moments(x)
        t_mom = med([gpu_ms(_C.feature_pca_moments, x) for _ in range(ROUNDS)])
        covd = cov.clone()
        t_eig_dev = med([host_ms(torch.linalg.eigh, covd) for _ in range(ROUNDS + 1)][1:])
        t_eig_host = med([host_ms(lambda c: torch.linalg.eigh(c.cpu()), covd) for _ in range(ROUNDS + 1)][1:])
        fit = fh.pca_fit(x)
        rng = torch.stack((fit.lo, fit.hi))
        t_rng = med([gpu_ms(_C.feature_pca_range, x, fit.mean, fit.components) for _ in range(ROUNDS)])
        t_img = med([gpu_ms(_C.feature_pca_image, x, fit.mean, fit.components, rng) for _ in range(ROUNDS)])
        gbs = (C * N * esize + N * 12) / (t_img * 1e-3) / 1e9
        print(f"  stages: moments {t_mom:.2f} ms, eigh {C}x{C} float64 host (LAPACK, incl. copy) {t_eig_host:.2f} ms / "
              f"device (cuSOLVER) {t_eig_dev:.2f} ms, range {t_rng:.2f} ms, image {t_img:.2f} ms = {gbs:.0f} GB/s "
              f"({100 * gbs / PEAK_GBS:.1f}% of 3.35 TB/s)")
        print(f"  speed-up (b)/(c): {med(times['(b) pytorch gpu']) / med(times['(c) native     ']):.2f}x"
              + (f", (a)/(c): {med(times['(a) reference  ']) / med(times['(c) native     ']):.1f}x" if have_sk else ""))
        del x, outs, mean, cov, covd, fit
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
