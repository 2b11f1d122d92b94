"""Per-call time of distCUDA2, the initial-scale computation of create_from_pcd:

  (a) the native exact 3-NN mean squared distance (simple_knn._C.distCUDA2 -> f3dgs_knn_mean_dist, csrc/knn.cu);
  (b) the reference's simple-knn build (tests/ref_knn.py), when a reference checkout is present, in alternating rounds.

Workloads: 100k points uniform in [-1.3, 1.3]^3 (the reference's synthetic-scene initialisation), and 1 M / 5 M points
in Gaussian clusters with 0.1 % far outliers at 100x the cluster radius.  Every path is warmed up, then timed with CUDA
events over ROUNDS rounds of ITERS calls; the median round is reported.  The card's name and power limit are printed by
the same run.  Development tool, not product code:
    python tools/time_knn.py
"""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "feature-3dgs_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
from simple_knn._C import distCUDA2  # noqa: E402

ROUNDS, WARMUP = 6, 3


def uniform(P, seed):
    return np.random.default_rng(seed).uniform(-1.3, 1.3, (P, 3)).astype(np.float32)


def clustered(P, seed, n_clusters=256, radius=0.01, outlier_frac=0.001):
    rng = np.random.default_rng(seed)
    centers = rng.uniform(-1, 1, (n_clusters, 3))
    n_out = int(P * outlier_frac)
    pts = centers[rng.integers(0, n_clusters, P - n_out)] + rng.normal(0, radius, (P - n_out, 3))
    d = rng.normal(size=(n_out, 3))
    far = centers[rng.integers(0, n_clusters, n_out)] + 100 * radius * d / np.linalg.norm(d, axis=1, keepdims=True)
    return rng.permutation(np.concatenate([pts, far])).astype(np.float32)


def time_calls(fn, x, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn(x)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                       text=True)
    print(q.stdout.strip() or q.stderr.strip())
    ref = None
    try:
        import ref_knn

        ref = ref_knn.load()
    except Exception as e:  # a failed reference build only drops column (b)
        print("reference simple-knn unavailable:", str(e).splitlines()[0] if str(e) else type(e).__name__)
    print("reference simple-knn:", "built" if ref is not None else "not present (column (b) not measured)")
    workloads = [("uniform 100k", uniform(100_000, 1), 20), ("clustered 1M", clustered(1_000_000, 2), 5),
                 ("clustered 5M", clustered(5_000_000, 3), 2)]
    paths = [("(a) native", distCUDA2)] + ([("(b) reference", ref.distCUDA2)] if ref is not None else [])
    rows = []
    for name, pts, iters in workloads:
        x = torch.from_numpy(pts).cuda()
        outs = {}
        for pname, fn in paths:
            outs[pname] = fn(x)
            time_calls(fn, x, WARMUP)
        if ref is not None:
            a, b = outs["(a) native"], outs["(b) reference"]
            fin = torch.isfinite(b)
            rel = float(((a[fin].double() - b[fin].double()).abs() / b[fin].double().abs().clamp_min(1e-30)).max())
            print(f"{name}: native vs reference max rel diff {rel:.2e}, bitwise equal: {bool(torch.equal(a, b))}")
        ts = {p: [] for p, _ in paths}
        for _ in range(ROUNDS):
            for pname, fn in paths:
                ts[pname].append(time_calls(fn, x, iters))
        for pname, _ in paths:
            t = sorted(ts[pname])
            print(f"  {name:14s} {pname:14s} {t[len(t) // 2]:9.3f} ms/call (median of {ROUNDS} rounds x {iters}; "
                  f"min {t[0]:.3f}, max {t[-1]:.3f})")
        rows.append((name, {p: sorted(v)[len(v) // 2] for p, v in ts.items()}))
    print("\n| workload | native ms | reference ms |")
    print("|---|---|---|")
    for name, med in rows:
        r = f"{med['(b) reference']:.3f}" if "(b) reference" in med else "not measured"
        print(f"| {name} | {med['(a) native']:.3f} | {r} |")


if __name__ == "__main__":
    main()
