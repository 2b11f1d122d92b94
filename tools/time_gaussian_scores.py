"""Time of the per-Gaussian blend-weight scores and of pruning:

  (a) score pass per view at config 3's cloud and camera (P = 1 M, 1920x1080): GaussianScores.add (C = 0 forward + the
      score walk) against FeatureLift(C = 1).add (the same forward + the lift walk, its instance lists and the feature
      kernel), alternating over ROUNDS rounds of ITERS calls, CUDA events, median; then, over one forward's buffers, the
      score walk alone against the lift call alone and the C = 0 forward alone;
  (b) GaussianState.prune at P = 1 M, M = 16, C = 128 and 512, a seeded 60 % prune: the native path (one plan, one
      compaction) against the PyTorch restatement {k: t[keep]} over the 21 tensors and max_radii2D; alternating, host
      clock around synchronised calls, median, with a bitwise comparison of both.

The card's name and power limit are printed by the same run.  Development tool:
    python tools/time_gaussian_scores.py
"""
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "feature-3dgs_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import scenegen  # noqa: E402
from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianScores, _C  # noqa: E402
from diff_gaussian_rasterization.feature_head import FeatureLift, _weights_forward  # noqa: E402
from diff_gaussian_rasterization.trainer import GaussianState  # noqa: E402

ROUNDS, ITERS, PRUNE_ROUNDS = 7, 10, 5
NAMES = GaussianState.NAMES


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else f"{torch.cuda.get_device_name()} (nvidia-smi failed)"


def events(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def med(x):
    return sorted(x)[len(x) // 2]


def bench_scores():
    sc = scenegen.make_config("c3_C0")
    t = scenegen.to_torch(sc, "cuda")
    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, sc.cameras[0], "cuda"))
    H, W, P = rs.image_height, rs.image_width, sc.P
    scores = GaussianScores(t["means3D"], t["opacities"], t["scales"], t["rotations"])
    lift = FeatureLift(t["means3D"], t["opacities"], t["scales"], t["rotations"], 1)
    fmap = torch.ones(1, H, W, device="cuda")
    arms = dict(score=lambda: scores.add(rs), lift=lambda: lift.add(rs, fmap))
    for f in arms.values():
        f()
    times = {k: [] for k in arms}
    for _ in range(ROUNDS):
        for k, f in arms.items():
            times[k].append(events(f, ITERS))
    ts, tl = med(times["score"]), med(times["lift"])
    print(f"score pass per view (P={P}, {W}x{H}): GaussianScores.add {ts:.3f} ms, FeatureLift(C=1).add {tl:.3f} ms "
          f"({(ts - tl) / tl * 100:+.1f} %)")
    # the walks alone over one forward's buffers, and that forward
    e = torch.empty(0, device="cuda")
    R, geom, binning, img = _weights_forward(scores._geom, scores._colors, e, False, rs, H, W)
    ws, mw = torch.zeros(P, device="cuda"), torch.zeros(P, device="cuda")
    pc = torch.zeros(P, dtype=torch.int64, device="cuda")
    fs, wl = torch.zeros(P, 1, device="cuda"), torch.zeros(P, device="cuda")
    walks = dict(score_walk=lambda: _C.gaussian_scores_accum(geom, R, binning, img, W, H, ws, mw, pc),
                 lift_call=lambda: _C.lift_features_accum(geom, R, binning, img, fmap, fs, wl),
                 forward_C0=lambda: _weights_forward(scores._geom, scores._colors, e, False, rs, H, W))
    for f in walks.values():
        f()
    times = {k: [] for k in walks}
    for _ in range(ROUNDS):
        for k, f in walks.items():
            times[k].append(events(f, ITERS))
    print("  alone, median: " + ", ".join(f"{k} {med(v):.3f} ms" for k, v in times.items()) + f"  (R = {R})")
    blended = int((scores.pixel_count > 0).sum())
    print(f"  Gaussians blended into the view: {blended} of {P}")


def make_state(P, C, M, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)  # noqa: E731
    st = GaussianState(r(P, 3), r(P, 1, 3), r(P, M - 1, 3), r(P, 1), r(P, 3), r(P, 4), r(P, 1, C))
    st.exp_avg = {k: torch.randn(v.shape, device="cuda", generator=g) for k, v in st.raw.items()}
    st.exp_avg_sq = {k: torch.rand(v.shape, device="cuda", generator=g) for k, v in st.raw.items()}
    st.max_radii2D = torch.rand(P, device="cuda", generator=g) * 40
    return st


def restate(st, keep):
    return [{k: g[k][keep] for k in NAMES} for g in (st.raw, st.exp_avg, st.exp_avg_sq)], st.max_radii2D[keep]


def bench_prune(P, C, M=16):
    g = torch.Generator(device="cuda").manual_seed(C)
    keep = torch.rand(P, device="cuda", generator=g) >= 0.6
    tn, tr = [], []
    ok = True
    for i in range(PRUNE_ROUNDS + 1):
        st = make_state(P, C, M, seed=i)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ref = restate(st, keep)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        st.prune(keep)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        if i:  # the first round warms both up
            tr.append((t1 - t0) * 1e3)
            tn.append((t2 - t1) * 1e3)
        for grp, a in zip(ref[0], (st.raw, st.exp_avg, st.exp_avg_sq)):
            ok &= all(torch.equal(grp[k].view(torch.int32), a[k].view(torch.int32)) for k in NAMES)
        ok &= torch.equal(ref[1], st.max_radii2D)
        del st, ref
        torch.cuda.empty_cache()
    width = 3 + 3 + 3 * (M - 1) + 1 + 3 + 4 + C
    gb = 3 * width * 4 * P * (1 + 0.4) / 1e9
    mn = med(tn)
    print(f"prune P={P} C={C} M={M}, 60 %: native {mn:.2f} ms ({gb / (mn / 1e3):.0f} GB/s of fields read + written), "
          f"restatement {med(tr):.2f} ms; bitwise equal: {ok}")


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    print("card:", card())
    bench_scores()
    torch.cuda.empty_cache()
    for C in (128, 512):
        bench_prune(1_000_000, C)


if __name__ == "__main__":
    main()
