"""Cost of the neighbour-graph features (csrc/knn.cu graph_kernel, csrc/neighbors.cu, neighbors.py):

  (a) the exact k-NN graph (knn_graph) at P = 1 M for k = 8, 16 and 32, on a uniform cloud and on a clustered one with
      far outliers (test_knn_init.clustered), with the reverse lists built once after it;
  (b) the total-variation loss + gradient (feature_tv_loss_and_grad) at P = 1 M, k = 8, C = 128 and 512, against a torch
      restatement (gather of both ends of every edge, sign, index_add_ of the signs onto both ends, abs().sum() for the
      loss).  GB/s count the bytes a row needs without cache reuse, P (2k + 2) C 4 + P k 4 (own row, k neighbour rows
      and about k source rows, the gradient read and written, the indices), from shapes.  The gradients are compared;
  (c) one training step per view at config 3's cloud and camera (P = 1 M, 1920x1080), C = 128: ViewBatch forward,
      colour and feature losses, backward, all_reduce, Adam, activate, with and without add_feature_tv_grads(k = 8) on
      a cached graph.
  The arms of each part alternate over ROUNDS rounds of ITERS calls after a warm-up, timed with CUDA events; medians
  (min-max).  The card's name and power limit are printed by the same run.  Development tool:
      python tools/time_neighbors.py [graph] [tv] [step]
"""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "feature-3dgs_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import scenegen  # noqa: E402
from diff_gaussian_rasterization import GaussianRasterizationSettings  # noqa: E402
from diff_gaussian_rasterization import feature_head as fh  # noqa: E402
from diff_gaussian_rasterization import neighbors as nb  # noqa: E402
from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid  # noqa: E402
from test_knn_init import clustered  # noqa: E402

P_ROWS = 1_000_000
ROUNDS, ITERS = 5, 3
STEP_C = 128
LRS = dict(xyz=1.6e-5, f_dc=2.5e-3, f_rest=1.25e-4, opacity=0.05, scaling=5e-3, rotation=1e-3, semantic_feature=1e-3)


def time_calls(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def alternate(arms, rounds=ROUNDS, iters=ITERS):
    """{name: sorted per-call ms over the rounds}, the arms alternating, each warmed up first"""
    for fn in arms.values():
        fn()
    t = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            t[k].append(time_calls(fn, iters))
    return {k: sorted(v) for k, v in t.items()}


def fmt(v):
    return f"{v[len(v) // 2]:8.3f} ({v[0]:.3f}-{v[-1]:.3f})"


def graph():
    rng = np.random.default_rng(0)
    clouds = {"uniform": torch.from_numpy(rng.uniform(-1.3, 1.3, (P_ROWS, 3)).astype(np.float32)).cuda(),
              "clustered": torch.from_numpy(clustered(P_ROWS, 1)).cuda()}
    print(f"\n(a) exact k-NN graph at P = {P_ROWS}: median of {ROUNDS} rounds x {ITERS} calls (min-max), ms per call")
    for name, pts in clouds.items():
        arms = {}
        for k in (8, 16, 32):
            arms[f"k={k}"] = lambda k=k: nb.knn_graph(pts, k)
            arms[f"k={k} + reverse"] = lambda k=k: nb.knn_graph(pts, k).reverse()
        t = alternate(arms)
        for a, v in t.items():
            print(f"  {name:>9} {a:<15} {fmt(v)}")


def torch_tv(f, idx, weight, grad):
    P, k = idx.shape
    C = f.shape[1]
    valid = idx >= 0
    rows = torch.arange(P, device=f.device)[:, None].expand(P, k)[valid]
    nbrs = idx[valid].long()
    d = f[rows] - f[nbrs]
    s = weight / (rows.numel() * C)
    sg = torch.sign(d) * s
    grad.index_add_(0, rows, sg)
    grad.index_add_(0, nbrs, -sg)
    return d.abs().sum() * s


def tv():
    g = torch.Generator(device="cuda").manual_seed(0)
    pts = torch.from_numpy(clustered(P_ROWS, 2)).cuda()
    k = 8
    graph = nb.knn_graph(pts, k)
    graph.reverse()
    print(f"\n(b) total variation loss + gradient at P = {P_ROWS}, k = {k}: median of {ROUNDS} rounds x {ITERS} calls "
          f"(min-max), ms per call")
    for C in (128, 512):
        f = torch.randn(P_ROWS, C, device="cuda", generator=g)
        ga, gb = torch.zeros_like(f), torch.zeros_like(f)
        t = alternate({"ours": lambda: nb.feature_tv_loss_and_grad(f, graph, 1.0, ga),
                       "torch": lambda: torch_tv(f, graph.idx, 1.0, gb)})
        ga.zero_(), gb.zero_()
        la, lb = nb.feature_tv_loss_and_grad(f, graph, 1.0, ga), torch_tv(f, graph.idx, 1.0, gb)
        med = {a: v[len(v) // 2] for a, v in t.items()}
        nbytes = P_ROWS * (2 * k + 2) * C * 4 + P_ROWS * k * 4
        print(f"  C = {C}: ours {fmt(t['ours'])}  torch {fmt(t['torch'])}  {med['torch'] / med['ours']:5.2f}x  | "
              f"{nbytes / med['ours'] / 1e6:7.1f} GB/s (bytes without reuse); gradients max |diff| "
              f"{float((ga - gb).abs().max()):.3g}, losses {float(la):.6g} / {float(lb):.6g}")
        del f, ga, gb
        torch.cuda.empty_cache()


def step():
    sc = scenegen.make_config("c3")
    sc.features = np.zeros((sc.P, 1, 0), np.float32)
    cam = sc.cameras[0]
    H, W = cam.image_height, cam.image_width
    t = scenegen.to_torch(sc, "cuda")
    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, "cuda"))
    gc, _, gd = [torch.from_numpy(a).cuda() for a in scenegen.upstream_grads(H, W, 0, seed=99)]
    Hg, Wg = max(round(H / 2.25), 1), max(round(W / 2.25), 1)
    gt = torch.rand(STEP_C, Hg, Wg, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    M = (sc.sh_degree + 1) ** 2
    shs = t["shs"][:, :M]
    sf = torch.randn(sc.P, 1, STEP_C, device="cuda", generator=torch.Generator("cuda").manual_seed(1)) * 0.1
    st = GaussianState(t["means3D"].clone(), shs[:, :1].clone(), shs[:, 1:].clone(),
                       inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                       t["rotations"].clone(), sf)
    del t
    st.activate()
    st.neighbor_graph(8).reverse()

    def step_of(tv_weight):
        def fn():
            vb = st.batch()
            vb.zero_()
            color, feat, radii, depth, ctx = vb.forward(rs)
            _, gfeat = fh.feature_l1_loss_and_grad(feat, gt, 1.0)
            vb.backward(ctx, gc, gfeat, gd, last=True)
            vb.all_reduce()
            if tv_weight:
                st.add_feature_tv_grads(tv_weight, k=8)
            st.step(LRS)
            st.activate()

        return fn

    t = alternate({"without": step_of(0.0), "with TV": step_of(0.1)})
    print(f"\n(c) one training step per view, config 3 cloud (P = {st.P}), {W}x{H}, C = {STEP_C}, k = 8 (graph cached): "
          f"median of {ROUNDS} rounds x {ITERS} steps (min-max)")
    for a, v in t.items():
        print(f"  {a:>8}: {fmt(v)} ms/step")


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    print(q.stdout.strip() or f"nvidia-smi unavailable: {q.stderr.strip()}")
    print(f"torch {torch.__version__}, device {torch.cuda.get_device_name()}")
    which = sys.argv[1:] or ["graph", "tv", "step"]
    if "graph" in which:
        graph()
    if "tv" in which:
        tv()
    if "step" in which:
        step()


if __name__ == "__main__":
    main()
