"""Cost of AbsGS's absolute-gradient statistic:

  (a) the backward composite stage (the library's per-stage events) and forward + ViewBatch.backward per view at config
      3's cloud and camera (P = 1 M, 1920x1080, scenegen seed 3), C = 0 and C = 128, with ViewBatch(absgrad=False)
      against ViewBatch(absgrad=True); alternating rounds, CUDA events, medians;
  (b) GaussianState.densify_and_prune at P = 1 M, M = 16, C = 128 with and without abs_grad, the same seeded state and
      statistics for both; alternating, host clock around synchronised calls, medians.

The card's name and power limit are printed by the same run.  Development tool:
    python tools/time_absgrad.py
"""
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "feature-3dgs_b200")):
    sys.path.insert(0, p)
import scenegen  # noqa: E402
from diff_gaussian_rasterization import GaussianRasterizationSettings, _C  # noqa: E402
from diff_gaussian_rasterization.parallel import ViewBatch  # noqa: E402
from diff_gaussian_rasterization.trainer import GaussianState  # noqa: E402

ROUNDS, ITERS, DENSIFY_ROUNDS = 7, 5, 5
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


def bench_backward(C, dev):
    sc = scenegen.make_scene(P=1_000_000, W=1920, H=1080, C=max(C, 1), sh_degree=3, views=1, seed=3)
    cam = sc.cameras[0]
    d = scenegen.to_torch(sc, dev)
    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, dev))
    keys = ("means3D", "scales", "rotations", "opacities", "shs") + (("semantic_feature",) if C else ())
    vbs = {a: ViewBatch({k: d[k] for k in keys}, absgrad=a) for a in (False, True)}
    H, W = cam.image_height, cam.image_width
    gc, gf, gd = (torch.from_numpy(a).to(dev) for a in scenegen.upstream_grads(H, W, max(C, 1)))

    def step(a):
        vb = vbs[a]
        *_, ctx = vb.forward(rs)
        vb.backward(ctx, gc, gf if C else None, gd)

    for a in vbs:  # warm-up
        step(a)
    torch.cuda.synchronize()
    t = {a: [] for a in vbs}
    for _ in range(ROUNDS):
        for a in vbs:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(ITERS):
                step(a)
            e1.record()
            torch.cuda.synchronize()
            t[a].append(e0.elapsed_time(e1) / ITERS)
    bwd = {a: [] for a in vbs}
    for _ in range(ROUNDS):
        for a in vbs:
            _C.profile_enable(True)
            _C.profile_read()
            for _ in range(ITERS):
                step(a)
            torch.cuda.synchronize()
            ms, cnt = _C.profile_read()
            _C.profile_enable(False)
            bwd[a].append(ms[STAGE_COMPOSITE_BWD] / max(cnt[STAGE_COMPOSITE_BWD], 1))
    # both arms accumulated the same views: their flat buffers agree up to the order of the float atomics, except for
    # the statistic's slice
    ref = vbs[False].flat
    same = torch.allclose(ref, vbs[True].flat[:ref.numel()], rtol=1e-4, atol=1e-5 * float(ref.abs().max()))
    for a in vbs:
        print(f"C={C} absgrad={a}: backward composite {median(bwd[a]):.3f} ms (profiled rounds); forward + "
              f"ViewBatch.backward {median(t[a]):.3f} ms per view (median of {ROUNDS}x{ITERS}, per-round ms: "
              f"{', '.join(f'{x:.3f}' for x in t[a])})")
    print(f"  extra: backward composite {(median(bwd[True]) / median(bwd[False]) - 1) * 100:+.2f} %, per view "
          f"{(median(t[True]) / median(t[False]) - 1) * 100:+.2f} %; other gradients agree: {same}")
    del vbs
    torch.cuda.empty_cache()


def make_state(P, C, M, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)  # noqa: E731
    st = GaussianState(r(P, 3), r(P, 1, 3), r(P, M - 1, 3), r(P, 1) + 2, r(P, 3) - 4, r(P, 4), r(P, 1, C))
    st.exp_avg = {k: torch.randn(v.shape, device="cuda", generator=g) for k, v in st.raw.items()}
    st.exp_avg_sq = {k: torch.rand(v.shape, device="cuda", generator=g) for k, v in st.raw.items()}
    denom = torch.randint(1, 4, (P,), device="cuda", generator=g).float()
    ga = torch.rand(P, device="cuda", generator=g) * denom * 4e-4
    gaa = ga + torch.rand(P, device="cuda", generator=g) * denom * 8e-4
    return st, ga, gaa, denom


def bench_densify(P=1_000_000, C=128, M=16):
    t = {a: [] for a in (False, True)}
    n = {}
    for i in range(DENSIFY_ROUNDS + 1):
        for a in (False, True):
            st, ga, gaa, dn = make_state(P, C, M, seed=i)
            gen = torch.Generator(device="cuda").manual_seed(i)
            kw = dict(abs_grad=6e-4, grad_accum_abs=gaa) if a else {}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n[a] = st.densify_and_prune(2e-4, 0.005, 3.7, 20, grad_accum=ga, denom=dn, generator=gen, **kw)
            torch.cuda.synchronize()
            if i:  # the first round warms both up
                t[a].append((time.perf_counter() - t0) * 1e3)
            del st, ga, gaa, dn
            torch.cuda.empty_cache()
    for a in (False, True):
        print(f"densify_and_prune P={P} C={C} M={M} abs_grad={'6e-4' if a else 'None'}: {median(t[a]):.2f} ms "
              f"(median of {DENSIFY_ROUNDS}; per-round ms: {', '.join(f'{x:.2f}' for x in t[a])}), P -> {n[a]}")


def main():
    if not torch.cuda.is_available():
        sys.exit("time_absgrad.py needs a CUDA device")
    dev = torch.device("cuda")
    print("card:", card())
    for C in (0, 128):
        bench_backward(C, dev)
    bench_densify()


if __name__ == "__main__":
    main()
