"""Per-call time of 3DGS-MCMC's densification step and position noise:

  (a) native: GaussianState.relocate_and_add -> f3dgs_mcmc_plan / _relocate / _add (csrc/mcmc.cu), one host read, and
      GaussianState.inject_noise -> f3dgs_mcmc_inject_noise;
  (b) restatement: the PyTorch tensor code of the official relocate_gs / add_new_gs / noise (tests/ref_mcmc.py).

Workloads: config 3's cloud (P = 1 M, M = 16) with C = 128 and C = 512, with 5 % and 30 % of the Gaussians dead
(opacity <= 0.005); cap_max = 1.05 P, so each call relocates the dead rows and adds 5 %.  The two paths alternate over
ROUNDS rounds after one warm-up call each; the state copy each call consumes is made outside the timed region, and each
call is timed with the host clock around work that ends in torch.cuda.synchronize() (both paths sync the host).  The
noise is timed with CUDA events over NOISE_ITERS back-to-back calls per path.  Bytes are computed from shapes: the
relocation reads each source row and writes its dead row and the source's two moment rows (4 W floats per dead row),
the addition reads 3 P W and writes 3 (P + n) W floats, the plan about 4 P ints and floats; the noise reads 14 and
writes 3 floats per Gaussian.  The card's name and power limit are printed by the same run.  Development tool:
    python tools/time_mcmc.py
"""
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "feature-3dgs_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import ref_mcmc  # noqa: E402
from diff_gaussian_rasterization.trainer import GaussianState  # noqa: E402

ROUNDS, NOISE_ITERS = 6, 20
NAMES = GaussianState.NAMES
MIN_OPACITY, XYZ_LR = 0.005, 1.6e-4


def make_state(P, M, C, dead, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)

    def rn(*shape):
        return torch.randn(*shape, generator=g, device="cuda")

    opacity = rn(P, 1)
    opacity[torch.rand(P, generator=g, device="cuda") < dead] = -8.0
    st = GaussianState(rn(P, 3), rn(P, 1, 3), rn(P, M - 1, 3), opacity, rn(P, 3) - 4.0, rn(P, 4), rn(P, 1, C))
    for k in NAMES:
        st.exp_avg[k] = rn(*st.raw[k].shape)
        st.exp_avg_sq[k] = torch.rand(st.raw[k].shape, generator=g, device="cuda")
    return st


def copy_state(st):
    c = GaussianState(*[st.raw[k].clone() for k in NAMES])
    c.exp_avg = {k: v.clone() for k, v in st.exp_avg.items()}
    c.exp_avg_sq = {k: v.clone() for k, v in st.exp_avg_sq.items()}
    c.steps = dict(st.steps)
    return c


def restatement(st, cap, g):
    # with torch's deterministic algorithms, as the native path draws: otherwise torch's CUDA multinomial is not bitwise
    # reproducible and the outputs could not be compared
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        return ref_mcmc.relocate_and_add(st, cap, MIN_OPACITY, generator=g)
    finally:
        torch.use_deterministic_algorithms(False)


PATHS = [("(a) native", lambda st, cap, g: st.relocate_and_add(cap, MIN_OPACITY, generator=g)),
         ("(b) restatement", restatement)]
NOISE = [("(a) native", lambda st, g: st.inject_noise(XYZ_LR, generator=g)),
         ("(b) restatement", lambda st, g: ref_mcmc.inject_noise(st, XYZ_LR, generator=g))]


def timed_call(fn, base, cap, seed):
    st = copy_state(base)
    g = torch.Generator(device="cuda").manual_seed(seed)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = fn(st, cap, g)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, n, st


def max_raw_diff(a, b):
    """(everything but the relocated opacity / scaling bitwise equal, max |diff| of raw opacity and scaling)"""
    if a.P != b.P:
        return False, float("nan")
    ok = all(torch.equal(getattr(a, d)[k].view(torch.int32), getattr(b, d)[k].view(torch.int32))
             for d in ("raw", "exp_avg", "exp_avg_sq") for k in NAMES if not (d == "raw" and k in ("opacity", "scaling")))
    dx = max(float((a.raw[k] - b.raw[k]).abs().max()) for k in ("opacity", "scaling"))
    return ok, dx


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                       text=True)
    print(q.stdout.strip() or q.stderr.strip())
    P, M = 1_000_000, 16
    rows = []
    for C in (128, 512):
        W = 14 + 3 * (M - 1) + C
        for dead in (0.05, 0.30):
            base = make_state(P, M, C, dead, seed=C + int(100 * dead))
            cap = int(1.05 * P)
            outs = {pname: timed_call(fn, base, cap, seed=1) for pname, fn in PATHS}  # warm-up and comparison
            (_, na, sa), (_, nb, sb) = outs["(a) native"], outs["(b) restatement"]
            bitwise, dx = max_raw_diff(sa, sb)
            del outs, sa, sb
            torch.cuda.empty_cache()
            ts = {p: [] for p, _ in PATHS}
            for r in range(ROUNDS):
                for pname, fn in PATHS:
                    ms, _, st = timed_call(fn, base, cap, seed=r + 2)
                    del st
                    ts[pname].append(ms)
            n_dead, n_add = na
            moved = (n_dead * 4 * W + 3 * P * W + 3 * (P + n_add) * W + 8 * P) * 4
            name = f"P=1M M=16 C={C} dead {int(100 * dead)} %"
            print(f"{name}: (relocated, added) native {na}, restatement {nb}; all but relocated opacity/scaling bitwise "
                  f"equal: {bitwise}, their max |raw diff| {dx:.3g}")
            res = {}
            for pname, _ in PATHS:
                t = sorted(ts[pname])
                med = (t[len(t) // 2 - 1] + t[len(t) // 2]) / 2
                res[pname] = med
                print(f"  relocate_and_add {pname:16s} {med:9.2f} ms (median of {ROUNDS}; min {t[0]:.2f}, max "
                      f"{t[-1]:.2f}), {moved / med / 1e6:.0f} GB/s of {moved / 1e9:.2f} GB")
            rows.append((name, "relocate_and_add", res, moved))
            if dead == 0.05:  # the noise does not depend on the dead share
                nres = {}
                for pname, fn in NOISE:
                    st = copy_state(base)
                    g = torch.Generator(device="cuda").manual_seed(0)
                    fn(st, g)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(NOISE_ITERS):
                        fn(st, g)
                    e1.record()
                    torch.cuda.synchronize()
                    nres[pname] = e0.elapsed_time(e1) / NOISE_ITERS
                    del st
                nmoved = P * 17 * 4
                for pname, ms in nres.items():
                    print(f"  inject_noise     {pname:16s} {ms:9.3f} ms (mean of {NOISE_ITERS}, normals included), "
                          f"{nmoved / ms / 1e6:.0f} GB/s of {nmoved / 1e9:.3f} GB")
                rows.append((f"P=1M M=16 C={C}", "inject_noise", nres, nmoved))
            del base
            torch.cuda.empty_cache()
    print("\n| workload | call | native ms | native GB/s | restatement ms | speed-up |")
    print("|---|---|---|---|---|---|")
    for name, call, res, moved in rows:
        ta, tb = res["(a) native"], res["(b) restatement"]
        print(f"| {name} | {call} | {ta:.3f} | {moved / ta / 1e6:.0f} | {tb:.3f} | {tb / ta:.1f}x |")


if __name__ == "__main__":
    main()
