"""Per-call time and peak memory of densify_and_prune (clone / split / prune with the Adam state carried along):

  (a) native: GaussianState.densify_and_prune -> f3dgs_densify_plan + f3dgs_densify_apply (csrc/densify.cu), one host
      sync;
  (b) restatement: the PyTorch tensor code of the reference (tests/ref_densify.py), the trainer's path before (a).

Workloads: a config-3-like state (P = 1 M, M = 16, C = 128, the LSeg --speedup width) and P = 5 M, C = 64 (SAM
--speedup).  Seeded statistics select about 10 % of the Gaussians for cloning and 5 % for splitting, and about 5 % are
transparent (pruned).  The two paths alternate over ROUNDS rounds after one warm-up call each; the copy of the state
each call consumes is made outside the timed region.  Each call is timed with the host clock around work that ends in
torch.cuda.synchronize() (both paths sync the host).  Reported: median ms, peak growth of max_memory_allocated during
the call, bytes moved (every old row read once, every new row written once: 3 P (59 + C) 4 + 3 P' (59 + C) 4 for
M = 16) over the median time, and a comparison of the outputs of both paths (bitwise except the split children's xyz).
The card's name and power limit are printed by the same run.  Development tool, not product code:
    python tools/time_densify.py
"""
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "feature-3dgs_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import ref_densify  # noqa: E402
from diff_gaussian_rasterization.trainer import GaussianState  # noqa: E402

ROUNDS = 6
NAMES = GaussianState.NAMES
PERCENT_DENSE, EXTENT, MAX_GRAD, MIN_OPACITY = 0.01, 4.0, 2e-4, 0.005


def make_state(P, M, C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)

    def rn(*shape):
        return torch.randn(*shape, generator=g, device="cuda")

    u = torch.rand(P, generator=g, device="cuda")
    sel = u < 0.15
    large = torch.rand(P, generator=g, device="cuda") < 1 / 3  # of the selected: 10 % clone, 5 % split
    dense = PERCENT_DENSE * EXTENT
    scale = torch.where(large, 2.0 * dense, 0.5 * dense)[:, None] * torch.exp(0.1 * torch.randn(P, 3, generator=g, device="cuda"))
    opacity = rn(P, 1)
    opacity[torch.rand(P, generator=g, device="cuda") < 0.05] = -8.0  # sigmoid < min_opacity
    st = GaussianState(rn(P, 3), rn(P, 1, 3), rn(P, M - 1, 3), opacity, torch.log(scale), rn(P, 4), rn(P, 1, C),
                       percent_dense=PERCENT_DENSE)
    for k in NAMES:
        st.exp_avg[k] = rn(*st.raw[k].shape)
        st.exp_avg_sq[k] = torch.rand(st.raw[k].shape, generator=g, device="cuda")
    denom = torch.ones(P, device="cuda")
    grad_accum = torch.where(sel, 2 * MAX_GRAD, 0.5 * MAX_GRAD).float()
    return st, grad_accum, denom


def copy_state(st):
    c = GaussianState(*[st.raw[k].clone() for k in NAMES], percent_dense=st.percent_dense)
    c.exp_avg = {k: v.clone() for k, v in st.exp_avg.items()}
    c.exp_avg_sq = {k: v.clone() for k, v in st.exp_avg_sq.items()}
    c.steps = dict(st.steps)
    return c


def native(st, ga, dn, gen, info):
    return st.densify_and_prune(MAX_GRAD, MIN_OPACITY, EXTENT, None, grad_accum=ga, denom=dn, generator=gen)


def restatement(st, ga, dn, gen, info):
    return ref_densify.densify_and_prune(st, MAX_GRAD, MIN_OPACITY, EXTENT, None, grad_accum=ga, denom=dn,
                                         generator=gen, info=info)


def timed_call(fn, base, ga, dn, seed):
    st = copy_state(base)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    info = {}
    torch.cuda.synchronize()
    a0 = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    n = fn(st, ga, dn, gen, info)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    return ms, torch.cuda.max_memory_allocated() - a0, n, st, info


def compare(a, b, info):
    """-> (all non-child-xyz tensors bitwise equal, max |diff| of the children's xyz)"""
    if a.P != b.P:
        return False, float("nan")
    nk = int(info["child_keep"].sum())
    ok = True
    for d in ("raw", "exp_avg", "exp_avg_sq"):
        for k in NAMES:
            x, y = getattr(a, d)[k], getattr(b, d)[k]
            if d == "raw" and k == "xyz":
                ok &= torch.equal(x[:a.P - nk].view(torch.int32), y[:b.P - nk].view(torch.int32))
            else:
                ok &= torch.equal(x.view(torch.int32), y.view(torch.int32))
    dx = float((a.raw["xyz"][a.P - nk:] - b.raw["xyz"][b.P - nk:]).abs().max()) if nk else 0.0
    return bool(ok), dx


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                       text=True)
    print(q.stdout.strip() or q.stderr.strip())
    workloads = [("config-3-like P=1M M=16 C=128", 1_000_000, 16, 128), ("P=5M M=16 C=64", 5_000_000, 16, 64)]
    paths = [("(a) native", native), ("(b) restatement", restatement)]
    rows = []
    for name, P, M, C in workloads:
        base, ga, dn = make_state(P, M, C, seed=P + C)
        W = 14 + 3 * (M - 1) + C
        outs = {}
        for pname, fn in paths:  # warm-up, and the outputs for the comparison
            _, _, n, st, info = timed_call(fn, base, ga, dn, seed=1)
            outs[pname] = (st, info)
        (sa, _), (sb, info) = outs["(a) native"], outs["(b) restatement"]
        bitwise, dx = compare(sa, sb, info)
        Pn = sa.P
        del outs, sa, sb, info, st
        torch.cuda.empty_cache()
        print(f"{name}: P' = {Pn}; native vs restatement: bitwise equal except split-child xyz: {bitwise}, "
              f"split-child xyz max |diff| {dx:.3g}")
        ts = {p: [] for p, _ in paths}
        peak = {p: 0 for p, _ in paths}
        for r in range(ROUNDS):
            for pname, fn in paths:
                ms, grow, n, st, _ = timed_call(fn, base, ga, dn, seed=r + 2)
                del st
                ts[pname].append(ms)
                peak[pname] = max(peak[pname], grow)
        moved = (3 * P * W + 3 * Pn * W) * 4
        res = {}
        for pname, _ in paths:
            t = sorted(ts[pname])
            med = (t[len(t) // 2 - 1] + t[len(t) // 2]) / 2
            res[pname] = (med, peak[pname])
            print(f"  {pname:16s} {med:9.2f} ms/call (median of {ROUNDS}; min {t[0]:.2f}, max {t[-1]:.2f}), peak growth "
                  f"{peak[pname] / 2**30:.2f} GiB, {moved / med / 1e6:.0f} GB/s of {moved / 1e9:.2f} GB moved")
        rows.append((name, res, moved, 3 * P * W * 4, bitwise))
        del base, ga, dn
        torch.cuda.empty_cache()
    print("\n| workload | state GB | native ms | native GB/s | native peak growth GiB | restatement ms "
          "| restatement peak growth GiB | bitwise |")
    print("|---|---|---|---|---|---|---|---|")
    for name, res, moved, state, bitwise in rows:
        (ta, pa), (tb, pb) = res["(a) native"], res["(b) restatement"]
        print(f"| {name} | {state / 1e9:.2f} | {ta:.2f} | {moved / ta / 1e6:.0f} | {pa / 2**30:.2f} | {tb:.2f} | "
              f"{pb / 2**30:.2f} | {bitwise} |")


if __name__ == "__main__":
    main()
