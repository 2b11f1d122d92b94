"""Cost of vector-quantised feature fields (csrc/vq.cu, codebook.py, GaussianState.quantize_features):

  (a) kernels at P = 1 M rows, D in {128, 512}, K in {256, 4096}: assign (f3dgs_vq_assign), plan, update, codebook
      gradient and decode, against the PyTorch restatement: a chunked `x @ c.T` (TF32 allowed) + `argmin` for the
      assignment, `index_add_` + `bincount` for the update, `index_add_` for the gradient and `c[code]` for the decode.
      The two arms alternate over ROUNDS rounds of ITERS calls after a warm-up, timed with CUDA events; medians (min-max).
      The assignment's TFLOP/s count 2 P K D operations (its share of the data-sheet dense TF32 peak, 495 TFLOP/s, is
      printed beside it); the update's and the decode's GB/s count P D + K D floats and 2 P ints (update) and P D + K D
      floats and P ints (decode), from shapes.  The codes of the two assignments are compared.
  (b) one fine-tuning step per view at config 3's cloud and camera (P = 1 M, 1920x1080), C = 128: ViewBatch forward,
      colour and feature losses, backward, all_reduce, Adam, activate, for per-row features against the same state after
      quantize_features(K = 4096); alternating, CUDA events; the memory each state holds between steps and its peak
      during a step, each measured with only that state allocated.
  (c) the PLY file of that state written by io.save_ply with and without the codebook.
The card's name and power limit are printed by the same run.  Development tool:
    python tools/time_vq.py
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "feature-3dgs_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import scenegen  # noqa: E402
from diff_gaussian_rasterization import GaussianRasterizationSettings  # noqa: E402
from diff_gaussian_rasterization import codebook as vq  # noqa: E402
from diff_gaussian_rasterization import feature_head as fh  # noqa: E402
from diff_gaussian_rasterization import io as ply  # noqa: E402
from diff_gaussian_rasterization.trainer import GaussianState, inverse_sigmoid  # noqa: E402

P_ROWS = 1_000_000
SHAPES = [(128, 256), (128, 4096), (512, 256), (512, 4096)]  # (D, K)
ROUNDS, ITERS = 5, 3
TF32_PEAK = 495e12  # H100 SXM data sheet, dense TF32
STEP_K, STEP_C = 4096, 128
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


def torch_assign(x, c, chunk=65536):
    cn = (c * c).sum(1)
    out = torch.empty(x.shape[0], dtype=torch.int64, device=x.device)
    for i in range(0, x.shape[0], chunk):
        out[i:i + chunk] = torch.argmin(cn - 2.0 * (x[i:i + chunk] @ c.T), dim=1)
    return out


def kernels():
    torch.backends.cuda.matmul.allow_tf32 = True
    g = torch.Generator(device="cuda").manual_seed(0)
    print(f"\n(a) kernels at P = {P_ROWS}: median of {ROUNDS} rounds x {ITERS} calls (min-max), ms per call")
    for D, K in SHAPES:
        x = torch.randn(P_ROWS, D, device="cuda", generator=g)
        c = x[torch.randperm(P_ROWS, device="cuda", generator=g)[:K]].contiguous()
        code = vq.assign(x, c)
        code64 = code.long()
        plan = vq.CodePlan(code, K)
        dx = torch.randn(P_ROWS, D, device="cuda", generator=g)
        c_upd = c.clone()

        def torch_update():
            s = torch.zeros(K, D, device="cuda").index_add_(0, code64, x)
            n = torch.bincount(code64, minlength=K).float()[:, None]
            return torch.where(n > 0, s / n, c)

        t = alternate({
            "assign": lambda: vq.assign(x, c), "assign_torch": lambda: torch_assign(x, c),
            "plan": lambda: vq.CodePlan(code, K),
            "update": lambda: plan.update(c_upd.copy_(c), x), "update_torch": torch_update,
            "grad": lambda: plan.grad(dx),
            "grad_torch": lambda: torch.zeros(K, D, device="cuda").index_add_(0, code64, dx),
            "decode": lambda: vq.decode(c, code), "decode_torch": lambda: c[code64],
            "decode_f16": lambda: vq.decode(c, code, torch.float16),
        })
        agree = float((torch_assign(x, c) == code64).float().mean())
        med = {k: v[len(v) // 2] for k, v in t.items()}
        flops = 2.0 * P_ROWS * K * D
        upd_bytes = 4.0 * (P_ROWS * D + K * D + 2 * P_ROWS)
        dec_bytes = 4.0 * (P_ROWS * D + K * D + P_ROWS)
        print(f"D = {D}, K = {K}")
        print(f"  assign   ours {fmt(t['assign'])}  torch {fmt(t['assign_torch'])}  {med['assign_torch'] / med['assign']:5.2f}x"
              f"  | {flops / med['assign'] / 1e9:6.1f} TFLOP/s = {flops / med['assign'] / 1e-3 / TF32_PEAK:5.1%} of the "
              f"data-sheet TF32 peak; torch {flops / med['assign_torch'] / 1e9:6.1f} TFLOP/s; codes agree {agree:.5f}")
        print(f"  plan     ours {fmt(t['plan'])}")
        print(f"  update   ours {fmt(t['update'])}  torch {fmt(t['update_torch'])}  {med['update_torch'] / med['update']:5.2f}x"
              f"  | {upd_bytes / med['update'] / 1e6:7.1f} GB/s")
        print(f"  grad     ours {fmt(t['grad'])}  torch {fmt(t['grad_torch'])}  {med['grad_torch'] / med['grad']:5.2f}x"
              f"  | {upd_bytes / med['grad'] / 1e6:7.1f} GB/s")
        print(f"  decode   ours {fmt(t['decode'])}  torch {fmt(t['decode_torch'])}  {med['decode_torch'] / med['decode']:5.2f}x"
              f"  | {dec_bytes / med['decode'] / 1e6:7.1f} GB/s; float16 out {fmt(t['decode_f16'])}")
        del x, c, code, code64, plan, dx, c_upd
        torch.cuda.empty_cache()


def make_state(sc, t, C):
    M = (sc.sh_degree + 1) ** 2
    shs = t["shs"][:, :M]
    sf = torch.randn(sc.P, 1, C, device="cuda", generator=torch.Generator("cuda").manual_seed(C)) * 0.1
    return GaussianState(t["means3D"].clone(), shs[:, :1].clone(), shs[:, 1:].clone(),
                         inverse_sigmoid(t["opacities"].clamp(1e-4, 1 - 1e-4)), torch.log(t["scales"]),
                         t["rotations"].clone(), sf)


def fine_tuning():
    sc = scenegen.make_config("c3")
    sc.features = np.zeros((sc.P, 1, 0), np.float32)
    cam = sc.cameras[0]
    H, W = cam.image_height, cam.image_width
    t = scenegen.to_torch(sc, "cuda")
    rs = GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, "cuda"))
    gc, _, gd = [torch.from_numpy(a).cuda() for a in scenegen.upstream_grads(H, W, 0, seed=99)]
    Hg, Wg = max(round(H / 2.25), 1), max(round(W / 2.25), 1)  # the teacher resolution of time_half_training.py
    gt = torch.rand(STEP_C, Hg, Wg, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    kinds = {}

    def state_of(kind):
        st = make_state(sc, t, STEP_C)
        if kind == "quantised":
            kinds["report"] = st.quantize_features(STEP_K, iters=10, generator=torch.Generator().manual_seed(0))
        return st

    def step_of(st):
        st.activate()
        vb = st.batch()

        def step():
            vb.zero_()
            color, feat, radii, depth, ctx = vb.forward(rs)
            _, gfeat = fh.feature_l1_loss_and_grad(feat, gt, 1.0)
            vb.backward(ctx, gc, gfeat, gd, last=True)
            vb.all_reduce()
            st.step(LRS)
            st.activate()

        return step

    # memory: one state at a time, above what is allocated without it (the scene and the loss inputs)
    mem = {}
    for k in ("per-row", "quantised"):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        st = state_of(k)
        fn = step_of(st)
        fn()
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        mem[k] = (before - base, torch.cuda.max_memory_allocated() - base)
        del st, fn
        torch.cuda.empty_cache()
    states = {k: state_of(k) for k in ("per-row", "quantised")}
    del t
    rep = kinds["report"]
    steps = {k: step_of(st) for k, st in states.items()}
    t = alternate(steps)
    print(f"\n(b) one fine-tuning step per view, config 3 cloud (P = {sc.P}), {W}x{H}, C = {STEP_C}, K = {STEP_K}: "
          f"median of {ROUNDS} rounds x {ITERS} steps (min-max); memory of one state on its own, above what the scene "
          f"and the loss inputs take")
    print(f"  feature field bytes (quantize_features): before {rep['before'] / 2**20:.1f} MiB, after "
          f"{rep['after'] / 2**20:.1f} MiB")
    for k in steps:
        b, pk = mem[k]
        print(f"  {k:>9}: {fmt(t[k])} ms/step  | held between steps {b / 2**30:6.2f} GiB, peak during it "
              f"{pk / 2**30:6.2f} GiB")
    q = states["quantised"]
    with tempfile.TemporaryDirectory() as d:
        r = q.raw
        common = [r["xyz"], r["f_dc"], r["f_rest"], r["opacity"], r["scaling"], r["rotation"]]
        common = [a.detach().cpu().numpy() for a in common]
        full = os.path.join(d, "full.ply")
        ply.save_ply(full, *common, q.act["semantic_feature"].float().cpu().numpy())
        comp = os.path.join(d, "quantised.ply")
        ply.save_ply(comp, *common, None, semantic_codebook=q.codebook, semantic_code=q.code)
        a, b = os.path.getsize(full), os.path.getsize(comp)
    print(f"\n(c) PLY of that state (P = {q.P}, SH degree {sc.sh_degree}, C = {STEP_C}): per-row features "
          f"{a / 1e6:.1f} MB, codebook K = {STEP_K} + ushort codes {b / 1e6:.1f} MB ({a / b:.2f}x smaller)")


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    print(q.stdout.strip() or f"nvidia-smi unavailable: {q.stderr.strip()}")
    print(f"torch {torch.__version__}, device {torch.cuda.get_device_name()}")
    which = sys.argv[1:] or ["kernels", "step"]
    if "kernels" in which:
        kernels()
    if "step" in which:
        fine_tuning()


if __name__ == "__main__":
    main()
