"""Per-call time and peak memory of a text query of a feature field, two ways, in one process:

  (a) PyTorch composition: F.conv2d (the 1x1 decoder, default cuDNN settings: TF32 allowed) -> F.normalize -> matmul
      with the normalised text (default matmul precision) -> argmax / softmax summed over the positive prompts.
  (b) feature_head.query: one prep for W, b and the text, then one fused kernel (csrc/feature_query.cu).

Workloads: a 1080x1920 view decoded 128 -> 512 (LSeg --speedup) with K = 2 and K = 150 prompts (labels + prob); a saved
float16 512-channel map without a decoder, K = 150 (labels); per-Gaussian scoring of P = 1M features 128 -> 512, K = 2
(prob + logits).  Both arms are warmed up on every shape, then timed with CUDA events in alternating rounds (median of
ROUNDS rounds of ITERS calls).  Peak memory is the growth of torch.cuda.max_memory_allocated plus the high watermark of
the default stream-ordered pool (the fused call's scratch).  FLOPs: 2 (D C + D K) per column (2 D K without a decoder);
the rate is printed against the H100 SXM data-sheet 495 TFLOP/s dense TF32.  Label agreement is measured on the timed
inputs.  Development tool, not product code:
    python tools/time_feature_query.py
"""
import ctypes
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "feature-3dgs_b200"))
from diff_gaussian_rasterization.feature_head import query  # noqa: E402

ROUNDS, ITERS, WARMUP = 5, 4, 2
PEAK_TFLOPS = 495.0
HW = (1080, 1920)
# name, C, D (None: no decoder, D = C), K, spatial shape, x dtype, outputs (labels, prob, logits)
WORKLOADS = [
    ("view 128->512, K=2", 128, 512, 2, HW, torch.float32, (True, True, False)),
    ("view 128->512, K=150", 128, 512, 150, HW, torch.float32, (True, True, False)),
    ("saved fp16 map 512, K=150", 512, None, 150, HW, torch.float16, (True, False, False)),
    ("per-Gaussian P=1M 128->512, K=2", 128, 512, 2, (1 << 20,), torch.float32, (False, True, True)),
]


def composition(x, W, b, T, scale, pos, want):
    C = x.shape[0]
    xs = x.float().reshape(1, C, -1, 1)
    y = xs[0, :, :, 0] if W is None else F.conv2d(xs, W, b)[0, :, :, 0]
    lg = scale * (F.normalize(T, dim=1) @ F.normalize(y, dim=0))
    lab = lg.argmax(0) if want[0] else None
    prob = lg.softmax(0)[pos].sum(0) if want[1] else None
    return lab, prob, lg if want[2] else None


def fused(x, W, b, T, scale, pos, want):
    lab, prob, lg = query(x, T, W, b, scale, positive=pos if want[1] else None, logits=want[2])
    return lab.view(-1) if want[0] else None, None if prob is None else prob.view(-1), lg


def time_calls(fn, args, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn(*args)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def pool_used_high(reset):
    cu = ctypes.CDLL("libcuda.so.1")
    dev, pool, v = ctypes.c_int(), ctypes.c_void_p(), ctypes.c_uint64(0)
    cu.cuDeviceGet(ctypes.byref(dev), torch.cuda.current_device())
    cu.cuDeviceGetDefaultMemPool(ctypes.byref(pool), dev)
    if reset:
        cu.cuMemPoolSetAttribute(pool, 8, ctypes.byref(v))  # CU_MEMPOOL_ATTR_USED_MEM_HIGH
    cu.cuMemPoolGetAttribute(pool, 8, ctypes.byref(v))
    return v.value


def peak_growth(fn, args):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    pool_used_high(True)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn(*args)
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base + pool_used_high(False)


def main():
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                       text=True)
    print(q.stdout.strip() or q.stderr.strip())
    print("torch", torch.__version__, " cudnn.allow_tf32 =", torch.backends.cudnn.allow_tf32,
          " matmul.allow_tf32 =", torch.backends.cuda.matmul.allow_tf32)
    gen = torch.Generator(device="cuda").manual_seed(0)
    scale = 10.0
    for name, C, D, K, shape, dt, want in WORKLOADS:
        N = 1
        for s in shape:
            N *= s
        x = torch.randn(C, *shape, device="cuda", generator=gen).to(dt)
        Dd = C if D is None else D
        W = None if D is None else torch.randn(D, C, 1, 1, device="cuda", generator=gen) / C ** 0.5
        b = None if D is None else 0.1 * torch.randn(D, device="cuda", generator=gen)
        T = torch.randn(K, Dd, device="cuda", generator=gen)
        pos = [0]
        args = (x, W, b, T, scale, pos, want)
        (la, pa, ga), ma = peak_growth(composition, args)
        (lb, pb, gb), mb = peak_growth(fused, args)
        agree = "n/a (labels not requested)"
        if want[0]:
            agree = f"{float((la == lb).double().mean()) * 100:.4f}% of {N} labels equal"
        diffs = []
        if want[1]:
            diffs.append(f"max|prob diff| {float((pa - pb).abs().max()):.2e}")
        if want[2]:
            diffs.append(f"max|logit diff| {float((ga - gb.view_as(ga)).abs().max()):.2e}")
        del la, pa, ga, lb, pb, gb
        for fn in (composition, fused):
            time_calls(fn, args, WARMUP)
        ta, tb = [], []
        for _ in range(ROUNDS):
            ta.append(time_calls(composition, args, ITERS))
            tb.append(time_calls(fused, args, ITERS))
        flops = 2 * (Dd * K + (0 if D is None else D * C)) * N
        print(f"{name}: N = {N}, C = {C}, D = {Dd}, K = {K}, x {str(dt).replace('torch.', '')}; {agree}; "
              + "; ".join(diffs))
        for label, ts, mem in (("(a) pytorch", ta, ma), ("(b) fused  ", tb, mb)):
            ts = sorted(ts)
            med = ts[len(ts) // 2]
            tfl = flops / (med * 1e-3) / 1e12
            print(f"  {label} {med:8.3f} ms/call (median of {ROUNDS} x {ITERS}; min {ts[0]:.3f}, max {ts[-1]:.3f})  "
                  f"{flops / 1e9:.0f} GFLOP -> {tfl:6.1f} TFLOP/s = {100 * tfl / PEAK_TFLOPS:5.1f}% of 495;  "
                  f"peak memory growth {mem / 2 ** 20:9.1f} MiB")
        print(f"  speed-up (a)/(b): {sorted(ta)[ROUNDS // 2] / sorted(tb)[ROUNDS // 2]:.2f}x")
        del x, W, b, T
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
