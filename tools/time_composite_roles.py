"""Who waits in the composite kernels: the share of each warp role's loop spent in each of its mbarrier waits.

Builds the library with -DF3DGS_ROLE_CLOCKS (composite_common.cuh: every producer, alpha and feature warp adds its
clock64() cycles per wait and per loop to a small global array) and its torch binding into a directory of its own
(--build-dir, default a temporary one; the normal build is not touched), renders config 3's cloud and camera
(1 M Gaussians, 1920x1080, C = 128; --config names another scenegen config) forward + backward for a few views through
the public GaussianRasterizer, and prints for composite_fwd and composite_bwd each wait as a share of its role's loop,
summed over all warps of the role and all views.  The clocks perturb what they measure a little (two CS2R per wait); the normal build has none of it.  The card's
name and power limit are read in the same run.  Development tool, fails without a GPU:
    python tools/time_composite_roles.py [--views N] [--config NAME] [--build-dir DIR]

Reading the table: the producer is the limit of a kernel only if its alpha warps spend a large share of their loop
waiting on `full` while the producer hardly waits on `empty`.
"""
import argparse
import ctypes
import glob
import os
import shutil
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "feature-3dgs_b200")
CLOCKS = ("prod_empty", "prod_loop", "alpha_full", "alpha_wempty", "alpha_loop", "feat_wfull", "feat_full",
          "feat_loop")  # enum RoleClock, composite_common.cuh
ROWS = (("producer", "prod_loop", (("empty", "prod_empty"),)),
        ("alpha warps", "alpha_loop", (("full", "alpha_full"), ("wempty", "alpha_wempty"))),
        ("feature warps", "feat_loop", (("wfull", "feat_wfull"), ("full", "feat_full"))))


def build_instrumented(out):
    """The instrumented library, its binding and a copy of the Python package under `out`."""
    sys.path.insert(0, PKG)
    import build as native_build

    native_build.build_all(out=out, defines=["F3DGS_ROLE_CLOCKS"])
    dst = os.path.join(out, "diff_gaussian_rasterization")
    for py in glob.glob(os.path.join(PKG, "diff_gaussian_rasterization", "*.py")):
        shutil.copy(py, dst)
    sys.path.remove(PKG)
    return os.path.join(out, "libf3dgs_b200.so")


def read_clocks(fn, reset=True):
    buf = (ctypes.c_ulonglong * len(CLOCKS))()
    rc = fn(buf, int(reset))
    assert rc == 0, f"reading the role clocks failed: cudaError {rc}"
    return dict(zip(CLOCKS, buf))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=4)
    ap.add_argument("--config", default="c3")
    ap.add_argument("--build-dir", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    print(q.stdout.strip() or f"nvidia-smi unavailable: {q.stderr.strip()}")
    print(f"torch {torch.__version__}, device {torch.cuda.get_device_name()}")

    out = args.build_dir or tempfile.mkdtemp(prefix="f3dgs_roleclocks_")
    lib_path = build_instrumented(os.path.abspath(out))
    sys.path[:0] = [ROOT, os.path.abspath(out)]
    import scenegen
    import diff_gaussian_rasterization as dgr

    assert os.path.abspath(dgr.__file__).startswith(os.path.abspath(out)), dgr.__file__
    lib = ctypes.CDLL(lib_path)  # the library the binding already loaded

    sc = scenegen.make_config(args.config, views=args.views)
    t = scenegen.to_torch(sc, "cuda", requires_grad=True)
    means2D = torch.zeros_like(t["means3D"], requires_grad=True)
    cam0 = sc.cameras[0]
    grads = [torch.from_numpy(g).cuda() for g in scenegen.upstream_grads(cam0.image_height, cam0.image_width, sc.C)]

    def view(cam):
        rast = dgr.GaussianRasterizer(dgr.GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, "cuda")))
        color, feat, _, depth = rast(means3D=t["means3D"], means2D=means2D, opacities=t["opacities"], shs=t["shs"],
                                     semantic_feature=t["semantic_feature"] if sc.C > 0 else None, scales=t["scales"],
                                     rotations=t["rotations"])
        outs, gos = ([color, depth, feat], [grads[0], grads[2], grads[1]]) if sc.C > 0 else ([color, depth],
                                                                                             [grads[0], grads[2]])
        torch.autograd.backward(outs, gos)
        torch.cuda.synchronize()

    view(cam0)  # warm-up: module load, shared-memory opt-in
    for fn in (lib.f3dgs_role_clocks_fwd, lib.f3dgs_role_clocks_bwd):
        read_clocks(fn)
    for cam in sc.cameras:
        view(cam)
    print(f"\nconfig {args.config} cloud (P = {sc.P}), {cam0.image_width}x{cam0.image_height}, C = {sc.C}, "
          f"forward + backward, {len(sc.cameras)} views; cycles summed over the role's warps")
    for name, fn in (("composite_fwd", lib.f3dgs_role_clocks_fwd), ("composite_bwd", lib.f3dgs_role_clocks_bwd)):
        c = read_clocks(fn)
        print(f"{name}")
        for role, loop, waits in ROWS:
            if c[loop] == 0:
                continue
            cells = ", ".join(f"wait on {w}: {100.0 * c[k] / c[loop]:5.1f} %" for w, k in waits)
            print(f"  {role:<14} loop {c[loop] / 1e6:10.1f} Mcycles | {cells}")


if __name__ == "__main__":
    main()
