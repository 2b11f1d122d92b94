#!/usr/bin/env python
"""In-tree build of the two native artefacts (no torch JIT cache: they live next to the package):

  feature-3dgs_b200/libf3dgs_b200.so           CUDA kernels + C ABI (include/f3dgs_b200.h); nvcc, sm_90a only
  feature-3dgs_b200/diff_gaussian_rasterization/_C*.so   torch/pybind11 binding over the C ABI; g++ only

Usage: python feature-3dgs_b200/build.py [--force]

build_all(out=DIR, defines=[...]) builds a variant (extra -D switches) with the same layout under DIR instead, for tools
that measure an instrumented library next to the normal one.
"""
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")


def _paths(out):
    """(object directory, library, torch extension) of a build under `out`"""
    return (os.path.join(out, "build"), os.path.join(out, "libf3dgs_b200.so"),
            os.path.join(out, "diff_gaussian_rasterization", "_C" + sysconfig.get_config_var("EXT_SUFFIX")))


OBJ, LIB, EXT = _paths(PKG)
CU = ["api.cu", "preprocess.cu", "binning.cu", "composite_fwd.cu", "composite_bwd.cu", "feature_bwd.cu",
      "feature_head.cu", "feature_decoder.cu", "feature_query.cu", "feature_pca.cu", "image_loss.cu", "optimizer.cu",
      "knn.cu", "densify.cu", "mcmc.cu", "filter3d.cu", "vq.cu", "neighbors.cu"]
HDRS = ["common.cuh", "kernels.h", "composite_common.cuh", "tf32_mma.cuh", os.path.join(ROOT, "include", "f3dgs_b200.h")]
NVCC_FLAGS = ["-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v", "--expt-relaxed-constexpr"]


def _run(cmd, log=None):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if log is not None:
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr + "\n")
        raise RuntimeError("build step failed: " + cmd[0])
    return r


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _flags_changed(obj_dir, flags):
    """Objects are only reusable for the flags they were built with."""
    import hashlib

    h = hashlib.sha256(" ".join(flags).encode()).hexdigest()
    stamp = os.path.join(obj_dir, "flags.sha256")
    old = open(stamp).read().strip() if os.path.exists(stamp) else None
    if old != h:
        with open(stamp, "w") as f:
            f.write(h)
        return True
    return False


def build_lib(force=False, out=PKG, defines=()):
    obj_dir, lib, _ = _paths(out)
    flags = NVCC_FLAGS + ["-D" + d for d in defines]
    os.makedirs(obj_dir, exist_ok=True)
    force = _flags_changed(obj_dir, flags) or force
    hdrs = [h if os.path.isabs(h) else os.path.join(CSRC, h) for h in HDRS]
    jobs, objs = [], []
    for cu in CU:
        src, obj = os.path.join(CSRC, cu), os.path.join(obj_dir, cu + ".o")
        objs.append(obj)
        if force or _newer(obj, [src] + hdrs):
            jobs.append((["nvcc", "-c", src, "-o", obj] + flags, os.path.join(obj_dir, cu + ".log")))
    with ThreadPoolExecutor(max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
        list(ex.map(lambda j: _run(*j), jobs))
    if force or jobs or not os.path.exists(lib):
        _run(["nvcc", "-shared", "-o", lib] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"])
    return lib


def build_ext(force=False, out=PKG):
    import torch
    from torch.utils import cpp_extension as ce

    _, lib, ext = _paths(out)
    src = os.path.join(CSRC, "torch_binding.cpp")
    if not (force or _newer(ext, [src, os.path.join(ROOT, "include", "f3dgs_b200.h"), lib])):
        return ext
    os.makedirs(os.path.dirname(ext), exist_ok=True)
    inc = []
    for p in ce.include_paths() + [sysconfig.get_paths()["include"], "/usr/local/cuda/include"]:
        inc += ["-I", p]
    libs = []
    for p in ce.library_paths():
        libs += ["-L", p, f"-Wl,-rpath,{p}"]
    _run(["g++", "-shared", "-fPIC", "-O2", "-std=c++17", src, "-o", ext,
          "-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H",
          f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}"] + inc + libs +
         ["-L", out, "-lf3dgs_b200", "-Wl,-rpath,$ORIGIN/..",
          "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python"])
    return ext


def build_all(force=False, out=PKG, defines=()):
    return build_lib(force, out, defines), build_ext(force, out)


if __name__ == "__main__":
    print(build_all("--force" in sys.argv))
