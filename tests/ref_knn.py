"""The reference's UNMODIFIED simple_knn extension (submodules/simple-knn: ext.cpp, spatial.cu, simple_knn.cu), built for
sm_90a from the sources where they lie in a reference checkout (the one oracle/build_ref.py uses) into oracle/_ref/
(git-ignored), and loaded as a module.  Test and timing infrastructure only: nothing on the product path imports it.

Two flags stand in for edits, as in oracle/build_ref.py: `-include cstdint` and `-include cfloat` (newer host compilers
no longer pull those headers in transitively)."""
import importlib.util
import os
import subprocess
import sys
import sysconfig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import build_ref  # noqa: E402

SRC = os.path.join(os.path.dirname(build_ref.REF), "simple-knn")  # REF is <checkout>/submodules/diff-gaussian-...
OUT = os.path.join(ROOT, "oracle", "_ref")
NAME = "ref_simple_knn"
TARGET = os.path.join(OUT, NAME + ".so")
_mod = None


def reference_present() -> bool:
    return os.path.isfile(os.path.join(SRC, "simple_knn.cu"))


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(" ".join(cmd) + "\n" + r.stdout + r.stderr)


def build() -> str:
    if os.path.exists(TARGET):
        return TARGET
    import torch
    from torch.utils import cpp_extension as ce

    bdir = os.path.join(OUT, "obj_simple_knn")
    os.makedirs(bdir, exist_ok=True)
    inc = []
    for p in ce.include_paths() + [sysconfig.get_paths()["include"], SRC]:
        inc += ["-I", p]
    common = [f"-DTORCH_EXTENSION_NAME={NAME}", "-DTORCH_API_INCLUDE_EXTENSION_H",
              f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}", "-include", "cstdint",
              "-include", "cfloat"] + inc
    objs = []
    for s in ("spatial.cu", "simple_knn.cu", "ext.cpp"):
        o = os.path.join(bdir, s + ".o")
        objs.append(o)
        if s.endswith(".cu"):
            _run(["nvcc", "-c", os.path.join(SRC, s), "-o", o, "-std=c++17", "-O3", "-gencode",
                  "arch=compute_90a,code=sm_90a", "-w", "-Xcompiler", "-fPIC"] + common)
        else:
            _run(["g++", "-c", os.path.join(SRC, s), "-o", o, "-std=c++17", "-O2", "-fPIC", "-w"] + common)
    libs = []
    for p in ce.library_paths():
        libs += ["-L", p, f"-Wl,-rpath,{p}"]
    tmp = TARGET + ".tmp"
    _run(["g++", "-shared", "-o", tmp] + objs + libs + ["-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch",
                                                       "-ltorch_python", "-L/usr/local/cuda/lib64", "-lcudart"])
    os.replace(tmp, TARGET)
    return TARGET


def load():
    """-> the reference module (with .distCUDA2), or None when there is no reference checkout and no prior build."""
    global _mod
    if _mod is None:
        if not os.path.exists(TARGET):
            if not reference_present():
                return None
            build()
        import torch  # noqa: F401  (the extension links against torch's libraries)

        spec = importlib.util.spec_from_file_location(NAME, TARGET)
        _mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(_mod)
    return _mod
