"""C-ABI surface: the shared library loads without a GPU and exports exactly what include/f3dgs_b200.h
declares; argument validation happens before any CUDA call; the private buffer layout is
self-consistent.  (No compute calls here -- those are the -m gpu parity tests.)"""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "f3dgs_b200.h")


class Layout(ctypes.Structure):
    _fields_ = [(n, ctypes.c_size_t) for n in (
        "geom_bytes", "geom_rec", "geom_cov3d", "geom_clamped", "geom_tiles", "geom_offsets", "geom_radii",
        "img_bytes", "img_final_T", "img_n_contrib", "img_ranges", "bin_bytes", "bin_point_list", "bin_keys")]


@pytest.fixture(scope="module")
def lib(built):
    return ctypes.CDLL(built)


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(f3dgs_[a-z_0-9]+)\s*\(", src)) - {"f3dgs_alloc_fn"})


def test_header_declares_the_reference_interface():
    names = declared_functions()
    for n in ("f3dgs_forward", "f3dgs_backward", "f3dgs_mark_visible", "f3dgs_get_layout", "f3dgs_last_error",
              "f3dgs_abi_version", "f3dgs_launch_count"):
        assert n in names
    text = open(HEADER).read()
    # every entry point cites the reference interface it replaces
    assert "rasterizer.h:31-58" in text and "rasterizer.h:60-93" in text and "rasterizer.h:24-29" in text


def test_library_exports_every_declared_symbol(lib):
    for name in declared_functions():
        assert hasattr(lib, name), f"{name} declared in include/f3dgs_b200.h but not exported"


def test_no_torch_or_python_dependency(built):
    import subprocess

    out = subprocess.run(["ldd", built], capture_output=True, text=True).stdout
    assert "torch" not in out and "python" not in out and "c10" not in out


def test_abi_version_and_launch_counter(lib):
    lib.f3dgs_launch_count.restype = ctypes.c_ulonglong
    assert lib.f3dgs_abi_version() == 2
    assert lib.f3dgs_launch_count() == 0  # nothing launched in a CPU-only process


def test_layout_is_aligned_and_ordered(lib):
    L = Layout()
    assert lib.f3dgs_get_layout(1000, 1920, 1080, 5000, ctypes.byref(L)) == 0
    vals = {n: getattr(L, n) for n, _ in Layout._fields_}
    for n, v in vals.items():
        assert v % 256 == 0, (n, v)
    assert vals["geom_rec"] == 0 and vals["geom_cov3d"] >= 48 * 1000
    assert vals["geom_bytes"] > vals["geom_radii"] >= vals["geom_offsets"] + 4000
    tiles = 120 * 68
    assert vals["img_ranges"] >= vals["img_n_contrib"] + 4 * 1920 * 1080
    assert vals["img_bytes"] >= vals["img_ranges"] + 8 * tiles
    assert vals["bin_keys"] >= vals["bin_point_list"] + 4 * 5000
    assert lib.f3dgs_get_layout(-1, 10, 10, 0, ctypes.byref(L)) == -1


def test_forward_rejects_bad_arguments_before_touching_cuda(lib):
    lib.f3dgs_last_error.restype = ctypes.c_char_p
    CB = ctypes.CFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t)
    cb = CB(lambda ctx, n: None)
    null = ctypes.c_void_p(0)

    def call(P=10, C=4, W=64, H=64, D=3, allocs=True):
        a = cb if allocs else ctypes.cast(null, CB)
        return lib.f3dgs_forward(a, null, a, null, a, null, P, D, 16, C, null, W, H, null, null, null, null, null,
                                 null, ctypes.c_float(1.0), null, null, null, null, null, ctypes.c_float(0.5),
                                 ctypes.c_float(0.5), 0, null, null, null, null, 0, null)

    assert call(P=-1) == -1 and b"bad sizes" in lib.f3dgs_last_error()
    assert call(C=4097) == -1 and b"bad sizes" in lib.f3dgs_last_error()  # F3DGS_MAX_FEATURE_DIM + 1
    assert call(C=4096) == -1 and b"NULL required pointer" in lib.f3dgs_last_error()  # the limit itself passes
    assert call(W=0) == -1
    assert call(D=4) == -1
    assert call(allocs=False) == -1 and b"allocator" in lib.f3dgs_last_error()
    assert call() == -1 and b"NULL required pointer" in lib.f3dgs_last_error()
    assert call(P=0) == 0  # empty cloud: nothing to do (the torch wrapper keeps the reference's zeros)


def test_mark_visible_and_backward_validate(lib):
    null = ctypes.c_void_p(0)
    assert lib.f3dgs_mark_visible(-1, null, null, null, null, null) == -1
    assert lib.f3dgs_mark_visible(0, null, null, null, null, null) == 0
    assert lib.f3dgs_mark_visible(5, null, null, null, null, null) == -1
    args = [5, 3, 16, 0, 4, null, 64, 64] + [null] * 4 + [null, ctypes.c_float(1.0), null, null, null, null, null,
            ctypes.c_float(0.5), ctypes.c_float(0.5), null, null, null, null] + [null] * 14 + [0, null]
    assert lib.f3dgs_backward(*args) == -1


def test_every_entry_point_reports_its_own_error(lib):
    """A rejected call names itself in the last error, also after another entry point failed."""
    lib.f3dgs_last_error.restype = ctypes.c_char_p
    null = ctypes.c_void_p(0)
    one = ctypes.c_float(1.0)
    calls = {
        b"f3dgs_adam_step": lambda: lib.f3dgs_adam_step(99, ctypes.c_size_t(4), 1, null, null, null, null, one, one,
                                                        one, one, 1, null),
        b"f3dgs_activate": lambda: lib.f3dgs_activate(-1, 1, null, null, null, null, null, null, null, null, null, null),
        b"f3dgs_knn_mean_dist": lambda: lib.f3dgs_knn_mean_dist(-1, null, null, null, null),
    }
    for name, call in calls.items():
        for other, fail_first in calls.items():
            if other != name:
                assert fail_first() == -1
                assert call() == -1
                assert lib.f3dgs_last_error().startswith(name + b": "), (name, lib.f3dgs_last_error())
    lib.f3dgs_launch_count.restype = ctypes.c_ulonglong
    assert lib.f3dgs_launch_count() == 0
