"""oracle -- CPU checker for the H100 rasterizer.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import
this package; the product (feature-3dgs_b200/) never does.

  oracle.forward(scene, cam)            -> dict of numpy arrays (images + every intermediate the
                                           reference keeps in its geometry/binning/image buffers)
  oracle.backward(scene, cam, fwd, dL_dcolor, dL_dfeature, dL_ddepth) -> dict of gradients
      in the layout the reference's autograd function returns them.

Backed by oracle/f3dgs_oracle.c (plain C restatement of the reference CUDA algorithm, each
function citing the reference file:line), compiled on first use into oracle/libf3dgs_oracle.so.
Parity pin: tests/golden/*.npz were produced by the UNMODIFIED reference extension (oracle/_ref)
via oracle/make_golden.py; tests/test_oracle_golden.py checks this restatement against
them.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "f3dgs_oracle.c")
_LIB = os.path.join(_HERE, "libf3dgs_oracle.so")
_lib = None


def build(force: bool = False) -> str:
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(_SRC):
        subprocess.run(["gcc", "-O2", "-fopenmp", "-ffp-contract=off", "-mfma", "-mavx2", "-shared", "-fPIC",
                        _SRC, "-o", _LIB, "-lm"], check=True)
    return _LIB


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build())
        _lib.oracle_preprocess.restype = ctypes.c_longlong
        _lib.oracle_max_threads.restype = ctypes.c_int
    return _lib


def _p(a):
    if a is None:
        return ctypes.c_void_p(0)
    assert a.flags["C_CONTIGUOUS"]
    return ctypes.c_void_p(a.ctypes.data)


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


def set_threads(n: int):
    lib().oracle_set_threads(ctypes.c_int(n))


def max_threads() -> int:
    return lib().oracle_max_threads()


def forward(scene, cam, colors_precomp=None, cov3D_precomp=None, scale_modifier=1.0, tile_range=None,
            render=True):
    """Reference Rasterizer::forward (rasterizer_impl.cu:198-342) on the CPU."""
    L = lib()
    P, C = scene.P, scene.C
    W, H = cam.image_width, cam.image_height
    gx, gy = (W + 15) // 16, (H + 15) // 16
    means = _f32(scene.means3D)
    use_sh = colors_precomp is None
    shs = _f32(scene.shs) if use_sh else None
    M = scene.shs.shape[1] if use_sh else 0
    scales = None if cov3D_precomp is not None else _f32(scene.scales)
    rots = None if cov3D_precomp is not None else _f32(scene.rotations)
    cov_pre = _f32(cov3D_precomp)
    col_pre = _f32(colors_precomp)
    opac = _f32(scene.opacities).reshape(-1)
    feats = _f32(scene.features).reshape(P, C)
    vm, pm, cp = _f32(cam.viewmatrix).reshape(-1), _f32(cam.projmatrix).reshape(-1), _f32(cam.campos)
    out = dict(
        radii=np.zeros(P, np.int32), means2D=np.zeros((P, 2), np.float32), depths=np.zeros(P, np.float32),
        cov3D=np.zeros((P, 6), np.float32), rgb=np.zeros((P, 3), np.float32),
        conic_opacity=np.zeros((P, 4), np.float32), clamped=np.zeros((P, 3), np.uint8),
        tiles_touched=np.zeros(P, np.uint32))
    R = L.oracle_preprocess(
        P, scene.sh_degree, M, _p(means), _p(scales), ctypes.c_float(scale_modifier), _p(rots), _p(opac), _p(shs),
        _p(cov_pre), _p(col_pre), _p(vm), _p(pm), _p(cp), W, H, ctypes.c_float(cam.tanfovx),
        ctypes.c_float(cam.tanfovy), _p(out["radii"]), _p(out["means2D"]), _p(out["depths"]), _p(out["cov3D"]),
        _p(out["rgb"]), _p(out["conic_opacity"]), _p(out["clamped"]), _p(out["tiles_touched"]))
    out["num_rendered"] = int(R)
    out["keys"] = np.zeros(R, np.uint64)
    out["point_list"] = np.zeros(R, np.uint32)
    out["ranges"] = np.zeros((gx * gy, 2), np.uint32)
    L.oracle_bin(P, ctypes.c_longlong(R), _p(out["radii"]), _p(out["means2D"]), _p(out["depths"]),
                 _p(out["tiles_touched"]), W, H, _p(out["keys"]), _p(out["point_list"]), _p(out["ranges"]))
    colors = col_pre if col_pre is not None else out["rgb"]
    out["colors"] = colors
    if cov_pre is not None:
        out["cov3D"] = cov_pre
    if render:
        out.update(final_T=np.ones((H, W), np.float32), n_contrib=np.zeros((H, W), np.uint32),
                   color=np.zeros((3, H, W), np.float32), feature_map=np.zeros((C, H, W), np.float32),
                   depth=np.zeros((1, H, W), np.float32))
        t0, t1 = tile_range if tile_range is not None else (0, -1)
        L.oracle_render(W, H, C, _p(out["ranges"]), _p(out["point_list"]), _p(out["means2D"]), _p(colors),
                        _p(feats), _p(out["depths"]), _p(out["conic_opacity"]), _p(_f32(scene.bg)),
                        _p(out["final_T"]), _p(out["n_contrib"]), _p(out["color"]), _p(out["feature_map"]),
                        _p(out["depth"]), t0, t1)
    return out


def backward(scene, cam, fwd, dL_dcolor, dL_dfeature, dL_ddepth, colors_precomp=None, cov3D_precomp=None,
             scale_modifier=1.0, tile_range=None):
    """Reference Rasterizer::backward (rasterizer_impl.cu:347-461) on the CPU."""
    L = lib()
    P, C = scene.P, scene.C
    W, H = cam.image_width, cam.image_height
    use_sh = colors_precomp is None
    M = scene.shs.shape[1] if use_sh else 0
    g = dict(
        means2D=np.zeros((P, 3), np.float32), conic=np.zeros((P, 4), np.float32), opacities=np.zeros((P, 1), np.float32),
        colors=np.zeros((P, 3), np.float32), semantic_feature=np.zeros((P, 1, C), np.float32),
        dz=np.zeros((P, 1), np.float32), means3D=np.zeros((P, 3), np.float32), cov3D=np.zeros((P, 6), np.float32),
        sh=np.zeros((P, M, 3), np.float32), scales=np.zeros((P, 3), np.float32), rotations=np.zeros((P, 4), np.float32))
    t0, t1 = tile_range if tile_range is not None else (0, -1)
    L.oracle_render_backward(
        W, H, C, _p(fwd["ranges"]), _p(fwd["point_list"]), _p(_f32(scene.bg)), _p(fwd["means2D"]),
        _p(fwd["conic_opacity"]), _p(fwd["colors"]), _p(fwd["depths"]), _p(fwd["final_T"]), _p(fwd["n_contrib"]),
        _p(_f32(dL_dcolor)), _p(_f32(dL_dfeature)), _p(_f32(dL_ddepth)), _p(g["means2D"]), _p(g["conic"]),
        _p(g["opacities"]), _p(g["colors"]), _p(g["semantic_feature"]), _p(g["dz"]), t0, t1)
    scales = None if cov3D_precomp is not None else _f32(scene.scales)
    rots = None if cov3D_precomp is not None else _f32(scene.rotations)
    shs = _f32(scene.shs) if use_sh else None
    vm, pm, cp = _f32(cam.viewmatrix).reshape(-1), _f32(cam.projmatrix).reshape(-1), _f32(cam.campos)
    L.oracle_preprocess_backward(
        P, scene.sh_degree, M, _p(_f32(scene.means3D)), _p(fwd["radii"]), _p(shs), _p(fwd["clamped"]), _p(scales),
        _p(rots), ctypes.c_float(scale_modifier), _p(_f32(fwd["cov3D"])), _p(vm), _p(pm), _p(cp), W, H,
        ctypes.c_float(cam.tanfovx), ctypes.c_float(cam.tanfovy), _p(g["means2D"]), _p(g["conic"]), _p(g["colors"]),
        _p(g["dz"]), _p(g["means3D"]), _p(g["cov3D"]), _p(g["sh"]), _p(g["scales"]), _p(g["rotations"]))
    return g


def mark_visible(means3D, viewmatrix):
    m = _f32(means3D)
    out = np.zeros(m.shape[0], np.uint8)
    lib().oracle_mark_visible(m.shape[0], _p(m), _p(_f32(viewmatrix).reshape(-1)), _p(out))
    return out.astype(bool)
