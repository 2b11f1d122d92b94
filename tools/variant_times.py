"""Time (and cross-check) several builds of libf3dgs_b200.so in ONE process through the C ABI.

    python tools/variant_times.py <config> <iters> base u1f0 timing ...

`base` is feature-3dgs_b200/libf3dgs_b200.so, any other name is feature-3dgs_b200/variants/<name>/libf3dgs_b200.so
(tools/build_variants.sh); `<name>+split` runs the same library in the two-pass mode (F3DGS_SPLIT=1, composite_split.cu) from a
private copy of the file, so that fused and two-pass results are compared in one process.  torch is only the device allocator / stream here; every library is dlopen'ed RTLD_LOCAL and
driven through include/f3dgs_b200.h (f3dgs_forward / f3dgs_backward / f3dgs_profile_*), so one import and one scene
serve all variants (a variant costs ~1 s instead of a fresh python process).  Prints per-stage mean milliseconds and the
largest difference of every output / gradient against the first variant.  Variants whose name starts with `timing` run
with F3DGS_TIMING=1 (per-role cycle counters on stderr, timing builds only).  Development tool, not product code.
"""
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import scenegen  # noqa: E402

STAGES = ["pre_fwd", "scan", "dup", "sort", "ranges", "comp_fwd", "comp_bwd", "pre_bwd"]
ALLOC = ctypes.CFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t)


def lib_path(name):
    pkg = os.path.join(ROOT, "feature-3dgs_b200")
    return os.path.join(pkg, "libf3dgs_b200.so") if name == "base" else os.path.join(pkg, "variants", name,
                                                                                      "libf3dgs_b200.so")


def ptr(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None and t.numel() else 0)


class Variant:
    def __init__(self, name):
        self.name = name
        path = lib_path(name.split("+")[0])
        if "+" in name:  # a distinct file = a distinct dlopen handle with its own cached settings
            import shutil
            import tempfile

            d = tempfile.mkdtemp(prefix="f3dgs_variant_")
            path = shutil.copy(path, os.path.join(d, "libf3dgs_b200.so"))
        self.lib = ctypes.CDLL(path, mode=os.RTLD_LOCAL)
        self.lib.f3dgs_last_error.restype = ctypes.c_char_p
        self.lib.f3dgs_forward.restype = ctypes.c_int
        self.lib.f3dgs_backward.restype = ctypes.c_int
        self.bufs = {}

    def _alloc(self, key):
        def cb(_ctx, nbytes):
            self.bufs[key] = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device="cuda")
            return self.bufs[key].data_ptr()

        return ALLOC(cb)

    def check(self, rc, what):
        if rc < 0:
            raise RuntimeError(f"{self.name}: {what} failed ({rc}): {self.lib.f3dgs_last_error().decode()}")
        return rc

    def forward(self, sc, cam, t, out):
        P, C, H, W = sc.P, sc.C, cam.image_height, cam.image_width
        M = t["shs"].shape[1]
        cbs = [self._alloc(k) for k in ("geom", "bin", "img")]
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        null = ctypes.c_void_p(0)
        R = self.lib.f3dgs_forward(
            cbs[0], null, cbs[1], null, cbs[2], null, P, sc.sh_degree, M, C, ptr(t["bg"]), W, H, ptr(t["means3D"]),
            ptr(t["shs"]), null, ptr(t["semantic_feature"]) if C else null, ptr(t["opacities"]), ptr(t["scales"]),
            ctypes.c_float(1.0), ptr(t["rotations"]), null, ptr(t["viewmatrix"]), ptr(t["projmatrix"]),
            ptr(t["campos"]), ctypes.c_float(cam.tanfovx), ctypes.c_float(cam.tanfovy), 0, ptr(out["color"]),
            ptr(out["feature"]) if C else null, ptr(out["depth"]), ptr(out["radii"]), 0, stream)
        return self.check(R, "f3dgs_forward")

    def backward(self, sc, cam, t, out, R, up, g):
        P, C, H, W = sc.P, sc.C, cam.image_height, cam.image_width
        M = t["shs"].shape[1]
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        null = ctypes.c_void_p(0)
        rc = self.lib.f3dgs_backward(
            P, sc.sh_degree, M, R, C, ptr(t["bg"]), W, H, ptr(t["means3D"]), ptr(t["shs"]), null,
            ptr(t["semantic_feature"]) if C else null, ptr(t["scales"]), ctypes.c_float(1.0), ptr(t["rotations"]), null,
            ptr(t["viewmatrix"]), ptr(t["projmatrix"]), ptr(t["campos"]), ctypes.c_float(cam.tanfovx),
            ctypes.c_float(cam.tanfovy), ptr(out["radii"]), ptr(self.bufs["geom"]), ptr(self.bufs["bin"]),
            ptr(self.bufs["img"]), ptr(up[0]), ptr(up[1]) if C else null, ptr(up[2]), ptr(g["mean2D"]), ptr(g["conic"]),
            ptr(g["opacity"]), ptr(g["color"]), ptr(g["feature"]) if C else null, ptr(g["mean3D"]), ptr(g["cov3D"]),
            ptr(g["sh"]), ptr(g["scale"]), ptr(g["rot"]), ptr(g["z"]), 0, stream)
        return self.check(rc, "f3dgs_backward")

    def profile(self, on=None):
        if on is not None:
            self.lib.f3dgs_profile_enable(1 if on else 0)
            return None
        ms = (ctypes.c_double * 8)()
        cnt = (ctypes.c_ulonglong * 8)()
        self.check(self.lib.f3dgs_profile_read(ms, cnt), "profile_read")
        return {n: round(ms[i] / max(cnt[i], 1), 4) for i, n in enumerate(STAGES)}


def main():
    cfg = sys.argv[1] if len(sys.argv) > 1 else "c3"
    iters = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    names = sys.argv[3:] or ["base"]
    sc = scenegen.make_config(cfg)
    cam = sc.cameras[0]
    P, C, H, W = sc.P, sc.C, cam.image_height, cam.image_width
    dev = "cuda"
    t = scenegen.to_torch(sc, dev, requires_grad=False)
    t["semantic_feature"] = t["semantic_feature"].reshape(P, C).contiguous() if C else None
    t["opacities"] = t["opacities"].reshape(P).contiguous()
    for k, v in (("viewmatrix", cam.viewmatrix), ("projmatrix", cam.projmatrix), ("campos", cam.campos)):
        t[k] = torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32).reshape(-1)).to(dev)
    up = [torch.from_numpy(x).to(dev).contiguous() for x in scenegen.upstream_grads(H, W, C)]  # colour, feature, depth
    up = [up[0], up[1], up[2]]
    M = t["shs"].shape[1]
    gshape = dict(mean2D=(P, 3), conic=(P, 4), opacity=(P,), color=(P, 3), feature=(P, max(C, 1)), mean3D=(P, 3),
                  cov3D=(P, 6), sh=(P, M, 3), scale=(P, 3), rot=(P, 4), z=(P,))
    ref = None
    report = {}
    for name in names:
        os.environ.pop("F3DGS_TIMING", None)
        os.environ.pop("F3DGS_SPLIT", None)
        os.environ.pop("F3DGS_TC", None)
        if name.endswith("+tc"):
            os.environ["F3DGS_TC"] = "1"  # tensor-core feature contraction (read once per library instance)
        if "+notc" in name:
            os.environ["F3DGS_TC"] = "0"
        os.environ.pop("F3DGS_BWD2", None)
        if "+bwd1" in name:
            os.environ["F3DGS_BWD2"] = "0"  # fused single-kernel backward
        if name.startswith("timing"):
            os.environ["F3DGS_TIMING"] = "1"
        v = Variant(name)
        out = dict(color=torch.empty(3, H, W, device=dev), feature=torch.empty(max(C, 1), H, W, device=dev),
                   depth=torch.empty(1, H, W, device=dev), radii=torch.empty(P, dtype=torch.int32, device=dev))
        g = None
        for it in range(iters + 2):
            if it == 2:
                torch.cuda.synchronize()
                v.profile(True)
            g = {k: torch.zeros(s, device=dev) for k, s in gshape.items()}
            R = v.forward(sc, cam, t, out)
            v.backward(sc, cam, t, out, R, up, g)
        torch.cuda.synchronize()
        ms = v.profile()
        v.profile(False)
        res = {k: x.clone() for k, x in out.items()}
        res.update({"g_" + k: x for k, x in g.items() if k not in ("conic", "z")})
        line = {"variant": name, "R": R, "ms": ms}
        if ref is None:
            ref = res
        else:
            diff = {}
            for k, x in res.items():
                a, b = x.float(), ref[k].float()
                scale = float(b.abs().max()) or 1.0
                diff[k] = float((a - b).abs().max()) / scale
            line["max_diff_vs_" + names[0]] = {k: (0 if d == 0 else float(f"{d:.2e}")) for k, d in diff.items()}
        report[name] = line
        print(json.dumps(line), flush=True)
    return report


if __name__ == "__main__":
    main()
