"""The argument checks of the rasterizer's forward and backward C entries, one fault at a time.

Each entry is called through ctypes with fake device addresses and allocators that return NULL.  A call with exactly one
fault must return -1 (F3DGS_ERR_INVALID_ARGUMENT) before any CUDA call, with the exact last error
"<entry>: <message>".  An otherwise well-formed call with P == 0 is a no-op that returns 0.  The parameter lists are
read from include/f3dgs_b200.h, so the arguments are named, not positional.  CPU only.
"""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32, F16 = 0, 1  # F3DGS_F32, F3DGS_F16
MAX_C = 4096  # F3DGS_MAX_FEATURE_DIM
P, C, W, H = 5, 4, 64, 64

FORWARD = ["f3dgs_forward", "f3dgs_forward_f16", "f3dgs_forward_antialiased", "f3dgs_forward_alpha_invdepth"]
BACKWARD = [f"f3dgs_backward{a}{v}" for a in ("", "_accum") for v in ("", "_f16", "_cam", "_cam_f16",
                                                                     "_feature_geometry", "_antialiased",
                                                                     "_alpha_invdepth")]
ENTRIES = FORWARD + BACKWARD

ALLOC_FN = ctypes.CFUNCTYPE(ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t)
NULL_ALLOC = ALLOC_FN(lambda ctx, nbytes: None)  # a check that did not fire reaches an allocator: it fails, no crash


def _signatures():
    """{entry: [(name, kind)]} with kind 'p' (pointer), 'i' (int) or 'f' (float), from the public header."""
    with open(os.path.join(ROOT, "include", "f3dgs_b200.h")) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    sigs = {}
    for name, params in re.findall(r"\bint (f3dgs_\w+)\(([^)]*)\);", text):
        if name not in ENTRIES:
            continue
        out = []
        for p in params.split(","):
            toks = p.replace("*", " * ").split()
            kind = "p" if "*" in toks or toks[0] == "f3dgs_alloc_fn" else "f" if toks[-2] == "float" else "i"
            out.append((toks[-1], kind))
        sigs[name] = out
    return sigs


SIGS = _signatures()
NAMES = sorted({n for e in ENTRIES for n, k in SIGS[e] if k == "p"})
ADDR = {n: (1 << 40) + i * (1 << 20) for i, n in enumerate(NAMES)}  # distinct, 1 MiB apart: nothing overlaps
# the precomputed inputs and their gradients, in the second half of another pointer's slot
COLOURS, COV, DCOL, DCOV = (ADDR[n] + (1 << 19) for n in ("shs", "scales", "dL_dsh", "dL_dscale"))
INTS = dict(P=P, D=0, M=1, R=10, C=C, width=W, height=H, prefiltered=0, debug=0, antialiasing=0,
            semantic_feature_dtype=F32, dL_dfeaturepix_dtype=F32)
FLOATS = dict(scale_modifier=1.0, tan_fovx=0.5, tan_fovy=0.5, dL_dfeaturepix_scale=1.0)
# absent by default: colours and cov3D come from shs and scales / rotations; no precomputed-input gradients, no event
# or stream.  Every other pointer is given, dL_dcamera, the planes and their gradients included.
ABSENT = {"colors_precomp", "cov3D_precomp", "dL_dcolors_precomp", "dL_dcov3D_precomp", "composite_done_event",
          "cuda_stream"}

BAD_FWD = "bad sizes (P, width, height, C or D)"
SCALE = "dL_dfeaturepix_scale must be finite and nonzero"
GO_WITH = "dL_dcolors_precomp / dL_dcov3D_precomp go with colors_precomp / cov3D_precomp"


@pytest.fixture(scope="module")
def lib(built):
    L = ctypes.CDLL(built)
    L.f3dgs_last_error.restype = ctypes.c_char_p
    L.f3dgs_backward_scratch_bytes.restype = ctypes.c_size_t
    return L


def _call(lib, entry, **kw):
    """entry(defaults, with kw by parameter name; None is NULL) -> (return code, last error)"""
    assert not set(kw) - {n for n, _ in SIGS[entry]}, (entry, kw)
    args = []
    for name, kind in SIGS[entry]:
        if kind == "p":
            v = kw[name] if name in kw else (None if name in ABSENT else ADDR[name])
            args.append(NULL_ALLOC if name.endswith("_alloc") and v == ADDR[name] else ctypes.c_void_p(v))
        elif kind == "f":
            args.append(ctypes.c_float(kw.get(name, FLOATS[name])))
        else:
            args.append(ctypes.c_int(kw.get(name, INTS[name])))
    rc = getattr(lib, entry)(*args)
    return rc, lib.f3dgs_last_error().decode()


def _has(entry, name):
    return any(n == name for n, _ in SIGS[entry])


def _forward_faults(entry):
    faults = [(dict(P=-1), BAD_FWD), (dict(width=0), BAD_FWD), (dict(height=0), BAD_FWD), (dict(C=-1), BAD_FWD),
              (dict(C=MAX_C + 1), BAD_FWD), (dict(D=-1), BAD_FWD), (dict(D=4), BAD_FWD)]
    faults += [({a: None}, "missing allocator") for a in ("geometry_alloc", "binning_alloc", "image_alloc")]
    faults += [({p: None}, "NULL required pointer") for p in ("means3D", "opacities", "background", "viewmatrix",
                                                              "projmatrix", "cam_pos", "out_color", "out_depth")]
    one_colour = "provide exactly one of shs / colors_precomp"
    faults += [(dict(shs=None), one_colour), (dict(colors_precomp=COLOURS), one_colour)]
    one_cov = "provide exactly one of (scales, rotations) / cov3D_precomp"
    faults += [(dict(scales=None), one_cov), (dict(rotations=None), one_cov),
               (dict(cov3D_precomp=COV), one_cov)]
    faults += [({p: None}, "C > 0 needs semantic_feature and out_feature_map")
               for p in ("semantic_feature", "out_feature_map")]
    faults += [(dict(D=1), "M < (D+1)^2 SH coefficients")]
    if _has(entry, "semantic_feature_dtype"):
        faults += [(dict(semantic_feature_dtype=t), "unknown dtype code") for t in (-1, 2)]
        faults += [(dict(semantic_feature_dtype=2, P=0), "unknown dtype code")]
    if _has(entry, "out_alpha"):
        faults += [({p: None}, "NULL out_alpha / out_invdepth") for p in ("out_alpha", "out_invdepth")]
        faults += [(dict(out_alpha=None, P=0), "NULL out_alpha / out_invdepth")]
        planes = "out_alpha / out_invdepth overlap another output"
        for aa in (0, 1):
            for o in ("out_color", "out_feature_map", "out_depth", "radii", "out_invdepth"):
                faults.append((dict(out_alpha=ADDR[o], antialiasing=aa), planes))
                faults.append((dict(out_invdepth=ADDR[o] if o != "out_invdepth" else ADDR["out_alpha"],
                                    antialiasing=aa), planes))
        # the last element of the feature map, at each element type
        for t, size in ((F32, 4), (F16, 2)):
            faults.append((dict(out_alpha=ADDR["out_feature_map"] + C * W * H * size - 4, semantic_feature_dtype=t),
                           planes))
            faults.append((dict(out_invdepth=ADDR["out_feature_map"] + C * W * H * size - 4,
                                semantic_feature_dtype=t), planes))
    return faults


def _outputs(entry, **kw):
    """The outputs of a backward call with arguments kw (defaults otherwise): [(name, address)]"""
    if "_accum" in entry:
        names = ["scratch", "dL_dopacity", "dL_dcolors_precomp", "dL_dsemantic_feature", "dL_dmean3D",
                 "dL_dcov3D_precomp", "dL_dsh", "dL_dscale", "dL_drot", "dL_dmean2D_out", "grad_accum", "denom"]
    else:
        names = ["dL_dmean2D", "dL_dconic", "dL_dopacity", "dL_dcolor", "dL_dsemantic_feature", "dL_dmean3D",
                 "dL_dcov3D", "dL_dsh", "dL_dscale", "dL_drot", "dL_dz"]
    if _has(entry, "dL_dcamera"):
        names.append("dL_dcamera")
    out = []
    for n in names:
        a = kw[n] if n in kw else (None if n in ABSENT else ADDR[n])
        if a is not None:
            out.append((n, a))
    return out


def _backward_faults(entry, scratch_bytes):
    accum = "_accum" in entry
    faults = []
    if entry.endswith(("_cam", "_cam_f16")):
        faults += [(dict(dL_dcamera=None), "NULL dL_dcamera"), (dict(dL_dcamera=None, P=0), "NULL dL_dcamera")]
    if _has(entry, "dL_dalpha"):
        faults += [({p: None}, "NULL dL_dalpha / dL_dinvdepth") for p in ("dL_dalpha", "dL_dinvdepth")]
        faults += [(dict(dL_dalpha=None, P=0), "NULL dL_dalpha / dL_dinvdepth")]
    typed = _has(entry, "semantic_feature_dtype")
    if typed:
        faults += [({p: t}, "unknown dtype code") for p in ("semantic_feature_dtype", "dL_dfeaturepix_dtype")
                   for t in (-1, 2)]
        faults += [(dict(dL_dfeaturepix_dtype=2, P=0), "unknown dtype code")]
    if "feature_geometry" in entry:
        faults += [(dict(semantic_feature=None), "NULL semantic_feature"),
                   (dict(semantic_feature=None, P=0), "NULL semantic_feature")]

    faults += [(d, "bad sizes") for d in (dict(P=-1), dict(width=0), dict(height=0), dict(C=-1), dict(C=MAX_C + 1),
                                          dict(R=-1))]
    faults += [({b: None}, "missing forward buffers") for b in ("geom_buffer", "binning_buffer", "image_buffer")]
    grads = ["dL_dpix", "dL_depths", "dL_dfeaturepix", "dL_dsemantic_feature", "dL_dopacity", "dL_dmean3D"]
    if not accum:
        grads += ["dL_dmean2D", "dL_dconic", "dL_dcolor", "dL_dcov3D", "dL_dz"]
    faults += [({g: None}, "NULL gradient pointer") for g in grads]
    faults += [(dict(dL_dsh=None), "shs given but dL_dsh NULL")]
    faults += [({p: None}, "scales given but rotations/dL_dscale/dL_drot NULL")
               for p in ("rotations", "dL_dscale", "dL_drot")]
    if accum:
        faults += [({p: None}, "grad_accum and denom go together") for p in ("grad_accum", "denom")]
        faults += [(dict(scratch=None), "NULL scratch")]
        faults += [(d, GO_WITH) for d in (dict(dL_dcolors_precomp=DCOL), dict(shs=None, colors_precomp=COLOURS),
                                          dict(dL_dcov3D_precomp=DCOV),
                                          dict(scales=None, rotations=None, cov3D_precomp=COV))]

    # a float16 map gradient: its scale, and the float32 feature gradient reduced while the map is read
    f16 = [dict()] if entry.endswith("_f16") else [dict(dL_dfeaturepix_dtype=F16)] if typed else []
    for d in f16:
        faults += [(dict(d, dL_dfeaturepix_scale=s), SCALE) for s in (0.0, -0.0, float("inf"), float("-inf"),
                                                                     float("nan"))]
        faults += [(dict(d, dL_dsemantic_feature=ADDR["dL_dfeaturepix"] + o),
                    "dL_dsemantic_feature overlaps dL_dfeaturepix") for o in (0, C * W * H * 2 - 4)]

    # with the optional inputs given, so that every output is present
    full = [dict()]
    if accum:
        full.append(dict(shs=None, colors_precomp=COLOURS, dL_dcolors_precomp=DCOL, scales=None, rotations=None,
                         cov3D_precomp=COV, dL_dcov3D_precomp=DCOV))
    for base in full:
        outs = _outputs(entry, **base)
        if _has(entry, "dL_dcamera"):
            msg = "dL_dcamera overlaps another output"
            # under antialiasing dL_dopacity on dL_dcamera is two faults (each overlaps another output)
            faults += [(dict(base, dL_dcamera=a), msg) for n, a in outs
                       if n != "dL_dcamera" and not (n == "dL_dopacity" and "antialiased" in entry)]
            if accum:  # inside the scratch: the per-view intermediates
                faults += [(dict(base, dL_dcamera=ADDR["scratch"] + o), msg) for o in (256, scratch_bytes - 4)]
        if typed:
            for t in (F32, F16):
                faults += [(dict(base, semantic_feature=a, semantic_feature_dtype=t),
                            "semantic_feature overlaps an output") for _, a in outs]
        aa = [dict(antialiasing=1)] if _has(entry, "antialiasing") else [dict()] if "antialiased" in entry else []
        for d in aa:
            faults += [(dict(base, dL_dopacity=a, **d), "dL_dopacity overlaps another output")
                       for n, a in outs if n not in ("dL_dopacity", "dL_dcamera")]
        if _has(entry, "dL_dalpha"):
            for aa_flag in (0, 1):
                faults += [(dict(base, antialiasing=aa_flag, **{p: a}), "dL_dalpha / dL_dinvdepth overlap an output")
                           for p in ("dL_dalpha", "dL_dinvdepth") for _, a in outs]
    return faults


@pytest.mark.parametrize("entry", ENTRIES)
def test_single_fault_is_rejected_with_its_message(lib, entry):
    if entry in FORWARD:
        faults = _forward_faults(entry)
    else:
        faults = _backward_faults(entry, lib.f3dgs_backward_scratch_bytes(P))
    for kw, msg in faults:
        assert _call(lib, entry, **kw) == (-1, f"{entry}: {msg}"), kw


@pytest.mark.parametrize("entry", ENTRIES)
def test_p_zero_is_a_no_op(lib, entry):
    assert _call(lib, entry, P=0) == (0, "")
    if "_accum" in entry:  # the accumulating entries return before the size checks
        assert _call(lib, entry, P=0, width=0) == (0, "")
    elif entry in BACKWARD:
        assert _call(lib, entry, P=0, width=0) == (-1, f"{entry}: bad sizes")
    else:
        assert _call(lib, entry, P=0, width=0) == (-1, f"{entry}: {BAD_FWD}")
