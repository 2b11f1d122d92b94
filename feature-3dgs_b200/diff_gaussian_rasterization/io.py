"""On-disk formats around the rasterizer (SURVEY.md section 8 f4), written and read without `plyfile`:

  * point_cloud.ply of the reference (scene/gaussian_model.py:192-229 save_ply, :236-281 load_ply): binary little-endian,
    one `vertex` element of float32 properties  x y z nx ny nz f_dc_* f_rest_* opacity scale_* rot_* semantic_*  in that
    order; f_dc / f_rest / semantic are stored channel-major (the reference transposes [P, K, 3] -> [P, 3, K] before
    flattening, :214-215, :220).  A vector-quantised feature field (GaussianState.quantize_features) is stored as
    LightGaussian / CompGS store theirs: the vertex element carries `ushort semantic_code` in place of semantic_*, and a
    second element `semantic_codebook` of K rows holds float32 semantic_0 .. semantic_{C-1}.
  * points3D.ply of a COLMAP / synthetic scene (scene/dataset_readers.py fetchPly): x y z nx ny nz red green blue, the
    input of GaussianState.from_point_cloud.
  * `<name>_fmap_CxHxW.pt` (render.py:179-180, scene/dataset_readers.py:110-112): the rendered / teacher feature map as a
    float16 tensor [C, H, W] saved with torch.save.
Pure host-side I/O (numpy / torch.save): nothing here runs on the hot path.
"""
import os
from typing import Dict

import numpy as np


def ply_attribute_names(n_dc: int, n_rest: int, n_scale: int, n_rot: int, n_sem: int):
    """scene/gaussian_model.py:192-208 (construct_list_of_attributes)."""
    names = ["x", "y", "z", "nx", "ny", "nz"]
    names += [f"f_dc_{i}" for i in range(n_dc)] + [f"f_rest_{i}" for i in range(n_rest)] + ["opacity"]
    names += [f"scale_{i}" for i in range(n_scale)] + [f"rot_{i}" for i in range(n_rot)]
    names += [f"semantic_{i}" for i in range(n_sem)]
    return names


def save_ply(path: str, xyz, features_dc, features_rest, opacity, scaling, rotation, semantic_feature,
             semantic_codebook=None, semantic_code=None):
    """Raw (pre-activation) parameters as numpy arrays: xyz [P,3], features_dc [P,1,3], features_rest [P,K,3], opacity
    [P,1], scaling [P,3], rotation [P,4], semantic_feature [P,1,C].

    With semantic_codebook [K,C] and semantic_code [P] (GaussianState.codebook and .code; tensors or arrays), the features
    are stored quantised and semantic_feature is not read: the vertex element ends with `property ushort semantic_code`
    instead of the C semantic_* floats (K <= 65536, so every code fits), and an element `semantic_codebook K` with
    `property float semantic_0 .. semantic_{C-1}` follows it.  That saves 4 C - 2 bytes per Gaussian for 4 K C bytes."""
    f32 = np.float32
    xyz = np.asarray(xyz, f32)
    P = xyz.shape[0]
    f_dc = np.asarray(features_dc, f32).transpose(0, 2, 1).reshape(P, -1)
    f_rest = np.asarray(features_rest, f32).transpose(0, 2, 1).reshape(P, -1)
    quantized = semantic_codebook is not None or semantic_code is not None
    if quantized:
        book, code = _as_numpy(semantic_codebook), _as_numpy(semantic_code)
        if book is None or code is None or book.ndim != 2 or code.shape != (P,):
            raise ValueError("save_ply: semantic_codebook must be [K,C] and semantic_code [P], both given")
        book = np.ascontiguousarray(book, dtype="<f4")
        if not 1 <= book.shape[0] <= 65536 or (P and (code.min() < 0 or code.max() >= book.shape[0])):
            raise ValueError(f"save_ply: codes must be in [0, K) with 1 <= K <= 65536 (K = {book.shape[0]})")
        sem = np.zeros((P, 0), f32)
    else:
        sem = np.asarray(semantic_feature, f32).transpose(0, 2, 1).reshape(P, -1)
    cols = np.concatenate((xyz, np.zeros_like(xyz), f_dc, f_rest, np.asarray(opacity, f32).reshape(P, 1),
                           np.asarray(scaling, f32).reshape(P, -1), np.asarray(rotation, f32).reshape(P, -1), sem), axis=1)
    names = ply_attribute_names(f_dc.shape[1], f_rest.shape[1], np.asarray(scaling).reshape(P, -1).shape[1],
                                np.asarray(rotation).reshape(P, -1).shape[1], sem.shape[1])
    assert cols.shape[1] == len(names)
    os.makedirs(os.path.dirname(os.path.abspath(path)) or ".", exist_ok=True)
    header = ["ply", "format binary_little_endian 1.0", f"element vertex {P}"]
    header += [f"property float {n}" for n in names]
    if quantized:
        C = book.shape[1]
        header += ["property ushort semantic_code", f"element semantic_codebook {book.shape[0]}"]
        header += [f"property float semantic_{i}" for i in range(C)]
        rows = np.empty(P, dtype=[("f", "<f4", (len(names),)), ("code", "<u2")])
        rows["f"] = cols
        rows["code"] = code.astype(np.uint16)
    header += ["end_header"]
    with open(path, "wb") as f:
        f.write(("\n".join(header) + "\n").encode("ascii"))
        if quantized:
            f.write(rows.tobytes())
            f.write(book.tobytes())
        else:
            f.write(np.ascontiguousarray(cols, dtype="<f4").tobytes())


def _as_numpy(a):
    if a is None:
        return None
    if hasattr(a, "detach"):
        a = a.detach().cpu().numpy()
    return np.asarray(a)


_PLY_TYPES = {"float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8", "uchar": "u1", "uint8": "u1",
              "char": "i1", "int8": "i1", "short": "<i2", "int16": "<i2", "ushort": "<u2", "uint16": "<u2", "int": "<i4",
              "int32": "<i4", "uint": "<u4", "uint32": "<u4"}


def read_ply_vertices(path: str) -> Dict[str, np.ndarray]:
    """Minimal reader for binary little-endian / ascii PLY files with a scalar-property `vertex` element first."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, count, props, in_vertex = None, None, [], False
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: truncated PLY header")
            tok = line.decode("ascii").split()
            if not tok:
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                in_vertex = tok[1] == "vertex" and count is None
                if in_vertex:
                    count = int(tok[2])
            elif tok[0] == "property" and in_vertex:
                if tok[1] == "list":
                    raise ValueError(f"{path}: list properties in the vertex element are not supported")
                props.append((tok[2], _PLY_TYPES[tok[1]]))
            elif tok[0] == "end_header":
                break
        if count is None:
            raise ValueError(f"{path}: no vertex element")
        if fmt == "binary_little_endian":
            data = np.frombuffer(f.read(count * np.dtype(props).itemsize), dtype=np.dtype(props), count=count)
            return {n: np.asarray(data[n]) for n, _ in props}
        if fmt == "ascii":
            arr = np.loadtxt(f, max_rows=count, ndmin=2)
            return {n: arr[:, i].astype(t) for i, (n, t) in enumerate(props)}
        raise ValueError(f"{path}: unsupported PLY format {fmt}")


def _read_ply_codebook(path: str):
    """The `semantic_codebook` element of a binary little-endian PLY written by save_ply (after a `vertex` element of
    scalar properties) as float32 [K,C], or None if the file has no such element."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, elements = None, []  # [name, count, [(property, dtype)]]
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: truncated PLY header")
            tok = line.decode("ascii").split()
            if not tok:
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                elements.append([tok[1], int(tok[2]), []])
            elif tok[0] == "property" and elements:
                if tok[1] == "list":
                    elements[-1][2].append((tok[-1], None))
                else:
                    elements[-1][2].append((tok[2], _PLY_TYPES[tok[1]]))
            elif tok[0] == "end_header":
                break
        names = [e[0] for e in elements]
        if "semantic_codebook" not in names:
            return None
        if fmt != "binary_little_endian" or names[:2] != ["vertex", "semantic_codebook"] or any(
                t is None for e in elements[:2] for _, t in e[2]):
            raise ValueError(f"{path}: semantic_codebook must follow a scalar vertex element in a binary little-endian "
                             "file")
        (_, n_v, p_v), (_, K, p_c) = elements[:2]
        f.seek(n_v * np.dtype(p_v).itemsize, 1)
        data = np.frombuffer(f.read(K * np.dtype(p_c).itemsize), dtype=np.dtype(p_c), count=K)
        cols = sorted((n for n, _ in p_c if n.startswith("semantic_")), key=lambda n: int(n.split("_")[-1]))
        return np.stack([data[n] for n in cols], axis=1).astype(np.float32) if cols else np.zeros((K, 0), np.float32)


def load_ply(path: str, max_sh_degree: int = 3) -> Dict[str, np.ndarray]:
    """-> raw parameters shaped like the reference's load_ply builds them (scene/gaussian_model.py:236-281).  For a file
    save_ply wrote with a codebook, also semantic_codebook [K,C] float32 and semantic_code [P] int32, with
    semantic_feature = semantic_codebook[semantic_code] as [P,1,C], so callers of the unquantised layout work unchanged."""
    v = read_ply_vertices(path)
    f32 = np.float32
    P = v["x"].shape[0]
    xyz = np.stack((v["x"], v["y"], v["z"]), axis=1).astype(f32)

    def numbered(prefix):
        names = sorted((n for n in v if n.startswith(prefix)), key=lambda n: int(n.split("_")[-1]))
        return np.stack([v[n] for n in names], axis=1).astype(f32) if names else np.zeros((P, 0), f32)

    f_dc = numbered("f_dc_").reshape(P, 3, -1).transpose(0, 2, 1)
    rest = numbered("f_rest_")
    if rest.shape[1] != 3 * (max_sh_degree + 1) ** 2 - 3:
        raise ValueError(f"{path}: {rest.shape[1]} f_rest properties, expected {3 * (max_sh_degree + 1) ** 2 - 3}")
    f_rest = rest.reshape(P, 3, -1).transpose(0, 2, 1)
    out = {}
    if "semantic_code" not in v:
        sem = numbered("semantic_")
    else:
        book = _read_ply_codebook(path)
        if book is None:
            raise ValueError(f"{path}: semantic_code without a semantic_codebook element")
        code = v["semantic_code"].astype(np.int32)
        if P and code.max() >= book.shape[0]:
            raise ValueError(f"{path}: a semantic_code is not below K = {book.shape[0]}")
        sem = book[code]
        out = dict(semantic_codebook=book, semantic_code=code)
    return dict(xyz=xyz, features_dc=np.ascontiguousarray(f_dc), features_rest=np.ascontiguousarray(f_rest),
                opacity=np.asarray(v["opacity"], f32).reshape(P, 1), scaling=numbered("scale_"), rotation=numbered("rot_"),
                semantic_feature=np.ascontiguousarray(sem.reshape(P, -1, 1).transpose(0, 2, 1)), **out)


def load_point_cloud(path: str):
    """-> (points [P,3], colors [P,3], normals [P,3]) as the reference's fetchPly reads a points3D.ply
    (scene/dataset_readers.py): x y z and nx ny nz as stored, red green blue (uchar) / 255.0 in float64."""
    v = read_ply_vertices(path)
    missing = [n for n in ("x", "y", "z", "nx", "ny", "nz", "red", "green", "blue") if n not in v]
    if missing:
        raise ValueError(f"{path}: vertex element lacks {', '.join(missing)}")
    points = np.vstack([v["x"], v["y"], v["z"]]).T
    colors = np.vstack([v["red"], v["green"], v["blue"]]).T / 255.0
    normals = np.vstack([v["nx"], v["ny"], v["nz"]]).T
    return points, colors, normals


def fmap_filename(stem: str, C: int, H: int, W: int) -> str:
    return f"{stem}_fmap_CxHxW.pt"  # the reference keeps the literal suffix (render.py:179)


def save_feature_map(path: str, feature_map):
    """float16 [C,H,W] tensor via torch.save, as render.py:179-180 writes it."""
    import torch

    t = feature_map if isinstance(feature_map, torch.Tensor) else torch.from_numpy(np.asarray(feature_map))
    os.makedirs(os.path.dirname(os.path.abspath(path)) or ".", exist_ok=True)
    torch.save(t.detach().to("cpu", torch.float16).contiguous(), path)


def load_feature_map(path: str, device="cpu", dtype="float32"):
    """-> [C,H,W] (scene/dataset_readers.py:110-112 loads the tensor and the trainer moves it to the GPU), float32 by
    default; dtype=None keeps the stored dtype (float16 as save_feature_map writes it), which the feature losses of
    feature_head take as it is, at half the memory.  (The default is spelt as a string because torch is imported lazily.)"""
    import torch

    t = torch.load(path, map_location="cpu")
    if t.dim() != 3:
        raise ValueError(f"{path}: expected a [C,H,W] tensor, got {tuple(t.shape)}")
    return t.to(device=device, dtype=torch.float32 if dtype == "float32" else dtype)
