"""Seeded synthetic Gaussian clouds and cameras for tests, golden vectors and bench.py.

Shapes and conventions follow what the reference's renderer feeds the rasterizer
(gaussian_renderer/__init__.py:188-252, scene/cameras.py:49-58, utils/graphics_utils.py:38-71):
  viewmatrix = world_view_transform = W2C^T (row-major torch tensor == column-major for the kernels)
  projmatrix = full_proj_transform  = W2C^T @ P^T          campos = inverse(viewmatrix)[3, :3]
Everything is generated with numpy's PCG64 (bit-reproducible on every host) as float32 and only
then moved to the requested device, so the CPU container and the GPU box see identical inputs.

Distributions (SURVEY.md section 8d): means uniform in [-1,1]^3; scales = exp(N(mu_s, 0.5^2)) with mu_s
chosen so that the median projected radius is about `target_radius_px`; rotations = normalised
N(0,1)^4; opacity = sigmoid(N(0, 2^2)); SH DC ~ N(0,1), higher bands ~ N(0, 0.2^2); features
N(0,1); background 0.  Cameras: pinhole, FoVx 60 deg, znear 0.01, zfar 100, on a ring of radius
3.5 around the origin looking at it, evenly spaced + seeded jitter.
"""
import math
from dataclasses import dataclass, field
from typing import Dict, List

import numpy as np

CONFIGS: Dict[str, dict] = {
    # BASELINE.json "configs" in order
    "c1": dict(P=10_000, W=256, H=256, C=0, sh_degree=3, views=1),
    "c2": dict(P=300_000, W=800, H=800, C=16, sh_degree=3, views=1),
    "c3": dict(P=1_000_000, W=1920, H=1080, C=128, sh_degree=3, views=1),
    "c4": dict(P=1_000_000, W=1920, H=1080, C=256, sh_degree=3, views=64),
    "c5": dict(P=5_000_000, W=3840, H=2160, C=64, sh_degree=3, views=1),
    # analysis variants of c3 (same cloud and camera, other feature widths)
    "c3_C0": dict(P=1_000_000, W=1920, H=1080, C=0, sh_degree=3, views=1),
    "c3_C32": dict(P=1_000_000, W=1920, H=1080, C=32, sh_degree=3, views=1),
    "c3_C64": dict(P=1_000_000, W=1920, H=1080, C=64, sh_degree=3, views=1),
    # small cases for parity tests / golden fixtures
    "tiny": dict(P=600, W=80, H=56, C=8, sh_degree=3, views=1),
    "small": dict(P=4000, W=160, H=112, C=16, sh_degree=2, views=1),
    # small cases with wide features: a full 128-channel chunk, and an odd image size with two channel chunks
    "small128": dict(P=4000, W=160, H=112, C=128, sh_degree=2, views=1),
    "small200": dict(P=3000, W=150, H=100, C=200, sh_degree=1, views=1),
}


@dataclass
class Camera:
    image_width: int
    image_height: int
    tanfovx: float
    tanfovy: float
    viewmatrix: np.ndarray   # [4,4] float32, = W2C^T
    projmatrix: np.ndarray   # [4,4] float32, = W2C^T @ P^T
    campos: np.ndarray       # [3]   float32


@dataclass
class Scene:
    means3D: np.ndarray      # [P,3]
    scales: np.ndarray       # [P,3]  (already exp-activated)
    rotations: np.ndarray    # [P,4]  (normalised, (w,x,y,z))
    opacities: np.ndarray    # [P,1]  (already sigmoid-activated)
    shs: np.ndarray          # [P,16,3]
    features: np.ndarray     # [P,1,C]
    bg: np.ndarray           # [3]
    sh_degree: int
    cameras: List[Camera] = field(default_factory=list)

    @property
    def P(self):
        return self.means3D.shape[0]

    @property
    def C(self):
        return self.features.shape[-1]


def _look_at(eye: np.ndarray, target: np.ndarray, up=np.array([0.0, 1.0, 0.0])) -> np.ndarray:
    """World-to-camera 4x4 (camera looks down +z, x right, y down-ish like COLMAP)."""
    f = target - eye
    f = f / np.linalg.norm(f)
    r = np.cross(up, f)
    r = r / np.linalg.norm(r)
    u = np.cross(f, r)
    R = np.stack([r, u, f], axis=0)  # rows = camera axes in world coords
    W2C = np.eye(4)
    W2C[:3, :3] = R
    W2C[:3, 3] = -R @ eye
    return W2C


def make_camera(W: int, H: int, eye, fovx_deg: float = 60.0, znear: float = 0.01, zfar: float = 100.0) -> Camera:
    tanx = math.tan(math.radians(fovx_deg) / 2)
    tany = tanx * H / W
    W2C = _look_at(np.asarray(eye, dtype=np.float64), np.zeros(3))
    P = np.zeros((4, 4))
    # utils/graphics_utils.py:51-71 with symmetric frustum
    P[0, 0] = 1.0 / tanx
    P[1, 1] = 1.0 / tany
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    view = W2C.T.astype(np.float32)
    proj = (W2C.T @ P.T).astype(np.float32)
    campos = np.linalg.inv(view.astype(np.float64))[3, :3].astype(np.float32)
    return Camera(W, H, float(np.float32(tanx)), float(np.float32(tany)), view, proj, campos)


def make_scene(P: int, W: int, H: int, C: int, sh_degree: int = 3, views: int = 1, seed: int = 0,
               target_radius_px: float = 6.0, ring_radius: float = 3.5, fovx_deg: float = 60.0) -> Scene:
    rng = np.random.Generator(np.random.PCG64(seed))
    f32 = np.float32
    means = rng.uniform(-1.0, 1.0, size=(P, 3)).astype(f32)
    focal = W / (2 * math.tan(math.radians(fovx_deg) / 2))
    sigma_px = math.sqrt(max((target_radius_px / 3.0) ** 2 - 0.3, 0.05))
    mu_s = math.log(sigma_px * ring_radius / focal) - 0.42  # median of max of 3 lognormals(0.5)
    scales = np.exp(rng.normal(mu_s, 0.5, size=(P, 3))).astype(f32)
    q = rng.normal(size=(P, 4))
    rotations = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(f32)
    opacities = (1.0 / (1.0 + np.exp(-rng.normal(0.0, 2.0, size=(P, 1))))).astype(f32)
    shs = np.concatenate([rng.normal(0.0, 1.0, size=(P, 1, 3)), rng.normal(0.0, 0.2, size=(P, 15, 3))], axis=1).astype(f32)
    features = rng.standard_normal(size=(P, 1, C), dtype=f32) if C > 0 else np.zeros((P, 1, 0), f32)
    cams = []
    for v in range(views):
        ang = 2 * math.pi * (v + rng.uniform(-0.2, 0.2)) / max(views, 1)
        elev = rng.uniform(-0.3, 0.3)
        eye = ring_radius * np.array([math.cos(ang) * math.cos(elev), math.sin(elev), math.sin(ang) * math.cos(elev)])
        cams.append(make_camera(W, H, eye, fovx_deg))
    return Scene(means, scales, rotations, opacities, shs, features, np.zeros(3, f32), sh_degree, cams)


def make_config(name: str, seed: int = None, views: int = None) -> Scene:
    cfg = dict(CONFIGS[name])
    if views is not None:
        cfg["views"] = views
    if seed is None:
        seed = 3 if name.startswith("c3_") else list(CONFIGS).index(name) + 1
    return make_scene(seed=seed, **cfg)


def upstream_grads(H: int, W: int, C: int, seed: int = 1234):
    """Fixed upstream gradients dL/dcolor, dL/dfeature, dL/ddepth ~ N(0,1) (SURVEY 8d)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    f32 = np.float32
    return (rng.standard_normal((3, H, W), dtype=f32), rng.standard_normal((C, H, W), dtype=f32),
            rng.standard_normal((1, H, W), dtype=f32))


def to_torch(scene: Scene, device, requires_grad: bool = False):
    """Scene -> dict of torch tensors shaped like the reference's render() passes them."""
    import torch

    def t(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(device)

    d = dict(means3D=t(scene.means3D), scales=t(scene.scales), rotations=t(scene.rotations),
             opacities=t(scene.opacities), shs=t(scene.shs), semantic_feature=t(scene.features), bg=t(scene.bg))
    if requires_grad:
        for k in ("means3D", "scales", "rotations", "opacities", "shs", "semantic_feature"):
            d[k].requires_grad_(True)
    return d


def settings_kwargs(scene: Scene, cam: Camera, device, debug: bool = False):
    import torch

    def t(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(device)

    return dict(image_height=cam.image_height, image_width=cam.image_width, tanfovx=cam.tanfovx,
                tanfovy=cam.tanfovy, bg=t(scene.bg), scale_modifier=1.0, viewmatrix=t(cam.viewmatrix),
                projmatrix=t(cam.projmatrix), sh_degree=scene.sh_degree, campos=t(cam.campos), prefiltered=False,
                debug=debug)
