"""One small forward + backward through the autograd API and one feature-head call, for compute-sanitizer:
    compute-sanitizer --tool memcheck python tools/sanitize_probe.py small128
Development tool, not product code."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "feature-3dgs_b200")]
import scenegen  # noqa: E402
from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer  # noqa: E402
from diff_gaussian_rasterization import feature_head as fh  # noqa: E402

name = sys.argv[1] if len(sys.argv) > 1 else "small128"
sc = scenegen.make_config(name)
cam = sc.cameras[0]
t = scenegen.to_torch(sc, "cuda", requires_grad=True)
rast = GaussianRasterizer(GaussianRasterizationSettings(**scenegen.settings_kwargs(sc, cam, "cuda")))
means2D = torch.zeros_like(t["means3D"], requires_grad=True)
color, feat, radii, depth = rast(means3D=t["means3D"], means2D=means2D, opacities=t["opacities"], shs=t["shs"],
                                 semantic_feature=t["semantic_feature"], scales=t["scales"], rotations=t["rotations"])
H, W = cam.image_height, cam.image_width
gt = torch.rand(feat.shape[0], max(int(round(H / 2.25)), 1), max(int(round(W / 2.25)), 1), device="cuda")
loss, gfeat = fh.feature_l1_loss_and_grad(feat.detach(), gt, 1.0)
torch.autograd.backward([color, depth, feat], [torch.ones_like(color), torch.ones_like(depth), gfeat])
torch.cuda.synchronize()
print("probe ok", name, float(loss), float(t["semantic_feature"].grad.abs().sum()))
