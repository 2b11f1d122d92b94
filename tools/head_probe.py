"""Two calls of the fused feature head at the config-3 shape (C = 128, 822x1237 -> 365x549), for an ncu capture:
    ncu --set full --clock-control none -k regex:resize_ -c 3 -o r02_head python tools/head_probe.py
Development tool, not product code."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "feature-3dgs_b200"))
from diff_gaussian_rasterization import feature_head as fh  # noqa: E402

C, H, W = 128, 822, 1237
x = torch.randn(C, H, W, device="cuda")
gt = torch.randn(C, int(round(H / 2.25)), int(round(W / 2.25)), device="cuda")
for _ in range(2):
    loss, grad = fh.feature_l1_loss_and_grad(x, gt, 1.0)
torch.cuda.synchronize()
print("loss", float(loss), "grad abs sum", float(grad.abs().sum()))
