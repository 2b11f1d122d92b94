"""Post-raster feature head (SURVEY.md section 8 f1): the reference's

    feature_map = F.interpolate(feature_map.unsqueeze(0), size=gt.shape[1:], mode='bilinear', align_corners=True).squeeze(0)
    [feature_map = cnn_decoder(feature_map)]          # 1x1 conv, only with --speedup (models/networks.py:107-119)
    Ll1_feature = l1_loss(feature_map, gt)            # train.py:98-104

on two CUDA kernels of libf3dgs_b200 (csrc/feature_head.cu): a resize that, given the teacher map, directly emits the loss
and dL/d(resized map), and a gather-style resize backward that writes every element of dL/dfeature_map exactly once.
With --speedup the 1x1 decoder and its loss run in between on csrc/feature_decoder.cu (TF32 tensor cores, like cuDNN's
default for the reference's nn.Conv2d): `decode`, `decoded_feature_l1_loss_and_grad`, `decoded_feature_l1_loss`.
`query` asks the trained field questions with text embeddings (csrc/feature_query.cu): LSeg's per-pixel labels and
render_edit's per-Gaussian selection score, without materialising the decoded map.  `pca_fit` and `pca_image` make
render.py's PCA picture of a feature map on the device (csrc/feature_pca.cu).  `FeatureLift` makes a feature field
without training: every Gaussian gets the blend-weighted mean of the teacher features of the pixels it is blended into
(the backward composite's lift mode, csrc/composite_bwd.cu, and feature_bwd.cu).
There is no CPU path (the extension raises on CPU tensors).

The teacher map `gt` may be float32 or float16, the dtype the data format stores it in (io.load_feature_map(path,
dtype=None)).  A float16 map is read as it is and upcast exactly inside the kernels, so no float32 copy is made and every
result equals the one for `gt.float()`; the loss and the gradients are float32, as PyTorch's `l1_loss(fp32, fp16)` gives.

Training a float16 feature field (GaussianState(feature_dtype=torch.float16), ViewBatch): the two `_and_grad` functions
also read a float16 rendered map exactly, and with grad_dtype=torch.float16 return dL/dfeature_map as a `ScaledGrad`, a
float16 map plus a float32 scale, for `ViewBatch.backward`.  The scale is needed: the L1 gradient is
sign * weight / (C*Hg*Wg), about 1.9e-8 at C = 128 and a 853x480 teacher, below float16's smallest subnormal (5.96e-8),
so a plain float16 cast of it is all zeros.  The autograd wrappers stay float32: autograd would cast the gradient to
float16 without a scale.
"""
from typing import NamedTuple, Optional

import torch


def _C():
    from . import _C as ext  # deferred: keeps this module importable for documentation tools without the extension

    return ext


class ScaledGrad(NamedTuple):
    """A float16 gradient map that stands for `scale * grad.float()`: grad [C,H,W] float16 holds dL/dO / scale, so that
    a gradient far below float16's range keeps its digits (ViewBatch.backward applies the scale in float32)."""

    grad: torch.Tensor
    scale: float


def _grad_half(grad_dtype) -> bool:
    if grad_dtype is None or grad_dtype == torch.float32:
        return False
    if grad_dtype == torch.float16:
        return True
    raise ValueError(f"grad_dtype must be None, torch.float32 or torch.float16, got {grad_dtype}")


def _reject_half(feature_map: torch.Tensor, fn: str):
    if feature_map.dtype == torch.float16:
        raise RuntimeError(
            f"{fn}: feature_map must be float32; train a float16 map without autograd: the ViewBatch path, "
            f"{fn}_and_grad(..., grad_dtype=torch.float16) -> ViewBatch.backward (autograd would cast the gradient to "
            "float16 without a scale, and it would underflow)")


def feature_l1_loss_and_grad(feature_map: torch.Tensor, gt: torch.Tensor, weight: float = 1.0, grad_dtype=None):
    """-> (loss, dL/dfeature_map) for loss = weight * mean|resize(feature_map) - gt|, no autograd graph (ViewBatch loops).

    feature_map may be float32 or float16 (read exactly).  grad_dtype=torch.float16 returns the gradient as a
    ScaledGrad: the float16 map resize^T(sign(resized - gt)) with scale = weight / (C*Hg*Wg), so no [C,H,W] float32
    tensor is made.  With the default arguments the results are the float32 ones."""
    C, Hg, Wg = gt.shape
    n = max(C * Hg * Wg, 1)
    H, W = feature_map.shape[1], feature_map.shape[2]
    if not _grad_half(grad_dtype):
        sign, loss_sum = _C().feature_resize_fwd(feature_map, gt, Hg, Wg, weight / n)
        grad = _C().feature_resize_bwd(sign, H, W)
        return loss_sum[0] * (weight / n), grad
    # exact signs (grad_scale 1) and the whole factor weight / n in the float32 scale; a zero weight gives zero signs
    scale = weight / n
    sign, loss_sum = _C().feature_resize_fwd(feature_map, gt, Hg, Wg, 1.0 if scale != 0 else 0.0)
    grad = _C().feature_resize_bwd(sign, H, W, torch.float16, 1.0)
    return loss_sum[0] * scale, ScaledGrad(grad, scale if scale != 0 else 1.0)


class _FeatureL1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feature_map, gt, weight):
        _reject_half(feature_map, "feature_l1_loss")
        loss, grad = feature_l1_loss_and_grad(feature_map, gt, weight)
        ctx.save_for_backward(grad)
        return loss

    @staticmethod
    def backward(ctx, g):
        (grad,) = ctx.saved_tensors
        return grad * g, None, None


def feature_l1_loss(feature_map: torch.Tensor, gt: torch.Tensor, weight: float = 1.0) -> torch.Tensor:
    """Autograd-aware drop-in for `l1_loss(F.interpolate(feature_map[None], gt.shape[1:], 'bilinear', True)[0], gt) * weight`."""
    return _FeatureL1.apply(feature_map, gt, float(weight))


class _Resize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feature_map, Hg, Wg):
        if feature_map.dtype != torch.float32:
            raise RuntimeError("resize_bilinear: feature_map must be float32 (autograd would cast its gradient to "
                               "float16 without a scale)")
        ctx.hw = (feature_map.shape[1], feature_map.shape[2])
        out, _ = _C().feature_resize_fwd(feature_map, torch.empty(0, device=feature_map.device), Hg, Wg, 0.0)
        return out

    @staticmethod
    def backward(ctx, dout):
        return _C().feature_resize_bwd(dout.contiguous(), ctx.hw[0], ctx.hw[1]), None, None


def resize_bilinear(feature_map: torch.Tensor, size) -> torch.Tensor:
    """`F.interpolate(feature_map[None], size, mode='bilinear', align_corners=True)[0]` with the gather backward; use
    it in front of the optional 1x1 decoder: `l1_loss(decoder(resize_bilinear(fm, gt.shape[1:])), gt)`."""
    return _Resize.apply(feature_map, int(size[0]), int(size[1]))


def _empty(like: torch.Tensor) -> torch.Tensor:
    return torch.empty(0, device=like.device, dtype=like.dtype)


def decode(feature_map: torch.Tensor, weight: torch.Tensor, bias=None, dtype=torch.float32) -> torch.Tensor:
    """The reference's `cnn_decoder(feature_map)` (nn.Conv2d(Cin, Cout, 1)) without a graph: feature_map [Cin,H,W],
    weight [Cout,Cin,1,1] or [Cout,Cin], bias [Cout] or None -> [Cout,H,W].  dtype=torch.float16 writes the map the way
    render.py saves it, bitwise `decode(...).half()` without the float32 map or the cast pass."""
    with torch.no_grad():
        return _C().decoder_forward(feature_map, weight, _empty(feature_map) if bias is None else bias, dtype)


def decoded_feature_l1_loss_and_grad(feature_map: torch.Tensor, gt: torch.Tensor, weight: torch.Tensor, bias=None,
                                     loss_weight: float = 1.0, dweight=None, dbias=None, grad_dtype=None):
    """-> (loss, dL/dfeature_map, dweight, dbias) for the --speedup feature loss

        loss = loss_weight * l1_loss(cnn_decoder(F.interpolate(feature_map[None], gt.shape[1:], 'bilinear', True)[0]), gt)

    with no autograd graph and no host sync: dL/dfeature_map is the `g_feature` a ViewBatch loop passes to `vb.backward`.
    feature_map [Cin,H,W], gt [Cout,Hg,Wg], weight [Cout,Cin,1,1] or [Cout,Cin], bias [Cout] or None.  The gradients of
    the decoder are ADDED into `dweight` / `dbias` (typically `conv.weight.grad` / `conv.bias.grad`, so the views of a step
    accumulate); they are allocated zeroed when None, and dbias stays None without a bias.  Step the decoder with the
    reference's `torch.optim.Adam(cnn_decoder.parameters())` on those tensors; with several ranks, all-reduce them (they
    are small) before the step.

    feature_map may be float32 or float16 (read exactly).  grad_dtype=torch.float16 returns dL/dfeature_map as a
    ScaledGrad with scale = loss_weight / (Cout*Hg*Wg): the decoder's gradients use the true scale, and the float16 map
    is resize^T(dL/d resized) / scale."""
    Cout, Hg, Wg = gt.shape
    with torch.no_grad():
        resized, _ = _C().feature_resize_fwd(feature_map, _empty(feature_map), Hg, Wg, 0.0)
        if dweight is None:
            dweight = torch.zeros_like(weight, memory_format=torch.contiguous_format)
        if dbias is None and bias is not None:
            dbias = torch.zeros_like(bias, memory_format=torch.contiguous_format)
        gs = float(loss_weight) / max(Cout * Hg * Wg, 1)
        loss_sum, dres = _C().decoder_l1(resized, gt, weight, _empty(resized) if bias is None else bias, gs, dweight,
                                         _empty(resized) if dbias is None else dbias)
        H, W = feature_map.shape[1], feature_map.shape[2]
        if _grad_half(grad_dtype):
            s = gs if gs != 0 else 1.0  # gs == 0: dres is zero
            grad = ScaledGrad(_C().feature_resize_bwd(dres, H, W, torch.float16, 1.0 / s), s)
        else:
            grad = _C().feature_resize_bwd(dres, H, W)
    return loss_sum[0] * gs, grad, dweight, dbias


def query(features: torch.Tensor, text: torch.Tensor, weight=None, bias=None, logit_scale: float = 1.0, positive=None,
          logits: bool = False):
    """Ask a feature field questions with text (csrc/feature_query.cu): -> (labels, prob or None, logits or None).

    features [C,H,W] or [C,N], float32 or float16 (a saved map is read as float16, with the result of `.float()`);
    text [K,D] embeddings (1 <= K <= 256); weight [D,C,1,1] or [D,C] and bias [D] the --speedup decoder, or None (then
    D == C).  Per column, with y the decoded feature and l_k = logit_scale * cos(y, text_k):
        labels  int64 argmax_k l_k                           (LSeg's segmentation head; first index on ties)
        prob    sum over k in `positive` of softmax_k(l)     (with `positive`, a sequence of prompt indices)
        logits  [K, ...] l                                   (with logits=True)
    shaped like `features` without its channel axis.  Nothing of size D x N is allocated.  No autograd: this is an
    inference path.

    render_edit's selection score of Gaussians: `query(state.raw["semantic_feature"][:, 0, :].t().contiguous(), text,
    w, b, positive=[0])`; the transposed [C,P] copy costs P x C x 4 bytes and one pass over the features.  Thresholding
    and the edit (zeroing opacity, recolouring) are plain tensor ops on the returned score."""
    K = text.shape[0]
    idx = None
    if positive is not None:
        idx = [int(i) for i in positive]
        bad = [i for i in idx if not 0 <= i < K]
        if bad:
            raise ValueError(f"query: positive indices {bad} out of range for {K} prompts")
    for name, t in (("features", features), ("text", text), ("weight", weight), ("bias", bias)):
        if t is not None and not t.is_cuda:
            raise ValueError(f"query: {name} must be a CUDA tensor (there is no CPU path)")
    with torch.no_grad():
        mask = torch.empty(0, dtype=torch.uint8, device=text.device)
        if idx is not None:
            mask = torch.zeros(K, dtype=torch.uint8, device=text.device)
            if idx:
                mask[idx] = 1
        lab, prob, lg = _C().feature_query(features, text, _empty(text) if weight is None else weight,
                                           _empty(text) if bias is None else bias, float(logit_scale), mask, True,
                                           idx is not None, bool(logits))
    return lab, (prob if idx is not None else None), (lg if logits else None)


class FeaturePCA(NamedTuple):
    """A PCA colour basis of a feature map (device tensors): mean [C] and components [3,C] float32, and the percentile
    range lo, hi (0-d float32) that maps the projections onto [0, 1]."""

    mean: torch.Tensor
    components: torch.Tensor
    lo: torch.Tensor
    hi: torch.Tensor


def _pca_check(x: torch.Tensor, fn: str, fit: Optional[FeaturePCA] = None):
    if not isinstance(x, torch.Tensor) or x.dim() not in (2, 3):
        raise ValueError(f"{fn}: x must be a tensor [C,H,W] or [C,N], got {getattr(x, 'shape', type(x))}")
    if x.dtype not in (torch.float32, torch.float16):
        raise ValueError(f"{fn}: x must be float32 or float16, got {x.dtype}")
    C = x.shape[0]
    N = x.numel() // max(C, 1)
    if not 3 <= C <= 1024:
        raise ValueError(f"{fn}: needs 3 <= C <= 1024 channels, got {C}")
    if (N + 2) // 3 < 3:
        raise ValueError(f"{fn}: needs at least 3 samples (every 3rd pixel: N >= 7), got N = {N}")
    if fit is not None and (tuple(fit.mean.shape) != (C,) or tuple(fit.components.shape) != (3, C)):
        raise ValueError(f"{fn}: the fit has {fit.mean.shape[0]} channels, x has {C}")
    if not x.is_cuda:
        raise ValueError(f"{fn}: x must be a CUDA tensor (there is no CPU path)")
    if not x.is_contiguous():
        raise ValueError(f"{fn}: x must be contiguous (the map is read in place, never copied)")


def pca_fit(x: torch.Tensor) -> FeaturePCA:
    """Fit render.py's PCA colour basis to a feature map x [C,H,W] or [C,N] (float32, or float16 with bitwise the result
    of `x.float()`, contiguous), on the device: the pixels are normalised (F.normalize, eps 1e-12), every 3rd pixel
    (p = y W + x, p % 3 == 0) is a sample, and the fit is scikit-learn's PCA(3) of the samples (components signed so that
    each one's largest |entry| is positive) with lo, hi = np.percentile(projections of the samples, [1, 99]).  x is read
    in place; nothing of size C x n is allocated.  One host sync, in the float64 eigensolver of the C x C covariance
    (torch.linalg.eigh on the device)."""
    _pca_check(x, "pca_fit")
    with torch.no_grad():
        mean, cov = _C().feature_pca_moments(x)
        # cuSOLVER on the device: at C = 512 it took 4.8 ms against 27-29 ms for LAPACK on the host, copy included
        # (tools/time_feature_pca.py, H100 80GB HBM3 at 700 W).  Its result check is the fit's one host sync.
        _, vec = torch.linalg.eigh(cov)
        comps = vec.flip(1)[:, :3].t()  # the three largest eigenvalues, descending
        first_max = comps.abs().argmax(dim=1, keepdim=True)  # first maximal |entry|
        comps = comps * torch.sign(comps.gather(1, first_max))
        comps = comps.float().contiguous()
        rng = _C().feature_pca_range(x, mean, comps)
    return FeaturePCA(mean, comps, rng[0], rng[1])


def pca_image(x: torch.Tensor, fit: Optional[FeaturePCA] = None) -> torch.Tensor:
    """PCA picture of a feature map x [C,H,W] or [C,N] -> [H,W,3] or [N,3] float32 on the device:
    clamp((c_k . (normalize(x_p) - mean) - lo) / (hi - lo), 0, 1).  fit=None fits on x itself, which is the drop-in for
    render.py's `feature_visualize_saving(x)` (== `pca_image(x).cpu()`); a fit from `pca_fit` on one frame gives the
    frames of a video consistent colours.  One read of the map; no autograd."""
    _pca_check(x, "pca_image", fit)
    if fit is None:
        fit = pca_fit(x)
    with torch.no_grad():
        rng = torch.stack((fit.lo, fit.hi)).to(device=x.device, dtype=torch.float32)
        return _C().feature_pca_image(x, fit.mean.contiguous(), fit.components.contiguous(), rng)


class _DecodedL1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feature_map, weight, bias, gt, loss_weight):
        _reject_half(feature_map, "decoded_feature_l1_loss")
        loss, g_fm, g_w, g_b = decoded_feature_l1_loss_and_grad(feature_map.detach(), gt.detach(), weight.detach(),
                                                                None if bias is None else bias.detach(), loss_weight)
        ctx.has_bias = bias is not None
        ctx.save_for_backward(g_fm, g_w, *((g_b,) if bias is not None else ()))
        return loss

    @staticmethod
    def backward(ctx, g):
        saved = ctx.saved_tensors
        g_b = saved[2] * g if ctx.has_bias else None
        return saved[0] * g, saved[1] * g, g_b, None, None


def decoded_feature_l1_loss(feature_map: torch.Tensor, gt: torch.Tensor, weight: torch.Tensor, bias=None,
                            loss_weight: float = 1.0) -> torch.Tensor:
    """Autograd-aware drop-in for the --speedup feature loss of train.py:
    `decoded_feature_l1_loss(feature_map, gt_feature_map, cnn_decoder.conv.weight, cnn_decoder.conv.bias)` equals
    `l1_loss(cnn_decoder(F.interpolate(feature_map[None], gt.shape[1:], 'bilinear', True)[0]), gt) * loss_weight`, with
    gradients for feature_map, weight and bias (gt is the constant target)."""
    return _DecodedL1.apply(feature_map, weight, bias, gt, float(loss_weight))


def _weights_forward(g, colors, e, antialiasing, rs, H, W):
    """The forward whose buffers FeatureLift and GaussianScores walk: C = 0 with zero colors_precomp (no SH work), at
    H x W, antialiased or not.  g holds means3D, opacities, scales, rotations and cov3D (e, empty, where absent).
    -> (R, geom, binning, img)"""
    fwd = _C().rasterize_gaussians_antialiased if antialiasing else _C().rasterize_gaussians
    R, _, _, _, _, geom, binning, img = fwd(
        rs.bg, g["means3D"], colors, e, g["opacities"], g["scales"], g["rotations"], rs.scale_modifier, g["cov3D"],
        rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, H, W, e, rs.sh_degree, rs.campos, rs.prefiltered,
        rs.debug)
    return R, geom, binning, img


class FeatureLift:
    """Lift 2-D feature maps onto Gaussians without training (blend-weighted back-projection over views):

        f_i = sum_{v,p} w_ivp F_v[:, p] / sum_{v,p} w_ivp,     w_ivp = alpha * T, Gaussian i's blend weight at pixel p of view v

        lift = FeatureLift(means3D, opacities, scales, rotations, C)     # or cov3D_precomp=...;  FeatureLift.from_state(state)
        for rs, fmap in views:        # fmap [C,Hg,Wg] float32 or float16; (rs.image_height, rs.image_width) == (Hg, Wg)
            lift.add(rs, fmap)
        feats, weight = lift.result(min_weight=0.0, dtype=torch.float32)     # [P,1,C] (semantic_feature layout), [P]

    Any trained 3DGS scene (a plain PLY from io.load_ply included) becomes a feature field in one pass over the views;
    the result can also initialise distillation.  Each `add` is a forward at C = 0 with zero colors_precomp (no SH
    work) and one native lift call (f3dgs_lift_features_accum), which accumulates into `feature_sum` and `weight_sum`:
    the two slices of the single float32 buffer `flat` ([P*C] then [P]), so a data-parallel caller that lifts a share
    of the views on each rank all-reduces `flat` once before `result`.

    Resolution: the map's pixels are the rasterizer's pixels of `rs`.  To lift at a teacher's resolution pass
    `rs._replace(image_height=Hg, image_width=Wg)`: pixel centres then follow the rasterizer's own projection at that
    resolution (pixel x covers [x, x+1) of Wg, the same field of view).  That is deliberately not the relation of the
    training loss, which resizes the W x H render to Hg x Wg with align_corners=True (corner pixel centres on corner
    pixel centres); the two differ by up to half a teacher pixel at the image borders.  There is no autograd.

    A teacher map is usually coarser than the training images, and there the rasterizer's 0.3 px^2 dilation makes
    small Gaussians blend over more of the map than they cover.  antialiasing=True weights with the antialiased
    opacities (AntialiasedGaussianRasterizer), which keep each Gaussian's integral at every resolution."""

    def __init__(self, means3D, opacities, scales=None, rotations=None, C: int = None, cov3D_precomp=None,
                 antialiasing: bool = False):
        if C is None or int(C) < 1 or int(C) > 4096:
            raise ValueError(f"FeatureLift: C must be 1..4096, got {C}")
        if (scales is None or rotations is None) == (cov3D_precomp is None):
            raise ValueError("FeatureLift: provide exactly one of (scales, rotations) / cov3D_precomp")
        if not means3D.is_cuda:
            raise ValueError("FeatureLift: means3D must be a CUDA tensor (there is no CPU path)")
        dev = means3D.device
        self.C, self.P = int(C), int(means3D.shape[0])
        self.antialiasing = bool(antialiasing)
        e = torch.empty(0, device=dev)
        self._geom = dict(means3D=means3D.detach(), opacities=opacities.detach(),
                          scales=e if scales is None else scales.detach(),
                          rotations=e if rotations is None else rotations.detach(),
                          cov3D=e if cov3D_precomp is None else cov3D_precomp.detach())
        self._colors = torch.zeros(self.P, 3, device=dev)
        self._empty = e
        self.flat = torch.zeros(self.P * (self.C + 1), device=dev)
        self.feature_sum = self.flat[: self.P * self.C].view(self.P, 1, self.C)
        self.weight_sum = self.flat[self.P * self.C:]

    @classmethod
    def from_state(cls, state, C: int = None, antialiasing: bool = False):
        """A lift over the Gaussians of a trainer.GaussianState (its activated geometry); C defaults to the state's
        feature width."""
        act = state.activate()
        C = state.raw["semantic_feature"].shape[-1] if C is None else C
        return cls(act["means3D"], act["opacities"], act["scales"], act["rotations"], C, antialiasing=antialiasing)

    def add(self, raster_settings, feature_map: torch.Tensor):
        """Accumulate one view: feature_map [C,H,W] (float32, or float16 read exactly) with (H, W) ==
        (raster_settings.image_height, raster_settings.image_width)."""
        rs = raster_settings
        if not isinstance(feature_map, torch.Tensor) or feature_map.dim() != 3:
            raise ValueError(f"FeatureLift.add: feature_map must be a tensor [C,H,W], got "
                             f"{getattr(feature_map, 'shape', type(feature_map))}")
        if feature_map.dtype not in (torch.float32, torch.float16):
            raise ValueError(f"FeatureLift.add: feature_map must be float32 or float16, got {feature_map.dtype}")
        C, H, W = feature_map.shape
        if C != self.C:
            raise ValueError(f"FeatureLift.add: the lift has C = {self.C} channels, feature_map has {C}")
        if (H, W) != (rs.image_height, rs.image_width):
            raise ValueError(f"FeatureLift.add: feature_map is {H}x{W} (HxW) but the settings render "
                             f"{rs.image_height}x{rs.image_width}; pass rs._replace(image_height={H}, image_width={W})")
        if feature_map.device != self.flat.device:
            raise ValueError(f"FeatureLift.add: feature_map must be on {self.flat.device}, got {feature_map.device}")
        if self.P == 0:
            return
        with torch.no_grad():
            R, geom, binning, img = _weights_forward(self._geom, self._colors, self._empty, self.antialiasing, rs, H, W)
            _C().lift_features_accum(geom, R, binning, img, feature_map, self.feature_sum, self.weight_sum)

    def result(self, min_weight: float = 0.0, dtype=torch.float32):
        """-> (features [P,1,C] of `dtype`, weight_sum [P] float32): feature_sum / weight_sum where weight_sum >
        min_weight, 0 elsewhere (Gaussians no view blended, radii == 0 ones among them)."""
        with torch.no_grad():
            w = self.weight_sum
            keep = w > min_weight
            f = torch.where(keep[:, None, None], self.feature_sum / torch.where(keep, w, 1.0)[:, None, None], 0.0)
            return f.to(dtype), w.clone()
