"""View-batch data parallelism for the rasterizer (additive to the reference API; the reference has no
multi-GPU path at all -- SURVEY.md section 2 "Parallelism strategies: none").

The path shards by *views*: every rank holds a full replica of the Gaussian parameters, renders its slice
of the step's camera batch (forward + backward), and the per-rank gradients -- accumulated over the local
views in ONE flat fp32 buffer -- are summed with a single all-reduce per step
(NCCL over NVLink 5 / NVSwitch on the GPU box; gloo in the CPU tests).  No collective sits on the
per-view data path.

    flat = FlatGradBuffer([means3D, scales, rotations, opacities, shs, features])   # .grad are views
    for v in shard_views(n_views, rank, world):
        render(v) -> loss.backward()          # autograd accumulates in place into the flat buffer
    flat.all_reduce()                         # exactly one collective per step

`ViewBatch` is the faster, autograd-free form of the same loop: the forward is `_C.rasterize_gaussians`, the user
computes dL/d(color, feature_map, depth) of one view, and `ViewBatch.backward` has the backward kernels ADD that view's
gradients straight into the flat buffer (`f3dgs_backward_accum`): no per-view zero-filled gradient tensors, no autograd
additions, densification statistics folded in.  The step's collective is issued in two buckets: the feature /
opacity slice, final after the last view's composite kernel, is reduced on a side stream while the last view's backward
preprocess still runs.
"""
from typing import Iterable, List, NamedTuple, Optional, Sequence

import torch
import torch.distributed as dist


def shard_views(n_views: int, rank: int, world_size: int) -> List[int]:
    """Round-robin assignment of view indices to ranks (rank r renders r, r+G, r+2G, ...)."""
    if not (0 <= rank < world_size):
        raise ValueError(f"rank {rank} outside world of size {world_size}")
    return list(range(rank, n_views, world_size))


class FlatGradBuffer:
    """One contiguous fp32 gradient buffer whose slices are the `.grad` of every parameter."""

    def __init__(self, params: Sequence[torch.Tensor], extra: int = 0):
        params = list(params)
        if not params:
            raise ValueError("no parameters")
        dev, dt = params[0].device, params[0].dtype
        for p in params:
            if p.device != dev or p.dtype != dt or not p.is_leaf or not p.requires_grad:
                raise ValueError("parameters must be leaf tensors requiring grad on one device with one dtype")
        self.params = params
        self.sizes = [p.numel() for p in params]
        self.offsets = [0]
        for n in self.sizes:
            self.offsets.append(self.offsets[-1] + n)
        # `extra` trailing floats for step statistics that ride in the same collective
        self.flat = torch.zeros(self.offsets[-1] + extra, device=dev, dtype=dt)
        for p, o, n in zip(params, self.offsets, self.sizes):
            p.grad = self.flat[o:o + n].view_as(p)

    @property
    def extra(self) -> torch.Tensor:
        return self.flat[self.offsets[-1]:]

    def zero_(self):
        self.flat.zero_()

    def check_views(self):
        """The .grad tensors must still alias the flat buffer (autograd accumulates in place)."""
        base = self.flat.data_ptr()
        for p, o in zip(self.params, self.offsets):
            if p.grad is None or p.grad.data_ptr() != base + o * self.flat.element_size():
                raise RuntimeError("a parameter's .grad no longer aliases the flat gradient buffer")

    def all_reduce(self, group: Optional[dist.ProcessGroup] = None, average: bool = False):
        """The single collective of a step.  No-op without an initialised process group."""
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group)
            if average:
                self.flat.div_(dist.get_world_size(group))
        return self.flat




class CameraGrad(NamedTuple):
    """One view's camera gradient (ViewBatch.backward(..., camera=True)): views of one 35-float buffer, each in the
    layout of the settings tensor it belongs to."""
    viewmatrix: torch.Tensor  # [4, 4]
    projmatrix: torch.Tensor  # [4, 4]
    campos: torch.Tensor  # [3]


class _ViewCtx:
    __slots__ = ("rs", "num_rendered", "radii", "geom", "binning", "img", "inputs", "antialiasing")


class ViewBatch:
    """Autograd-free view-batch rendering with in-kernel gradient accumulation (additive API).

        vb = ViewBatch(dict(means3D=..., scales=..., rotations=..., opacities=..., shs=..., semantic_feature=...))
        vb.zero_()
        for settings in local_views:
            color, feat, radii, depth, ctx = vb.forward(settings)
            g_color, g_feat, g_depth = my_loss_gradients(color, feat, depth)
            vb.backward(ctx, g_color, g_feat, g_depth)
        vb.all_reduce()              # gradients: vb.grads[name] (views of vb.flat.flat); stats: vb.grad_accum, vb.denom

    Parameter order inside the flat buffer: the feature and opacity gradients come first -- they are complete as soon as
    the last view's backward composite has run, so their bucket of the all-reduce overlaps the last backward preprocess.

    `semantic_feature` may be float16 (a float16 feature field): the forward then renders a float16 map, and the
    feature gradient still accumulates in float32, in a slot of the same shape.
    """

    ORDER = ("semantic_feature", "opacities", "means3D", "shs", "scales", "rotations")

    def __init__(self, params: dict, densify_stats: bool = True):
        from . import _C  # deferred: this module must stay importable without the extension (bench reference arm)

        self._C = _C
        self.names = [k for k in self.ORDER if params.get(k) is not None and params[k].numel() > 0]
        self.params = {k: params[k] for k in self.names}
        P = params["means3D"].shape[0]
        dev = params["means3D"].device
        self.P = P
        sizes = [self.params[k].numel() for k in self.names]
        extra = 2 * P if densify_stats else 0
        # every view starts on a 16-byte boundary: the backward and the optimizer move the rotation gradient as float4,
        # and P, which sets the offsets, is arbitrary once densification has run
        offs, o = [], 0
        for n in sizes:
            offs.append(o)
            o += -(-n // 4) * 4
        self.flat = torch.zeros(o + extra, device=dev, dtype=torch.float32)
        self.grads = {k: self.flat[s:s + n].view_as(self.params[k]) for k, s, n in zip(self.names, offs, sizes)}
        self.n_param = o
        self.early = next((s for k, s in zip(self.names, offs) if k not in ("semantic_feature", "opacities")), o)
        self.grad_accum = self.flat[o:o + P] if densify_stats else None
        self.denom = self.flat[o + P:o + 2 * P] if densify_stats else None
        self.scratch = torch.empty(int(_C.backward_scratch_bytes(P)), dtype=torch.uint8, device=dev)
        self._empty = torch.empty(0, device=dev)
        self._side = torch.cuda.Stream(device=dev) if dev.type == "cuda" else None
        self._ev = None
        if self._side is not None:
            self._ev = torch.cuda.Event()
            self._ev.record()  # materialises the cudaEvent_t handle
        self._early_pending = False

    def zero_(self):
        self.flat.zero_()

    def visible(self) -> torch.Tensor:
        """bool [P]: the Gaussians with radii > 0 in at least one view of the step (denom > 0), the rows outside which
        every gradient slot is exactly zero.  After all_reduce() it is the union over every rank's views, the same on
        every rank: the mask of GaussianState.step(lrs, visible=...).  Needs densify_stats=True."""
        if self.denom is None:
            raise RuntimeError("ViewBatch.visible() needs the densification statistics (densify_stats=True)")
        return self.denom > 0

    def forward(self, rs, antialiasing: bool = False):
        """One view's forward (no autograd graph).  `rs` is a GaussianRasterizationSettings.  antialiasing=True renders
        with the antialiased opacities (AntialiasedGaussianRasterizer); the returned ctx remembers it, so that
        `backward` differentiates the same model."""
        fn = self._C.rasterize_gaussians_antialiased if antialiasing else self._C.rasterize_gaussians
        (color, feat, depth), ctx = self._forward(fn, rs, antialiasing)
        return color, feat, ctx.radii, depth, ctx

    def forward_alpha_invdepth(self, rs, antialiasing: bool = False):
        """forward() that also renders the opacity plane alpha = 1 - T_final and the inverse-depth plane
        invdepth = sum_i w_i / z_i ([1,H,W] float32 each; AlphaInvDepthGaussianRasterizer) ->
        (color, feat, radii, depth, alpha, invdepth, ctx).  Their gradients go to backward(..., g_alpha=, g_invdepth=)."""
        fn = lambda *args: self._C.rasterize_gaussians_alpha_invdepth(*args, antialiasing=antialiasing)  # noqa: E731
        (color, feat, depth, alpha, invdepth), ctx = self._forward(fn, rs, antialiasing)
        return color, feat, ctx.radii, depth, alpha, invdepth, ctx

    def _forward(self, fn, rs, antialiasing):
        """The native forward `fn` of one view -> (its images, the view's ctx)"""
        p = self.params
        e = torch.Tensor([])
        sf = p.get("semantic_feature", self._empty)
        out = fn(rs.bg, p["means3D"], e, sf, p["opacities"], p["scales"], p["rotations"], rs.scale_modifier, e,
                 rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width, p["shs"],
                 rs.sh_degree, rs.campos, rs.prefiltered, rs.debug)
        ctx = _ViewCtx()
        ctx.rs = rs
        ctx.antialiasing = bool(antialiasing)
        ctx.num_rendered, *images, ctx.radii, ctx.geom, ctx.binning, ctx.img = out
        return images, ctx

    def backward(self, ctx, g_color, g_feature, g_depth, means2D_out=None, last: bool = False, camera: bool = False,
                 feature_geometry: bool = False, g_alpha=None, g_invdepth=None):
        """Add this view's parameter gradients into the flat buffer.  `last=True` on the rank's last view of the step
        lets all_reduce() start the feature/opacity bucket early.  g_feature: dL/dfeature_map as a float32 or float16
        [C,H,W] tensor, a feature_head.ScaledGrad (a float16 map and its float32 scale), or None.

        camera=True also returns this view's CameraGrad (dL/dviewmatrix, dL/dprojmatrix, dL/dcampos of its settings,
        f3dgs_backward_accum_cam); the flat buffer and the densification statistics are bitwise those of camera=False.
        A camera gradient belongs to its view and stays on the rank that rendered it: all_reduce() does not touch it.

        feature_geometry=True also feeds g_feature into dL/dalpha, so that the feature loss reaches the opacities, means,
        scales, rotations, the densification statistics and the camera gradient (f3dgs_backward_accum_feature_geometry,
        which reads the batch's semantic_feature).

        A view rendered by forward(rs, antialiasing=True) is differentiated in that mode
        (f3dgs_backward_accum_antialiased); its opacity gradient is final only after the backward preprocess, so the
        early bucket of a `last=True` view then starts after it.

        g_alpha / g_invdepth: dL/dalpha and dL/dinvdepth [1,H,W] float32 of forward_alpha_invdepth's planes
        (f3dgs_backward_accum_alpha_invdepth; one given alone: the other is zero).  The buffers of either forward take
        them, and they combine with camera, feature_geometry and a ScaledGrad g_feature; with both None the call is the
        one without them."""
        rs, p, g, e = ctx.rs, self.params, self.grads, torch.Tensor([])
        none = self._empty
        scale = 1.0
        if isinstance(g_feature, tuple):  # ScaledGrad (not imported: this module loads without the package)
            g_feature, scale = g_feature
        cam = torch.zeros(35, device=self.flat.device, dtype=torch.float32) if camera else None
        self._C.rasterize_gaussians_backward_accum(
            rs.bg, p["means3D"], ctx.radii, e, p["scales"], p["rotations"], rs.scale_modifier, e, rs.viewmatrix,
            rs.projmatrix, rs.tanfovx, rs.tanfovy, g_color, g_feature if g_feature is not None else none, g_depth,
            p["shs"], rs.sh_degree, rs.campos, ctx.geom, ctx.num_rendered, ctx.binning, ctx.img, self.scratch,
            g["means3D"], g["shs"], none, g.get("semantic_feature", none), g["opacities"], g["scales"], g["rotations"],
            none, means2D_out if means2D_out is not None else none,
            self.grad_accum if self.grad_accum is not None else none, self.denom if self.denom is not None else none,
            int(self._ev.cuda_event) if (last and self._ev is not None) else 0, rs.debug, float(scale), cam,
            p.get("semantic_feature") if feature_geometry else None, ctx.antialiasing, g_alpha, g_invdepth)
        self._early_pending = bool(last and self._ev is not None)
        if cam is not None:
            return CameraGrad(cam[:16].view(4, 4), cam[16:32].view(4, 4), cam[32:35])
        return None

    def all_reduce(self, group: Optional[dist.ProcessGroup] = None):
        """The step's collective (sum over ranks).  After backward(..., last=True): two buckets, the feature/opacity one
        starting on a side stream as soon as the last composite kernel is done; otherwise one call over the buffer."""
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1):
            self._early_pending = False
            return self.flat
        if self._early_pending and 0 < self.early < self.flat.numel():
            main = torch.cuda.current_stream(self.flat.device)
            self._side.wait_event(self._ev)
            with torch.cuda.stream(self._side):
                dist.all_reduce(self.flat[:self.early], op=dist.ReduceOp.SUM, group=group)
            dist.all_reduce(self.flat[self.early:], op=dist.ReduceOp.SUM, group=group)
            main.wait_stream(self._side)
        else:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group)
        self._early_pending = False
        return self.flat
