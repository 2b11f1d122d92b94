"""Vector quantisation of per-row features on the GPU (csrc/vq.cu, include/f3dgs_b200.h f3dgs_vq_*): the k-means
codebook of LightGaussian (NeurIPS 2024) and CompGS (ECCV 2024), which store a trained scene's per-Gaussian features as a
codebook [K, D] plus one code per Gaussian.

  kmeans(x, K)        Lloyd's algorithm: a TF32 tensor-core assignment with the argmin fused into the GEMM (no P x K
                      distance matrix), a code plan (a stable sort by code) and a float64 segment mean per round;
  decode(c, code)     c[code] as float32, or float16 (bitwise c.half()[code]);
  CodePlan(code, K)   the codes with their plan, made once while the codes stay fixed (a fine-tuning run): grad(dL_dx) is
                      the codebook gradient of decode, update(codebook, x) one k-means update.
"""
from typing import Optional, Tuple

import torch


def _check_matrix(x: torch.Tensor, name: str):
    if not isinstance(x, torch.Tensor) or x.dim() != 2 or x.dtype != torch.float32 or not x.is_cuda:
        raise ValueError(f"{name} must be a float32 CUDA tensor [rows, D], got "
                         f"{getattr(x, 'dtype', type(x))} {tuple(getattr(x, 'shape', ()))}")


def _check_weights(weights: Optional[torch.Tensor], P: int, device) -> Optional[torch.Tensor]:
    """weights as a contiguous float32 [P] tensor on `device`; ValueError unless every weight is finite and >= 0 (one host
    read)"""
    if weights is None:
        return None
    w = weights.reshape(-1)
    if w.numel() != P or w.device != device:
        raise ValueError(f"weights must have {P} elements on {device}, got {w.numel()} on {w.device}")
    w = w.float().contiguous()
    if not bool((torch.isfinite(w) & (w >= 0)).all()):
        raise ValueError("weights must be finite and >= 0")
    return w


class CodePlan:
    """The codes [P] (int32, each in [0, K)) and their plan: a stable sort of the rows by code and the segment offsets,
    built once (f3dgs_vq_plan).  While the codes do not change the plan serves every grad() and update().  A code outside
    [0, K) is detected on the device: grad() then returns an unwritten tensor and update() leaves the codebook as it is
    (no host read is made to find out)."""

    def __init__(self, code: torch.Tensor, K: int):
        from . import _C

        if code.dtype != torch.int32 or code.dim() != 1 or not code.is_cuda:
            raise ValueError(f"code must be a 1-D int32 CUDA tensor, got {code.dtype} {tuple(code.shape)}")
        self.code, self.K = code.contiguous(), int(K)
        self.scratch = _C.vq_plan(self.code, self.K)

    @property
    def P(self) -> int:
        return self.code.shape[0]

    def grad(self, dL_dx: torch.Tensor) -> torch.Tensor:
        """dL/dcodebook [K, D] of x = codebook[code]: the sum of dL_dx [P, D] over the rows of each code, in float64 and
        rounded once (0 for an empty code)."""
        from . import _C

        return _C.vq_codebook_grad(dL_dx.reshape(self.P, -1), self.scratch, self.K)

    def update(self, codebook: torch.Tensor, x: torch.Tensor, weights: Optional[torch.Tensor] = None) -> torch.Tensor:
        """One k-means update, in place: codebook[k] = sum w_i x_i / sum w_i over the rows of code k (float64 sums,
        rounded once; weights default to ones and must be finite and >= 0, checked on the device: otherwise nothing is
        written).  A code with zero total weight keeps its row bitwise.  Returns codebook."""
        from . import _C

        _C.vq_update(x.reshape(self.P, -1), weights, self.scratch, codebook)
        return codebook


def assign(x: torch.Tensor, codebook: torch.Tensor) -> torch.Tensor:
    """code[i] = argmin_k ||x_i - c_k||^2 as int32 [P] (f3dgs_vq_assign: TF32 products, ties to the lower index; the
    header states the error bound)."""
    from . import _C

    return _C.vq_assign(x, codebook)


def kmeans(x: torch.Tensor, K: int, iters: int = 10, weights: Optional[torch.Tensor] = None,
           generator: Optional[torch.Generator] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """k-means of the rows of x [P, D] (float32 CUDA) -> (codebook [K, D] float32, code [P] int32).

    The initial codebook is x[torch.randperm(P, generator=generator)[:K]] (randperm on the generator's device, CPU
    without one).  Then `iters` rounds of assign, plan and update (CodePlan.update, with `weights` [P], e.g.
    GaussianScores.weight_sum to follow what renders), and a final assign, so the codes are those of the returned
    codebook.  No host read inside the loop; equal inputs and generator state give bitwise-equal results, so data-parallel
    ranks that fit from the same state stay identical.  ValueError for K > P, K outside [1, 65536], or weights that are
    not finite and >= 0."""
    from . import _C

    _check_matrix(x, "x")
    P = x.shape[0]
    if not 1 <= K <= 65536:
        raise ValueError(f"K must be in [1, 65536], got {K}")
    if K > P:
        raise ValueError(f"K = {K} codes need at least as many rows, got P = {P}")
    x = x.contiguous()
    w = _check_weights(weights, P, x.device)
    dev = generator.device if generator is not None else "cpu"
    first = torch.randperm(P, generator=generator, device=dev)[:K].to(x.device)
    codebook = x[first].contiguous()
    for _ in range(iters):
        code = _C.vq_assign(x, codebook)
        CodePlan(code, K).update(codebook, x, w)
    return codebook, _C.vq_assign(x, codebook)


def decode(codebook: torch.Tensor, code: torch.Tensor, dtype: torch.dtype = torch.float32,
           out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """codebook[code] -> [P, D] of `dtype`: float32, or float16 rounded to nearest even (bitwise codebook.half()[code]).
    A bandwidth-bound gather (f3dgs_vq_decode / _f16out); a code outside [0, K) decodes to a NaN row.  out (optional): a
    contiguous tensor of P D elements of `dtype`, written instead of a new one."""
    from . import _C

    if dtype not in (torch.float32, torch.float16):
        raise ValueError(f"dtype must be torch.float32 or torch.float16, got {dtype}")
    return _C.vq_decode(codebook, code, dtype == torch.float16, out)
