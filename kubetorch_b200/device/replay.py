"""Prioritized experience replay on the device, the proportional sampler of Ape-X, R2D2 and Rainbow, each call one C
entry on the caller's current stream (include/ktb200.h):
  per_sample  ktb_per_sample_f32: the sum tree of a priority vector, stratified draws from it and their importance
              weights, bit for bit the torch body of tests/policy_per_cases.py on the GPU;
  per_update  ktb_per_update_f32: the new priorities (|td| + eps)^alpha written in place, a repeated index taking its
              last occurrence, deterministically."""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

from ..mapped import check_beta, check_finite
from ..sampling import _check_seed
from . import lib as L
from . import ops

MAX_BATCH = 8192
MAX_CAPACITY = 1 << 30
# The exponents at which torch's pow of an fp32 CUDA tensor leaves powf for sqrt, rsqrt, a reciprocal or multiplies,
# chosen on the exponent's double value (include/ktb200.h); 0 is not here: powf(x, 0) is 1 as ATen's fill is
_POW_SPECIAL = (1.0, 0.5, -0.5, -1.0, 2.0, 3.0, -2.0)


def _fp32(v) -> float:
    return torch.tensor(float(v), dtype=torch.float32).item()


def per_scalars(**scalars) -> Tuple[float, ...]:
    """The given beta, alpha and eps (keyword arguments, in their order) as the fp32 values the C entries take, each
    rounded as torch rounds a Python scalar that meets an fp32 tensor.  ValueError naming the first bad one: each must
    be a finite number, finite in float32, beta >= 0; and an exponent (beta is one as -beta) whose fp32 rounding is
    one of the exponents torch's pow computes another way must be exactly that value, since torch chooses the way from
    the double and the kernel from the fp32 rounding."""
    out = []
    for name, v in scalars.items():
        if name not in ("beta", "alpha", "eps"):
            raise TypeError(f"per_scalars() got an unexpected keyword argument {name!r}")
        check_beta(v) if name == "beta" else check_finite(name, v)
        f = _fp32(v)
        if not math.isfinite(f):
            raise ValueError(f"{name}={v!r} must be finite in float32")
        exponent = -f if name == "beta" else f
        if name != "eps" and exponent in _POW_SPECIAL and float(v) != f:
            raise ValueError(f"{name}={v!r} rounds to {f!r} in float32, where torch's pow takes a special path only "
                             f"for exactly {f!r}: pass {f!r}")
        out.append(f)
    return tuple(out)


def _check(name: str, t, dtype, shape, device) -> None:
    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{name} must be a torch.Tensor, got {type(t).__name__}")
    if t.dtype != dtype:
        raise ValueError(f"{name} must be {str(dtype).replace('torch.', '')}, got {t.dtype}")
    if tuple(t.shape) != shape:
        raise ValueError(f"{name} must have shape {list(shape)}, got {list(t.shape)}")
    if not t.is_cuda or t.device != device:
        raise ValueError(f"{name} must be a CUDA tensor on the device of priorities ({device}), got {t.device}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")


def _priorities(priorities) -> Tuple[int, torch.device]:
    if not isinstance(priorities, torch.Tensor) or priorities.dim() != 1:
        raise ValueError(f"priorities must be a 1-D [C] tensor, got "
                         f"{list(priorities.shape) if isinstance(priorities, torch.Tensor) else type(priorities).__name__}")
    c, device = priorities.numel(), priorities.device
    _check("priorities", priorities, torch.float32, (c,), device)
    if not 1 <= c <= MAX_CAPACITY:
        raise ValueError(f"priorities must hold 1 to 2**30 items, got {c}")
    return c, device


def tree_size(capacity: int) -> int:
    """The fp32 scratch words of per_sample's tree for `capacity` priorities: the least power of two >= capacity, and
    at least 2."""
    return max(2, 1 << (capacity - 1).bit_length())


def per_sample(priorities: torch.Tensor, batch: int, seed: int, beta, j0: int = 0, rows: Optional[int] = None,
               tree: Optional[torch.Tensor] = None, indices: Optional[torch.Tensor] = None,
               weights: Optional[torch.Tensor] = None,
               stream: Optional[torch.cuda.Stream] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(indices, weights) of strata j0 .. j0 + rows - 1 (rows: all of them from j0 by default) of a stratified draw of
    `batch` from the fp32 [C] priorities p_i^α, in proportion to them: stratum j lands at mass (j + u_j)·(total / batch)
    of the sum tree, u_j = kubetorch_b200.sampling.replay_noise(seed, j, 1), and its importance weight is (C·p_i /
    total)^-β over the largest such weight, (C·min p / total)^-β.  int64 indices [rows] in [0, C) whatever the
    priorities hold, fp32 weights [rows].  batch is an int in [1, 8192], seed an int in [0, 2**64), beta a number >= 0.
    tree is fp32 [tree_size(C)] scratch, left holding the min, the total and the internal nodes (include/ktb200.h);
    tree, indices and weights are fresh tensors unless given, and given ones must not overlap priorities or each other.
    Every tensor is contiguous and on one CUDA device.  Enqueued on `stream` (default: the current stream of that
    device)."""
    c, device = _priorities(priorities)
    if isinstance(batch, bool) or not isinstance(batch, int) or not 1 <= batch <= MAX_BATCH:
        raise ValueError(f"batch must be an int in [1, {MAX_BATCH}], got {batch!r}")
    seed = _check_seed(seed)
    rows = batch - j0 if rows is None else rows
    if any(isinstance(v, bool) or not isinstance(v, int) for v in (j0, rows)) or j0 < 0 or rows < 0 \
            or j0 + rows > batch:
        raise ValueError(f"j0={j0!r} and rows={rows!r} must be ints with 0 <= j0 and j0 + rows <= batch={batch}")
    b, = per_scalars(beta=beta)
    tree = torch.empty(tree_size(c), dtype=torch.float32, device=device) if tree is None else tree
    indices = torch.empty(rows, dtype=torch.int64, device=device) if indices is None else indices
    weights = torch.empty(rows, dtype=torch.float32, device=device) if weights is None else weights
    _check("tree", tree, torch.float32, (tree_size(c),), device)
    _check("indices", indices, torch.int64, (rows,), device)
    _check("weights", weights, torch.float32, (rows,), device)
    if rows:
        dev = device.index
        ops.ensure_init([dev])
        L.call("ktb_per_sample_f32", dev, priorities.data_ptr(), c, batch, j0, rows, seed, b, tree.data_ptr(),
               indices.data_ptr(), weights.data_ptr(), ops._stream(dev, stream))
    return indices, weights


def per_update(priorities: torch.Tensor, indices: torch.Tensor, td: torch.Tensor, alpha, eps=1e-6,
               stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
    """priorities[indices] = (|td| + eps)^alpha in place, as torch computes it on the GPU, where a repeated index takes
    its LAST occurrence (deterministic, unlike `priorities[indices] = new` on CUDA).  An index outside [0, C) is
    skipped.  priorities fp32 [C], indices int64 [B] and td fp32 [B] (B <= 8192; 0 does nothing), contiguous, on one
    CUDA device; indices and td must not overlap priorities.  alpha and eps are finite numbers.  Enqueued on `stream`
    (default: the current stream of that device).  Returns priorities."""
    c, device = _priorities(priorities)
    if not isinstance(indices, torch.Tensor) or indices.dim() != 1:
        raise ValueError("indices must be a 1-D [B] tensor")
    n = indices.numel()
    _check("indices", indices, torch.int64, (n,), device)
    _check("td", td, torch.float32, (n,), device)
    if n > MAX_BATCH:
        raise ValueError(f"indices must hold at most {MAX_BATCH} items, got {n}")
    a, e = per_scalars(alpha=alpha, eps=eps)
    if n:
        dev = device.index
        ops.ensure_init([dev])
        L.call("ktb_per_update_f32", dev, priorities.data_ptr(), c, indices.data_ptr(), td.data_ptr(), n, a, e,
               ops._stream(dev, stream))
    return priorities
