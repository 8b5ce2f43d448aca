"""Generalized advantage estimation on the device: ktb_gae_f32 (include/ktb200.h) over torch tensors.

The advantages and λ-returns of env-major fp32 rollouts [N, T], bit for bit the per-step torch loop of CleanRL
(tests/policy_gae_cases.py), in one kernel launch on the caller's current stream."""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

from ..mapped import check_finite
from . import lib as L
from . import ops


def _check(name: str, t, shape, device) -> None:
    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{name} must be a torch.Tensor, got {type(t).__name__}")
    if t.dtype != torch.float32:
        raise ValueError(f"{name} must be float32, got {t.dtype}")
    if tuple(t.shape) != shape:
        raise ValueError(f"{name} must have shape {list(shape)}, got {list(t.shape)}")
    if not t.is_cuda or t.device != device:
        raise ValueError(f"{name} must be a CUDA tensor on the device of rewards ({device}), got {t.device}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")


def gae_scalars(gamma, lam) -> Tuple[float, float]:
    """(gamma, gamma_lam) as the fp32 values ktb_gae_f32 takes: fp32(γ) and fp32(γ·λ) with the product taken in double,
    as torch rounds the Python scalars γ and γ * λ when they meet an fp32 tensor; ValueError unless both are finite."""
    check_finite("gamma", gamma)
    check_finite("lam", lam)
    g, gl = (torch.tensor(float(v), dtype=torch.float32).item() for v in (gamma, float(gamma) * float(lam)))
    if not (math.isfinite(g) and math.isfinite(gl)):
        raise ValueError(f"gamma={gamma!r} and gamma * lam={float(gamma) * float(lam)!r} must be finite in float32")
    return g, gl


def gae(rewards: torch.Tensor, values: torch.Tensor, dones: torch.Tensor, last_values: torch.Tensor, gamma, lam,
        adv: Optional[torch.Tensor] = None, ret: Optional[torch.Tensor] = None,
        stream: Optional[torch.cuda.Stream] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(advantages, returns) of env-major rollouts: rewards, values and dones fp32 [N, T] (row i is environment i's
    trajectory; dones[i, t] = 1 when the episode ended after the action at step t), last_values fp32 [N] = V(s_T).
    Every tensor is contiguous and on one CUDA device.  adv and ret are fresh fp32 [N, T] tensors unless given; given
    ones must not overlap the inputs or each other.  Enqueued on `stream` (default: the current stream of that device)."""
    if not isinstance(rewards, torch.Tensor) or rewards.dim() != 2:
        raise ValueError(f"rewards must be a 2-D [N, T] tensor, got "
                         f"{list(rewards.shape) if isinstance(rewards, torch.Tensor) else type(rewards).__name__}")
    shape, device = tuple(rewards.shape), rewards.device
    _check("rewards", rewards, shape, device)
    _check("values", values, shape, device)
    _check("dones", dones, shape, device)
    _check("last_values", last_values, shape[:1], device)
    g, gl = gae_scalars(gamma, lam)
    adv = torch.empty(shape, dtype=torch.float32, device=device) if adv is None else adv
    ret = torch.empty(shape, dtype=torch.float32, device=device) if ret is None else ret
    _check("adv", adv, shape, device)
    _check("ret", ret, shape, device)
    dev = device.index
    ops.ensure_init([dev])
    L.call("ktb_gae_f32", dev, rewards.data_ptr(), values.data_ptr(), dones.data_ptr(), last_values.data_ptr(),
           shape[0], shape[1], g, gl, adv.data_ptr(), ret.data_ptr(), ops._stream(dev, stream))
    return adv, ret
