"""The learner targets of env-major fp32 rollouts [N, T] on the device, each in one kernel launch on the caller's
current stream (include/ktb200.h):
  gae     ktb_gae_f32: PPO's advantages and λ-returns, bit for bit CleanRL's per-step torch loop
          (tests/policy_gae_cases.py);
  vtrace  ktb_vtrace_f32: IMPALA's V-trace targets and policy-gradient advantages, bit for bit TorchBeast's
          from_importance_weights made env-major (tests/policy_vtrace_cases.py);
  nstep   ktb_nstep_f32: Ape-X's, R2D2's and A3C's n-step bootstrapped returns and their TD errors, bit for bit rlax's
          n_step_bootstrapped_returns at lambda_t = 1 made env-major (tests/policy_nstep_cases.py);
  retrace ktb_retrace_f32: Retrace(λ), the off-policy Q-value targets of ACER, Reactor, MPO and Q(λ), and their TD
          errors, bit for bit rlax's retrace_continuous made env-major (tests/policy_retrace_cases.py)."""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

from ..mapped import check_finite, check_threshold
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


def _fp32(v) -> float:
    return torch.tensor(float(v), dtype=torch.float32).item()


def vtrace_scalars(gamma, lam, rho_bar, c_bar, pg_rho_bar) -> Tuple[float, float, float, float, float]:
    """(gamma, lam, rho_bar, c_bar, pg_rho_bar) as the fp32 values ktb_vtrace_f32 takes, each rounded as torch rounds a
    Python scalar that meets an fp32 tensor, a threshold of None as +inf (no clip); ValueError naming the first bad
    argument: gamma and lam must be finite numbers, finite in float32, and each threshold a number > 0 in float32."""
    check_finite("gamma", gamma)
    check_finite("lam", lam)
    out = []
    for name, v in (("gamma", gamma), ("lam", lam)):
        out.append(_fp32(v))
        if not math.isfinite(out[-1]):
            raise ValueError(f"{name}={v!r} must be finite in float32")
    for name, v in (("rho_bar", rho_bar), ("c_bar", c_bar), ("pg_rho_bar", pg_rho_bar)):
        check_threshold(name, v)
        out.append(math.inf if v is None else _fp32(v))
        if not out[-1] > 0:
            raise ValueError(f"{name}={v!r} must be > 0 in float32")
    return tuple(out)


def vtrace(log_rhos: torch.Tensor, rewards: torch.Tensor, values: torch.Tensor, dones: torch.Tensor,
           bootstrap_value: torch.Tensor, gamma, lam=1.0, rho_bar=1.0, c_bar=1.0, pg_rho_bar=1.0,
           vs: Optional[torch.Tensor] = None, pg_adv: Optional[torch.Tensor] = None,
           stream: Optional[torch.cuda.Stream] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(vs, pg_advantages) of env-major rollouts: log_rhos (target less behaviour log-probabilities of the taken
    actions), rewards, values and dones fp32 [N, T] (row i is environment i's trajectory; dones[i, t] = 1 when the
    episode ended after the action at step t), bootstrap_value fp32 [N] = V(s_T).  rho_bar, c_bar and pg_rho_bar clip
    ρ in the TD errors, the traces and the policy gradient (None: no clip); lam is seed_rl's lambda_.  Every tensor is
    contiguous and on one CUDA device.  vs and pg_adv are fresh fp32 [N, T] tensors unless given; given ones must not
    overlap the inputs or each other.  Enqueued on `stream` (default: the current stream of that device)."""
    if not isinstance(rewards, torch.Tensor) or rewards.dim() != 2:
        raise ValueError(f"rewards must be a 2-D [N, T] tensor, got "
                         f"{list(rewards.shape) if isinstance(rewards, torch.Tensor) else type(rewards).__name__}")
    shape, device = tuple(rewards.shape), rewards.device
    _check("rewards", rewards, shape, device)
    _check("log_rhos", log_rhos, shape, device)
    _check("values", values, shape, device)
    _check("dones", dones, shape, device)
    _check("bootstrap_value", bootstrap_value, shape[:1], device)
    scalars = vtrace_scalars(gamma, lam, rho_bar, c_bar, pg_rho_bar)
    vs = torch.empty(shape, dtype=torch.float32, device=device) if vs is None else vs
    pg_adv = torch.empty(shape, dtype=torch.float32, device=device) if pg_adv is None else pg_adv
    _check("vs", vs, shape, device)
    _check("pg_adv", pg_adv, shape, device)
    dev = device.index
    ops.ensure_init([dev])
    L.call("ktb_vtrace_f32", dev, log_rhos.data_ptr(), rewards.data_ptr(), values.data_ptr(), dones.data_ptr(),
           bootstrap_value.data_ptr(), shape[0], shape[1], *scalars, vs.data_ptr(), pg_adv.data_ptr(),
           ops._stream(dev, stream))
    return vs, pg_adv


def nstep_scalars(n, gamma) -> Tuple[int, float]:
    """(n, gamma) as ktb_nstep_f32 takes them: n an int (not a bool) in [1, 32], gamma rounded to fp32 as torch rounds
    a Python scalar that meets an fp32 tensor; ValueError naming the first bad argument: gamma must be a finite number,
    finite in float32."""
    if isinstance(n, bool) or not isinstance(n, int) or not 1 <= n <= 32:
        raise ValueError(f"n must be an int in [1, 32], got {n!r}")
    check_finite("gamma", gamma)
    g = _fp32(gamma)
    if not math.isfinite(g):
        raise ValueError(f"gamma={gamma!r} must be finite in float32")
    return n, g


def nstep(rewards: torch.Tensor, values: torch.Tensor, dones: torch.Tensor, baseline: torch.Tensor,
          last_values: torch.Tensor, n, gamma, ret: Optional[torch.Tensor] = None, td: Optional[torch.Tensor] = None,
          stream: Optional[torch.cuda.Stream] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(returns, td_errors) of env-major rollouts: the n-step bootstrapped returns G_t = r_t + γ r_{t+1} + … +
    γ^{n−1} r_{t+n−1} + γ^n values[:, t + n], cut at episode ends and bootstrapped from last_values past the rollout's
    end, and G_t − baseline[:, t].  rewards, values (the bootstrap value of each state), dones (dones[i, t] = 1 when the
    episode ended after the action at step t) and baseline (Q(s_t, a_t), or values for A3C) are fp32 [N, T];
    last_values fp32 [N] = V(s_T).  Every tensor is contiguous and on one CUDA device; inputs may alias one another.
    ret and td are fresh fp32 [N, T] tensors unless given; given ones must not overlap the inputs or each other.
    Enqueued on `stream` (default: the current stream of that device)."""
    if not isinstance(rewards, torch.Tensor) or rewards.dim() != 2:
        raise ValueError(f"rewards must be a 2-D [N, T] tensor, got "
                         f"{list(rewards.shape) if isinstance(rewards, torch.Tensor) else type(rewards).__name__}")
    shape, device = tuple(rewards.shape), rewards.device
    _check("rewards", rewards, shape, device)
    _check("values", values, shape, device)
    _check("dones", dones, shape, device)
    _check("baseline", baseline, shape, device)
    _check("last_values", last_values, shape[:1], device)
    n, g = nstep_scalars(n, gamma)
    ret = torch.empty(shape, dtype=torch.float32, device=device) if ret is None else ret
    td = torch.empty(shape, dtype=torch.float32, device=device) if td is None else td
    _check("ret", ret, shape, device)
    _check("td", td, shape, device)
    dev = device.index
    ops.ensure_init([dev])
    L.call("ktb_nstep_f32", dev, rewards.data_ptr(), values.data_ptr(), dones.data_ptr(), baseline.data_ptr(),
           last_values.data_ptr(), shape[0], shape[1], n, g, ret.data_ptr(), td.data_ptr(), ops._stream(dev, stream))
    return ret, td


def retrace_scalars(gamma, lam) -> Tuple[float, float]:
    """(gamma, lam) as the fp32 values ktb_retrace_f32 takes, each rounded as torch rounds a Python scalar that meets an
    fp32 tensor; ValueError naming the first bad argument: each must be a finite number, finite in float32."""
    out = []
    for name, v in (("gamma", gamma), ("lam", lam)):
        out.append(_fp32(check_finite(name, v)))
        if not math.isfinite(out[-1]):
            raise ValueError(f"{name}={v!r} must be finite in float32")
    return tuple(out)


def retrace(log_rhos: torch.Tensor, rewards: torch.Tensor, q: torch.Tensor, values: torch.Tensor, dones: torch.Tensor,
            baseline: torch.Tensor, bootstrap_value: torch.Tensor, gamma, lam, ret: Optional[torch.Tensor] = None,
            td: Optional[torch.Tensor] = None,
            stream: Optional[torch.cuda.Stream] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(returns, td_errors) of env-major rollouts under Retrace(λ): G_t = r_t + γ(1 − d_t)·(values[:, t + 1] −
    c_{t+1}·q[:, t + 1] + c_{t+1}·G_{t+1}) with traces c = λ·min(1, exp(log_rhos)), bootstrapped from bootstrap_value at
    the rollout's end, and G_t − baseline[:, t].  log_rhos (target less behaviour log-probabilities of the taken
    actions), rewards, q (Q_target(s_t, a_t)), values (E_π Q_target(s_t, ·)), dones (dones[i, t] = 1 when the episode
    ended after the action at step t) and baseline (Q_online(s_t, a_t), or q itself) are fp32 [N, T]; bootstrap_value
    fp32 [N] = E_π Q_target(s_T, ·).  Columns 0 of log_rhos, q and values are not read.  Every tensor is contiguous and
    on one CUDA device; inputs may alias one another.  ret and td are fresh fp32 [N, T] tensors unless given; given ones
    must not overlap the inputs or each other.  Enqueued on `stream` (default: the current stream of that device)."""
    if not isinstance(rewards, torch.Tensor) or rewards.dim() != 2:
        raise ValueError(f"rewards must be a 2-D [N, T] tensor, got "
                         f"{list(rewards.shape) if isinstance(rewards, torch.Tensor) else type(rewards).__name__}")
    shape, device = tuple(rewards.shape), rewards.device
    _check("rewards", rewards, shape, device)
    _check("log_rhos", log_rhos, shape, device)
    _check("q", q, shape, device)
    _check("values", values, shape, device)
    _check("dones", dones, shape, device)
    _check("baseline", baseline, shape, device)
    _check("bootstrap_value", bootstrap_value, shape[:1], device)
    g, lm = retrace_scalars(gamma, lam)
    ret = torch.empty(shape, dtype=torch.float32, device=device) if ret is None else ret
    td = torch.empty(shape, dtype=torch.float32, device=device) if td is None else td
    _check("ret", ret, shape, device)
    _check("td", td, shape, device)
    dev = device.index
    ops.ensure_init([dev])
    L.call("ktb_retrace_f32", dev, log_rhos.data_ptr(), rewards.data_ptr(), q.data_ptr(), values.data_ptr(),
           dones.data_ptr(), baseline.data_ptr(), bootstrap_value.data_ptr(), shape[0], shape[1], g, lm, ret.data_ptr(),
           td.data_ptr(), ops._stream(dev, stream))
    return ret, td
