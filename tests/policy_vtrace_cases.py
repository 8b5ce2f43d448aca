"""User callables of V-trace (IMPALA's off-policy learner target), written as a kubetorch user writes SPMD functions:
rank r takes its `x.chunk(WORLD_SIZE)[RANK]` rows of env-major rollouts (row i is environment i's trajectory, column t
its step t) and runs TorchBeast's from_importance_weights over them.

TEST INFRASTRUCTURE.  vtrace() is the semantic definition of @kt.mapped("vtrace", gamma=GAMMA, ...): TorchBeast's loop
made env-major, with dones[:, t] the done flag of transition t (TorchBeast's batch["done"][1:]), bootstrap_value V(s_T)
and seed_rl's lambda_ as lam.  include/ktb200.h restates it as fp32 operations (header_vtrace below), and the CUDA path
must reproduce its bits.  The oracle restatement (oracle/ref_dispatch.spmd_call) executes the bodies on CPU.
"""
import os

import numpy as np

GAMMA = 0.99


def _shard(t):
    """This rank's rows of t, as obs.chunk(WORLD_SIZE)[RANK] (an empty shard for ranks past the data)."""
    r, w = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    rows = t.chunk(w, dim=0)
    return rows[r] if r < len(rows) else t[:0]


def vtrace(log_rhos, rewards, values, dones, bootstrap_value, gamma, lam=1.0, rho_bar=1.0, c_bar=1.0, pg_rho_bar=1.0):
    import torch

    discounts = gamma * (1.0 - dones)
    rhos = torch.exp(log_rhos)
    clipped_rhos = rhos if rho_bar is None else torch.clamp(rhos, max=rho_bar)
    cs = lam * (rhos if c_bar is None else torch.clamp(rhos, max=c_bar))
    v_next = torch.cat([values[:, 1:], bootstrap_value[:, None]], 1)
    deltas = clipped_rhos * (rewards + discounts * v_next - values)
    acc = torch.zeros_like(bootstrap_value)
    vs_minus_v = torch.empty_like(values)
    for t in reversed(range(values.shape[1])):
        acc = deltas[:, t] + discounts[:, t] * cs[:, t] * acc
        vs_minus_v[:, t] = acc
    vs = vs_minus_v + values
    vs_next = torch.cat([vs[:, 1:], bootstrap_value[:, None]], 1)
    pg_rhos = rhos if pg_rho_bar is None else torch.clamp(rhos, max=pg_rho_bar)
    return vs, pg_rhos * (rewards + discounts * vs_next - values)


def _shards(*xs):
    return tuple(_shard(t) for t in xs)


def mapped_vtrace(log_rhos, rewards, values, dones, bootstrap_value):
    """@kt.mapped("vtrace", gamma=GAMMA): TorchBeast's defaults, λ = 1 and every threshold 1."""
    return vtrace(*_shards(log_rhos, rewards, values, dones, bootstrap_value), GAMMA)


def mapped_vtrace_args(log_rhos, rewards, values, dones, bootstrap_value, gamma, lam):
    """gamma and lam as call arguments: @kt.mapped("vtrace", gamma="gamma", lam="lam")."""
    return vtrace(*_shards(log_rhos, rewards, values, dones, bootstrap_value), gamma, lam)


def mapped_vtrace_shifted(log_rhos, rewards, values, dones, bootstrap_value):
    """A body that reads episode-start flags: dones[:, t + 1] as step t's flag (CleanRL's and TorchBeast's unshifted
    batch["done"]) and the last step as nonterminal.  Not the op's body: the deployment's self-check refuses it."""
    import torch

    log_rhos, rewards, values, dones, bootstrap_value = _shards(log_rhos, rewards, values, dones, bootstrap_value)
    shifted = torch.cat([dones[:, 1:], torch.zeros_like(dones[:, :1])], 1)
    return vtrace(log_rhos, rewards, values, shifted, bootstrap_value, GAMMA)


def mapped_vtrace_other_gamma(log_rhos, rewards, values, dones, bootstrap_value):
    """The body with γ = 0.98: not what a deployment declaring gamma=GAMMA computes."""
    return vtrace(*_shards(log_rhos, rewards, values, dones, bootstrap_value), 0.98)


def mapped_vtrace_fixed_c(log_rhos, rewards, values, dones, bootstrap_value):
    """TorchBeast's hardcoded c̄ = 1: cs is clamped at 1.0 whatever c_bar a deployment declares, so a deployment with
    c_bar=0.9 does not compute it."""
    return vtrace(*_shards(log_rhos, rewards, values, dones, bootstrap_value), GAMMA, c_bar=1.0)


def header_vtrace(log_rhos, rewards, values, dones, bootstrap_value, gamma, lam=1.0, rho_bar=1.0, c_bar=1.0,
                  pg_rho_bar=1.0):
    """include/ktb200.h's restatement in numpy fp32, one rounding per operation: (vs, pg_adv) as float32 arrays.  ρ is
    torch.exp of log_rhos on the device they are on (CUDA's expf on a GPU), so only the arithmetic after it is
    restated here."""
    import torch

    f = np.float32
    rho_all = torch.exp(log_rhos).cpu().numpy().astype(f)
    r, v, d, bv = (np.asarray(x.cpu() if isinstance(x, torch.Tensor) else x, dtype=f)
                   for x in (rewards, values, dones, bootstrap_value))
    g, lm = f(gamma), f(lam)
    rb, cb, pb = (f(np.inf) if x is None else f(x) for x in (rho_bar, c_bar, pg_rho_bar))
    vs, pg = np.empty_like(r), np.empty_like(r)
    acc, nv, nvs = np.zeros(r.shape[0], dtype=f), bv.copy(), bv.copy()
    with np.errstate(all="ignore"):
        for t in reversed(range(r.shape[1])):
            rho = rho_all[:, t]
            disc = g * (f(1) - d[:, t])
            cr = np.where(rho > rb, rb, rho)
            c = lm * np.where(rho > cb, cb, rho)
            pr = np.where(rho > pb, pb, rho)
            delta = cr * ((r[:, t] + disc * nv) - v[:, t])
            acc = delta + (disc * c) * acc
            vs[:, t] = acc + v[:, t]
            pg[:, t] = pr * ((r[:, t] + disc * nvs) - v[:, t])
            nv, nvs = v[:, t], vs[:, t]
    return vs, pg
