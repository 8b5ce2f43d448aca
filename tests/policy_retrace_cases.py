"""User callables of Retrace(λ) (Munos et al. 2016: the off-policy Q-value target of ACER, Reactor, MPO and Q(λ) agents),
written as a kubetorch user writes SPMD functions: rank r takes its `x.chunk(WORLD_SIZE)[RANK]` rows of env-major
rollouts (row i is environment i's trajectory, column t its step t) and runs the Retrace loop over them.

TEST INFRASTRUCTURE.  retrace() is the semantic definition of @kt.mapped("retrace", gamma=GAMMA, lam=LAM): rlax's
retrace_continuous (general_off_policy_returns_from_q_and_v) made env-major, with dones[:, t] the done flag of transition
t, log_rhos the log-ratios of the taken actions, q = Q_target(s_t, a_t), values = E_π Q_target(s_t, ·), baseline =
Q_online(s_t, a_t) (rlax's q_tm1; it may be q itself) and bootstrap_value = E_π Q_target(s_T, ·).  As in rlax, columns 0
of log_rhos, q and values are never read.  log_rhos = 0 is Harutyunyan's Q(λ) (c = λ); log_rhos = −inf on the actions
the target policy does not take is Watkins' Q(λ) (the trace is cut there).  include/ktb200.h restates it as fp32
operations (header_retrace below), and the CUDA path must reproduce its bits.  The oracle restatement
(oracle/ref_dispatch.spmd_call) executes the bodies on CPU.
"""
import os

import numpy as np

GAMMA, LAM = 0.99, 0.95


def _shard(t):
    """This rank's rows of t, as obs.chunk(WORLD_SIZE)[RANK] (an empty shard for ranks past the data)."""
    r, w = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    rows = t.chunk(w, dim=0)
    return rows[r] if r < len(rows) else t[:0]


def retrace(log_rhos, rewards, q, values, dones, baseline, bootstrap_value, gamma, lam):
    import torch

    T = rewards.shape[1]
    discounts = gamma * (1.0 - dones)
    cs = torch.clamp(torch.exp(log_rhos), max=1.0) * lam
    g = rewards[:, -1] + discounts[:, -1] * bootstrap_value
    ret = torch.empty_like(rewards)
    ret[:, -1] = g
    for t in reversed(range(T - 1)):
        g = rewards[:, t] + discounts[:, t] * (values[:, t + 1] - cs[:, t + 1] * q[:, t + 1] + cs[:, t + 1] * g)
        ret[:, t] = g
    return ret, ret - baseline


def _shards(*xs):
    return tuple(_shard(t) for t in xs)


def mapped_retrace(log_rhos, rewards, q, values, dones, baseline, bootstrap_value):
    """@kt.mapped("retrace", gamma=GAMMA, lam=LAM)."""
    return retrace(*_shards(log_rhos, rewards, q, values, dones, baseline, bootstrap_value), GAMMA, LAM)


def mapped_retrace_args(log_rhos, rewards, q, values, dones, baseline, bootstrap_value, gamma, lam):
    """gamma and lam as call arguments: @kt.mapped("retrace", gamma="gamma", lam="lam")."""
    return retrace(*_shards(log_rhos, rewards, q, values, dones, baseline, bootstrap_value), gamma, lam)


def mapped_retrace_shifted(log_rhos, rewards, q, values, dones, baseline, bootstrap_value):
    """A body that reads episode-start flags: dones[:, t + 1] as step t's flag (CleanRL's dones[t] says observation t
    starts an episode) and the last step as nonterminal.  Not the op's body: the deployment's self-check refuses it."""
    import torch

    xs = list(_shards(log_rhos, rewards, q, values, dones, baseline, bootstrap_value))
    xs[4] = torch.cat([xs[4][:, 1:], torch.zeros_like(xs[4][:, :1])], 1)
    return retrace(*xs, GAMMA, LAM)


def mapped_retrace_other_gamma(log_rhos, rewards, q, values, dones, baseline, bootstrap_value):
    """The body with γ = 0.98: not what a deployment declaring gamma=GAMMA computes."""
    return retrace(*_shards(log_rhos, rewards, q, values, dones, baseline, bootstrap_value), 0.98, LAM)


def mapped_retrace_other_lam(log_rhos, rewards, q, values, dones, baseline, bootstrap_value):
    """The body with λ = 0.9: not what a deployment declaring lam=LAM computes."""
    return retrace(*_shards(log_rhos, rewards, q, values, dones, baseline, bootstrap_value), GAMMA, 0.9)


def mapped_retrace_unclipped(log_rhos, rewards, q, values, dones, baseline, bootstrap_value):
    """Importance-sampled traces c = λ·ρ without Retrace's min(1, ρ): not the op's body."""
    import torch

    lr, r, q_, v, d, b, bv = _shards(log_rhos, rewards, q, values, dones, baseline, bootstrap_value)
    T = r.shape[1]
    discounts = GAMMA * (1.0 - d)
    cs = torch.exp(lr) * LAM
    g = r[:, -1] + discounts[:, -1] * bv
    ret = torch.empty_like(r)
    ret[:, -1] = g
    for t in reversed(range(T - 1)):
        g = r[:, t] + discounts[:, t] * (v[:, t + 1] - cs[:, t + 1] * q_[:, t + 1] + cs[:, t + 1] * g)
        ret[:, t] = g
    return ret, ret - b


def mapped_retrace_current_value(log_rhos, rewards, q, values, dones, baseline, bootstrap_value):
    """A body that reads values[:, t] where the target reads the next state's values[:, t + 1]: not the op's body."""
    import torch

    lr, r, q_, v, d, b, bv = _shards(log_rhos, rewards, q, values, dones, baseline, bootstrap_value)
    return retrace(lr, r, q_, torch.cat([v[:, :1], v[:, :-1]], 1), d, b, bv, GAMMA, LAM)


def header_retrace(log_rhos, rewards, q, values, dones, baseline, bootstrap_value, gamma, lam):
    """include/ktb200.h's restatement in numpy fp32, one rounding per operation: (ret, td) as float32 arrays.  ρ is
    torch.exp of log_rhos on the device they are on (CUDA's expf on a GPU), so only the arithmetic after it is
    restated here."""
    import torch

    f = np.float32
    rho_all = torch.exp(log_rhos).cpu().numpy().astype(f)
    r, qq, v, d, b, bv = (np.asarray(x.cpu() if isinstance(x, torch.Tensor) else x, dtype=f)
                          for x in (rewards, q, values, dones, baseline, bootstrap_value))
    g, lm = f(gamma), f(lam)
    ret, td = np.empty_like(r), np.empty_like(r)
    n = r.shape[0]
    acc, nv = np.zeros(n, dtype=f), bv.copy()
    nq, nc = np.full(n, -0.0, dtype=f), np.full(n, -0.0, dtype=f)
    with np.errstate(all="ignore"):
        for t in reversed(range(r.shape[1])):
            disc = g * (f(1) - d[:, t])
            acc = r[:, t] + disc * ((nv - nc * nq) + nc * acc)
            ret[:, t] = acc
            td[:, t] = acc - b[:, t]
            rho = rho_all[:, t]
            nc = lm * np.where(rho > f(1), f(1), rho)
            nv, nq = v[:, t], qq[:, t]
    return ret, td
