"""User callables of n-step bootstrapped returns (Ape-X's, R2D2's and A3C's learner targets), written as a kubetorch user
writes SPMD functions: rank r takes its `x.chunk(WORLD_SIZE)[RANK]` rows of env-major rollouts (row i is environment
i's trajectory, column t its step t) and runs the padded n-step loop over them.

TEST INFRASTRUCTURE.  nstep() is the semantic definition of @kt.mapped("nstep", n=N_STEP, gamma=GAMMA): rlax's
n_step_bootstrapped_returns with lambda_t = 1 made env-major, dones[:, t] the done flag of transition t, values[:, t]
the bootstrap value of state s_t, baseline what the TD error is taken against and last_values V(s_T).  The λ-mixing
term (1 − λ)·v + λ·g is dropped rather than evaluated at λ = 1, so the body differs from rlax only in the sign of a
zero result and where 0·v would be 0·inf.  include/ktb200.h restates it as fp32 operations (header_nstep below), and
the CUDA path must reproduce its bits.  The oracle restatement (oracle/ref_dispatch.spmd_call) executes the bodies on
CPU.
"""
import os

import numpy as np

N_STEP, GAMMA = 5, 0.99


def _shard(t):
    """This rank's rows of t, as obs.chunk(WORLD_SIZE)[RANK] (an empty shard for ranks past the data)."""
    r, w = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    rows = t.chunk(w, dim=0)
    return rows[r] if r < len(rows) else t[:0]


def nstep(rewards, values, dones, baseline, last_values, n, gamma):
    import torch

    N, T = rewards.shape
    pad = n - 1
    disc = gamma * (1.0 - dones)
    v_next = torch.cat([values[:, 1:], last_values[:, None]], 1)
    r = torch.cat([rewards, rewards.new_zeros(N, pad)], 1)
    dc = torch.cat([disc, disc.new_ones(N, pad)], 1)
    v = torch.cat([v_next, last_values[:, None].expand(N, pad)], 1)
    g = v[:, pad:]
    for i in reversed(range(n)):
        g = r[:, i:i + T] + dc[:, i:i + T] * g
    return g, g - baseline


def _shards(*xs):
    return tuple(_shard(t) for t in xs)


def mapped_nstep(rewards, values, dones, baseline, last_values):
    """@kt.mapped("nstep", n=N_STEP, gamma=GAMMA)."""
    return nstep(*_shards(rewards, values, dones, baseline, last_values), N_STEP, GAMMA)


def mapped_nstep_args(rewards, values, dones, baseline, last_values, gamma):
    """gamma as a call argument: @kt.mapped("nstep", n=N_STEP, gamma="gamma")."""
    return nstep(*_shards(rewards, values, dones, baseline, last_values), N_STEP, gamma)


def mapped_nstep_shifted(rewards, values, dones, baseline, last_values):
    """A body that reads episode-start flags: dones[:, t + 1] as step t's flag (CleanRL's dones[t] says observation t
    starts an episode) and the last step as nonterminal.  Not the op's body: the deployment's self-check refuses it."""
    import torch

    rewards, values, dones, baseline, last_values = _shards(rewards, values, dones, baseline, last_values)
    shifted = torch.cat([dones[:, 1:], torch.zeros_like(dones[:, :1])], 1)
    return nstep(rewards, values, shifted, baseline, last_values, N_STEP, GAMMA)


def mapped_nstep_other_gamma(rewards, values, dones, baseline, last_values):
    """The body with γ = 0.98: not what a deployment declaring gamma=GAMMA computes."""
    return nstep(*_shards(rewards, values, dones, baseline, last_values), N_STEP, 0.98)


def mapped_nstep_other_n(rewards, values, dones, baseline, last_values):
    """The body with n = 3: not what a deployment declaring n=N_STEP computes."""
    return nstep(*_shards(rewards, values, dones, baseline, last_values), 3, GAMMA)


def mapped_nstep_zero_bootstrap(rewards, values, dones, baseline, last_values):
    """A body that bootstraps 0 past the rollout's end instead of V(s_T): the op's padding carries last_values."""
    import torch

    rewards, values, dones, baseline, last_values = _shards(rewards, values, dones, baseline, last_values)
    return nstep(rewards, values, dones, baseline, torch.zeros_like(last_values), N_STEP, GAMMA)


def header_nstep(rewards, values, dones, baseline, last_values, n, gamma):
    """include/ktb200.h's restatement in numpy fp32, one rounding per operation: (ret, td) as float32 arrays."""
    f = np.float32
    r, v, d, b, lv = (np.asarray(x.cpu() if hasattr(x, "cpu") else x, dtype=f)
                      for x in (rewards, values, dones, baseline, last_values))
    N, T = r.shape
    g = f(gamma)
    ret = np.empty_like(r)
    with np.errstate(all="ignore"):
        for t in range(T):
            acc = v[:, t + n] if t + n < T else lv.copy()
            for k in reversed(range(n)):
                if t + k < T:
                    rk, disc = r[:, t + k], g * (f(1) - d[:, t + k])
                else:
                    rk, disc = f(0), f(1)
                acc = rk + disc * acc
            ret[:, t] = acc
        td = ret - b
    return ret, td
