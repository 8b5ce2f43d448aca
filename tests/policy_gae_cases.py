"""User callables of generalized advantage estimation, written as a kubetorch user writes SPMD functions: rank r takes
its `x.chunk(WORLD_SIZE)[RANK]` rows of env-major rollouts (row i is environment i's trajectory, column t its step t)
and runs CleanRL's backward loop over them.

TEST INFRASTRUCTURE.  gae() is the semantic definition of @kt.mapped("gae", gamma=GAMMA, lam=LAM): dones[:, t] is the
done flag of transition t (the episode ended after the action at step t) and last_values is V(s_T).  The expression
order is CleanRL's; include/ktb200.h restates it as fp32 operations (header_gae below), and the CUDA path must
reproduce its bits.  The oracle restatement (oracle/ref_dispatch.spmd_call) executes the bodies on CPU.
"""
import os

import numpy as np

GAMMA, LAM = 0.99, 0.95


def _shard(t):
    """This rank's rows of t, as obs.chunk(WORLD_SIZE)[RANK] (an empty shard for ranks past the data)."""
    r, w = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    rows = t.chunk(w, dim=0)
    return rows[r] if r < len(rows) else t[:0]


def gae(rewards, values, dones, last_values, gamma, lam):
    import torch

    adv = torch.empty_like(rewards)
    acc = torch.zeros_like(last_values)
    next_v = last_values
    for t in reversed(range(rewards.shape[1])):
        nonterminal = 1.0 - dones[:, t]
        delta = rewards[:, t] + gamma * next_v * nonterminal - values[:, t]
        acc = delta + gamma * lam * nonterminal * acc
        adv[:, t] = acc
        next_v = values[:, t]
    return adv, adv + values


def mapped_gae(rewards, values, dones, last_values):
    return gae(*(_shard(t) for t in (rewards, values, dones, last_values)), GAMMA, LAM)


def mapped_gae_args(rewards, values, dones, last_values, gamma, lam):
    """gamma and lam as call arguments: @kt.mapped("gae", gamma="gamma", lam="lam")."""
    return gae(*(_shard(t) for t in (rewards, values, dones, last_values)), gamma, lam)


def mapped_gae_shifted(rewards, values, dones, last_values):
    """A CleanRL buffer's loop run on transition-t done flags: it reads dones[:, t + 1] as step t's flag (CleanRL's
    dones[t] says observation t starts an episode) and treats the last step as nonterminal.  Not the op's body: the
    deployment's self-check refuses it."""
    import torch

    rewards, values, dones, last_values = (_shard(t) for t in (rewards, values, dones, last_values))
    adv = torch.empty_like(rewards)
    acc = torch.zeros_like(last_values)
    T = rewards.shape[1]
    for t in reversed(range(T)):
        if t == T - 1:
            nonterminal, next_v = torch.ones_like(last_values), last_values
        else:
            nonterminal, next_v = 1.0 - dones[:, t + 1], values[:, t + 1]
        delta = rewards[:, t] + GAMMA * next_v * nonterminal - values[:, t]
        acc = delta + GAMMA * LAM * nonterminal * acc
        adv[:, t] = acc
    return adv, adv + values


def mapped_gae_other_gamma(rewards, values, dones, last_values):
    """The body with γ = 0.98: not what a deployment declaring gamma=GAMMA computes."""
    return gae(*(_shard(t) for t in (rewards, values, dones, last_values)), 0.98, LAM)


def header_gae(rewards, values, dones, last_values, gamma, lam):
    """include/ktb200.h's restatement in numpy fp32, one rounding per operation: (adv, ret) as float32 arrays."""
    f = np.float32
    r, v, d, lv = (np.asarray(x, dtype=f) for x in (rewards, values, dones, last_values))
    g, gl = f(gamma), f(float(gamma) * float(lam))
    adv, ret = np.empty_like(r), np.empty_like(r)
    acc, nv = np.zeros(r.shape[0], dtype=f), lv.copy()
    with np.errstate(all="ignore"):
        for t in reversed(range(r.shape[1])):
            nt = f(1) - d[:, t]
            delta = (r[:, t] + (g * nv) * nt) - v[:, t]
            acc = delta + (gl * nt) * acc
            adv[:, t] = acc
            ret[:, t] = acc + v[:, t]
            nv = v[:, t]
    return adv, ret
