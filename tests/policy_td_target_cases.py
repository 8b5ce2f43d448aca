"""User callables of the TD targets of TD3, DDPG and SAC, written as a kubetorch user writes SPMD functions: rank r takes
its `next_obs.chunk(WORLD_SIZE)[RANK]` rows, runs the (target) actor on them for the next actions (the deterministic
actor of policy_deterministic_cases, or the state-dependent Gaussian head of policy_gaussian_state_cases, with the noise
of the rows' GLOBAL indices), the (target) critics of policy_critic_cases over those actions, and returns the Bellman
target  reward + gamma * (1 - done) * t  of its rows, t the critic's q, the twin's minimum, less alpha * log_prob for SAC.

TEST INFRASTRUCTURE.  These functions are the semantic definition of @kt.mapped("mlp", bias=True, output="td_target",
actor=(...), policy=..., twin=(...), reward="r", done="d", gamma=..., ...).  The oracle restatement
(oracle/ref_dispatch.spmd_call) executes them on CPU; the CUDA path must reproduce their results.
"""
from policy_critic_cases import critic_q
from policy_deterministic_cases import deterministic
from policy_gaussian_state_cases import gaussian_state
from policy_value_cases import _row0, _shard, _trunk

GAMMA = 0.99


def td_target(reward, done, gamma, t, alpha=None, logp=None):
    """y as users write it: reward + gamma * (1 - done) * (t - alpha * logp), the α term only with logp."""
    if logp is not None:
        t = t - alpha * logp
    return reward + gamma * (1 - done) * t


def header_y(reward, done, gamma, t, alpha=None, logp=None):
    """The header's restatement, one fp32 rounding per operation in its order, element by element in numpy."""
    import numpy as np
    import torch

    f = np.float32
    r, d, tt = (x.reshape(-1).numpy().astype(np.float32) for x in (reward, done, t))
    lp = None if logp is None else logp.reshape(-1).numpy().astype(np.float32)
    out = np.empty_like(r)
    with np.errstate(all="ignore"):
        for i in range(r.shape[0]):
            ti = tt[i]
            if lp is not None:
                ti = f(ti - f(f(alpha) * lp[i]))
            out[i] = f(r[i] + f(f(f(gamma) * f(f(1.0) - d[i])) * ti))
    return torch.from_numpy(out).reshape(reward.shape)


def _rows(t):
    return _shard(t)


def mlp_td3_target(next_obs, w1, b1, w2, b2, w3, b3, a1, ab1, a2, ab2, a3, ab3, v1, c1, v2, c2, v3, c3, r, d, seed):
    """TD3's target: smoothed target actions (σ 0.2, clip 0.5) and the minimum of the twin target critics."""
    import torch
    import torch.nn.functional as F

    o = _shard(next_obs)
    act = deterministic(F.linear(_trunk(next_obs, a1, ab1, a2, ab2), a3, ab3), seed, _row0(next_obs), noise=0.2,
                        noise_clip=0.5)
    t = torch.minimum(critic_q(o, act, w1, b1, w2, b2, w3, b3), critic_q(o, act, v1, c1, v2, c2, v3, c3))
    return td_target(_rows(r), _rows(d), GAMMA, t)


def mlp_ddpg_target(next_obs, w1, b1, w2, b2, w3, b3, a1, ab1, a2, ab2, a3, ab3, r, d):
    """DDPG's target: the noise-free target actor and one target critic."""
    import torch.nn.functional as F

    o = _shard(next_obs)
    act = deterministic(F.linear(_trunk(next_obs, a1, ab1, a2, ab2), a3, ab3), None, _row0(next_obs))
    return td_target(_rows(r), _rows(d), GAMMA, critic_q(o, act, w1, b1, w2, b2, w3, b3))


def mlp_sac_target(next_obs, w1, b1, w2, b2, w3, b3, a1, ab1, a2, ab2, a3, ab3, w_ls, b_ls, v1, c1, v2, c2, v3, c3,
                   r, d, seed, alpha):
    """SAC's target: squashed next actions with their log-probabilities, the twin's minimum less α·log π."""
    import torch

    o = _shard(next_obs)
    act, logp = gaussian_state(_trunk(next_obs, a1, ab1, a2, ab2), a3, ab3, w_ls, b_ls, seed, _row0(next_obs),
                               squash=True)
    t = torch.minimum(critic_q(o, act, w1, b1, w2, b2, w3, b3), critic_q(o, act, v1, c1, v2, c2, v3, c3))
    return td_target(_rows(r), _rows(d), GAMMA, t, float(alpha), logp)
