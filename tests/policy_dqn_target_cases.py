"""User callables of the DQN and Double DQN targets, written as a kubetorch user writes SPMD functions: rank r takes its
`next_obs.chunk(WORLD_SIZE)[RANK]` rows, runs the target Q-network (and for Double DQN the online Q-network) on them,
picks the greedy next action with the selecting network's (masked) Q-values, and returns the Bellman target
reward + gamma * (1 - done) * q of its rows, q the target network's UNMASKED Q-value at that action.

TEST INFRASTRUCTURE.  These functions are the semantic definition of @kt.mapped("mlp", bias=True, output="dqn_target",
online=(...), mask="legal", reward="r", done="d", gamma=...).  The oracle restatement (oracle/ref_dispatch.spmd_call)
executes them on CPU; the CUDA path must reproduce their results.
"""
from policy_value_cases import _shard, _trunk

GAMMA = 0.99


def dqn_target(q_target, reward, done, gamma, q_online=None, legal=None):
    """y of the rows' bf16 Q-values [rows, d_out] as users write it: the selector (the online network's Q for Double DQN,
    the target's for DQN) masked with the legal actions, its argmax, the target's unmasked Q there widened to fp32, and
    reward + gamma * (1 - done) * q, of reward's shape ([rows] or [rows, 1])."""
    s = q_online if q_online is not None else q_target
    if legal is not None:
        s = s.masked_fill(~legal, float("-inf"))
    q = q_target.float().gather(1, s.argmax(-1, keepdim=True)).squeeze(1)
    return reward + gamma * (1 - done) * q.reshape(reward.shape)


def header_y(reward, done, gamma, q):
    """The header's restatement, one fp32 rounding per operation in its order, element by element in numpy."""
    import numpy as np
    import torch

    f = np.float32
    r, d, qq = (x.reshape(-1).numpy().astype(np.float32) for x in (reward, done, q))
    out = np.empty_like(r)
    with np.errstate(all="ignore"):
        for i in range(r.shape[0]):
            out[i] = f(r[i] + f(f(f(gamma) * f(f(1.0) - d[i])) * qq[i]))
    return torch.from_numpy(out).reshape(reward.shape)


def _q(next_obs, w1, b1, w2, b2, w3, b3):
    import torch.nn.functional as F

    return F.linear(_trunk(next_obs, w1, b1, w2, b2), w3, b3)


def mlp_dqn_target(next_obs, w1, b1, w2, b2, w3, b3, r, d):
    """DQN's target: the target network picks and scores the next action."""
    return dqn_target(_q(next_obs, w1, b1, w2, b2, w3, b3), _shard(r), _shard(d), GAMMA)


def mlp_dqn_target_masked(next_obs, w1, b1, w2, b2, w3, b3, legal, r, d):
    """As mlp_dqn_target over the legal actions of each next state (legal: bool [M, d_out], True: legal)."""
    return dqn_target(_q(next_obs, w1, b1, w2, b2, w3, b3), _shard(r), _shard(d), GAMMA, legal=_shard(legal))


def mlp_double_dqn_target(next_obs, w1, b1, w2, b2, w3, b3, o1, ob1, o2, ob2, o3, ob3, r, d):
    """Double DQN's target: the online network (o1 .. ob3) picks the next action, the target network scores it."""
    return dqn_target(_q(next_obs, w1, b1, w2, b2, w3, b3), _shard(r), _shard(d), GAMMA,
                      q_online=_q(next_obs, o1, ob1, o2, ob2, o3, ob3))


def mlp_double_dqn_target_masked(next_obs, w1, b1, w2, b2, w3, b3, o1, ob1, o2, ob2, o3, ob3, legal, r, d):
    """As mlp_double_dqn_target over the legal actions of each next state."""
    return dqn_target(_q(next_obs, w1, b1, w2, b2, w3, b3), _shard(r), _shard(d), GAMMA,
                      q_online=_q(next_obs, o1, ob1, o2, ob2, o3, ob3), legal=_shard(legal))
