"""User callables of the Q(s, a) critics of SAC and TD3, written as a kubetorch user writes SPMD functions: rank r runs
the critic  Linear(d_in + d_act, d_h) → ReLU → Linear(d_h, d_h) → ReLU → Linear(d_h, 1)  on torch.cat of its
`obs.chunk(WORLD_SIZE)[RANK]` rows and the same rows of the actions, rounded to bf16, and returns the fp32 Q-value of
each row; the twin runs two independent critics on the same rows and also returns their minimum.

TEST INFRASTRUCTURE.  These functions are the semantic definition of @kt.mapped("mlp", bias=True, output="critic",
action="act") (with twin=("v1", "c1", "v2", "c2", "v3", "c3"): the twin): q = F.linear(h, w3, b3).float().squeeze(-1)
over x = torch.cat([obs, act.to(torch.bfloat16)], -1), and q_min = torch.minimum(q1, q2).  The oracle restatement
(oracle/ref_dispatch.spmd_call) executes them on CPU; the CUDA path must reproduce their results.
"""
from policy_value_cases import _shard


def critic_q(obs, act, w1, b1, w2, b2, w3, b3):
    """fp32 q [rows] of one critic over rows obs (bf16 [rows, d_in]) and act (fp32 [rows, d_act]): the header's
    definition."""
    import torch
    import torch.nn.functional as F

    x = torch.cat([obs, act.to(torch.bfloat16)], -1)
    h = torch.relu(F.linear(torch.relu(F.linear(x, w1, b1)), w2, b2))
    return F.linear(h, w3, b3).float().squeeze(-1)


def q_min(q1, q2):
    """The twin's minimum as the header states it: q2 < q1 ? q2 : q1, NaN when either is (q1 on ties, signed zeros
    included); torch.minimum(q1, q2) of 0-d CPU tensors."""
    import torch

    return torch.where(q2.isnan(), q2, torch.where(q2 < q1, q2, q1))


def mlp_critic(obs, w1, b1, w2, b2, w3, b3, act):
    """Q(s, a) of this rank's rows: a TD3 or SAC critic, or an Ape-X DPG actor's initial priority."""
    return critic_q(_shard(obs), _shard(act), w1, b1, w2, b2, w3, b3)


def mlp_critic_twin(obs, w1, b1, w2, b2, w3, b3, act, v1, c1, v2, c2, v3, c3):
    """Clipped double Q of this rank's rows: (q1, q2, min(q1, q2)), the min of TD3's and SAC's targets."""
    import torch

    o, a = _shard(obs), _shard(act)
    q1 = critic_q(o, a, w1, b1, w2, b2, w3, b3)
    q2 = critic_q(o, a, v1, c1, v2, c2, v3, c3)
    return q1, q2, torch.minimum(q1, q2)


def mlp_critic_nobias(obs, w1, w2, w3, act):
    """A bias-free critic (bias=False)."""
    return critic_q(_shard(obs), _shard(act), w1, None, w2, None, w3, None)
