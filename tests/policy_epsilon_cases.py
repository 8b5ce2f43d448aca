"""User callables of the ε-greedy Q-network actor (DQN, Ape-X, R2D2), written as a kubetorch user writes SPMD
functions: rank r runs the trunk  Linear → ReLU → Linear → ReLU  on its `obs.chunk(WORLD_SIZE)[RANK]` rows and a Q head
nn.Linear(d_hidden, d_out) (w3, b3), explores with the draws of its rows' GLOBAL indices, and returns (actions, q,
q_max): the action taken, its Q-value and the greedy Q-value, for the initial replay priorities of Ape-X.

TEST INFRASTRUCTURE.  These functions are the semantic definition of @kt.mapped("mlp", bias=True,
output="epsilon_greedy", seed="seed", epsilon="eps") (masked: mask="legal" too).  `eps` is a float, or a per-row fp32
tensor [M] that each rank shards like obs.  The oracle restatement (oracle/ref_dispatch.spmd_call) executes them on
CPU; the CUDA path must reproduce their results.
"""
from policy_value_cases import _row0, _shard, _trunk


def epsilon_greedy(q, eps, seed, row0, legal=None):
    """(int64 actions, float32 q, float32 q_max) of the bf16 Q-values q [rows, d_out] of global rows row0, ...: a row
    explores iff u < ε (fp32) and then takes the legal column with the largest exploration word, else the argmax."""
    import torch

    from kubetorch_b200.sampling import explore_noise

    rows, d_out = q.shape
    if legal is None:
        legal = torch.ones(rows, d_out, dtype=torch.bool, device=q.device)
    q = q.masked_fill(~legal, float("-inf"))
    eps_r = eps if isinstance(eps, torch.Tensor) else torch.full((rows,), float(eps), dtype=torch.float32)
    u, w = explore_noise(seed, row0, rows, d_out, device=q.device)
    greedy = q.argmax(-1)
    explore_a = w.masked_fill(~legal, -1).argmax(-1)   # words are >= 0, so -1 never wins over a legal column
    actions = torch.where(u < eps_r.to(q.device), explore_a, greedy)
    qf = q.float()
    return actions, qf.gather(1, actions[:, None])[:, 0], qf.gather(1, greedy[:, None])[:, 0]


def _eps_rows(eps):
    import torch

    return _shard(eps) if isinstance(eps, torch.Tensor) else eps


def mlp_policy_epsilon_greedy(obs, w1, b1, w2, b2, w3, b3, eps, seed):
    """(int64 actions, float32 q, float32 q_max) of this rank's rows, exploring with probability eps."""
    import torch.nn.functional as F

    q = F.linear(_trunk(obs, w1, b1, w2, b2), w3, b3)
    return epsilon_greedy(q, _eps_rows(eps), seed, _row0(obs))


def mlp_policy_epsilon_greedy_masked(obs, w1, b1, w2, b2, w3, b3, legal, eps, seed):
    """As mlp_policy_epsilon_greedy over the legal actions of each row (legal: bool [M, d_out], True: legal)."""
    import torch.nn.functional as F

    q = F.linear(_trunk(obs, w1, b1, w2, b2), w3, b3)
    return epsilon_greedy(q, _eps_rows(eps), seed, _row0(obs), _shard(legal))
