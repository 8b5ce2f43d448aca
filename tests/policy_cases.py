"""User callables of the nn.Linear policy cases, written as a kubetorch user writes SPMD functions: each rank reads
RANK / WORLD_SIZE, takes its `obs.chunk(WORLD_SIZE)[RANK]` rows (an empty shard for ranks past the data) and runs
the policy  Linear → ReLU → Linear → ReLU → Linear  with biases.

TEST INFRASTRUCTURE.  These functions are the semantic definition of @kt.mapped("mlp", bias=True, output=...):
F.linear adds the bias inside the matmul (one bf16 rounding per layer) and the actions are torch.argmax over the
last dimension of the bf16 logits.  The oracle restatement (oracle/ref_dispatch.spmd_call) executes them on CPU; the
CUDA path must reproduce their results.
"""
import os


def _obs_shard(obs):
    r, w = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    rows = obs.chunk(w, dim=0)
    return rows[r] if r < len(rows) else obs[:0]


def mlp_policy_biased(obs, w1, b1, w2, b2, w3, b3):
    """Logits of the policy on this rank's shard of observations (rows)."""
    import torch
    import torch.nn.functional as F

    h = torch.relu(F.linear(_obs_shard(obs), w1, b1))
    h = torch.relu(F.linear(h, w2, b2))
    return F.linear(h, w3, b3)


def mlp_policy_actions(obs, w1, b1, w2, b2, w3, b3):
    """Greedy actions (int64) of the policy on this rank's shard."""
    return mlp_policy_biased(obs, w1, b1, w2, b2, w3, b3).argmax(-1)


def mlp_policy_both(obs, w1, b1, w2, b2, w3, b3):
    """(logits, actions) of the policy on this rank's shard."""
    logits = mlp_policy_biased(obs, w1, b1, w2, b2, w3, b3)
    return logits, logits.argmax(-1)
