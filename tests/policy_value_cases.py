"""User callables of the shared-trunk actor-critic, written as a kubetorch user writes SPMD functions: rank r runs the
trunk  Linear → ReLU → Linear → ReLU  on its `obs.chunk(WORLD_SIZE)[RANK]` rows, the sampled policy head of
policy_sample_cases / policy_masked_cases / policy_gaussian_cases on it, and a critic nn.Linear(d_hidden, 1) (weight
wv [1, d_hidden], bias bv [1]) on the same trunk, and returns (actions, log_probs, values).

TEST INFRASTRUCTURE.  These functions are the semantic definition of @kt.mapped("mlp", bias=True, output="sample" or
"gaussian", seed="seed", value=("wv", "bv")) (masked: mask="legal" too): the actions and log-probabilities are those of
the policy without a value head, and values = F.linear(h, wv, bv).float().squeeze(-1), the bf16 value widened to fp32.
The oracle restatement (oracle/ref_dispatch.spmd_call) executes them on CPU; the CUDA path must reproduce their
results.
"""
import math
import os


def _shard(t):
    """This rank's rows of t, as obs.chunk(WORLD_SIZE)[RANK] (an empty shard for ranks past the data)."""
    r, w = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    rows = t.chunk(w, dim=0)
    return rows[r] if r < len(rows) else t[:0]


def _row0(obs):
    """Where this rank's shard begins in obs: the global index of its first row."""
    r, w = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    return min(r * -(-obs.shape[0] // w), obs.shape[0])


def _trunk(obs, w1, b1, w2, b2):
    """h2 of this rank's rows: the shared trunk of the actor and the critic."""
    import torch
    import torch.nn.functional as F

    return torch.relu(F.linear(torch.relu(F.linear(_shard(obs), w1, b1)), w2, b2))


def _value(h, wv, bv):
    import torch.nn.functional as F

    return F.linear(h, wv, bv).float().squeeze(-1)


def _sample(logits, seed, row0):
    import torch

    from kubetorch_b200.sampling import gumbel_noise

    g = gumbel_noise(seed, row0, logits.shape[0], logits.shape[1], device=logits.device)
    actions = (logits + g).argmax(-1)
    return actions, torch.log_softmax(logits, -1).gather(-1, actions[:, None]).squeeze(-1)


def mlp_policy_sample_value(obs, w1, b1, w2, b2, w3, b3, wv, bv, seed):
    """(int64 actions, float32 log_probs, float32 values) of this rank's rows, sampled with `seed`."""
    import torch.nn.functional as F

    h = _trunk(obs, w1, b1, w2, b2)
    return (*_sample(F.linear(h, w3, b3).float(), seed, _row0(obs)), _value(h, wv, bv))


def mlp_policy_masked_sample_value(obs, w1, b1, w2, b2, w3, b3, legal, wv, bv, seed):
    """As mlp_policy_sample_value, with actions drawn from the legal ones only; the mask does not touch the values."""
    import torch.nn.functional as F

    h = _trunk(obs, w1, b1, w2, b2)
    logits = F.linear(h, w3, b3).masked_fill(~_shard(legal), float("-inf")).float()
    return (*_sample(logits, seed, _row0(obs)), _value(h, wv, bv))


def mlp_policy_gaussian_value(obs, w1, b1, w2, b2, w3, b3, log_std, wv, bv, seed):
    """(float32 actions [rows, d_out], float32 log_probs, float32 values) of this rank's rows, drawn with `seed`."""
    import torch
    import torch.nn.functional as F

    from kubetorch_b200.sampling import normal_noise

    h = _trunk(obs, w1, b1, w2, b2)
    mu = F.linear(h, w3, b3).float()
    z = normal_noise(seed, _row0(obs), mu.shape[0], mu.shape[1], device=mu.device)
    log_std = log_std.float().to(mu.device)
    actions = mu + torch.exp(log_std) * z
    log_probs = (-0.5 * z * z - log_std - 0.5 * math.log(2 * math.pi)).sum(-1)
    return actions, log_probs, _value(h, wv, bv)
