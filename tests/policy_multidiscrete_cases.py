"""User callables of the multi-discrete categorical policy, written as a kubetorch user writes SPMD functions: rank r
runs the policy of policy_cases on its `obs.chunk(WORLD_SIZE)[RANK]` rows (with the rows of the legal-action mask of
policy_masked_cases, and the critic of policy_value_cases where they take one), splits the bf16 logits into the groups
of NVEC and picks one action per group.

TEST INFRASTRUCTURE.  These functions are the semantic definition of @kt.mapped("mlp", bias=True, output="actions",
"both" or "sample", nvec=NVEC) (masked: mask="legal"; with a critic: value=("wv", "bv")): over the kernel's bf16
logits y (y.masked_fill(~legal, -inf) with a mask), the greedy actions are torch.stack([p.argmax(-1) for p in
y.split(nvec, -1)], -1); the sampled ones the same stack over y.float() + gumbel_noise(seed, row0, rows, d_out), the
noise of output="sample"; and log_probs the fp32 sum, in group order and starting from group 0's term, of each group's
log_softmax(p.float(), -1)[a_g].  The oracle restatement (oracle/ref_dispatch.spmd_call) executes them on CPU; the CUDA
path must reproduce their results.
"""
import os

from policy_cases import mlp_policy_biased
from policy_masked_cases import masked_logits
from policy_value_cases import _trunk, _value

NVEC = (3, 1, 2)   # d_out = 6: a boundary inside a column pair (3 | 4), a group of one, and one on a pair (4 | 5)


def _row0(obs):
    """Where this rank's shard begins in obs: the global index of its first row."""
    r, w = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    return min(r * -(-obs.shape[0] // w), obs.shape[0])


def grouped_actions(y, nvec):
    """int64 [rows, G]: the argmax of each group of columns of y, relative to the group."""
    import torch

    return torch.stack([p.argmax(-1) for p in y.split(tuple(nvec), -1)], -1)


def grouped_log_probs(y, nvec, actions):
    """fp32 [rows]: the sum in group order, from group 0's term, of log_softmax(group.float())[a_g]."""
    import torch

    terms = [torch.log_softmax(p.float(), -1).gather(-1, actions[:, g:g + 1]).squeeze(-1)
             for g, p in enumerate(y.split(tuple(nvec), -1))]
    lp = terms[0]
    for t in terms[1:]:
        lp = lp + t
    return lp


def grouped_sample(y, nvec, seed, row0):
    """(int64 actions [rows, G], fp32 log_probs [rows]) drawn per group with the noise of output="sample"."""
    from kubetorch_b200.sampling import gumbel_noise

    y = y.float()
    g = gumbel_noise(seed, row0, y.shape[0], y.shape[1], device=y.device)
    actions = grouped_actions(y + g, nvec)
    return actions, grouped_log_probs(y, nvec, actions)


def mlp_policy_multidiscrete_actions(obs, w1, b1, w2, b2, w3, b3):
    """Greedy int64 actions [rows, G] of this rank's rows, one per group of NVEC."""
    return grouped_actions(mlp_policy_biased(obs, w1, b1, w2, b2, w3, b3), NVEC)


def mlp_policy_multidiscrete_both(obs, w1, b1, w2, b2, w3, b3):
    """(bf16 logits, greedy int64 actions [rows, G]) of this rank's rows."""
    logits = mlp_policy_biased(obs, w1, b1, w2, b2, w3, b3)
    return logits, grouped_actions(logits, NVEC)


def mlp_policy_multidiscrete_sample(obs, w1, b1, w2, b2, w3, b3, seed):
    """(int64 actions [rows, G], fp32 log_probs) of this rank's rows sampled with `seed`."""
    return grouped_sample(mlp_policy_biased(obs, w1, b1, w2, b2, w3, b3), NVEC, seed, _row0(obs))


def mlp_policy_multidiscrete_masked_actions(obs, w1, b1, w2, b2, w3, b3, legal):
    """Greedy int64 actions [rows, G] of this rank's rows over the legal actions of each group."""
    return grouped_actions(masked_logits(obs, w1, b1, w2, b2, w3, b3, legal), NVEC)


def mlp_policy_multidiscrete_masked_sample(obs, w1, b1, w2, b2, w3, b3, legal, seed):
    """(int64 actions [rows, G], fp32 log_probs) of this rank's rows sampled from the legal actions of each group."""
    return grouped_sample(masked_logits(obs, w1, b1, w2, b2, w3, b3, legal), NVEC, seed, _row0(obs))


def mlp_policy_multidiscrete_sample_value(obs, w1, b1, w2, b2, w3, b3, wv, bv, seed):
    """(int64 actions [rows, G], fp32 log_probs, fp32 values) of this rank's rows: the critic of policy_value_cases
    beside the grouped sample."""
    import torch.nn.functional as F

    h = _trunk(obs, w1, b1, w2, b2)
    return (*grouped_sample(F.linear(h, w3, b3), NVEC, seed, _row0(obs)), _value(h, wv, bv))
