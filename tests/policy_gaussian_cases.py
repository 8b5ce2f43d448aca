"""User callable of the Gaussian nn.Linear policy, written as a kubetorch user writes SPMD functions: rank r runs the
policy of policy_cases on its `obs.chunk(WORLD_SIZE)[RANK]` rows as the mean, adds exp(log_std) times the Gaussian
noise of those rows' GLOBAL indices (its shard begins at row0 of obs), and returns (actions, log_probs).

TEST INFRASTRUCTURE.  This function is the semantic definition of
@kt.mapped("mlp", bias=True, output="gaussian", seed="seed", log_std="log_std"): with μ the fp32 logits and
z = normal_noise(seed, row0, ...), actions = μ + exp(log_std)·z and log_probs = (-0.5·z² - log_std - 0.5·log 2π)
summed over the head, the log-density of the action under Normal(μ, exp(log_std)).  The oracle restatement
(oracle/ref_dispatch.spmd_call) executes it on CPU; the CUDA path must reproduce its results.
"""
import math
import os

from policy_cases import mlp_policy_biased


def mlp_policy_gaussian(obs, w1, b1, w2, b2, w3, b3, log_std, seed):
    """(float32 actions [rows, d_out], float32 log_probs [rows]) of the policy on this rank's shard, drawn with
    `seed`."""
    import torch

    from kubetorch_b200.sampling import normal_noise

    r, w = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    row0 = min(r * -(-obs.shape[0] // w), obs.shape[0])   # where obs.chunk(w)[r] begins
    mu = mlp_policy_biased(obs, w1, b1, w2, b2, w3, b3).float()
    z = normal_noise(seed, row0, mu.shape[0], mu.shape[1], device=mu.device)
    log_std = log_std.float().to(mu.device)
    actions = mu + torch.exp(log_std) * z
    log_probs = (-0.5 * z * z - log_std - 0.5 * math.log(2 * math.pi)).sum(-1)
    return actions, log_probs
