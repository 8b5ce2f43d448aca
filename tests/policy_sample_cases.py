"""User callable of the sampled nn.Linear policy, written as a kubetorch user writes SPMD functions: rank r runs the
policy of policy_cases on its `obs.chunk(WORLD_SIZE)[RANK]` rows, adds the Gumbel noise of those rows' GLOBAL indices
(its shard begins at row0 of obs), and returns (actions, log_probs).

TEST INFRASTRUCTURE.  This function is the semantic definition of
@kt.mapped("mlp", bias=True, output="sample", seed="seed"): actions = argmax(float(logits) + gumbel_noise) under the
torch.argmax rules, log_probs = log_softmax(float(logits))[action].  The oracle restatement
(oracle/ref_dispatch.spmd_call) executes it on CPU; the CUDA path must reproduce its results.
"""
import os

from policy_cases import mlp_policy_biased


def mlp_policy_sample(obs, w1, b1, w2, b2, w3, b3, seed):
    """(int64 actions, float32 log_probs) of the policy on this rank's shard, sampled with `seed`."""
    import torch

    from kubetorch_b200.sampling import gumbel_noise

    r, w = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    row0 = min(r * -(-obs.shape[0] // w), obs.shape[0])   # where obs.chunk(w)[r] begins
    logits = mlp_policy_biased(obs, w1, b1, w2, b2, w3, b3).float()
    g = gumbel_noise(seed, row0, logits.shape[0], logits.shape[1], device=logits.device)
    actions = (logits + g).argmax(-1)
    log_probs = torch.log_softmax(logits, -1).gather(-1, actions[:, None]).squeeze(-1)
    return actions, log_probs
