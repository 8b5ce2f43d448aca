"""User callables of the masked categorical policy, written as a kubetorch user writes SPMD functions: rank r runs the
policy of policy_cases on its `obs.chunk(WORLD_SIZE)[RANK]` rows, takes the same rows of the legal-action mask
`legal.chunk(WORLD_SIZE)[RANK]` and fills the logits of illegal actions with -inf before it picks an action.

TEST INFRASTRUCTURE.  These functions are the semantic definition of @kt.mapped("mlp", bias=True, output="actions",
mask="legal") and of @kt.mapped("mlp", bias=True, output="sample", seed="seed", mask="legal"): masked =
logits.masked_fill(~legal, -inf) on the bf16 logits, then torch.argmax, or Gumbel-max over float(masked) with the
noise of the rows' global indices and log_softmax(float(masked))[action].  The oracle restatement
(oracle/ref_dispatch.spmd_call) executes them on CPU; the CUDA path must reproduce their results.
"""
import os

from policy_cases import mlp_policy_biased


def _shard_of(t):
    """This rank's rows of t, as the policy takes its rows of obs (an empty shard for ranks past the data)."""
    r, w = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    rows = t.chunk(w, dim=0)
    return rows[r] if r < len(rows) else t[:0]


def masked_logits(obs, w1, b1, w2, b2, w3, b3, legal):
    """The bf16 logits of this rank's rows with -inf in every illegal column."""
    return mlp_policy_biased(obs, w1, b1, w2, b2, w3, b3).masked_fill(~_shard_of(legal), float("-inf"))


def mlp_policy_masked_actions(obs, w1, b1, w2, b2, w3, b3, legal):
    """Greedy int64 actions of this rank's rows, over the legal actions only."""
    return masked_logits(obs, w1, b1, w2, b2, w3, b3, legal).argmax(-1)


def mlp_policy_masked_sample(obs, w1, b1, w2, b2, w3, b3, legal, seed):
    """(int64 actions, float32 log_probs) of this rank's rows sampled with `seed` from the legal actions only."""
    import torch

    from kubetorch_b200.sampling import gumbel_noise

    r, w = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    row0 = min(r * -(-obs.shape[0] // w), obs.shape[0])   # where obs.chunk(w)[r] begins
    logits = masked_logits(obs, w1, b1, w2, b2, w3, b3, legal).float()
    g = gumbel_noise(seed, row0, logits.shape[0], logits.shape[1], device=logits.device)
    actions = (logits + g).argmax(-1)
    log_probs = torch.log_softmax(logits, -1).gather(-1, actions[:, None]).squeeze(-1)
    return actions, log_probs
