"""User callables that score actions the caller already holds under the MLP policy heads (SB3's
policy.evaluate_actions, RLlib's dist.logp / dist.entropy), written as a kubetorch user writes SPMD functions: rank r
runs the trunk  Linear → ReLU → Linear → ReLU  on its `obs.chunk(WORLD_SIZE)[RANK]` rows and the head nn.Linear(d_hidden,
d_out) (w3, b3), takes its rows of the actions with `acts.chunk(WORLD_SIZE)[RANK]`, and returns (log_probs, entropy),
or (log_probs, entropy, values) with a critic (wv, bv) on the same trunk.

TEST INFRASTRUCTURE.  These functions are the semantic definition of @kt.mapped("mlp", bias=True, output="evaluate",
taken="acts") (mask="legal", nvec=(...) and value=("wv", "bv") as given) and of output="gaussian_evaluate" with
log_std="log_std".  The oracle restatement (oracle/ref_dispatch.spmd_call) executes them on CPU; the CUDA path must
reproduce their results.  An action out of range makes torch's gather raise here, where the device route, which does
not check (that would need a host synchronisation), gives a NaN row.
"""
from policy_value_cases import _shard, _trunk, _value


def evaluate(y, a, legal=None, nvec=None):
    """(float32 log_probs, float32 entropy) of the group-relative actions a [rows] or [rows, G] under the bf16 logits
    y [rows, d_out], masked by legal (True: legal) and split by nvec (None: one group of every column)."""
    import torch

    if legal is None:
        legal = torch.ones_like(y, dtype=torch.bool)
    if nvec is None:
        nvec, a = (y.shape[1],), a[:, None]
    parts = y.masked_fill(~legal, float("-inf")).float().split(list(nvec), -1)
    lp = sum(p.log_softmax(-1).gather(-1, a[:, g:g + 1])[:, 0] for g, p in enumerate(parts))
    ent = sum(torch.special.entr(p.softmax(-1)).sum(-1) for p in parts)
    return lp, ent


def gaussian_evaluate(mu, log_std, a):
    """(float32 log_probs, float32 entropy) of the fp32 actions a [rows, d_out] under Normal(mu, exp(log_std))."""
    import torch

    dist = torch.distributions.Normal(mu.float(), log_std.exp())
    return dist.log_prob(a).sum(-1), dist.entropy().sum(-1).expand(a.shape[0]).contiguous()


def mlp_policy_evaluate(obs, w1, b1, w2, b2, w3, b3, acts):
    """(log_probs, entropy) of this rank's rows' actions under the categorical policy."""
    import torch.nn.functional as F

    return evaluate(F.linear(_trunk(obs, w1, b1, w2, b2), w3, b3), _shard(acts))


def mlp_policy_evaluate_masked_nvec_value(obs, w1, b1, w2, b2, w3, b3, wv, bv, legal, acts, nvec):
    """(log_probs, entropy, values) of this rank's rows' multi-discrete actions under the masked policy, and the
    critic's values."""
    import torch.nn.functional as F

    h = _trunk(obs, w1, b1, w2, b2)
    return (*evaluate(F.linear(h, w3, b3), _shard(acts), _shard(legal), nvec), _value(h, wv, bv))


def mlp_policy_gaussian_evaluate(obs, w1, b1, w2, b2, w3, b3, log_std, acts):
    """(log_probs, entropy) of this rank's rows' continuous actions under the state-independent Gaussian policy."""
    import torch.nn.functional as F

    return gaussian_evaluate(F.linear(_trunk(obs, w1, b1, w2, b2), w3, b3), log_std, _shard(acts))
