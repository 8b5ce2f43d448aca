"""not-gpu: the masked categorical policy (@kt.mapped("mlp", mask="legal")) without a GPU — the semantic definitions
on 1, 3 and 4 ranks (sharding is invisible), their edge rows, the decoration option and the Python mask checks."""
import pytest
import torch

import policy_masked_cases
from oracle import ref_dispatch

from kubetorch_b200.sampling import gumbel_noise


def _policy(seed, d_in=64, d_hidden=256, d_out=6):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).bfloat16()   # noqa: E731
    return (r(d_hidden, d_in, scale=0.1), r(d_hidden, scale=0.5), r(d_hidden, d_hidden, scale=0.05),
            r(d_hidden, scale=0.5), r(d_out, d_hidden, scale=0.05), r(d_out, scale=0.5))


def _legal(rows, d_out, seed):
    """About half the actions legal; row 0 has none, row 1 exactly one (column 3), row 2 all of them."""
    legal = torch.rand(rows, d_out, generator=torch.Generator().manual_seed(seed)) < 0.5
    for i, row in enumerate((torch.zeros(d_out, dtype=torch.bool), torch.arange(d_out) == 3,
                             torch.ones(d_out, dtype=torch.bool))):
        if i < rows:
            legal[i] = row
    return legal


def _same(a, b):
    """Equal values, NaN where the other has NaN: the same bits for these computations."""
    return a.dtype == b.dtype and a.shape == b.shape and bool(((a == b) | (a.isnan() & b.isnan())).all())


def _whole_batch_logits(obs, p, legal):
    import torch.nn.functional as F

    h = torch.relu(F.linear(obs, p[0], p[1]))
    h = torch.relu(F.linear(h, p[2], p[3]))
    return F.linear(h, p[4], p[5]).masked_fill(~legal, float("-inf"))


# ---- the semantic definitions ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [0, 2, 10, 13, 100])
def test_masked_greedy_body_is_the_same_on_every_rank_count(rows):
    """1, 3 and 4 ranks (ragged shards, and empty shards past the data) give the same concatenated actions, equal to
    the argmax of the whole batch's masked logits: never an illegal action on a row that has a legal one, action 0 on
    a row with none."""
    p = _policy(rows + 11)
    obs = torch.randn(rows, 64, generator=torch.Generator().manual_seed(rows)).bfloat16()
    legal = _legal(rows, 6, rows + 1)
    runs = {n: ref_dispatch.spmd_call(policy_masked_cases.mlp_policy_masked_actions, obs, *p, legal, num_proc=n)
            for n in (1, 3, 4)}
    want = torch.cat(runs[1])
    for n in (3, 4):
        assert len(runs[n]) == n
        assert torch.equal(torch.cat(runs[n]), want), n
    assert want.dtype == torch.int64
    assert torch.equal(want, _whole_batch_logits(obs, p, legal).argmax(-1))
    has_legal = legal.any(-1)
    assert bool(legal[has_legal].gather(1, want[has_legal][:, None]).all())
    if rows >= 2:
        assert int(want[0]) == 0 and int(want[1]) == 3


@pytest.mark.parametrize("rows", [0, 2, 10, 13, 100])
def test_masked_sampled_body_is_the_same_on_every_rank_count(rows):
    """The sampled body: the same concatenated actions and log-probabilities bit for bit on 1, 3 and 4 ranks, equal to
    Gumbel-max over the whole batch's masked logits; no legal row draws an illegal action, a row with no legal action
    gets action 0 and a NaN log-probability, a row with one legal action gets it with log-probability exactly 0."""
    p = _policy(rows + 3)
    obs = torch.randn(rows, 64, generator=torch.Generator().manual_seed(rows)).bfloat16()
    legal = _legal(rows, 6, rows + 2)
    seed = 2**40 + rows
    runs = {n: ref_dispatch.spmd_call(policy_masked_cases.mlp_policy_masked_sample, obs, *p, legal, seed, num_proc=n)
            for n in (1, 3, 4)}

    def concat(res):
        return torch.cat([a for a, _ in res]), torch.cat([lp for _, lp in res])

    want_a, want_lp = concat(runs[1])
    for n in (3, 4):
        a, lp = concat(runs[n])
        assert torch.equal(a, want_a) and _same(lp, want_lp), n
    logits = _whole_batch_logits(obs, p, legal).float()
    assert torch.equal(want_a, (logits + gumbel_noise(seed, 0, rows, 6)).argmax(-1))
    assert _same(want_lp, torch.log_softmax(logits, -1).gather(-1, want_a[:, None]).squeeze(-1))
    has_legal = legal.any(-1)
    assert bool(legal[has_legal].gather(1, want_a[has_legal][:, None]).all())
    if rows >= 2:
        assert int(want_a[0]) == 0 and bool(torch.isnan(want_lp[0]))
        assert int(want_a[1]) == 3 and float(want_lp[1]) == 0.0


def test_masked_fill_hides_nan_and_inf_in_illegal_columns():
    """NaN and +inf logits in illegal columns do not reach the argmax or the log-softmax."""
    logits = torch.tensor([[float("nan"), 1.0, float("inf"), 0.5]]).bfloat16()
    legal = torch.tensor([[False, True, False, True]])
    masked = logits.masked_fill(~legal, float("-inf")).float()
    assert int(masked.argmax(-1)) == 1
    lp = torch.log_softmax(masked, -1)
    assert bool(torch.isfinite(lp[0, [1, 3]]).all())


# ---- decoration ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("output", ["logits", "actions", "both", "sample"])
@pytest.mark.parametrize("bias", [True, False])
def test_mask_option_is_recorded_on_the_spec(output, bias):
    import kubetorch_b200 as kt
    from kubetorch_b200.mapped import mapped_spec

    def body(obs, w1, b1, w2, b2, w3, b3, legal, seed):
        return None

    extra = {"seed": "seed"} if output == "sample" else {}
    spec = mapped_spec(kt.mapped("mlp", bias=bias, output=output, mask="legal", **extra)(body))
    assert spec.extra["mask"] == "legal" and spec.extra["output"] == output


@pytest.mark.parametrize("kwargs", [
    {"output": "gaussian", "seed": 1, "log_std": "log_std", "mask": "legal"},   # no mask with the Gaussian head
    {"output": "actions", "mask": 1},                                           # a name, not a value
    {"output": "actions", "mask": None},
])
def test_bad_mask_options_raise_at_decoration(kwargs):
    import kubetorch_b200 as kt

    with pytest.raises(ValueError, match="mask"):
        kt.mapped("mlp", bias=True, **kwargs)


def test_mask_must_name_a_parameter():
    import kubetorch_b200 as kt

    deco = kt.mapped("mlp", bias=True, output="actions", mask="legal")
    with pytest.raises(ValueError, match="mask='legal'"):
        deco(lambda obs, w1, b1, w2, b2, w3, b3, allowed: None)


@pytest.mark.parametrize("op", ["identity", "scale", "affine"])
def test_mask_belongs_to_the_mlp_op(op):
    import kubetorch_b200 as kt

    with pytest.raises(ValueError):
        kt.mapped(op, mask="legal")


# ---- Python argument checks -----------------------------------------------------------------------------------------
def _w(d_in=256, d_hidden=1024, d_out=18):
    return (torch.zeros(d_hidden, d_in, dtype=torch.bfloat16), torch.zeros(d_out, d_hidden, dtype=torch.bfloat16))


@pytest.mark.parametrize("bad,reason", [
    ("not a tensor", "torch.bool"),
    (torch.ones(8, 18, dtype=torch.uint8), "torch.bool"),
    (torch.ones(8, 17, dtype=torch.bool), "shape"),
    (torch.ones(7, 18, dtype=torch.bool), "shape"),
    (torch.ones(18, 8, dtype=torch.bool).t(), "contiguous"),
    (torch.ones(8, 18, dtype=torch.bool), "CUDA"),
])
def test_check_policy_rejects_a_bad_mask(bad, reason):
    """Each bad mask is refused for its own reason: the checks run in the order type and dtype, shape, layout, device,
    so a CPU tensor reaches the device check only when everything before it holds."""
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    obs = torch.zeros(8, 256, dtype=torch.bfloat16)
    for output, seed in (("logits", None), ("actions", None), ("both", None), ("sample", 1)):
        with pytest.raises(ValueError, match=reason):
            mlp._check_policy(w1, w3, (None, None, None), output, seed, mask=bad, obs=obs)


def test_check_policy_needs_obs_with_a_mask():
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    with pytest.raises(ValueError, match="obs"):
        mlp._check_policy(w1, w3, (None, None, None), "actions", mask=torch.ones(8, 18, dtype=torch.bool))


def test_check_policy_rejects_a_mask_with_the_gaussian_head():
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    obs = torch.zeros(8, 256, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="gaussian"):
        mlp._check_policy(w1, w3, (None, None, None), "gaussian", 1, None, torch.ones(8, 18, dtype=torch.bool), obs)


def test_check_policy_keeps_its_positional_signature():
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    assert mlp._check_policy(w1, w3, (None, None, None), "sample", 5) is None
    assert mlp._check_policy(w1, w3, (None, None, None), "actions", None, None, None, None) is None
