"""not-gpu: the value head of the sampled MLP policies (@kt.mapped("mlp", value=("wv", "bv"))) without a GPU — the
semantic definitions on 1, 3 and 4 ranks (sharding is invisible), the decoration option, the stacked head and the
Python value checks."""
import pytest
import torch
import torch.nn.functional as F

import policy_value_cases
from oracle import ref_dispatch

from kubetorch_b200.sampling import gumbel_noise, normal_noise


def _policy(seed, d_in=64, d_hidden=256, d_out=6):
    """(w1, b1, w2, b2, w3, b3, wv, bv) of a small biased actor-critic."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).bfloat16()   # noqa: E731
    return (r(d_hidden, d_in, scale=0.1), r(d_hidden, scale=0.5), r(d_hidden, d_hidden, scale=0.05),
            r(d_hidden, scale=0.5), r(d_out, d_hidden, scale=0.05), r(d_out, scale=0.5), r(1, d_hidden, scale=0.05),
            r(1, scale=0.5))


def _same(a, b):
    """Equal values, NaN where the other has NaN: the same bits for these computations."""
    return a.dtype == b.dtype and a.shape == b.shape and bool(((a == b) | (a.isnan() & b.isnan())).all())


def _trunk(obs, p):
    return torch.relu(F.linear(torch.relu(F.linear(obs, p[0], p[1])), p[2], p[3]))


def _concat(res):
    return tuple(torch.cat([r[k] for r in res]) for k in range(3))


# ---- the semantic definitions ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["sample", "masked", "gaussian"])
@pytest.mark.parametrize("rows", [0, 2, 10, 13, 100])
def test_value_bodies_are_the_same_on_every_rank_count(kind, rows):
    """1, 3 and 4 ranks (ragged shards, and empty shards past the data) give the same concatenated actions,
    log-probabilities and values bit for bit; the values are the whole batch's F.linear(h, wv, bv) in fp32, and the
    actions and log-probabilities those of the policy without a value head."""
    p = _policy(rows + 21)
    obs = torch.randn(rows, 64, generator=torch.Generator().manual_seed(rows)).bfloat16()
    seed = 2**41 + rows
    legal = torch.rand(rows, 6, generator=torch.Generator().manual_seed(rows + 5)) < 0.5
    log_std = torch.linspace(-1.0, 0.5, 6)
    if kind == "sample":
        body, args = policy_value_cases.mlp_policy_sample_value, (*p, seed)
    elif kind == "masked":
        body, args = policy_value_cases.mlp_policy_masked_sample_value, (*p[:6], legal, *p[6:], seed)
    else:
        body, args = policy_value_cases.mlp_policy_gaussian_value, (*p[:6], log_std, *p[6:], seed)
    runs = {n: _concat(ref_dispatch.spmd_call(body, obs, *args, num_proc=n)) for n in (1, 3, 4)}
    for n in (3, 4):
        assert all(_same(a, b) for a, b in zip(runs[n], runs[1])), n
    actions, log_probs, values = runs[1]
    h = _trunk(obs, p)
    assert values.dtype == torch.float32 and values.shape == (rows,)
    assert torch.equal(values, F.linear(h, p[6], p[7]).float()[:, 0])
    logits = F.linear(h, p[4], p[5])
    if kind == "masked":
        logits = logits.masked_fill(~legal, float("-inf"))
    logits = logits.float()
    if kind == "gaussian":
        z = normal_noise(seed, 0, rows, 6)
        assert torch.equal(actions, logits + torch.exp(log_std) * z)
    else:
        assert torch.equal(actions, (logits + gumbel_noise(seed, 0, rows, 6)).argmax(-1))
        assert _same(log_probs, torch.log_softmax(logits, -1).gather(-1, actions[:, None]).squeeze(-1))


def test_value_is_the_last_column_of_the_stacked_head():
    """F.linear over W3v = [w3; wv] and b3v = [b3; bv]: its first d_out columns are the policy's logits and its last
    the critic's value, each bit for bit (one bf16 rounding per output, with its own bias)."""
    p = _policy(7)
    h = _trunk(torch.randn(50, 64, generator=torch.Generator().manual_seed(7)).bfloat16(), p)
    both = F.linear(h, torch.cat((p[4], p[6])), torch.cat((p[5], p[7])))
    assert torch.equal(both[:, :6], F.linear(h, p[4], p[5]))
    assert torch.equal(both[:, 6], F.linear(h, p[6], p[7])[:, 0])


# ---- decoration ----------------------------------------------------------------------------------------------------
def _body(obs, w1, b1, w2, b2, w3, b3, log_std, legal, wv, bv, seed):
    return None


@pytest.mark.parametrize("output,extra", [
    ("sample", {}), ("sample", {"mask": "legal"}), ("gaussian", {"log_std": "log_std"}),
])
def test_value_option_is_recorded_on_the_spec(output, extra):
    import kubetorch_b200 as kt
    from kubetorch_b200.mapped import mapped_spec

    spec = mapped_spec(kt.mapped("mlp", bias=True, output=output, seed="seed", value=("wv", "bv"), **extra)(_body))
    assert tuple(spec.extra["value"]) == ("wv", "bv") and spec.extra["output"] == output


@pytest.mark.parametrize("kwargs,reason", [
    ({"bias": True, "output": "actions"}, 'value= is not an option of output="actions"'),
    ({"bias": True, "output": "logits"}, 'value= is not an option of output="logits"'),
    ({"bias": True, "output": "both"}, 'value= is not an option of output="both"'),
    ({"bias": True}, 'value= is not an option of output="logits"'),
    ({"bias": False, "output": "sample", "seed": 1}, "bias=True"),
    ({"output": "sample", "seed": 1}, "bias=True"),
    ({"bias": True, "output": "sample", "seed": 1, "value_": "wv"}, "two call arguments"),
    ({"bias": True, "output": "sample", "seed": 1, "value_": ("wv",)}, "two call arguments"),
    ({"bias": True, "output": "sample", "seed": 1, "value_": ("wv", 1)}, "two call arguments"),
    ({"bias": True, "output": "sample", "seed": 1, "value_": None}, "two call arguments"),
])
def test_bad_value_options_raise_at_decoration(kwargs, reason):
    import kubetorch_b200 as kt

    kwargs = dict(kwargs)
    value = kwargs.pop("value_", ("wv", "bv"))
    with pytest.raises(ValueError, match=reason):
        kt.mapped("mlp", value=value, **kwargs)


@pytest.mark.parametrize("names", [("wv", "critic_b"), ("critic_w", "bv")])
def test_value_must_name_parameters(names):
    import kubetorch_b200 as kt

    deco = kt.mapped("mlp", bias=True, output="sample", seed="seed", value=names)
    missing = names[0] if names[0] != "wv" else names[1]
    with pytest.raises(ValueError, match=f"'{missing}' is not an argument"):
        deco(lambda obs, w1, b1, w2, b2, w3, b3, wv, bv, seed: None)


@pytest.mark.parametrize("op", ["identity", "scale", "affine"])
def test_value_belongs_to_the_mlp_op(op):
    import kubetorch_b200 as kt

    with pytest.raises(ValueError, match="value="):
        kt.mapped(op, value=("wv", "bv"))


# ---- the stacked head ------------------------------------------------------------------------------------------------
@pytest.fixture
def heads():
    from kubetorch_b200.device import mlp

    saved = dict(mlp._stacked_heads)
    mlp._stacked_heads.clear()
    yield mlp
    mlp._stacked_heads.clear()
    mlp._stacked_heads.update(saved)


def test_stacked_head_layout_and_biases(heads):
    """W3v = [w3; wv] and b3v = [b3; bv]; without biases b3v is None."""
    p = _policy(11)
    w3v, b3v = heads._stacked_head(p[4], p[5], p[6], p[7])
    assert w3v.shape == (7, 256) and w3v.is_contiguous() and b3v.shape == (7,)
    assert torch.equal(w3v[:6], p[4]) and torch.equal(w3v[6:], p[6])
    assert torch.equal(b3v[:6], p[5]) and torch.equal(b3v[6:], p[7])
    w3v, b3v = heads._stacked_head(p[4], None, p[6], None)
    assert b3v is None and torch.equal(w3v, torch.cat((p[4], p[6])))


def test_stacked_head_follows_in_place_updates_with_one_entry(heads):
    """The same head again is the same tensors; an in-place update of any of w3, b3, wv, bv rewrites them in place
    (their own _version moves on, so copies on other devices follow), and the cache keeps one entry for the head."""
    p = list(_policy(12))
    w3v, b3v = heads._stacked_head(p[4], p[5], p[6], p[7])
    again = heads._stacked_head(p[4], p[5], p[6], p[7])
    assert again[0] is w3v and again[1] is b3v
    for i in (6, 4, 7, 5):
        v0, vb0 = w3v._version, b3v._version
        p[i].add_(1.0)
        got = heads._stacked_head(p[4], p[5], p[6], p[7])
        assert got[0] is w3v and got[1] is b3v
        assert (w3v._version, b3v._version) != (v0, vb0), i
        assert torch.equal(w3v, torch.cat((p[4], p[6]))) and torch.equal(b3v, torch.cat((p[5], p[7]))), i
        assert len(heads._stacked_heads) == 1
    other = _policy(13)
    heads._stacked_head(other[4], other[5], other[6], other[7])
    assert len(heads._stacked_heads) == 2


def test_stacked_head_forgets_heads_that_are_gone(heads):
    import gc

    p = _policy(14)
    w3 = p[4].clone()
    heads._stacked_head(w3, p[5], p[6], p[7])
    del w3
    gc.collect()
    heads._stacked_head(p[4], p[5], p[6], p[7])
    assert len(heads._stacked_heads) == 1


# ---- Python argument checks -----------------------------------------------------------------------------------------
def _w(d_in=256, d_hidden=1024, d_out=18):
    return (torch.zeros(d_hidden, d_in, dtype=torch.bfloat16), torch.zeros(d_out, d_hidden, dtype=torch.bfloat16))


BIASED = (None, None, torch.zeros(18, dtype=torch.bfloat16))


@pytest.mark.parametrize("output", ["logits", "actions", "both"])
def test_check_policy_refuses_a_value_naming_the_output(output):
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    with pytest.raises(ValueError, match=f'value is not an argument of output="{output}"'):
        mlp._check_policy(w1, w3, (None, None, None), output, value=(torch.zeros(1, 1024, dtype=torch.bfloat16), None))


@pytest.mark.parametrize("bad,biases,reason", [
    ("not a pair", BIASED, "value must be"),
    ((torch.zeros(1, 1024, dtype=torch.bfloat16),), BIASED, "value must be"),
    ((torch.zeros(1, 1024, dtype=torch.bfloat16), None), BIASED, "bv is given exactly when b3 is"),
    ((torch.zeros(1, 1024, dtype=torch.bfloat16), torch.zeros(1, dtype=torch.bfloat16)), (None, None, None),
     "bv is given exactly when b3 is"),
    ((torch.zeros(1, 1024), torch.zeros(1, dtype=torch.bfloat16)), BIASED, "wv must be a bfloat16"),
    ((torch.zeros(1024, dtype=torch.bfloat16), torch.zeros(1, dtype=torch.bfloat16)), BIASED, "shape"),
    ((torch.zeros(2, 1024, dtype=torch.bfloat16), torch.zeros(1, dtype=torch.bfloat16)), BIASED, "shape"),
    ((torch.zeros(1024, 2, dtype=torch.bfloat16)[:, :1].t(), torch.zeros(1, dtype=torch.bfloat16)), BIASED,
     "contiguous"),
    ((torch.zeros(1, 1024, dtype=torch.bfloat16), torch.zeros(1, dtype=torch.bfloat16)), BIASED, "CUDA"),
])
def test_check_policy_rejects_a_bad_value(bad, biases, reason):
    """Each bad value head is refused for its own reason, in the order: its form, the bias rule, wv's dtype and
    shape, layout, device; a CPU wv reaches the device check only when everything before it holds."""
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    with pytest.raises(ValueError, match=reason):
        mlp._check_policy(w1, w3, biases, "sample", 1, value=bad)


def test_check_policy_refuses_a_value_beside_a_256_wide_policy():
    from kubetorch_b200.device import mlp

    w1, w3 = _w(d_out=256)
    with pytest.raises(ValueError, match="d_out=256"):
        mlp._check_policy(w1, w3, (None, None, None), "sample", 1,
                          value=(torch.zeros(1, 1024, dtype=torch.bfloat16), None))


def test_check_policy_keeps_its_positional_signature():
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    assert mlp._check_policy(w1, w3, (None, None, None), "sample", 5) is None
    assert mlp._check_policy(w1, w3, (None, None, None), "actions", None, None, None, None, None) is None
