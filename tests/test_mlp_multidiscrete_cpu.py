"""not-gpu: the multi-discrete categorical heads (@kt.mapped("mlp", nvec=...)) without a GPU — the semantic
definitions on 1, 3 and 4 ranks (sharding is invisible), their reduction to the single categorical at nvec = (d_out,),
the decoration option and the Python nvec checks."""
import pytest
import torch
import torch.nn.functional as F

import policy_cases
import policy_masked_cases
import policy_multidiscrete_cases as cases
import policy_value_cases
from oracle import ref_dispatch

from kubetorch_b200.sampling import gumbel_noise

D_OUT = sum(cases.NVEC)


def _policy(seed, d_in=64, d_hidden=256, d_out=D_OUT):
    """(w1, b1, w2, b2, w3, b3, wv, bv) of a small biased actor-critic."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).bfloat16()   # noqa: E731
    return (r(d_hidden, d_in, scale=0.1), r(d_hidden, scale=0.5), r(d_hidden, d_hidden, scale=0.05),
            r(d_hidden, scale=0.5), r(d_out, d_hidden, scale=0.05), r(d_out, scale=0.5), r(1, d_hidden, scale=0.05),
            r(1, scale=0.5))


def _same(a, b):
    """Equal values, NaN where the other has NaN: the same bits for these computations."""
    return a.dtype == b.dtype and a.shape == b.shape and bool(((a == b) | (a.isnan() & b.isnan())).all())


def _concat(res):
    if isinstance(res[0], torch.Tensor):
        return (torch.cat(res),)
    return tuple(torch.cat([r[k] for r in res]) for k in range(len(res[0])))


def _legal(rows, seed):
    legal = torch.rand(rows, D_OUT, generator=torch.Generator().manual_seed(seed)) < 0.5
    legal[::7, :3] = False   # group 0 without a legal action
    legal[::5] = False       # rows without any
    return legal


KINDS = ("actions", "both", "sample", "masked_actions", "masked_sample", "sample_value")


def _call(kind, p, legal, seed):
    """(body, its arguments after obs)."""
    body = getattr(cases, "mlp_policy_multidiscrete_" + kind)
    if kind in ("actions", "both"):
        return body, p[:6]
    if kind == "sample":
        return body, (*p[:6], seed)
    if kind == "masked_actions":
        return body, (*p[:6], legal)
    if kind == "masked_sample":
        return body, (*p[:6], legal, seed)
    return body, (*p, seed)


# ---- the semantic definitions ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("rows", [0, 2, 10, 13, 100])
def test_bodies_are_the_same_on_every_rank_count(kind, rows):
    """1, 3 and 4 ranks (ragged shards, and empty shards past the data) give the same concatenated outputs bit for
    bit, and those are the per-group definition over the whole batch: int64 actions [rows, G] relative to each group,
    and fp32 log-probabilities summed over the groups in group order."""
    p = _policy(rows + 31)
    obs = torch.randn(rows, 64, generator=torch.Generator().manual_seed(rows)).bfloat16()
    seed = 2**40 + rows
    legal = _legal(rows, rows + 3)
    body, args = _call(kind, p, legal, seed)
    runs = {n: _concat(ref_dispatch.spmd_call(body, obs, *args, num_proc=n)) for n in (1, 3, 4)}
    for n in (3, 4):
        assert all(_same(a, b) for a, b in zip(runs[n], runs[1])), n
    h = torch.relu(F.linear(torch.relu(F.linear(obs, p[0], p[1])), p[2], p[3]))
    y = F.linear(h, p[4], p[5])
    if kind.startswith("masked"):
        y = y.masked_fill(~legal, float("-inf"))
    got = runs[1]
    actions = got[1] if kind == "both" else got[0]
    assert actions.dtype == torch.int64 and actions.shape == (rows, len(cases.NVEC))
    for g, (lo, n) in enumerate(zip((0, 3, 4), cases.NVEC)):
        part = y[:, lo:lo + n].float()
        if "sample" in kind:
            part = part + gumbel_noise(seed, 0, rows, D_OUT)[:, lo:lo + n]
        assert torch.equal(actions[:, g], part.argmax(-1)), g
    if kind == "both":
        assert torch.equal(got[0], y)
    if "sample" in kind:
        want = sum((torch.log_softmax(y[:, lo:lo + n].float(), -1).gather(-1, actions[:, g:g + 1]).squeeze(-1)
                    for g, (lo, n) in enumerate(zip((0, 3, 4), cases.NVEC))), torch.zeros(rows))
        assert torch.allclose(got[1], want, equal_nan=True)
    if kind.startswith("masked") and rows:
        assert bool((actions[::5] == 0).all())
        if kind == "masked_sample":
            assert bool(got[1][::7].isnan().all())


@pytest.mark.parametrize("rows", [0, 13, 100])
def test_one_group_is_the_single_categorical(rows):
    """nvec = (d_out,): the grouped definitions give the bits of the single categorical's bodies, actions as [rows, 1]."""
    d_out = 9
    p = _policy(rows + 41, d_out=d_out)
    obs = torch.randn(rows, 64, generator=torch.Generator().manual_seed(rows + 1)).bfloat16()
    legal = torch.rand(rows, d_out, generator=torch.Generator().manual_seed(rows + 2)) < 0.5
    legal[::4] = False
    seed = 2**33 + rows
    env = {"RANK": "0", "WORLD_SIZE": "1"}
    from unittest import mock

    with mock.patch.dict("os.environ", env):
        y = policy_cases.mlp_policy_biased(obs, *p[:6])
        assert torch.equal(cases.grouped_actions(y, (d_out,))[:, 0], policy_cases.mlp_policy_actions(obs, *p[:6]))
        ym = policy_masked_cases.masked_logits(obs, *p[:6], legal)
        assert torch.equal(cases.grouped_actions(ym, (d_out,))[:, 0],
                           policy_masked_cases.mlp_policy_masked_actions(obs, *p[:6], legal))
        a, lp = cases.grouped_sample(ym, (d_out,), seed, 0)
        wa, wlp = policy_masked_cases.mlp_policy_masked_sample(obs, *p[:6], legal, seed)
        assert torch.equal(a[:, 0], wa) and _same(lp, wlp)
        a, lp = cases.grouped_sample(y, (d_out,), seed, 0)
        wa, wlp, _ = policy_value_cases.mlp_policy_sample_value(obs, *p, seed)
        assert torch.equal(a[:, 0], wa) and _same(lp, wlp)


# ---- decoration ----------------------------------------------------------------------------------------------------
def _body(obs, w1, b1, w2, b2, w3, b3, legal, wv, bv, seed):
    return None


@pytest.mark.parametrize("output,extra", [
    ("actions", {}), ("both", {}), ("sample", {"seed": "seed"}), ("actions", {"mask": "legal"}),
    ("sample", {"seed": 3, "mask": "legal", "value": ("wv", "bv")}),
])
@pytest.mark.parametrize("nvec", [(6,), [3, 1, 2], (1,) * 6])
def test_nvec_is_recorded_on_the_spec_as_a_tuple(output, extra, nvec):
    import kubetorch_b200 as kt
    from kubetorch_b200.mapped import mapped_spec

    spec = mapped_spec(kt.mapped("mlp", bias=True, output=output, nvec=nvec, **extra)(_body))
    assert spec.extra["nvec"] == tuple(nvec) and isinstance(spec.extra["nvec"], tuple)


BAD_NVEC = [
    ("3, 1, 2", "tuple of ints"),
    (6, "tuple of ints"),
    ((3.0, 3), "tuple of ints"),
    ((True, 5), "tuple of ints"),
    (("3", 3), "tuple of ints"),
    (None, "tuple of ints"),
    ((), "empty"),
    ([], "empty"),
    ((3, 0, 3), ">= 1"),
    ((7, -1), ">= 1"),
]


@pytest.mark.parametrize("nvec,reason", BAD_NVEC)
def test_bad_nvec_raises_at_decoration(nvec, reason):
    import kubetorch_b200 as kt

    with pytest.raises(ValueError, match=reason):
        kt.mapped("mlp", bias=True, output="actions", nvec=nvec)


@pytest.mark.parametrize("kwargs", [{}, {"output": "logits"}, {"output": "gaussian", "seed": 1, "log_std": "s"}])
def test_mapped_refuses_nvec_naming_the_output(kwargs):
    import kubetorch_b200 as kt

    with pytest.raises(ValueError, match=f'nvec= is not an option of output="{kwargs.get("output", "logits")}"'):
        kt.mapped("mlp", bias=True, nvec=(3, 3), **kwargs)


@pytest.mark.parametrize("op", ["identity", "scale", "affine"])
def test_nvec_belongs_to_the_mlp_op(op):
    import kubetorch_b200 as kt

    with pytest.raises(ValueError, match="nvec="):
        kt.mapped(op, nvec=(3, 3))


# ---- Python argument checks -----------------------------------------------------------------------------------------
def _w(d_in=256, d_hidden=1024, d_out=18):
    return (torch.zeros(d_hidden, d_in, dtype=torch.bfloat16), torch.zeros(d_out, d_hidden, dtype=torch.bfloat16))


@pytest.mark.parametrize("nvec,reason", [c for c in BAD_NVEC if c[0] is not None] + [
    ((9, 8), "sums to 17, not d_out=18"),
    ((9, 10), "sums to 19, not d_out=18"),
    ((1,) * 19, "sums to 19"),
])
@pytest.mark.parametrize("output", ["actions", "both", "sample"])
def test_check_policy_rejects_a_bad_nvec(nvec, reason, output):
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    with pytest.raises(ValueError, match=reason):
        mlp._check_policy(w1, w3, (None, None, None), output, 1 if output == "sample" else None, nvec=nvec)


@pytest.mark.parametrize("output,extra", [("logits", {}), ("gaussian", {"seed": 1})])
def test_check_policy_refuses_nvec_naming_the_output(output, extra):
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    with pytest.raises(ValueError, match=f'nvec is not an argument of output="{output}"'):
        mlp._check_policy(w1, w3, (None, None, None), output, nvec=(9, 9), **extra)


@pytest.mark.parametrize("nvec", [(18,), (9, 9), [1] * 18, (2, 7, 9)])
def test_check_policy_accepts_a_good_nvec(nvec):
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    for output, seed in (("actions", None), ("both", None), ("sample", 5)):
        assert mlp._check_policy(w1, w3, (None, None, None), output, seed, nvec=nvec) is None


def test_outputs_shape_grouped_actions():
    """_outputs allocates int64 actions [M, G] with nvec and refuses a given actions buffer of another shape."""
    from kubetorch_b200.device import mlp

    logits, actions, log_probs, values = mlp._outputs("both", 5, 18, "cpu", None, None, None, nvec=(9, 9))
    assert actions.shape == (5, 2) and actions.dtype == torch.int64 and logits.shape == (5, 18)
    assert log_probs is None and values is None
    for bad in (torch.zeros(5, dtype=torch.int64), torch.zeros(5, 3, dtype=torch.int64)):
        with pytest.raises(ValueError, match=r"actions must have shape \(5, 2\)"):
            mlp._outputs("sample", 5, 18, "cpu", None, bad, None, nvec=(9, 9))
