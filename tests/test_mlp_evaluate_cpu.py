"""not-gpu: evaluating given actions under the MLP policy heads (@kt.mapped("mlp", output="evaluate" or
"gaussian_evaluate")) without a GPU — the semantic definitions against torch.distributions on 1, 3 and 4 ranks, the
decoration options and every Python check of mlp_forward's taken."""
import inspect
import math

import pytest
import torch
import torch.nn.functional as F

import policy_evaluate_cases as cases
from oracle import ref_dispatch

import kubetorch_b200 as kt


def _policy(seed, d_in=64, d_hidden=256, d_out=6):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).bfloat16()   # noqa: E731
    return (r(d_hidden, d_in, scale=0.1), r(d_hidden, scale=0.5), r(d_hidden, d_hidden, scale=0.05),
            r(d_hidden, scale=0.5), r(d_out, d_hidden, scale=0.05), r(d_out, scale=0.5))


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and bool(((a == b) | (a.isnan() & b.isnan())).all())


def _concat(res, k):
    return tuple(torch.cat([r[i] for r in res]) for i in range(k))


# ---- the semantic definitions ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [0, 2, 10, 13, 100])
def test_categorical_body_is_the_same_on_every_rank_count(rows):
    """1, 3 and 4 ranks give the same concatenated outputs bit for bit, and those are Categorical(logits)'s."""
    p = _policy(rows + 1)
    obs = torch.randn(rows, 64, generator=torch.Generator().manual_seed(rows)).bfloat16()
    acts = torch.randint(0, 6, (rows,), generator=torch.Generator().manual_seed(2))
    runs = {n: _concat(ref_dispatch.spmd_call(cases.mlp_policy_evaluate, obs, *p, acts, num_proc=n), 2)
            for n in (1, 3, 4)}
    for n in (3, 4):
        assert all(_same(a, b) for a, b in zip(runs[n], runs[1])), n
    if rows == 0:   # torch.distributions refuses an empty batch
        return
    h = torch.relu(F.linear(torch.relu(F.linear(obs, p[0], p[1])), p[2], p[3]))
    dist = torch.distributions.Categorical(logits=F.linear(h, p[4], p[5]).float())
    lp, ent = runs[1]
    assert torch.allclose(lp, dist.log_prob(acts), atol=1e-5) and torch.allclose(ent, dist.entropy(), atol=1e-5)


@pytest.mark.parametrize("rows", [0, 3, 13, 64])
def test_masked_multidiscrete_value_body_is_per_group_categoricals(rows):
    """Each group is a Categorical of its masked columns; the row sums them; the values are the critic's."""
    nvec = (3, 1, 4, 2)
    p = _policy(rows + 7, d_out=sum(nvec))
    g = torch.Generator().manual_seed(rows + 3)
    wv, bv = (torch.randn(1, 256, generator=g) * 0.05).bfloat16(), torch.randn(1, generator=g).bfloat16()
    obs = torch.randn(rows, 64, generator=g).bfloat16()
    legal = torch.rand(rows, sum(nvec), generator=g) < 0.7
    acts = torch.stack([torch.randint(0, n, (rows,), generator=g) for n in nvec], -1)
    for k, lo in enumerate((0, 3, 4, 8)):   # every taken action legal, so every term is finite
        legal[torch.arange(rows), lo + acts[:, k]] = True
    runs = {n: _concat(ref_dispatch.spmd_call(cases.mlp_policy_evaluate_masked_nvec_value, obs, *p, wv, bv, legal,
                                              acts, nvec, num_proc=n), 3) for n in (1, 3)}
    assert all(_same(a, b) for a, b in zip(runs[3], runs[1]))
    if rows == 0:   # torch.distributions refuses an empty batch
        return
    h = torch.relu(F.linear(torch.relu(F.linear(obs, p[0], p[1])), p[2], p[3]))
    y = F.linear(h, p[4], p[5]).masked_fill(~legal, float("-inf")).float()
    lp, ent, values = runs[1]
    want_lp, want_ent, lo = torch.zeros(rows), torch.zeros(rows), 0
    for k, n in enumerate(nvec):
        dist = torch.distributions.Categorical(logits=y[:, lo:lo + n])
        want_lp += dist.log_prob(acts[:, k])
        want_ent += dist.entropy()
        lo += n
    assert torch.allclose(lp, want_lp, atol=1e-5) and torch.allclose(ent, want_ent, atol=1e-5)
    assert _same(values, F.linear(h, wv, bv).float().squeeze(-1))


def test_categorical_edge_rows():
    """An illegal action's log-probability is -inf; one legal column gives lp = 0 and H = 0; n equal logits H = log n;
    a group with no legal column gives NaN, as torch's log_softmax of an all -inf row."""
    y = torch.tensor([[1.0, 2.0, 3.0], [1.0, 2.0, 3.0], [0.5, 0.5, 0.5], [1.0, 2.0, 3.0]]).bfloat16()
    legal = torch.tensor([[True, False, True], [False, True, False], [True, True, True], [False, False, False]])
    lp, ent = cases.evaluate(y, torch.tensor([1, 1, 2, 0]), legal)
    assert float(lp[0]) == -math.inf
    assert float(lp[1]) == 0.0 and float(ent[1]) == 0.0
    assert math.isclose(float(ent[2]), math.log(3), rel_tol=1e-6)
    assert math.isnan(float(lp[3])) and math.isnan(float(ent[3]))


@pytest.mark.parametrize("bad", [-1, 3])
def test_out_of_range_actions_raise_in_the_body(bad):
    """The body's gather raises on an out-of-range action (the device route writes a NaN row instead)."""
    y = torch.zeros(2, 3).bfloat16()
    with pytest.raises((RuntimeError, IndexError)):
        cases.evaluate(y, torch.tensor([0, bad]))
    with pytest.raises((RuntimeError, IndexError)):
        cases.evaluate(torch.zeros(2, 5).bfloat16(), torch.tensor([[0, 0], [bad if bad < 0 else 2, 0]]), nvec=(2, 3))


@pytest.mark.parametrize("rows", [0, 5, 13])
def test_gaussian_body_is_normal(rows):
    p = _policy(rows + 11, d_out=4)
    g = torch.Generator().manual_seed(rows)
    obs = torch.randn(rows, 64, generator=g).bfloat16()
    log_std = torch.randn(4, generator=g) * 0.5
    acts = torch.randn(rows, 4, generator=g)
    runs = {n: _concat(ref_dispatch.spmd_call(cases.mlp_policy_gaussian_evaluate, obs, *p, log_std, acts,
                                              num_proc=n), 2) for n in (1, 3, 4)}
    for n in (3, 4):
        assert all(_same(a, b) for a, b in zip(runs[n], runs[1])), n
    h = torch.relu(F.linear(torch.relu(F.linear(obs, p[0], p[1])), p[2], p[3]))
    mu = F.linear(h, p[4], p[5]).double()
    z = (acts.double() - mu) / log_std.double().exp()
    want_lp = (-0.5 * z * z - log_std.double() - 0.5 * math.log(2 * math.pi)).sum(-1)
    want_ent = float((log_std.double() + 0.5 + 0.5 * math.log(2 * math.pi)).sum())
    lp, ent = runs[1]
    assert torch.allclose(lp.double(), want_lp, atol=1e-4)
    assert torch.allclose(ent.double(), torch.full((rows,), want_ent, dtype=torch.float64), atol=1e-5)


# ---- kt.mapped options -------------------------------------------------------------------------------------------------
def _body(obs, w1, b1, w2, b2, w3, b3, acts, legal, log_std):
    return obs


def test_evaluate_options_at_decoration():
    from kubetorch_b200.mapped import MLP_OUTPUTS, mapped_spec

    assert "evaluate" in MLP_OUTPUTS and "gaussian_evaluate" in MLP_OUTPUTS
    spec = mapped_spec(kt.mapped("mlp", bias=True, output="evaluate", taken="acts", mask="legal", nvec=(2, 4),
                                 value=("w3", "b3"))(_body))
    assert spec.extra["taken"] == "acts" and spec.extra["nvec"] == (2, 4)
    spec = mapped_spec(kt.mapped("mlp", bias=True, output="gaussian_evaluate", taken="acts", log_std="log_std")(_body))
    assert spec.extra["output"] == "gaussian_evaluate"


EV = dict(bias=True, output="evaluate", taken="acts")
GEV = dict(bias=True, output="gaussian_evaluate", taken="acts", log_std="log_std")


@pytest.mark.parametrize("kwargs,reason", [
    (dict(bias=True, output="evaluate"), "taken= is required"),
    (dict(bias=True, output="gaussian_evaluate", log_std="log_std"), "taken= is required"),
    (dict(bias=True, output="sample", seed=1, taken="acts"), 'taken= is not an option of output="sample"'),
    (dict(bias=True, output="actions", taken="acts"), 'taken= is not an option of output="actions"'),
    (dict(EV, taken=3), "taken must be the name of a call argument"),
    (dict(EV, seed=1), "seed= is not an option"),
    (dict(GEV, seed="seed"), "seed= is not an option"),
    (dict(EV, epsilon=0.1), 'epsilon= is not an option of output="evaluate"'),
    (dict(GEV, squash=True), 'squash= is not an option of output="gaussian_evaluate"'),
    (dict(GEV, log_std_bounds=(-5, 2)), 'log_std_bounds= is not an option of output="gaussian_evaluate"'),
    (dict(GEV, log_std=("w_ls", "b_ls")), "not a log_std=\\(w_ls, b_ls\\) pair"),
    (dict(GEV, mask="legal"), 'mask= is not an option of output="gaussian_evaluate"'),
    (dict(EV, log_std="log_std"), 'log_std= is not an option of output="evaluate"'),
    (dict(GEV, nvec=(3, 3)), 'nvec= is not an option of output="gaussian_evaluate"'),
])
def test_bad_evaluate_options_raise_at_decoration(kwargs, reason):
    with pytest.raises(ValueError, match=reason):
        kt.mapped("mlp", **kwargs)


def test_taken_name_must_be_an_argument():
    with pytest.raises(ValueError, match="'acts_missing' is not an argument"):
        kt.mapped("mlp", **dict(EV, taken="acts_missing"))(_body)


@pytest.mark.parametrize("op", ["identity", "scale", "affine"])
def test_taken_belongs_to_the_mlp_op(op):
    with pytest.raises(ValueError, match="options of the 'mlp' op"):
        kt.mapped(op, taken="acts")


# ---- mlp_forward's Python checks ---------------------------------------------------------------------------------------
def _check(output="evaluate", taken="default", obs=None, **kw):
    from kubetorch_b200.device import mlp

    w1 = torch.zeros(1024, 256, dtype=torch.bfloat16)
    w3 = torch.zeros(18, 1024, dtype=torch.bfloat16)
    obs = torch.zeros(8, 256, dtype=torch.bfloat16) if obs is None else obs
    if isinstance(taken, str):
        taken = torch.zeros(8, 18) if output == "gaussian_evaluate" else torch.zeros(8, dtype=torch.int64)
    mlp._check_policy(w1, w3, (None, None, None), output, kw.pop("seed", None), kw.pop("log_std", None), obs=obs,
                      taken=taken, **kw)


LS = torch.zeros(18)   # a CPU log_std: the checks of taken come first


@pytest.mark.parametrize("case,reason", [
    (dict(taken=None), "taken is required"),
    (dict(taken=[0] * 8), "taken must be a tensor"),
    (dict(taken=torch.zeros(8, dtype=torch.int32)), "int64 tensor of shape \\(8,\\)"),
    (dict(taken=torch.zeros(7, dtype=torch.int64)), "int64 tensor of shape \\(8,\\)"),
    (dict(taken=torch.zeros(8, dtype=torch.int64), nvec=(9, 9)), "int64 tensor of shape \\(8, 2\\)"),
    (dict(taken=torch.zeros(16, dtype=torch.int64)[::2]), "taken must be contiguous"),
    (dict(taken=torch.zeros(2, 8, dtype=torch.int64).t(), nvec=(9, 9)), "taken must be contiguous"),
    (dict(), "taken must be a CUDA tensor on the device of obs"),
    (dict(output="gaussian_evaluate", log_std=LS, taken=torch.zeros(8, 18, dtype=torch.float64)),
     "float32 tensor of shape \\(8, 18\\)"),
    (dict(output="gaussian_evaluate", log_std=LS, taken=torch.zeros(8, 17)), "float32 tensor of shape \\(8, 18\\)"),
    (dict(output="gaussian_evaluate", log_std=LS, taken=torch.zeros(18, 8).t()), "taken must be contiguous"),
    (dict(output="gaussian_evaluate", log_std=LS), "taken must be a CUDA tensor on the device of obs"),
    (dict(seed=1), 'seed is not an argument of output="evaluate"'),
    (dict(epsilon=0.1), "epsilon is not an argument"),
    (dict(output="gaussian_evaluate", squash=True), "squash is not an argument"),
    (dict(output="gaussian_evaluate", log_std_bounds=(-5.0, 2.0)), "log_std_bounds is not an argument"),
    (dict(output="gaussian_evaluate", log_std=(torch.zeros(18, 1024), None)), "not a log_std=\\(w_ls, b_ls\\) pair"),
    (dict(output="gaussian_evaluate", mask=torch.zeros(8, 18, dtype=torch.bool)),
     'mask is not an argument of output="gaussian_evaluate"'),
    (dict(output="sample", seed=1), 'taken is not an argument of output="sample"'),
    (dict(output="actions"), 'taken is not an argument of output="actions"'),
    (dict(output="gaussian", seed=1), 'taken is not an argument of output="gaussian"'),
    (dict(output="epsilon_greedy", seed=1, epsilon=0.1), 'taken is not an argument of output="epsilon_greedy"'),
])
def test_check_policy_rejects_bad_evaluate_arguments(case, reason):
    with pytest.raises(ValueError, match=reason):
        _check(**case)


def test_mlp_forward_and_scatter_gather_take_taken():
    from kubetorch_b200.device import mlp

    for fn in (mlp.mlp_forward, mlp.mlp_scatter_gather):
        assert inspect.signature(fn).parameters["taken"].default is None
    assert inspect.signature(mlp.mlp_forward).parameters["entropy"].default is None
    assert inspect.signature(mlp.mlp_scatter_gather).parameters["entropy_root"].default is None
    assert "evaluate" in mlp.OUTPUTS and "gaussian_evaluate" in mlp.OUTPUTS


def test_c_entries_are_declared():
    """The twelve evaluating entries have ctypes signatures of the header's arity."""
    from kubetorch_b200.device import lib as L

    n = {name: len(L._SIGNATURES[name][1]) for name in L._SIGNATURES}
    for form in ("", "_pushed"):
        base = n["ktb_mlp_bf16_policy" + form]   # (logits, actions) -> (nvec, n_groups, taken, log_probs, entropy)
        assert n["ktb_mlp_bf16_policy_evaluate" + form] == base + 3
        assert n["ktb_mlp_bf16_policy_evaluate_masked" + form] == base + 4
        assert n["ktb_mlp_bf16_policy_evaluate_value" + form] == base + 4
        assert n["ktb_mlp_bf16_policy_evaluate_masked_value" + form] == base + 5
        assert n["ktb_mlp_bf16_policy_gaussian_evaluate" + form] == base + 2
        assert n["ktb_mlp_bf16_policy_gaussian_evaluate_value" + form] == base + 3
