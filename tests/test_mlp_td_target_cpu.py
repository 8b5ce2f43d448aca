"""The TD-target heads without a GPU: the header's fp32 restatement of y equals the torch expression users write, on
vectorised and 0-d tensors; the bodies of tests/policy_td_target_cases.py give the same bits on any number of ranks;
and kt.mapped() and _check_policy refuse the options a TD target does not take, each with a message that names its
reason."""
import math
import os
from unittest import mock

import pytest
import torch

import kubetorch_b200 as kt
from kubetorch_b200.device import mlp
from policy_td_target_cases import header_y, mlp_ddpg_target, mlp_sac_target, mlp_td3_target, td_target

SPECIAL = [0.0, -0.0, 1.0, -1.5, 1e30, -1e-30, math.inf, -math.inf, math.nan]


def _bits(t):
    return t.view(torch.int32)


def _same(got, want):
    nan = want.isnan()
    assert torch.equal(got.isnan(), nan)
    assert torch.equal(_bits(got[~nan]), _bits(want[~nan]))


def _grid():
    """Every combination of special and random r, d, t, logp: 9^4 = 6561 rows, past torch's vectorised width."""
    g = torch.Generator().manual_seed(0)
    s = torch.tensor(SPECIAL, dtype=torch.float32)
    grid = torch.cartesian_prod(s, s, s, s)
    rnd = torch.randn(4096, 4, generator=g) * torch.tensor([3.0, 1.0, 50.0, 5.0])
    rnd[:, 1] = torch.randint(0, 2, (4096,), generator=g).float()
    x = torch.cat([grid, rnd])
    return [x[:, i].contiguous() for i in range(4)]


@pytest.mark.parametrize("alpha", [None, 0.0, 0.2, 0.05])
@pytest.mark.parametrize("gamma", [0.99, 0.0, 1.0, 0.9])
def test_header_restatement_equals_the_torch_expression(gamma, alpha):
    r, d, t, lp = _grid()
    logp = None if alpha is None else lp
    want = header_y(r, d, gamma, t, alpha, logp)
    _same(td_target(r, d, gamma, t, alpha, logp), want)
    for i in range(0, r.shape[0], 97):   # the 0-d path, which differs from the vectorised one on signed-zero ties
        _same(td_target(r[i], d[i], gamma, t[i], alpha, None if logp is None else logp[i]).reshape(1), want[i:i + 1])


def test_done_with_an_infinite_t_is_nan():
    r = torch.tensor([1.0, 1.0, 1.0])
    d = torch.tensor([1.0, 1.0, 0.0])
    t = torch.tensor([math.inf, -math.inf, math.inf])
    y = header_y(r, d, 0.99, t)
    assert y[:2].isnan().all() and y[2] == math.inf
    _same(td_target(r, d, 0.99, t), y)


def _case(d_in=64, d_act=6, d_ha=256, d_hidden=256, rows=37, seed=0):
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(rows, d_in, generator=g).bfloat16()

    def lin(*shapes):
        return [(torch.randn(*s, generator=g) * 0.05).bfloat16() for s in shapes]

    def critic():
        w = lin((d_hidden, d_in + d_act), (d_hidden,), (d_hidden, d_hidden), (d_hidden,), (1, d_hidden), (1,))
        return tuple(w)

    actor = tuple(lin((d_ha, d_in), (d_ha,), (d_ha, d_ha), (d_ha,), (d_act, d_ha), (d_act,)))
    ls = tuple(lin((d_act, d_ha), (d_act,)))
    r = torch.randn(rows, generator=g)
    d = (torch.rand(rows, generator=g) < 0.3).float()
    return obs, critic(), critic(), actor, ls, r, d


def _ranks(body, n, *args):
    outs = []
    for k in range(n):
        with mock.patch.dict(os.environ, {"RANK": str(k), "WORLD_SIZE": str(n)}):
            outs.append(body(*args))
    return torch.cat(outs)


@pytest.mark.parametrize("n", [1, 3, 4])
@pytest.mark.parametrize("d_act", [1, 6, 17])
def test_bodies_are_independent_of_the_rank_count(n, d_act):
    obs, c1, c2, actor, ls, r, d = _case(d_act=d_act, d_ha=512)
    for body, args in ((mlp_td3_target, (obs, *c1, *actor, *c2, r, d, 5)),
                       (mlp_ddpg_target, (obs, *c1, *actor, r, d)),
                       (mlp_sac_target, (obs, *c1, *actor, *ls, *c2, r, d, 5, 0.2))):
        want = _ranks(body, 1, *args)
        assert want.shape == (obs.shape[0],)
        assert torch.equal(_bits(_ranks(body, n, *args)), _bits(want)), body.__name__


# ---- refusals -----------------------------------------------------------------------------------------------------
def _check(**over):
    """_check_policy of a TD3 target over meta-device stand-ins patched to look like CUDA tensors."""
    obs, c1, c2, actor, ls, r, d = _case()
    kw = dict(output="td_target", obs=obs, twin=c2, td=(actor, "deterministic", r, d, 0.99, None), seed=1, noise=0.2,
              noise_clip=0.5)
    kw.update(over)
    with mock.patch.object(torch.Tensor, "is_cuda", property(lambda self: True)):
        mlp._check_policy(c1[0], c1[4], (c1[1], c1[3], c1[5]), kw.pop("output"), w2=c1[2], **kw)


def test_a_well_formed_td3_target_passes_the_checks():
    _check()


def _td(**over):
    obs, c1, c2, actor, ls, r, d = _case()
    t = dict(actor=actor, policy="deterministic", reward=r, done=d, gamma=0.99, alpha=None)
    t.update(over)
    return tuple(t.values())


REFUSALS = [
    (dict(mask=torch.ones(37, 1, dtype=torch.bool)), "mask is not an argument"),
    (dict(value=(None, None)), "value is not an argument"),
    (dict(nvec=(1,)), "nvec is not an argument"),
    (dict(epsilon=0.1), "epsilon is not an argument"),
    (dict(taken=torch.zeros(37, dtype=torch.int64)), "taken is not an argument"),
    (dict(action=torch.zeros(37, 6)), "action is not an argument"),
    (dict(td=_td(policy="greedy")), "policy must be one of"),
    (dict(td=_td(alpha=0.2)), 'alpha is not an argument of output="td_target", policy="deterministic"'),
    (dict(log_std_bounds=(-5, 2)), 'log_std_bounds is not an argument of output="td_target", policy="deterministic"'),
    (dict(seed=None), "takes a seed exactly when it takes noise"),
    (dict(noise=-1.0), "noise must be >= 0"),
    (dict(td=_td(policy="gaussian", alpha=0.2)), 'noise is not an argument of output="td_target", policy="gaussian"'),
    (dict(td=_td(policy="gaussian"), noise=None, noise_clip=None), "alpha is required"),
    (dict(td=_td(policy="gaussian", alpha=0.2), noise=None, noise_clip=None),
     'log_std is required with output="td_target", policy="gaussian"'),
    (dict(td=_td(actor=(None,) * 5)), "actor must be (w1, b1, w2, b2, w3, b3)"),
    (dict(td=_td(reward=torch.zeros(37, dtype=torch.float64))), "reward must be a float32 tensor"),
    (dict(td=_td(done=torch.zeros(37, dtype=torch.bfloat16))), "done must be a float32 tensor"),
    (dict(td=_td(done=torch.zeros(37, 1))), "reward and done must have one shape"),
    (dict(td=_td(reward=torch.zeros(36))), "reward must be a float32 tensor of shape (37,)"),
    (dict(td=_td(gamma=math.nan)), "gamma must be a finite number"),
    (dict(td=_td(gamma="0.99")), "gamma must be a finite number, got '0.99'"),
    (dict(twin=(None,) * 3), "twin must be (w1, b1, w2, b2, w3, b3)"),
]


@pytest.mark.parametrize("over,msg", REFUSALS, ids=[m for _, m in REFUSALS])
def test_mlp_forward_checks_refuse_with_a_reason(over, msg):
    with pytest.raises(ValueError, match=None) as e:
        _check(**over)
    assert msg in str(e.value), str(e.value)


def test_the_actor_width_must_match_the_critic():
    obs, c1, c2, actor, ls, r, d = _case(d_act=6)
    bad = actor[:4] + (actor[4][:5].contiguous(), actor[5][:5].contiguous())
    with pytest.raises(ValueError, match=r"w1 must be \[d_hidden, d_in \+ d_act\]"):
        _check(td=(bad, "deterministic", r, d, 0.99, None))


def test_check_policy_refuses_td_arguments_naming_the_output():
    obs, c1, c2, actor, ls, r, d = _case()
    with mock.patch.object(torch.Tensor, "is_cuda", property(lambda self: True)):
        with pytest.raises(ValueError, match='actor is not an argument of output="logits"'):
            mlp._check_policy(c1[0], c1[4], (c1[1], c1[3], c1[5]), "logits", obs=obs, w2=c1[2],
                              td=(actor, None, None, None, None, None))


def _mapped(**over):
    kw = dict(bias=True, output="td_target", actor=("a1", "ab1", "a2", "ab2", "a3", "ab3"), policy="deterministic",
              twin=("v1", "c1", "v2", "c2", "v3", "c3"), reward="r", done="d", gamma=0.99, seed="seed", noise=0.2,
              noise_clip=0.5)
    kw.update(over)
    return kt.mapped("mlp", **{k: v for k, v in kw.items() if v is not None})(mlp_td3_target)


def test_mapped_td3_and_sac_targets_are_accepted():
    _mapped()
    _mapped(twin=None)
    kt.mapped("mlp", bias=True, output="td_target", actor=("a1", "ab1", "a2", "ab2", "a3", "ab3"), policy="gaussian",
              log_std=("w_ls", "b_ls"), twin=("v1", "c1", "v2", "c2", "v3", "c3"), reward="r", done="d", gamma=0.99,
              seed="seed", alpha="alpha")(mlp_sac_target)


MAPPED_REFUSALS = [
    (dict(mask="r"), "mask= is not an option of output=\"td_target\""),
    (dict(value=("a", "b")), "value= is not an option"),
    (dict(nvec=(1,)), "nvec= is not an option"),
    (dict(epsilon=0.1), "epsilon= is not an option"),
    (dict(taken="r"), "taken= is not an option"),
    (dict(action="r"), "action= is not an option"),
    (dict(policy="sample"), "policy= must be"),
    (dict(alpha=0.2), 'alpha= is not an option of output="td_target", policy="deterministic"'),
    (dict(log_std=("a", "b")), 'log_std= is not an option of output="td_target", policy="deterministic"'),
    (dict(seed=None), "seed= exactly when it takes noise="),
    (dict(noise=-1.0), "noise must be >= 0"),
    (dict(policy="gaussian"), 'noise= is not an option of output="td_target", policy="gaussian"'),
    (dict(policy="gaussian", noise=None, noise_clip=None, seed=None),
     'seed= is required with output="td_target", policy="gaussian"'),
    (dict(policy="gaussian", noise=None, noise_clip=None), "alpha= is required"),
    (dict(policy="gaussian", noise=None, noise_clip=None, alpha=math.inf, log_std=("a", "b")),
     "alpha must be a finite number"),
    (dict(policy="gaussian", noise=None, noise_clip=None, alpha=0.2),
     'log_std= is required with output="td_target", policy="gaussian"'),
    (dict(squash=1), "squash must be True or False"),
    (dict(actor=("a1", "a2", "a3")), "actor must name the actor's 6 call arguments"),
    (dict(twin=("v1",)), "twin must name the second critic's 6"),
    (dict(reward=None), "reward= is required"),
    (dict(done=3), "done must be the name of a call argument"),
    (dict(gamma=None), "gamma= is required"),
    (dict(gamma=math.nan), "gamma must be a finite number, got nan"),
    (dict(reward="nope"), "'nope' is not an argument"),
]


@pytest.mark.parametrize("over,msg", MAPPED_REFUSALS, ids=[m for _, m in MAPPED_REFUSALS])
def test_mapped_refuses_td_options_with_a_reason(over, msg):
    with pytest.raises(ValueError) as e:
        _mapped(**over)
    assert msg in str(e.value), str(e.value)


def test_mapped_refuses_td_options_naming_the_output():
    with pytest.raises(ValueError, match='gamma= is not an option of output="critic"'):
        kt.mapped("mlp", output="critic", action="act", gamma=0.99)(lambda obs, w1, w2, w3, act: None)
    with pytest.raises(ValueError, match="options of the 'mlp' op"):
        kt.mapped("scale", reward="r")(lambda x, r: None)
