"""The Q(s, a) critic heads without a GPU: the bodies of tests/policy_critic_cases.py give the same bits on any number
of ranks, the twin's minimum is torch.minimum's, and kt.mapped() and _check_policy refuse the options a critic does not
take, each with a message that names its reason."""
import math
import os
from unittest import mock

import pytest
import torch

import kubetorch_b200 as kt
from kubetorch_b200.device import mlp
from policy_critic_cases import critic_q, mlp_critic, mlp_critic_nobias, mlp_critic_twin, q_min


def _case(d_in=64, d_act=6, d_hidden=256, rows=37, bias=True, seed=0):
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(rows, d_in, generator=g).bfloat16()
    act = torch.rand(rows, d_act, generator=g) * 2 - 1

    def critic():
        w = [(torch.randn(*s, generator=g) * 0.05).bfloat16()
             for s in ((d_hidden, d_in + d_act), (d_hidden, d_hidden), (1, d_hidden))]
        b = [(torch.randn(n, generator=g) * 0.1).bfloat16() if bias else None for n in (d_hidden, d_hidden, 1)]
        return (w[0], b[0], w[1], b[1], w[2], b[2])

    return obs, act, critic(), critic()


def _ranks(body, n, *args):
    outs = []
    for r in range(n):
        with mock.patch.dict(os.environ, {"RANK": str(r), "WORLD_SIZE": str(n)}):
            outs.append(body(*args))
    return outs


def _bits(t):
    return t.view(torch.int32)


@pytest.mark.parametrize("n", [1, 3, 4])
@pytest.mark.parametrize("d_act", [1, 6, 17, 64])
def test_critic_body_is_independent_of_the_rank_count(n, d_act):
    obs, act, c1, c2 = _case(d_act=d_act)
    want = critic_q(obs, act, *c1)
    got = torch.cat(_ranks(mlp_critic, n, obs, *c1, act))
    assert torch.equal(_bits(got), _bits(want))
    twin = _ranks(mlp_critic_twin, n, obs, *c1, act, *c2)
    for i, w in enumerate((want, critic_q(obs, act, *c2))):
        assert torch.equal(_bits(torch.cat([t[i] for t in twin])), _bits(w)), i


@pytest.mark.parametrize("n", [1, 3, 4])
def test_bias_free_critic_body_is_independent_of_the_rank_count(n):
    obs, act, c1, _ = _case(bias=False)
    want = critic_q(obs, act, *c1)
    got = torch.cat(_ranks(mlp_critic_nobias, n, obs, c1[0], c1[2], c1[4], act))
    assert torch.equal(_bits(got), _bits(want))


def test_critic_body_rounds_the_action_once_to_nearest_even():
    """The body's action block is act.to(torch.bfloat16): a tie between two bf16 values goes to the even one."""
    obs, act, c1, _ = _case(d_act=2, rows=2)
    act = torch.tensor([[1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8], [-(1 + 2.0 ** -8), 0.0]])
    x = act.to(torch.bfloat16).float()
    assert x.tolist() == [[1.0, 1 + 2.0 ** -6], [-1.0, 0.0]]


SPECIAL = [0.0, -0.0, math.inf, -math.inf, math.nan, 1.0, -2.5]


def test_twin_minimum_restatement_equals_torch_minimum():
    """q_min's restatement and torch.minimum of each pair (0-d CPU tensors) agree bit for bit on every ordered pair of
    ±0, ±inf, NaN and numbers: q1 on ties (signed zeros included), NaN when either is.  (torch.minimum's vectorised CPU
    kernel returns q2 on a tie of signed zeros, so the pairs are taken one at a time; on every other pair the two paths
    agree, which the last assertion checks.)"""
    a = torch.tensor([x for x in SPECIAL for _ in SPECIAL])
    b = torch.tensor([y for _ in SPECIAL for y in SPECIAL])
    got = q_min(a, b)
    want = torch.stack([torch.minimum(x, y) for x, y in zip(a, b)])
    nan = want.isnan()
    assert torch.equal(got.isnan(), nan)
    assert torch.equal(_bits(got[~nan]), _bits(want[~nan]))
    zeros = (a == 0) & (b == 0)
    assert torch.equal(_bits(got[zeros]), _bits(a[zeros]))   # q1 on a tie of zeros
    vec = torch.minimum(a, b)
    assert torch.equal(_bits(vec[~zeros & ~nan]), _bits(want[~zeros & ~nan]))


REFUSED = {"seed": 1, "mask": "legal", "value": ("wv", "bv"), "nvec": (2, 2), "log_std": "ls",
           "log_std_bounds": (-5.0, 2.0), "squash": True, "epsilon": 0.1, "taken": "taken", "noise": 0.2,
           "noise_clip": 0.5}


@pytest.mark.parametrize("option", list(REFUSED))
def test_mapped_critic_refuses_the_options_of_other_heads(option):
    with pytest.raises(ValueError, match=f'{option}= is not an option of output="critic"'):
        kt.mapped("mlp", bias=True, output="critic", action="act", **{option: REFUSED[option]})


def test_mapped_critic_requires_action_as_a_name():
    with pytest.raises(ValueError, match='action= is required with output="critic"'):
        kt.mapped("mlp", bias=True, output="critic")
    with pytest.raises(ValueError, match="action must be the name of a call argument"):
        kt.mapped("mlp", bias=True, output="critic", action=3)


@pytest.mark.parametrize("output", ["logits", "actions", "sample", "deterministic"])
@pytest.mark.parametrize("option", ["action", "twin"])
def test_mapped_refuses_action_and_twin_naming_the_output(output, option):
    extra = dict(seed=1) if output == "sample" else {}
    with pytest.raises(ValueError, match=f'{option}= is not an option of output="{output}"'):
        kt.mapped("mlp", bias=True, output=output, **extra, **{option: "act" if option == "action" else ("a",) * 6})


def test_mapped_refuses_action_on_elementwise_ops():
    with pytest.raises(ValueError, match="options of the 'mlp' op"):
        kt.mapped("scale", alpha=2.0, action="act")


@pytest.mark.parametrize("bias,twin", [(True, ("v1", "c1", "v2")), (False, ("v1", "c1", "v2", "c2", "v3", "c3")),
                                       (True, "v1"), (True, ("v1", "c1", "v2", "c2", "v3", 3))])
def test_mapped_twin_names_six_or_three_arguments(bias, twin):
    with pytest.raises(ValueError, match="twin must name the second critic's"):
        kt.mapped("mlp", bias=bias, output="critic", action="act", twin=twin)


def test_mapped_critic_names_must_be_arguments():
    deco = kt.mapped("mlp", bias=True, output="critic", action="act", twin=("v1", "c1", "v2", "c2", "v3", "c9"))
    with pytest.raises(ValueError, match="'c9' is not an argument"):
        deco(mlp_critic_twin)
    assert kt.mapped("mlp", bias=True, output="critic", action="act",
                     twin=("v1", "c1", "v2", "c2", "v3", "c3"))(mlp_critic_twin) is mlp_critic_twin
    assert kt.mapped("mlp", output="critic", action="act")(mlp_critic_nobias) is mlp_critic_nobias


def _check(output="critic", w3_rows=1, **kw):
    obs, act, c1, _ = _case()
    w1, b1, w2, b2, w3, b3 = c1
    if w3_rows != 1:
        w3, b3 = torch.zeros(w3_rows, w3.shape[1], dtype=torch.bfloat16), None
    mlp._check_policy(w1, w3, (b1, b2, b3), output, obs=obs, w2=w2, **kw)


@pytest.mark.parametrize("option", ["seed", "mask", "value", "nvec", "log_std", "log_std_bounds", "squash", "epsilon",
                                    "taken", "noise", "noise_clip"])
def test_check_policy_critic_refuses_the_options_of_other_heads(option):
    with pytest.raises(ValueError, match=f'{option} is not an argument of output="critic"'):
        _check(**{option: REFUSED[option]})


def test_check_policy_critic_refuses_a_wide_head_and_requires_action():
    obs, act, _, _ = _case()
    with pytest.raises(ValueError, match=r"d_out=4: a critic's w3 is \[1, d_hidden\]"):
        _check(w3_rows=4, action=act)
    with pytest.raises(ValueError, match='action is required with output="critic"'):
        _check()


@pytest.mark.parametrize("output", ["logits", "sample", "deterministic"])
def test_check_policy_refuses_action_naming_the_output(output):
    extra = dict(seed=1) if output == "sample" else {}
    with pytest.raises(ValueError, match=f'action is not an argument of output="{output}"'):
        _check(output=output, action=torch.zeros(37, 6), **extra)
