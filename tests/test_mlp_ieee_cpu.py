"""The reference of the MLP IEEE suite (tests/mlp_ieee_ref.py) pinned on CPU: its trunk against an fp64 restatement on
the constructed inputs, the overflow and subnormal constructions against their hand-computed results, the class
helper, and the policy_*_cases definitions returning NaN rows for NaN inputs."""
import math

import pytest
import torch

import policy_cases
import policy_critic_cases
import policy_deterministic_cases
import policy_evaluate_cases
import policy_gaussian_state_cases
import policy_td_target_cases
import policy_value_cases
from mlp_ieee_ref import (BF16_MAX, D_OUT, FINITE, FP32_ULP_AT_TIE, NAN, NEG_INF, POISON_SITES, POS_INF, SUB, TIE,
                          TIE_A, TIE_B, assert_matches, classes, overflow_case, poisoned, random_net, same_bits,
                          subnormal_case, trunk, trunk64)

NAN_F, INF = float("nan"), float("inf")


def test_classes():
    t = torch.tensor([0.0, -0.0, 1.0, NAN_F, INF, -INF, 5e-45, -3.0e38], dtype=torch.float32)
    want = [FINITE, FINITE, FINITE, NAN, POS_INF, NEG_INF, FINITE, FINITE]
    assert classes(t).tolist() == want
    assert classes(t.bfloat16()).tolist() == want


def test_assert_matches_and_same_bits_reject_what_they_should():
    a = torch.tensor([1.0, NAN_F, INF, -INF])
    assert_matches(a, a.clone(), "itself")
    for b in (torch.tensor([1.0, 0.0, INF, -INF]), torch.tensor([1.0, NAN_F, -INF, -INF]),
              torch.tensor([1.0, NAN_F, INF, 3.0]), torch.tensor([1.5, NAN_F, INF, -INF])):
        with pytest.raises(AssertionError):
            assert_matches(a, b, "other")
    same_bits(a, a.clone(), "itself")
    with pytest.raises(AssertionError):
        same_bits(torch.tensor([0.0]), torch.tensor([-0.0]), "signed zero")


def test_the_tie_construction_lands_on_the_tie():
    """TIE_A and TIE_B are bf16 values whose product is (2 - 2^-8) · 2^127, exactly halfway between the bf16 maximum and
    2^128, representable in fp32; bf16 rounding sends it to +inf and one fp32 ulp less to BF16_MAX, as .bfloat16()
    does."""
    a, b = torch.tensor(TIE_A).bfloat16(), torch.tensor(TIE_B).bfloat16()
    assert float(a) == TIE_A and float(b) == TIE_B
    assert TIE_A * TIE_B == TIE == 511 * 2.0 ** 119
    tie32 = torch.tensor(TIE, dtype=torch.float32)
    assert float(tie32) == TIE
    assert float(tie32.bfloat16()) == INF and float((-tie32).bfloat16()) == -INF
    below = torch.tensor(TIE - FP32_ULP_AT_TIE, dtype=torch.float32)
    assert float(below) == TIE - FP32_ULP_AT_TIE and float(torch.nextafter(below, tie32)) == TIE
    assert float(below.bfloat16()) == BF16_MAX == float(torch.finfo(torch.bfloat16).max)
    assert float(torch.tensor(1.5 * 2.0 ** 127, dtype=torch.float32) * 2) == INF


@pytest.mark.parametrize("layer", ["hidden", "head"])
def test_overflow_case_reference(layer):
    """The reference trunk on the overflow construction: the fp64 restatement's classes and bits, and the results the
    construction was built for."""
    net = overflow_case(layer)
    got = trunk(*net)
    same_bits(got, trunk64(*net), layer)
    g, kind = got.float(), torch.arange(got.shape[0]) % 4
    sign = torch.tensor([1.0, -1.0]).repeat(D_OUT // 2)
    if layer == "hidden":
        assert torch.equal(g[kind == 0], (sign * INF).expand(int((kind == 0).sum()), -1))
        assert torch.equal(g[kind == 1], (sign * 255 * 2.0 ** 112).expand(int((kind == 1).sum()), -1))
        assert torch.equal(g[kind == 2], (sign * INF).expand(int((kind == 2).sum()), -1))
        assert torch.equal(g[kind == 3], (sign * 1.5 * 2.0 ** 119).expand(int((kind == 3).sum()), -1))
    else:
        want = {0: [INF, -INF, 0, 0], 1: [BF16_MAX, -BF16_MAX, 0, 0], 2: [0, 0, INF, -INF],
                3: [0, 0, 1.5 * 2.0 ** 127, -1.5 * 2.0 ** 127]}
        for k, w in want.items():
            assert torch.equal(g[kind == k, :4], torch.tensor(w).expand(int((kind == k).sum()), -1)), k
        assert bool((g[:, 4:] == 0).all())


@pytest.mark.parametrize("bias", [False, True])
def test_subnormal_case_reference_is_not_flushed(bias):
    net = subnormal_case(bias)
    got = trunk(*net)
    same_bits(got, trunk64(*net), f"bias={bias}")
    g = got.double()
    m = (1 + torch.arange(got.shape[0]) % 127).double()
    assert torch.equal(g[:, 0], m * 2.0 ** -33)
    assert bool((g[:, 1] == 5 * 2.0 ** -33).all())
    assert torch.equal(g[:, 2], m * SUB) and torch.equal(g[:, D_OUT - 1], -m * SUB)
    if bias:
        assert g[0, 3:11].tolist() == [k * SUB for k in (3, 17, 33, 64, 65, 100, 126, 127)]
    else:
        assert bool((g[:, 3:11] == 0).all())


@pytest.mark.parametrize("value", [NAN_F, INF, -INF])
@pytest.mark.parametrize("site", list(POISON_SITES))
def test_poisoned_net_classes_match_fp64(site, value):
    """Random weights with a NaN or ±inf site, and NaN / ±inf observation rows: the fp32 reference's class of every
    output equals the fp64 restatement's (the sums hold no overflow, so the class cannot depend on precision), and
    its finite values are within the end-to-end bar."""
    net = poisoned(random_net(31), site, value)
    obs = torch.randn(64, 256, generator=torch.Generator().manual_seed(32)).bfloat16()
    obs[3, 10], obs[4, 20], obs[5, 30] = NAN_F, INF, -INF
    got, want = trunk(obs, *net), trunk64(obs, *net)
    assert_matches(got, want, f"{site} {value}", rtol=2 ** -7, atol=1e-2)
    assert bool(got[3].isnan().all())


# ---- the definitions keep NaN -------------------------------------------------------------------------------------
ROWS = [0, 5, 31]


@pytest.fixture
def one_rank(monkeypatch):
    monkeypatch.setenv("RANK", "0")
    monkeypatch.setenv("WORLD_SIZE", "1")


def _nan_obs(M=32, d_in=64):
    obs = torch.randn(M, d_in, generator=torch.Generator().manual_seed(3)).bfloat16()
    obs[ROWS, 7] = NAN_F
    return obs


def _rows_nan(t, what):
    t = t.float()
    hit = torch.zeros(t.shape[0], dtype=torch.bool)
    hit[ROWS] = True
    assert bool(t[hit].isnan().all()), what
    assert not bool(t[~hit].isnan().any()), what


def test_policy_definitions_give_nan_rows(one_rank):
    obs = _nan_obs()
    w1, b1, w2, b2, w3, b3 = random_net(4, d_in=64, d_hidden=256, d_out=6)
    g = torch.Generator().manual_seed(5)
    w_ls, b_ls = (torch.randn(6, 256, generator=g) * 0.02).bfloat16(), (torch.randn(6, generator=g) * 0.1).bfloat16()
    wv, bv = (torch.randn(1, 256, generator=g) * 0.02).bfloat16(), (torch.randn(1, generator=g) * 0.1).bfloat16()
    p = (obs, w1, b1, w2, b2, w3, b3)
    _rows_nan(policy_cases.mlp_policy_biased(*p), "logits")
    _rows_nan(policy_deterministic_cases.mlp_policy_deterministic(*p), "deterministic")
    for i, t in enumerate(policy_gaussian_state_cases.mlp_policy_gaussian_state_squashed(*p, w_ls, b_ls, 9)):
        _rows_nan(t, f"gaussian_state output {i}")
    _, lp, v = policy_value_cases.mlp_policy_sample_value(*p, wv, bv, 9)
    _rows_nan(lp, "sample log_probs")
    _rows_nan(v, "values")
    for i, t in enumerate(policy_evaluate_cases.mlp_policy_evaluate(*p, torch.zeros(32, dtype=torch.int64))):
        _rows_nan(t, f"evaluate output {i}")


def test_critic_and_td_definitions_give_nan_rows(one_rank):
    """d_in + d_act = 128: at some odd widths (67 on an AVX-512 host) torch's CPU bf16 F.linear lets a NaN reach the
    neighbouring row, which is torch's own behaviour and not the definition's."""
    obs, d_act = _nan_obs(), 64
    g = torch.Generator().manual_seed(6)
    act = torch.randn(32, d_act, generator=g)
    act[ROWS[1:], 0] = torch.tensor([INF, -INF])      # rows already NaN through obs stay NaN
    c = random_net(7, d_in=64 + d_act, d_hidden=256, d_out=1)
    c2 = random_net(8, d_in=64 + d_act, d_hidden=256, d_out=1)
    _rows_nan(policy_critic_cases.mlp_critic(obs, *c, act), "critic")
    actor = random_net(9, d_in=64, d_hidden=256, d_out=d_act)
    r = torch.randn(32, generator=g)
    d = torch.ones(32)                                   # done: 0 · NaN is still NaN
    _rows_nan(policy_td_target_cases.mlp_ddpg_target(obs, *c, *actor, r, d), "ddpg y")
    _rows_nan(policy_td_target_cases.mlp_td3_target(obs, *c, *actor, *c2, r, d, 9), "td3 y")
    assert not math.isnan(float(policy_td_target_cases.mlp_ddpg_target(obs, *c, *actor, r, d)[1]))
