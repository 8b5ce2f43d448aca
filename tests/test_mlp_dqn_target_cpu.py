"""The DQN-target head without a GPU: the header's fp32 restatement of y equals the torch expression on random and
special values; the bodies of tests/policy_dqn_target_cases.py give the same bits on any number of ranks; the ctypes
prototypes match the header; kt.mapped() and _check_policy take exactly the options of output="dqn_target" and refuse
the rest with a reason; and the supervisor passes online=, reward=, done= and gamma= only with this output."""
import ctypes
import math
import os
import re
from unittest import mock

import pytest
import torch

import kubetorch_b200 as kt
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp
from kubetorch_b200.mapped import MLP_FORMS, MLP_TAKES
from oracle import ref_dispatch
from policy_dqn_target_cases import (dqn_target, header_y, mlp_double_dqn_target, mlp_double_dqn_target_masked,
                                     mlp_dqn_target, mlp_dqn_target_masked)
from test_mlp_options_cpu import _call, _want

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "ktb200.h")
SPECIAL = [0.0, -0.0, 1.0, -1.5, 1e30, -1e-30, math.inf, -math.inf, math.nan]


def _bits(t):
    return t.view(torch.int32)


def _same(got, want):
    nan = want.isnan()
    assert torch.equal(got.isnan(), nan)
    assert torch.equal(_bits(got[~nan]), _bits(want[~nan]))


# ---- the formula ----------------------------------------------------------------------------------------------------
def _grid():
    """Every combination of special and random r, d, q: 9^3 rows, then 4096 random ones."""
    g = torch.Generator().manual_seed(1)
    s = torch.tensor(SPECIAL, dtype=torch.float32)
    grid = torch.cartesian_prod(s, s, s)
    rnd = torch.randn(4096, 3, generator=g) * torch.tensor([3.0, 1.0, 50.0])
    rnd[:, 1] = torch.randint(0, 2, (4096,), generator=g).float()
    x = torch.cat([grid, rnd])
    return [x[:, i].contiguous() for i in range(3)]


@pytest.mark.parametrize("gamma", [0.99, 0.0, 1.0, 0.9])
def test_header_restatement_equals_the_torch_expression(gamma):
    r, d, q = _grid()
    want = header_y(r, d, gamma, q)
    # one column per row: the gather reads q itself, widened exactly from bf16
    qb = q.bfloat16()
    _same(dqn_target(qb[:, None], r, d, gamma), header_y(r, d, gamma, qb.float()))
    _same(r + gamma * (1 - d) * q, want)


def test_selection_rules():
    """Ties to the lowest column, the first NaN wins, -0 equals +0, all -inf or no legal column gives column 0, and the
    target's value is read unmasked."""
    nan, inf = math.nan, math.inf
    q = torch.tensor([[1.0, 3.0, 3.0, 2.0],
                      [1.0, nan, 5.0, nan],
                      [-0.0, 0.0, -1.0, -2.0],
                      [-inf, -inf, -inf, -inf],
                      [4.0, 9.0, 8.0, 7.0],
                      [4.0, 9.0, 8.0, 7.0]]).bfloat16()
    legal = torch.ones(6, 4, dtype=torch.bool)
    legal[4] = False                     # a terminal state with no legal action
    legal[5, 1] = False                  # the best column is illegal
    r = torch.arange(6, dtype=torch.float32)
    d = torch.tensor([0.0, 0.0, 0.0, 0.0, 1.0, 0.0])
    y = dqn_target(q, r, d, 1.0, legal=legal)
    want_cols = [1, 1, 0, 0, 0, 2]
    want = r + (1 - d) * q.float()[torch.arange(6), torch.tensor(want_cols)]
    _same(y, want)
    assert float(y[4]) == 4.0            # done = 1 with no legal action: y = r, not 0 * -inf
    assert math.isnan(float(y[1]))       # DQN: the NaN column is picked and scored
    # Double DQN scores the NaN column the online network picks with the target's value there
    qt = torch.tensor([[1.0, 2.0, 3.0]]).bfloat16()
    qo = torch.tensor([[0.0, nan, 9.0]]).bfloat16()
    _same(dqn_target(qt, torch.zeros(1), torch.zeros(1), 0.5, q_online=qo), torch.tensor([1.0]))


def test_infinite_q_with_done_or_zero_gamma_is_nan():
    q = torch.tensor([[math.inf], [-math.inf], [math.inf], [math.inf]]).bfloat16()
    r = torch.ones(4)
    d = torch.tensor([1.0, 1.0, 0.0, 0.0])
    y = dqn_target(q, r, d, 0.99)
    assert y[:2].isnan().all() and y[2] == math.inf
    assert dqn_target(q[3:], r[3:], d[3:], 0.0).isnan().all()


def test_dqn_equals_double_dqn_with_online_equal_to_target():
    g = torch.Generator().manual_seed(2)
    q = (torch.randn(300, 18, generator=g) * 3).bfloat16()
    q[::7, 3] = math.nan
    legal = torch.rand(300, 18, generator=g) < 0.6
    r, d = torch.randn(300, generator=g), (torch.rand(300, generator=g) < 0.3).float()
    for lg in (None, legal):
        _same(dqn_target(q, r, d, 0.99, q_online=q, legal=lg), dqn_target(q, r, d, 0.99, legal=lg))


def test_reward_of_shape_m_1_gives_y_of_that_shape():
    q = torch.randn(5, 3).bfloat16()
    y = dqn_target(q, torch.zeros(5, 1), torch.zeros(5, 1), 0.9)
    assert y.shape == (5, 1)


# ---- the bodies on any number of ranks --------------------------------------------------------------------------------
def _case(d_in=64, d_out=18, d_hidden=256, rows=37, seed=0):
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(rows, d_in, generator=g).bfloat16()

    def net():
        shapes = ((d_hidden, d_in), (d_hidden,), (d_hidden, d_hidden), (d_hidden,), (d_out, d_hidden), (d_out,))
        return tuple((torch.randn(*s, generator=g) * 0.05).bfloat16() for s in shapes)

    legal = torch.rand(rows, d_out, generator=g) < 0.5
    legal[::5] = False
    r = torch.randn(rows, generator=g)
    d = (torch.rand(rows, generator=g) < 0.3).float()
    return obs, net(), net(), legal, r, d


@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_bodies_through_the_oracle_are_independent_of_the_rank_count(n):
    obs, t, o, legal, r, d = _case()
    for body, args in ((mlp_dqn_target, (obs, *t, r, d)), (mlp_dqn_target_masked, (obs, *t, legal, r, d)),
                       (mlp_double_dqn_target, (obs, *t, *o, r, d)),
                       (mlp_double_dqn_target_masked, (obs, *t, *o, legal, r, d))):
        with mock.patch.dict(os.environ, {"RANK": "0", "WORLD_SIZE": "1"}):
            want = body(*args)
        got = ref_dispatch.spmd_call(body, *args, num_proc=n, serialization="pickle")
        assert len(got) == n
        assert torch.equal(_bits(torch.cat(got)), _bits(want)), (body.__name__, n)


# ---- the C ABI ----------------------------------------------------------------------------------------------------------
ENTRIES = ("ktb_mlp_dqn_target_scratch_bytes", "ktb_mlp_bf16_dqn_target", "ktb_mlp_bf16_dqn_target_pushed",
           "ktb_mlp_bf16_dqn_target_masked", "ktb_mlp_bf16_dqn_target_masked_pushed")


def _header_params(name):
    text = open(HEADER).read()
    m = re.search(r"\b" + name + r"\(([^)]*)\);", text)
    assert m, name
    return [p.strip() for p in m.group(1).split(",")]


@pytest.mark.parametrize("name", ENTRIES)
def test_ctypes_prototypes_match_the_header(name):
    params = _header_params(name)
    argtypes = L._SIGNATURES[name][1]
    assert len(argtypes) == len(params), (name, len(argtypes), len(params))
    for p, t in zip(params, argtypes):
        if "*" in p:
            assert t in (ctypes.c_void_p,), (name, p, t)
        elif p.startswith("float"):
            assert t is ctypes.c_float, (name, p, t)
        elif p.startswith("size_t"):
            assert t is ctypes.c_size_t, (name, p, t)
        elif p.startswith("int "):
            assert t is ctypes.c_int, (name, p, t)


def test_entries_take_mask_and_rd_where_the_header_says():
    plain = _header_params("ktb_mlp_bf16_dqn_target_masked")
    assert [p.split()[-1].lstrip("*") for p in plain[12:22]] == \
        ["oW1", "ob1", "oW2", "ob2", "oW3", "ob3", "mask", "reward", "done", "gamma"]
    pushed = _header_params("ktb_mlp_bf16_dqn_target_masked_pushed")
    assert [p.split()[-1].lstrip("*") for p in pushed[19:23]] == ["mask_offset", "rd_offset", "gamma", "y"]


# ---- options ------------------------------------------------------------------------------------------------------------
def test_the_option_row():
    assert MLP_TAKES[("dqn_target", None)] == dict(reward=True, done=True, gamma=True, online=False, mask=False)
    assert MLP_FORMS["online"] == "names"


OTHERS = [o for o in MLP_FORMS if o not in MLP_TAKES[("dqn_target", None)]]
DECO = dict(seed=1, log_std="ls", value=("wv", "bv"), nvec=(2, 2), log_std_bounds=(-5.0, 2.0), squash=True,
            epsilon=0.1, taken="t", noise=0.1, noise_clip=0.5, action="a", twin=("t1", "tb1", "t2", "tb2", "t3", "tb3"),
            actor=("a1", "ab1", "a2", "ab2", "a3", "ab3"), policy="deterministic", alpha=0.2)
PARAMS = ("obs", "w1", "b1", "w2", "b2", "w3", "b3", "o1", "ob1", "o2", "ob2", "o3", "ob3", "legal", "r", "d", "ls",
          "wv", "bv", "t", "a", "t1", "tb1", "t2", "tb2", "t3", "tb3", "a1", "ab1", "a2", "ab2", "a3", "ab3")


def _body(*params):
    ns = {}
    exec(f"def body({', '.join(params)}):\n    pass", ns)
    return ns["body"]


def _mapped(**over):
    kw = dict(bias=True, output="dqn_target", online=("o1", "ob1", "o2", "ob2", "o3", "ob3"), mask="legal", reward="r",
              done="d", gamma=0.99)
    kw.update(over)
    return kt.mapped("mlp", **{k: v for k, v in kw.items() if v is not None})(_body(*PARAMS))


def test_mapped_accepts_dqn_and_double_dqn_targets():
    _mapped()
    _mapped(online=None, mask=None)
    kt.mapped("mlp", output="dqn_target", online=("o1", "o2", "o3"), reward="r", done="d", gamma=0.5)(
        _body("obs", "w1", "w2", "w3", "o1", "o2", "o3", "r", "d"))


@pytest.mark.parametrize("option", OTHERS)
def test_mapped_refuses_every_other_option(option):
    if option == "alpha":
        pytest.skip("mapped()'s alpha= is the element-wise ops' scale with every output but td_target")
    with pytest.raises(ValueError) as e:
        _mapped(**{option: DECO[option]})
    assert f'{option}= is not an option of output="dqn_target", which takes' in str(e.value), str(e.value)


@pytest.mark.parametrize("option", ["reward", "done", "gamma"])
def test_mapped_reports_a_missing_required_option(option):
    with pytest.raises(ValueError, match=f'{option}= is required with output="dqn_target"'):
        _mapped(**{option: None})


MAPPED_REFUSALS = [
    (dict(online=("o1", "o2", "o3")), "online must name the online network's 6 call arguments"),
    (dict(online="o1"), "online must name the online network's 6"),
    (dict(gamma=math.nan), "gamma must be a finite number, got nan"),
    (dict(gamma="g"), "gamma must be a finite number"),
    (dict(reward=3), "reward must be the name of a call argument"),
    (dict(mask="nope"), "'nope' is not an argument"),
]


@pytest.mark.parametrize("over,msg", MAPPED_REFUSALS, ids=[m for _, m in MAPPED_REFUSALS])
def test_mapped_refuses_malformed_options_with_a_reason(over, msg):
    with pytest.raises(ValueError) as e:
        _mapped(**over)
    assert msg in str(e.value), str(e.value)


@pytest.mark.parametrize("output", sorted({o for o, _ in MLP_TAKES} - {"dqn_target"}))
def test_online_is_refused_by_every_other_output(output):
    policy = dict(policy="deterministic") if output == "td_target" else {}
    with pytest.raises(ValueError) as e:
        kt.mapped("mlp", output=output, online=("o1", "o2", "o3"), **policy)(_body(*PARAMS))
    assert f'online= is not an option of output="{output}"' in str(e.value), str(e.value)
    w1, w3 = torch.zeros(64, 32, dtype=torch.bfloat16), torch.zeros(4, 64, dtype=torch.bfloat16)
    with pytest.raises(ValueError) as e:
        mlp._check_policy(w1, w3, (None,) * 3, output, online=(None,) * 6,
                          td=(None, "deterministic" if output == "td_target" else None, None, None, None, None))
    assert f'online is not an argument of output="{output}"' in str(e.value), str(e.value)


def _nets_meta(d_in=64, d_out=18, d_hidden=256, rows=37, bias=True):
    obs, t, o, legal, r, d = _case(d_in, d_out, d_hidden, rows)
    if not bias:
        t = (t[0], None, t[2], None, t[4], None)
        o = (o[0], None, o[2], None, o[4], None)
    return obs, t, o, legal, r, d


def _check(bias=True, **over):
    """_check_policy of a masked Double DQN target over CPU tensors patched to look like CUDA tensors."""
    obs, t, o, legal, r, d = _nets_meta(bias=bias)
    kw = dict(output="dqn_target", obs=obs, mask=legal, online=o, td=(None, None, r, d, 0.99, None))
    kw.update(over)
    with mock.patch.object(torch.Tensor, "is_cuda", property(lambda self: True)):
        mlp._check_policy(t[0], t[4], (t[1], t[3], t[5]), kw.pop("output"), w2=t[2], **kw)


def test_a_well_formed_target_passes_the_checks():
    _check()
    _check(online=None)
    _check(mask=None)
    _check(bias=False)


def _td(r=None, d=None, gamma=0.99):
    obs, t, o, legal, rr, dd = _nets_meta()
    return (None, None, rr if r is None else r, dd if d is None else d, gamma, None)


CHECK_REFUSALS = [
    (dict(seed=1), 'seed is not an argument of output="dqn_target", which takes reward, done, gamma, online, mask'),
    (dict(epsilon=0.1), 'epsilon is not an argument of output="dqn_target"'),
    (dict(twin=(None,) * 6), 'twin is not an argument of output="dqn_target"'),
    (dict(action=torch.zeros(37, 6)), 'action is not an argument of output="dqn_target"'),
    (dict(td=(None, None, None, None, 0.99, None)), 'reward is required with output="dqn_target"'),
    (dict(td=(None, "deterministic") + _td()[2:]), 'policy is not an argument of output="dqn_target"'),
    (dict(td=_td(gamma=math.inf)), "gamma must be a finite number"),
    (dict(online=(None,) * 3), "online must be (w1, b1, w2, b2, w3, b3) of the online network"),
    (dict(online=(torch.zeros(256, 64, dtype=torch.bfloat16), None) + (None,) * 4),
     "online: b1 is given exactly when the target network's is"),
    (dict(td=_td(r=torch.zeros(37, dtype=torch.float64))), "reward must be a float32 tensor"),
    (dict(td=_td(d=torch.zeros(37, 1))), "reward and done must have one shape"),
    (dict(mask=torch.ones(37, 17, dtype=torch.bool)), "mask must have shape (37, 18)"),
    (dict(mask=torch.ones(37, 18, dtype=torch.uint8)), "mask must be a torch.bool tensor"),
]


@pytest.mark.parametrize("over,msg", CHECK_REFUSALS, ids=[m for _, m in CHECK_REFUSALS])
def test_check_policy_refuses_with_a_reason(over, msg):
    with pytest.raises(ValueError) as e:
        _check(**over)
    assert msg in str(e.value), str(e.value)


def test_online_weights_must_match_the_target_shapes():
    obs, t, o, legal, r, d = _nets_meta()
    bad = (o[0], o[1], o[2], o[3], o[4][:17].contiguous(), o[5][:17].contiguous())
    with pytest.raises(ValueError, match=r"online: w3 must be a contiguous CUDA bfloat16 tensor of shape \(18, 256\)"):
        _check(online=bad)


def test_a_d_out_past_256_is_refused():
    obs, t, o, legal, r, d = _case(d_out=257)
    with mock.patch.object(torch.Tensor, "is_cuda", property(lambda self: True)):
        with pytest.raises(ValueError, match="d_out=257"):
            mlp._check_policy(t[0], t[4], (t[1], t[3], t[5]), "dqn_target", obs=obs, w2=t[2],
                              td=(None, None, r, d, 0.99, None))


# ---- the supervisor ---------------------------------------------------------------------------------------------------
BIASED = ("obs", "w1", "b1", "w2", "b2", "w3", "b3")


def test_supervisor_passes_the_target_options_with_dqn_target_only():
    v, args, kwargs = _call(dict(bias=True, output="dqn_target", online=("o1", "ob1", "o2", "ob2", "o3", "ob3"),
                                 mask="legal", reward="r", done="d", gamma=0.9),
                            BIASED + ("o1", "ob1", "o2", "ob2", "o3", "ob3", "legal", "r", "d"))
    assert args == (v["obs"], v["w1"], v["w2"], v["w3"])
    want = _want(v, "dqn_target", mask=v["legal"], reward=v["r"], done=v["d"], gamma=0.9,
                 online=tuple(v[n] for n in ("o1", "ob1", "o2", "ob2", "o3", "ob3")))
    assert kwargs == want, (kwargs, want)


def test_supervisor_expands_a_bias_free_online_network_and_leaves_it_none_for_dqn():
    v, args, kwargs = _call(dict(output="dqn_target", online=("o1", "o2", "o3"), reward="r", done="d", gamma=0.5),
                            ("obs", "w1", "w2", "w3", "o1", "o2", "o3", "r", "d"))
    assert kwargs == _want(v, "dqn_target", bias=False, reward=v["r"], done=v["d"], gamma=0.5,
                           online=(v["o1"], None, v["o2"], None, v["o3"], None))
    v, args, kwargs = _call(dict(bias=True, output="dqn_target", reward="r", done="d", gamma=0.5), BIASED + ("r", "d"))
    assert kwargs == _want(v, "dqn_target", reward=v["r"], done=v["d"], gamma=0.5, online=None)


def test_supervisor_keeps_online_from_every_other_output():
    v, args, kwargs = _call(dict(bias=True, output="epsilon_greedy", seed=3, epsilon=0.1), BIASED)
    assert "online" not in kwargs and "reward" not in kwargs
    v, args, kwargs = _call(dict(output="td_target", policy="deterministic", actor=("a1", "a2", "a3"), reward="r",
                                 done="d", gamma=0.99), ("obs", "w1", "w2", "w3", "a1", "a2", "a3", "r", "d"))
    assert "online" not in kwargs and kwargs["reward"] is v["r"]
