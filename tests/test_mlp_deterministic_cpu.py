"""not-gpu: the deterministic actor head (@kt.mapped("mlp", output="deterministic")) without a GPU — the semantic
definitions on 1, 3 and 4 ranks (sharding is invisible), the header's IEEE cases in the body, the decoration options,
every Python check of the output and the two C entries' declarations."""
import inspect
import math

import pytest
import torch
import torch.nn.functional as F

import policy_deterministic_cases as cases
from oracle import ref_dispatch

from kubetorch_b200.sampling import normal_noise


def _policy(seed, d_in=64, d_hidden=256, d_out=6):
    """(w1, b1, w2, b2, w3, b3) of a small biased actor whose means span tanh's curved range."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).bfloat16()   # noqa: E731
    return (r(d_hidden, d_in, scale=0.1), r(d_hidden, scale=0.5), r(d_hidden, d_hidden, scale=0.05),
            r(d_hidden, scale=0.5), r(d_out, d_hidden, scale=0.3), r(d_out, scale=0.5))


def _same(a, b):
    """The same bits, NaN where the other has NaN."""
    return a.dtype == b.dtype and a.shape == b.shape and \
        bool(((a.view(torch.int32) == b.view(torch.int32)) | (a.isnan() & b.isnan())).all())


BODIES = {
    "noise_free": (cases.mlp_policy_deterministic, (), dict()),
    "explore": (cases.mlp_policy_deterministic_explore, ("seed",), dict(noise=0.1)),
    "smoothing": (cases.mlp_policy_deterministic_smoothing, ("seed",), dict(noise=0.2, noise_clip=0.5)),
    "unsquashed": (cases.mlp_policy_deterministic_unsquashed, ("sigma", "seed"), dict(noise=0.3, squash=False)),
}


@pytest.mark.parametrize("kind", list(BODIES))
@pytest.mark.parametrize("rows", [0, 2, 10, 13, 100])
def test_bodies_are_the_same_on_every_rank_count(kind, rows):
    """1, 3 and 4 ranks (ragged shards, and empty shards past the data) give the same concatenated actions bit for bit,
    and those are the whole batch's: t = tanh(μ) (μ unsquashed), plus (σ·z).clamp(-c, c), clamped to [-1, 1] when
    squashed."""
    body, names, opts = BODIES[kind]
    p = _policy(rows + 41)
    obs = torch.randn(rows, 64, generator=torch.Generator().manual_seed(rows)).bfloat16()
    seed = 2**41 + rows
    tail = tuple({"seed": seed, "sigma": 0.3}[n] for n in names)
    runs = {n: torch.cat(ref_dispatch.spmd_call(body, obs, *p, *tail, num_proc=n)) for n in (1, 3, 4)}
    for n in (3, 4):
        assert _same(runs[n], runs[1]), n
    h = torch.relu(F.linear(torch.relu(F.linear(obs, p[0], p[1])), p[2], p[3]))
    mu = F.linear(h, p[4], p[5]).float()
    squash = opts.get("squash", True)
    t = torch.tanh(mu) if squash else mu
    if "noise" in opts:
        t = t + (opts["noise"] * normal_noise(seed, 0, rows, 6)).clamp(-opts.get("noise_clip", math.inf),
                                                                         opts.get("noise_clip", math.inf))
    assert _same(runs[1], t.clamp(-1, 1) if squash else t)
    assert runs[1].dtype == torch.float32 and runs[1].shape == (rows, 6)
    if squash:
        assert bool((runs[1].abs() <= 1).all())


def test_body_follows_the_header_ieee_cases():
    """NaN μ stays NaN; μ = ±inf is ±1 squashed; σ = inf with c = inf is ±1 squashed and ±inf (or NaN against an
    opposite infinite μ) unsquashed; c = 0 leaves every value unchanged; σ = 0 draws nothing."""
    mu = torch.tensor([[math.nan, math.inf, -math.inf, 0.0, 0.5, -3.0]]).bfloat16().expand(50, 6)
    z = normal_noise(9, 0, 50, 6)
    a = cases.deterministic(mu, None, 0)
    assert bool(a[:, 0].isnan().all()) and torch.equal(a[:, 1:3], torch.tensor([1.0, -1.0]).expand(50, 2))
    a = cases.deterministic(mu, 9, 0, noise=math.inf)
    assert torch.equal(a[:, 1:], z[:, 1:].sign())
    a = cases.deterministic(mu, 9, 0, noise=math.inf, squash=False)
    assert torch.equal(a[:, 3:], z[:, 3:].sign() * math.inf)
    assert torch.equal(a[:, 1].isnan(), z[:, 1] < 0) and torch.equal(a[:, 2].isnan(), z[:, 2] > 0)
    for squash in (True, False):
        a = cases.deterministic(mu, 9, 0, noise=0.7, noise_clip=0.0, squash=squash)
        r = cases.deterministic(mu, None, 0, squash=squash)
        assert bool(((a == r) | (a.isnan() & r.isnan())).all()), squash
    with pytest.raises(Exception):   # a seed of None draws nothing: σ = 0 never reaches the noise
        cases.deterministic(mu, None, 0, noise=0.1)
    assert _same(cases.deterministic(mu, None, 0, noise=0.0, squash=False), mu.float())


# ---- decoration ------------------------------------------------------------------------------------------------------
def _body(obs, w1, b1, w2, b2, w3, b3, sigma, seed):
    return None


def _bias_free(obs, w1, w2, w3, sigma, seed):
    return None


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("extra", [{}, {"squash": False}, {"noise": 0.1, "seed": "seed"},
                                   {"noise": "sigma", "seed": "seed", "noise_clip": 0.5, "squash": True},
                                   {"noise": 0, "seed": 7, "noise_clip": math.inf}])
def test_deterministic_options_are_recorded_on_the_spec(extra, bias):
    import kubetorch_b200 as kt
    from kubetorch_b200.mapped import MLP_OUTPUTS, mapped_spec

    assert "deterministic" in MLP_OUTPUTS
    spec = mapped_spec(kt.mapped("mlp", bias=bias, output="deterministic", **extra)(_body if bias else _bias_free))
    assert spec.extra["output"] == "deterministic"
    for k, v in extra.items():
        assert spec.extra[k] == v


D = dict(output="deterministic")


@pytest.mark.parametrize("kwargs,reason", [
    (dict(**D, noise=0.1), "seed= exactly when it takes noise="),
    (dict(**D, seed="seed"), "seed= exactly when it takes noise="),
    (dict(**D, noise_clip=0.5), "noise_clip= is an option of noise= only"),
    (dict(**D, noise=-0.1, seed="seed"), ">= 0 and not NaN"),
    (dict(**D, noise=float("nan"), seed="seed"), ">= 0 and not NaN"),
    (dict(**D, noise=True, seed="seed"), "noise must be a number"),
    (dict(**D, noise=[0.1], seed="seed"), "noise must be a number"),
    (dict(**D, noise=0.1, seed="seed", noise_clip=-1.0), ">= 0 and not NaN"),
    (dict(**D, noise=0.1, seed="seed", noise_clip="clip"), "noise_clip must be a number"),
    (dict(**D, noise=0.1, seed=-1), "seed must be an int"),
    (dict(**D, squash=1), "True or False"),
    (dict(**D, mask="legal"), 'mask= is not an option of output="deterministic"'),
    (dict(**D, value=("wv", "bv"), bias=True), 'value= is not an option of output="deterministic"'),
    (dict(**D, nvec=(3, 3)), 'nvec= is not an option of output="deterministic"'),
    (dict(**D, log_std="log_std"), 'log_std= is not an option of output="deterministic"'),
    (dict(**D, log_std_bounds=(-1, 1)), 'log_std_bounds= is not an option of output="deterministic"'),
    (dict(**D, epsilon=0.1), 'epsilon= is not an option of output="deterministic"'),
    (dict(**D, taken="acts"), 'taken= is not an option of output="deterministic"'),
    (dict(output="gaussian", seed="seed", log_std="log_std", noise=0.1), 'noise= is not an option of output="gaussian"'),
    (dict(output="sample", seed="seed", noise_clip=0.5), 'noise_clip= is not an option of output="sample"'),
    (dict(output="sample", seed="seed", squash=True), 'squash= is not an option of output="sample"'),
])
def test_bad_deterministic_options_raise_at_decoration(kwargs, reason):
    import kubetorch_b200 as kt

    with pytest.raises(ValueError, match=reason):
        kt.mapped("mlp", **kwargs)


@pytest.mark.parametrize("op", ["identity", "scale", "affine"])
@pytest.mark.parametrize("option", [{"noise": 0.1}, {"noise_clip": 0.5}])
def test_noise_options_belong_to_the_mlp_op(op, option):
    import kubetorch_b200 as kt

    with pytest.raises(ValueError, match="options of the 'mlp' op"):
        kt.mapped(op, **option)


def test_a_named_noise_must_be_a_parameter():
    import kubetorch_b200 as kt

    deco = kt.mapped("mlp", bias=True, output="deterministic", noise="sd", seed="seed")
    with pytest.raises(ValueError, match="'sd' is not an argument"):
        deco(_body)


# ---- Python argument checks --------------------------------------------------------------------------------------------
def _check(**kw):
    from kubetorch_b200.device import mlp

    w1, w3 = torch.zeros(1024, 256, dtype=torch.bfloat16), torch.zeros(18, 1024, dtype=torch.bfloat16)
    mlp._check_policy(w1, w3, (None, None, None), kw.pop("output", "deterministic"), **kw)


@pytest.mark.parametrize("kw,reason", [
    (dict(noise=0.1), "seed exactly when it takes noise"),
    (dict(seed=1), "seed exactly when it takes noise"),
    (dict(noise_clip=0.5), "noise_clip is an option of noise only"),
    (dict(noise=0.1, seed=2**64), "seed must be an int"),
    (dict(noise=0.1, seed=True), "seed must be an int"),
    (dict(noise="0.1", seed=1), "noise must be a number"),
    (dict(noise=False, seed=1), "noise must be a number"),
    (dict(noise=-1e-30, seed=1), "noise must be >= 0"),
    (dict(noise=float("nan"), seed=1), "noise must be >= 0"),
    (dict(noise=0.1, seed=1, noise_clip=float("nan")), "noise_clip must be >= 0"),
    (dict(noise=0.1, seed=1, noise_clip=-0.5), "noise_clip must be >= 0"),
    (dict(noise=0.1, seed=1, noise_clip=torch.tensor(0.5)), "noise_clip must be a number"),
    (dict(squash="yes"), "squash must be True or False"),
    (dict(mask=torch.ones(4, 18, dtype=torch.bool)), "mask is not an argument"),
    (dict(value=(None, None)), "value is not an argument"),
    (dict(nvec=(9, 9)), "nvec is not an argument"),
    (dict(log_std=torch.zeros(18)), "log_std is not an argument"),
    (dict(log_std_bounds=(-1.0, 1.0)), "log_std_bounds is not an argument"),
    (dict(epsilon=0.5), "epsilon is not an argument"),
    (dict(taken=torch.zeros(4, 18)), "taken is not an argument"),
    (dict(output="gaussian", seed=1, noise=0.1), 'noise is not an argument of output="gaussian"'),
    (dict(output="logits", noise_clip=1.0), 'noise_clip is not an argument of output="logits"'),
    (dict(output="sample", seed=1, squash=True), 'squash is not an argument of output="sample"'),
])
def test_check_policy_rejects_bad_deterministic_arguments(kw, reason):
    with pytest.raises(ValueError, match=reason):
        _check(**kw)


@pytest.mark.parametrize("kw", [{}, dict(squash=False), dict(noise=0.0, seed=0), dict(noise=0.2, noise_clip=0.5, seed=5),
                                dict(noise=math.inf, noise_clip=0, seed=2**64 - 1, squash=True)])
def test_check_policy_accepts_good_deterministic_arguments(kw):
    _check(**kw)


def test_entry_arguments_and_defaults():
    """_det's defaults (σ = 0, c = +inf, squashed), the entry each form picks, and the arguments it passes; both entries
    are declared in the header, exported by the library and have ctypes prototypes of the documented layout."""
    import ctypes

    from kubetorch_b200.device import lib as L
    from kubetorch_b200.device import mlp

    assert mlp._det(None, None, None) == (0.0, math.inf, 1)
    assert mlp._det(0.2, 0.5, False) == (0.2, 0.5, 0)
    ptr = lambda t: 0 if t is None else 1234   # noqa: E731
    entry, args = mlp._head("deterministic", None, object(), None, None, 17, None, ptr, det=(0.0, math.inf, 1))
    assert entry == "ktb_mlp_bf16_policy_deterministic" and args == (0.0, math.inf, 1, 0, 17, 1234)
    entry, args = mlp._head("deterministic", None, object(), None, 5, 0, None, ptr, pushed=True, det=(0.2, 0.5, 0))
    assert entry == "ktb_mlp_bf16_policy_deterministic_pushed" and args == (0.2, 0.5, 0, 5, 0, 1234)
    header = open(inspect.getfile(L).replace("kubetorch_b200/device/lib.py", "include/ktb200.h")).read()
    lib = L.load()
    for name in ("ktb_mlp_bf16_policy_deterministic", "ktb_mlp_bf16_policy_deterministic_pushed"):
        assert f"int {name}(" in header and hasattr(lib, name)
        restype, argtypes = L._SIGNATURES[name]
        assert restype is ctypes.c_int
    plain_args = L._SIGNATURES["ktb_mlp_bf16_policy_deterministic"][1]
    assert len(plain_args) == 21 and plain_args[12:15] == [ctypes.c_float, ctypes.c_float, ctypes.c_int]
    pushed_args = L._SIGNATURES["ktb_mlp_bf16_policy_deterministic_pushed"][1]
    assert len(pushed_args) == 26 and pushed_args[13:16] == [ctypes.c_float, ctypes.c_float, ctypes.c_int]


def test_mlp_forward_and_scatter_gather_take_the_new_options():
    """Both take noise and noise_clip by keyword, default None, and return the actions tensor (views) alone."""
    from kubetorch_b200.device import mlp

    for fn in (mlp.mlp_forward, mlp.mlp_scatter_gather):
        params = inspect.signature(fn).parameters
        assert params["noise"].default is None and params["noise_clip"].default is None
    assert "deterministic" in mlp.OUTPUTS
    actions = torch.zeros(3, 2)
    assert mlp._result("deterministic", None, actions, None) is actions
