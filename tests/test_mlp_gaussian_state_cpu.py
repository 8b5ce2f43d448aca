"""not-gpu: the state-dependent Gaussian policy head (@kt.mapped("mlp", output="gaussian", log_std=("w_ls", "b_ls")))
without a GPU — the semantic definitions on 1, 3 and 4 ranks (sharding is invisible), the tanh correction, the
interleaved head and its cache, the decoration options and every Python check of the pair form."""
import math

import pytest
import torch
import torch.nn.functional as F

import policy_gaussian_state_cases as cases
from oracle import ref_dispatch

from kubetorch_b200.sampling import normal_noise


def _policy(seed, d_in=64, d_hidden=256, d_out=6):
    """(w1, b1, w2, b2, w3, b3, w_ls, b_ls, wv, bv) of a small biased actor with a log-std head and a critic."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).bfloat16()   # noqa: E731
    return (r(d_hidden, d_in, scale=0.1), r(d_hidden, scale=0.5), r(d_hidden, d_hidden, scale=0.05),
            r(d_hidden, scale=0.5), r(d_out, d_hidden, scale=0.05), r(d_out, scale=0.5),
            r(d_out, d_hidden, scale=0.2), r(d_out, scale=2.0), r(1, d_hidden, scale=0.05), r(1, scale=0.5))


def _same(a, b):
    """Equal values, NaN where the other has NaN: the same bits for these computations."""
    return a.dtype == b.dtype and a.shape == b.shape and bool(((a == b) | (a.isnan() & b.isnan())).all())


def _trunk(obs, p):
    return torch.relu(F.linear(torch.relu(F.linear(obs, p[0], p[1])), p[2], p[3]))


def _concat(res, n):
    return tuple(torch.cat([r[k] for r in res]) for k in range(n))


# ---- the semantic definitions ------------------------------------------------------------------------------------------
BODIES = {
    "unsquashed": (cases.mlp_policy_gaussian_state, False, False),
    "squashed": (cases.mlp_policy_gaussian_state_squashed, True, False),
    "squashed_value": (cases.mlp_policy_gaussian_state_squashed_value, True, True),
}


@pytest.mark.parametrize("kind", list(BODIES))
@pytest.mark.parametrize("rows", [0, 2, 10, 13, 100])
def test_bodies_are_the_same_on_every_rank_count(kind, rows):
    """1, 3 and 4 ranks (ragged shards, and empty shards past the data) give the same concatenated outputs bit for bit,
    and those are the whole batch's: u = μ + exp(clamp(ℓ, -20, 2))·z, tanh(u) when squashed, and the log-density with
    its correction."""
    body, squash, valued = BODIES[kind]
    p = _policy(rows + 31)
    obs = torch.randn(rows, 64, generator=torch.Generator().manual_seed(rows)).bfloat16()
    seed = 2**41 + rows
    args = p if valued else p[:8]
    n_out = 3 if valued else 2
    runs = {n: _concat(ref_dispatch.spmd_call(body, obs, *args, seed, num_proc=n), n_out) for n in (1, 3, 4)}
    for n in (3, 4):
        assert all(_same(a, b) for a, b in zip(runs[n], runs[1])), n
    h = _trunk(obs, p)
    mu = F.linear(h, p[4], p[5]).float()
    ls = F.linear(h, p[6], p[7]).float().clamp(-20.0, 2.0)
    z = normal_noise(seed, 0, rows, 6)
    u = mu + torch.exp(ls) * z
    lp = (-0.5 * z * z - ls - 0.5 * math.log(2 * math.pi)).sum(-1)
    if squash:
        au = u.abs()
        lp = lp - (2 * (math.log(2) - au - torch.log1p(torch.exp(-2 * au)))).sum(-1)
    assert _same(runs[1][0], torch.tanh(u) if squash else u)
    assert _same(runs[1][1], lp)
    if valued:
        assert torch.equal(runs[1][2], F.linear(h, p[8], p[9]).float()[:, 0])


def test_tanh_correction_is_exact_and_finite():
    """2·(log 2 - |u| - softplus(-2|u|)) is log(1 - tanh²u) in fp64 wherever the latter is finite, is even in u, and
    stays finite where tanh(u) rounds to ±1 in fp32, unlike the fp32 log(1 - tanh²u).  (Near u = 0 both sides cancel
    to about 2u², so the fp64 agreement is relative to that cancellation.)"""
    u = torch.tensor([0.0, 1e-3, 0.5, 3.0, 9.0, 20.0, 80.0], dtype=torch.float64)
    c = 2 * (math.log(2) - u.abs() - F.softplus(-2 * u.abs()))
    assert torch.allclose(c[:5], torch.log1p(-torch.tanh(u[:5]) ** 2), rtol=1e-9, atol=1e-15)
    assert torch.equal(c, 2 * (math.log(2) - (-u).abs() - F.softplus(-2 * (-u).abs())))
    u32 = u.float()
    assert bool(torch.isfinite(2 * (math.log(2) - u32.abs() - F.softplus(-2 * u32.abs()))).all())
    assert torch.tanh(u32[-2:]).eq(1.0).all() and torch.isinf(torch.log(1 - torch.tanh(u32[-2:]) ** 2)).all()


def test_interleaved_head_gives_the_mean_and_log_std_columns():
    """F.linear over W3s = [w3_0; w_ls_0; ...] and its interleaved bias: columns 2j and 2j + 1 are the mean's and
    the log-std's column j, bit for bit (one bf16 rounding per output, with its own bias)."""
    from kubetorch_b200.device import mlp

    p = _policy(7)
    h = _trunk(torch.randn(50, 64, generator=torch.Generator().manual_seed(7)).bfloat16(), p)
    w3s, b3s = mlp._stacked_head(p[4], p[5], w_ls=p[6], b_ls=p[7])
    y = F.linear(h, w3s, b3s)
    assert torch.equal(y[:, 0::2], F.linear(h, p[4], p[5])) and torch.equal(y[:, 1::2], F.linear(h, p[6], p[7]))
    mlp._stacked_heads.clear()


# ---- the interleaved head and its cache ------------------------------------------------------------------------------
@pytest.fixture
def heads():
    from kubetorch_b200.device import mlp

    saved = dict(mlp._stacked_heads)
    mlp._stacked_heads.clear()
    yield mlp
    mlp._stacked_heads.clear()
    mlp._stacked_heads.update(saved)


def test_interleaved_head_layout(heads):
    """W3s rows alternate w3 and w_ls, W3sv adds wv last; the biases likewise; without biases b3s is None."""
    p = _policy(11)
    w3s, b3s = heads._stacked_head(p[4], p[5], w_ls=p[6], b_ls=p[7])
    assert w3s.shape == (12, 256) and w3s.is_contiguous() and b3s.shape == (12,)
    assert torch.equal(w3s[0::2], p[4]) and torch.equal(w3s[1::2], p[6])
    assert torch.equal(b3s[0::2], p[5]) and torch.equal(b3s[1::2], p[7])
    w3sv, b3sv = heads._stacked_head(p[4], p[5], p[8], p[9], p[6], p[7])
    assert w3sv.shape == (13, 256) and torch.equal(w3sv[:12], w3s) and torch.equal(w3sv[12:], p[8])
    assert torch.equal(b3sv[:12], b3s) and torch.equal(b3sv[12:], p[9])
    w3s, b3s = heads._stacked_head(p[4], None, w_ls=p[6], b_ls=None)
    assert b3s is None and torch.equal(w3s[1::2], p[6])


def test_interleaved_head_follows_in_place_updates_with_one_entry(heads):
    """An in-place update of any of w3, b3, w_ls, b_ls, wv, bv rewrites the head in place (its own _version moves on,
    so copies on other devices follow), and the cache keeps one entry per head."""
    p = list(_policy(12))

    def get():
        return heads._stacked_head(p[4], p[5], p[8], p[9], p[6], p[7])

    w, b = get()
    again = get()
    assert again[0] is w and again[1] is b
    for i in (6, 7, 4, 5, 8, 9):
        v0 = (w._version, b._version)
        p[i].add_(1.0)
        got = get()
        assert got[0] is w and got[1] is b and (w._version, b._version) != v0, i
        assert torch.equal(w[0:12:2], p[4]) and torch.equal(w[1:12:2], p[6]) and torch.equal(w[12:], p[8]), i
        assert torch.equal(b[0:12:2], p[5]) and torch.equal(b[1:12:2], p[7]) and torch.equal(b[12:], p[9]), i
        assert len(heads._stacked_heads) == 1
    heads._stacked_head(p[4], p[5], w_ls=p[6], b_ls=p[7])   # the same w3 with another head: still one entry
    assert len(heads._stacked_heads) == 1


# ---- decoration ------------------------------------------------------------------------------------------------------
def _body(obs, w1, b1, w2, b2, w3, b3, w_ls, b_ls, wv, bv, seed):
    return None


@pytest.mark.parametrize("extra", [{}, {"squash": True}, {"log_std_bounds": (-5, 1)}, {"value": ("wv", "bv")},
                                   {"squash": False, "log_std_bounds": (-20.0, 2.0), "value": ("wv", "bv")}])
def test_state_options_are_recorded_on_the_spec(extra):
    import kubetorch_b200 as kt
    from kubetorch_b200.mapped import mapped_spec

    spec = mapped_spec(kt.mapped("mlp", bias=True, output="gaussian", seed="seed", log_std=("w_ls", "b_ls"),
                                 **extra)(_body))
    assert tuple(spec.extra["log_std"]) == ("w_ls", "b_ls")
    if "log_std_bounds" in extra:
        assert spec.extra["log_std_bounds"] == tuple(float(b) for b in extra["log_std_bounds"])
    if "squash" in extra:
        assert spec.extra["squash"] is extra["squash"]


G = dict(output="gaussian", seed="seed")


@pytest.mark.parametrize("kwargs,reason", [
    (dict(bias=True, **G, log_std=("w_ls",)), "one call argument or two"),
    (dict(bias=True, **G, log_std=("w_ls", 1)), "one call argument or two"),
    (dict(bias=True, **G, log_std=("a", "b", "c")), "one call argument or two"),
    (dict(bias=False, **G, log_std=("w_ls", "b_ls")), "bias=True"),
    (dict(bias=True, **G, log_std="log_std", squash=True), "state-dependent"),
    (dict(bias=True, **G, log_std="log_std", log_std_bounds=(-5, 1)), "state-dependent"),
    (dict(bias=True, output="sample", seed="seed", squash=True), 'squash= is not an option of output="sample"'),
    (dict(bias=True, **G, log_std=("w_ls", "b_ls"), log_std_bounds=(1.0,)), "two numbers"),
    (dict(bias=True, **G, log_std=("w_ls", "b_ls"), log_std_bounds=(True, 2.0)), "two numbers"),
    (dict(bias=True, **G, log_std=("w_ls", "b_ls"), log_std_bounds="(-20, 2)"), "two numbers"),
    (dict(bias=True, **G, log_std=("w_ls", "b_ls"), log_std_bounds=(float("nan"), 2.0)), "NaN"),
    (dict(bias=True, **G, log_std=("w_ls", "b_ls"), log_std_bounds=(2.0, -2.0)), "low <= high"),
    (dict(bias=True, **G, log_std=("w_ls", "b_ls"), squash=1), "True or False"),
])
def test_bad_state_options_raise_at_decoration(kwargs, reason):
    import kubetorch_b200 as kt

    with pytest.raises(ValueError, match=reason):
        kt.mapped("mlp", **kwargs)


@pytest.mark.parametrize("op", ["identity", "scale", "affine"])
@pytest.mark.parametrize("option", [{"squash": True}, {"log_std_bounds": (-1, 1)}])
def test_state_options_belong_to_the_mlp_op(op, option):
    import kubetorch_b200 as kt

    with pytest.raises(ValueError, match="options of the 'mlp' op"):
        kt.mapped(op, **option)


def test_log_std_pair_must_name_parameters():
    import kubetorch_b200 as kt

    deco = kt.mapped("mlp", bias=True, output="gaussian", seed="seed", log_std=("w_ls", "ls_bias"))
    with pytest.raises(ValueError, match="'ls_bias' is not an argument"):
        deco(_body)


# ---- Python argument checks --------------------------------------------------------------------------------------------
def _w(d_out=18, d_hidden=1024):
    return (torch.zeros(d_hidden, 256, dtype=torch.bfloat16), torch.zeros(d_out, d_hidden, dtype=torch.bfloat16))


def _check(d_out=18, log_std=None, biased=True, output="gaussian", value=None, **kw):
    from kubetorch_b200.device import mlp

    w1, w3 = _w(d_out)
    b3 = torch.zeros(d_out, dtype=torch.bfloat16) if biased else None
    if log_std is None:
        log_std = (torch.zeros(d_out, 1024, dtype=torch.bfloat16), b3)
    mlp._check_policy(w1, w3, (None, None, b3), output, 1, log_std, value=value, **kw)


def _zw(*shape, dtype=torch.bfloat16):
    return torch.zeros(*shape, dtype=dtype)


@pytest.mark.parametrize("case,reason", [
    (dict(output="sample"), 'log_std is not an argument of output="sample"'),
    (dict(log_std=(_zw(18, 1024),)), "tensor or \\(w_ls, b_ls\\)"),
    (dict(log_std=(_zw(18, 1024), _zw(18), _zw(18))), "tensor or \\(w_ls, b_ls\\)"),
    (dict(d_out=129), "1 to 128 actions"),
    (dict(d_out=128, value=(_zw(1, 1024), _zw(1))), "1 to 127 actions"),
    (dict(log_std=(_zw(18, 1024), None)), "b_ls is given exactly when b3 is"),
    (dict(biased=False, log_std=(_zw(18, 1024), _zw(18))), "b_ls is given exactly when b3 is"),
    (dict(log_std=(_zw(18, 1024, dtype=torch.float32), _zw(18))), "bfloat16 tensor of shape \\(18, 1024\\)"),
    (dict(log_std=(_zw(17, 1024), _zw(18))), "bfloat16 tensor of shape \\(18, 1024\\)"),
    (dict(log_std=(_zw(18, 512), _zw(18))), "bfloat16 tensor of shape \\(18, 1024\\)"),
    (dict(log_std=(_zw(1024, 18).t(), _zw(18))), "w_ls must be contiguous"),
    (dict(log_std=(_zw(18, 1024), _zw(18))), "w_ls must be a CUDA tensor"),
    (dict(log_std=("w", _zw(18))), "bfloat16 tensor"),
])
def test_check_policy_rejects_a_bad_log_std_pair(case, reason):
    with pytest.raises(ValueError, match=reason):
        _check(**case)


@pytest.mark.parametrize("kw,reason", [
    (dict(log_std_bounds=(-1.0, 1.0)), "state-dependent"),
    (dict(squash=True), "state-dependent"),
    (dict(squash=False), "state-dependent"),
])
def test_bounds_and_squash_need_a_log_std_pair(kw, reason):
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    with pytest.raises(ValueError, match=reason):
        mlp._check_policy(w1, w3, (None, None, None), "gaussian", 1, torch.zeros(18), **kw)
    with pytest.raises(ValueError, match=f'{next(iter(kw))} is not an argument of output="sample"'):
        mlp._check_policy(w1, w3, (None, None, None), "sample", 1, None, **kw)


def test_mlp_forward_and_scatter_gather_take_the_new_options():
    """Both keep their positional parameters and take log_std_bounds and squash by keyword."""
    import inspect

    from kubetorch_b200.device import mlp

    for fn in (mlp.mlp_forward, mlp.mlp_scatter_gather):
        params = inspect.signature(fn).parameters
        assert params["log_std_bounds"].default is None and params["squash"].default is None
        assert params["log_std_bounds"].kind is inspect.Parameter.POSITIONAL_OR_KEYWORD
    assert mlp.LOG_STD_BOUNDS == cases.LOG_STD_BOUNDS == (-20.0, 2.0)
    assert mlp._std((None, None), None, None) == (-20.0, 2.0, 0)
    assert mlp._std((None, None), (-5, 1), True) == (-5.0, 1.0, 1)
    assert mlp._std(torch.zeros(3), None, None) is None
