"""not-gpu: the ε-greedy Q-network head (@kt.mapped("mlp", output="epsilon_greedy")) without a GPU — the exploration
streams against a plain-int Philox, the semantic definitions on 1, 3 and 4 ranks (sharding is invisible), the
decoration options and every Python check of mlp_forward's epsilon."""
import inspect

import pytest
import torch
import torch.nn.functional as F

import policy_epsilon_cases as cases
from oracle import ref_dispatch

import kubetorch_b200 as kt
from kubetorch_b200.sampling import explore_noise, gumbel_noise, normal_noise

M32 = 0xFFFFFFFF


# ---- the exploration streams --------------------------------------------------------------------------------------------
def _philox_int(c, k):
    """Philox4x32-10 on Python ints (Random123's round), independent of the torch restatement."""
    c, k = list(c), list(k)
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k[0]) & M32, p1 & M32, ((p0 >> 32) ^ c[3] ^ k[1]) & M32, p0 & M32]
        k = [(k[0] + 0x9E3779B9) & M32, (k[1] + 0xBB67AE85) & M32]
    return c


@pytest.mark.parametrize("seed,row0", [(0, 0), (7, 123), (2**64 - 1, 2**32 - 3), (0x1234_5678_9ABC_DEF0, 2**40 + 5)])
def test_explore_noise_is_the_documented_philox_counters(seed, row0):
    """u[r] = (2·(x >> 9) + 1)·2^-24 of word 0 of counter (i, 0, 3), and words[r, j] = word j & 1 of counter (i, j >> 1,
    2), for global row i = row0 + r, under key (seed mod 2^32, seed >> 32); row indices above 2^32 carry into word 1."""
    rows, cols = 5, 7
    u, w = explore_noise(seed, row0, rows, cols)
    assert u.dtype == torch.float32 and tuple(u.shape) == (rows,)
    assert w.dtype == torch.int64 and tuple(w.shape) == (rows, cols)
    key = (seed & M32, seed >> 32)
    for r in range(rows):
        i = row0 + r
        x = _philox_int((i & M32, i >> 32, 0, 3), key)[0]
        assert float(u[r]) == (2 * (x >> 9) + 1) * 2.0 ** -24
        for j in range(cols):
            assert int(w[r, j]) == _philox_int((i & M32, i >> 32, j >> 1, 2), key)[j & 1]


def test_explore_streams_are_new_and_sharding_independent():
    """The streams of counter word 2 and 3 are not the Gumbel (0) or Gaussian (1) draws of the same seed, and a row's
    draws depend on its global index only."""
    u, w = explore_noise(11, 0, 64, 8)
    g = gumbel_noise(11, 0, 64, 8)
    z = normal_noise(11, 0, 64, 8)
    g_u = torch.exp(-torch.exp(-g))   # the Gumbel stream's uniforms, up to rounding
    assert not torch.allclose(g_u[:, 0], u) and not torch.allclose((w >> 9).float() * 2.0 ** -23, g_u, atol=1e-3)
    assert not torch.allclose(torch.special.ndtr(z.double()).float()[:, 0], u, atol=1e-3)
    u2, w2 = explore_noise(11, 40, 24, 8)
    assert torch.equal(u2, u[40:]) and torch.equal(w2, w[40:])


# ---- the semantic definitions ------------------------------------------------------------------------------------------
def _policy(seed, d_in=64, d_hidden=256, d_out=6):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).bfloat16()   # noqa: E731
    return (r(d_hidden, d_in, scale=0.1), r(d_hidden, scale=0.5), r(d_hidden, d_hidden, scale=0.05),
            r(d_hidden, scale=0.5), r(d_out, d_hidden, scale=0.05), r(d_out, scale=0.5))


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and bool(((a == b) | (a.isnan() & b.isnan())).all())


def _concat(res):
    return tuple(torch.cat([r[k] for r in res]) for k in range(3))


def _legal(rows, d_out, seed):
    legal = torch.rand(rows, d_out, generator=torch.Generator().manual_seed(seed)) < 0.5
    if rows > 1:
        legal[1] = False            # a row with no legal action
    return legal


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("eps_kind", ["float", "tensor"])
@pytest.mark.parametrize("rows", [0, 2, 10, 13, 100])
def test_bodies_are_the_same_on_every_rank_count(masked, eps_kind, rows):
    """1, 3 and 4 ranks (ragged shards, and empty shards past the data) give the same concatenated outputs bit for bit,
    and those are the whole batch's: explore where u < ε, the legal column with the largest word there, the argmax
    elsewhere, and the (masked) Q-values of the taken and the greedy action."""
    p = _policy(rows + 5)
    obs = torch.randn(rows, 64, generator=torch.Generator().manual_seed(rows)).bfloat16()
    seed = 2**37 + rows
    eps = 0.3 if eps_kind == "float" else torch.rand(rows, generator=torch.Generator().manual_seed(1))
    legal = _legal(rows, 6, rows)
    body = cases.mlp_policy_epsilon_greedy_masked if masked else cases.mlp_policy_epsilon_greedy
    args = (*p, legal, eps) if masked else (*p, eps)
    runs = {n: _concat(ref_dispatch.spmd_call(body, obs, *args, seed, num_proc=n)) for n in (1, 3, 4)}
    for n in (3, 4):
        assert all(_same(a, b) for a, b in zip(runs[n], runs[1])), n
    h = torch.relu(F.linear(torch.relu(F.linear(obs, p[0], p[1])), p[2], p[3]))
    q = F.linear(h, p[4], p[5])
    if masked:
        q = q.masked_fill(~legal, float("-inf"))
    u, w = explore_noise(seed, 0, rows, 6)
    e = torch.full((rows,), 0.3) if eps_kind == "float" else eps
    actions, qa, qm = runs[1]
    for i in range(rows):
        lg = legal[i] if masked else torch.ones(6, dtype=torch.bool)
        g = int(q[i].argmax())
        if float(u[i]) < float(e[i]):
            want = max((int(w[i, j]), -j) for j in range(6) if lg[j])[1] * -1 if bool(lg.any()) else 0
        else:
            want = g
        assert int(actions[i]) == want, i
        assert _same(qa[i:i + 1], q[i, want:want + 1].float())
        assert _same(qm[i:i + 1], q[i, g:g + 1].float())
    if masked and rows > 1:
        assert int(actions[1]) == 0 and float(qa[1]) == float("-inf") and float(qm[1]) == float("-inf")


@pytest.mark.parametrize("eps,explores", [(0.0, False), (-1.0, False), (float("nan"), False), (1.0, True),
                                          (float("inf"), True)])
def test_epsilon_edges(eps, explores):
    """ε <= 0 and a NaN ε never explore; ε >= 1 always does (every u is below 1)."""
    q = torch.randn(64, 5, generator=torch.Generator().manual_seed(3)).bfloat16()
    actions, _, _ = cases.epsilon_greedy(q, torch.full((64,), eps), 9, 0)
    u, w = explore_noise(9, 0, 64, 5)
    assert torch.equal(actions, w.argmax(-1) if explores else q.argmax(-1))


def test_nan_q_is_greedy_but_does_not_move_exploration():
    """A NaN Q-value in a legal column is the greedy action and q_max; an exploring row ranks the words only."""
    q = torch.zeros(4, 5, dtype=torch.bfloat16)
    q[:, 3] = float("nan")
    a0, q0, m0 = cases.epsilon_greedy(q, 0.0, 5, 0)
    assert torch.equal(a0, torch.full((4,), 3)) and bool(q0.isnan().all()) and bool(m0.isnan().all())
    a1, _, m1 = cases.epsilon_greedy(q, 1.0, 5, 0)
    assert torch.equal(a1, explore_noise(5, 0, 4, 5)[1].argmax(-1)) and bool(m1.isnan().all())


# ---- kt.mapped options -------------------------------------------------------------------------------------------------
def _body(obs, w1, b1, w2, b2, w3, b3, eps, seed):
    return obs


def test_epsilon_option_at_decoration():
    from kubetorch_b200.mapped import MLP_OUTPUTS, mapped_spec

    assert "epsilon_greedy" in MLP_OUTPUTS
    for e in (0.05, "eps", 1, 0.0):
        spec = mapped_spec(kt.mapped("mlp", bias=True, output="epsilon_greedy", seed="seed", epsilon=e)(_body))
        assert spec.extra["epsilon"] == e and spec.extra["output"] == "epsilon_greedy"
    spec = mapped_spec(kt.mapped("mlp", bias=True, output="epsilon_greedy", seed=3, epsilon=0.1, mask="eps")(_body))
    assert spec.extra["mask"] == "eps"


E = dict(output="epsilon_greedy", seed="seed")


@pytest.mark.parametrize("kwargs,reason", [
    (dict(bias=True, output="epsilon_greedy", epsilon=0.1), "seed= is required"),
    (dict(bias=True, **E), "epsilon= is required"),
    (dict(bias=True, output="sample", seed="seed", epsilon=0.1), 'epsilon= is not an option of output="sample"'),
    (dict(bias=True, output="actions", epsilon=0.1), 'epsilon= is not an option of output="actions"'),
    (dict(bias=True, **E, epsilon=float("nan")), "NaN"),
    (dict(bias=True, **E, epsilon=True), "epsilon must be a number"),
    (dict(bias=True, **E, epsilon=[0.1]), "epsilon must be a number"),
    (dict(bias=True, **E, epsilon=0.1, value=("wv", "bv")), 'value= is not an option of output="epsilon_greedy"'),
    (dict(bias=True, **E, epsilon=0.1, nvec=(3, 3)), 'nvec= is not an option of output="epsilon_greedy"'),
    (dict(bias=True, **E, epsilon=0.1, log_std="ls"), 'log_std= is not an option of output="epsilon_greedy"'),
    (dict(bias=True, output="epsilon_greedy", seed=-1, epsilon=0.1), "seed must be an int"),
])
def test_bad_epsilon_options_raise_at_decoration(kwargs, reason):
    with pytest.raises(ValueError, match=reason):
        kt.mapped("mlp", **kwargs)


def test_epsilon_name_must_be_an_argument():
    with pytest.raises(ValueError, match="'eps_missing' is not an argument"):
        kt.mapped("mlp", bias=True, **E, epsilon="eps_missing")(_body)


@pytest.mark.parametrize("op", ["identity", "scale", "affine"])
def test_epsilon_belongs_to_the_mlp_op(op):
    with pytest.raises(ValueError, match="options of the 'mlp' op"):
        kt.mapped(op, epsilon=0.1)


# ---- mlp_forward's Python checks ---------------------------------------------------------------------------------------
def _check(output="epsilon_greedy", epsilon=0.1, obs=None, **kw):
    from kubetorch_b200.device import mlp

    w1 = torch.zeros(1024, 256, dtype=torch.bfloat16)
    w3 = torch.zeros(18, 1024, dtype=torch.bfloat16)
    obs = torch.zeros(8, 256, dtype=torch.bfloat16) if obs is None else obs
    mlp._check_policy(w1, w3, (None, None, None), output, kw.pop("seed", 1), kw.pop("log_std", None), obs=obs,
                      epsilon=epsilon, **kw)


@pytest.mark.parametrize("case,reason", [
    (dict(epsilon=None), "epsilon is required"),
    (dict(epsilon=float("nan")), "must not be NaN"),
    (dict(epsilon=True), "epsilon must be a number"),
    (dict(epsilon="0.1"), "epsilon must be a number"),
    (dict(epsilon=torch.zeros(8, dtype=torch.float64)), "float32 tensor of shape \\(8,\\)"),
    (dict(epsilon=torch.zeros(7)), "float32 tensor of shape \\(8,\\)"),
    (dict(epsilon=torch.zeros(8, 1)), "float32 tensor of shape \\(8,\\)"),
    (dict(epsilon=torch.zeros(16)[::2]), "epsilon must be contiguous"),
    (dict(epsilon=torch.zeros(8)), "must be a CUDA tensor on the device of obs"),
    (dict(seed=None), 'seed is required with output="epsilon_greedy"'),
    (dict(output="sample"), 'epsilon is not an argument of output="sample"'),
    (dict(output="actions", seed=None), 'epsilon is not an argument of output="actions"'),
    (dict(value=(torch.zeros(1, 1024, dtype=torch.bfloat16), None)), 'value is not an argument of output="epsilon_greedy"'),
    (dict(nvec=(9, 9)), 'nvec is not an argument of output="epsilon_greedy"'),
    (dict(log_std=torch.zeros(18)), 'log_std is not an argument of output="epsilon_greedy"'),
])
def test_check_policy_rejects_bad_epsilon_options(case, reason):
    with pytest.raises(ValueError, match=reason):
        _check(**case)


def test_check_policy_accepts_numbers():
    for e in (0.0, 0.05, 1, 1.0, -3.0, float("inf")):
        _check(epsilon=e)


def test_mlp_forward_and_scatter_gather_take_epsilon():
    from kubetorch_b200.device import mlp

    for fn in (mlp.mlp_forward, mlp.mlp_scatter_gather):
        assert inspect.signature(fn).parameters["epsilon"].default is None
    assert "epsilon_greedy" in mlp.OUTPUTS


def test_c_entries_are_declared():
    """The four ε-greedy entries and ktb_push_scatter_ce_sides have ctypes signatures of the header's arity."""
    from kubetorch_b200.device import lib as L

    n = {name: len(L._SIGNATURES[name][1]) for name in L._SIGNATURES}
    assert n["ktb_mlp_bf16_policy_epsilon_greedy"] == n["ktb_mlp_bf16_policy_sample"] + 2
    assert n["ktb_mlp_bf16_policy_epsilon_greedy_masked"] == n["ktb_mlp_bf16_policy_sample_masked"] + 2
    assert n["ktb_mlp_bf16_policy_epsilon_greedy_pushed"] == n["ktb_mlp_bf16_policy_sample_pushed"] + 2
    assert n["ktb_mlp_bf16_policy_epsilon_greedy_masked_pushed"] == n["ktb_mlp_bf16_policy_sample_masked_pushed"] + 2
    assert n["ktb_push_scatter_ce_sides"] == n["ktb_push_scatter_ce"] + 4
