"""-m gpu: the state-dependent Gaussian head of the bf16 MLP policy (ktb_mlp_bf16_policy_gaussian_state*,
log_std=(w_ls, b_ls) of mlp_forward, mlp_scatter_gather and kt.mapped) — tied bit for bit to the Gaussian head under a
constant log-std, its actions and log-probabilities against fp64 restatements built from the greedy kernel's logits
over the interleaved head, squashed against unsquashed, clamping, NaN and infinite cases, the tanh-Normal
distribution, every form, chunking and row split, guard bands, status codes, the public API and two GPUs."""
import math
import os
from unittest import mock

import pytest
import torch

from conftest import mapped_copy
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp
from mlp_rig import (SHIPPED_CHUNK, Head, K, config, deployed, expect_status, plain, policy_weights,  # noqa: F401
                     pushed, randn, run_guarded, tuning)

pytestmark = pytest.mark.gpu

import policy_gaussian_state_cases as cases  # noqa: E402
from oracle import ref_dispatch  # noqa: E402

from kubetorch_b200.sampling import gumbel_uniform  # noqa: E402

HALF_LOG_2PI = 0.5 * math.log(2 * math.pi)
LOG2 = math.log(2)


def _state_head(entry, valued):
    outputs = {"actions": lambda d: 4 * d, "log_probs": lambda d: 4}
    if valued:
        outputs["values"] = lambda d: 4
    return Head(entry, entry, entry + "_pushed", True, 0, outputs,
                lambda a: (a.get("lo", -20.0), a.get("hi", 2.0), a.get("squash", 0), a["seed"], a["row_base"],
                           a["actions"], a["log_probs"], *((a["values"],) if valued else ())))


STATE = _state_head("ktb_mlp_bf16_policy_gaussian_state", False)
STATE_VALUE = _state_head("ktb_mlp_bf16_policy_gaussian_state_value", True)


# ---- inputs and helpers ---------------------------------------------------------------------------------------------
def actor(seed, d_out, bias=True, ls_scale=0.05, ls_bias=(-1.5, 0.5)):
    """(W1, W2, W3), (b1, b2, b3) of mlp_rig.config, a log-std head (w_ls, b_ls) and a critic (wv, bv); b_ls spread
    over ls_bias.  Without biases b3, b_ls and bv are None."""
    w, b = config(seed, d_out, bias)
    w = (w[0], w[1], w[2] * 50)
    w_ls = randn((d_out, 1024), seed + 8, ls_scale)
    b_ls = torch.linspace(*ls_bias, d_out, device="cuda").bfloat16() if bias else None
    value = (randn((1, 1024), seed + 6, 0.02), randn((1,), seed + 7, 0.1) if bias else None)
    return w, b, (w_ls, b_ls), value


def interleaved(w, b, ls, value=None):
    """W3s / b3s (W3sv / b3sv with a value head), built as the package builds them."""
    wv, bv = value if value is not None else (None, None)
    w3s, b3s = mlp._stacked_head(w[2], b[2], wv, bv, *ls)
    return w3s.clone(), None if b3s is None else b3s.clone()


def bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def same(got, want, what):
    assert len(got) == len(want), what
    for i, (g, h) in enumerate(zip(got, want)):
        assert g.shape == h.shape, (what, i)
        nan = g.isnan() & h.isnan()
        assert bool(((bits(g) == bits(h)) | nan).all()), (what, i, (bits(g) != bits(h)).nonzero()[:4].tolist())


def state(obs, w, b, ls, seed, **kw):
    return mlp.mlp_forward(obs, *w, biases=b, output="gaussian", log_std=ls, seed=seed, **kw)


def _z64(seed, row0, rows, cols):
    return torch.special.ndtri(gumbel_uniform(seed, row0, rows, cols, device="cuda", word3=1).double())


def _c64(u):
    """log(1 - tanh²u) in fp64, as 2·(log 2 - |u| - log1p(e^-2|u|))."""
    au = u.abs()
    return 2 * (LOG2 - au - torch.log1p(torch.exp(-2 * au)))


def _check_state(y, bounds, seed, row0, actions, log_probs, squash, what, rows=None):
    """y: the greedy kernel's bf16 logits over the interleaved head (μ in even, ℓ in odd columns) of global rows row0,
    row0 + 1, ..., all finite; only the rows where `rows` (a bool [M]) is set are held to the bars, when it is given.

    With lc = clamp(ℓ) (exact in fp32), σ64 = exp(lc), z64 = ndtri(u) in fp64:
      u (the kernel's, before tanh) is within tol_u = 2^-19·σ64·(1 + |z64|) + 2^-23·|μ| of u64 = μ + σ64·z64: the bar
      of the Gaussian head (test_gpu_mlp_gaussian.py), which derives it from normcdfinvf's 2^-20·(1 + |z|), expf's 2 ulp
      and the two roundings of the action.
      Squashed: tanh is 1-Lipschitz with slope sech²; over [u64 - tol_u, u64 + tol_u] the slope is at most
      sech²(max(|u64| - tol_u, 0)), and tanhf adds CUDA's documented 2 ulp (<= 2^-22·|tanh|, plus the smallest normal
      near 0).
    Log-probability: ref64 = -Σ_j (0.5·z64² + lc + [squash]·c64(u64)) - d·0.5·log 2π.  The unsquashed terms carry the
      Gaussian head's 2^-20·(1 + |z64|)² each.  c(u) = 2·(log 2 - |u| - log1p(e^-2|u|)) has slope at most 2 in u, so
      the kernel's u costs 2·tol_u per term; its fp32 evaluation (a subtraction, expf and log1pf of 1-2 ulp, the sum
      and the doubling) adds at most 2^-21·(|u| + 1).  The per-thread sums, the quad's two shuffles and the constant
      add at most (2d + 8)·2^-23 of the running magnitudes, bounded by Σ_j |term_j| + d.  The 2·tol_u term is looser
      than (2d + 8)·2^-22·(1 + Σ|term|) where σ is large: it is the action's own error carried through c."""
    M, d2 = y.shape
    d = d2 // 2
    assert actions.dtype == torch.float32 and actions.shape == (M, d), what
    assert log_probs.dtype == torch.float32 and log_probs.shape == (M,), what
    yd = y.double()
    assert bool(torch.isfinite(yd).all()), what
    mu, lc = yd[:, 0::2], yd[:, 1::2].clamp(*bounds)
    s64 = lc.exp()
    z64 = _z64(seed, row0, M, d)
    u64 = mu + s64 * z64
    tol_u = 2.0 ** -19 * s64 * (1 + z64.abs()) + 2.0 ** -23 * mu.abs()
    a = actions.double()
    if squash:
        t64 = torch.tanh(u64)
        slope = 1 / torch.cosh((u64.abs() - tol_u).clamp(min=0)) ** 2
        tol = tol_u * slope + 2.0 ** -22 * t64.abs() + 2.0 ** -126
        err = (a - t64).abs()
        assert bool((a.abs() <= 1).all()), what
    else:
        tol, err = tol_u, (a - u64).abs()
    if rows is not None:
        err, tol = err[rows], tol[rows]
    assert bool((err <= tol).all()), (what, float((err / tol).max()), (err > tol).nonzero()[:4].tolist())
    t = 0.5 * z64 * z64 + lc
    tol_t = 2.0 ** -20 * (1 + z64.abs()) ** 2
    if squash:
        c = _c64(u64)
        t = t + c
        tol_t = tol_t + 2 * tol_u + 2.0 ** -21 * (u64.abs() + 1)
    ref = -t.sum(-1) - d * HALF_LOG_2PI
    tol_lp = tol_t.sum(-1) + (2 * d + 8) * 2.0 ** -23 * (t.abs().sum(-1) + d)
    err_lp = (log_probs.double() - ref).abs()
    if rows is not None:
        err_lp, tol_lp = err_lp[rows], tol_lp[rows]
    assert bool((err_lp <= tol_lp).all()), (what, float((err_lp / tol_lp).max()))
    return u64, tol_u


# ---- 1. a constant log-std ties to the Gaussian head -------------------------------------------------------------------
@pytest.mark.parametrize("valued", [False, True], ids=["policy", "value"])
@pytest.mark.parametrize("bias", [True, False], ids=["biased", "bias_free"])
@pytest.mark.parametrize("d_out", [1, 2, 6, 17, 32, 63, 64, 100, 127, 128])
def test_constant_log_std_ties_to_the_gaussian_head(K, d_out, bias, valued):
    """w_ls = 0 and b_ls = c inside the bounds: the unsquashed actions equal ktb_mlp_bf16_policy_gaussian's with
    log_std = c.float() bit for bit (bias-free: ℓ = 0 and log_std = 0), values equal the _gaussian_value entry's bit
    for bit, and the log-probabilities agree within the reassociation of the same fp32 terms: each sum of d terms
    rounds at most (d + 2)·2^-24 of Σ|t_j| + d·0.92, and a term may round once more (2^-23·|t_j|) where the compiler
    fuses differently, so |Δ| <= (2d + 8)·2^-23·(Σ|t_j| + d)."""
    if valued and d_out == 128:
        pytest.skip("a value head allows 127 actions")
    M, seed = SHIPPED_CHUNK + 1005, 2**33 + 5 * d_out
    w, b, (w_ls, b_ls), value = actor(4000 + d_out, d_out, bias)
    w_ls = torch.zeros_like(w_ls)
    obs = randn((M, 256), 4010 + d_out)
    log_std = b_ls.float() if bias else torch.zeros(d_out, device="cuda")
    kw = dict(value=value) if valued else {}
    got = state(obs, w, b, (w_ls, b_ls), seed, **kw)
    want = mlp.mlp_forward(obs, *w, biases=b, output="gaussian", log_std=log_std, seed=seed, **kw)
    same([got[0]], [want[0]], (d_out, "actions"))
    if valued:
        same([got[2]], [want[2]], (d_out, "values"))
    z64 = _z64(seed, 0, M, d_out)
    t = 0.5 * z64 * z64 + log_std.double()
    tol = (2 * d_out + 8) * 2.0 ** -23 * (t.abs().sum(-1) + d_out)
    err = (got[1].double() - want[1].double()).abs()
    assert bool((err <= tol).all()), (d_out, float((err / tol).max()))


# ---- 2. μ and ℓ tie to the greedy head's logits, and 3. squashed against unsquashed -----------------------------------
@pytest.mark.parametrize("d_out", [1, 6, 17, 64, 127, 128])
@pytest.mark.parametrize("chunk", [256, SHIPPED_CHUNK])
def test_bars_against_the_greedy_logits_of_the_interleaved_head(K, d_out, chunk):
    """17 901 rows, a seed past 2^32, ℓ spread across both bounds (some rows clamped at -3 and at 1): both the
    unsquashed and the squashed call meet their fp64 bars against columns 2j (μ) and 2j + 1 (ℓ) of
    ktb_mlp_bf16_policy's logits over the interleaved head.  In the same call pair, the unsquashed action is the
    squashed one's u bit for bit: tanh64(u) is within tanhf's 2 ulp of the squashed action, and the squashed
    log-probability equals the unsquashed one minus Σ_j c64(u_j) within c's fp32 evaluation and the two sums."""
    M, seed, bounds = SHIPPED_CHUNK + 1005, 2**33 + 11 * d_out, (-3.0, 1.0)
    w, b, ls, _ = actor(4100 + d_out, d_out, ls_scale=0.5, ls_bias=(-4.0, 2.0))
    obs = randn((M, 256), 4110 + d_out)
    w3s, b3s = interleaved(w, b, ls)
    with tuning(chunk):
        y = mlp.mlp_forward(obs, w[0], w[1], w3s, biases=(b[0], b[1], b3s))
        a0, lp0 = state(obs, w, b, ls, seed, log_std_bounds=bounds)
        a1, lp1 = state(obs, w, b, ls, seed, log_std_bounds=bounds, squash=True)
    lc = y.double()[:, 1::2]
    assert bool((lc < bounds[0]).any()) and bool((lc > bounds[1]).any()) or d_out < 6, "both bounds clamp"
    _check_state(y, bounds, seed, 0, a0, lp0, False, f"d_out={d_out} chunk={chunk}")
    _check_state(y, bounds, seed, 0, a1, lp1, True, f"d_out={d_out} chunk={chunk} squash")
    u = a0.double()
    t64 = torch.tanh(u)
    assert bool(((a1.double() - t64).abs() <= 2.0 ** -22 * t64.abs() + 2.0 ** -126).all())
    c = _c64(u)
    z64 = _z64(seed, 0, M, d_out)
    t = 0.5 * z64 * z64 + lc.clamp(*bounds)
    tol = (2.0 ** -21 * (u.abs() + 1)).sum(-1) + 2 * (2 * d_out + 8) * 2.0 ** -23 * ((t.abs() + c.abs()).sum(-1) + d_out)
    err = (lp1.double() - (lp0.double() - c.sum(-1))).abs()
    assert bool((err <= tol).all()), (d_out, float((err / tol).max()))


# ---- 4. edge cases ------------------------------------------------------------------------------------------------------
def _edge(d_out, b_ls_values, b3_values=None, seed=77, M=1000):
    """A head with w_ls = 0 and b_ls = b_ls_values (so ℓ is b_ls in every row), and b3 = b3_values when given."""
    w, b, ls, _ = actor(4200, d_out)
    w_ls = torch.zeros_like(ls[0])
    b_ls = torch.tensor(b_ls_values, device="cuda").bfloat16()
    if b3_values is not None:
        w = (w[0], w[1], torch.zeros_like(w[2]))
        b = (b[0], b[1], torch.tensor(b3_values, device="cuda").bfloat16())
    return randn((M, 256), 4201), w, b, (w_ls, b_ls)


@pytest.mark.parametrize("bounds", [(-1.0, 0.5), (0.25, 0.25), (-math.inf, math.inf), (-20.0, math.inf)],
                         ids=["inside", "lo_eq_hi", "infinite", "upper_infinite"])
def test_clamping_matches_the_gaussian_head_with_the_clamped_log_std(K, bounds):
    """ℓ below, above and at each bound: the unsquashed actions equal the Gaussian head's with log_std =
    clamp(ℓ, lo, hi) bit for bit, and the log-probabilities agree within the reassociation bar."""
    vals = [-3.0, -1.0, -0.5, 0.25, 0.5, 1.5, -0.0, 3.0]
    obs, w, b, ls = _edge(len(vals), vals)
    got = state(obs, w, b, ls, 5, log_std_bounds=bounds)
    log_std = ls[1].float().clamp(*bounds)
    want = mlp.mlp_forward(obs, *w, biases=b, output="gaussian", log_std=log_std.contiguous(), seed=5)
    same([got[0]], [want[0]], bounds)
    assert bool(((got[1] - want[1]).abs() <= 1e-4 * (1 + want[1].abs())).all()), bounds


def test_a_nan_log_std_gives_a_nan_column_and_log_probability(K):
    vals = [0.0, float("nan"), -1.0]
    obs, w, b, ls = _edge(3, vals)
    for squash in (False, True):
        a, lp = state(obs, w, b, ls, 9, squash=squash)
        assert bool(a[:, 1].isnan().all()) and bool(lp.isnan().all()), squash
        assert bool(torch.isfinite(a[:, [0, 2]]).all()), squash


def test_large_u_gives_exactly_one_with_a_finite_log_probability(K):
    """μ = ±100 and ±30 (|u| > 21): tanh rounds to exactly ±1.0 in fp32, and the log-probability stays finite (c(u) is taken from
    u, about -2|u| + 2·log 2 each)."""
    obs, w, b, ls = _edge(4, [0.0, -1.0, 0.0, 0.5], [100.0, -100.0, 30.0, -30.0])
    a, lp = state(obs, w, b, ls, 3, squash=True)
    assert torch.equal(a.sign(), torch.tensor([1.0, -1.0, 1.0, -1.0], device="cuda").expand_as(a))
    assert bool((a.abs() == 1.0).all()) and bool(torch.isfinite(lp).all())
    u, lp0 = state(obs, w, b, ls, 3)
    assert bool(((lp.double() - (lp0.double() - _c64(u.double()).sum(-1))).abs() <= 1e-3 * lp.double().abs()).all())


def test_infinite_u_through_an_infinite_upper_bound_follows_the_header(K):
    """ℓ = 100 with log_std_max = +inf: expf overflows, u = ±inf.  Squashed: actions ±1.0 and log_probs = +inf
    (c(±inf) = -inf).  Unsquashed: actions ±inf and a finite log-probability (lc = 100 is finite).  With
    log_std_max = +inf and ℓ = +inf itself (b_ls = inf): unsquashed log_probs = -inf, squashed NaN (-inf + inf)."""
    obs, w, b, ls = _edge(2, [100.0, 0.0])
    a, lp = state(obs, w, b, ls, 4, log_std_bounds=(-20.0, math.inf), squash=True)
    assert bool((a[:, 0].abs() == 1.0).all()) and bool((lp == math.inf).all())
    a, lp = state(obs, w, b, ls, 4, log_std_bounds=(-20.0, math.inf))
    assert bool(a[:, 0].isinf().all()) and bool(torch.isfinite(lp).all())
    obs, w, b, ls = _edge(2, [math.inf, 0.0])
    a, lp = state(obs, w, b, ls, 4, log_std_bounds=(-20.0, math.inf))
    assert bool(a[:, 0].isinf().all()) and bool((lp == -math.inf).all())
    a, lp = state(obs, w, b, ls, 4, log_std_bounds=(-20.0, math.inf), squash=True)
    assert bool((a[:, 0].abs() == 1.0).all()) and bool(lp.isnan().all())


# ---- 5. the distribution ------------------------------------------------------------------------------------------------
def test_actions_follow_the_tanh_normal_of_their_row(K):
    """2^20 copies of one observation: each action column's empirical CDF against the tanh-Normal CDF
    P(a <= x) = Φ((atanh x - μ) / σ) of that row's fp64 (μ, σ) from the greedy logits passes a KS test at p > 1e-4."""
    from scipy.special import ndtr
    from scipy.stats import kstest

    d_out, M, seed = 4, 1 << 20, 20261017
    w, b, ls, _ = actor(4300, d_out, ls_scale=0.3, ls_bias=(-1.0, 0.3))
    w = (w[0], w[1], w[2] * 0.1)
    obs = randn((1, 256), 4301).expand(M, 256).contiguous()
    a, _ = state(obs, w, b, ls, seed, squash=True)
    w3s, b3s = interleaved(w, b, ls)
    y = mlp.mlp_forward(obs[:1], w[0], w[1], w3s, biases=(b[0], b[1], b3s)).double().cpu()[0]
    for j in range(d_out):
        mu, sigma = float(y[2 * j]), math.exp(float(y[2 * j + 1].clamp(-20.0, 2.0)))
        x = a[:, j].double().cpu().numpy()
        p = kstest(x, lambda v: ndtr((torch.atanh(torch.from_numpy(v).clamp(-1, 1)).numpy() - mu) / sigma)).pvalue
        assert p > 1e-4, (j, mu, sigma, p)


# ---- 6. forms, chunkings and row splits ------------------------------------------------------------------------------------
@pytest.mark.parametrize("squash", [False, True], ids=["u", "tanh"])
@pytest.mark.parametrize("valued", [False, True], ids=["policy", "value"])
@pytest.mark.parametrize("d_out", [1, 7, 32, 33, 64, 127])
def test_every_form_gives_the_same_bits(K, d_out, valued, squash):
    """The plain form at the shipped and 256-row chunks, the staged form (pull kernel and copy engine), row splits with
    row_offset, mlp_scatter_gather on ranks [0, 0, 0] and the pushed form on ranks [0, 0, 0]: the same bits."""
    M, seed = 3 * 1408, 2**34 + 3 * d_out
    w, b, ls, value = actor(4400 + d_out, d_out, ls_scale=0.3)
    obs = randn((M, 256), 4410 + d_out)
    kw = dict(squash=squash, **(dict(value=value) if valued else {}))
    got = state(obs, w, b, ls, seed, **kw)
    assert len(got) == (3 if valued else 2)
    for chunk in (256, SHIPPED_CHUNK):
        for ce in (None, 0, 1):
            with tuning(chunk, ce):
                same(state(obs, w, b, ls, seed, staged=ce is not None, **kw), got, (chunk, ce))
    for split in (1, 1000, 2 * 1408 + 5):
        lo = state(obs[:split], w, b, ls, seed, **kw)
        hi = state(obs[split:], w, b, ls, seed, row_offset=split, **kw)
        same([torch.cat([p, q]) for p, q in zip(lo, hi)], got, ("split", split))
    views = mlp.mlp_scatter_gather(obs, *w, devices=[0, 0, 0], biases=b, output="gaussian", log_std=ls, seed=seed,
                                   **kw)
    torch.cuda.synchronize()
    same([torch.cat([v[k] for v in views]) for k in range(len(got))], got, "scatter_gather")
    w3s, b3s = interleaved(w, b, ls, value if valued else None)
    bounds = [K.shard_bounds(M, 3, r) for r in range(3)]
    actions = torch.full((M, d_out), -1.0, device="cuda")
    log_probs, values = (torch.full((M,), -1.0, device="cuda") for _ in range(2))
    mlp._mlp_scatter_gather_pushed(obs, [0, 0, 0], bounds, {0: (w[0], w[1], w3s, b[0], b[1], b3s)}, "gaussian", None,
                                   actions, log_probs, seed, {0: ls}, None, values if valued else None, None,
                                   (-20.0, 2.0, int(squash)))
    torch.cuda.synchronize()
    same((actions, log_probs, values)[:len(got)], got, "pushed")


def rig_weights(w, b, ls, value=None):
    """(w, b) for the rig's named arguments: the head replaced by views of the first d_out rows of the interleaved
    head, so the rig passes the action width d_out and the interleaved head's address."""
    w3s, b3s = interleaved(w, b, ls, value)
    d_out = w[2].shape[0]
    return (w[0], w[1], w3s[:d_out]), (b[0], b[1], None if b3s is None else b3s[:d_out])


@pytest.mark.parametrize("head", [STATE, STATE_VALUE], ids=["policy", "value"])
@pytest.mark.parametrize("form,M,chunk,d_out", [
    ("plain", 1000, SHIPPED_CHUNK, 7), ("plain", 1000, 256, 18), ("plain", 1000, 256, 127),
    ("staged", 1408, 256, 63), ("staged", 1408, 256, 64), ("pushed", 3 * 1408, 256, 7), ("pushed", 3 * 1408, 256, 32),
])
def test_writes_stay_inside_the_outputs(K, head, form, M, chunk, d_out):
    """Every output, the scratch and the stage between guard bands (the fp32 actions [M, d_out] as scalars, one at a
    4-byte offset); the results equal mlp_forward's bit for bit."""
    seed = 6
    valued = head is STATE_VALUE
    w, b, ls, value = actor(4500 + d_out, d_out, ls_scale=0.3)
    obs = randn((M, 256), 4501)
    want = state(obs, w, b, ls, seed, squash=True, **(dict(value=value) if valued else {}))
    rw, rb = rig_weights(w, b, ls, value if valued else None)
    bufs = run_guarded(form, head._replace(args=lambda a: head.args(dict(a, squash=1))), K, chunk, obs, rw, rb, seed,
                       offsets={"actions": 4})
    for name, buf in bufs.items():
        buf.check(f"{form} M={M} chunk={chunk} d_out={d_out}: {name}")
    for name, h in zip(("actions", "log_probs", "values"), want):
        assert torch.equal(bufs[name].view(torch.int32).view(h.shape), bits(h)), (form, name)


# ---- status codes ----------------------------------------------------------------------------------------------------------
_VALUES = {}


def _values():
    if "v" not in _VALUES:
        _VALUES["v"] = torch.zeros(4096, device="cuda")
    return _VALUES["v"].data_ptr()


NAN = float("nan")
STATUS_CASES = {
    "d_out_129": (plain, dict(d_out=129), L.ERR_UNSUPPORTED, None),
    "value_d_out_128": (plain, dict(d_out=128), L.ERR_UNSUPPORTED, "value"),
    "value_d_out_127_runs_its_other_checks": (plain, dict(d_out=127, values=0), L.ERR_ARG, "value"),
    "nan_low": (plain, dict(lo=NAN), L.ERR_ARG, None),
    "nan_high": (plain, dict(hi=NAN), L.ERR_ARG, None),
    "low_above_high": (plain, dict(lo=1.0, hi=0.5), L.ERR_ARG, None),
    "null_actions": (plain, dict(actions=0), L.ERR_ARG, None),
    "null_log_probs": (plain, dict(log_probs=0), L.ERR_ARG, None),
    "actions_2_bytes_in": (plain, dict(actions_off=2), L.ERR_ARG, None),
    "staged_nan_low": (plain, dict(lo=NAN, stage=0), L.ERR_ARG, None),
    "inherited_d_out_first": (plain, dict(d_out=257, lo=NAN), L.ERR_UNSUPPORTED, None),
    "width_before_bounds": (plain, dict(d_out=129, lo=NAN), L.ERR_UNSUPPORTED, None),
    "inherited_d_in": (plain, dict(d_in=100), L.ERR_ARG, None),
    "pushed_d_out_129": (pushed, dict(d_out=129), L.ERR_UNSUPPORTED, None),
    "pushed_nan_high": (pushed, dict(hi=NAN), L.ERR_ARG, None),
    "pushed_low_above_high": (pushed, dict(lo=0.0, hi=-1.0), L.ERR_ARG, None),
    "pushed_inherited_seq": (pushed, dict(seq=0, lo=NAN), L.ERR_ARG, None),
    "pushed_inherited_stride": (pushed, dict(stride=(1 << 20) + 8), L.ERR_ARG, None),
}


@pytest.mark.parametrize("valued", [False, True], ids=["policy", "value"])
@pytest.mark.parametrize("name", list(STATUS_CASES))
def test_bad_arguments_get_the_documented_status(K, name, valued):
    form, overrides, status, only = STATUS_CASES[name]
    if only == "value" and not valued:
        pytest.skip("a case of the value entries")
    o = dict(overrides)
    if valued:
        o.setdefault("values", _values())
    expect_status(form(STATE_VALUE if valued else STATE, **o), status)


@pytest.mark.parametrize("valued", [False, True], ids=["policy", "value"])
def test_empty_pushed_shard_runs_its_checks_and_acks(K, valued):
    """An empty shard (M = 0) with null outputs publishes ack[rank] = seq in the root's control block (its bounds are
    not read); with a bad inherited argument it returns that entry's status."""
    head = STATE_VALUE if valued else STATE
    ctrl_root = torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda")
    L.call(*pushed(head, M=0, actions=0, log_probs=0, values=0, ctrl_root=ctrl_root.data_ptr(), seq=3, rank=2,
                   lo=NAN))
    torch.cuda.synchronize()
    assert int(ctrl_root[512 + 8 * 2:512 + 8 * 3].view(torch.int64)) == 3
    expect_status(pushed(head, M=0, actions=0, log_probs=0, values=0, seq=0), L.ERR_ARG)


# ---- Python checks and in-place updates ------------------------------------------------------------------------------------
def test_python_checks_name_the_output_in_mlp_forward_and_scatter_gather(K):
    (w1, w2, w3), b = config(4600, 18)
    obs = randn((256, 256), 4601)
    w_ls, b_ls = randn((18, 1024), 4602), randn((18,), 4603)
    bad = [
        (dict(log_std=(w_ls, b_ls), output="sample"), 'log_std is not an argument of output="sample"'),
        (dict(log_std=(w_ls,)), "tensor or"),
        (dict(log_std=(w_ls, None)), "b_ls is given exactly when b3 is"),
        (dict(log_std=(w_ls[:17], b_ls)), "shape"),
        (dict(log_std=(w_ls.float(), b_ls)), "bfloat16"),
        (dict(log_std=(w_ls.cpu(), b_ls)), "CUDA"),
        (dict(log_std=(w_ls, b_ls.cpu())), "b_ls must be"),
        (dict(log_std=(w_ls, b_ls), log_std_bounds=(NAN, 1.0)), "NaN"),
        (dict(log_std=(w_ls, b_ls), log_std_bounds=(1.0, 0.0)), "low <= high"),
        (dict(log_std=(w_ls, b_ls), log_std_bounds=(1.0,)), "two numbers"),
        (dict(log_std=(w_ls, b_ls), squash="yes"), "True or False"),
        (dict(log_std=torch.zeros(18, device="cuda"), squash=True), "state-dependent"),
        (dict(log_std=torch.zeros(18, device="cuda"), log_std_bounds=(-1, 1)), "state-dependent"),
    ]
    for kw, reason in bad:
        kw = dict(dict(output="gaussian", seed=1), **kw)
        with pytest.raises(ValueError, match=reason):
            mlp.mlp_forward(obs, w1, w2, w3, biases=b, **kw)
        with pytest.raises(ValueError, match=reason):
            mlp.mlp_scatter_gather(obs, w1, w2, w3, devices=[0], biases=b, **kw)
    (w1, w2, w3), b = config(4610, 129)
    for fn, extra in ((mlp.mlp_forward, {}), (mlp.mlp_scatter_gather, dict(devices=[0]))):
        with pytest.raises(ValueError, match="d_out=129"):
            fn(obs, w1, w2, w3, biases=b, output="gaussian", seed=1,
               log_std=(randn((129, 1024), 1), randn((129,), 2)), **extra)


def test_in_place_weight_updates_reach_the_next_call(K):
    """After w_ls.add_(...), then b_ls, w3 and wv: the next call equals a fresh call's (fresh tensors, so a new head),
    and the head cache keeps one entry for the head."""
    d_out, M, seed = 18, 2048, 31
    w, b, ls, value = actor(4700, d_out, ls_scale=0.3)
    w, b, ls, value = list(w), list(b), list(ls), list(value)
    obs = randn((M, 256), 4701)
    kw = dict(squash=True, value=value)
    state(obs, w, b, ls, seed, **kw)
    entries = len(mlp._stacked_heads)
    for t in (ls[0], ls[1], w[2], value[0]):
        t.add_(0.125)
        got = state(obs, w, b, ls, seed, **kw)
        fresh = state(obs, [t.clone() for t in w], [t.clone() for t in b], [t.clone() for t in ls], seed,
                      squash=True, value=[t.clone() for t in value])
        same(got, fresh, "update")
        assert len(mlp._stacked_heads) <= entries + 1
    assert len(mlp._stacked_heads) <= entries + 1


# ---- 7. the public API ------------------------------------------------------------------------------------------------------
def _public_case(golden, valued):
    obs = torch.randn(1000, 256, generator=torch.Generator().manual_seed(1000)).bfloat16()
    d_out = 6
    p = policy_weights(golden, d_out)
    g = torch.Generator().manual_seed(78)
    ls = ((torch.randn(d_out, 1024, generator=g) * 0.01).bfloat16(), torch.linspace(-1.0, 0.0, d_out).bfloat16())
    value = ((torch.randn(1, 1024, generator=g) * 0.02).bfloat16(), (torch.randn(1, generator=g) * 0.1).bfloat16())
    seed = 2**35 + 29
    if valued:
        body, extra, tail = cases.mlp_policy_gaussian_state_squashed_value, dict(value=("wv", "bv")), value
    else:
        body, extra, tail = cases.mlp_policy_gaussian_state_squashed, {}, ()
    policy = mapped_copy(body, "mlp", bias=True, output="gaussian", seed="seed", log_std=("w_ls", "b_ls"),
                         log_std_bounds=(-20.0, 2.0), squash=True, **extra)
    return obs, p, ls, tail, seed, body, policy


def _mine(obs, p, ls, tail, seed):
    pc = [t.cuda() for t in p]
    kw = dict(value=tuple(t.cuda() for t in tail)) if tail else {}
    return mlp.mlp_forward(obs.cuda(), pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]), output="gaussian",
                           log_std=tuple(t.cuda() for t in ls), seed=seed, squash=True, **kw)


def _against_body(K, obs, p, ls, seed, got, want, n):
    """Each rank's outputs against the oracle's run of the body: values within rtol 2^-7, atol 1e-2 everywhere; where
    the body's bf16 μ and ℓ equal the kernel's (elsewhere they differ by a bf16 rounding of the logits, which the other
    tests tie down), actions within rtol 2^-7, atol 1e-2, and, in rows where all of them are equal, the kernel's and the
    body's actions and log-probabilities each within _check_state's bar of the same fp64 reference.  At least 90 % of
    the (μ, ℓ) pairs must agree."""
    from policy_value_cases import _trunk

    pc = [t.cuda() for t in p]
    w3s, b3s = mlp._stacked_head(pc[4], pc[5], None, None, *(t.cuda() for t in ls))
    agree, total = 0, 0
    for r, (g, h) in enumerate(zip(got, want)):
        lo, hi = K.shard_bounds(obs.shape[0], n, r)
        g, h = [t.cuda() for t in g], [t.cuda() for t in h]
        if len(g) == 3:
            assert torch.allclose(g[2], h[2], rtol=2.0 ** -7, atol=1e-2), r
        with mock.patch.dict(os.environ, {"RANK": str(r), "WORLD_SIZE": str(n)}):
            hb = _trunk(obs, *p[:4])
        y_body = torch.stack((torch.nn.functional.linear(hb, p[4], p[5]),
                              torch.nn.functional.linear(hb, ls[0], ls[1])), -1).flatten(1).cuda()
        y = mlp.mlp_forward(obs[lo:hi].cuda(), pc[0], pc[2], w3s, biases=(pc[1], pc[3], b3s))
        eq = (y_body == y).view(hi - lo, -1, 2).all(-1)
        agree += int(eq.sum())
        total += eq.numel()
        assert bool(torch.isclose(g[0], h[0], rtol=2.0 ** -7, atol=1e-2)[eq].all()), r
        rows = eq.all(-1)
        for outs, who in ((g, "kernel"), (h, "body")):
            _check_state(y, (-20.0, 2.0), seed, lo, outs[0], outs[1], True, (r, who), rows=rows)
    assert agree >= 0.9 * total, (agree, total)


@pytest.mark.parametrize("valued", [False, True], ids=["policy", "value"])
@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["1_rank", "3_ranks"])
def test_mapped_state_head_through_public_api(K, golden, devices, valued):
    """@kt.mapped("mlp", bias=True, output="gaussian", seed="seed", log_std=("w_ls", "b_ls"), log_std_bounds=(-20, 2),
    squash=True[, value=("wv", "bv")]) on Compute(gpus=1): each rank returns the bits of mlp_forward over its rows,
    and agrees with the oracle's run of the body as _against_body states."""
    obs, p, ls, tail, seed, body, policy = _public_case(golden, valued)
    n = len(devices)
    want = ref_dispatch.spmd_call(body, obs, *p, *ls, *tail, seed, num_proc=n, serialization="pickle")
    mine = _mine(obs, p, ls, tail, seed)
    with deployed(policy, f"t-gstate-{int(valued)}-{n}", devices) as remote:
        got = remote(obs.cuda(), *[t.cuda() for t in p], *[t.cuda() for t in ls], *[t.cuda() for t in tail], seed,
                     serialization="pickle")
        torch.cuda.synchronize()
    assert len(got) == len(want) == n
    for r, g in enumerate(got):
        lo, hi = K.shard_bounds(obs.shape[0], n, r)
        assert isinstance(g, tuple) and len(g) == (3 if valued else 2), r
        same([t.cpu() for t in g], [t[lo:hi].cpu() for t in mine], r)
    _against_body(K, obs, p, ls, seed, got, want, n)


def test_mapped_state_head_on_a_workers_subset(K, golden):
    """Two workers of one rank each on cuda:0; a call with workers=[1] returns rank 1's outputs only, with the bits of
    mlp_forward over its rows."""
    import kubetorch_b200 as kt

    obs, p, ls, tail, seed, body, policy = _public_case(golden, True)
    mine = _mine(obs, p, ls, tail, seed)
    remote = kt.fn(policy, name="t-gstate-workers").to(
        kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute("b200", workers=2, num_proc=1,
                                                                                 devices=[0, 0]))
    try:
        got = remote(obs.cuda(), *[t.cuda() for t in p], *[t.cuda() for t in ls], *[t.cuda() for t in tail], seed,
                     serialization="pickle", workers=[1])
        torch.cuda.synchronize()
    finally:
        remote.teardown()
    lo, hi = K.shard_bounds(obs.shape[0], 2, 1)
    assert len(got) == 1
    same([t.cpu() for t in got[0]], [t[lo:hi].cpu() for t in mine], "workers=[1]")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("transfer", ["pull", "push"])
def test_mapped_state_head_on_two_gpus(K, golden, transfer):
    """Two ranks on two GPUs, staged pull and pushed form (the interleaved head copied to cuda:1), three calls, the
    log-std head updated in place before the last: the bits of one plain call."""
    obs, p, ls, tail, seed, body, policy = _public_case(golden, True)
    with deployed(policy, f"t-gstate-2gpu-{transfer}", [0, 1], transfer=transfer) as remote:
        pc = [t.cuda(0) for t in p]
        lc = [t.cuda(0) for t in ls]
        vc = [t.cuda(0) for t in tail]
        for it in range(3):
            x = torch.randn(2 * 1408, 256, generator=torch.Generator().manual_seed(5 + it)).bfloat16().cuda(0)
            if it == 2:
                lc[0].add_(0.125)
            got = remote(x, *pc, *lc, *vc, seed, serialization="pickle")
            torch.cuda.synchronize(0)
            torch.cuda.synchronize(1)
            want = mlp.mlp_forward(x, pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]), output="gaussian",
                                   log_std=tuple(lc), seed=seed, squash=True, value=tuple(vc))
            same([torch.cat([g[k].cpu() for g in got]) for k in range(3)], [t.cpu() for t in want], it)
