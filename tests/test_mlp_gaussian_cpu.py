"""not-gpu: the Gaussian policy head (@kt.mapped("mlp", output="gaussian")) without a GPU — the Gaussian noise of
kubetorch_b200.sampling against a plain-int restatement, its separation from the Gumbel stream, the semantic definition
on 1, 3 and 4 ranks (sharding is invisible) and its distribution, the decoration options and the Python log_std
checks."""
import math
import random
from unittest import mock

import pytest
import torch

import policy_gaussian_cases
from oracle import ref_dispatch

from kubetorch_b200.sampling import gumbel_uniform, normal_noise, random_words

Z_MAX = 5.29471   # |Φ⁻¹(2^-24)| = 5.2947041, in fp32 too


def _philox_int(c, k):
    """Philox4x32-10 restated on plain Python ints."""
    c, k = list(c), list(k)
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k[0], p1 & 0xFFFFFFFF, (p0 >> 32) ^ c[3] ^ k[1], p0 & 0xFFFFFFFF]
        k = [(k[0] + 0x9E3779B9) & 0xFFFFFFFF, (k[1] + 0xBB67AE85) & 0xFFFFFFFF]
    return c


def _word_int(seed, i, j, word3):
    return _philox_int((i & 0xFFFFFFFF, i >> 32, j >> 1, word3), (seed & 0xFFFFFFFF, seed >> 32))[j & 1]


def _ndtri64(u):
    from scipy.special import ndtri

    return float(ndtri(u))


# ---- the Gaussian noise ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,row0", [(0, 0), (12345, 7), (2**32 + 5, 2**32 - 3), (2**64 - 1, 2**40 + 11),
                                       (0x9E3779B97F4A7C15, 3 * 2**33)])
def test_normal_noise_equals_a_plain_int_restatement(seed, row0):
    """Random words with counter word 3 = 1 exactly, u exactly (strictly inside (0, 1), never 0.5), and z = fp32 of the
    fp64 ndtri of the exact u, bit for bit; never 0 and within ±5.29471.  Rows and seeds past 2^32, odd widths."""
    rows, cols = 9, 7
    words = random_words(seed, row0, rows, cols, word3=1)
    u = gumbel_uniform(seed, row0, rows, cols, word3=1)
    z = normal_noise(seed, row0, rows, cols)
    assert z.shape == (rows, cols) and z.dtype == torch.float32
    for r in range(rows):
        for j in range(cols):
            x = _word_int(seed, row0 + r, j, 1)
            assert int(words[r, j]) == x, (r, j)
            u_exact = (2 * (x >> 9) + 1) * 2.0 ** -24
            assert float(u[r, j]) == u_exact and 0.0 < u_exact < 1.0 and u_exact != 0.5
            want = torch.tensor(_ndtri64(u_exact), dtype=torch.float64).float()
            assert float(z[r, j]) == float(want), (r, j)
            assert float(z[r, j]) != 0.0 and abs(float(z[r, j])) <= Z_MAX


def test_normal_noise_of_random_coordinates():
    """Random (seed, row, col) from the whole range, each drawn alone, against the restatement."""
    rng = random.Random(11)
    for _ in range(200):
        seed, i, j = rng.getrandbits(64), rng.getrandbits(rng.choice((8, 32, 40, 62))), rng.randrange(256)
        x = _word_int(seed, i, j, 1)
        assert int(random_words(seed, i, 1, j + 1, word3=1)[0, j]) == x
        u = (2 * (x >> 9) + 1) * 2.0 ** -24
        assert float(normal_noise(seed, i, 1, j + 1)[0, j]) == float(torch.tensor(_ndtri64(u)).float())


def test_the_extreme_uniforms_give_the_documented_tail():
    """u = 2^-24 and 1 - 2^-24 are the extreme uniforms: |z| there is the truncation point 5.29471 of the contract."""
    lo, hi = _ndtri64(2.0 ** -24), _ndtri64(1 - 2.0 ** -24)
    assert lo == -hi and 5.2947 < hi < Z_MAX
    assert 1.1e-7 < 2 * 0.5 * math.erfc(hi / math.sqrt(2)) < 1.3e-7


def test_gaussian_words_are_not_the_gumbel_words():
    """The same (seed, row, column) draws different words in the two streams, and the Gumbel default is word 3 = 0."""
    for seed, row0 in ((0, 0), (77, 2**33)):
        g = random_words(seed, row0, 64, 18)
        assert torch.equal(g, random_words(seed, row0, 64, 18, word3=0))
        n = random_words(seed, row0, 64, 18, word3=1)
        assert float((g == n).double().mean()) < 0.01


def test_normal_noise_depends_on_the_global_row_only():
    full = normal_noise(99, 0, 50, 18)
    assert torch.equal(normal_noise(99, 17, 20, 18), full[17:37])
    assert torch.equal(normal_noise(99, 0, 50, 5), full[:, :5])
    assert not torch.equal(normal_noise(100, 0, 50, 18), full)
    many = normal_noise(3, 0, 4096, 64)
    assert bool((many != 0).all()) and bool((many.abs() <= Z_MAX).all())


@pytest.mark.parametrize("bad", [-1, 2**64, True, 1.0, "7", None])
def test_normal_noise_rejects_a_bad_seed(bad):
    with pytest.raises(ValueError):
        normal_noise(bad, 0, 2, 2)


@pytest.mark.parametrize("bad", [-1, 2**32, True, 0.0])
def test_random_words_rejects_a_bad_counter_word(bad):
    with pytest.raises(ValueError):
        random_words(1, 0, 2, 2, word3=bad)


# ---- the semantic definition ----------------------------------------------------------------------------------------
def _policy(seed, d_in=64, d_hidden=256, d_out=6):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).bfloat16()   # noqa: E731
    return (r(d_hidden, d_in, scale=0.1), r(d_hidden, scale=0.5), r(d_hidden, d_hidden, scale=0.05),
            r(d_hidden, scale=0.5), r(d_out, d_hidden, scale=0.05), r(d_out, scale=0.5))


@pytest.mark.parametrize("rows", [0, 2, 10, 13, 100])
def test_gaussian_body_is_the_same_on_every_rank_count(rows):
    """1, 3 and 4 ranks (ragged shards, and empty shards past the data) give the same concatenated actions and
    log-probabilities bit for bit: each rank draws the noise of its rows' global indices.  The result is the
    reparameterised draw of the whole batch, and log_probs is Normal(μ, σ).log_prob(actions).sum(-1)."""
    p = _policy(rows + 5)
    obs = torch.randn(rows, 64, generator=torch.Generator().manual_seed(rows)).bfloat16()
    log_std = torch.linspace(-3, 1, 6)
    seed = 2**40 + rows
    runs = {n: ref_dispatch.spmd_call(policy_gaussian_cases.mlp_policy_gaussian, obs, *p, log_std, seed, num_proc=n)
            for n in (1, 3, 4)}
    for n, res in runs.items():
        assert len(res) == n
        for a, lp in res:
            assert a.dtype == lp.dtype == torch.float32 and a.shape == (lp.shape[0], 6)
    want_a = torch.cat([a for a, _ in runs[1]])
    want_lp = torch.cat([lp for _, lp in runs[1]])
    for n in (3, 4):
        assert torch.equal(torch.cat([a for a, _ in runs[n]]), want_a), n
        assert torch.equal(torch.cat([lp for _, lp in runs[n]]), want_lp), n
    import torch.nn.functional as F

    h = torch.relu(F.linear(obs, p[0], p[1]))
    h = torch.relu(F.linear(h, p[2], p[3]))
    mu = F.linear(h, p[4], p[5]).float()
    assert torch.equal(want_a, mu + torch.exp(log_std) * normal_noise(seed, 0, rows, 6))
    if rows:
        ref = torch.distributions.Normal(mu.double(), log_std.double().exp()).log_prob(want_a.double()).sum(-1)
        assert torch.allclose(want_lp.double(), ref, rtol=1e-5, atol=1e-4)


def test_gaussian_draws_follow_their_normal():
    """Many rows of one mean: per-column mean and variance within 5 standard errors of (μ, σ²), and a KS test of the
    standardised draws against N(0, 1) gives p > 1e-4."""
    from scipy.stats import kstest

    n = 1 << 17
    mu = torch.tensor([0.5, -2.0, 0.0, 3.0, 1.0])
    log_std = torch.tensor([0.0, -1.0, 0.5, -3.0, 1.0])
    sigma = log_std.exp()
    a = (mu + sigma * normal_noise(2024, 0, n, 5)).double()
    mean, var = a.mean(0), a.var(0)
    assert bool(((mean - mu.double()).abs() <= 5 * sigma.double() / math.sqrt(n)).all()), mean
    assert bool(((var / sigma.double() ** 2 - 1).abs() <= 5 * math.sqrt(2 / n)).all()), var
    stat = kstest(((a - mu.double()) / sigma.double()).flatten().numpy(), "norm")
    assert stat.pvalue > 1e-4, stat


# ---- decoration -----------------------------------------------------------------------------------------------------
def test_gaussian_options_are_recorded_on_the_spec():
    import kubetorch_b200 as kt
    from kubetorch_b200.mapped import mapped_spec

    assert kt.normal_noise is normal_noise
    fn = kt.mapped("mlp", bias=True, output="gaussian", seed="seed", log_std="log_std")(
        policy_gaussian_cases.mlp_policy_gaussian)
    spec = mapped_spec(fn)
    assert spec.extra["output"] == "gaussian" and spec.extra["seed"] == "seed" and spec.extra["log_std"] == "log_std"
    const = mapped_spec(kt.mapped("mlp", output="gaussian", seed=2**64 - 1, log_std="s")(lambda obs, s: None))
    assert const.extra["seed"] == 2**64 - 1


@pytest.mark.parametrize("kwargs", [
    {"output": "gaussian", "log_std": "log_std"}, {"output": "gaussian", "seed": 1},
    {"output": "gaussian", "seed": "seed", "log_std": None}, {"output": "gaussian", "seed": "seed", "log_std": 0.5},
    {"output": "gaussian", "seed": 1, "log_std": torch.zeros(3)}, {"output": "sample", "seed": 1, "log_std": "s"},
    {"output": "logits", "log_std": "s"}, {"log_std": "s"}, {"output": "gaussian", "seed": -1, "log_std": "s"},
    {"output": "gaussian", "seed": 2**64, "log_std": "s"}, {"output": "gaussian", "seed": True, "log_std": "s"},
    {"output": "gaussian", "seed": 1.5, "log_std": "s"},
])
def test_bad_gaussian_options_raise_at_decoration(kwargs):
    """output="gaussian" needs seed= and log_std=; log_std= belongs to output="gaussian" only and names a call
    argument; a constant seed is an int in [0, 2**64)."""
    import kubetorch_b200 as kt

    with pytest.raises(ValueError):
        kt.mapped("mlp", **kwargs)


def test_log_std_must_name_an_argument_of_the_callable():
    import kubetorch_b200 as kt

    deco = kt.mapped("mlp", bias=True, output="gaussian", seed="seed", log_std="sigma")
    with pytest.raises(ValueError):
        deco(policy_gaussian_cases.mlp_policy_gaussian)


@pytest.mark.parametrize("op", ["identity", "scale", "affine"])
def test_log_std_belongs_to_the_mlp_op(op):
    import kubetorch_b200 as kt

    with pytest.raises(ValueError):
        kt.mapped(op, log_std="log_std")


# ---- Python argument checks -----------------------------------------------------------------------------------------
def _w(d_in=256, d_hidden=1024, d_out=18):
    return (torch.zeros(d_hidden, d_in, dtype=torch.bfloat16), torch.zeros(d_out, d_hidden, dtype=torch.bfloat16))


def _as_cuda():
    """Make CPU tensors report is_cuda, so that the checks' acceptance can be tested without a GPU."""
    return mock.patch.object(torch.Tensor, "is_cuda", property(lambda self: True))


def test_python_checks_accept_gaussian_with_a_seed_and_log_std():
    from kubetorch_b200.device import mlp

    assert "gaussian" in mlp.OUTPUTS
    with _as_cuda():
        for d_out in (1, 6, 18, 64, 256):
            w1, w3 = _w(d_out=d_out)
            for seed in (0, 2**32, 2**64 - 1):
                assert mlp._check_policy(w1, w3, (None, None, None), "gaussian", seed, torch.zeros(d_out)) is None


@pytest.mark.parametrize("case", ["missing", "cpu", "float64", "bfloat16", "short", "long", "2d", "strided", "list"])
def test_python_checks_reject_a_bad_log_std(case):
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    log_std = {"missing": None, "cpu": torch.zeros(18), "float64": torch.zeros(18, dtype=torch.float64),
               "bfloat16": torch.zeros(18, dtype=torch.bfloat16), "short": torch.zeros(17), "long": torch.zeros(19),
               "2d": torch.zeros(1, 18), "strided": torch.zeros(36)[::2], "list": [0.0] * 18}[case]
    with _as_cuda() if case != "cpu" else mock.patch.dict({}):
        with pytest.raises(ValueError):
            mlp._check_policy(w1, w3, (None, None, None), "gaussian", 1, log_std)


@pytest.mark.parametrize("output", ["logits", "actions", "both", "sample"])
def test_python_checks_refuse_log_std_with_another_output(output):
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    with _as_cuda():
        with pytest.raises(ValueError):
            mlp._check_policy(w1, w3, (None, None, None), output, 1, torch.zeros(18))


@pytest.mark.parametrize("seed", [None, -1, 2**64, True, 1.0, "1"])
def test_python_checks_reject_a_bad_gaussian_seed(seed):
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    with _as_cuda():
        with pytest.raises(ValueError):
            mlp._check_policy(w1, w3, (None, None, None), "gaussian", seed, torch.zeros(18))
