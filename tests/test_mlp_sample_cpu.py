"""not-gpu: the sampled policy (@kt.mapped("mlp", output="sample")) without a GPU — the Philox generator and Gumbel
noise of kubetorch_b200.sampling against the Random123 known answers and a plain-int restatement, the semantic
definition on 1, 3 and 4 ranks (sharding is invisible), the decoration options and the Python seed checks."""
import math
import random

import pytest
import torch

import policy_sample_cases
from oracle import ref_dispatch

from kubetorch_b200.sampling import gumbel_noise, gumbel_uniform, philox4x32_10, random_words


# ---- Philox4x32-10 ----------------------------------------------------------------------------------------------------
KNOWN_ANSWERS = [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


def test_philox_reproduces_the_known_answers():
    for counter, key, want in KNOWN_ANSWERS:
        got = philox4x32_10(torch.tensor(counter, dtype=torch.int64), torch.tensor(key, dtype=torch.int64))
        assert got.tolist() == list(want), [f"{v:08x}" for v in got.tolist()]
    # batched: every vector in one call
    c = torch.tensor([k[0] for k in KNOWN_ANSWERS], dtype=torch.int64)
    k = torch.tensor([k[1] for k in KNOWN_ANSWERS], dtype=torch.int64)
    assert philox4x32_10(c, k).tolist() == [list(k[2]) for k in KNOWN_ANSWERS]


def _philox_int(c, k):
    """Philox4x32-10 restated on plain Python ints."""
    c, k = list(c), list(k)
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k[0], p1 & 0xFFFFFFFF, (p0 >> 32) ^ c[3] ^ k[1], p0 & 0xFFFFFFFF]
        k = [(k[0] + 0x9E3779B9) & 0xFFFFFFFF, (k[1] + 0xBB67AE85) & 0xFFFFFFFF]
    return c


def _word_int(seed, i, j):
    return _philox_int((i & 0xFFFFFFFF, i >> 32, j >> 1, 0), (seed & 0xFFFFFFFF, seed >> 32))[j & 1]


@pytest.mark.parametrize("seed,row0", [(0, 0), (12345, 7), (2**32 + 5, 2**32 - 3), (2**64 - 1, 2**40 + 11),
                                       (0x9E3779B97F4A7C15, 3 * 2**33)])
def test_gumbel_noise_equals_a_plain_int_restatement(seed, row0):
    """Random words exactly, u exactly (and strictly inside (0, 1)), and g = -log(-log u) within the error of two fp32
    logs of the exact u (finite, inside about [-2.81, 16.6]); rows and seeds past 2^32 included, odd widths too."""
    rows, cols = 9, 7
    words = random_words(seed, row0, rows, cols)
    u = gumbel_uniform(seed, row0, rows, cols)
    g = gumbel_noise(seed, row0, rows, cols)
    assert words.shape == u.shape == g.shape == (rows, cols) and u.dtype == g.dtype == torch.float32
    for r in range(rows):
        for j in range(cols):
            x = _word_int(seed, row0 + r, j)
            assert int(words[r, j]) == x, (r, j)
            u_exact = (2 * (x >> 9) + 1) * 2.0 ** -24
            assert float(u[r, j]) == u_exact and 0.0 < u_exact < 1.0
            g_exact = -math.log(-math.log(u_exact))
            assert math.isfinite(float(g[r, j])) and -2.82 < float(g[r, j]) < 16.7
            assert abs(float(g[r, j]) - g_exact) <= 2.0 ** -20 * (1.0 + abs(g_exact)), (r, j, float(g[r, j]), g_exact)


def test_gumbel_noise_of_random_coordinates():
    """Random (seed, row, col) from the whole range, each drawn alone, against the restatement."""
    rng = random.Random(7)
    for _ in range(200):
        seed, i, j = rng.getrandbits(64), rng.getrandbits(rng.choice((8, 32, 40, 62))), rng.randrange(256)
        x = _word_int(seed, i, j)
        assert int(random_words(seed, i, 1, j + 1)[0, j]) == x
        assert float(gumbel_uniform(seed, i, 1, j + 1)[0, j]) == (2 * (x >> 9) + 1) * 2.0 ** -24


def test_gumbel_noise_depends_on_the_global_row_only():
    """Rows [a, b) drawn alone equal rows a.. of a longer draw: the noise of a row does not depend on its shard."""
    full = gumbel_noise(99, 0, 50, 18)
    assert torch.equal(gumbel_noise(99, 17, 20, 18), full[17:37])
    assert torch.equal(gumbel_noise(99, 0, 50, 5), full[:, :5])
    assert not torch.equal(gumbel_noise(100, 0, 50, 18), full)
    extremes = gumbel_uniform(3, 0, 4096, 64)
    assert bool((extremes > 0).all()) and bool((extremes < 1).all())
    assert bool(torch.isfinite(gumbel_noise(3, 0, 4096, 64)).all())


@pytest.mark.parametrize("bad", [-1, 2**64, True, 1.0, "7", None])
def test_gumbel_noise_rejects_a_bad_seed(bad):
    with pytest.raises(ValueError):
        gumbel_noise(bad, 0, 2, 2)


# ---- the semantic definition ------------------------------------------------------------------------------------------
def _policy(seed, d_in=64, d_hidden=256, d_out=6):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).bfloat16()   # noqa: E731
    return (r(d_hidden, d_in, scale=0.1), r(d_hidden, scale=0.5), r(d_hidden, d_hidden, scale=0.05),
            r(d_hidden, scale=0.5), r(d_out, d_hidden, scale=0.05), r(d_out, scale=0.5))


def _concat(results):
    acts = torch.cat([a for a, _ in results])
    lps = torch.cat([lp for _, lp in results])
    return acts, lps


@pytest.mark.parametrize("rows", [0, 2, 10, 13, 100])
def test_sampled_body_is_the_same_on_every_rank_count(rows):
    """1, 3 and 4 ranks (ragged shards, and empty shards past the data) give the same concatenated actions and
    log-probabilities bit for bit: each rank draws the noise of its rows' global indices.  The result is the
    Gumbel-max of the whole batch's logits."""
    p = _policy(rows + 3)
    obs = torch.randn(rows, 64, generator=torch.Generator().manual_seed(rows)).bfloat16()
    seed = 2**40 + rows
    runs = {n: ref_dispatch.spmd_call(policy_sample_cases.mlp_policy_sample, obs, *p, seed, num_proc=n)
            for n in (1, 3, 4)}
    for n, res in runs.items():
        assert len(res) == n
        for a, lp in res:
            assert a.dtype == torch.int64 and lp.dtype == torch.float32 and a.shape == lp.shape
    want_a, want_lp = _concat(runs[1])
    for n in (3, 4):
        a, lp = _concat(runs[n])
        assert torch.equal(a, want_a) and torch.equal(lp, want_lp), n
    import torch.nn.functional as F

    h = torch.relu(F.linear(obs, p[0], p[1]))
    h = torch.relu(F.linear(h, p[2], p[3]))
    logits = F.linear(h, p[4], p[5]).float()
    assert torch.equal(want_a, (logits + gumbel_noise(seed, 0, rows, 6)).argmax(-1))
    assert torch.equal(want_lp, torch.log_softmax(logits, -1).gather(-1, want_a[:, None]).squeeze(-1))


def test_sampled_body_follows_its_logits_distribution():
    """Many rows of one logit vector: the empirical frequencies follow softmax, and masked columns are never drawn."""
    logits = torch.tensor([1.0, 0.0, float("-inf"), 2.0, -1.0, float("-inf")])
    n = 200_000
    a = (logits + gumbel_noise(5, 0, n, 6)).argmax(-1)
    freq = torch.bincount(a, minlength=6).double() / n
    want = torch.softmax(logits.double(), -1)
    assert freq[2] == 0 and freq[5] == 0
    assert bool(((freq - want).abs() <= 5 * (want * (1 - want) / n).sqrt() + 1e-12).all()), (freq, want)


# ---- decoration ----------------------------------------------------------------------------------------------------
def test_sample_options_are_recorded_on_the_spec():
    import kubetorch_b200 as kt
    from kubetorch_b200.mapped import mapped_spec

    fn = kt.mapped("mlp", bias=True, output="sample", seed="seed")(policy_sample_cases.mlp_policy_sample)
    spec = mapped_spec(fn)
    assert spec.extra["output"] == "sample" and spec.extra["seed"] == "seed"
    const = mapped_spec(kt.mapped("mlp", bias=True, output="sample", seed=2**64 - 1)(lambda *a: None))
    assert const.extra["seed"] == 2**64 - 1


@pytest.mark.parametrize("kwargs", [
    {"output": "sample"}, {"bias": True, "output": "sample"}, {"output": "logits", "seed": 1},
    {"output": "both", "seed": "seed"}, {"seed": 1}, {"output": "sample", "seed": -1},
    {"output": "sample", "seed": 2**64}, {"output": "sample", "seed": True}, {"output": "sample", "seed": 1.5},
])
def test_bad_sample_options_raise_at_decoration(kwargs):
    """output="sample" needs seed=; seed= belongs to output="sample" only; a constant seed is an int in [0, 2**64)."""
    import kubetorch_b200 as kt

    with pytest.raises(ValueError):
        kt.mapped("mlp", **kwargs)


@pytest.mark.parametrize("op", ["identity", "scale", "affine"])
def test_seed_belongs_to_the_mlp_op(op):
    import kubetorch_b200 as kt

    with pytest.raises(ValueError):
        kt.mapped(op, seed=1)


# ---- Python argument checks -----------------------------------------------------------------------------------------
def _w(d_in=256, d_hidden=1024, d_out=18):
    return (torch.zeros(d_hidden, d_in, dtype=torch.bfloat16), torch.zeros(d_out, d_hidden, dtype=torch.bfloat16))


def test_python_checks_accept_sample_with_a_seed():
    from kubetorch_b200.device import mlp

    assert "sample" in mlp.OUTPUTS
    for d_out in (1, 18, 64, 256):
        w1, w3 = _w(d_out=d_out)
        for seed in (0, 1, 2**32, 2**64 - 1):
            assert mlp._check_policy(w1, w3, (None, None, None), "sample", seed) is None


@pytest.mark.parametrize("seed", [None, -1, 2**64, True, False, 1.0, "1"])
def test_python_checks_reject_a_bad_seed(seed):
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    with pytest.raises(ValueError):
        mlp._check_policy(w1, w3, (None, None, None), "sample", seed)
