"""-m gpu: the Gaussian head of the bf16 MLP policy (ktb_mlp_bf16_policy_gaussian*, output="gaussian") — its actions
and log-probabilities against fp64 restatements built from the kernel's own logits, its noise against fp64 ndtri and
N(0, 1), deterministic columns, bit identity across chunkings, forms, row offsets and repeat calls, seeds, planted NaN
and infinite logits and log_std, guard bands, status codes, and the mapped op through the public API."""
import ctypes
import math
import os
from unittest import mock

import pytest
import torch

from conftest import mapped_copy
from test_gpu_mlp import SHIPPED_CHUNK, _Guarded
from test_gpu_mlp_policy import _PolicyPushRig, _config, _policy_weights, _randn, _stream

pytestmark = pytest.mark.gpu

import policy_gaussian_cases  # noqa: E402
from oracle import ref_dispatch  # noqa: E402

from kubetorch_b200.sampling import gumbel_uniform  # noqa: E402


@pytest.fixture(scope="module")
def K():
    assert torch.cuda.is_available()
    from kubetorch_b200.device import lib as L
    from kubetorch_b200.device import ops

    L.load()
    ops.ensure_init([0])
    return ops


def _L():
    from kubetorch_b200.device import lib as L

    return L


def _mlp():
    from kubetorch_b200.device import mlp

    return mlp


def _ptr(t):
    return 0 if t is None else t.data_ptr()


HALF_LOG_2PI = 0.5 * math.log(2 * math.pi)


# ---- the bars ----------------------------------------------------------------------------------------------------------
def _z64(seed, row0, rows, cols, device="cuda"):
    """z in fp64: ndtri of the exact uniform of the Gaussian stream (Philox counter word 3 = 1)."""
    return torch.special.ndtri(gumbel_uniform(seed, row0, rows, cols, device=device, word3=1).double())


def _check_gaussian(y, log_std, seed, row0, actions, log_probs, what):
    """y: the kernel's own bf16 logits of global rows row0, row0 + 1, ..., all finite; log_std finite.

    With z64 = ndtri(u) and σ64 = exp(log_std) in fp64 and z, σ the kernel's fp32 values:
      |z - z64| <= 2^-20·(1 + |z64|)        (the bar of the contract on normcdfinvf)
      |σ - σ64| <= 2^-22·σ64                 (expf: 2 ulp)
      a = fl(y + fl(σ·z)): each rounding adds at most 2^-24 of its result, and |a| <= |y| + σ|z|.
    So |a - (y + σ64·z64)| <= σ64·(2^-20·(1 + |z64|) + |z64|·(2^-22 + 2^-24)) + 2^-24·(|y| + σ64·|z64|) (to first
    order) <= 2^-19·σ64·(1 + |z64|) + 2^-23·|y|.
    For the log-probability, each term t_j = 0.5·z_j² + log_std_j differs from its fp64 value by at most
    |z|·|Δz| + 2^-23·|t_j| <= 2^-20·(1 + |z64_j|)² + 2^-23·|t_j| (the square, the half and the add each round once
    or fuse); the sum of d_out terms over a quad and the final subtraction add at most (d_out + 8)·2^-24 of the
    running magnitudes, which are bounded by Σ|t_j| + d_out·0.92.  Hence
      |lp - ref64| <= 2^-20·Σ_j(1 + |z64_j|)² + (d_out + 8)·2^-23·(Σ_j|t_j| + d_out·0.92)."""
    M, d_out = y.shape
    assert actions.dtype == torch.float32 and actions.shape == (M, d_out), what
    assert log_probs.dtype == torch.float32 and log_probs.shape == (M,), what
    yd = y.double()
    assert bool(torch.isfinite(yd).all()), what
    z64 = _z64(seed, row0, M, d_out, device=y.device)
    ls64 = log_std.double().to(y.device)
    s64 = ls64.exp()
    ref = yd + s64 * z64
    err = (actions.to(y.device).double() - ref).abs()
    tol = 2.0 ** -19 * s64 * (1 + z64.abs()) + 2.0 ** -23 * yd.abs()
    assert bool((err <= tol).all()), (what, float((err / tol).max()), (err > tol).nonzero()[:4].tolist())
    t = 0.5 * z64 * z64 + ls64
    ref_lp = -t.sum(-1) - d_out * HALF_LOG_2PI
    err_lp = (log_probs.to(y.device).double() - ref_lp).abs()
    tol_lp = 2.0 ** -20 * ((1 + z64.abs()) ** 2).sum(-1) + (d_out + 8) * 2.0 ** -23 * (t.abs().sum(-1) + d_out * 0.92)
    assert bool((err_lp <= tol_lp).all()), (what, float((err_lp / tol_lp).max()))


def _gauss(obs, w, b, log_std, seed, **kw):
    return _mlp().mlp_forward(obs, *w, biases=b, output="gaussian", log_std=log_std, seed=seed, **kw)


def _logits(obs, w, b):
    return _mlp().mlp_forward(obs, *w, biases=b, output="logits")


def _log_std(d_out, lo=-3.0, hi=1.0):
    return torch.linspace(lo, hi, d_out, device="cuda") if d_out > 1 else torch.tensor([lo], device="cuda")


# ---- 1. the bars at every head width -----------------------------------------------------------------------------------
@pytest.mark.parametrize("d_out", [1, 6, 17, 64, 129, 256])
@pytest.mark.parametrize("chunk", [256, SHIPPED_CHUNK])
def test_gaussian_bars_at_every_head_width(K, d_out, chunk):
    """17 901 rows: more than one chunk at either chunk size, and a partial last tile; a seed past 2^32; log_std spread
    over [-3, 1]; logits of a few units."""
    M, seed = SHIPPED_CHUNK + 1005, 2**33 + 7 * d_out
    w, b = _config(200 + d_out, d_out)
    w = (w[0], w[1], w[2] * 50)
    obs = _randn((M, 256), 210 + d_out)
    log_std = _log_std(d_out)
    K.set_tuning(8, chunk)
    try:
        y = _logits(obs, w, b)
        actions, log_probs = _gauss(obs, w, b, log_std, seed)
    finally:
        K.set_tuning(8, SHIPPED_CHUNK)
    _check_gaussian(y, log_std, seed, 0, actions, log_probs, f"d_out={d_out} chunk={chunk}")


# ---- 2. the noise and its distribution ---------------------------------------------------------------------------------
def _zero_head(seed_cfg, d_out):
    (w1, w2, _), (b1, b2, _) = _config(seed_cfg, d_out)
    w3 = torch.zeros(d_out, 1024, dtype=torch.bfloat16, device="cuda")
    b3 = torch.zeros(d_out, dtype=torch.bfloat16, device="cuda")
    return (w1, w2, w3), (b1, b2, b3)


def test_noise_meets_its_bar_and_follows_the_standard_normal(K):
    """W3 = 0, b3 = 0, log_std = 0: the actions are z itself (0 + 1·z is exact).  Over 2^20 × 8 draws: every z within
    2^-20·(1 + |z64|) of the fp64 ndtri of the exact u, none 0, all within ±5.29471; a KS test against N(0, 1) gives
    p > 1e-4; per-column mean and variance within 5 standard errors; the correlation of columns 2p and 2p + 1 (one
    Philox call) and of adjacent rows below 5/√n."""
    from scipy.stats import kstest

    d_out, M, seed = 8, 1 << 20, 20240611
    w, b = _zero_head(300, d_out)
    obs = _randn((M, 256), 301)
    z, log_probs = _gauss(obs, w, b, torch.zeros(d_out, device="cuda"), seed)
    z64 = _z64(seed, 0, M, d_out)
    err = (z.double() - z64).abs()
    ulp = torch.abs(torch.nextafter(z64.float(), torch.full_like(z, float("inf"))) - z64.float()).double()
    print(f"largest |z - ndtri64(u)|: {float((err / ulp).max()):.2f} ulp; largest error / bar: "
          f"{float((err / (2.0 ** -20 * (1 + z64.abs()))).max()):.4f}")
    assert bool((err <= 2.0 ** -20 * (1 + z64.abs())).all())
    assert bool((z != 0).all()) and bool((z.abs() <= 5.29471).all())
    stat = kstest(z.flatten().double().cpu().numpy(), "norm")
    print(f"KS over {z.numel()} draws: D={stat.statistic:.3g} p={stat.pvalue:.4f}")
    assert stat.pvalue > 1e-4, stat
    zd = z.double()
    mean, var = zd.mean(0), zd.var(0)
    assert bool((mean.abs() <= 5 / math.sqrt(M)).all()), mean.tolist()
    assert bool(((var - 1).abs() <= 5 * math.sqrt(2 / M)).all()), var.tolist()
    bound = 5 / math.sqrt(M)
    for p in range(d_out // 2):
        c = float(torch.corrcoef(torch.stack([zd[:, 2 * p], zd[:, 2 * p + 1]]))[0, 1])
        assert abs(c) < bound, ("columns", p, c)
    for j in range(d_out):
        c = float(torch.corrcoef(torch.stack([zd[:-1, j], zd[1:, j]]))[0, 1])
        assert abs(c) < 5 / math.sqrt(M - 1), ("rows", j, c)
    ref_lp = -(0.5 * z64 * z64).sum(-1) - d_out * HALF_LOG_2PI
    tol = 2.0 ** -20 * ((1 + z64.abs()) ** 2).sum(-1) + (d_out + 8) * 2.0 ** -23 * (
        (0.5 * z64 * z64).sum(-1) + d_out * 0.92)
    assert bool(((log_probs.double() - ref_lp).abs() <= tol).all())


# ---- 3. deterministic columns ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d_out", [6, 17, 200])
def test_minus_inf_log_std_gives_the_logits(K, d_out):
    """log_std = -inf on some columns: σ = 0, so those actions equal the logits of output="logits" (==), and every
    row's log-probability is +inf; the other columns still meet the bar."""
    w, b = _config(350 + d_out, d_out)
    obs = _randn((3000, 256), 351)
    log_std = _log_std(d_out).clone()
    det = list(range(0, d_out, 3))
    log_std[det] = float("-inf")
    y = _logits(obs, w, b)
    actions, log_probs = _gauss(obs, w, b, log_std, 5)
    assert bool((actions[:, det] == y[:, det].float()).all())
    assert bool(torch.isposinf(log_probs).all())
    live = [j for j in range(d_out) if j not in det]
    if live:
        z64 = _z64(5, 0, 3000, d_out)[:, live]
        s64 = log_std[live].double().exp()
        ref = y[:, live].double() + s64 * z64
        tol = 2.0 ** -19 * s64 * (1 + z64.abs()) + 2.0 ** -23 * y[:, live].double().abs()
        assert bool(((actions[:, live].double() - ref).abs() <= tol).all())


# ---- 4. identical bits ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d_out", [6, 17, 200])
def test_every_chunking_form_and_row_split_gives_identical_bits(K, d_out):
    """Repeat calls, chunk sizes 256 / 512 / shipped, plain and staged (kernel or copy-engine pull), and one call over
    M rows against two calls over [0, b) and [b, M) with row_offset = b."""
    w, b = _config(400 + d_out, d_out)
    M, seed = SHIPPED_CHUNK + 1000, 77
    obs = _randn((M, 256), 401)
    log_std = _log_std(d_out)
    want_a, want_lp = _gauss(obs, w, b, log_std, seed)
    again = _gauss(obs, w, b, log_std, seed)
    assert torch.equal(again[0], want_a) and torch.equal(again[1], want_lp)
    try:
        for chunk in (256, 512, SHIPPED_CHUNK):
            K.set_tuning(8, chunk)
            a, lp = _gauss(obs, w, b, log_std, seed)
            assert torch.equal(a, want_a) and torch.equal(lp, want_lp), ("plain", chunk)
            for ce in (0, 1):
                K.set_tuning(22, ce)
                a, lp = _gauss(obs, w, b, log_std, seed, staged=True)
                assert torch.equal(a, want_a) and torch.equal(lp, want_lp), ("staged", chunk, ce)
    finally:
        K.set_tuning(8, SHIPPED_CHUNK)
        K.set_tuning(22, 0)
    for split in (1, 1000, 16896, 16900):
        a0, lp0 = _gauss(obs[:split], w, b, log_std, seed)
        a1, lp1 = _gauss(obs[split:], w, b, log_std, seed, row_offset=split)
        assert torch.equal(torch.cat([a0, a1]), want_a) and torch.equal(torch.cat([lp0, lp1]), want_lp), split
    shifted = _gauss(obs, w, b, log_std, seed, row_offset=5)
    assert not torch.equal(shifted[0], want_a)


class _GaussianPushRig(_PolicyPushRig):
    """_PolicyPushRig driving ktb_mlp_bf16_policy_gaussian_pushed; rank r's row_base is its shard's begin."""

    def call(self, obs, w, b, d_out, log_std, seed, actions_ptr, log_probs_ptr):
        L = _L()
        self.seq += 1
        seq, n, d_in, st = self.seq, self.n, self.d_in, _stream()
        stage_ptrs = L.arr(ctypes.c_void_p, [0] + [s.ptr() for s in self.stage[1:]])
        ctrl_ptrs = L.arr(ctypes.c_void_p, [c.data_ptr() for c in self.ctrl])
        if self.engine == "sm":
            L.call("ktb_push_scatter_chunked", 0, obs.data_ptr(), obs.numel(), d_in, L.BF16, n, 0, stage_ptrs,
                   self.stride, ctrl_ptrs, self.ctrl[0].data_ptr(), self.chunk_rows * d_in, 0, seq, st)
        else:
            L.call("ktb_push_scatter_ce", 0, obs.data_ptr(), obs.numel(), d_in, L.BF16, n, 0,
                   L.arr(ctypes.c_int, [0] * n), stage_ptrs, self.stride, ctrl_ptrs, self.ctrl[0].data_ptr(),
                   self.chunk_rows * d_in, seq, st)
        for r in range(1, n):
            lo, hi = self.bounds[r]
            L.call("ktb_mlp_bf16_policy_gaussian_pushed", 0, self.stage[r].ptr(), self.stride, hi - lo, d_in,
                   self.d_hidden, d_out, w[0].data_ptr(), _ptr(b[0]), w[1].data_ptr(), _ptr(b[1]), w[2].data_ptr(),
                   _ptr(b[2]), log_std.data_ptr(), seed, lo, actions_ptr + lo * d_out * 4, log_probs_ptr + lo * 4,
                   self.scratch[r].ptr(), self.ctrl[r].data_ptr(), self.ctrl[0].data_ptr(), r, self.chunk_rows, seq, st)
        lo, hi = self.bounds[0]
        scratch = _mlp()._scratch_for(0, hi - lo, self.d_hidden)
        L.call("ktb_mlp_bf16_policy_gaussian", 0, obs.data_ptr() + lo * d_in * 2, hi - lo, d_in, self.d_hidden, d_out,
               w[0].data_ptr(), _ptr(b[0]), w[1].data_ptr(), _ptr(b[1]), w[2].data_ptr(), _ptr(b[2]),
               log_std.data_ptr(), seed, lo, actions_ptr + lo * d_out * 4, log_probs_ptr + lo * 4, scratch.data_ptr(),
               0, st)
        L.call("ktb_push_wait", 0, self.ctrl[0].data_ptr(), n, 0, seq, st)


@pytest.mark.parametrize("engine", ["sm", "ce"])
def test_pushed_form_on_one_gpu_matches_plain_bits(K, engine):
    """ktb_mlp_bf16_policy_gaussian_pushed fed by either scatter engine with ranks [0, 0, 0] on cuda:0, three
    consecutive calls with fresh observations: the actions and log-probabilities equal one plain call over all rows,
    bit for bit."""
    M, d_out, seed = 3 * 1408, 17, 2**40 + 3
    w, b = _config(500, d_out)
    log_std = _log_std(d_out)
    rig = _GaussianPushRig(K, M, 256, 1024, 512, engine)
    for it in range(3):
        obs = _randn((M, 256), 501 + it)
        want_a, want_lp = _gauss(obs, w, b, log_std, seed)
        actions = torch.full((M, d_out), float("nan"), dtype=torch.float32, device="cuda")
        log_probs = torch.full((M,), float("nan"), dtype=torch.float32, device="cuda")
        rig.call(obs, w, b, d_out, log_std, seed, actions.data_ptr(), log_probs.data_ptr())
        torch.cuda.synchronize()
        assert torch.equal(actions, want_a) and torch.equal(log_probs, want_lp), (engine, it)
    assert rig.statuses() == [0] * rig.n


def test_package_push_path_on_one_gpu_matches_plain_bits(K):
    """mlp_scatter_gather's pushed form (a cached PushSession, copy-engine scatter, the root's shard on the side
    stream) with ranks [0, 0, 0] on cuda:0 and output="gaussian": equal to one plain call over all rows."""
    mlp = _mlp()
    devs, rows, d_out, seed = [0, 0, 0], 35072, 6, 9
    M = 3 * rows
    bounds = [K.shard_bounds(M, 3, r) for r in range(3)]
    w, b = _config(510, d_out)
    log_std = _log_std(d_out)
    weights = {0: (*w, *b)}
    for it in range(2):
        obs = _randn((M, 256), 511 + it)
        want_a, want_lp = _gauss(obs, w, b, log_std, seed)
        actions = torch.full((M, d_out), float("nan"), dtype=torch.float32, device="cuda")
        log_probs = torch.full((M,), float("nan"), dtype=torch.float32, device="cuda")
        mlp._mlp_scatter_gather_pushed(obs, devs, bounds, weights, "gaussian", None, actions, log_probs, seed,
                                       {0: log_std})
        torch.cuda.synchronize()
        assert torch.equal(actions, want_a) and torch.equal(log_probs, want_lp), it
    mlp._push_sessions[tuple(devs)].check()


# ---- 5. seeds ------------------------------------------------------------------------------------------------------------
def test_nearby_seeds_draw_different_noise_and_not_the_gumbel_stream(K):
    """Seeds s, s + 1 and s + 2^32 give different draws (no two agree on any element of 8192 × 6), and the draws of a
    seed are not the Gaussian transform of the Gumbel stream's uniforms at the same seed."""
    d_out = 6
    w, b = _zero_head(600, d_out)
    obs = _randn((8192, 256), 601)
    zeros = torch.zeros(d_out, device="cuda")
    s = 123456789
    draws = [_gauss(obs, w, b, zeros, seed)[0] for seed in (s, s + 1, s + 2**32)]
    for i in range(3):
        for j in range(i + 1, 3):
            assert float((draws[i] == draws[j]).double().mean()) < 1e-3, (i, j)
    gumbel_z = torch.special.ndtri(gumbel_uniform(s, 0, 8192, d_out, device="cuda").double())
    assert float(((draws[0].double() - gumbel_z).abs() < 1e-5).double().mean()) < 1e-3


# ---- 6. planted values ---------------------------------------------------------------------------------------------------
def test_planted_nan_and_infinite_logits_touch_their_column_only(K):
    """NaN, +inf and -inf logits from b3 (columns 3, 5, 6): those action columns are NaN, +inf and -inf, every other
    column and every log-probability equal a call with a finite b3 bit for bit."""
    d_out = 9
    w, b = _config(650, d_out)
    obs = _randn((2000, 256), 651)
    log_std = _log_std(d_out)
    want_a, want_lp = _gauss(obs, w, b, log_std, 44)
    b3 = b[2].clone()
    b3[3], b3[5], b3[6] = float("nan"), float("inf"), float("-inf")
    a, lp = _gauss(obs, w, (b[0], b[1], b3), log_std, 44)
    assert bool(torch.isnan(a[:, 3]).all())
    assert bool(torch.isposinf(a[:, 5]).all()) and bool(torch.isneginf(a[:, 6]).all())
    keep = [j for j in range(d_out) if j not in (3, 5, 6)]
    assert torch.equal(a[:, keep], want_a[:, keep])
    assert torch.equal(lp, want_lp)


def test_overflowing_logits_touch_their_column_only(K):
    """Identity hidden layers pass non-negative observations through exactly; trigger units of 2^100 times W3 entries
    of ±2^100 overflow the head's accumulator to ±inf in columns 1 and 4 on every other row."""
    from test_gpu_mlp import _identity

    d, d_out, M, big = 256, 6, 2048, 2.0 ** 100
    obs = torch.rand(M, d, generator=torch.Generator(device="cuda").manual_seed(7), device="cuda") * 0.5
    obs[:, 200:] = 0
    w3 = torch.randn(d_out, d, generator=torch.Generator(device="cuda").manual_seed(8), device="cuda") * 0.5
    w3[:, 200:] = 0
    w3[1, 255], w3[4, 255] = big, -big
    rows = torch.arange(0, M, 2, device="cuda")
    obs[rows, 255] = big
    obs, w3 = obs.bfloat16(), w3.bfloat16()
    w, b = (_identity(d), _identity(d), w3), (None, None, None)
    log_std = _log_std(d_out)
    y = _logits(obs, w, b)
    a, lp = _gauss(obs, w, b, log_std, 3)
    assert bool(torch.isposinf(y[rows, 1]).all()) and bool(torch.isneginf(y[rows, 4]).all())
    assert bool(torch.isposinf(a[rows, 1]).all()) and bool(torch.isneginf(a[rows, 4]).all())
    finite = torch.isfinite(y.float()).all(1)
    assert int(finite.sum()) == M // 2
    assert bool(torch.isfinite(lp).all())
    ref_lp = -(0.5 * _z64(3, 0, M, d_out) ** 2 + log_std.double()).sum(-1) - d_out * HALF_LOG_2PI
    assert bool(((lp.double() - ref_lp).abs() <= 1e-4).all())
    idx = finite.nonzero()[:, 0]
    z64 = _z64(3, 0, M, d_out)[idx]
    s64 = log_std.double().exp()
    tol = 2.0 ** -19 * s64 * (1 + z64.abs()) + 2.0 ** -23 * y[idx].double().abs()
    assert bool(((a[idx].double() - (y[idx].double() + s64 * z64)).abs() <= tol).all())


def test_planted_nan_and_infinite_log_std(K):
    """log_std = +inf at column 1: σ = inf, the action is ±inf with the sign of z (never 0) and the log-probability
    -inf; NaN at column 2: a NaN column and NaN log-probabilities; -inf at column 0 with +inf elsewhere: NaN
    log-probabilities (inf - inf), and the column equals the logits."""
    d_out, M, seed = 5, 3000, 81
    w, b = _config(660, d_out)
    obs = _randn((M, 256), 661)
    y = _logits(obs, w, b).float()
    z64 = _z64(seed, 0, M, d_out)
    base = _log_std(d_out)

    ls = base.clone()
    ls[1] = float("inf")
    a, lp = _gauss(obs, w, b, ls, seed)
    assert torch.equal(a[:, 1], torch.where(z64[:, 1] > 0, float("inf"), float("-inf")).float())
    assert bool(torch.isneginf(lp).all())

    ls = base.clone()
    ls[2] = float("nan")
    a, lp = _gauss(obs, w, b, ls, seed)
    assert bool(torch.isnan(a[:, 2]).all()) and bool(torch.isnan(lp).all())
    keep = [0, 1, 3, 4]
    want_a, _ = _gauss(obs, w, b, base, seed)
    assert torch.equal(a[:, keep], want_a[:, keep])

    ls = base.clone()
    ls[0], ls[3] = float("-inf"), float("inf")
    a, lp = _gauss(obs, w, b, ls, seed)
    assert torch.equal(a[:, 0], y[:, 0]) and bool(torch.isnan(lp).all())


# ---- 7. guard bands --------------------------------------------------------------------------------------------------
class _Offset4(_Guarded):
    """A _Guarded buffer whose base is 4 bytes past an 8-byte boundary: float2 stores would be misaligned."""

    def __init__(self, nbytes):
        super().__init__(nbytes)
        self.band += 4
        self.raw = torch.full((self.nbytes + 2 * self.band,), self.FILL, dtype=torch.uint8, device="cuda")


@pytest.mark.parametrize("form,M,chunk,d_out,offset", [
    ("plain", 1000, SHIPPED_CHUNK, 7, False), ("plain", 1000, 256, 18, True), ("plain", 1000, 256, 130, False),
    ("staged", 1408, 256, 17, False), ("staged", 1408, 256, 18, True), ("pushed", 3 * 1408, 256, 7, False),
    ("pushed", 3 * 1408, 256, 18, True),
])
def test_writes_stay_inside_actions_and_log_probs(K, form, M, chunk, d_out, offset):
    """actions (M·d_out·4 bytes), log_probs (M·4), scratch and stage between guard bands; an odd d_out (scalar
    stores) and an even d_out with the actions base 4 bytes past an 8-byte boundary (the scalar fallback); a logits
    buffer passed to no one stays untouched; the results equal mlp_forward's bit for bit."""
    L = _L()
    d_in, d_hidden, seed = 256, 1024, 5
    w, b = _config(700, d_out)
    obs = _randn((M, d_in), 701)
    log_std = _log_std(d_out)
    want_a, want_lp = _gauss(obs, w, b, log_std, seed)
    K.set_tuning(8, chunk)
    try:
        actions = (_Offset4 if offset else _Guarded)(M * d_out * 4)
        assert (actions.ptr() % 8 == 4) == offset
        log_probs, logits = _Guarded(M * 4), _Guarded(M * d_out * 2)
        buffers = {"actions": actions, "log_probs": log_probs}
        if form == "pushed":
            rig = _GaussianPushRig(K, M, d_in, d_hidden, 512, "sm")
            for _ in range(3):
                rig.call(obs, w, b, d_out, log_std, seed, actions.ptr(), log_probs.ptr())
            torch.cuda.synchronize()
            assert rig.statuses() == [0] * rig.n
            buffers.update({f"stage[{r}]": rig.stage[r] for r in range(1, rig.n)})
            buffers.update({f"scratch[{r}]": rig.scratch[r] for r in range(1, rig.n)})
        else:
            scratch = _Guarded(L.load().ktb_mlp_scratch_bytes(M, d_hidden))
            buffers["scratch"] = scratch
            stage = 0
            if form == "staged":
                buffers["stage"] = _Guarded(L.load().ktb_mlp_stage_bytes(M, d_in))
                stage = buffers["stage"].ptr()
            L.call("ktb_mlp_bf16_policy_gaussian", 0, obs.data_ptr(), M, d_in, d_hidden, d_out, w[0].data_ptr(),
                   b[0].data_ptr(), w[1].data_ptr(), b[1].data_ptr(), w[2].data_ptr(), b[2].data_ptr(),
                   log_std.data_ptr(), seed, 0, actions.ptr(), log_probs.ptr(), scratch.ptr(), stage, _stream())
        for name, buf in buffers.items():
            buf.check(f"{form} M={M} chunk={chunk} d_out={d_out} offset={offset}: {name}")
        assert bool((logits.view() == _Guarded.FILL).all()), "a logits buffer nobody was given changed"
        assert torch.equal(actions.view(torch.float32).view(M, d_out), want_a)
        assert torch.equal(log_probs.view(torch.float32), want_lp)
    finally:
        K.set_tuning(8, SHIPPED_CHUNK)


# ---- 8. status codes -------------------------------------------------------------------------------------------------
def _arg_case(name):
    L = _L()
    w1, w2, w3 = (torch.zeros(s, dtype=torch.bfloat16, device="cuda") for s in ((1024, 256), (1024, 1024), (512, 1024)))
    bias = torch.zeros(1024, dtype=torch.bfloat16, device="cuda")
    obs = torch.zeros(2048, 256, dtype=torch.bfloat16, device="cuda")
    act = torch.zeros(2048 * 512, dtype=torch.float32, device="cuda")
    lp = torch.zeros(2048, dtype=torch.float32, device="cuda")
    ls = torch.zeros(512, dtype=torch.float32, device="cuda")
    scratch = torch.zeros(1 << 24, dtype=torch.uint8, device="cuda")
    ctrl = torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda")
    p = lambda t, off=0: t.data_ptr() + off   # noqa: E731

    def plain(d_out=18, actions=None, log_probs=None, log_std=None):
        return ("ktb_mlp_bf16_policy_gaussian", 0, p(obs), 256, 256, 1024, d_out, p(w1), p(bias), p(w2), p(bias),
                p(w3), p(bias), p(ls) if log_std is None else log_std, 1, 0, p(act) if actions is None else actions,
                p(lp) if log_probs is None else log_probs, p(scratch), 0, _stream())

    def pushed(d_out=18, actions=None, log_probs=None, log_std=None):
        return ("ktb_mlp_bf16_policy_gaussian_pushed", 0, p(scratch), 1 << 20, 256, 256, 1024, d_out, p(w1), p(bias),
                p(w2), p(bias), p(w3), p(bias), p(ls) if log_std is None else log_std, 1, 0,
                p(act) if actions is None else actions, p(lp) if log_probs is None else log_probs, p(scratch),
                p(ctrl), p(ctrl), 1, 256, 1, _stream())

    table = {
        "null_actions": (plain(actions=0), L.ERR_ARG),
        "null_log_probs": (plain(log_probs=0), L.ERR_ARG),
        "null_log_std": (plain(log_std=0), L.ERR_ARG),
        "misaligned_actions": (plain(actions=p(act, 2)), L.ERR_ARG),
        "misaligned_log_probs": (plain(log_probs=p(lp, 2)), L.ERR_ARG),
        "misaligned_log_std": (plain(log_std=p(ls, 1)), L.ERR_ARG),
        "d_out_257": (plain(d_out=257), L.ERR_UNSUPPORTED),
        "pushed_null_actions": (pushed(actions=0), L.ERR_ARG),
        "pushed_null_log_probs": (pushed(log_probs=0), L.ERR_ARG),
        "pushed_null_log_std": (pushed(log_std=0), L.ERR_ARG),
        "pushed_misaligned_actions": (pushed(actions=p(act, 1)), L.ERR_ARG),
        "pushed_misaligned_log_probs": (pushed(log_probs=p(lp, 1)), L.ERR_ARG),
        "pushed_misaligned_log_std": (pushed(log_std=p(ls, 2)), L.ERR_ARG),
        "pushed_d_out_257": (pushed(d_out=257), L.ERR_UNSUPPORTED),
    }
    return table[name]


@pytest.mark.parametrize("name", [
    "null_actions", "null_log_probs", "null_log_std", "misaligned_actions", "misaligned_log_probs",
    "misaligned_log_std", "d_out_257", "pushed_null_actions", "pushed_null_log_probs", "pushed_null_log_std",
    "pushed_misaligned_actions", "pushed_misaligned_log_probs", "pushed_misaligned_log_std", "pushed_d_out_257",
])
def test_bad_arguments_get_the_documented_status(K, name):
    L = _L()
    args, status = _arg_case(name)
    with pytest.raises(L.KtbError) as ei:
        L.call(*args)
    assert ei.value.status == status, (name, str(ei.value))
    torch.cuda.synchronize()    # nothing was launched; the device stays healthy


def test_python_checks_reach_mlp_forward(K):
    (w1, w2, w3), b = _config(800, 18)
    obs = _randn((256, 256), 801)
    ls = torch.zeros(18, device="cuda")
    for bad in (None, -1, 2**64, True, 1.0):
        with pytest.raises(ValueError):
            _mlp().mlp_forward(obs, w1, w2, w3, biases=b, output="gaussian", seed=bad, log_std=ls)
    for bad in (None, torch.zeros(18), torch.zeros(17, device="cuda"), torch.zeros(18, device="cuda").double(),
                torch.zeros(36, device="cuda")[::2]):
        with pytest.raises(ValueError):
            _mlp().mlp_forward(obs, w1, w2, w3, biases=b, output="gaussian", seed=1, log_std=bad)
    with pytest.raises(ValueError):
        _mlp().mlp_forward(obs, w1, w2, w3, biases=b, output="gaussian", seed=1, log_std=ls, row_offset=-1)
    with pytest.raises(ValueError):
        _mlp().mlp_forward(obs, w1, w2, w3, biases=b, output="sample", seed=1, log_std=ls)
    a, lp = _mlp().mlp_forward(obs, w1, w2, w3, biases=b, output="gaussian", seed=1, log_std=ls)
    assert a.shape == (256, 18) and lp.shape == (256,)


# ---- 9. the public API ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["recorded", "ragged_1000_rows_3_ranks", "2_rows_3_ranks"])
def test_mapped_gaussian_through_public_api(K, golden, case):
    """@kt.mapped("mlp", bias=True, output="gaussian", seed="seed", log_std="log_std") on Compute(gpus=1) with three
    ranks on cuda:0, against the oracle's run of the body: each rank's draws satisfy the bars over its rows' global
    indices, and agree with the body's actions within the action bar wherever the body's bf16 logits equal the
    kernel's."""
    import kubetorch_b200 as kt

    if case == "recorded":
        obs, d_out = golden["all_inputs"]["mlp_obs"], 64
    else:
        rows = 1000 if case.startswith("ragged") else 2
        obs, d_out = torch.randn(rows, 256, generator=torch.Generator().manual_seed(rows)).bfloat16(), 6
    p = _policy_weights(golden, d_out)
    log_std = torch.linspace(-3, 1, d_out)
    n_ranks, seed = 3, 2**35 + 17
    want = ref_dispatch.spmd_call(policy_gaussian_cases.mlp_policy_gaussian, obs, *p, log_std, seed,
                                  num_proc=n_ranks, serialization="pickle")
    policy = mapped_copy(policy_gaussian_cases.mlp_policy_gaussian, "mlp", bias=True, output="gaussian", seed="seed",
                         log_std="log_std")
    remote = kt.fn(policy, name=f"t-gaussian-{case}").to(
        kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute(
            "b200", workers=1, num_proc=n_ranks, devices=[0] * n_ranks))
    try:
        pc = [t.cuda() for t in p]
        lsc = log_std.cuda()
        got = remote(obs.cuda(), *pc, lsc, seed, serialization="pickle")
        torch.cuda.synchronize()
        assert len(got) == len(want) == n_ranks
        y = _mlp().mlp_forward(obs.cuda(), pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]))
        from policy_cases import mlp_policy_biased

        same, total = 0, 0
        for r, (g, h) in enumerate(zip(got, want)):
            lo, hi = K.shard_bounds(obs.shape[0], n_ranks, r)
            with mock.patch.dict(os.environ, {"RANK": str(r), "WORLD_SIZE": str(n_ranks)}):
                y_shard = mlp_policy_biased(obs, *p).float()   # the body's own μ of rank r's rows
            assert isinstance(g, tuple) and len(g) == 2, (case, r)
            assert g[0].shape == h[0].shape == (hi - lo, d_out) and g[1].shape == h[1].shape == (hi - lo,)
            if hi == lo:
                continue
            _check_gaussian(y[lo:hi], lsc, seed, lo, g[0].cuda(), g[1].cuda(), (case, r))
            eq = y_shard == y[lo:hi].float().cpu()
            z64 = _z64(seed, lo, hi - lo, d_out, device="cpu")
            s64 = log_std.double().exp()
            tol = 2.0 ** -19 * s64 * (1 + z64.abs()) + 2.0 ** -23 * y_shard.double().abs()
            close = (g[0].cpu().double() - h[0].double()).abs() <= tol
            assert bool(close[eq].all()), (case, r)
            same += int(eq.sum())
            total += eq.numel()
        print(f"{case}: the body's logits equal the kernel's on {same} of {total} elements")
    finally:
        remote.teardown()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("transfer", ["pull", "push"])
def test_mapped_gaussian_on_two_gpus(K, golden, transfer):
    """Two ranks on two GPUs, staged pull and pushed form: the same bits as one plain call over all rows."""
    import kubetorch_b200 as kt

    obs = torch.randn(2 * 1408, 256, generator=torch.Generator().manual_seed(5)).bfloat16()
    p = _policy_weights(golden, 18)
    log_std = torch.linspace(-2, 0.5, 18)
    seed = 4242
    policy = mapped_copy(policy_gaussian_cases.mlp_policy_gaussian, "mlp", bias=True, output="gaussian", seed="seed",
                         log_std="log_std")
    remote = kt.fn(policy, name=f"t-gaussian-2gpu-{transfer}").to(
        kt.Compute(gpus=2, allowed_serialization=["json", "pickle"]).distribute(
            "b200", workers=1, num_proc=2, devices=[0, 1], transfer=transfer))
    try:
        pc = [t.cuda(0) for t in p]
        lsc = log_std.cuda(0)
        got = remote(obs.cuda(0), *pc, lsc, seed, serialization="pickle")
        torch.cuda.synchronize(0)
        torch.cuda.synchronize(1)
        want_a, want_lp = _mlp().mlp_forward(obs.cuda(0), pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]),
                                             output="gaussian", seed=seed, log_std=lsc)
        assert torch.equal(torch.cat([g[0].cpu() for g in got]), want_a.cpu())
        assert torch.equal(torch.cat([g[1].cpu() for g in got]), want_lp.cpu())
    finally:
        remote.teardown()
