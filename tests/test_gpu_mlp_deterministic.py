"""-m gpu: the deterministic actor head of the bf16 MLP policy (ktb_mlp_bf16_policy_deterministic*, output="deterministic"
of mlp_forward, mlp_scatter_gather and kt.mapped) — tied bit for bit to the Gaussian head and to the greedy head's
logits, its squashed and noisy actions against fp64 bars built from the greedy kernel's logits, the noise clip, the
clipped fraction, the header's IEEE cases, every form, chunking and row split, guard bands, status codes, the public
API and two GPUs."""
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

import policy_deterministic_cases as cases  # noqa: E402
from oracle import ref_dispatch  # noqa: E402

from kubetorch_b200.sampling import gumbel_uniform  # noqa: E402

INF, NAN = math.inf, float("nan")
EXPLORE = dict(noise=0.1)
SMOOTH = dict(noise=0.2, noise_clip=0.5)


def det_head(noise=0.0, noise_clip=INF, squash=1):
    """The C entries of the deterministic actor with these options."""
    entry = "ktb_mlp_bf16_policy_deterministic"
    return Head(entry, entry, entry + "_pushed", True, 0, {"actions": lambda d: 4 * d},
                lambda a: (a.get("noise", noise), a.get("noise_clip", noise_clip), a.get("squash", squash), a["seed"],
                           a["row_base"], a["actions"]))


DET = det_head()


# ---- inputs and helpers ---------------------------------------------------------------------------------------------
def actor(seed, d_out, bias=True):
    """(W1, W2, W3), (b1, b2, b3) of mlp_rig.config with the head scaled so that μ spans tanh's curved range."""
    w, b = config(seed, d_out, bias)
    return (w[0], w[1], w[2] * 50), b


def bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def same(got, want, what):
    assert len(got) == len(want), what
    for i, (g, h) in enumerate(zip(got, want)):
        assert g.shape == h.shape, (what, i)
        nan = g.isnan() & h.isnan()
        assert bool(((bits(g) == bits(h)) | nan).all()), (what, i, (bits(g) != bits(h)).nonzero()[:4].tolist())


def det(obs, w, b, seed=None, **kw):
    return mlp.mlp_forward(obs, *w, biases=b, output="deterministic", seed=seed, **kw)


def _z64(seed, row0, rows, cols):
    return torch.special.ndtri(gumbel_uniform(seed, row0, rows, cols, device="cuda", word3=1).double())


def _check_actions(mu, got, seed, row0, noise, noise_clip, squash, what, keep=None):
    """mu: the greedy kernel's bf16 logits of global rows row0, row0 + 1, ..., all finite; only entries where `keep` is
    set are held to the bar, when it is given.

    With t64 = tanh(μ) (μ unsquashed) and n64 = clamp(σ·z64, ±c), z64 = ndtri(u) in fp64, the reference is
    clamp(t64 + n64, ±1) squashed and t64 + n64 otherwise; both clamps are 1-Lipschitz, so the bar before them holds
    after.  tanhf is within CUDA's documented 2 ulp (<= 2^-22·|t64|, plus the smallest subnormals near 0); z is within
    normcdfinvf's 2^-20·(1 + |z64|) of z64 and σ·z is rounded once, so n is within σ·2^-19·(1 + |z64|) of σ·z64 (the
    Gaussian head's bar with σ in place of exp(log_std)); the sum is rounded once, 2^-24·(|t| + |n|)."""
    m = mu.double()
    assert bool(torch.isfinite(m).all()), what
    assert got.dtype == torch.float32 and got.shape == mu.shape, what
    t64 = torch.tanh(m) if squash else m
    tol = (2.0 ** -22 * t64.abs() + 2.0 ** -148) if squash else torch.zeros_like(t64)
    ref = t64
    if noise != 0:
        z64 = _z64(seed, row0, *mu.shape)
        n64 = (noise * z64).clamp(-noise_clip, noise_clip)
        ref = t64 + n64
        tol = tol + noise * 2.0 ** -19 * (1 + z64.abs()) + 2.0 ** -23 * (t64.abs() + n64.abs())
    if squash:
        ref = ref.clamp(-1, 1)
        assert bool((got.abs() <= 1).all()), what
    err = (got.double() - ref).abs()
    if keep is not None:
        err, tol = err[keep], tol[keep]
    assert bool((err <= tol).all()), (what, float((err / tol.clamp(min=1e-300)).max()), (err > tol).nonzero()[:4].tolist())


D_OUTS = [1, 2, 6, 17, 32, 63, 64, 100, 128, 129, 255, 256]


# ---- 1. ties to the heads already checked against fp64 --------------------------------------------------------------------
@pytest.mark.parametrize("bias", [True, False], ids=["biased", "bias_free"])
@pytest.mark.parametrize("d_out", D_OUTS)
def test_unsquashed_ties_to_the_gaussian_and_the_greedy_heads(K, d_out, bias):
    """Unsquashed with σ = 1 and c = +inf: ktb_mlp_bf16_policy_gaussian's actions with log_std = 0, bit for bit (both
    add __fmul_rn(1, z) = z to μ once).  Unsquashed with σ = 0: ktb_mlp_bf16_policy's logits widened to fp32, bit for
    bit (no noise is drawn or added, so -0.0 stays -0.0)."""
    M, seed = SHIPPED_CHUNK + 1005, 2**33 + 7 * d_out
    w, b = actor(5000 + d_out, d_out, bias)
    obs = randn((M, 256), 5010 + d_out)
    got = det(obs, w, b, seed, noise=1.0, squash=False)
    want, _ = mlp.mlp_forward(obs, *w, biases=b, output="gaussian", seed=seed,
                              log_std=torch.zeros(d_out, device="cuda"))
    same([got], [want], (d_out, "gaussian"))
    logits = mlp.mlp_forward(obs, *w, biases=b)
    same([det(obs, w, b, squash=False)], [logits.float()], (d_out, "logits"))


# ---- 2. fp64 bars against the greedy logits -----------------------------------------------------------------------------------
@pytest.mark.parametrize("d_out", [1, 6, 17, 64, 129, 256])
@pytest.mark.parametrize("chunk", [256, SHIPPED_CHUNK])
def test_bars_against_the_greedy_logits(K, d_out, chunk):
    """17 901 rows, a seed past 2^32: the noise-free squashed actions within tanhf's 2 ulp of fp64 tanh(μ), and the
    exploring (σ = 0.1) and smoothing (σ = 0.2, c = 0.5) actions, squashed and not, within _check_actions' bar, all
    against ktb_mlp_bf16_policy's logits of the same call."""
    M, seed = SHIPPED_CHUNK + 1005, 2**33 + 13 * d_out
    w, b = actor(5100 + d_out, d_out)
    obs = randn((M, 256), 5110 + d_out)
    with tuning(chunk):
        mu = mlp.mlp_forward(obs, *w, biases=b)
        assert float(mu.float().abs().max()) > 1.0, "μ reaches tanh's flat range"
        _check_actions(mu, det(obs, w, b), seed, 0, 0.0, INF, True, (d_out, chunk, "tanh"))
        for opts in (EXPLORE, SMOOTH):
            for squash in (True, False):
                got = det(obs, w, b, seed, squash=squash, **opts)
                _check_actions(mu, got, seed, 0, opts["noise"], opts.get("noise_clip", INF), squash,
                               (d_out, chunk, opts, squash))


@pytest.mark.parametrize("d_out", [6, 64, 256])
def test_clipped_noise_is_exactly_the_clip(K, d_out):
    """σ = 0.2, c = 0.5, unsquashed: where |σ·z64| exceeds c by more than the noise's own error, the action is
    fp32(μ) + ±c rounded once, bit for bit; and such entries exist."""
    M, seed, c = 20000, 2**36 + d_out, 0.5
    w, b = actor(5200 + d_out, d_out)
    obs = randn((M, 256), 5210 + d_out)
    mu = mlp.mlp_forward(obs, *w, biases=b).float()
    got = det(obs, w, b, seed, noise=0.2, noise_clip=c, squash=False)
    z64 = _z64(seed, 0, M, d_out)
    over = (0.2 * z64).abs() > c * (1 + 2.0 ** -10)
    assert int(over.sum()) > 100
    want = mu + torch.where(z64 > 0, c, -c).float()
    assert torch.equal(bits(got[over]), bits(want[over]))


def test_clipped_fraction_matches_the_normal_tail(K):
    """2^20 rows of μ = 0 (a zero head, no biases), σ = 0.2, c = 0.5, unsquashed: the action is the clipped noise
    itself, and the fraction equal to ±c is within 5 standard deviations of P(|z| > c/σ) = 2·(1 - Φ(2.5))."""
    from scipy.special import ndtr

    d_out, M, seed = 8, 1 << 20, 20261018
    w, _ = actor(5300, d_out, False)
    w = (w[0], w[1], torch.zeros_like(w[2]))
    obs = randn((1, 256), 5301).expand(M, 256).contiguous()
    a = det(obs, w, (None, None, None), seed, noise=0.2, noise_clip=0.5, squash=False)
    n = a.numel()
    frac = float((a.abs() == 0.5).double().mean())
    p = 2 * (1 - float(ndtr(2.5)))
    assert abs(frac - p) <= 5 * math.sqrt(p * (1 - p) / n), (frac, p)
    assert float(a.abs().max()) == 0.5


# ---- 3. the header's IEEE cases --------------------------------------------------------------------------------------------
EDGE_MU = [NAN, INF, -INF, 0.0, 0.25, 0.5, -3.0, 100.0]


def _edge(seed=77, M=1000):
    """A zero head with b3 = EDGE_MU: μ is EDGE_MU in every row (0·h + b, rounded to bf16 exactly)."""
    w, b = actor(5400, len(EDGE_MU))
    w = (w[0], w[1], torch.zeros_like(w[2]))
    b = (b[0], b[1], torch.tensor(EDGE_MU, device="cuda").bfloat16())
    return randn((M, 256), 5401), w, b


def test_edge_rows_follow_the_header(K):
    obs, w, b = _edge()
    M, d = obs.shape[0], len(EDGE_MU)
    seed = 12
    sign = torch.where(_z64(seed, 0, M, d) > 0, 1.0, -1.0).float()
    # a NaN μ stays NaN in every mode, and squashed actions stay in [-1, 1]
    for kw in (dict(), dict(noise=0.3, seed=seed), dict(noise=0.2, noise_clip=0.5, seed=seed)):
        a = det(obs, w, b, **kw)
        assert bool(a[:, 0].isnan().all()) and not bool(a[:, 1:].isnan().any()), kw
        assert bool((a.abs()[:, 1:] <= 1).all()), kw
    # noise-free, μ = ±inf gives ±1 squashed (and μ = 100 exactly 1)
    a = det(obs, w, b)
    assert bool((a[:, 1] == 1).all()) and bool((a[:, 2] == -1).all()) and bool((a[:, 7] == 1).all())
    # σ = inf, c = inf: every non-NaN μ gives ±1 squashed (the sign of z), and unsquashed ±inf, NaN where an infinite
    # μ meets noise of the opposite sign
    a = det(obs, w, b, seed, noise=INF)
    assert torch.equal(a[:, 1:], sign[:, 1:])
    a = det(obs, w, b, seed, noise=INF, squash=False)
    assert torch.equal(a[:, 3:], sign[:, 3:] * INF)
    assert torch.equal(a[:, 1].isnan(), sign[:, 1] < 0) and bool((a[:, 1][sign[:, 1] > 0] == INF).all())
    assert torch.equal(a[:, 2].isnan(), sign[:, 2] > 0) and bool((a[:, 2][sign[:, 2] < 0] == -INF).all())
    # c = 0 adds a signed zero: the values of the noise-free call, and a +0.0 μ stays +0.0
    for squash in (True, False):
        a = det(obs, w, b, seed, noise=0.7, noise_clip=0.0, squash=squash)
        r = det(obs, w, b, squash=squash)
        assert bool(((a == r) | (a.isnan() & r.isnan())).all()), squash
        assert not bool(torch.signbit(a[:, 3]).any()), squash


# ---- 4. forms, chunkings and row splits ------------------------------------------------------------------------------------
@pytest.mark.parametrize("opts", [{}, EXPLORE, SMOOTH], ids=["noise_free", "explore", "smooth"])
@pytest.mark.parametrize("squash", [True, False], ids=["tanh", "mu"])
@pytest.mark.parametrize("d_out", [1, 7, 32, 33, 64, 129, 256])
def test_every_form_gives_the_same_bits(K, d_out, squash, opts):
    """The plain form at the shipped and 256-row chunks, the staged form (pull kernel and copy engine), row splits with
    row_offset, mlp_scatter_gather on ranks [0, 0, 0] and the pushed form on ranks [0, 0, 0]: the same bits."""
    M, seed = 3 * 1408, (2**34 + 3 * d_out) if opts else None
    w, b = actor(5500 + d_out, d_out)
    obs = randn((M, 256), 5510 + d_out)
    kw = dict(squash=squash, **opts)
    got = det(obs, w, b, seed, **kw)
    for chunk in (256, SHIPPED_CHUNK):
        for ce in (None, 0, 1):
            with tuning(chunk, ce):
                same([det(obs, w, b, seed, staged=ce is not None, **kw)], [got], (chunk, ce))
    for split in (1, 1000, 2 * 1408 + 5):
        lo = det(obs[:split], w, b, seed, **kw)
        hi = det(obs[split:], w, b, seed, row_offset=split, **kw)
        same([torch.cat([lo, hi])], [got], ("split", split))
    views = mlp.mlp_scatter_gather(obs, *w, devices=[0, 0, 0], biases=b, output="deterministic", seed=seed, **kw)
    torch.cuda.synchronize()
    same([torch.cat(views)], [got], "scatter_gather")
    bounds = [K.shard_bounds(M, 3, r) for r in range(3)]
    actions = torch.full((M, d_out), -1.0, device="cuda")
    mlp._mlp_scatter_gather_pushed(obs, [0, 0, 0], bounds, {0: (w[0], w[1], w[2], b[0], b[1], b[2])}, "deterministic",
                                   None, actions, seed=seed, det=dict(noise=opts.get("noise"),
                                                                      noise_clip=opts.get("noise_clip"), squash=squash))
    torch.cuda.synchronize()
    same([actions], [got], "pushed")


@pytest.mark.parametrize("form,M,chunk,d_out,offset", [
    ("plain", 1000, SHIPPED_CHUNK, 7, 4), ("plain", 1000, 256, 18, 4), ("plain", 1000, 256, 256, 0),
    ("staged", 1408, 256, 63, 4), ("staged", 1408, 256, 64, 0), ("pushed", 3 * 1408, 256, 7, 4),
    ("pushed", 3 * 1408, 256, 32, 0), ("pushed", 3 * 1408, 256, 129, 4),
])
def test_writes_stay_inside_the_outputs(K, form, M, chunk, d_out, offset):
    """The fp32 actions [M, d_out] (as scalars at a 4-byte offset, as float2 where the stride and base allow), the
    scratch and the stage between guard bands; the results equal mlp_forward's bit for bit."""
    seed = 6
    w, b = actor(5600 + d_out, d_out)
    obs = randn((M, 256), 5601)
    want = det(obs, w, b, seed, **SMOOTH)
    bufs = run_guarded(form, det_head(**SMOOTH), K, chunk, obs, w, b, seed, offsets={"actions": offset})
    for name, buf in bufs.items():
        buf.check(f"{form} M={M} chunk={chunk} d_out={d_out}: {name}")
    assert torch.equal(bufs["actions"].view(torch.int32).view(want.shape), bits(want)), form


# ---- status codes ----------------------------------------------------------------------------------------------------------
STATUS_CASES = {
    "null_actions": (plain, dict(actions=0), L.ERR_ARG),
    "actions_2_bytes_in": (plain, dict(actions_off=2), L.ERR_ARG),
    "d_out_257": (plain, dict(d_out=257), L.ERR_UNSUPPORTED),
    "null_actions_before_d_out": (plain, dict(d_out=257, actions=0), L.ERR_ARG),
    "nan_noise": (plain, dict(noise=NAN), L.ERR_ARG),
    "negative_noise": (plain, dict(noise=-0.1), L.ERR_ARG),
    "nan_clip": (plain, dict(noise_clip=NAN), L.ERR_ARG),
    "negative_clip": (plain, dict(noise_clip=-1.0), L.ERR_ARG),
    "d_out_before_noise": (plain, dict(d_out=257, noise=NAN), L.ERR_UNSUPPORTED),
    "staged_nan_noise": (plain, dict(noise=NAN, stage=0), L.ERR_ARG),
    "inherited_d_in": (plain, dict(d_in=100, noise=NAN), L.ERR_ARG),
    "inherited_d_hidden": (plain, dict(d_hidden=384), L.ERR_ARG),
    "pushed_null_actions": (pushed, dict(actions=0), L.ERR_ARG),
    "pushed_d_out_257": (pushed, dict(d_out=257), L.ERR_UNSUPPORTED),
    "pushed_nan_clip": (pushed, dict(noise_clip=NAN), L.ERR_ARG),
    "pushed_negative_noise": (pushed, dict(noise=-INF), L.ERR_ARG),
    "pushed_inherited_seq": (pushed, dict(seq=0, noise=NAN), L.ERR_ARG),
    "pushed_inherited_stride": (pushed, dict(stride=(1 << 20) + 8), L.ERR_ARG),
}


@pytest.mark.parametrize("name", list(STATUS_CASES))
def test_bad_arguments_get_the_documented_status(K, name):
    form, overrides, status = STATUS_CASES[name]
    expect_status(form(DET, **overrides), status)


def test_empty_pushed_shard_runs_its_checks_and_acks(K):
    """An empty shard (M = 0) with null actions publishes ack[rank] = seq in the root's control block (its noise is not
    read); with a bad inherited argument it returns that entry's status."""
    ctrl_root = torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda")
    L.call(*pushed(DET, M=0, actions=0, ctrl_root=ctrl_root.data_ptr(), seq=3, rank=2, noise=NAN))
    torch.cuda.synchronize()
    assert int(ctrl_root[512 + 8 * 2:512 + 8 * 3].view(torch.int64)) == 3
    expect_status(pushed(DET, M=0, actions=0, seq=0), L.ERR_ARG)


# ---- Python checks -----------------------------------------------------------------------------------------------------------
def test_python_checks_name_the_output_in_mlp_forward_and_scatter_gather(K):
    (w1, w2, w3), b = config(5700, 18)
    obs = randn((256, 256), 5701)
    bad = [
        (dict(noise=0.1), "seed exactly when"),
        (dict(seed=1), "seed exactly when"),
        (dict(noise=0.1, seed=1, noise_clip=NAN), "noise_clip must be >= 0"),
        (dict(noise=-0.1, seed=1), "noise must be >= 0"),
        (dict(noise_clip=0.5), "noise_clip is an option of noise"),
        (dict(squash=1), "True or False"),
        (dict(mask=torch.ones(256, 18, dtype=torch.bool, device="cuda")), "mask is not an argument"),
        (dict(log_std=torch.zeros(18, device="cuda")), "log_std is not an argument"),
        (dict(output="gaussian", noise=0.1, seed=1, log_std=torch.zeros(18, device="cuda")),
         'noise is not an argument of output="gaussian"'),
    ]
    for kw, reason in bad:
        kw = dict(dict(output="deterministic"), **kw)
        with pytest.raises(ValueError, match=reason):
            mlp.mlp_forward(obs, w1, w2, w3, biases=b, **kw)
        with pytest.raises(ValueError, match=reason):
            mlp.mlp_scatter_gather(obs, w1, w2, w3, devices=[0], biases=b, **kw)


# ---- 5. the public API ------------------------------------------------------------------------------------------------------
PUBLIC = {
    "noise_free": (cases.mlp_policy_deterministic, dict(), (), dict()),
    "smoothing": (cases.mlp_policy_deterministic_smoothing, dict(noise=0.2, noise_clip=0.5, seed="seed"), ("seed",),
                  dict(noise=0.2, noise_clip=0.5, squash=True)),
    "unsquashed_named_sigma": (cases.mlp_policy_deterministic_unsquashed,
                               dict(noise="sigma", seed="seed", squash=False), ("sigma", "seed"),
                               dict(noise=0.3, squash=False)),
}


def _public_case(golden, kind):
    obs = torch.randn(1000, 256, generator=torch.Generator().manual_seed(1001)).bfloat16()
    p = list(policy_weights(golden, 6))
    p[4] = (p[4].float() * 50).bfloat16()
    body, options, names, mine_kw = PUBLIC[kind]
    seed = 2**35 + 41
    tail = tuple({"seed": seed, "sigma": 0.3}[n] for n in names)
    policy = mapped_copy(body, "mlp", bias=True, output="deterministic", **options)
    return obs, p, tail, seed if names else None, body, policy, mine_kw


def _mine(obs, p, seed, mine_kw):
    pc = [t.cuda() for t in p]
    return mlp.mlp_forward(obs.cuda(), pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]), output="deterministic",
                           seed=seed, **mine_kw)


def _against_body(K, obs, p, got, want, n):
    """Each rank's actions against the oracle's run of the body within rtol 2^-7, atol 1e-2 where the body's bf16 μ
    equals the kernel's (elsewhere they differ by a bf16 rounding of the logits, which the other tests tie down); at
    least 90 % of the μ must agree."""
    from policy_value_cases import _trunk

    pc = [t.cuda() for t in p]
    agree, total = 0, 0
    for r, (g, h) in enumerate(zip(got, want)):
        lo, hi = K.shard_bounds(obs.shape[0], n, r)
        with mock.patch.dict(os.environ, {"RANK": str(r), "WORLD_SIZE": str(n)}):
            mu_body = torch.nn.functional.linear(_trunk(obs, *p[:4]), p[4], p[5]).cuda()
        mu = mlp.mlp_forward(obs[lo:hi].cuda(), pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]))
        eq = mu_body == mu
        agree += int(eq.sum())
        total += eq.numel()
        assert bool(torch.isclose(g.cuda(), h.cuda(), rtol=2.0 ** -7, atol=1e-2)[eq].all()), r
    assert agree >= 0.9 * total, (agree, total)


@pytest.mark.parametrize("kind", list(PUBLIC))
@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["1_rank", "3_ranks"])
def test_mapped_deterministic_head_through_public_api(K, golden, devices, kind):
    """@kt.mapped("mlp", bias=True, output="deterministic", ...) on Compute(gpus=1): each rank returns the bits of
    mlp_forward over its rows, and agrees with the oracle's run of the body as _against_body states."""
    obs, p, tail, seed, body, policy, mine_kw = _public_case(golden, kind)
    n = len(devices)
    want = ref_dispatch.spmd_call(body, obs, *p, *tail, num_proc=n, serialization="pickle")
    mine = _mine(obs, p, seed, mine_kw)
    with deployed(policy, f"t-det-{kind}-{n}", devices) as remote:
        got = remote(obs.cuda(), *[t.cuda() for t in p], *tail, serialization="pickle")
        torch.cuda.synchronize()
    assert len(got) == len(want) == n
    for r, g in enumerate(got):
        lo, hi = K.shard_bounds(obs.shape[0], n, r)
        assert isinstance(g, torch.Tensor) and g.dtype == torch.float32, r
        same([g.cpu()], [mine[lo:hi].cpu()], r)
    _against_body(K, obs, p, got, want, n)


def test_mapped_deterministic_head_on_a_workers_subset(K, golden):
    """Two workers of one rank each on cuda:0; a call with workers=[1] returns rank 1's actions only, with the bits of
    mlp_forward over its rows."""
    import kubetorch_b200 as kt

    obs, p, tail, seed, body, policy, mine_kw = _public_case(golden, "smoothing")
    mine = _mine(obs, p, seed, mine_kw)
    remote = kt.fn(policy, name="t-det-workers").to(
        kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute("b200", workers=2, num_proc=1,
                                                                                 devices=[0, 0]))
    try:
        got = remote(obs.cuda(), *[t.cuda() for t in p], *tail, serialization="pickle", workers=[1])
        torch.cuda.synchronize()
    finally:
        remote.teardown()
    lo, hi = K.shard_bounds(obs.shape[0], 2, 1)
    assert len(got) == 1
    same([got[0].cpu()], [mine[lo:hi].cpu()], "workers=[1]")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("transfer", ["pull", "push"])
def test_mapped_deterministic_head_on_two_gpus(K, golden, transfer):
    """Two ranks on two GPUs, staged pull and pushed form, three calls, the head updated in place before the last: the
    bits of one plain call."""
    obs, p, tail, seed, body, policy, mine_kw = _public_case(golden, "smoothing")
    with deployed(policy, f"t-det-2gpu-{transfer}", [0, 1], transfer=transfer) as remote:
        pc = [t.cuda(0) for t in p]
        for it in range(3):
            x = torch.randn(2 * 1408, 256, generator=torch.Generator().manual_seed(5 + it)).bfloat16().cuda(0)
            if it == 2:
                pc[4].add_(0.125)
            got = remote(x, *pc, *tail, serialization="pickle")
            torch.cuda.synchronize(0)
            torch.cuda.synchronize(1)
            want = mlp.mlp_forward(x, pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]), output="deterministic",
                                   seed=seed, **mine_kw)
            same([torch.cat([g.cpu() for g in got])], [want.cpu()], it)
