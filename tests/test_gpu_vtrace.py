"""ktb_vtrace_f32 on the H100 against the header's restatement and the body of tests/policy_vtrace_cases.py run with
torch on the same GPU, bit for bit (NaN against NaN): every row count around the warp's 32 rows, every step count around
the 32-step tile, random episode boundaries, special values, several option sets, inputs and outputs at 4-byte offsets
that are not 16-byte aligned, and guard bands that must stay untouched.  Then ρ = expf(log_rho) against torch.exp over
all 2³² fp32 bit patterns; on-policy V-trace against ktb_gae_f32's λ = 1 returns; IMPALA's learner target from the MLP
sampling and evaluating heads; the entry's statuses in the header's order, the wrapper's checks, kt.mapped("vtrace")
through the public API and the deployment's self-check."""
import math
import os
from unittest import mock

import numpy as np
import pytest
import torch

from conftest import mapped_copy
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp, ops, returns
from mlp_rig import K, config, randn  # noqa: F401
from policy_vtrace_cases import (GAMMA, header_vtrace, mapped_vtrace, mapped_vtrace_args, mapped_vtrace_fixed_c,
                                 mapped_vtrace_other_gamma, mapped_vtrace_shifted, vtrace)
from test_gpu_gae import deployed, guarded, guards_untouched, placed

pytestmark = pytest.mark.gpu

# (gamma, lam, rho_bar, c_bar, pg_rho_bar): TorchBeast's defaults, λ < 1, unclipped, three different thresholds
OPTIONS = [(0.99, 1.0, 1.0, 1.0, 1.0), (0.99, 0.95, 1.0, 1.0, 1.0), (0.997, 1.0, None, None, None),
           (0.9, 0.9, 2.0, 0.8, 1.5), (0.0, 0.5, 0.5, None, 3.0)]
SPECIAL = [0.0, -0.0, 1.0, -1.5, 1e30, -1e30, 1e-40, math.inf, -math.inf, math.nan]


@pytest.fixture(scope="module")
def dev():
    ops.ensure_init([0])
    return 0


def same(got, want, what=""):
    got = torch.as_tensor(np.asarray(got.cpu() if isinstance(got, torch.Tensor) else got, dtype=np.float32))
    want = torch.as_tensor(np.asarray(want.cpu() if isinstance(want, torch.Tensor) else want, dtype=np.float32))
    assert got.shape == want.shape, (what, got.shape, want.shape)
    nan = want.isnan()
    assert torch.equal(got.isnan(), nan), what
    assert torch.equal(got[~nan].view(torch.int32), want[~nan].view(torch.int32)), what


def rollouts(n, t, seed, special=True):
    """Seeded env-major (log_rhos, rewards, values, dones, bootstrap_value) on the CPU: log-ratios on both sides of
    every threshold, random episode boundaries (done = 1), and with `special` a few done = 0.5 and NaN and the special
    values sprinkled over every other input."""
    g = torch.Generator().manual_seed(seed)
    lr = torch.randn(n, t, generator=g)
    r, v = torch.randn(n, t, generator=g) * 2, torch.randn(n, t, generator=g) * 5
    bv = torch.randn(n, generator=g) * 5
    d = (torch.rand(n, t, generator=g) < 0.05).float()
    if special:
        s = torch.tensor(SPECIAL)
        for x in (lr, r, v, bv):
            hit = torch.rand(x.shape, generator=g) < 0.01
            x[hit] = s[torch.randint(0, len(SPECIAL), (int(hit.sum()),), generator=g)]
        odd = torch.rand(n, t, generator=g)
        d[odd < 0.002] = 0.5
        d[odd > 0.999] = math.nan
    return lr, r, v, d, bv


def entry(dev, lr, r, v, d, bv, n, t, scalars, vs, pg):
    ptr = lambda x: x if isinstance(x, int) else x.data_ptr()   # noqa: E731
    return L.load().ktb_vtrace_f32(dev, ptr(lr), ptr(r), ptr(v), ptr(d), ptr(bv), n, t, *scalars, ptr(vs), ptr(pg),
                                   ops.current_stream_handle(0) if dev == 0 else 0)


def run_entry(dev, lr, r, v, d, bv, opts):
    """The C entry on offset copies of the inputs into guarded outputs: (vs, pg_adv) on the CPU, guards checked."""
    n, t = r.shape
    ins = [placed(x.contiguous(), o) for x, o in zip((lr, r, v, d, bv), (3, 1, 2, 3, 1))]
    (vbuf, vs), (pbuf, pg) = guarded(n * t, 1), guarded(n * t, 3)
    assert entry(dev, *ins, n, t, returns.vtrace_scalars(*opts), vs, pg) == L.OK, L.last_error()
    torch.cuda.synchronize()
    guards_untouched(vbuf, 1, n * t)
    guards_untouched(pbuf, 3, n * t)
    return vs.view(n, t).cpu(), pg.view(n, t).cpu()


# ---- the kernel against the header and the body -----------------------------------------------------------------------
NS = [0, 1, 31, 32, 33, 1000, 4097]
TS = [1, 2, 3, 31, 32, 33, 127, 128, 129, 2048]


@pytest.mark.parametrize("t", TS)
@pytest.mark.parametrize("n", NS)
def test_kernel_equals_header_and_body(dev, n, t):
    opts = OPTIONS[(NS.index(n) + TS.index(t)) % len(OPTIONS)]
    lr, r, v, d, bv = rollouts(n, t, seed=1000 * n + t)
    got = run_entry(dev, lr, r, v, d, bv, opts)
    cuda = [x.cuda() for x in (lr, r, v, d, bv)]
    for g, h, what in zip(got, header_vtrace(*cuda, *opts), ("vs", "pg_adv")):
        same(g, h, (n, t, "header " + what))
    if n * t <= 1000 * 129 or (n, t) == (8, 2048):
        for g, w, what in zip(got, vtrace(*cuda, *opts), ("vs", "pg_adv")):
            same(g, w, (n, t, "torch " + what))


@pytest.mark.parametrize("opts", OPTIONS, ids=[str(o) for o in OPTIONS])
def test_every_option_set_on_special_values(dev, opts):
    lr, r, v, d, bv = rollouts(97, 129, seed=7)
    s = torch.tensor(SPECIAL)
    lr[:40, 90] = s.repeat(4)[:40]
    r[:40, 100] = s.repeat(4)[:40]
    v[:40, 64] = s.repeat(4)[:40]
    bv[:40] = s.repeat(4)[:40]
    d[:, 63] = torch.tensor([0.0, 1.0, 0.5, math.nan]).repeat(25)[:97]
    got = run_entry(dev, lr, r, v, d, bv, opts)
    cuda = [x.cuda() for x in (lr, r, v, d, bv)]
    for g, w, h in zip(got, vtrace(*cuda, *opts), header_vtrace(*cuda, *opts)):
        same(g, w, opts)
        same(g, h, opts)


def test_expf_equals_torch_exp_at_every_fp32_bit_pattern(dev):
    """At T = 1 with r = 1, v = 0, done = 1, bootstrap = 0, ρ̄ = ρ̄_pg = +inf and c̄ = 1, disc = 0 and both outputs are
    ρ = expf(log_rho) exactly (c̄ stays finite: disc·c would be 0·inf).  All 2³² log-ratio bit patterns, 2²⁸ rows per
    launch, against torch.exp on the same GPU, NaN against NaN."""
    rows = 1 << 28
    r, v = torch.ones(rows, device="cuda:0"), torch.zeros(rows, device="cuda:0")
    d, bv = torch.ones(rows, device="cuda:0"), torch.zeros(rows, device="cuda:0")
    vs, pg = torch.empty(rows, device="cuda:0"), torch.empty(rows, device="cuda:0")
    scalars = returns.vtrace_scalars(GAMMA, 1.0, None, 1.0, None)
    differ, first = 0, []
    for lo in range(-(1 << 31), 1 << 31, rows):
        lr = torch.arange(lo, lo + rows, dtype=torch.int32, device="cuda:0").view(torch.float32)
        assert entry(dev, lr, r, v, d, bv, rows, 1, scalars, vs, pg) == L.OK, L.last_error()
        want = torch.exp(lr)
        nan = want.isnan()
        for got in (vs, pg):
            bad = (got.isnan() != nan) | (~nan & (got.view(torch.int32) != want.view(torch.int32)))
            differ += int(bad.sum())
            first += [hex(x) for x in lr.view(torch.int32)[bad][:8 - len(first)].tolist()]
        del lr, want, nan
    assert differ == 0, (differ, first)


def test_on_policy_vtrace_equals_the_gae_kernels_lambda_one_returns(dev):
    lr, r, v, d, bv = (x.cuda() for x in rollouts(1000, 129, seed=8, special=False))
    lr.zero_()
    vs, _ = returns.vtrace(lr, r, v, d, bv, GAMMA)
    _, ret = returns.gae(r, v, d, bv, GAMMA, 1.0)
    same(vs, ret)


def test_impala_learner_target_from_the_mlp_heads(K):
    """Behaviour log-probabilities and values from output="sample", target log-probabilities from output="evaluate":
    under the same weights log_rhos are 0 exactly and V-trace is the GAE λ = 1 return; under perturbed target weights
    the kernel equals the body on the GPU."""
    n, t, d_out = 64, 40, 18
    w, b = config(31, d_out)
    obs = randn((n * t, 256), 32)
    value = (randn((1, 1024), 33, 0.02), randn((1,), 34, 0.1))
    actions, behaviour_lp, values = mlp.mlp_forward(obs, *w, biases=b, output="sample", seed=35, value=value)
    target_lp = mlp.mlp_forward(obs, *w, biases=b, output="evaluate", taken=actions)[0]
    log_rhos = (target_lp - behaviour_lp).view(n, t)
    assert torch.equal(log_rhos, torch.zeros_like(log_rhos))
    g = torch.Generator().manual_seed(36)
    rewards = torch.randn(n, t, generator=g).cuda()
    dones = (torch.rand(n, t, generator=g) < 0.05).float().cuda()
    values = values.float().view(n, t).contiguous()
    bootstrap = torch.randn(n, generator=g).cuda()
    vs, pg = returns.vtrace(log_rhos, rewards, values, dones, bootstrap, GAMMA)
    same(vs, returns.gae(rewards, values, dones, bootstrap, GAMMA, 1.0)[1])
    w_t = tuple((x.float() + randn(x.shape, 40 + i, 0.004).float()).bfloat16() for i, x in enumerate(w))
    target_lp = mlp.mlp_forward(obs, *w_t, biases=b, output="evaluate", taken=actions)[0]
    log_rhos = (target_lp - behaviour_lp).view(n, t)
    assert (log_rhos > 0).any() and (log_rhos < 0).any()
    vs, pg = returns.vtrace(log_rhos, rewards, values, dones, bootstrap, GAMMA, 0.95)
    for got, want in zip((vs, pg), vtrace(log_rhos, rewards, values, dones, bootstrap, GAMMA, 0.95)):
        same(got, want)


def test_wrapper_takes_given_outputs_and_a_stream(dev):
    args = [x.cuda() for x in rollouts(100, 77, seed=9)]
    want = header_vtrace(*args, GAMMA, 0.9, 1.0, 0.9, 2.0)
    got = returns.vtrace(*args, GAMMA, 0.9, 1.0, 0.9, 2.0)
    vs, pg = torch.empty_like(args[0]), torch.empty_like(args[0])
    out = returns.vtrace(*args, GAMMA, 0.9, 1.0, 0.9, 2.0, vs=vs, pg_adv=pg, stream=torch.cuda.Stream())
    torch.cuda.synchronize()
    assert out[0] is vs and out[1] is pg
    for g, o, h in zip(got, out, want):
        same(g, h)
        same(o, h)


@pytest.mark.parametrize("case,match", [
    ("dtype", "values must be float32"),
    ("shape", "dones must have shape"),
    ("log_rhos", "log_rhos must have shape"),
    ("bootstrap", "bootstrap_value must have shape"),
    ("host", "values must be a CUDA tensor"),
    ("strided", "rewards must be contiguous"),
    ("dim", "rewards must be a 2-D"),
    ("out", "vs must have shape"),
    ("gamma", "gamma must be a finite number"),
    ("bar", "rho_bar must be a number > 0 or None"),
])
def test_wrapper_refuses_bad_arguments(dev, case, match):
    lr, r, v, d, bv = (x.cuda() for x in rollouts(10, 6, seed=10))
    kw = {}
    if case == "dtype":
        v = v.double()
    elif case == "shape":
        d = d[:, :5]
    elif case == "log_rhos":
        lr = lr[:9]
    elif case == "bootstrap":
        bv = bv[:9]
    elif case == "host":
        v = v.cpu()
    elif case == "strided":
        r = torch.empty(6, 10, device="cuda:0").t()
    elif case == "dim":
        r = r[0]
    elif case == "out":
        kw["vs"] = torch.empty(10, 5, device="cuda:0")
    elif case == "bar":
        kw["rho_bar"] = 0.0
    with pytest.raises(ValueError, match=match):
        returns.vtrace(lr, r, v, d, bv, math.nan if case == "gamma" else GAMMA, **kw)


def test_statuses_follow_the_header_order(dev):
    x = torch.zeros(64, device="cuda:0")
    nan, inf = math.nan, math.inf
    ok_scalars = (0.99, 0.9, 1.0, 1.0, 1.0)
    # an unregistered device comes first, before gamma
    assert entry(15, 0, 0, 0, 0, 0, 4, 4, (nan, 0.9, 1.0, 1.0, 1.0), 0, 0) == L.ERR_STATE
    # a non-finite gamma or lam, or a NaN or non-positive threshold, before the empty-input check
    for bad in [(nan, 0.9, 1, 1, 1), (0.99, inf, 1, 1, 1), (0.99, 0.9, nan, 1, 1), (0.99, 0.9, 1, 0.0, 1),
                (0.99, 0.9, 1, 1, -1.0), (0.99, 0.9, -inf, 1, 1)]:
        assert entry(dev, 0, 0, 0, 0, 0, 0, 4, bad, 0, 0) == L.ERR_ARG, bad
    # +inf thresholds are allowed; N·T == 0: nothing to do, NULL pointers allowed
    assert entry(dev, 0, 0, 0, 0, 0, 0, 4, (0.99, 0.9, inf, inf, inf), 0, 0) == L.OK
    assert entry(dev, 0, 0, 0, 0, 0, 4, 0, ok_scalars, 0, 0) == L.OK
    p = x.data_ptr()
    ok = dict(lr=p, r=p + 16, v=p + 32, d=p + 48, bv=p + 64, vs=p + 80, pg=p + 96)   # 2 x 2 rows of 4 bytes each

    def call(**over):
        a = dict(ok, **over)
        return entry(dev, a["lr"], a["r"], a["v"], a["d"], a["bv"], 2, 2, ok_scalars, a["vs"], a["pg"])

    assert call() == L.OK
    for name in ok:
        assert call(**{name: 0}) == L.ERR_ARG, name
        assert call(**{name: ok[name] + 2}) == L.ERR_ARG, name
    assert call(vs=p + 56) == L.ERR_ARG             # vs overlaps dones and bootstrap
    assert call(pg=p + 68) == L.ERR_ARG             # pg_adv overlaps bootstrap (8 bytes) and vs
    assert call(vs=p + 112, pg=p + 120) == L.ERR_ARG
    assert call(vs=p + 72, pg=p + 112) == L.OK      # vs right after bootstrap
    torch.cuda.synchronize()


# ---- kt.mapped("vtrace") through the public API -------------------------------------------------------------------------
def parts(got):
    return [(a.cpu(), b.cpu()) for a, b in got]


def oracle_on_gpu(body, args, n, *more):
    """The body rank by rank on the GPU, where its exp is the kernel's expf (torch's CPU exp is not)."""
    out = []
    for k in range(n):
        with mock.patch.dict(os.environ, {"RANK": str(k), "WORLD_SIZE": str(n)}):
            out.append(body(*(a.cuda() for a in args), *more))
    return out


@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["1_rank", "3_ranks"])
def test_mapped_equals_body_and_wrapper(dev, devices):
    n = len(devices)
    args = rollouts(1003, 200, seed=11)
    want = oracle_on_gpu(mapped_vtrace, args, n)
    mine = returns.vtrace(*(a.cuda() for a in args), GAMMA)
    fn = mapped_copy(mapped_vtrace, "vtrace", gamma=GAMMA)
    with deployed(fn, f"t-vtrace-{n}", devices) as remote:
        got = parts(remote(*(a.cuda() for a in args), serialization="pickle"))
    assert len(got) == len(want) == n
    for k, (g, w) in enumerate(zip(got, want)):
        lo, hi = ops.shard_bounds(1003, n, k)
        for i in range(2):
            same(g[i], w[i], (k, i))
            same(g[i], mine[i][lo:hi], (k, i))


def test_mapped_with_a_workers_subset(dev):
    """Three workers of one rank each on cuda:0; workers=[0, 2] computes ranks 0 and 2 only, workers=[1] rank 1."""
    args = rollouts(50, 33, seed=12)
    want = oracle_on_gpu(mapped_vtrace, args, 3)
    fn = mapped_copy(mapped_vtrace, "vtrace", gamma=GAMMA)
    with deployed(fn, "t-vtrace-workers", [0, 0, 0], workers=3, num_proc=1) as remote:
        gpu = [a.cuda() for a in args]
        two = parts(remote(*gpu, serialization="pickle", workers=[0, 2]))
        one = parts(remote(*gpu, serialization="pickle", workers=[1]))
    assert len(two) == 2 and len(one) == 1
    for g, k in zip(two + one, (0, 2, 1)):
        same(g[0], want[k][0], k)
        same(g[1], want[k][1], k)


def test_mapped_with_gamma_and_lam_as_call_arguments(dev):
    args = rollouts(77, 40, seed=13)
    fn = mapped_copy(mapped_vtrace_args, "vtrace", gamma="gamma", lam="lam")
    with deployed(fn, "t-vtrace-args", [0, 0]) as remote:
        for gamma, lam in [(0.99, 1.0), (0.9, 0.95), (0.0, 0.5)]:
            want = oracle_on_gpu(mapped_vtrace_args, args, 2, gamma, lam)
            got = parts(remote(*(a.cuda() for a in args), gamma, lam, serialization="pickle"))
            for g, w in zip(got, want):
                same(g[0], w[0], (gamma, lam))
                same(g[1], w[1], (gamma, lam))
        with pytest.raises(Exception, match="lam must be a finite number"):
            remote(*(a.cuda() for a in args), 0.99, math.nan, serialization="pickle")


def test_mapped_refuses_host_tensors(dev):
    args = rollouts(8, 4, seed=14)
    fn = mapped_copy(mapped_vtrace, "vtrace", gamma=GAMMA)
    with deployed(fn, "t-vtrace-host", [0]) as remote:
        with pytest.raises(Exception, match="'vtrace' op takes CUDA tensors on the root GPU"):
            remote(*args, serialization="pickle")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_mapped_on_two_gpus(dev):
    args = rollouts(4097, 129, seed=15)
    want = oracle_on_gpu(mapped_vtrace, args, 2)
    fn = mapped_copy(mapped_vtrace, "vtrace", gamma=GAMMA)
    with deployed(fn, "t-vtrace-2gpu", [0, 1]) as remote:
        got = parts(remote(*(a.cuda() for a in args), serialization="pickle"))
    for g, w in zip(got, want):
        same(g[0], w[0])
        same(g[1], w[1])


# ---- the deployment's self-check ----------------------------------------------------------------------------------------
WRONG = [(mapped_vtrace_shifted, {}), (mapped_vtrace_other_gamma, {}), (mapped_vtrace_fixed_c, dict(c_bar=0.9))]


@pytest.mark.parametrize("body,options", WRONG, ids=["shifted_done", "other_gamma", "fixed_c"])
def test_self_check_refuses_a_body_the_op_does_not_compute(dev, body, options):
    fn = mapped_copy(body, "vtrace", gamma=GAMMA, **options)
    with pytest.raises(ValueError, match="self-check failed.*clamping the traces at c_bar.*done flag of transition t"):
        with deployed(fn, f"t-vtrace-wrong-{body.__name__}", [0, 0]):
            pass
    # self_check=False deploys it anyway: the op computes the declared options with transition-t dones
    fn = mapped_copy(body, "vtrace", gamma=GAMMA, self_check=False, **options)
    args = [a.cuda() for a in rollouts(9, 9, seed=16)]
    with deployed(fn, f"t-vtrace-unchecked-{body.__name__}", [0, 0]) as remote:
        got = parts(remote(*args, serialization="pickle"))
    same(torch.cat([g[0] for g in got]), vtrace(*args, GAMMA, **options)[0])


def test_self_check_accepts_the_body(dev):
    for body, options in [(mapped_vtrace, {}), (mapped_vtrace_fixed_c, {})]:
        fn = mapped_copy(body, "vtrace", gamma=GAMMA, **options)
        with deployed(fn, f"t-vtrace-right-{body.__name__}", [0, 0, 0]) as remote:
            assert len(remote(*(a.cuda() for a in rollouts(5, 3, seed=17)), serialization="pickle")) == 3
