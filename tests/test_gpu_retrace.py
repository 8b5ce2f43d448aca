"""ktb_retrace_f32 on the H100 against the header's restatement and the body of tests/policy_retrace_cases.py run with
torch on the same GPU, bit for bit (NaN against NaN): every row count around the warp's 32 rows, every step count around
the 32-step tile, random episode boundaries, special values, several (γ, λ) pairs, inputs and outputs at 4-byte offsets
that are not 16-byte aligned, guard bands that must stay untouched, and baseline aliasing q.  Then on-policy Retrace at
λ = 1 against ktb_nstep_f32 at n = 32; λ = 0 over the ε-greedy head's q_max against output="dqn_target"; Watkins' Q(λ)
over ε-greedy behaviour; the entry's statuses in the header's order, the wrapper's checks, kt.mapped("retrace") through
the public API and the deployment's self-check.  ρ = expf(log_rho) is the kernel test_gpu_vtrace.py pins against
torch.exp at every fp32 bit pattern, so that sweep is not repeated here."""
import math
import os
from unittest import mock

import pytest
import torch

from conftest import mapped_copy
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp, ops, returns
from mlp_rig import K, config, randn  # noqa: F401
from policy_retrace_cases import (GAMMA, LAM, header_retrace, mapped_retrace, mapped_retrace_args,
                                  mapped_retrace_current_value, mapped_retrace_other_gamma, mapped_retrace_other_lam,
                                  mapped_retrace_shifted, mapped_retrace_unclipped, retrace)
from test_gpu_gae import deployed, guarded, guards_untouched, parts, placed, same

pytestmark = pytest.mark.gpu

# (gamma, lam): the usual pair, λ = 1, λ = 0, γ = 0, and γ = 1
OPTIONS = [(0.99, 0.95), (0.997, 1.0), (0.9, 0.0), (0.0, 0.5), (1.0, 0.9)]
SPECIAL = [0.0, -0.0, 1.0, -1.5, 1e30, -1e30, 1e-40, math.inf, -math.inf, math.nan]


@pytest.fixture(scope="module")
def dev():
    ops.ensure_init([0])
    return 0


def rollouts(n, t, seed, special=True):
    """Seeded env-major (log_rhos, rewards, q, values, dones, baseline, bootstrap_value) on the CPU: log-ratios on both
    sides of the clip at ρ = 1, random episode boundaries (done = 1), and with `special` a few done = 0.5 and NaN and
    the special values sprinkled over every other input."""
    g = torch.Generator().manual_seed(seed)
    lr = torch.randn(n, t, generator=g)
    r, q = torch.randn(n, t, generator=g) * 2, torch.randn(n, t, generator=g) * 5
    v, b = torch.randn(n, t, generator=g) * 5, torch.randn(n, t, generator=g) * 5
    bv = torch.randn(n, generator=g) * 5
    d = (torch.rand(n, t, generator=g) < 0.05).float()
    if special:
        s = torch.tensor(SPECIAL)
        for x in (lr, r, q, v, b, bv):
            hit = torch.rand(x.shape, generator=g) < 0.01
            x[hit] = s[torch.randint(0, len(SPECIAL), (int(hit.sum()),), generator=g)]
        odd = torch.rand(n, t, generator=g)
        d[odd < 0.002] = 0.5
        d[odd > 0.999] = math.nan
    return lr, r, q, v, d, b, bv


def entry(dev, lr, r, q, v, d, b, bv, n, t, scalars, ret, td):
    ptr = lambda x: x if isinstance(x, int) else x.data_ptr()   # noqa: E731
    return L.load().ktb_retrace_f32(dev, ptr(lr), ptr(r), ptr(q), ptr(v), ptr(d), ptr(b), ptr(bv), n, t, *scalars,
                                    ptr(ret), ptr(td), ops.current_stream_handle(0) if dev == 0 else 0)


def run_entry(dev, lr, r, q, v, d, b, bv, opts):
    """The C entry on offset copies of the inputs into guarded outputs: (ret, td) on the CPU, guards checked."""
    n, t = r.shape
    ins = [placed(x.contiguous(), o) for x, o in zip((lr, r, q, v, d, b, bv), (3, 1, 2, 3, 1, 2, 1))]
    (rbuf, ret), (tbuf, td) = guarded(n * t, 1), guarded(n * t, 3)
    assert entry(dev, *ins, n, t, returns.retrace_scalars(*opts), ret, td) == L.OK, L.last_error()
    torch.cuda.synchronize()
    guards_untouched(rbuf, 1, n * t)
    guards_untouched(tbuf, 3, n * t)
    return ret.view(n, t).cpu(), td.view(n, t).cpu()


# ---- the kernel against the header and the body -----------------------------------------------------------------------
NS = [0, 1, 31, 32, 33, 1000, 4097]
TS = [1, 2, 3, 31, 32, 33, 127, 128, 129, 2048]


@pytest.mark.parametrize("t", TS)
@pytest.mark.parametrize("n", NS)
def test_kernel_equals_header_and_body(dev, n, t):
    opts = OPTIONS[(NS.index(n) + TS.index(t)) % len(OPTIONS)]
    args = rollouts(n, t, seed=1000 * n + t)
    got = run_entry(dev, *args, opts)
    cuda = [x.cuda() for x in args]
    for g, h, what in zip(got, header_retrace(*cuda, *opts), ("ret", "td")):
        same(g, h, (n, t, "header " + what))
    if n * t <= 1000 * 129 or (n, t) == (8, 2048):
        for g, w, what in zip(got, retrace(*cuda, *opts), ("ret", "td")):
            same(g, w, (n, t, "torch " + what))


@pytest.mark.parametrize("opts", OPTIONS, ids=[str(o) for o in OPTIONS])
def test_every_option_set_on_special_values(dev, opts):
    lr, r, q, v, d, b, bv = rollouts(97, 129, seed=7)
    s = torch.tensor(SPECIAL)
    lr[:40, 90] = s.repeat(4)[:40]
    r[:40, 100] = s.repeat(4)[:40]
    q[:40, 70] = s.repeat(4)[:40]
    v[:40, 64] = s.repeat(4)[:40]
    b[:40, 110] = s.repeat(4)[:40]
    bv[:40] = s.repeat(4)[:40]
    r[40:80, 128] = -0.0   # with a −0 bootstrap, the last step's r + disc·bootstrap is −0
    bv[40:80] = -0.0
    d[:, 63] = torch.tensor([0.0, 1.0, 0.5, math.nan]).repeat(25)[:97]
    args = (lr, r, q, v, d, b, bv)
    got = run_entry(dev, *args, opts)
    cuda = [x.cuda() for x in args]
    for g, w, h in zip(got, retrace(*cuda, *opts), header_retrace(*cuda, *opts)):
        same(g, w, opts)
        same(g, h, opts)
    assert torch.signbit(got[0][40:80, 128]).all()


def test_baseline_may_alias_q(dev):
    """baseline is q (the TD error against the target network's own Q), and dones is rewards: inputs may alias."""
    lr, r, q, v, d, _, bv = (x.cuda() for x in rollouts(100, 77, seed=8))
    for opts in OPTIONS:
        for args in ((lr, r, q, v, d, q, bv), (lr, r, q, v, r, r, bv)):
            for g, w in zip(returns.retrace(*args, *opts), retrace(*args, *opts)):
                same(g, w, opts)


@pytest.mark.parametrize("t", [1, 2, 3, 31, 32])
def test_on_policy_lambda_one_equals_the_nstep_kernel(dev, t):
    """log_rhos = 0, λ = 1, values = q = baseline: Retrace is the discounted sum to the rollout's end, ktb_nstep_f32 at
    n = 32 ≥ T, bit for bit in both outputs."""
    lr, r, _, v, d, _, bv = (x.cuda() for x in rollouts(1000, t, seed=9 + t, special=False))
    got = returns.retrace(torch.zeros_like(lr), r, v, v, d, v, bv, GAMMA, 1.0)
    for g, w in zip(got, returns.nstep(r, v, d, v, bv, 32, GAMMA)):
        same(g, w, t)


def test_lambda_zero_over_epsilon_greedy_q_max_is_the_dqn_target(K):
    """The ε-greedy head (ε = 0, the target network, no mask) over the N·(T + 1) observations of a rollout gives q_max;
    λ = 0 over values = q_max[:, :T] and bootstrap_value = q_max[:, T] is then output="dqn_target"'s y on the next
    observations, bit for bit: both are r + (γ(1 − d))·fp32(Q_target[argmax])."""
    n_env, t, d_out = 48, 40, 18
    w, b = config(61, d_out)
    obs = randn((n_env * (t + 1), 256), 62)
    _, _, q_max = mlp.mlp_forward(obs, *w, biases=b, output="epsilon_greedy", seed=63, epsilon=0.0)
    q_max = q_max.float().view(n_env, t + 1)
    g = torch.Generator().manual_seed(64)
    rewards = torch.randn(n_env, t, generator=g).cuda()
    dones = (torch.rand(n_env, t, generator=g) < 0.1).float().cuda()
    log_rhos = torch.randn(n_env, t, generator=g).cuda()
    values, bootstrap = q_max[:, :t].contiguous(), q_max[:, t].contiguous()
    ret, _ = returns.retrace(log_rhos, rewards, values, values, dones, values, bootstrap, GAMMA, 0.0)
    next_obs = obs.view(n_env, t + 1, 256)[:, 1:].reshape(n_env * t, 256).contiguous()
    y = mlp.mlp_forward(next_obs, *w, biases=b, output="dqn_target", reward=rewards.view(-1), done=dones.view(-1),
                        gamma=GAMMA)
    y = y[0] if isinstance(y, (tuple, list)) else y
    same(ret.view(-1), y)


def test_watkins_q_lambda_over_epsilon_greedy_behaviour(K):
    """ε-greedy behaviour (ε = 0.3) on perturbed online weights; the greedy target policy on the target weights.
    log_rhos is 0 where the taken action is the target's greedy one and −inf elsewhere, values and bootstrap_value are
    the target's q_max, q = values (q only meets a trace that is 0 off the greedy action), and baseline is the
    behaviour's Q_online(s_t, a_t): the kernel equals the body on the GPU."""
    n_env, t, d_out = 64, 40, 18
    w, b = config(71, d_out)
    w_o = tuple((x.float() + randn(x.shape, 80 + i, 0.004).float()).bfloat16() for i, x in enumerate(w))
    obs = randn((n_env * (t + 1), 256), 72)
    taken, q_online, _ = mlp.mlp_forward(obs, *w_o, biases=b, output="epsilon_greedy", seed=73, epsilon=0.3)
    greedy, _, q_max = mlp.mlp_forward(obs, *w, biases=b, output="epsilon_greedy", seed=74, epsilon=0.0)
    on = (taken == greedy).view(n_env, t + 1)[:, :t]
    assert on.any() and not on.all()
    log_rhos = torch.where(on, 0.0, -math.inf).float().contiguous()
    q_max = q_max.float().view(n_env, t + 1)
    values, bootstrap = q_max[:, :t].contiguous(), q_max[:, t].contiguous()
    baseline = q_online.float().view(n_env, t + 1)[:, :t].contiguous()
    g = torch.Generator().manual_seed(75)
    rewards = torch.randn(n_env, t, generator=g).cuda()
    dones = (torch.rand(n_env, t, generator=g) < 0.05).float().cuda()
    args = (log_rhos, rewards, values, values, dones, baseline, bootstrap)
    for got, want in zip(returns.retrace(*args, GAMMA, LAM), retrace(*args, GAMMA, LAM)):
        same(got, want)


def test_wrapper_takes_given_outputs_and_a_stream(dev):
    args = [x.cuda() for x in rollouts(100, 77, seed=10)]
    want = header_retrace(*args, GAMMA, LAM)
    got = returns.retrace(*args, GAMMA, LAM)
    ret, td = torch.empty_like(args[0]), torch.empty_like(args[0])
    out = returns.retrace(*args, GAMMA, LAM, ret=ret, td=td, stream=torch.cuda.Stream())
    torch.cuda.synchronize()
    assert out[0] is ret and out[1] is td
    for g, o, h in zip(got, out, want):
        same(g, h)
        same(o, h)


@pytest.mark.parametrize("case,match", [
    ("dtype", "values must be float32"),
    ("shape", "dones must have shape"),
    ("log_rhos", "log_rhos must have shape"),
    ("q", "q must have shape"),
    ("baseline", "baseline must have shape"),
    ("bootstrap", "bootstrap_value must have shape"),
    ("host", "q must be a CUDA tensor"),
    ("strided", "rewards must be contiguous"),
    ("dim", "rewards must be a 2-D"),
    ("out", "td must have shape"),
    ("gamma", "gamma must be a finite number"),
    ("lam", "lam=1e\\+39 must be finite in float32"),
])
def test_wrapper_refuses_bad_arguments(dev, case, match):
    lr, r, q, v, d, b, bv = (x.cuda() for x in rollouts(10, 6, seed=11))
    kw = {}
    gamma, lam = GAMMA, LAM
    if case == "dtype":
        v = v.double()
    elif case == "shape":
        d = d[:, :5]
    elif case == "log_rhos":
        lr = lr[:9]
    elif case == "q":
        q = q[:, :5]
    elif case == "baseline":
        b = b[:9]
    elif case == "bootstrap":
        bv = bv[:9]
    elif case == "host":
        q = q.cpu()
    elif case == "strided":
        r = torch.empty(6, 10, device="cuda:0").t()
    elif case == "dim":
        r = r[0]
    elif case == "out":
        kw["td"] = torch.empty(10, 5, device="cuda:0")
    elif case == "gamma":
        gamma = math.nan
    elif case == "lam":
        lam = 1e39
    with pytest.raises(ValueError, match=match):
        returns.retrace(lr, r, q, v, d, b, bv, gamma, lam, **kw)


def test_statuses_follow_the_header_order(dev):
    x = torch.zeros(64, device="cuda:0")
    nan, inf = math.nan, math.inf
    # an unregistered device comes first, before gamma and lam
    assert entry(15, 0, 0, 0, 0, 0, 0, 0, 4, 4, (nan, 0.9), 0, 0) == L.ERR_STATE
    # a non-finite gamma or lam, before the empty-input check
    for bad in [(nan, 0.9), (0.99, inf), (-inf, 0.9), (0.99, nan)]:
        assert entry(dev, 0, 0, 0, 0, 0, 0, 0, 0, 4, bad, 0, 0) == L.ERR_ARG, bad
    # N·T == 0: nothing to do, NULL pointers allowed
    assert entry(dev, 0, 0, 0, 0, 0, 0, 0, 0, 4, (0.99, 0.95), 0, 0) == L.OK
    assert entry(dev, 0, 0, 0, 0, 0, 0, 0, 4, 0, (0.99, 0.95), 0, 0) == L.OK
    p = x.data_ptr()
    # 2 x 2 rows of 4 bytes each, bootstrap 8 bytes
    ok = dict(lr=p, r=p + 16, q=p + 32, v=p + 48, d=p + 64, b=p + 80, bv=p + 96, ret=p + 112, td=p + 128)

    def call(**over):
        a = dict(ok, **over)
        return entry(dev, a["lr"], a["r"], a["q"], a["v"], a["d"], a["b"], a["bv"], 2, 2, (0.99, 0.95), a["ret"],
                     a["td"])

    assert call() == L.OK
    for name in ok:
        assert call(**{name: 0}) == L.ERR_ARG, name
        assert call(**{name: ok[name] + 2}) == L.ERR_ARG, name
    assert call(ret=p + 88) == L.ERR_ARG            # ret overlaps baseline and bootstrap
    assert call(td=p + 100) == L.ERR_ARG            # td overlaps bootstrap (8 bytes)
    assert call(ret=p + 144, td=p + 152) == L.ERR_ARG
    assert call(ret=p + 104, td=p + 144) == L.OK    # ret right after bootstrap
    assert call(b=p + 32) == L.OK                   # baseline is q: inputs may alias
    torch.cuda.synchronize()


# ---- kt.mapped("retrace") through the public API ------------------------------------------------------------------------
def oracle_on_gpu(body, args, n, *more):
    """The body rank by rank on the GPU, where its exp is the kernel's expf (torch's CPU exp is not)."""
    out = []
    for k in range(n):
        with mock.patch.dict(os.environ, {"RANK": str(k), "WORLD_SIZE": str(n)}):
            out.append(body(*(a.cuda() for a in args), *more))
    return out


@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["1_rank", "3_ranks"])
def test_mapped_equals_oracle_and_wrapper(dev, devices):
    ranks = len(devices)
    args = rollouts(1003, 200, seed=12)
    want = oracle_on_gpu(mapped_retrace, args, ranks)
    mine = returns.retrace(*(a.cuda() for a in args), GAMMA, LAM)
    fn = mapped_copy(mapped_retrace, "retrace", gamma=GAMMA, lam=LAM)
    with deployed(fn, f"t-retrace-{ranks}", devices) as remote:
        got = parts(remote(*(a.cuda() for a in args), serialization="pickle"))
    assert len(got) == len(want) == ranks
    for k, (g, w) in enumerate(zip(got, want)):
        lo, hi = ops.shard_bounds(1003, ranks, k)
        for i in range(2):
            same(g[i], w[i], (k, i))
            same(g[i], mine[i][lo:hi], (k, i))


def test_mapped_with_a_workers_subset(dev):
    """Three workers of one rank each on cuda:0; workers=[0, 2] computes ranks 0 and 2 only, workers=[1] rank 1."""
    args = rollouts(50, 33, seed=13)
    want = oracle_on_gpu(mapped_retrace, args, 3)
    fn = mapped_copy(mapped_retrace, "retrace", gamma=GAMMA, lam=LAM)
    with deployed(fn, "t-retrace-workers", [0, 0, 0], workers=3, num_proc=1) as remote:
        gpu = [a.cuda() for a in args]
        two = parts(remote(*gpu, serialization="pickle", workers=[0, 2]))
        one = parts(remote(*gpu, serialization="pickle", workers=[1]))
    assert len(two) == 2 and len(one) == 1
    for g, k in zip(two + one, (0, 2, 1)):
        same(g[0], want[k][0], k)
        same(g[1], want[k][1], k)


def test_mapped_with_gamma_and_lam_as_call_arguments(dev):
    args = rollouts(77, 40, seed=14)
    fn = mapped_copy(mapped_retrace_args, "retrace", gamma="gamma", lam="lam")
    with deployed(fn, "t-retrace-args", [0, 0]) as remote:
        for gamma, lam in OPTIONS:
            want = oracle_on_gpu(mapped_retrace_args, args, 2, gamma, lam)
            got = parts(remote(*(a.cuda() for a in args), gamma, lam, serialization="pickle"))
            for g, w in zip(got, want):
                same(g[0], w[0], (gamma, lam))
                same(g[1], w[1], (gamma, lam))
        with pytest.raises(Exception, match="lam must be a finite number"):
            remote(*(a.cuda() for a in args), 0.99, math.nan, serialization="pickle")


def test_mapped_refuses_host_tensors(dev):
    args = rollouts(8, 4, seed=15)
    fn = mapped_copy(mapped_retrace, "retrace", gamma=GAMMA, lam=LAM)
    with deployed(fn, "t-retrace-host", [0]) as remote:
        with pytest.raises(Exception, match="'retrace' op takes CUDA tensors on the root GPU"):
            remote(*args, serialization="pickle")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_mapped_on_two_gpus(dev):
    args = rollouts(4097, 129, seed=16)
    want = oracle_on_gpu(mapped_retrace, args, 2)
    fn = mapped_copy(mapped_retrace, "retrace", gamma=GAMMA, lam=LAM)
    with deployed(fn, "t-retrace-2gpu", [0, 1]) as remote:
        got = parts(remote(*(a.cuda() for a in args), serialization="pickle"))
    for g, w in zip(got, want):
        same(g[0], w[0])
        same(g[1], w[1])


# ---- the deployment's self-check ----------------------------------------------------------------------------------------
WRONG = [mapped_retrace_shifted, mapped_retrace_other_gamma, mapped_retrace_other_lam, mapped_retrace_unclipped,
         mapped_retrace_current_value]


@pytest.mark.parametrize("body", WRONG, ids=["shifted_done", "other_gamma", "other_lam", "unclipped", "current_value"])
def test_self_check_refuses_a_body_the_op_does_not_compute(dev, body):
    fn = mapped_copy(body, "retrace", gamma=GAMMA, lam=LAM)
    with pytest.raises(ValueError, match="self-check failed.*lam \\* min\\(1, exp\\(log_rhos\\)\\).*values\\[:, t \\+ "
                                         "1\\].*done flag of transition t"):
        with deployed(fn, f"t-retrace-wrong-{body.__name__}", [0, 0]):
            pass
    # self_check=False deploys it anyway: the op computes the declared γ and λ with transition-t dones
    fn = mapped_copy(body, "retrace", gamma=GAMMA, lam=LAM, self_check=False)
    args = [a.cuda() for a in rollouts(9, 9, seed=17)]
    with deployed(fn, f"t-retrace-unchecked-{body.__name__}", [0, 0]) as remote:
        got = parts(remote(*args, serialization="pickle"))
    for i in range(2):
        same(torch.cat([g[i] for g in got]), retrace(*args, GAMMA, LAM)[i])


def test_self_check_accepts_the_body(dev):
    fn = mapped_copy(mapped_retrace, "retrace", gamma=GAMMA, lam=LAM)
    with deployed(fn, "t-retrace-right", [0, 0, 0]) as remote:
        assert len(remote(*(a.cuda() for a in rollouts(5, 3, seed=18)), serialization="pickle")) == 3
