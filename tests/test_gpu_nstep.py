"""ktb_nstep_f32 on the H100 against the header's restatement and the body of tests/policy_nstep_cases.py run with torch
on the same GPU, bit for bit (NaN against NaN): every row count around the warp's 32 rows, every step count around the
32-step tile and its span, every n at the small and medium shapes, random episode boundaries, special values, inputs
and outputs at 4-byte offsets that are not 16-byte aligned, guard bands that must stay untouched, and aliased inputs.
Then the one-step target over the ε-greedy head's q_max against output="dqn_target"; the entry's statuses in the
header's order, the wrapper's checks, kt.mapped("nstep") through the public API and the deployment's self-check."""
import math

import pytest
import torch

from conftest import mapped_copy
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp, ops, returns
from mlp_rig import K, config, randn  # noqa: F401
from oracle import ref_dispatch
from policy_nstep_cases import (GAMMA, N_STEP, header_nstep, mapped_nstep, mapped_nstep_args, mapped_nstep_other_gamma,
                                mapped_nstep_other_n, mapped_nstep_shifted, mapped_nstep_zero_bootstrap, nstep)
from test_gpu_gae import deployed, guarded, guards_untouched, parts, placed, same

pytestmark = pytest.mark.gpu

SPECIAL = [0.0, -0.0, 1.0, -1.5, 1e30, -1e30, 3e38, 1e-40, -1e-45, math.inf, -math.inf, math.nan]
N_ALL = [1, 2, 3, 5, 31, 32]
GAMMAS = [0.99, 0.9, 0.0, 1.0]


@pytest.fixture(scope="module")
def dev():
    ops.ensure_init([0])
    return 0


def rollouts(n, t, seed, special=True):
    """Seeded env-major (rewards, values, dones, baseline, last_values) on the CPU: random episode boundaries
    (done = 1), and with `special` a few done = 0.5 and NaN and the special values sprinkled over every other input."""
    g = torch.Generator().manual_seed(seed)
    r, v, b = torch.randn(n, t, generator=g) * 2, torch.randn(n, t, generator=g) * 5, torch.randn(n, t, generator=g)
    lv = torch.randn(n, generator=g) * 5
    d = (torch.rand(n, t, generator=g) < 0.05).float()
    if special:
        s = torch.tensor(SPECIAL)
        for x in (r, v, b, lv):
            hit = torch.rand(x.shape, generator=g) < 0.01
            x[hit] = s[torch.randint(0, len(SPECIAL), (int(hit.sum()),), generator=g)]
        odd = torch.rand(n, t, generator=g)
        d[odd < 0.002] = 0.5
        d[odd > 0.999] = math.nan
    return r, v, d, b, lv


def entry(dev, r, v, d, b, lv, N, T, n, gamma, ret, td):
    ptr = lambda x: x if isinstance(x, int) else x.data_ptr()   # noqa: E731
    return L.load().ktb_nstep_f32(dev, ptr(r), ptr(v), ptr(d), ptr(b), ptr(lv), N, T, n, gamma, ptr(ret), ptr(td),
                                  ops.current_stream_handle(0) if dev == 0 else 0)


def run_entry(dev, r, v, d, b, lv, n, gamma):
    """The C entry on offset copies of the inputs into guarded outputs: (ret, td) on the CPU, guards checked."""
    N, T = r.shape
    ins = [placed(x.contiguous(), o) for x, o in zip((r, v, d, b, lv), (1, 2, 3, 1, 3))]
    (rbuf, ret), (tbuf, td) = guarded(N * T, 3), guarded(N * T, 1)
    assert entry(dev, *ins, N, T, *returns.nstep_scalars(n, gamma), ret, td) == L.OK, L.last_error()
    torch.cuda.synchronize()
    guards_untouched(rbuf, 3, N * T)
    guards_untouched(tbuf, 1, N * T)
    return ret.view(N, T).cpu(), td.view(N, T).cpu()


# ---- the kernel against the header and the body -----------------------------------------------------------------------
NS = [0, 1, 31, 32, 33, 1000, 4097]
TS = [1, 2, 3, 31, 32, 33, 63, 64, 65, 127, 128, 129, 2048]


def _steps(N, T):
    """Every n at the small and medium shapes, 1, 5 and 32 at the largest."""
    return [1, 5, 32] if N * T > 1000 * 129 else N_ALL


@pytest.mark.parametrize("t", TS)
@pytest.mark.parametrize("N", NS)
def test_kernel_equals_header_and_body(dev, N, t):
    r, v, d, b, lv = rollouts(N, t, seed=1000 * N + t)
    cuda = [x.cuda() for x in (r, v, d, b, lv)]
    for i, n in enumerate(_steps(N, t)):
        gamma = GAMMAS[(NS.index(N) + TS.index(t) + i) % len(GAMMAS)]
        got = run_entry(dev, r, v, d, b, lv, n, gamma)
        for g, w, what in zip(got, nstep(*cuda, n, gamma), ("ret", "td")):
            same(g, w, (N, t, n, gamma, "torch " + what))
        if N * t <= 1000 * 129 or n == 5:
            for g, h, what in zip(got, header_nstep(r, v, d, b, lv, n, gamma), ("ret", "td")):
                same(g, h, (N, t, n, gamma, "header " + what))


@pytest.mark.parametrize("n", N_ALL)
def test_every_n_on_special_values(dev, n):
    r, v, d, b, lv = rollouts(97, 129, seed=7)
    s = torch.tensor(SPECIAL)
    r[:48, 100] = s.repeat(4)[:48]
    v[:48, 64] = s.repeat(4)[:48]
    v[48:96, 127] = s.repeat(4)[:48]
    b[:48, 90] = s.repeat(4)[:48]
    lv[:48] = s.repeat(4)[:48]
    d[:, 63] = torch.tensor([0.0, 1.0, 0.5, math.nan]).repeat(25)[:97]
    d[:, 128] = torch.tensor([0.0, 1.0, 0.5, math.nan]).repeat(25)[:97]
    got = run_entry(dev, r, v, d, b, lv, n, GAMMA)
    cuda = [x.cuda() for x in (r, v, d, b, lv)]
    for g, w, h in zip(got, nstep(*cuda, n, GAMMA), header_nstep(r, v, d, b, lv, n, GAMMA)):
        same(g, w, n)
        same(g, h, n)


def test_aliased_inputs(dev):
    """baseline is values (A3C's n-step advantages), and dones is rewards: inputs may alias one another."""
    r, v, d, _, lv = (x.cuda() for x in rollouts(100, 77, seed=8))
    for n in (1, 5, 32):
        ret, td = returns.nstep(r, v, d, v, lv, n, GAMMA)
        for g, w in zip((ret, td), nstep(r, v, d, v, lv, n, GAMMA)):
            same(g, w, n)
        ret, td = returns.nstep(r, v, r, r, lv, n, GAMMA)
        for g, w in zip((ret, td), nstep(r, v, r, r, lv, n, GAMMA)):
            same(g, w, n)


def test_one_step_over_epsilon_greedy_q_max_is_the_dqn_target(K):
    """The ε-greedy head (ε = 0, the target network, no mask) over the N·(T + 1) observations of a rollout gives q_max,
    V(s) = max_a Q_target(s, a); n = 1 over values = q_max[:, :T] and last_values = q_max[:, T] is then
    output="dqn_target"'s y on the next observations, bit for bit: both are r + (γ(1 − d))·fp32(Q_target[argmax])."""
    n_env, t, d_out = 48, 40, 18
    w, b = config(51, d_out)
    obs = randn((n_env * (t + 1), 256), 52)
    _, _, q_max = mlp.mlp_forward(obs, *w, biases=b, output="epsilon_greedy", seed=53, epsilon=0.0)
    q_max = q_max.float().view(n_env, t + 1)
    g = torch.Generator().manual_seed(54)
    rewards = torch.randn(n_env, t, generator=g).cuda()
    dones = (torch.rand(n_env, t, generator=g) < 0.1).float().cuda()
    values, last_values = q_max[:, :t].contiguous(), q_max[:, t].contiguous()
    ret, _ = returns.nstep(rewards, values, dones, values, last_values, 1, GAMMA)
    next_obs = obs.view(n_env, t + 1, 256)[:, 1:].reshape(n_env * t, 256).contiguous()
    y = mlp.mlp_forward(next_obs, *w, biases=b, output="dqn_target", reward=rewards.view(-1), done=dones.view(-1),
                        gamma=GAMMA)
    y = y[0] if isinstance(y, (tuple, list)) else y
    same(ret.view(-1), y)


def test_wrapper_takes_given_outputs_and_a_stream(dev):
    args = [x.cuda() for x in rollouts(100, 77, seed=9)]
    want = header_nstep(*args, 7, GAMMA)
    got = returns.nstep(*args, 7, GAMMA)
    ret, td = torch.empty_like(args[0]), torch.empty_like(args[0])
    out = returns.nstep(*args, 7, GAMMA, ret=ret, td=td, stream=torch.cuda.Stream())
    torch.cuda.synchronize()
    assert out[0] is ret and out[1] is td
    for g, o, h in zip(got, out, want):
        same(g, h)
        same(o, h)


@pytest.mark.parametrize("case,match", [
    ("dtype", "values must be float32"),
    ("shape", "dones must have shape"),
    ("baseline", "baseline must have shape"),
    ("last_values", "last_values must have shape"),
    ("host", "values must be a CUDA tensor"),
    ("strided", "rewards must be contiguous"),
    ("dim", "rewards must be a 2-D"),
    ("out", "td must have shape"),
    ("gamma", "gamma must be a finite number"),
    ("n", "n must be an int in \\[1, 32\\]"),
])
def test_wrapper_refuses_bad_arguments(dev, case, match):
    r, v, d, b, lv = (x.cuda() for x in rollouts(10, 6, seed=10))
    kw = {}
    if case == "dtype":
        v = v.double()
    elif case == "shape":
        d = d[:, :5]
    elif case == "baseline":
        b = b[:9]
    elif case == "last_values":
        lv = lv[:9]
    elif case == "host":
        v = v.cpu()
    elif case == "strided":
        r = torch.empty(6, 10, device="cuda:0").t()
    elif case == "dim":
        r = r[0]
    elif case == "out":
        kw["td"] = torch.empty(10, 5, device="cuda:0")
    with pytest.raises(ValueError, match=match):
        returns.nstep(r, v, d, b, lv, 33 if case == "n" else 5, math.nan if case == "gamma" else GAMMA, **kw)


def test_statuses_follow_the_header_order(dev):
    x = torch.zeros(64, device="cuda:0")
    nan = math.nan
    # an unregistered device comes first, before n and gamma
    assert entry(15, 0, 0, 0, 0, 0, 4, 4, 0, nan, 0, 0) == L.ERR_STATE
    # n outside [1, 32] or a non-finite gamma, before the empty-input check
    for n, gamma in [(0, 0.99), (33, 0.99), (-1, 0.99), (5, nan), (5, math.inf)]:
        assert entry(dev, 0, 0, 0, 0, 0, 0, 4, n, gamma, 0, 0) == L.ERR_ARG, (n, gamma)
    # N·T == 0: nothing to do, NULL pointers allowed
    assert entry(dev, 0, 0, 0, 0, 0, 0, 4, 32, 0.99, 0, 0) == L.OK
    assert entry(dev, 0, 0, 0, 0, 0, 4, 0, 1, 0.99, 0, 0) == L.OK
    p = x.data_ptr()
    ok = dict(r=p, v=p + 16, d=p + 32, b=p + 48, lv=p + 64, ret=p + 80, td=p + 96)   # 2 x 2 rows of 4 bytes each

    def call(**over):
        a = dict(ok, **over)
        return entry(dev, a["r"], a["v"], a["d"], a["b"], a["lv"], 2, 2, 3, 0.99, a["ret"], a["td"])

    assert call() == L.OK
    for name in ok:
        assert call(**{name: 0}) == L.ERR_ARG, name
        assert call(**{name: ok[name] + 2}) == L.ERR_ARG, name
    assert call(ret=p + 56) == L.ERR_ARG            # ret overlaps baseline and last_values
    assert call(td=p + 68) == L.ERR_ARG             # td overlaps last_values (8 bytes) and ret
    assert call(ret=p + 112, td=p + 120) == L.ERR_ARG
    assert call(ret=p + 72, td=p + 112) == L.OK     # ret right after last_values
    assert call(b=p + 16) == L.OK                   # baseline is values: inputs may alias
    torch.cuda.synchronize()


# ---- kt.mapped("nstep") through the public API --------------------------------------------------------------------------
@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["1_rank", "3_ranks"])
def test_mapped_equals_oracle_and_wrapper(dev, devices):
    ranks = len(devices)
    args = rollouts(1003, 200, seed=11)
    want = ref_dispatch.spmd_call(mapped_nstep, *args, num_proc=ranks, serialization="pickle")
    mine = returns.nstep(*(a.cuda() for a in args), N_STEP, GAMMA)
    fn = mapped_copy(mapped_nstep, "nstep", n=N_STEP, gamma=GAMMA)
    with deployed(fn, f"t-nstep-{ranks}", devices) as remote:
        got = parts(remote(*(a.cuda() for a in args), serialization="pickle"))
    assert len(got) == len(want) == ranks
    for k, (g, w) in enumerate(zip(got, want)):
        lo, hi = ops.shard_bounds(1003, ranks, k)
        for i in range(2):
            same(g[i], w[i], (k, i))
            same(g[i], mine[i][lo:hi], (k, i))


def test_mapped_with_a_workers_subset(dev):
    """Three workers of one rank each on cuda:0; workers=[0, 2] computes ranks 0 and 2 only, workers=[1] rank 1."""
    args = rollouts(50, 33, seed=12)
    want = ref_dispatch.spmd_call(mapped_nstep, *args, num_proc=3, serialization="pickle")
    fn = mapped_copy(mapped_nstep, "nstep", n=N_STEP, gamma=GAMMA)
    with deployed(fn, "t-nstep-workers", [0, 0, 0], workers=3, num_proc=1) as remote:
        gpu = [a.cuda() for a in args]
        two = parts(remote(*gpu, serialization="pickle", workers=[0, 2]))
        one = parts(remote(*gpu, serialization="pickle", workers=[1]))
    assert len(two) == 2 and len(one) == 1
    for g, k in zip(two + one, (0, 2, 1)):
        same(g[0], want[k][0], k)
        same(g[1], want[k][1], k)


def test_mapped_with_gamma_as_a_call_argument(dev):
    args = rollouts(77, 40, seed=13)
    fn = mapped_copy(mapped_nstep_args, "nstep", n=N_STEP, gamma="gamma")
    with deployed(fn, "t-nstep-args", [0, 0]) as remote:
        for gamma in GAMMAS:
            want = ref_dispatch.spmd_call(mapped_nstep_args, *args, gamma, num_proc=2, serialization="pickle")
            got = parts(remote(*(a.cuda() for a in args), gamma, serialization="pickle"))
            for g, w in zip(got, want):
                same(g[0], w[0], gamma)
                same(g[1], w[1], gamma)
        with pytest.raises(Exception, match="gamma must be a finite number"):
            remote(*(a.cuda() for a in args), math.inf, serialization="pickle")


def test_mapped_refuses_host_tensors(dev):
    args = rollouts(8, 4, seed=14)
    fn = mapped_copy(mapped_nstep, "nstep", n=N_STEP, gamma=GAMMA)
    with deployed(fn, "t-nstep-host", [0]) as remote:
        with pytest.raises(Exception, match="'nstep' op takes CUDA tensors on the root GPU"):
            remote(*args, serialization="pickle")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_mapped_on_two_gpus(dev):
    args = rollouts(4097, 129, seed=15)
    want = ref_dispatch.spmd_call(mapped_nstep, *args, num_proc=2, serialization="pickle")
    fn = mapped_copy(mapped_nstep, "nstep", n=N_STEP, gamma=GAMMA)
    with deployed(fn, "t-nstep-2gpu", [0, 1]) as remote:
        got = parts(remote(*(a.cuda() for a in args), serialization="pickle"))
    for g, w in zip(got, want):
        same(g[0], w[0])
        same(g[1], w[1])


# ---- the deployment's self-check ----------------------------------------------------------------------------------------
WRONG = [mapped_nstep_shifted, mapped_nstep_other_gamma, mapped_nstep_other_n, mapped_nstep_zero_bootstrap]


@pytest.mark.parametrize("body", WRONG, ids=["shifted_done", "other_gamma", "other_n", "zero_bootstrap"])
def test_self_check_refuses_a_body_the_op_does_not_compute(dev, body):
    fn = mapped_copy(body, "nstep", n=N_STEP, gamma=GAMMA)
    with pytest.raises(ValueError, match="self-check failed.*n=5 discounted rewards with gamma=0.99.*done flag of "
                                         "transition t.*bootstraps from last_values"):
        with deployed(fn, f"t-nstep-wrong-{body.__name__}", [0, 0]):
            pass
    # self_check=False deploys it anyway: the op computes the declared n and γ with transition-t dones
    fn = mapped_copy(body, "nstep", n=N_STEP, gamma=GAMMA, self_check=False)
    args = rollouts(9, 9, seed=16)
    with deployed(fn, f"t-nstep-unchecked-{body.__name__}", [0, 0]) as remote:
        got = parts(remote(*(a.cuda() for a in args), serialization="pickle"))
    for i in range(2):
        same(torch.cat([g[i] for g in got]), nstep(*args, N_STEP, GAMMA)[i])


def test_self_check_accepts_the_body(dev):
    fn = mapped_copy(mapped_nstep, "nstep", n=N_STEP, gamma=GAMMA)
    with deployed(fn, "t-nstep-right", [0, 0, 0]) as remote:
        assert len(remote(*(a.cuda() for a in rollouts(5, 3, seed=17)), serialization="pickle")) == 3
