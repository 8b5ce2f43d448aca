"""ktb_gae_f32 on the H100 against the header's restatement and the body of tests/policy_gae_cases.py run with torch on
the same GPU, bit for bit (NaN against NaN): every row count around the warp's 32 rows, every step count around the
32-step tile, random episode boundaries, special values, every (γ, λ) pair, inputs and outputs at 4-byte offsets that
are not 16-byte aligned, and guard bands that must stay untouched.  Then the entry's statuses in the header's order,
the wrapper's checks, kt.mapped("gae") through the public API and the deployment's self-check."""
import contextlib
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import kubetorch_b200 as kt
from conftest import mapped_copy
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import ops, returns
from oracle import ref_dispatch
from policy_gae_cases import (GAMMA, LAM, gae, header_gae, mapped_gae, mapped_gae_args, mapped_gae_other_gamma,
                              mapped_gae_shifted)

pytestmark = pytest.mark.gpu

PAIRS = [(0.99, 0.95), (0.0, 0.95), (1.0, 1.0), (0.99, 0.0), (0.997, 0.93)]
SPECIAL = [0.0, -0.0, 1.0, -1.5, 1e30, -1e30, 1e-40, math.inf, -math.inf, math.nan]
GUARD = 67                      # guard words on each side of every output
SENTINEL = 0x7FA5A5A5           # a NaN payload no computation produces


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
    """Seeded env-major (rewards, values, dones, last_values) on the CPU: random episode boundaries (done = 1), a few
    done = 0.5 and NaN, and with `special` the special values sprinkled over rewards, values and last_values."""
    g = torch.Generator().manual_seed(seed)
    r, v = torch.randn(n, t, generator=g) * 2, torch.randn(n, t, generator=g) * 5
    lv = torch.randn(n, generator=g) * 5
    d = (torch.rand(n, t, generator=g) < 0.05).float()
    if special:
        s = torch.tensor(SPECIAL)
        for x in (r, v, lv):
            hit = torch.rand(x.shape, generator=g) < 0.01
            x[hit] = s[torch.randint(0, len(SPECIAL), (int(hit.sum()),), generator=g)]
        odd = torch.rand(n, t, generator=g)
        d[odd < 0.002] = 0.5
        d[odd > 0.999] = math.nan
    return r, v, d, lv


def placed(x, offset):
    """x copied into a fresh fp32 CUDA buffer at `offset` words past its (256-byte aligned) start: the view's address
    is 4-byte but not 16-byte aligned for offsets 1-3."""
    buf = torch.empty(x.numel() + offset + 1, dtype=torch.float32, device="cuda:0")
    view = buf[offset:offset + x.numel()].view(x.shape)
    view.copy_(x)
    return view


def guarded(n, offset):
    """An output of n words at `offset` words past GUARD sentinel words, GUARD more after it: (buffer, view)."""
    buf = torch.full((GUARD + offset + n + GUARD,), SENTINEL, dtype=torch.int32, device="cuda:0").view(torch.float32)
    return buf, buf[GUARD + offset:GUARD + offset + n]


def guards_untouched(buf, offset, n):
    bits = buf.view(torch.int32).cpu()
    assert (bits[:GUARD + offset] == SENTINEL).all() and (bits[GUARD + offset + n:] == SENTINEL).all()


def entry(dev, r, v, d, lv, n, t, g, gl, adv, ret):
    ptr = lambda x: x if isinstance(x, int) else x.data_ptr()   # noqa: E731
    return L.load().ktb_gae_f32(dev, ptr(r), ptr(v), ptr(d), ptr(lv), n, t, g, gl, ptr(adv), ptr(ret),
                                ops.current_stream_handle(0) if dev == 0 else 0)


def run_entry(dev, r, v, d, lv, gamma, lam):
    """The C entry on offset copies of the inputs into guarded outputs: (adv, ret) on the CPU, guards checked."""
    n, t = r.shape
    g, gl = returns.gae_scalars(gamma, lam)
    ins = [placed(x.contiguous(), o) for x, o in zip((r, v, d, lv), (1, 2, 3, 1))]
    (abuf, adv), (rbuf, ret) = guarded(n * t, 1), guarded(n * t, 3)
    assert entry(dev, *ins, n, t, g, gl, adv, ret) == L.OK, L.last_error()
    torch.cuda.synchronize()
    guards_untouched(abuf, 1, n * t)
    guards_untouched(rbuf, 3, n * t)
    return adv.view(n, t).cpu(), ret.view(n, t).cpu()


# ---- the kernel against the header and the body -----------------------------------------------------------------------
NS = [0, 1, 31, 32, 33, 1000, 4097]
TS = [1, 2, 3, 31, 32, 33, 127, 128, 129, 2048]


@pytest.mark.parametrize("t", TS)
@pytest.mark.parametrize("n", NS)
def test_kernel_equals_header_and_body(dev, n, t):
    gamma, lam = PAIRS[(NS.index(n) + TS.index(t)) % len(PAIRS)]
    r, v, d, lv = rollouts(n, t, seed=1000 * n + t)
    adv, ret = run_entry(dev, r, v, d, lv, gamma, lam)
    hadv, hret = header_gae(r, v, d, lv, gamma, lam)
    same(adv, hadv, (n, t, "header adv"))
    same(ret, hret, (n, t, "header ret"))
    if n * t <= 1000 * 129 or (n, t) == (8, 2048):
        badv, bret = gae(*(x.cuda() for x in (r, v, d, lv)), gamma, lam)
        same(adv, badv, (n, t, "torch adv"))
        same(ret, bret, (n, t, "torch ret"))


@pytest.mark.parametrize("gamma,lam", PAIRS)
def test_every_pair_on_special_values(dev, gamma, lam):
    r, v, d, lv = rollouts(97, 129, seed=7)
    s = torch.tensor(SPECIAL)
    r[:40, 100] = s.repeat(4)[:40]
    v[:40, 64] = s.repeat(4)[:40]
    lv[:40] = s.repeat(4)[:40]
    d[:, 63] = torch.tensor([0.0, 1.0, 0.5, math.nan]).repeat(25)[:97]
    adv, ret = run_entry(dev, r, v, d, lv, gamma, lam)
    badv, bret = gae(*(x.cuda() for x in (r, v, d, lv)), gamma, lam)
    same(adv, badv, "adv")
    same(ret, bret, "ret")
    same(adv, header_gae(r, v, d, lv, gamma, lam)[0], "header")


def test_wrapper_equals_entry_and_takes_given_outputs(dev):
    r, v, d, lv = (x.cuda() for x in rollouts(100, 77, seed=9))
    adv, ret = returns.gae(r, v, d, lv, GAMMA, LAM)
    hadv, hret = header_gae(*(x.cpu() for x in (r, v, d, lv)), GAMMA, LAM)
    same(adv, hadv)
    same(ret, hret)
    a2, r2 = torch.empty_like(r), torch.empty_like(r)
    out = returns.gae(r, v, d, lv, GAMMA, LAM, adv=a2, ret=r2, stream=torch.cuda.Stream())
    torch.cuda.synchronize()
    assert out[0] is a2 and out[1] is r2
    same(a2, hadv)
    same(r2, hret)


@pytest.mark.parametrize("case,match", [
    ("dtype", "values must be float32"),
    ("shape", "dones must have shape"),
    ("last", "last_values must have shape"),
    ("host", "values must be a CUDA tensor"),
    ("strided", "rewards must be contiguous"),
    ("dim", "rewards must be a 2-D"),
    ("out", "adv must have shape"),
    ("gamma", "gamma must be a finite number"),
])
def test_wrapper_refuses_bad_arguments(dev, case, match):
    r, v, d, lv = (x.cuda() for x in rollouts(10, 6, seed=10))
    kw = {}
    if case == "dtype":
        v = v.double()
    elif case == "shape":
        d = d[:, :5]
    elif case == "last":
        lv = lv[:9]
    elif case == "host":
        v = v.cpu()
    elif case == "strided":
        r = torch.empty(6, 10, device="cuda:0").t()
    elif case == "dim":
        r = r[0]
    elif case == "out":
        kw["adv"] = torch.empty(10, 5, device="cuda:0")
    with pytest.raises(ValueError, match=match):
        returns.gae(r, v, d, lv, math.nan if case == "gamma" else GAMMA, LAM, **kw)


def test_statuses_follow_the_header_order(dev):
    x = torch.zeros(64, device="cuda:0")
    nan, inf = math.nan, math.inf
    # an unregistered device comes first, before gamma
    assert entry(15, 0, 0, 0, 0, 4, 4, nan, 0.5, 0, 0) == L.ERR_STATE
    # a non-finite gamma or gamma_lam, before the empty-input check
    assert entry(dev, 0, 0, 0, 0, 0, 4, nan, 0.5, 0, 0) == L.ERR_ARG
    assert entry(dev, 0, 0, 0, 0, 0, 4, 0.5, inf, 0, 0) == L.ERR_ARG
    # N·T == 0: nothing to do, NULL pointers allowed
    assert entry(dev, 0, 0, 0, 0, 0, 4, 0.99, 0.9, 0, 0) == L.OK
    assert entry(dev, 0, 0, 0, 0, 4, 0, 0.99, 0.9, 0, 0) == L.OK
    p = x.data_ptr()
    ok = dict(r=p, v=p + 16, d=p + 32, lv=p + 48, adv=p + 64, ret=p + 80)   # 2 x 2 rows of 4 bytes each

    def call(**over):
        a = dict(ok, **over)
        return entry(dev, a["r"], a["v"], a["d"], a["lv"], 2, 2, 0.99, 0.9, a["adv"], a["ret"])

    assert call() == L.OK
    for name in ok:
        assert call(**{name: 0}) == L.ERR_ARG, name
        assert call(**{name: ok[name] + 2}) == L.ERR_ARG, name
    assert call(adv=p + 40) == L.ERR_ARG            # adv overlaps dones and last_values
    assert call(ret=p + 52) == L.ERR_ARG            # ret overlaps last_values (8 bytes) and adv
    assert call(adv=p + 96, ret=p + 104) == L.ERR_ARG
    assert call(adv=p + 56, ret=p + 100) == L.OK    # adv right after last_values
    torch.cuda.synchronize()


# ---- kt.mapped("gae") through the public API ----------------------------------------------------------------------------
@contextlib.contextmanager
def deployed(fn, name, devices, **distribute):
    remote = kt.fn(fn, name=name).to(
        kt.Compute(gpus=len(set(devices)), allowed_serialization=["json", "pickle"]).distribute(
            "b200", num_proc=distribute.pop("num_proc", len(devices)), devices=list(devices),
            **dict(dict(workers=1), **distribute)))
    try:
        yield remote
    finally:
        remote.teardown()


def parts(got):
    return [(a.cpu(), b.cpu()) for a, b in got]


@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["1_rank", "3_ranks"])
def test_mapped_equals_oracle_and_wrapper(dev, devices):
    n = len(devices)
    args = rollouts(1003, 200, seed=11)
    want = ref_dispatch.spmd_call(mapped_gae, *args, num_proc=n, serialization="pickle")
    mine = returns.gae(*(a.cuda() for a in args), GAMMA, LAM)
    fn = mapped_copy(mapped_gae, "gae", gamma=GAMMA, lam=LAM)
    with deployed(fn, f"t-gae-{n}", devices) as remote:
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
    want = ref_dispatch.spmd_call(mapped_gae, *args, num_proc=3, serialization="pickle")
    fn = mapped_copy(mapped_gae, "gae", gamma=GAMMA, lam=LAM)
    with deployed(fn, "t-gae-workers", [0, 0, 0], workers=3, num_proc=1) as remote:
        gpu = [a.cuda() for a in args]
        two = parts(remote(*gpu, serialization="pickle", workers=[0, 2]))
        one = parts(remote(*gpu, serialization="pickle", workers=[1]))
    assert len(two) == 2 and len(one) == 1
    for g, k in zip(two + one, (0, 2, 1)):
        same(g[0], want[k][0], k)
        same(g[1], want[k][1], k)


def test_mapped_with_gamma_and_lam_as_call_arguments(dev):
    args = rollouts(77, 40, seed=13)
    fn = mapped_copy(mapped_gae_args, "gae", gamma="gamma", lam="lam")
    with deployed(fn, "t-gae-args", [0, 0]) as remote:
        for gamma, lam in PAIRS:
            want = ref_dispatch.spmd_call(mapped_gae_args, *args, gamma, lam, num_proc=2, serialization="pickle")
            got = parts(remote(*(a.cuda() for a in args), gamma, lam, serialization="pickle"))
            for g, w in zip(got, want):
                same(g[0], w[0], (gamma, lam))
                same(g[1], w[1], (gamma, lam))
        with pytest.raises(Exception, match="gamma must be a finite number"):
            remote(*(a.cuda() for a in args), math.inf, 0.9, serialization="pickle")


def test_mapped_refuses_host_tensors(dev):
    args = rollouts(8, 4, seed=14)
    fn = mapped_copy(mapped_gae, "gae", gamma=GAMMA, lam=LAM)
    with deployed(fn, "t-gae-host", [0]) as remote:
        with pytest.raises(Exception, match="CUDA tensors on the root GPU"):
            remote(*args, serialization="pickle")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_mapped_on_two_gpus(dev):
    args = rollouts(4097, 129, seed=15)
    want = ref_dispatch.spmd_call(mapped_gae, *args, num_proc=2, serialization="pickle")
    fn = mapped_copy(mapped_gae, "gae", gamma=GAMMA, lam=LAM)
    with deployed(fn, "t-gae-2gpu", [0, 1]) as remote:
        got = parts(remote(*(a.cuda() for a in args), serialization="pickle"))
    for g, w in zip(got, want):
        same(g[0], w[0])
        same(g[1], w[1])


# ---- the deployment's self-check ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("body", [mapped_gae_shifted, mapped_gae_other_gamma], ids=["shifted_done", "other_gamma"])
def test_self_check_refuses_a_body_the_op_does_not_compute(dev, body):
    fn = mapped_copy(body, "gae", gamma=GAMMA, lam=LAM)
    with pytest.raises(ValueError, match="self-check failed.*done flag of transition t"):
        with deployed(fn, f"t-gae-wrong-{body.__name__}", [0, 0]):
            pass
    # self_check=False deploys it anyway: the op computes the declared γ and λ with transition-t dones
    fn = mapped_copy(body, "gae", gamma=GAMMA, lam=LAM, self_check=False)
    args = rollouts(9, 9, seed=16)
    with deployed(fn, f"t-gae-unchecked-{body.__name__}", [0, 0]) as remote:
        got = parts(remote(*(a.cuda() for a in args), serialization="pickle"))
    same(torch.cat([g[0] for g in got]), gae(*args, GAMMA, LAM)[0])


def test_self_check_accepts_the_body(dev):
    fn = mapped_copy(mapped_gae, "gae", gamma=GAMMA, lam=LAM)
    with deployed(fn, "t-gae-right", [0, 0, 0]) as remote:
        assert len(remote(*(a.cuda() for a in rollouts(5, 3, seed=17)), serialization="pickle")) == 3
