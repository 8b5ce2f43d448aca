"""ktb_per_sample_f32 and ktb_per_update_f32 on the H100 against the bodies of tests/policy_per_cases.py run with torch on
the same GPU, and against the header's restatement, bit for bit (NaN against NaN): the tree, the indices and the
weights over capacities around powers of two up to 2^21 + 1, batches of 1 to 8192, every usual β (each of torch's pow
paths among them), special values, a total that overflows, priorities at 4-byte offsets that are not 16-byte aligned,
guard bands around every output, and splits of the strata into calls.  Then the update's last-occurrence rule; the
entries' statuses in the header's order; the wrappers' checks; kt.mapped("per") through the public API; and the
deployment's self-check."""
import math
import os
from unittest import mock

import numpy as np
import pytest
import torch

from conftest import mapped_copy
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import ops, replay
from policy_per_cases import (BATCH, BETA, header_per_sample, mapped_per, mapped_per_beta, mapped_per_local,
                              mapped_per_other_stream, mapped_per_seeded, mapped_per_strict, mapped_per_uniform,
                              mapped_per_unnormalised, per_sample, per_update, sum_tree)
from test_gpu_gae import GUARD, deployed, guarded, guards_untouched, placed, same

pytestmark = pytest.mark.gpu

BETAS = [0.0, 0.4, 0.5, 1.0, 2.0]
SPECIAL = [0.0, 1e-45, 1e-40, 3e38, math.inf, math.nan, 1.0, 0.25]
LONG_SENTINEL = -0x5A5A5A5A5A5A5A5B


@pytest.fixture(scope="module")
def dev():
    ops.ensure_init([0])
    return 0


def priorities(c, seed, zeros=0.3):
    g = torch.Generator().manual_seed(seed)
    p = torch.rand(c, generator=g) * 2
    p[torch.rand(c, generator=g) < zeros] = 0.0
    p[int(torch.randint(0, c, (1,), generator=g))] = 1.0 + c / 8   # one dominant item
    return p


def body_tree(p):
    """The body's levels on the GPU in the header's layout (min, total, internal nodes), on the CPU."""
    levels = sum_tree(p)
    n = levels[0].numel()
    out = torch.zeros(max(n, 2), device=p.device)
    for lv in levels[1:]:
        out[lv.numel():2 * lv.numel()] = lv
    out[1] = levels[-1][0]
    out[0] = p.min()
    return out.cpu()


def guarded_long(n):
    buf = torch.full((GUARD + n + GUARD,), LONG_SENTINEL, dtype=torch.int64, device="cuda:0")
    return buf, buf[GUARD:GUARD + n]


def run_sample(dev, p, seed, batch, beta, j0=0, rows=None, offset=1):
    """The C entry on an offset copy of p into guarded outputs: (tree, indices, weights) on the CPU, guards checked."""
    rows = batch - j0 if rows is None else rows
    c = p.numel()
    prio = placed(p, offset)
    tn = replay.tree_size(c)
    (tbuf, tree), (wbuf, w) = guarded(tn, 3), guarded(rows, 2)
    ibuf, idx = guarded_long(rows)
    rc = L.load().ktb_per_sample_f32(dev, prio.data_ptr(), c, batch, j0, rows, seed, replay.per_scalars(beta=beta)[0],
                                     tree.data_ptr(), idx.data_ptr(), w.data_ptr(), ops.current_stream_handle(0))
    assert rc == L.OK, L.last_error()
    torch.cuda.synchronize()
    guards_untouched(tbuf, 3, tn)
    guards_untouched(wbuf, 2, rows)
    bits = ibuf.cpu()
    assert (bits[:GUARD] == LONG_SENTINEL).all() and (bits[GUARD + rows:] == LONG_SENTINEL).all()
    return tree.cpu(), idx.cpu(), w.cpu()


def check_against_body(dev, p, seed, batch, beta, j0=0, rows=None, header=True):
    tree, idx, w = run_sample(dev, p, seed, batch, beta, j0, rows)
    pc = p.cuda()
    want_idx, want_w = per_sample(pc, seed, batch, beta, j0, rows)
    same(tree, body_tree(pc), (p.numel(), batch, beta, "tree"))
    assert torch.equal(idx, want_idx.cpu()), (p.numel(), batch, beta)
    same(w, want_w, (p.numel(), batch, beta, "weights"))
    if header:
        h_tree, h_idx, h_w = header_per_sample(pc, seed, batch, beta, j0, rows)
        same(tree, h_tree, "header tree")
        assert np.array_equal(idx.numpy(), h_idx)
        same(w, h_w, "header weights")
    return tree, idx, w


# ---- the kernel against the body and the header -----------------------------------------------------------------------
CS = [1, 2, 3, 31, 32, 33, 1000, 2047, 2048, 2049, 4097, 65536, (1 << 20) + 3, (1 << 21) + 1]
BATCHES = [1, 7, 512, 8192]


@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("c", CS)
def test_kernel_equals_body_and_header(dev, c, batch):
    beta = BETAS[(CS.index(c) + BATCHES.index(batch)) % len(BETAS)]
    p = priorities(c, seed=c + batch)
    _, idx, _ = check_against_body(dev, p, 1000 * c + batch, batch, beta, header=c <= 65536)
    assert (p[idx] > 0).all() and (idx[1:] >= idx[:-1]).all()


@pytest.mark.parametrize("beta", BETAS)
def test_every_beta_with_zero_free_priorities(dev, beta):
    """No zero priority, so the weights are finite and each of torch's pow paths (fill, powf, rsqrt, reciprocal and
    1 / (x·x)) is what decides their bits."""
    for c in (33, 4097, 100000):
        p = torch.rand(c, generator=torch.Generator().manual_seed(c)) + 0.01
        _, _, w = check_against_body(dev, p, c, 512, beta)
        assert (w > 0).all() and (w <= 1.0 + 1e-6).all()


def test_special_values(dev):
    s = torch.tensor(SPECIAL)
    for c in (8, 33, 1000, 5000):
        p = s.repeat(c // 8 + 1)[:c][torch.randperm(c, generator=torch.Generator().manual_seed(c))].contiguous()
        for beta in BETAS:
            _, idx, _ = check_against_body(dev, p, c, 512, beta)
            assert ((idx >= 0) & (idx < c)).all()


def test_subnormal_priorities_and_a_total_that_overflows(dev):
    for c in (1000, 4097):
        p = priorities(c, seed=c)
        tiny = torch.where(p > 0, torch.tensor(1e-45), torch.tensor(0.0))   # masses equal partial sums
        huge = torch.where(p > 0, torch.tensor(3e38), torch.tensor(0.0))    # the total overflows to inf
        sub = p * 1e-39                                                     # subnormal priorities
        for q in (tiny, huge, sub):
            for beta in (0.4, 1.0):
                _, idx, _ = check_against_body(dev, q, 5, 512, beta)
                assert ((idx >= 0) & (idx < c)).all()


def test_negative_zero_priorities_stay_in_bounds(dev):
    """torch.min's choice between −0 and +0 is its own, so only memory safety and the range are checked here."""
    p = priorities(1000, seed=3)
    p[p == 0] = -0.0
    tree, idx, _ = run_sample(dev, p, 4, 512, 0.4)
    assert ((idx >= 0) & (idx < 1000)).all() and (p[idx] > 0).all()


@pytest.mark.parametrize("offset", [0, 1, 2, 3])
def test_priorities_at_every_alignment(dev, offset):
    p = priorities(5001, seed=offset)
    want = run_sample(dev, p, 9, 512, 0.4, offset=0)
    got = run_sample(dev, p, 9, 512, 0.4, offset=offset)
    for g, w in zip(got, want):
        assert torch.equal(g.view(torch.int32) if g.dtype == torch.float32 else g,
                           w.view(torch.int32) if w.dtype == torch.float32 else w)


def test_splits_of_the_strata_equal_the_whole(dev):
    p = priorities(70001, seed=11)
    _, idx, w = check_against_body(dev, p, 12, 8192, 0.4, header=False)
    for cuts in ([0, 4096, 8192], [0, 1, 2, 8191, 8192], [0, 2731, 5462, 8192], [0, 100, 101, 8192]):
        for a, b in zip(cuts, cuts[1:]):
            _, i2, w2 = check_against_body(dev, p, 12, 8192, 0.4, a, b - a, header=False)
            assert torch.equal(i2, idx[a:b])
            same(w2, w[a:b])


def test_wrapper_takes_given_outputs_and_a_stream(dev):
    p = priorities(3000, seed=13).cuda()
    idx, w = replay.per_sample(p, 512, 14, BETA)
    tree = torch.empty(replay.tree_size(3000), device="cuda:0")
    i2, w2 = torch.empty(100, dtype=torch.int64, device="cuda:0"), torch.empty(100, device="cuda:0")
    out = replay.per_sample(p, 512, 14, BETA, j0=200, rows=100, tree=tree, indices=i2, weights=w2,
                            stream=torch.cuda.Stream())
    torch.cuda.synchronize()
    assert out[0] is i2 and out[1] is w2
    assert torch.equal(i2, idx[200:300])
    same(w2, w[200:300])
    same(tree, body_tree(p))


# ---- the update -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alpha", [0.5, 0.6, 1.0, 2.0])
def test_update_equals_the_body(dev, alpha):
    g = torch.Generator().manual_seed(int(alpha * 10))
    c = 100003
    cases = [torch.full((512,), 77), torch.randint(0, 300, (8192,), generator=g), torch.randint(0, c, (8192,),
             generator=g), torch.randperm(c, generator=g)[:4096], torch.tensor([5]), torch.randint(0, 9, (7,),
             generator=g)]
    for indices in cases:
        td = torch.randn(len(indices), generator=g) * 3
        td[::97] = torch.tensor([0.0, -0.0, math.inf, math.nan, 1e-40])[torch.arange(len(td[::97])) % 5]
        p = torch.rand(c, generator=g).cuda()
        want = p.clone()
        per_update(want, indices.cuda(), td.cuda(), alpha, 1e-6)
        got = replay.per_update(p, indices.cuda(), td.cuda(), alpha, 1e-6)
        torch.cuda.synchronize()
        assert got is p
        same(p, want, (alpha, len(indices)))


def test_update_skips_indices_out_of_range(dev):
    c = 1000
    p = torch.rand(c + 2 * GUARD, device="cuda:0")
    before = p.clone()
    prio = p[GUARD:GUARD + c]
    indices = torch.tensor([-1, c, c + 5, 1 << 40, -(1 << 62), 3, 999, 0, 3], device="cuda:0")
    td = torch.arange(9, dtype=torch.float32, device="cuda:0")
    replay.per_update(prio, indices, td, 1.0, 0.0)
    torch.cuda.synchronize()
    want = before.clone()
    want[GUARD + 999], want[GUARD + 0], want[GUARD + 3] = 6.0, 7.0, 8.0
    same(p, want)


def test_update_of_nothing_is_a_no_op(dev):
    p = torch.rand(10, device="cuda:0")
    before = p.clone()
    replay.per_update(p, torch.empty(0, dtype=torch.int64, device="cuda:0"), torch.empty(0, device="cuda:0"), 0.6)
    same(p, before)


# ---- statuses and wrapper checks --------------------------------------------------------------------------------------
def sample_entry(dev, prio, c, batch, j0, rows, beta, tree, idx, w):
    return L.load().ktb_per_sample_f32(dev, prio, c, batch, j0, rows, 1, beta, tree, idx, w,
                                       ops.current_stream_handle(0) if dev == 0 else 0)


def update_entry(dev, prio, c, idx, td, b, alpha, eps):
    return L.load().ktb_per_update_f32(dev, prio, c, idx, td, b, alpha, eps,
                                       ops.current_stream_handle(0) if dev == 0 else 0)


def test_sample_statuses_follow_the_header_order(dev):
    x = torch.zeros(256, device="cuda:0")
    p = x.data_ptr()
    nan, inf = math.nan, math.inf
    assert sample_entry(15, 0, 0, 0, 0, 0, nan, 0, 0, 0) == L.ERR_STATE
    for beta in (nan, inf, -0.5):
        assert sample_entry(dev, 0, 0, 0, 0, 0, beta, 0, 0, 0) == L.ERR_ARG, beta
    assert sample_entry(dev, 0, 0, 8, 0, 1, 0.4, 0, 0, 0) == L.ERR_ARG             # C = 0
    assert sample_entry(dev, 0, (1 << 30) + 1, 8, 0, 1, 0.4, 0, 0, 0) == L.ERR_ARG
    assert sample_entry(dev, 0, 8, 0, 0, 0, 0.4, 0, 0, 0) == L.ERR_ARG             # batch = 0
    assert sample_entry(dev, 0, 8, 8193, 0, 0, 0.4, 0, 0, 0) == L.ERR_UNSUPPORTED
    assert sample_entry(dev, 0, 8, 8, 5, 4, 0.4, 0, 0, 0) == L.ERR_ARG             # j0 + rows > batch
    assert sample_entry(dev, 0, 8, 8, 8, 0, 0.4, 0, 0, 0) == L.OK                  # rows = 0: nothing to do
    # C = 8 priorities, tree of 8, 4 rows of indices (8 bytes) and weights
    ok = dict(prio=p, tree=p + 64, idx=p + 128, w=p + 192)

    def call(**over):
        a = dict(ok, **over)
        return sample_entry(dev, a["prio"], 8, 8, 4, 4, 0.4, a["tree"], a["idx"], a["w"])

    assert call() == L.OK
    for name in ok:
        assert call(**{name: 0}) == L.ERR_ARG, name
        assert call(**{name: ok[name] + 2}) == L.ERR_ARG, name
    assert call(idx=p + 132) == L.ERR_ARG           # 4-byte but not 8-byte aligned
    assert call(tree=p + 4) == L.ERR_ARG            # tree overlaps priorities
    assert call(idx=p + 88) == L.ERR_ARG            # indices overlap the tree
    assert call(w=p + 152) == L.ERR_ARG             # weights overlap indices
    assert call(w=p + 16) == L.ERR_ARG              # weights overlap priorities
    assert call(w=p + 160) == L.OK
    torch.cuda.synchronize()


def test_update_statuses_follow_the_header_order(dev):
    x = torch.zeros(256, device="cuda:0")
    p = x.data_ptr()
    nan = math.nan
    assert update_entry(15, 0, 0, 0, 0, 0, nan, nan) == L.ERR_STATE
    for a, e in ((nan, 0.0), (0.6, math.inf), (-math.inf, 1e-6)):
        assert update_entry(dev, 0, 0, 0, 0, 0, a, e) == L.ERR_ARG
    assert update_entry(dev, 0, 0, 0, 0, 1, 0.6, 0.0) == L.ERR_ARG                 # C = 0
    assert update_entry(dev, 0, 8, 0, 0, 0, 0.6, 0.0) == L.ERR_ARG                 # B = 0
    assert update_entry(dev, 0, 8, 0, 0, 8193, 0.6, 0.0) == L.ERR_UNSUPPORTED
    ok = dict(prio=p, idx=p + 64, td=p + 128)

    def call(**over):
        a = dict(ok, **over)
        return update_entry(dev, a["prio"], 8, a["idx"], a["td"], 4, 0.6, 1e-6)

    assert call() == L.OK
    for name in ok:
        assert call(**{name: 0}) == L.ERR_ARG, name
        assert call(**{name: ok[name] + 2}) == L.ERR_ARG, name
    assert call(idx=p + 68) == L.ERR_ARG
    assert call(idx=p + 24) == L.ERR_ARG            # indices overlap priorities
    assert call(td=p + 28) == L.ERR_ARG             # td overlaps priorities
    assert call(td=p + 64) == L.OK                  # inputs may alias
    torch.cuda.synchronize()


@pytest.mark.parametrize("case,match", [
    ("dtype", "priorities must be float32"),
    ("dim", "priorities must be a 1-D"),
    ("host", "priorities must be a CUDA tensor"),
    ("strided", "priorities must be contiguous"),
    ("batch", "batch must be an int in \\[1, 8192\\]"),
    ("seed", "seed must be an int"),
    ("rows", "j0=0 and rows=600 must be ints"),
    ("beta", "beta must be >= 0"),
    ("tree", "tree must have shape \\[1024\\]"),
    ("indices", "indices must be int64"),
])
def test_sample_wrapper_refuses_bad_arguments(dev, case, match):
    p = priorities(1000, seed=15).cuda()
    kw, batch, seed, beta = {}, 512, 1, 0.4
    if case == "dtype":
        p = p.double()
    elif case == "dim":
        p = p.view(10, 100)
    elif case == "host":
        p = p.cpu()
    elif case == "strided":
        p = torch.empty(2000, device="cuda:0")[::2]
    elif case == "batch":
        batch = 8193
    elif case == "seed":
        seed = -1
    elif case == "rows":
        kw["rows"] = 600
    elif case == "beta":
        beta = -1.0
    elif case == "tree":
        kw["tree"] = torch.empty(1000, device="cuda:0")
    elif case == "indices":
        kw["indices"] = torch.empty(512, dtype=torch.int32, device="cuda:0")
    with pytest.raises(ValueError, match=match):
        replay.per_sample(p, batch, seed, beta, **kw)


# ---- kt.mapped("per") through the public API --------------------------------------------------------------------------
def oracle_on_gpu(body, args, n):
    """The body rank by rank on the GPU, where its pow is CUDA's."""
    out = []
    for k in range(n):
        with mock.patch.dict(os.environ, {"RANK": str(k), "WORLD_SIZE": str(n)}):
            out.append(body(*(a.cuda() if isinstance(a, torch.Tensor) else a for a in args)))
    return out


def parts(got):
    return [(a.cpu(), b.cpu()) for a, b in got]


def check_parts(got, want):
    assert len(got) == len(want)
    for k, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g[0], w[0].cpu()), k
        same(g[1], w[1], k)


@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["1_rank", "3_ranks"])
def test_mapped_equals_oracle_and_wrapper(dev, devices):
    ranks = len(devices)
    p = priorities(100003, seed=16)
    want = oracle_on_gpu(mapped_per, (p, 17), ranks)
    mine = replay.per_sample(p.cuda(), BATCH, 17, BETA)
    fn = mapped_copy(mapped_per, "per", batch=BATCH, beta=BETA, seed="seed")
    with deployed(fn, f"t-per-{ranks}", devices) as remote:
        got = parts(remote(p.cuda(), 17, serialization="pickle"))
    check_parts(got, want)
    for k, g in enumerate(got):
        lo, hi = ops.shard_bounds(BATCH, ranks, k)
        assert torch.equal(g[0], mine[0][lo:hi].cpu())
        same(g[1], mine[1][lo:hi])


def test_mapped_with_a_workers_subset(dev):
    """Three workers of one rank each on cuda:0; workers=[0, 2] draws ranks 0 and 2 only, workers=[1] rank 1."""
    p = priorities(5000, seed=18)
    want = oracle_on_gpu(mapped_per, (p, 19), 3)
    fn = mapped_copy(mapped_per, "per", batch=BATCH, beta=BETA, seed="seed")
    with deployed(fn, "t-per-workers", [0, 0, 0], workers=3, num_proc=1) as remote:
        two = parts(remote(p.cuda(), 19, serialization="pickle", workers=[0, 2]))
        one = parts(remote(p.cuda(), 19, serialization="pickle", workers=[1]))
    check_parts(two + one, [want[0], want[2], want[1]])


def test_mapped_with_beta_as_a_call_argument_and_a_constant_seed(dev):
    p = priorities(3001, seed=20)
    fn = mapped_copy(mapped_per_beta, "per", batch=BATCH, beta="beta", seed="seed")
    with deployed(fn, "t-per-beta", [0, 0]) as remote:
        for beta in BETAS:
            got = parts(remote(p.cuda(), 21, beta, serialization="pickle"))
            check_parts(got, oracle_on_gpu(mapped_per_beta, (p, 21, beta), 2))
        with pytest.raises(Exception, match="beta must be >= 0"):
            remote(p.cuda(), 21, -0.5, serialization="pickle")
    fn = mapped_copy(mapped_per_seeded, "per", batch=BATCH, beta=BETA, seed=7)
    with deployed(fn, "t-per-seeded", [0, 0, 0]) as remote:
        check_parts(parts(remote(p.cuda(), serialization="pickle")), oracle_on_gpu(mapped_per_seeded, (p,), 3))


def test_mapped_refuses_host_tensors(dev):
    fn = mapped_copy(mapped_per, "per", batch=BATCH, beta=BETA, seed="seed")
    with deployed(fn, "t-per-host", [0]) as remote:
        with pytest.raises(Exception, match="'per' op takes CUDA tensors on the root GPU"):
            remote(priorities(100, seed=22), 1, serialization="pickle")


# ---- the deployment's self-check --------------------------------------------------------------------------------------
WRONG = [mapped_per_uniform, mapped_per_local, mapped_per_strict, mapped_per_unnormalised, mapped_per_other_stream]


@pytest.mark.parametrize("body", WRONG, ids=["uniform", "local_strata", "strict", "unnormalised", "other_stream"])
def test_self_check_refuses_a_body_the_op_does_not_compute(dev, body):
    fn = mapped_copy(body, "per", batch=BATCH, beta=BETA, seed="seed")
    with pytest.raises(ValueError, match="self-check failed.*'per' op.*mass >= left.*\\(min p / total \\* C\\)"):
        with deployed(fn, f"t-per-wrong-{body.__name__}", [0, 0]):
            pass
    # self_check=False deploys it anyway: the op computes the declared draw
    fn = mapped_copy(body, "per", batch=BATCH, beta=BETA, seed="seed", self_check=False)
    p = priorities(999, seed=23)
    with deployed(fn, f"t-per-unchecked-{body.__name__}", [0, 0]) as remote:
        check_parts(parts(remote(p.cuda(), 24, serialization="pickle")), oracle_on_gpu(mapped_per, (p, 24), 2))


@pytest.mark.parametrize("body,kw", [(mapped_per, dict(beta=BETA, seed="seed")),
                                     (mapped_per_beta, dict(beta="beta", seed="seed")),
                                     (mapped_per_seeded, dict(beta=BETA, seed=7))], ids=["seed", "beta", "constant"])
def test_self_check_accepts_the_body(dev, body, kw):
    fn = mapped_copy(body, "per", batch=BATCH, **kw)
    with deployed(fn, f"t-per-right-{body.__name__}", [0, 0, 0]) as remote:
        args = {"seed": (1,), "beta": (1, 0.4), "constant": ()}[
            "constant" if body is mapped_per_seeded else "beta" if body is mapped_per_beta else "seed"]
        assert len(remote(priorities(50, seed=25).cuda(), *args, serialization="pickle")) == 3
