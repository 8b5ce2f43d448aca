"""The Q(s, a) critic heads (ktb_mlp_bf16_critic and _twin, plain, staged and pushed) on the GPU.  Every q is tied bit
for bit to ktb_mlp_bf16_policy at d_out = 1, an entry already checked against fp64, over x = [obs | bf16(act) | 0] and
W1p: both issue the same K blocks over the same bytes."""
import ctypes
import math
import os
from unittest import mock

import pytest
import torch

from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp
from mlp_rig import K, Guarded, PushRig, deployed, expect_status, stream, tuning  # noqa: F401
from oracle import ref_dispatch
from policy_critic_cases import critic_q, mlp_critic, mlp_critic_nobias, mlp_critic_twin, q_min

pytestmark = pytest.mark.gpu


def _critic(d_in, d_act, d_hidden, bias, seed, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    w = [(torch.randn(*s, generator=g) * 0.05).bfloat16().to(device)
         for s in ((d_hidden, d_in + d_act), (d_hidden, d_hidden), (1, d_hidden))]
    b = [(torch.randn(n, generator=g) * 0.1).bfloat16().to(device) if bias else None for n in (d_hidden, d_hidden, 1)]
    return (w[0], b[0], w[1], b[1], w[2], b[2])


def _inputs(M, d_in, d_act, seed=7, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(M, d_in, generator=g).bfloat16().to(device),
            (torch.rand(M, d_act, generator=g) * 4 - 2).to(device))


def _tied(obs, act, c):
    """ktb_mlp_bf16_policy's logits at d_out = 1 over x = [obs | bf16(act) | 0] and W1p, widened to fp32."""
    M, d_in = obs.shape
    x = torch.zeros(M, d_in + 64, dtype=torch.bfloat16, device=obs.device)
    x[:, :d_in] = obs
    x[:, d_in:d_in + act.shape[1]] = act.to(torch.bfloat16)
    w1p = mlp._padded_w1(c[0], d_in)
    return mlp.mlp_forward(x, w1p, c[2], c[4], biases=(c[1], c[3], c[5])).float().squeeze(-1)


def _bits(t):
    return t.view(torch.int32)


def same(got, want, what):
    assert torch.equal(_bits(got), _bits(want)), (what, (got != want).sum())


@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("d_hidden", [256, 1024])
@pytest.mark.parametrize("d_in", [64, 256])
@pytest.mark.parametrize("d_act", [1, 2, 6, 17, 63, 64])
def test_critic_equals_the_policy_entry_over_the_padded_input(K, d_act, d_in, d_hidden, bias):
    obs, act = _inputs(1000, d_in, d_act)
    c = _critic(d_in, d_act, d_hidden, bias, seed=d_act)
    q = mlp.mlp_forward(obs, c[0], c[2], c[4], biases=(c[1], c[3], c[5]), output="critic", action=act)
    assert q.dtype == torch.float32 and q.shape == (1000,)
    same(q, _tied(obs, act, c), "critic vs policy entry")
    torch.testing.assert_close(q.cpu(), critic_q(obs.cpu(), act.cpu(), *[None if t is None else t.cpu() for t in c]),
                               rtol=2.0 ** -7, atol=1e-2)


@pytest.mark.parametrize("d_act", [6, 17, 64])
def test_twin_equals_two_single_critics_and_their_minimum(K, d_act):
    obs, act = _inputs(1000, 256, d_act)
    c1, c2 = _critic(256, d_act, 1024, True, 1), _critic(256, d_act, 1024, True, 2)
    q1, q2, qm = mlp.mlp_forward(obs, c1[0], c1[2], c1[4], biases=(c1[1], c1[3], c1[5]), output="critic", action=act,
                                 twin=c2)
    for got, c in ((q1, c1), (q2, c2)):
        same(got, mlp.mlp_forward(obs, c[0], c[2], c[4], biases=(c[1], c[3], c[5]), output="critic", action=act),
             "twin vs single")
    same(qm, q_min(q1, q2), "q_min")


SPECIAL = [0.0, -0.0, math.inf, -math.inf, math.nan, 0.5]


@pytest.mark.parametrize("v2", SPECIAL, ids=str)
@pytest.mark.parametrize("v1", SPECIAL, ids=str)
def test_twin_minimum_of_special_values_set_through_b3(K, v1, v2):
    """w3 = 0 with the sign of b3, so every product is a zero and q = b3: NaN, ±inf and numbers reach the minimum.  q1
    and q2 are checked bit for bit.  A zero q is +0 whatever the signs: the tensor cores sum all-zero products to +0 (on
    H100, even when every product is −0), and +0 + −0 = +0.  So no signed-zero tie of q1 and q2 reaches q_min from the
    kernel; the rule for one is pinned on the host (tests/test_mlp_critic_cpu.py)."""
    obs, act = _inputs(300, 64, 6)
    cs = []
    for i, v in enumerate((v1, v2)):
        c = list(_critic(64, 6, 256, True, 10 + i))
        c[4] = torch.full_like(c[4], -0.0 if math.copysign(1, v) < 0 else 0.0)
        c[5] = torch.full_like(c[5], v)
        cs.append(tuple(c))
    c1, c2 = cs
    q1, q2, qm = mlp.mlp_forward(obs, c1[0], c1[2], c1[4], biases=(c1[1], c1[3], c1[5]), output="critic", action=act,
                                 twin=c2)
    for got, v in ((q1, v1), (q2, v2)):
        want = torch.full((300,), 0.0 if v == 0 else v, device="cuda").bfloat16().float()
        if math.isnan(v):
            assert bool(got.isnan().all()), v
        else:
            same(got, want, ("intended q", v))
    nan = qm.isnan()
    ref = q_min(q1, q2)
    assert torch.equal(nan, ref.isnan()) and torch.equal(_bits(qm[~nan]), _bits(ref[~nan]))
    assert bool(nan.all()) == (math.isnan(v1) or math.isnan(v2)) and bool(nan.any()) == bool(nan.all())
    if v1 == 0 and v2 == 0:   # a tie of zeros gives q1
        same(qm, q1, "tie of zeros")


def test_nan_and_infinite_actions_follow_the_policy_entry(K):
    obs, act = _inputs(640, 64, 17)
    act[::7, 3] = math.nan
    act[1::7, 0] = math.inf
    act[2::7, 16] = -math.inf
    act[3::7] = math.nan
    c = _critic(64, 17, 256, True, 3)
    q = mlp.mlp_forward(obs, c[0], c[2], c[4], biases=(c[1], c[3], c[5]), output="critic", action=act)
    want = _tied(obs, act, c)
    nan = want.isnan()
    assert torch.equal(q.isnan(), nan)
    same(q[~nan], want[~nan], "edge rows")


def _push_call(K, obs, act, c, twin, chunk_rows, n=3):
    """The pushed forms through the push rig, ranks [0] * n on cuda:0 and one stream, the actions a side input beside
    the rows: ranks 1.. on the _pushed entry, the root's shard on the plain one."""
    M, d_in = obs.shape
    d_act, d_h = act.shape[1], c[0].shape[0]
    rig = PushRig(K, M, d_in, d_h, chunk_rows, "ce", n_ranks=n, sides=[("act", d_act * 4)],
                  scratch_bytes=lambda rows: mlp.pushed_scratch_bytes(rows, d_h, chunk_rows, True))
    outs = [torch.full((M,), 7.0, device="cuda") for _ in range(3 if twin else 1)]
    w1p = [mlp._padded_w1(c[0], d_in)] + ([mlp._padded_w1(twin[0], d_in)] if twin else [])
    ptr = lambda t: 0 if t is None else t.data_ptr()   # noqa: E731
    weights = [ptr(t) for t in (w1p[0],) + c[1:]]
    twin_ptrs = [ptr(t) for t in (w1p[1],) + tuple(twin[1:])] if twin else []
    entry = "ktb_mlp_bf16_critic" + ("_twin" if twin else "")

    def rank(r, b, e, p):
        L.call(entry + "_pushed", 0, p["stage"], p["stride"], e - b, d_in, d_h, d_act, *weights, *twin_ptrs, p["act"],
               *[o.data_ptr() + 4 * b for o in outs], p["scratch"], p["ctrl"], p["ctrl_root"], r, chunk_rows, p["seq"],
               stream())

    def root(b, e, rows):
        L.call(entry, 0, obs.data_ptr() + b * d_in * 2, e - b, d_in, d_h, d_act, *weights, *twin_ptrs, rows["act"],
               *[o.data_ptr() + 4 * b for o in outs], mlp._scratch_for(0, e - b, d_h, True).data_ptr(), 0, stream())

    for _ in (1, 2):
        rig.push(obs, {"act": act}, rank, root)
    rig.check()
    return outs


@pytest.mark.parametrize("ranks", [2, 3, 4])
@pytest.mark.parametrize("chunk", [None, 256])
@pytest.mark.parametrize("twin", [False, True], ids=["single", "twin"])
def test_every_form_gives_the_same_bits(K, twin, chunk, ranks):
    """Plain, staged and pushed.  A pushed split has shards of whole 128-row blocks, which torch.chunk's split makes
    equal; the rank count moves every rank's row and action offsets."""
    M = ranks * 640
    obs, act = _inputs(M, 128, 17)
    c = _critic(128, 17, 512, True, 4)
    t = _critic(128, 17, 512, True, 5) if twin else None
    kw = dict(biases=(c[1], c[3], c[5]), output="critic", action=act, twin=t)
    with tuning(chunk):
        plain = mlp.mlp_forward(obs, c[0], c[2], c[4], **kw)
        staged = mlp.mlp_forward(obs, c[0], c[2], c[4], staged=True, **kw)
        pushed = _push_call(K, obs, act, c, t, chunk or 16896, n=ranks)
    plain = plain if twin else (plain,)
    staged = staged if twin else (staged,)
    for p, s, u in zip(plain, staged, pushed):
        same(s, p, "staged")
        same(u, p, "pushed")


@pytest.mark.parametrize("M", [1003, 2, 0])
@pytest.mark.parametrize("twin", [False, True], ids=["single", "twin"])
def test_pull_scatter_gather_over_uneven_and_empty_shards(K, twin, M):
    """mlp_scatter_gather on four ranks of cuda:0 (the pull form): shards of 251 / 251 / 251 / 250 rows, two shards of
    one row and two empty ones, or none at all; each rank reads its action rows in place at its own offset."""
    obs, act = _inputs(M, 64, 6)
    c = _critic(64, 6, 256, True, 14)
    t = _critic(64, 6, 256, True, 15) if twin else None
    kw = dict(biases=(c[1], c[3], c[5]), output="critic", action=act, twin=t)
    got = mlp.mlp_scatter_gather(obs, c[0], c[2], c[4], [0, 0, 0, 0], **kw)
    torch.cuda.synchronize()
    want = mlp.mlp_forward(obs, c[0], c[2], c[4], **kw)
    for i, w in enumerate(want if twin else (want,)):
        same(torch.cat([g[i] if twin else g for g in got]), w, (M, i))


@pytest.mark.parametrize("twin", [False, True], ids=["single", "twin"])
def test_outputs_scratch_and_action_tile_stay_inside_their_bytes(K, twin):
    M, d_in, d_act, d_h = 700, 64, 6, 256
    obs, act = _inputs(M, d_in, d_act)
    c = _critic(d_in, d_act, d_h, True, 6)
    t = _critic(d_in, d_act, d_h, True, 7) if twin else None
    outs = [Guarded(4 * M, off) for off in ((4, 8, 12) if twin else (4,))]
    ptr = lambda x: 0 if x is None else x.data_ptr()   # noqa: E731
    w = [ptr(x) for x in (mlp._padded_w1(c[0], d_in),) + c[1:]]
    tw = [ptr(x) for x in (mlp._padded_w1(t[0], d_in),) + t[1:]] if twin else []
    with tuning(256):   # the scratch as documented for 256-row chunks: its action tile ends at the band
        scratch = Guarded(L.load().ktb_mlp_critic_scratch_bytes(M, d_h))
        assert scratch.nbytes == 2 * 256 * d_h * 2 + 256 * 64 * 2
        L.call("ktb_mlp_bf16_critic" + ("_twin" if twin else ""), 0, obs.data_ptr(), M, d_in, d_h, d_act, *w, *tw,
               act.data_ptr(), *[o.ptr() for o in outs], scratch.ptr(), 0, stream())
    for i, o in enumerate(outs):
        o.check(f"output {i}")
    scratch.check("scratch (hidden activations and action tile)")
    want = mlp.mlp_forward(obs, c[0], c[2], c[4], biases=(c[1], c[3], c[5]), output="critic", action=act, twin=t)
    for o, q in zip(outs, want if twin else (want,)):
        same(o.view(torch.float32), q, "guarded")


_PTRS = dict(obs=0, w1=0, b1=0, w2=0, b2=0, w3=0, b3=0, act=4096, q1=8192, q2=12288, q_min=16384, scratch=1 << 20,
             stage=0)


def _status_call(entry, pushed=False, **over):
    """(args, buffers kept alive) of `entry` over zero buffers: 256 rows, d_in 256, d_hidden 256, d_act 6.  An override
    `<pointer>_off=k` points that argument k bytes past its place, `<pointer>=0` makes it null, anything else replaces
    the argument."""
    z = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda")
    ctrl = torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda")
    a = {k: z.data_ptr() + v for k, v in _PTRS.items()}
    a.update(M=256, d_in=256, d_hidden=256, d_act=6, act_off=1 << 17, stride=1 << 20)
    for k, v in over.items():
        if k.endswith("_ptr"):
            a[k[:-4]] += v
        else:
            a[k] = v
    twin = entry.endswith("_twin")
    weights = [a[k] for k in ("w1", "b1", "w2", "b2", "w3", "b3")] * (2 if twin else 1)
    outs = [a["q1"], a["q2"], a["q_min"]] if twin else [a["q1"]]
    body = (a["M"], a["d_in"], a["d_hidden"], a["d_act"], *weights)
    if pushed:
        return (entry + "_pushed", 0, a["stage"], a["stride"], *body, a["act_off"], *outs, a["scratch"],
                ctrl.data_ptr(), ctrl.data_ptr(), 1, 256, 1, stream()), (z, ctrl)
    return (entry, 0, a["obs"], *body, a["act"], *outs, a["scratch"], 0, stream()), (z, ctrl)


STATUS_CASES = [   # in the entries' check order
    ("d_in", dict(d_in=100), L.ERR_ARG), ("d_hidden", dict(d_hidden=300), L.ERR_ARG),
    ("bias_align", dict(b1_ptr=1), L.ERR_ARG), ("w1_align", dict(w1_ptr=8), L.ERR_ARG),
    ("d_act_0", dict(d_act=0), L.ERR_ARG), ("d_act_65", dict(d_act=65), L.ERR_UNSUPPORTED),
    ("d_act_before_outputs", dict(d_act=65, q1=0), L.ERR_UNSUPPORTED),
    ("act_null", dict(act=0), L.ERR_ARG), ("act_align", dict(act_ptr=2), L.ERR_ARG),
    ("q_null", dict(q1=0), L.ERR_ARG), ("q_align", dict(q1_ptr=2), L.ERR_ARG),
]


@pytest.mark.parametrize("entry", ["ktb_mlp_bf16_critic", "ktb_mlp_bf16_critic_twin"])
@pytest.mark.parametrize("case,over,status", STATUS_CASES, ids=[c[0] for c in STATUS_CASES])
def test_plain_entry_statuses(K, entry, case, over, status):
    args, keep = _status_call(entry, **over)
    expect_status(args, status)


@pytest.mark.parametrize("over", [dict(q2=0), dict(q_min=0), dict(q2_ptr=2), dict(q_min_ptr=1)], ids=str)
def test_twin_statuses_cover_its_outputs(K, over):
    expect_status(_status_call("ktb_mlp_bf16_critic_twin", **over)[0], L.ERR_ARG)


def test_twin_statuses_cover_the_second_critic(K):
    args, keep = _status_call("ktb_mlp_bf16_critic_twin")
    for i, off in ((13, 8), (14, 1)):   # the second W1p not 16-byte aligned, its b1 not 2-byte aligned
        bad = list(args)
        bad[i] += off
        expect_status(tuple(bad), L.ERR_ARG)


@pytest.mark.parametrize("entry", ["ktb_mlp_bf16_critic", "ktb_mlp_bf16_critic_twin"])
@pytest.mark.parametrize("case,over,status", [
    ("region_before_d_act", dict(d_act=65, act_off=2), L.ERR_ARG),
    ("act_overlaps_rows", dict(act_off=256 * 256 * 2 - 4), L.ERR_ARG),
    ("act_past_stride", dict(act_off=(1 << 20) - 4), L.ERR_ARG),
    ("act_align", dict(act_off=(1 << 17) + 2), L.ERR_ARG),
], ids=lambda x: x if isinstance(x, str) else "")
def test_pushed_entry_statuses(K, entry, case, over, status):
    args, keep = _status_call(entry, pushed=True, **over)
    expect_status(args, status)


@pytest.mark.parametrize("entry", ["ktb_mlp_bf16_critic", "ktb_mlp_bf16_critic_twin"])
def test_empty_pushed_shard_with_null_outputs_acks(K, entry):
    args, (z, ctrl) = _status_call(entry, pushed=True, M=0, q1=0, q2=0, q_min=0)
    L.call(*args)
    torch.cuda.synchronize()
    assert int(ctrl.count_nonzero()) > 0   # ack[1] = 1 published in the (root's) control block


def test_in_place_polyak_update_reaches_the_next_call(K):
    obs, act = _inputs(512, 64, 6)
    c = list(_critic(64, 6, 256, True, 8))
    t = _critic(64, 6, 256, True, 9)
    kw = lambda: dict(biases=(c[1], c[3], c[5]), output="critic", action=act)   # noqa: E731
    before = mlp.mlp_forward(obs, c[0], c[2], c[4], **kw())
    with torch.no_grad():
        c[0].mul_(0.995).add_(t[0], alpha=0.005)
    after = mlp.mlp_forward(obs, c[0], c[2], c[4], **kw())
    assert not torch.equal(before, after)
    same(after, _tied(obs, act, c), "after the update")
    fresh = c[0].clone()
    same(after, mlp.mlp_forward(obs, fresh, c[2], c[4], **kw()), "a fresh copy of the updated weight")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("transfer", ["pull", "push"])
def test_in_place_polyak_update_through_two_devices(K, transfer):
    M = 2 * 1408
    obs, act = _inputs(M, 64, 6)
    c = list(_critic(64, 6, 256, True, 8))
    t = _critic(64, 6, 256, True, 9)
    for it in range(3):
        if it == 2:
            with torch.no_grad():
                c[0].mul_(0.995).add_(t[0], alpha=0.005)
                t[0].mul_(0.5)
        got = mlp.mlp_scatter_gather(obs, c[0], c[2], c[4], [0, 1], transfer=transfer, biases=(c[1], c[3], c[5]),
                                     output="critic", action=act, twin=t)
        torch.cuda.synchronize(0)
        torch.cuda.synchronize(1)
        want = mlp.mlp_forward(obs, c[0], c[2], c[4], biases=(c[1], c[3], c[5]), output="critic", action=act, twin=t)
        for i in range(3):
            same(torch.cat([g[i] for g in got]), want[i], (it, i))


def _public(bias=True, twin=False):
    g = torch.Generator().manual_seed(11)
    obs = torch.randn(1003, 128, generator=g).bfloat16()
    act = torch.rand(1003, 17, generator=g) * 2 - 1
    c1 = _critic(128, 17, 256, bias, 12, device="cpu")
    c2 = _critic(128, 17, 256, bias, 13, device="cpu")
    return obs, act, c1, c2


def _against_oracle(got, want):
    for g, w in zip(got, want):
        for a, b in zip(g if isinstance(g, tuple) else (g,), w if isinstance(w, tuple) else (w,)):
            torch.testing.assert_close(a.cpu(), b.cpu(), rtol=2.0 ** -7, atol=1e-2)


@pytest.mark.parametrize("twin", [False, True], ids=["single", "twin"])
@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["1_rank", "3_ranks"])
def test_mapped_critic_through_public_api(K, devices, twin):
    import kubetorch_b200 as kt

    obs, act, c1, c2 = _public(twin=twin)
    n = len(devices)
    body = mlp_critic_twin if twin else mlp_critic
    args = (obs, *c1, act) + (tuple(c2) if twin else ())
    want = ref_dispatch.spmd_call(body, *args, num_proc=n, serialization="pickle")
    policy = kt.mapped("mlp", bias=True, output="critic", action="act",
                       **(dict(twin=("v1", "c1", "v2", "c2", "v3", "c3")) if twin else {}))(body)
    gpu = [t.cuda() for t in args]
    mine = mlp.mlp_forward(gpu[0], gpu[1], gpu[3], gpu[5], biases=(gpu[2], gpu[4], gpu[6]), output="critic",
                           action=gpu[7], twin=tuple(gpu[8:]) if twin else None)
    with deployed(policy, f"t-critic-{int(twin)}-{n}", devices) as remote:
        got = remote(*gpu, serialization="pickle")
        torch.cuda.synchronize()
    assert len(got) == len(want) == n
    for r, g in enumerate(got):
        lo, hi = K.shard_bounds(obs.shape[0], n, r)
        for a, b in zip(g if twin else (g,), mine if twin else (mine,)):
            same(a.cuda(), b[lo:hi], r)
    _against_oracle(got, want)


def test_mapped_bias_free_critic_on_a_workers_subset(K):
    import kubetorch_b200 as kt

    obs, act, c1, _ = _public(bias=False)
    policy = kt.mapped("mlp", output="critic", action="act")(mlp_critic_nobias)
    gpu = [t.cuda() for t in (obs, c1[0], c1[2], c1[4], act)]
    mine = mlp.mlp_forward(gpu[0], gpu[1], gpu[2], gpu[3], output="critic", action=gpu[4])
    remote = kt.fn(policy, name="t-critic-workers").to(
        kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute("b200", workers=2, num_proc=1,
                                                                                 devices=[0, 0]))
    try:
        got = remote(*gpu, serialization="pickle", workers=[1])
        torch.cuda.synchronize()
    finally:
        remote.teardown()
    lo, hi = K.shard_bounds(obs.shape[0], 2, 1)
    assert len(got) == 1
    same(got[0].cuda(), mine[lo:hi], "workers=[1]")
    with mock.patch.dict(os.environ, {"RANK": "1", "WORLD_SIZE": "2"}):
        want = mlp_critic_nobias(obs, c1[0], c1[2], c1[4], act)
    torch.testing.assert_close(got[0].cpu(), want, rtol=2.0 ** -7, atol=1e-2)
