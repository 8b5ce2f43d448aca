"""The TD-target heads (ktb_mlp_bf16_td_target_deterministic and _gaussian, plain, staged and pushed) on the GPU.  Every
y is tied bit for bit to entries that are already checked against fp64: the header's formula over the actions (and
log-probabilities) of the standalone _deterministic / _gaussian_state entry with the same seed and row_base, and the q
of the standalone _critic (_twin) entry over those actions."""
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
from policy_td_target_cases import header_y, mlp_ddpg_target, mlp_sac_target, mlp_td3_target

pytestmark = pytest.mark.gpu

# (policy, options, twin, alpha): TD3, noise-free DDPG with one critic, SAC squashed and unsquashed
POLICIES = {
    "td3": ("deterministic", dict(noise=0.2, noise_clip=0.5, seed=11), True, None),
    "ddpg": ("deterministic", dict(), False, None),
    "sac": ("gaussian", dict(squash=True, seed=12), True, 0.2),
    "sac_unsquashed_a0": ("gaussian", dict(squash=False, seed=13), True, 0.0),
}


def _lin(g, shapes, scale, device):
    return [(torch.randn(*s, generator=g) * scale).bfloat16().to(device) for s in shapes]


def _nets(d_in, d_act, d_ha, d_h, bias, seed, device="cuda"):
    """(critic, second critic, actor, log-std head), each a tuple of weights and biases (None without biases)."""
    g = torch.Generator().manual_seed(seed)

    def net(w_shapes, b_lens, scale=0.05):
        w = _lin(g, w_shapes, scale, device)
        b = _lin(g, [(n,) for n in b_lens], 0.1, device) if bias else [None] * 3
        return (w[0], b[0], w[1], b[1], w[2], b[2])

    critic = lambda: net(((d_h, d_in + d_act), (d_h, d_h), (1, d_h)), (d_h, d_h, 1))   # noqa: E731
    c1, c2 = critic(), critic()
    actor = net(((d_ha, d_in), (d_ha, d_ha), (d_act, d_ha)), (d_ha, d_ha, d_act))
    w_ls = _lin(g, [(d_act, d_ha)], 0.05, device)[0]
    b_ls = _lin(g, [(d_act,)], 0.1, device)[0] if bias else None
    return c1, c2, actor, (w_ls, b_ls)


def _inputs(M, d_in, seed=7, device="cuda"):
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(M, d_in, generator=g).bfloat16().to(device)
    r = (torch.randn(M, generator=g) * 2).to(device)
    d = (torch.rand(M, generator=g) < 0.25).float().to(device)
    return obs, r, d


def _kw(name, c1, c2, actor, ls, r, d, gamma=0.99, **over):
    policy, opts, twin, alpha = POLICIES[name]
    kw = dict(biases=(c1[1], c1[3], c1[5]), output="td_target", actor=actor, policy=policy, reward=r, done=d,
              gamma=gamma, twin=c2 if twin else None, **opts)
    if policy == "gaussian":
        kw.update(log_std=ls, alpha=alpha)
    kw.update(over)
    return kw


def _fused(obs, c1, kw):
    return mlp.mlp_forward(obs, c1[0], c1[2], c1[4], **kw)


def _composed(obs, c1, kw, row_offset=0):
    """y of the header's formula over the standalone actor entry's outputs and the standalone critic entry's q."""
    a = kw["actor"]
    ab = (a[1], a[3], a[5])
    if kw["policy"] == "deterministic":
        act = mlp.mlp_forward(obs, a[0], a[2], a[4], biases=ab, output="deterministic", noise=kw.get("noise"),
                              noise_clip=kw.get("noise_clip"), seed=kw.get("seed"), squash=kw.get("squash"),
                              row_offset=row_offset)
        logp = None
    else:
        act, logp = mlp.mlp_forward(obs, a[0], a[2], a[4], biases=ab, output="gaussian", log_std=kw["log_std"],
                                    log_std_bounds=kw.get("log_std_bounds"), squash=kw.get("squash"), seed=kw["seed"],
                                    row_offset=row_offset)
    q = mlp.mlp_forward(obs, c1[0], c1[2], c1[4], biases=kw["biases"], output="critic", action=act, twin=kw["twin"])
    t = q[2] if kw["twin"] is not None else q
    return header_y(kw["reward"].cpu(), kw["done"].cpu(), kw["gamma"], t.cpu(), kw.get("alpha"),
                    None if logp is None else logp.cpu())


def _bits(t):
    return t.view(torch.int32)


def same(got, want, what):
    got, want = got.cpu(), want.cpu()
    nan = want.isnan()
    assert torch.equal(got.isnan(), nan), (what, int((got.isnan() != nan).sum()))
    assert torch.equal(_bits(got[~nan]), _bits(want[~nan])), (what, int((got[~nan] != want[~nan]).sum()))


SHAPES = [(64, 256, 256, True), (256, 1024, 256, False), (256, 256, 1024, True), (64, 1024, 1024, False)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "din{}-dha{}-dh{}-{}".format(*s[:3], "bias" if s[3] else "nobias"))
@pytest.mark.parametrize("d_act", [1, 2, 6, 17, 63, 64])
@pytest.mark.parametrize("name", list(POLICIES))
def test_target_equals_the_composed_entries(K, name, d_act, shape):
    d_in, d_ha, d_h, bias = shape
    obs, r, d = _inputs(1000, d_in)
    c1, c2, actor, ls = _nets(d_in, d_act, d_ha, d_h, bias, seed=d_act)
    kw = _kw(name, c1, c2, actor, ls, r, d)
    y = _fused(obs, c1, kw)
    assert y.dtype == torch.float32 and y.shape == (1000,)
    same(y, _composed(obs, c1, kw), (name, d_act, shape))


@pytest.mark.parametrize("case", ["done", "gamma0", "gamma1", "q_inf", "q_ninf", "q_nan", "sac_big_u", "sac_bounds"])
@pytest.mark.parametrize("name", list(POLICIES))
def test_special_values_follow_the_header(K, name, case):
    """done ∈ {0, 1, 0.5}; γ 0 and 1; q = ±inf and NaN set through b3 (w3 = 0, so q = b3; with done = 1 an infinite q
    gives NaN); SAC rows with |u| > 21 (a large actor mean through b3) and narrow log-std bounds."""
    M, d_in, d_act = 640, 64, 6
    obs, r, d = _inputs(M, d_in)
    d = torch.tensor([0.0, 1.0, 0.5], device="cuda").repeat(M // 3 + 1)[:M].contiguous()
    c1, c2, actor, ls = _nets(d_in, d_act, 256, 256, True, seed=3)
    over = {}
    if case == "gamma0":
        over["gamma"] = 0.0
    elif case == "gamma1":
        over["gamma"] = 1.0
    elif case.startswith("q_"):
        v = {"q_inf": math.inf, "q_ninf": -math.inf, "q_nan": math.nan}[case]
        c1 = c1[:4] + (torch.zeros_like(c1[4]), torch.full_like(c1[5], v))
    elif case == "sac_big_u":
        actor = actor[:5] + (torch.tensor([30.0, -25.0, 22.0, 0.5, -40.0, 3.0]).bfloat16().cuda(),)
    elif case == "sac_bounds":
        over["log_std_bounds"] = (-1.0, -0.5)
    if case.startswith("sac") and POLICIES[name][0] != "gaussian":
        pytest.skip("a SAC case")
    kw = _kw(name, c1, c2, actor, ls, r, d, **over)
    y = _fused(obs, c1, kw)
    same(y, _composed(obs, c1, kw), (name, case))
    if case == "q_inf" and POLICIES[name][2] is False:   # DDPG's t is q itself: done = 1 with q = inf is NaN
        assert bool(y[1::3].isnan().all()) and bool((y[0::3] == math.inf).all())


def _push_call(K, obs, c1, kw, chunk_rows, n):
    """The pushed forms through the push rig, ranks [0] * n on cuda:0 and one stream, reward and done side inputs
    beside the rows: ranks 1.. on the _pushed entry, the root's shard on the plain one through mlp_forward."""
    M, d_in = obs.shape
    policy, gaussian = kw["policy"], kw["policy"] == "gaussian"
    a = list(kw["actor"])
    if gaussian:
        a[4], a[5] = mlp._stacked_head(a[4], a[5], None, None, *kw["log_std"])
    d_act, d_ha, d_h = a[4].shape[0] // (2 if gaussian else 1), a[0].shape[0], c1[0].shape[0]
    rig = PushRig(K, M, d_in, d_h, chunk_rows, "ce", n_ranks=n, sides=[("reward", 4), ("done", 4)],
                  scratch_bytes=lambda rows: mlp.pushed_td_scratch_bytes(rows, d_ha, d_h, d_act, chunk_rows))
    y = torch.full((M,), 7.0, device="cuda")
    ptr = lambda t: 0 if t is None else t.data_ptr()   # noqa: E731
    crit = [ptr(t) for t in (mlp._padded_w1(c1[0], d_in),) + c1[1:]]
    tw = kw["twin"]
    twin = [ptr(t) for t in (mlp._padded_w1(tw[0], d_in),) + tuple(tw[1:])] if tw else [0] * 6

    def rank(r, b, e, p):
        args = mlp._td_args(policy, kw.get("seed"), kw.get("log_std"), kw.get("log_std_bounds"), kw.get("squash"),
                            kw.get("noise"), kw.get("noise_clip"), b)
        L.call("ktb_mlp_bf16_td_target_" + policy + "_pushed", 0, p["stage"], p["stride"], e - b, d_in, d_h, d_act,
               *crit, *twin, d_ha, *[ptr(t) for t in a], *args, p["reward"], p["done"], float(kw["gamma"]),
               *((float(kw["alpha"]),) if gaussian else ()), y.data_ptr() + 4 * b, p["scratch"], p["ctrl"],
               p["ctrl_root"], r, chunk_rows, p["seq"], stream())

    def root(b, e, rows):
        sub = dict(kw, reward=kw["reward"][b:e], done=kw["done"][b:e], target=y[b:e], row_offset=b)
        _fused(obs[b:e], c1, dict(sub, stream=torch.cuda.current_stream()))

    for _ in (1, 2):
        rig.push(obs, {"reward": kw["reward"], "done": kw["done"]}, rank, root)
    rig.check()
    return y


@pytest.mark.parametrize("ranks", [2, 3, 4])
@pytest.mark.parametrize("chunk", [None, 256])
@pytest.mark.parametrize("name", ["td3", "ddpg", "sac"])
def test_every_form_gives_the_same_bits(K, name, chunk, ranks):
    """Plain, staged, pushed and row_offset splits, at the shipped chunk and at 256-row chunks."""
    M = ranks * 640
    obs, r, d = _inputs(M, 128)
    c1, c2, actor, ls = _nets(128, 17, 512, 256, True, 4)
    kw = _kw(name, c1, c2, actor, ls, r, d)
    with tuning(chunk):
        plain = _fused(obs, c1, kw)
        staged = _fused(obs, c1, dict(kw, staged=True))
        split = torch.cat([_fused(obs[b:e], c1, dict(kw, reward=r[b:e], done=d[b:e], row_offset=b))
                           for b, e in ((0, 384), (384, 1000), (1000, M))])
        pushed = _push_call(K, obs, c1, kw, chunk or 16896, ranks)
    same(plain, _composed(obs, c1, kw), "composed")
    for what, got in (("staged", staged), ("split", split), ("pushed", pushed)):
        same(got, plain, what)


@pytest.mark.parametrize("M", [1003, 2, 0])
@pytest.mark.parametrize("name", ["td3", "sac"])
def test_pull_scatter_gather_over_uneven_and_empty_shards(K, name, M):
    obs, r, d = _inputs(M, 64)
    c1, c2, actor, ls = _nets(64, 6, 256, 256, True, 14)
    kw = _kw(name, c1, c2, actor, ls, r, d)
    kw.pop("biases")
    got = mlp.mlp_scatter_gather(obs, c1[0], c1[2], c1[4], [0, 0, 0, 0], biases=(c1[1], c1[3], c1[5]), **kw)
    torch.cuda.synchronize()
    want = _fused(obs, c1, dict(kw, biases=(c1[1], c1[3], c1[5])))
    same(torch.cat(got), want, M)


@pytest.mark.parametrize("name", ["td3", "ddpg", "sac"])
def test_package_push_path_on_one_gpu_matches_plain_bits(K, name):
    """mlp_scatter_gather's pushed form (the rows, reward and done pushed into each staging half, the root's shard on
    the side stream) with ranks [0, 0, 0] on cuda:0, back to back with fresh inputs: equal to one plain call over all
    rows."""
    devs, M, d_in = [0, 0, 0], 3 * 1280, 128
    bounds = [K.shard_bounds(M, 3, r) for r in range(3)]
    c1, c2, actor, ls = _nets(d_in, 17, 512, 256, True, 4)
    policy, opts, twin, alpha = POLICIES[name]
    gaussian = policy == "gaussian"
    a = (*actor[:4], *mlp._stacked_head(actor[4], actor[5], None, None, *ls)) if gaussian else actor
    weights = {0: (mlp._padded_w1(c1[0], d_in), c1[2], c1[4], c1[1], c1[3], c1[5])}
    tw = {0: (mlp._padded_w1(c2[0], d_in), *c2[1:])} if twin else None
    std = mlp._std(ls, None, opts.get("squash")) if gaussian else None
    det = None if gaussian else dict(noise=opts.get("noise"), noise_clip=opts.get("noise_clip"),
                                     squash=opts.get("squash"))
    for it in range(3):
        obs, r, d = _inputs(M, d_in, seed=20 + it)
        want = _fused(obs, c1, _kw(name, c1, c2, actor, ls, r, d))
        y = torch.full((M,), 7.0, device="cuda")
        mlp._mlp_scatter_gather_pushed(obs, devs, bounds, weights, "td_target", y, None, None, opts.get("seed"),
                                       {0: ls} if gaussian else None, std=std, det=det, twin=tw,
                                       td=({0: a}, policy, r, d, 0.99, alpha))
        torch.cuda.synchronize()
        same(y, want, (name, it))
    mlp._push_sessions[tuple(devs)].check()


@pytest.mark.parametrize("name", ["td3", "ddpg", "sac"])
def test_y_and_scratch_stay_inside_their_bytes(K, name):
    M, d_in, d_act, d_ha, d_h = 700, 64, 6, 512, 256
    obs, r, d = _inputs(M, d_in)
    c1, c2, actor, ls = _nets(d_in, d_act, d_ha, d_h, True, 6)
    kw = _kw(name, c1, c2, actor, ls, r, d)
    want = _fused(obs, c1, kw)
    y = Guarded(4 * M, 4)
    with tuning(256):   # the scratch as documented for 256-row chunks: the q1 slot ends at the band
        nbytes = L.load().ktb_mlp_td_target_scratch_bytes(M, d_ha, d_h, d_act)
        assert nbytes == 2 * 256 * 512 * 2 + 256 * 64 * 2 + 256 * (4 * d_act + 8)
        scratch = Guarded(nbytes)
        with mock.patch.object(mlp, "_cached_buffer", lambda cache, key, dev, n: scratch.view()):
            _fused(obs, c1, dict(kw, target=y.view(torch.float32)))
    y.check("y")
    scratch.check("scratch (hidden activations, action tile, actions, log-probabilities, q1)")
    same(y.view(torch.float32), want, "guarded")


def test_scratch_size_function(K):
    lib = L.load()
    assert lib.ktb_mlp_td_target_scratch_bytes(0, 256, 256, 6) == 0
    assert lib.ktb_mlp_td_target_scratch_bytes(100, 1024, 256, 17) == 100 * (4 * 1024 + 128 + 4 * 17 + 8)
    assert lib.ktb_mlp_td_target_scratch_bytes(1 << 20, 256, 512, 64) == 16896 * (4 * 512 + 128 + 4 * 64 + 8)


_PTRS = dict(obs=0, w1=0, b1=0, w2=0, b2=0, w3=0, b3=0, r=4096, d=8192, y=12288, scratch=1 << 20, stage=0)


def _status_call(policy, pushed=False, twin=True, **over):
    """(args, buffers kept alive) over zero buffers: 256 rows, d_in 256, every d_hidden 256, d_act 6.  `<ptr>_ptr=k`
    moves a pointer k bytes, `<ptr>=0` makes it null, anything else replaces the argument."""
    z = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda")
    ctrl = torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda")
    a = {k: z.data_ptr() + v for k, v in _PTRS.items()}
    a.update(M=256, d_in=256, d_hidden=256, d_ha=256, d_act=6, r_off=1 << 17, d_off=(1 << 17) + 4096, stride=1 << 20,
             gamma=0.99, alpha=0.2, noise=0.2, clip=0.5, lo=-20.0, hi=2.0, tw_w1=a["w1"])
    for k, v in over.items():
        if k.endswith("_ptr"):
            a[k[:-4]] += v
        else:
            a[k] = v
    w = [a[k] for k in ("w1", "b1", "w2", "b2", "w3", "b3")]
    tw = [a["tw_w1"], a["b1"], a["w2"], a["b2"], a["w3"], a["b3"]] if twin else [0] * 6
    body = (a["M"], a["d_in"], a["d_hidden"], a["d_act"], *w, *tw, a["d_ha"], *w)
    pol = (a["noise"], a["clip"], 1, 5, 0) if policy == "deterministic" else (a["lo"], a["hi"], 1, 5, 0)
    tail = (a["gamma"],) + ((a["alpha"],) if policy == "gaussian" else ()) + (a["y"], a["scratch"])
    entry = "ktb_mlp_bf16_td_target_" + policy
    if pushed:
        return (entry + "_pushed", 0, a["stage"], a["stride"], *body, *pol, a["r_off"], a["d_off"], *tail,
                ctrl.data_ptr(), ctrl.data_ptr(), 1, 256, 1, stream()), (z, ctrl)
    return (entry, 0, a["obs"], *body, *pol, a["r"], a["d"], *tail, 0, stream()), (z, ctrl)


STATUS_CASES = [   # in the entries' check order
    ("d_in", dict(d_in=100), L.ERR_ARG), ("d_hidden", dict(d_hidden=300), L.ERR_ARG),
    ("bias_align", dict(b1_ptr=1), L.ERR_ARG), ("w1_align", dict(w1_ptr=8), L.ERR_ARG),
    ("twin_partial", dict(tw_w1=0), L.ERR_ARG),
    ("d_act_0", dict(d_act=0), L.ERR_ARG), ("d_act_65", dict(d_act=65), L.ERR_UNSUPPORTED),
    ("d_act_before_actor", dict(d_act=65, d_ha=300), L.ERR_UNSUPPORTED),
    ("actor_hidden", dict(d_ha=300), L.ERR_ARG),
    ("actor_before_gamma", dict(d_ha=300, gamma=math.nan), L.ERR_ARG),
    ("gamma_nan", dict(gamma=math.nan), L.ERR_ARG), ("gamma_inf", dict(gamma=math.inf), L.ERR_ARG),
    ("gamma_before_y", dict(gamma=math.inf, y=0), L.ERR_ARG),
    ("y_null", dict(y=0), L.ERR_ARG), ("y_align", dict(y_ptr=2), L.ERR_ARG),
    ("reward_null", dict(r=0), L.ERR_ARG), ("done_align", dict(d_ptr=1), L.ERR_ARG),
]


@pytest.mark.parametrize("policy", ["deterministic", "gaussian"])
@pytest.mark.parametrize("case,over,status", STATUS_CASES, ids=[c[0] for c in STATUS_CASES])
def test_plain_entry_statuses(K, policy, case, over, status):
    args, keep = _status_call(policy, **over)
    expect_status(args, status)


@pytest.mark.parametrize("policy,over", [("deterministic", dict(noise=-1.0)), ("deterministic", dict(clip=math.nan)),
                                         ("gaussian", dict(lo=3.0)), ("gaussian", dict(alpha=math.nan)),
                                         ("gaussian", dict(alpha=math.inf))], ids=str)
def test_policy_statuses(K, policy, over):
    expect_status(_status_call(policy, **over)[0], L.ERR_ARG)


@pytest.mark.parametrize("policy", ["deterministic", "gaussian"])
@pytest.mark.parametrize("case,over,status", [
    ("region_before_d_act", dict(d_act=65, r_off=2), L.ERR_ARG),
    ("gamma_first", dict(gamma=math.nan, r_off=2), L.ERR_ARG),
    ("reward_overlaps_rows", dict(r_off=256 * 256 * 2 - 4), L.ERR_ARG),
    ("done_past_stride", dict(d_off=(1 << 20) - 4), L.ERR_ARG),
    ("reward_align", dict(r_off=(1 << 17) + 2), L.ERR_ARG),
    ("regions_overlap", dict(d_off=(1 << 17) + 512), L.ERR_ARG),
], ids=lambda x: x if isinstance(x, str) else "")
def test_pushed_entry_statuses(K, policy, case, over, status):
    args, keep = _status_call(policy, pushed=True, **over)
    expect_status(args, status)


@pytest.mark.parametrize("policy", ["deterministic", "gaussian"])
def test_empty_pushed_shard_with_null_outputs_acks(K, policy):
    args, (z, ctrl) = _status_call(policy, pushed=True, M=0, y=0)
    L.call(*args)
    torch.cuda.synchronize()
    assert int(ctrl.count_nonzero()) > 0   # ack[1] = 1 published in the (root's) control block


@pytest.mark.parametrize("name", ["td3", "sac"])
def test_in_place_polyak_updates_reach_the_next_call(K, name):
    obs, r, d = _inputs(512, 64)
    c1, c2, actor, ls = _nets(64, 6, 256, 256, True, 8)
    src = _nets(64, 6, 256, 256, True, 9)
    kw = _kw(name, c1, c2, actor, ls, r, d)
    before = _fused(obs, c1, kw)
    with torch.no_grad():
        c2[0].mul_(0.995).add_(src[1][0], alpha=0.005)   # the second target critic's w1
        actor[4].mul_(0.5)                                 # the actor's mean head w3
        ls[0].mul_(0.5)                                    # the actor's log-std head w_ls
    after = _fused(obs, c1, kw)
    assert not torch.equal(before, after)
    same(after, _composed(obs, c1, kw), "after the update")


def _public(seed=21):
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(1003, 128, generator=g).bfloat16()
    r = torch.randn(1003, generator=g)
    d = (torch.rand(1003, generator=g) < 0.2).float()
    c1, c2, actor, ls = _nets(128, 17, 256, 512, True, seed, device="cpu")
    return obs, r, d, c1, c2, actor, ls


def _close_where_the_actions_agree(got, want):
    """rtol 2^-7, atol 1e-2 against the fp32 body, as the critic's bar.  The body's actor runs bf16 GEMMs on the CPU,
    whose fp32 sums round differently; where a rounding moves a bf16 actor output the actions differ and q moves by
    up to Lipschitz × one bf16 ulp, so the bar is widened to atol 5e-2 for those few rows rather than dropped."""
    got, want = got.cpu(), want.cpu()
    torch.testing.assert_close(got, want, rtol=2.0 ** -7, atol=5e-2)
    close = torch.isclose(got, want, rtol=2.0 ** -7, atol=1e-2)
    assert float(close.float().mean()) > 0.97


@pytest.mark.parametrize("name", ["td3", "sac"])
@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["1_rank", "3_ranks"])
def test_mapped_target_through_public_api(K, devices, name):
    import kubetorch_b200 as kt

    obs, r, d, c1, c2, actor, ls = _public()
    n = len(devices)
    names = dict(actor=("a1", "ab1", "a2", "ab2", "a3", "ab3"), twin=("v1", "c1", "v2", "c2", "v3", "c3"),
                 reward="r", done="d", gamma=0.99, seed="seed")
    if name == "td3":
        body, args = mlp_td3_target, (obs, *c1, *actor, *c2, r, d, 11)
        policy = kt.mapped("mlp", bias=True, output="td_target", policy="deterministic", noise=0.2, noise_clip=0.5,
                           **names)(body)
    else:
        body, args = mlp_sac_target, (obs, *c1, *actor, *ls, *c2, r, d, 12, torch.tensor([0.2]))
        policy = kt.mapped("mlp", bias=True, output="td_target", policy="gaussian", log_std=("w_ls", "b_ls"),
                           alpha="alpha", squash=True, **names)(body)
    want = ref_dispatch.spmd_call(body, *args, num_proc=n, serialization="pickle")
    gpu = [t.cuda() if isinstance(t, torch.Tensor) else t for t in args]
    cg, ag = gpu[1:7], gpu[7:13]
    kw = _kw(name, cg, gpu[13 + 2 * (name == "sac"):19 + 2 * (name == "sac")], ag,
             tuple(gpu[13:15]) if name == "sac" else None, gpu[-4 if name == "sac" else -3],
             gpu[-3 if name == "sac" else -2])
    mine = _fused(gpu[0], cg, kw)
    with deployed(policy, f"t-td-{name}-{n}", devices) as remote:
        got = remote(*gpu, serialization="pickle")
        torch.cuda.synchronize()
    assert len(got) == len(want) == n
    for k, g in enumerate(got):
        lo, hi = K.shard_bounds(obs.shape[0], n, k)
        same(g.cuda(), mine[lo:hi], k)
        _close_where_the_actions_agree(g, want[k])


def test_mapped_ddpg_target_on_a_workers_subset(K):
    import kubetorch_b200 as kt

    obs, r, d, c1, _, actor, _ = _public(23)
    policy = kt.mapped("mlp", bias=True, output="td_target", policy="deterministic",
                       actor=("a1", "ab1", "a2", "ab2", "a3", "ab3"), reward="r", done="d", gamma=0.99)(mlp_ddpg_target)
    args = (obs, *c1, *actor, r, d)
    gpu = [t.cuda() for t in args]
    kw = _kw("ddpg", gpu[1:7], None, gpu[7:13], None, gpu[13], gpu[14])
    mine = _fused(gpu[0], gpu[1:7], kw)
    remote = kt.fn(policy, name="t-td-workers").to(
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
        want = mlp_ddpg_target(*args)
    _close_where_the_actions_agree(got[0], want)
