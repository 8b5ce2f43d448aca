"""The DQN-target heads (ktb_mlp_bf16_dqn_target and _masked, plain, staged and pushed) on the GPU.  Every y is tied bit
for bit to entries that are already checked against fp64: the header's formula over the actions entry on the selecting
network (ktb_mlp_bf16_policy(_masked)) and the logits entry on the target network, gathered unmasked."""
import math
from unittest import mock

import pytest
import torch

from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp
from mlp_rig import K, Guarded, PushRig, deployed, expect_status, stream, tuning  # noqa: F401
from oracle import ref_dispatch
from policy_dqn_target_cases import (header_y, mlp_double_dqn_target, mlp_double_dqn_target_masked, mlp_dqn_target,
                                     mlp_dqn_target_masked)

pytestmark = pytest.mark.gpu


def _net(g, d_in, d_h, d_out, bias, device="cuda"):
    """(w1, b1, w2, b2, w3, b3) of a Q-network (biases None without biases)."""
    w = [(torch.randn(*s, generator=g) * 0.05).bfloat16().to(device) for s in ((d_h, d_in), (d_h, d_h), (d_out, d_h))]
    b = [(torch.randn(n, generator=g) * 0.1).bfloat16().to(device) for n in (d_h, d_h, d_out)] if bias else [None] * 3
    return (w[0], b[0], w[1], b[1], w[2], b[2])


def _case(M, d_out, d_in=64, d_h=256, bias=True, seed=0, device="cuda"):
    """(obs, target, online, legal, reward, done): about 5 % of the rows have no legal action."""
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(M, d_in, generator=g).bfloat16().to(device)
    target, online = _net(g, d_in, d_h, d_out, bias, device), _net(g, d_in, d_h, d_out, bias, device)
    legal = torch.rand(M, d_out, generator=g) < 0.6
    legal[torch.rand(M, generator=g) < 0.05] = False
    r = (torch.randn(M, generator=g) * 2).to(device)
    d = (torch.rand(M, generator=g) < 0.25).float().to(device)
    return obs, target, online, legal.to(device), r, d


def _fused(obs, t, online=None, mask=None, r=None, d=None, gamma=0.99, **kw):
    return mlp.mlp_forward(obs, t[0], t[2], t[4], biases=(t[1], t[3], t[5]), output="dqn_target", online=online,
                           mask=mask, reward=r, done=d, gamma=gamma, **kw)


def _composed(obs, t, online=None, mask=None, r=None, d=None, gamma=0.99):
    """The two-call composition: the actions entry on the selector, the logits entry on the target, the header's y."""
    s = online if online is not None else t
    a = mlp.mlp_forward(obs, s[0], s[2], s[4], biases=(s[1], s[3], s[5]), output="actions", mask=mask)
    qt = mlp.mlp_forward(obs, t[0], t[2], t[4], biases=(t[1], t[3], t[5]), output="logits")
    q = qt.float().gather(1, a[:, None]).squeeze(1)
    return header_y(r.cpu(), d.cpu(), gamma, q.cpu())


def _bits(t):
    return t.view(torch.int32)


def same(got, want, what):
    got, want = got.cpu(), want.cpu()
    nan = want.isnan()
    assert torch.equal(got.isnan(), nan), (what, int((got.isnan() != nan).sum()))
    assert torch.equal(_bits(got[~nan]), _bits(want[~nan])), (what, int((got[~nan] != want[~nan]).sum()))


D_OUTS = [1, 2, 6, 18, 63, 64, 65, 128, 255, 256]


@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("double", [False, True], ids=["dqn", "double"])
@pytest.mark.parametrize("d_out", D_OUTS)
def test_target_equals_the_composed_entries(K, d_out, double, masked, bias):
    obs, t, o, legal, r, d = _case(1000, d_out, bias=bias, seed=d_out)
    kw = dict(online=o if double else None, mask=legal if masked else None, r=r, d=d)
    y = _fused(obs, t, **kw)
    assert y.dtype == torch.float32 and y.shape == (1000,)
    same(y, _composed(obs, t, **kw), (d_out, double, masked, bias))


@pytest.mark.parametrize("M,chunk", [(0, None), (1, None), (127, None), (129, None), (5 * 256 + 128 + 37, 256)],
                         ids=["M0", "M1", "M127", "M129", "chunks256-ragged"])
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("double", [False, True], ids=["dqn", "double"])
def test_row_counts_and_chunks(K, M, chunk, double, masked):
    obs, t, o, legal, r, d = _case(M, 18, seed=M + 1)
    kw = dict(online=o if double else None, mask=legal if masked else None, r=r, d=d)
    with tuning(chunk):
        y = _fused(obs, t, **kw)
        want = _composed(obs, t, **kw)
    assert y.shape == (M,)
    same(y, want, (M, chunk))


@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("d_out", [6, 18, 256])
def test_dqn_equals_double_dqn_with_online_equal_to_target(K, d_out, masked):
    obs, t, o, legal, r, d = _case(777, d_out, seed=5)
    mask = legal if masked else None
    same(_fused(obs, t, online=t, mask=mask, r=r, d=d), _fused(obs, t, mask=mask, r=r, d=d), d_out)


def _special(t, cols, values):
    """t with w3 rows `cols` zero and b3 there `values`: the head's Q-value there is the bias on every row."""
    w3, b3 = t[4].clone(), t[5].clone()
    w3[cols] = 0
    b3[cols] = torch.tensor(values, device="cuda").bfloat16()
    return (*t[:4], w3, b3)


def test_nan_selectors(K):
    """A NaN in the selector picks the first NaN column: DQN's y is NaN, Double DQN's the target's value there."""
    obs, t, o, legal, r, d = _case(640, 18, seed=9)
    tn = _special(t, [3, 7], [math.nan, math.nan])
    y = _fused(obs, tn, r=r, d=d)
    same(y, _composed(obs, tn, r=r, d=d), "dqn")
    assert bool(y.isnan().all())
    on = _special(o, [3, 7], [math.nan, math.nan])
    y2 = _fused(obs, t, online=on, r=r, d=d)
    same(y2, _composed(obs, t, online=on, r=r, d=d), "double")
    qt = mlp.mlp_forward(obs, t[0], t[2], t[4], biases=(t[1], t[3], t[5]), output="logits")
    same(y2, header_y(r.cpu(), d.cpu(), 0.99, qt[:, 3].float().cpu()), "double reads the target at the NaN column")
    # the mask hides the NaN columns from the ranking: illegal NaNs are never picked
    mask = torch.ones_like(legal)
    mask[:, [3, 7]] = False
    same(_fused(obs, tn, mask=mask, r=r, d=d), _composed(obs, tn, mask=mask, r=r, d=d), "masked nan")
    assert not bool(_fused(obs, tn, mask=mask, r=r, d=d).isnan().any())


@pytest.mark.parametrize("gamma", [0.99, 0.0])
@pytest.mark.parametrize("v", [math.inf, -math.inf])
def test_infinite_q_with_done_and_gamma(K, v, gamma):
    """q = ±inf in every column (w3 = 0, b3 = ±inf): done = 1 or γ = 0 gives NaN, done = 0 with γ > 0 gives ±inf."""
    obs, t, o, legal, r, d = _case(640, 6, seed=10)
    d = torch.tensor([0.0, 1.0], device="cuda").repeat(320).contiguous()
    ti = _special(t, list(range(6)), [v] * 6)
    y = _fused(obs, ti, r=r, d=d, gamma=gamma)
    same(y, _composed(obs, ti, r=r, d=d, gamma=gamma), (v, gamma))
    if gamma == 0.0:
        assert bool(y.isnan().all())
    else:
        assert bool(y[1::2].isnan().all()) and bool((y[0::2] == v).all())


@pytest.mark.parametrize("double", [False, True], ids=["dqn", "double"])
def test_rows_with_no_legal_action_give_the_reward_when_done(K, double):
    obs, t, o, legal, r, d = _case(1000, 18, seed=11)
    legal[::3] = False
    d[::3] = 1.0
    y = _fused(obs, t, online=o if double else None, mask=legal, r=r, d=d)
    same(y, _composed(obs, t, online=o if double else None, mask=legal, r=r, d=d), double)
    assert torch.equal(_bits(y[::3].cpu()), _bits(r[::3].cpu()))


def test_reward_of_shape_m_1(K):
    obs, t, o, legal, r, d = _case(300, 18, seed=12)
    y = _fused(obs, t, online=o, r=r[:, None].contiguous(), d=d[:, None].contiguous())
    assert y.shape == (300, 1)
    same(y[:, 0], _fused(obs, t, online=o, r=r, d=d), "[M, 1]")


# ---- forms ----------------------------------------------------------------------------------------------------------
def _push_call(K, obs, t, online, mask, r, d, chunk_rows, n, gamma=0.99):
    """The pushed forms through the push rig, ranks [0] * n on cuda:0 and one stream, (the mask and) the (reward, done)
    pairs as side inputs beside the rows: ranks 1.. on the _pushed entry, the root's shard on the plain one."""
    M, d_in = obs.shape
    d_h, d_out = t[0].shape[0], t[4].shape[0]
    sides = ([("mask", d_out)] if mask is not None else []) + [("rd", 8)]
    rig = PushRig(K, M, d_in, d_h, chunk_rows, "ce", n_ranks=n, sides=sides,
                  scratch_bytes=lambda rows: mlp.pushed_scratch_bytes(rows, d_h, chunk_rows) +
                  min(rows, chunk_rows) * 8)
    y = torch.full((M,), 7.0, device="cuda")
    ptr = lambda x: 0 if x is None else x.data_ptr()   # noqa: E731
    rd = torch.stack((r, d), 1)
    entry = "ktb_mlp_bf16_dqn_target" + ("" if mask is None else "_masked") + "_pushed"

    def rank(k, b, e, p):
        L.call(entry, 0, p["stage"], p["stride"], e - b, d_in, d_h, d_out, *[ptr(x) for x in t],
               *[ptr(x) for x in (online or (None,) * 6)], *(() if mask is None else (p["mask"],)), p["rd"],
               float(gamma), y.data_ptr() + 4 * b, p["scratch"], p["ctrl"], p["ctrl_root"], k, chunk_rows, p["seq"],
               stream())

    def root(b, e, rows):
        _fused(obs[b:e], t, online=online, mask=None if mask is None else mask[b:e], r=r[b:e], d=d[b:e], gamma=gamma,
               target=y[b:e], stream=torch.cuda.current_stream())

    side_t = {"rd": rd, **({} if mask is None else {"mask": mask})}
    for _ in (1, 2):
        rig.push(obs, side_t, rank, root)
    rig.check()
    return y


@pytest.mark.parametrize("ranks", [2, 3])
@pytest.mark.parametrize("chunk", [None, 256])
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("double", [False, True], ids=["dqn", "double"])
def test_every_form_gives_the_same_bits(K, double, masked, chunk, ranks):
    """Plain, staged, pushed and split calls, at the shipped chunk and at 256-row chunks."""
    M = ranks * 640
    obs, t, o, legal, r, d = _case(M, 18, d_in=128, seed=13)
    kw = dict(online=o if double else None, mask=legal if masked else None)
    with tuning(chunk):
        plain = _fused(obs, t, r=r, d=d, **kw)
        staged = _fused(obs, t, r=r, d=d, staged=True, **kw)
        split = torch.cat([_fused(obs[b:e], t, online=kw["online"], mask=None if not masked else legal[b:e], r=r[b:e],
                                  d=d[b:e]) for b, e in ((0, 384), (384, 1000), (1000, M))])
        pushed = _push_call(K, obs, t, kw["online"], kw["mask"], r, d, chunk or 16896, ranks)
    same(plain, _composed(obs, t, r=r, d=d, **kw), "composed")
    for what, got in (("staged", staged), ("split", split), ("pushed", pushed)):
        same(got, plain, what)


@pytest.mark.parametrize("M", [1003, 2, 0])
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
def test_pull_scatter_gather_over_uneven_and_empty_shards(K, masked, M):
    obs, t, o, legal, r, d = _case(M, 18, seed=14)
    mask = legal if masked else None
    got = mlp.mlp_scatter_gather(obs, t[0], t[2], t[4], [0, 0, 0, 0], biases=(t[1], t[3], t[5]), output="dqn_target",
                                 online=o, mask=mask, reward=r, done=d, gamma=0.99)
    torch.cuda.synchronize()
    same(torch.cat(got), _fused(obs, t, online=o, mask=mask, r=r, d=d), M)


@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("double", [False, True], ids=["dqn", "double"])
def test_package_push_path_on_one_gpu_matches_plain_bits(K, double, masked):
    """mlp_scatter_gather's pushed form (the rows, the mask and the (reward, done) pairs pushed into each staging half,
    the root's shard on the side stream) with ranks [0, 0, 0] on cuda:0, back to back with fresh inputs."""
    devs, M, d_in = [0, 0, 0], 3 * 1280, 128
    bounds = [K.shard_bounds(M, 3, k) for k in range(3)]
    _, t, o, _, _, _ = _case(16, 18, d_in=d_in, seed=15)
    weights = {0: (t[0], t[2], t[4], t[1], t[3], t[5])}
    for it in range(3):
        obs, _, _, legal, r, d = _case(M, 18, d_in=d_in, seed=20 + it)
        mask = legal if masked else None
        want = _fused(obs, t, online=o if double else None, mask=mask, r=r, d=d)
        y = torch.full((M,), 7.0, device="cuda")
        mlp._mlp_scatter_gather_pushed(obs, devs, bounds, weights, "dqn_target", y, None, None, mask=mask,
                                       td=({0: o} if double else None, None, r, d, 0.99, None))
        torch.cuda.synchronize()
        same(y, want, (double, masked, it))
    mlp._push_sessions[tuple(devs)].check()


@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("double", [False, True], ids=["dqn", "double"])
def test_y_and_scratch_stay_inside_their_bytes(K, double, masked):
    M, d_h = 700, 256
    obs, t, o, legal, r, d = _case(M, 18, d_h=d_h, seed=16)
    kw = dict(online=o if double else None, mask=legal if masked else None, r=r, d=d)
    want = _fused(obs, t, **kw)
    y = Guarded(4 * M, 4)
    with tuning(256):   # the scratch as documented for 256-row chunks: the actions end at the band
        nbytes = L.load().ktb_mlp_dqn_target_scratch_bytes(M, d_h)
        assert nbytes == 2 * 256 * d_h * 2 + 256 * 8
        scratch = Guarded(nbytes)
        stage = Guarded(L.load().ktb_mlp_stage_bytes(M, obs.shape[1]))
        with mock.patch.object(mlp, "_cached_buffer", lambda cache, key, dev, n: scratch.view()), \
                mock.patch.object(mlp, "_stage_for", lambda dev, m, d_in: stage.view()):
            _fused(obs, t, target=y.view(torch.float32), staged=True, **kw)
    y.check("y")
    scratch.check("scratch (hidden activations and actions)")
    stage.check("stage")
    same(y.view(torch.float32), want, "guarded")


def test_scratch_size_function(K):
    lib = L.load()
    assert lib.ktb_mlp_dqn_target_scratch_bytes(0, 256) == 0
    assert lib.ktb_mlp_dqn_target_scratch_bytes(100, 1024) == 100 * (4 * 1024 + 8)
    assert lib.ktb_mlp_dqn_target_scratch_bytes(1 << 20, 512) == 16896 * (4 * 512 + 8)


# ---- statuses -----------------------------------------------------------------------------------------------------------
_PTRS = dict(obs=0, w1=0, b1=0, w2=0, b2=0, w3=0, b3=0, mask=0, r=4096, d=8192, y=12288, scratch=1 << 20, stage=0)


def _status_call(masked=False, pushed=False, **over):
    """(args, buffers kept alive) over zero buffers: 256 rows, d_in 256, d_hidden 256, d_out 18, Double DQN with the
    online network on the same zero weights.  `<ptr>_ptr=k` moves a pointer k bytes, `<ptr>=0` makes it null, anything
    else replaces the argument."""
    z = torch.zeros(1 << 22, dtype=torch.uint8, device="cuda")
    ctrl = torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda")
    a = {k: z.data_ptr() + v for k, v in _PTRS.items()}
    a.update(M=256, d_in=256, d_hidden=256, d_out=18, m_off=1 << 17, rd_off=(1 << 17) + 8192, stride=1 << 20,
             gamma=0.99, o_w1=a["w1"], o_w2=a["w2"], o_b1=a["b1"])
    for k, v in over.items():
        if k.endswith("_ptr"):
            a[k[:-4]] += v
        else:
            a[k] = v
    w = [a[k] for k in ("w1", "b1", "w2", "b2", "w3", "b3")]
    on = [a["o_w1"], a["o_b1"], a["o_w2"], a["b2"], a["w3"], a["b3"]]
    body = (a["M"], a["d_in"], a["d_hidden"], a["d_out"], *w, *on)
    entry = "ktb_mlp_bf16_dqn_target" + ("_masked" if masked else "")
    if pushed:
        return (entry + "_pushed", 0, a["stage"], a["stride"], *body, *((a["m_off"],) if masked else ()), a["rd_off"],
                a["gamma"], a["y"], a["scratch"], ctrl.data_ptr(), ctrl.data_ptr(), 1, 256, 1, stream()), (z, ctrl)
    return (entry, 0, a["obs"], *body, *((a["mask"],) if masked else ()), a["r"], a["d"], a["gamma"], a["y"],
            a["scratch"], 0, stream()), (z, ctrl)


STATUS_CASES = [   # in the entries' check order
    ("d_in", dict(d_in=100), L.ERR_ARG), ("d_hidden", dict(d_hidden=300), L.ERR_ARG),
    ("d_out_0", dict(d_out=0), L.ERR_ARG), ("d_out_257", dict(d_out=257), L.ERR_UNSUPPORTED),
    ("bias_align", dict(b1_ptr=1), L.ERR_ARG), ("w1_align", dict(w1_ptr=8), L.ERR_ARG),
    ("scratch_null", dict(scratch=0), L.ERR_ARG),
    ("d_out_before_online", dict(d_out=257, o_w1=0), L.ERR_UNSUPPORTED),
    ("online_partial", dict(o_w1=0), L.ERR_ARG), ("online_w2_null", dict(o_w2=0), L.ERR_ARG),
    ("online_align", dict(o_w1_ptr=8), L.ERR_ARG), ("online_bias_align", dict(o_b1_ptr=1), L.ERR_ARG),
    ("online_before_gamma", dict(o_w1=0, gamma=math.nan), L.ERR_ARG),
    ("gamma_nan", dict(gamma=math.nan), L.ERR_ARG), ("gamma_inf", dict(gamma=-math.inf), L.ERR_ARG),
    ("gamma_before_y", dict(gamma=math.inf, y=0), L.ERR_ARG),
    ("y_null", dict(y=0), L.ERR_ARG), ("y_align", dict(y_ptr=2), L.ERR_ARG),
    ("reward_null", dict(r=0), L.ERR_ARG), ("done_align", dict(d_ptr=1), L.ERR_ARG),
]


@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("case,over,status", STATUS_CASES, ids=[c[0] for c in STATUS_CASES])
def test_plain_entry_statuses(K, masked, case, over, status):
    args, keep = _status_call(masked, **over)
    expect_status(args, status)


def test_masked_entry_mask_comes_after_the_unmasked_checks(K):
    expect_status(_status_call(True, mask=0)[0], L.ERR_ARG)
    expect_status(_status_call(True, mask=0, d_out=257)[0], L.ERR_UNSUPPORTED)


def test_mask_is_checked_before_the_online_network(K):
    """A null mask is a check of ktb_mlp_bf16_policy_masked, so it is reported before the online network's defects."""
    args, keep = _status_call(True, mask=0, o_w1=0)
    with pytest.raises(L.KtbError) as e:
        L.call(*args)
    assert e.value.status == L.ERR_ARG and "null mask" in str(e.value), str(e.value)


@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("case,over,status", [
    ("rd_overlaps_rows", dict(rd_off=256 * 256 * 2 - 8), L.ERR_ARG),
    ("rd_past_stride", dict(rd_off=(1 << 20) - 8), L.ERR_ARG),
    ("rd_align", dict(rd_off=(1 << 17) + 8192 + 4), L.ERR_ARG),
    ("rd_first", dict(gamma=math.nan, rd_off=4), L.ERR_ARG),
], ids=lambda x: x if isinstance(x, str) else "")
def test_pushed_entry_statuses(K, masked, case, over, status):
    args, keep = _status_call(masked, pushed=True, **over)
    expect_status(args, status)


def test_pushed_mask_and_rd_must_not_overlap(K):
    expect_status(_status_call(True, pushed=True, rd_off=(1 << 17) + 8)[0], L.ERR_ARG)


@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
def test_empty_pushed_shard_with_null_outputs_acks(K, masked):
    args, (z, ctrl) = _status_call(masked, pushed=True, M=0, y=0)
    L.call(*args)
    torch.cuda.synchronize()
    assert int(ctrl.count_nonzero()) > 0   # ack[1] = 1 published in the (root's) control block


# ---- weights updated in place -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["forward", "scatter_gather"])
def test_a_hard_target_update_reaches_the_next_call(K, devices):
    obs, t, o, legal, r, d = _case(512, 18, seed=17)

    def call():
        if len(devices) == 1:
            return _fused(obs, t, online=o, mask=legal, r=r, d=d)
        return torch.cat(mlp.mlp_scatter_gather(obs, t[0], t[2], t[4], devices, biases=(t[1], t[3], t[5]),
                                                output="dqn_target", online=o, mask=legal, reward=r, done=d,
                                                gamma=0.99))

    before = call()
    with torch.no_grad():
        for dst, src in zip(t, o):   # target ← online, the hard update of DQN
            dst.copy_(src)
    after = call()
    torch.cuda.synchronize()
    assert not torch.equal(before.cpu(), after.cpu())
    same(after, _composed(obs, t, online=o, mask=legal, r=r, d=d), "after the update")


# ---- the public API -----------------------------------------------------------------------------------------------------
BODIES = {
    "dqn": (mlp_dqn_target, dict()),
    "dqn_masked": (mlp_dqn_target_masked, dict(mask="legal")),
    "double": (mlp_double_dqn_target, dict(online=("o1", "ob1", "o2", "ob2", "o3", "ob3"))),
    "double_masked": (mlp_double_dqn_target_masked, dict(online=("o1", "ob1", "o2", "ob2", "o3", "ob3"),
                                                         mask="legal")),
}


def _public(name, M=1003, seed=21):
    obs, t, o, legal, r, d = _case(M, 18, d_in=128, d_h=512, seed=seed, device="cpu")
    args = (obs, *t, *(o if "double" in name else ()), *((legal,) if "masked" in name else ()), r, d)
    return args, (obs, t, o if "double" in name else None, legal if "masked" in name else None, r, d)


def _mine(parts):
    """mlp_forward over all rows of the public case, on cuda:0."""
    obs, t, o, legal, r, d = parts
    cuda = lambda x: None if x is None else x.cuda()   # noqa: E731
    return _fused(cuda(obs), tuple(cuda(w) for w in t), online=None if o is None else tuple(cuda(w) for w in o),
                  mask=cuda(legal), r=cuda(r), d=cuda(d))


def _close_where_the_actions_agree(got, want):
    """The body runs bf16 GEMMs on the CPU, whose fp32 sums round differently: where a rounding moves the argmax of a
    near tie the rows score a different column, so most rows must be close and every finite one within a wide bar."""
    got, want = got.cpu(), want.cpu()
    close = torch.isclose(got, want, rtol=2.0 ** -7, atol=1e-2, equal_nan=True)
    assert float(close.float().mean()) > 0.97


@pytest.mark.parametrize("name", list(BODIES))
@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["1_rank", "3_ranks"])
def test_mapped_target_through_public_api(K, devices, name):
    import kubetorch_b200 as kt

    body, opts = BODIES[name]
    args, parts = _public(name)
    n = len(devices)
    fn = kt.mapped("mlp", bias=True, output="dqn_target", reward="r", done="d", gamma=0.99, **opts)(body)
    want = ref_dispatch.spmd_call(body, *args, num_proc=n, serialization="pickle")
    mine = _mine(parts)
    gpu = [a.cuda() for a in args]
    with deployed(fn, f"t-dqn-{name}-{n}", devices) as remote:
        got = remote(*gpu, serialization="pickle")
        torch.cuda.synchronize()
    assert len(got) == len(want) == n
    for k, g in enumerate(got):
        lo, hi = K.shard_bounds(args[0].shape[0], n, k)
        same(g.cuda(), mine[lo:hi], k)
        _close_where_the_actions_agree(g, want[k])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("transfer", ["pull", "push"])
@pytest.mark.parametrize("name", ["dqn_masked", "double_masked"])
def test_mapped_target_on_two_gpus(K, name, transfer):
    """Two ranks on two GPUs, staged pull and pushed form, three calls with fresh inputs: the bits of one plain call,
    and the oracle's values."""
    import kubetorch_b200 as kt

    body, opts = BODIES[name]
    fn = kt.mapped("mlp", bias=True, output="dqn_target", reward="r", done="d", gamma=0.99, **opts)(body)
    with deployed(fn, f"t-dqn-2gpu-{name}-{transfer}", [0, 1], transfer=transfer) as remote:
        for it in range(3):
            args, parts = _public(name, M=2 * 1408, seed=30 + it)
            got = remote(*[a.cuda() for a in args], serialization="pickle")
            torch.cuda.synchronize(0)
            torch.cuda.synchronize(1)
            same(torch.cat([g.cpu() for g in got]), _mine(parts), (it, transfer))
            want = ref_dispatch.spmd_call(body, *args, num_proc=2, serialization="pickle")
            _close_where_the_actions_agree(torch.cat([g.cpu() for g in got]), torch.cat(want))
