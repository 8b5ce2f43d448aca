"""-m gpu: the value head of the sampled MLP policies (ktb_mlp_bf16_policy_sample_value*, _sample_masked_value*,
_gaussian_value*, value= of mlp_forward, mlp_scatter_gather and kt.mapped) — values bit for bit against column d_out of
the greedy kernel's logits over the stacked head, actions and log-probabilities bit for bit against the entries without
a value head, with and without a mask, in every form, chunking and row split; guard bands, status codes, the Python
checks, in-place weight updates, the public API and two GPUs."""
import os

import pytest
import torch

from conftest import mapped_copy
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp
from mlp_rig import (SHIPPED_CHUNK, Head, K, config, deployed, expect_status, plain, policy_weights,  # noqa: F401
                     pushed, randn, run_guarded, tuning)

pytestmark = pytest.mark.gpu

import policy_value_cases  # noqa: E402
from oracle import ref_dispatch  # noqa: E402

from kubetorch_b200.sampling import normal_noise  # noqa: E402

WIDTHS = [1, 2, 7, 18, 63, 64, 127, 128, 200, 255]
SAMPLE_VALUE = Head("ktb_mlp_bf16_policy_sample_value", "ktb_mlp_bf16_policy_sample_value",
                    "ktb_mlp_bf16_policy_sample_value_pushed", True, 0,
                    {"actions": lambda d: 8, "log_probs": lambda d: 4, "values": lambda d: 4},
                    lambda a: (a["seed"], a["row_base"], a["actions"], a["log_probs"], a["values"]))
MASKED_SAMPLE_VALUE = Head("ktb_mlp_bf16_policy_sample_masked_value", "ktb_mlp_bf16_policy_sample_masked_value",
                           "ktb_mlp_bf16_policy_sample_masked_value_pushed", True, 0,
                           {"actions": lambda d: 8, "log_probs": lambda d: 4, "values": lambda d: 4},
                           lambda a: (a["mask"], a["seed"], a["row_base"], a["actions"], a["log_probs"], a["values"]))
GAUSSIAN_VALUE = Head("ktb_mlp_bf16_policy_gaussian_value", "ktb_mlp_bf16_policy_gaussian_value",
                      "ktb_mlp_bf16_policy_gaussian_value_pushed", True, 0,
                      {"actions": lambda d: 4 * d, "log_probs": lambda d: 4, "values": lambda d: 4},
                      lambda a: (a["log_std"], a["seed"], a["row_base"], a["actions"], a["log_probs"], a["values"]))
KINDS = ("sample", "masked", "gaussian")


# ---- inputs -------------------------------------------------------------------------------------------------------------
def actor_critic(seed, d_out, bias=True):
    """(W1, W2, W3), (b1, b2, b3) of mlp_rig.config and a critic (wv [1, 1024], bv [1] or None without biases)."""
    w, b = config(seed, d_out, bias)
    return w, b, (randn((1, 1024), seed + 6, 0.02), randn((1,), seed + 7, 0.1) if bias else None)


def stacked(w, b, value):
    """W3v = [w3; wv] and b3v = [b3; bv] (None without biases)."""
    return torch.cat((w[2], value[0])), None if b[2] is None else torch.cat((b[2], value[1]))


def rig_weights(w, b, value):
    """(w, b) for the rig's named arguments with the head replaced by views of the first d_out rows of the stacked
    head: the rig then passes the policy's d_out and the stacked head's address."""
    w3v, b3v = stacked(w, b, value)
    d_out = w[2].shape[0]
    return (w[0], w[1], w3v[:d_out]), (b[0], b[1], None if b3v is None else b3v[:d_out])


def random_legal(M, d_out, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    legal = torch.rand(M, d_out, generator=g, device="cuda") < 0.5
    legal[::61] = False   # rows with no legal action
    return legal


def bits(t):
    """The bit patterns of a 16- or 32-bit float tensor; other tensors as they are."""
    if not t.is_floating_point():
        return t
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def same(got, want, what):
    assert len(got) == len(want), what
    for i, (g, h) in enumerate(zip(got, want)):
        assert torch.equal(bits(g), bits(h)), (what, i)


def kind_args(kind, M, d_out, seed):
    """The mlp_forward arguments of a head kind (output, mask or log_std, seed)."""
    if kind == "gaussian":
        return dict(output="gaussian", seed=seed, log_std=torch.linspace(-2, 0.5, d_out, device="cuda"))
    kw = dict(output="sample", seed=seed)
    if kind == "masked":
        kw["mask"] = random_legal(M, d_out, seed + 1)
    return kw


def forward(obs, w, b, **kw):
    return mlp.mlp_forward(obs, *w, biases=b, **kw)


# ---- 1. bit for bit in every form ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("bias", [True, False], ids=["biased", "bias_free"])
@pytest.mark.parametrize("d_out", WIDTHS)
def test_values_and_draws_are_exact_in_every_form(K, d_out, bias):
    """Values are column d_out of ktb_mlp_bf16_policy's logits over the stacked head, widened to fp32, bit for bit;
    the actions and log-probabilities of every value entry are those of the entry without a value head (also at d_out
    64 and 128, where the value column moves the head into the next tile width); a mask leaves the values alone; and
    the plain form at the shipped and 256-row chunks, the staged form (pull kernel and copy engine), row splits with
    row_offset and the package's pushed form on ranks [0, 0, 0] all give the same bits."""
    M, seed = 3 * 1408, 2**34 + 7 * d_out
    w, b, value = actor_critic(2000 + d_out, d_out, bias)
    obs = randn((M, 256), 2010 + d_out)
    w3v, b3v = stacked(w, b, value)
    y = mlp.mlp_forward(obs, w[0], w[1], w3v, biases=(b[0], b[1], b3v))
    want_values = y[:, d_out].float()
    results = {}
    for kind in KINDS:
        kw = kind_args(kind, M, d_out, seed)
        want = forward(obs, w, b, **kw)
        got = forward(obs, w, b, value=value, **kw)
        assert len(got) == 3 and got[2].dtype == torch.float32 and got[2].shape == (M,), kind
        same(got[:2], want, (kind, "draws"))
        assert torch.equal(bits(got[2]), bits(want_values)), (kind, "values")
        for chunk in (256, SHIPPED_CHUNK):
            for ce in (None, 0, 1):
                with tuning(chunk, ce):
                    same(forward(obs, w, b, value=value, staged=ce is not None, **kw), got, (kind, chunk, ce))
        for split in (1, 1000, 2 * 1408 + 5):
            lo_kw, hi_kw = dict(kw), dict(kw)
            if "mask" in kw:
                lo_kw["mask"], hi_kw["mask"] = kw["mask"][:split], kw["mask"][split:]
            lo = forward(obs[:split], w, b, value=value, **lo_kw)
            hi = forward(obs[split:], w, b, value=value, row_offset=split, **hi_kw)
            same([torch.cat([p, q]) for p, q in zip(lo, hi)], got, (kind, "split", split))
        devs = [0, 0, 0]
        bounds = [K.shard_bounds(M, 3, r) for r in range(3)]
        weights = {0: (w[0], w[1], w3v, b[0], b[1], b3v)}
        gaussian = kind == "gaussian"
        actions = torch.full((M, d_out) if gaussian else (M,), -1, dtype=torch.float32 if gaussian else torch.int64,
                             device="cuda")
        log_probs, values = (torch.full((M,), -1.0, device="cuda") for _ in range(2))
        mlp._mlp_scatter_gather_pushed(obs, devs, bounds, weights, kw["output"], None, actions, log_probs, seed,
                                       {0: kw["log_std"]} if gaussian else None, kw.get("mask"), values)
        torch.cuda.synchronize()
        same((actions, log_probs, values), got, (kind, "pushed"))
        results[kind] = got
    assert torch.equal(bits(results["masked"][2]), bits(results["sample"][2]))


# ---- 2. guard bands ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("head", [SAMPLE_VALUE, GAUSSIAN_VALUE], ids=["sample", "gaussian"])
@pytest.mark.parametrize("form,M,chunk,d_out", [
    ("plain", 1000, SHIPPED_CHUNK, 7), ("plain", 1000, 256, 18), ("plain", 1000, 256, 255),
    ("staged", 1408, 256, 63), ("staged", 1408, 256, 64),
    ("pushed", 3 * 1408, 256, 7), ("pushed", 3 * 1408, 256, 128),
])
def test_writes_stay_inside_the_outputs(K, head, form, M, chunk, d_out):
    """Every output (values included), the scratch and the stage between guard bands, at odd and even d_out (the
    Gaussian actions [M, d_out] as float2 pairs, and at d_out 64 four bytes past an 8-byte boundary, as scalars); the
    results equal mlp_forward's bit for bit."""
    seed = 6
    w, b, value = actor_critic(2100 + d_out, d_out)
    obs = randn((M, 256), 2101)
    kind = "gaussian" if head is GAUSSIAN_VALUE else "sample"
    kw = kind_args(kind, M, d_out, seed)
    want = forward(obs, w, b, value=value, **kw)
    rw, rb = rig_weights(w, b, value)
    bufs = run_guarded(form, head, K, chunk, obs, rw, rb, seed, kw.get("log_std"),
                       offsets={"actions": 4} if kind == "gaussian" and d_out == 64 else None)
    for name, buf in bufs.items():
        buf.check(f"{form} M={M} chunk={chunk} d_out={d_out}: {name}")
    dtypes = {"actions": torch.int32 if kind == "gaussian" else torch.int64, "log_probs": torch.int32,
              "values": torch.int32}
    for name, h in zip(("actions", "log_probs", "values"), want):
        assert torch.equal(bufs[name].view(dtypes[name]).view(h.shape), bits(h)), (form, name)


# ---- 3. status codes ----------------------------------------------------------------------------------------------------
_BUFS = {}


def _buf(name, n, dtype=torch.float32):
    if name not in _BUFS:
        _BUFS[name] = torch.zeros(n, dtype=dtype, device="cuda")
    return _BUFS[name].data_ptr()


ROWS_BYTES = 256 * 256 * 2      # the status cases' M * d_in * 2: where a pushed mask may begin
STATUS_CASES = {
    "null_values": (plain, dict(values=0), L.ERR_ARG),
    "values_2_bytes_in": (plain, dict(values=2), L.ERR_ARG),
    "d_out_256": (plain, dict(d_out=256), L.ERR_UNSUPPORTED),
    "staged_null_values": (plain, dict(values=0, stage="stage"), L.ERR_ARG),
    "inherited_checks_first": (plain, dict(values=0, d_out=257), L.ERR_UNSUPPORTED),
    "inherited_d_in": (plain, dict(d_in=100), L.ERR_ARG),
    "pushed_null_values": (pushed, dict(values=0), L.ERR_ARG),
    "pushed_values_2_bytes_in": (pushed, dict(values=2), L.ERR_ARG),
    "pushed_d_out_256": (pushed, dict(d_out=256), L.ERR_UNSUPPORTED),
    "pushed_inherited_checks_first": (pushed, dict(values=0, d_out=257), L.ERR_UNSUPPORTED),
    "pushed_inherited_seq": (pushed, dict(seq=0), L.ERR_ARG),
    "pushed_inherited_stride": (pushed, dict(stride=(1 << 20) + 8), L.ERR_ARG),
}
MASKED_CASES = {
    "null_mask": (plain, dict(mask=0), L.ERR_ARG),
    "null_mask_before_null_values": (plain, dict(mask=0, values=0, d_out=256), L.ERR_ARG),
    "pushed_mask_offset_over_the_rows": (pushed, dict(mask=ROWS_BYTES - 1), L.ERR_ARG),
    "pushed_mask_past_stage_stride": (pushed, dict(mask=(1 << 20) - 256 * 18 + 1), L.ERR_ARG),
}
HEADS = {"sample": SAMPLE_VALUE, "masked": MASKED_SAMPLE_VALUE, "gaussian": GAUSSIAN_VALUE}


def _status_overrides(form, overrides):
    o = dict(overrides)
    values = _buf("values", 4096)
    o["values"] = values + o["values"] if o.get("values", 0) else o.get("values", values)
    if o.get("stage") == "stage":
        o["stage"] = _buf("stage", 1 << 22, torch.uint8)
    if "mask" not in o:
        o["mask"] = ROWS_BYTES if form is pushed else _buf("mask", 2048 * 512, torch.uint8)
    return o


@pytest.mark.parametrize("head,name", [(h, n) for n in STATUS_CASES for h in HEADS] +
                         [("masked", n) for n in MASKED_CASES])
def test_bad_arguments_get_the_documented_status(K, head, name):
    form, overrides, status = {**STATUS_CASES, **MASKED_CASES}[name]
    expect_status(form(HEADS[head], **_status_overrides(form, overrides)), status)


@pytest.mark.parametrize("head", list(HEADS))
def test_empty_pushed_shard_runs_its_checks_and_acks(K, head):
    """An empty shard (M = 0) with null outputs publishes ack[rank] = seq in the root's control block; with a bad
    argument it returns the status of the entry without a value head."""
    ctrl_root = torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda")
    args = pushed(HEADS[head], M=0, actions=0, log_probs=0, values=0, ctrl_root=ctrl_root.data_ptr(), seq=3, rank=2,
                  mask=0)
    L.call(*args)
    torch.cuda.synchronize()
    assert int(ctrl_root[512 + 8 * 2:512 + 8 * 3].view(torch.int64)) == 3
    expect_status(pushed(HEADS[head], M=0, actions=0, log_probs=0, values=0, mask=0, seq=0), L.ERR_ARG)


# ---- 4. Python checks ---------------------------------------------------------------------------------------------------
def test_python_checks_name_the_output_in_mlp_forward_and_scatter_gather(K):
    (w1, w2, w3), b = config(2200, 18)
    obs = randn((256, 256), 2201)
    wv, bv = randn((1, 1024), 2202), randn((1,), 2203)
    log_std = torch.zeros(18, device="cuda")
    bad = [
        ("actions", {}, b, (wv, bv), 'value is not an argument of output="actions"'),
        ("both", {}, b, (wv, bv), 'value is not an argument of output="both"'),
        ("logits", {}, b, (wv, bv), 'value is not an argument of output="logits"'),
        ("sample", dict(seed=1), b, (wv,), "value must be"),
        ("sample", dict(seed=1), b, (wv, None), "bv is given exactly when b3 is"),
        ("gaussian", dict(seed=1, log_std=log_std), (b[0], b[1], None), (wv, bv), "bv is given exactly when b3 is"),
        ("sample", dict(seed=1), b, (randn((2, 1024), 1), bv), "shape"),
        ("sample", dict(seed=1), b, (randn((1, 512), 1), bv), "shape"),
        ("sample", dict(seed=1), b, (wv.float(), bv), "bfloat16"),
        ("sample", dict(seed=1), b, (randn((1024, 2), 1)[:, :1].t(), bv), "contiguous"),
        ("sample", dict(seed=1), b, (wv.cpu(), bv), "CUDA"),
        ("gaussian", dict(seed=1, log_std=log_std), b, (wv, bv.cpu()), "bv must be"),
        ("sample", dict(seed=1), b, (wv, bv.float()), "bv must be"),
    ]
    for output, kw, biases, value, reason in bad:
        with pytest.raises(ValueError, match=reason):
            mlp.mlp_forward(obs, w1, w2, w3, biases=biases, output=output, value=value, **kw)
        with pytest.raises(ValueError, match=reason):
            mlp.mlp_scatter_gather(obs, w1, w2, w3, devices=[0], biases=biases, output=output, value=value, **kw)
    (w1, w2, w3), b = config(2210, 256)
    for fn, extra in ((mlp.mlp_forward, {}), (mlp.mlp_scatter_gather, dict(devices=[0]))):
        with pytest.raises(ValueError, match="d_out=256"):
            fn(obs, w1, w2, w3, biases=b, output="sample", seed=1, value=(wv, bv), **extra)


# ---- 5. in-place updates --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_in_place_weight_updates_reach_the_next_call(K, kind):
    """After wv.add_(...), and again after w3.add_(...) and bv.add_(...), the next call's values and draws equal a
    fresh call's (fresh tensors, so a new stacked head); the stacked-head cache keeps one entry for the head."""
    d_out, M, seed = 18, 2048, 31
    w, b, value = actor_critic(2300, d_out)
    w, b, value = list(w), list(b), list(value)
    obs = randn((M, 256), 2301)
    kw = kind_args(kind, M, d_out, seed)
    forward(obs, w, b, value=value, **kw)
    entries = len(mlp._stacked_heads)
    for t in (value[0], w[2], value[1], b[2]):
        t.add_(0.25)
        got = forward(obs, w, b, value=value, **kw)
        fresh = forward(obs, [t.clone() for t in w], [t.clone() for t in b], value=[t.clone() for t in value], **kw)
        same(got, fresh, kind)
        assert len(mlp._stacked_heads) <= entries + 1   # at most the fresh call's own head beside this one
    assert len(mlp._stacked_heads) <= entries + 1


# ---- 6. the public API ----------------------------------------------------------------------------------------------------
def _public_case(golden, kind):
    obs = torch.randn(1000, 256, generator=torch.Generator().manual_seed(1000)).bfloat16()
    d_out = 6
    p = policy_weights(golden, d_out)
    g = torch.Generator().manual_seed(77)
    value = ((torch.randn(1, 1024, generator=g) * 0.02).bfloat16(), (torch.randn(1, generator=g) * 0.1).bfloat16())
    seed = 2**35 + 23
    if kind == "sample":
        body, extra, middle = policy_value_cases.mlp_policy_sample_value, {}, ()
    elif kind == "masked":
        legal = torch.rand(obs.shape[0], d_out, generator=g) < 0.5
        legal[::50] = False
        body, extra, middle = policy_value_cases.mlp_policy_masked_sample_value, dict(mask="legal"), (legal,)
    else:
        body, extra, middle = (policy_value_cases.mlp_policy_gaussian_value, dict(log_std="log_std"),
                               (torch.linspace(-3, 1, d_out),))
    output = "gaussian" if kind == "gaussian" else "sample"
    policy = mapped_copy(body, "mlp", bias=True, output=output, seed="seed", value=("wv", "bv"), **extra)
    return obs, p, value, seed, body, middle, policy, output


def _mine(obs, p, value, seed, middle, kind, with_value=True):
    """mlp_forward over all rows on cuda:0."""
    pc = [t.cuda() for t in p]
    kw = dict(output="gaussian" if kind == "gaussian" else "sample", seed=seed)
    if kind == "masked":
        kw["mask"] = middle[0].cuda()
    if kind == "gaussian":
        kw["log_std"] = middle[0].cuda()
    if with_value:
        kw["value"] = tuple(t.cuda() for t in value)
    return mlp.mlp_forward(obs.cuda(), pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]), **kw)


@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["1_rank", "3_ranks"])
@pytest.mark.parametrize("kind", KINDS)
def test_mapped_value_through_public_api(K, golden, kind, devices):
    """@kt.mapped("mlp", bias=True, output=..., seed="seed", value=("wv", "bv")) on Compute(gpus=1): each rank returns
    (actions, log_probs, values) with the bits of mlp_forward over its rows (actions and log-probabilities also those
    of the call without a value head), and against the oracle's run of the body the values agree within rtol 2^-7,
    atol 1e-2, the sampled actions on at least 99 % of the rows and the Gaussian actions within their bar wherever the
    body's bf16 logits equal the kernel's."""
    from unittest import mock

    from policy_value_cases import _trunk

    obs, p, value, seed, body, middle, policy, output = _public_case(golden, kind)
    n = len(devices)
    want = ref_dispatch.spmd_call(body, obs, *p, *middle, *value, seed, num_proc=n, serialization="pickle")
    mine = _mine(obs, p, value, seed, middle, kind)
    plain_draws = _mine(obs, p, value, seed, middle, kind, with_value=False)
    same(mine[:2], plain_draws, kind)
    with deployed(policy, f"t-value-{kind}-{n}", devices) as remote:
        got = remote(obs.cuda(), *[t.cuda() for t in p], *[t.cuda() for t in middle], *[t.cuda() for t in value],
                     seed, serialization="pickle")
        torch.cuda.synchronize()
    assert len(got) == len(want) == n
    agree, total = 0, 0
    for r, (g, h) in enumerate(zip(got, want)):
        lo, hi = K.shard_bounds(obs.shape[0], n, r)
        assert isinstance(g, tuple) and len(g) == 3, (kind, r)
        same([t.cpu() for t in g], [t[lo:hi].cpu() for t in mine], (kind, r))
        assert torch.allclose(g[2].cpu(), h[2], rtol=2.0 ** -7, atol=1e-2), (kind, r)
        if kind != "gaussian":
            agree += int((g[0].cpu() == h[0]).sum())
            total += hi - lo
            continue
        with mock.patch.dict(os.environ, {"RANK": str(r), "WORLD_SIZE": str(n)}):
            y_body = torch.nn.functional.linear(_trunk(obs, *p[:4]), p[4], p[5]).float()
        pc = [t.cuda() for t in p]
        y = mlp.mlp_forward(obs[lo:hi].cuda(), pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5])).float().cpu()
        eq = y_body == y
        z = normal_noise(seed, lo, hi - lo, 6).double()
        tol = 2.0 ** -19 * middle[0].double().exp() * (1 + z.abs()) + 2.0 ** -23 * y.double().abs()
        assert bool(((g[0].cpu().double() - h[0].double()).abs() <= tol)[eq].all()), (kind, r)
    if kind != "gaussian":
        assert agree >= 0.99 * total, (agree, total)


def test_mapped_value_on_a_workers_subset(K, golden):
    """Two workers of one rank each on cuda:0; a call with workers=[1] returns rank 1's (actions, log_probs, values)
    only, with the bits of mlp_forward over its rows."""
    import kubetorch_b200 as kt

    obs, p, value, seed, body, middle, policy, output = _public_case(golden, "sample")
    mine = _mine(obs, p, value, seed, middle, "sample")
    remote = kt.fn(policy, name="t-value-workers").to(
        kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute("b200", workers=2, num_proc=1,
                                                                                 devices=[0, 0]))
    try:
        got = remote(obs.cuda(), *[t.cuda() for t in p], *[t.cuda() for t in value], seed, serialization="pickle",
                     workers=[1])
        torch.cuda.synchronize()
    finally:
        remote.teardown()
    lo, hi = K.shard_bounds(obs.shape[0], 2, 1)
    assert len(got) == 1
    same([t.cpu() for t in got[0]], [t[lo:hi].cpu() for t in mine], "workers=[1]")


# ---- 7. two GPUs ----------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("transfer", ["pull", "push"])
@pytest.mark.parametrize("kind", KINDS)
def test_mapped_value_on_two_gpus(K, golden, kind, transfer):
    """Two ranks on two GPUs, staged pull and pushed form (the stacked head copied to cuda:1), three back-to-back
    calls with fresh observations, the critic updated in place before the last: the bits of one plain call."""
    obs, p, value, seed, body, middle, policy, output = _public_case(golden, kind)
    with deployed(policy, f"t-value-2gpu-{kind}-{transfer}", [0, 1], transfer=transfer) as remote:
        pc = [t.cuda(0) for t in p]
        vc = [t.cuda(0) for t in value]
        mc = [t.cuda(0) for t in middle]
        for it in range(3):
            x = torch.randn(2 * 1408, 256, generator=torch.Generator().manual_seed(5 + it)).bfloat16().cuda(0)
            if kind == "masked":
                mc = [(torch.rand(x.shape[0], 6, generator=torch.Generator().manual_seed(9 + it)) < 0.5).cuda(0)]
            if it == 2:
                vc[0].add_(0.125)
            got = remote(x, *pc, *mc, *vc, seed, serialization="pickle")
            torch.cuda.synchronize(0)
            torch.cuda.synchronize(1)
            kw = dict(output=output, seed=seed, value=tuple(vc))
            if kind == "masked":
                kw["mask"] = mc[0]
            if kind == "gaussian":
                kw["log_std"] = mc[0]
            want = mlp.mlp_forward(x, pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]), **kw)
            same([torch.cat([g[k].cpu() for g in got]) for k in range(3)], [t.cpu() for t in want], (kind, it))
