"""-m gpu: the multi-discrete categorical heads (ktb_mlp_bf16_policy_multidiscrete*, _sample_multidiscrete*, nvec= of
mlp_forward, mlp_scatter_gather and kt.mapped) — nvec = (d_out,) bit for bit against the single categorical in every
form, chunking and row split; every group bit for bit against the masked single categorical under the mask legal ∧
(column in the group); the joint distribution of two groups; guard bands, status codes, the Python checks, the public
API and two GPUs."""
import ctypes

import pytest
import torch

from conftest import mapped_copy
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp
from mlp_rig import (SHIPPED_CHUNK, Head, K, config, deployed, expect_status, plain, policy_weights,  # noqa: F401
                     pushed, randn, run_guarded, tuning)

pytestmark = pytest.mark.gpu

import policy_multidiscrete_cases as cases  # noqa: E402
from oracle import ref_dispatch  # noqa: E402

WIDTHS = [1, 2, 7, 18, 63, 64, 127, 128, 200, 255, 256]
# (output, masked, valued) of every multi-discrete entry
KINDS = [("actions", False, False), ("both", False, False), ("sample", False, False), ("actions", True, False),
         ("both", True, False), ("sample", True, False), ("sample", False, True), ("sample", True, True)]


def kind_id(kind):
    output, masked, valued = kind
    return output + ("_masked" if masked else "") + ("_value" if valued else "")


# ---- inputs and comparisons ---------------------------------------------------------------------------------------------
def random_legal(M, d_out, seed, p=0.5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    legal = torch.rand(M, d_out, generator=g, device="cuda") < p
    legal[::61] = False   # rows with no legal action
    return legal


def critic(seed, bias=True):
    return randn((1, 1024), seed, 0.02), randn((1,), seed + 1, 0.1) if bias else None


def bits(t):
    """The bit patterns of a 16- or 32-bit float tensor; other tensors as they are."""
    if not t.is_floating_point():
        return t
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def same(got, want, what):
    assert len(got) == len(want), what
    for i, (g, h) in enumerate(zip(got, want)):
        assert g.shape == h.shape and g.dtype == h.dtype, (what, i, g.shape, h.shape)
        assert torch.equal(bits(g), bits(h)), (what, i)


def same_or_nan(got, want, what):
    """The same bits, or NaN in both (a NaN's sign and payload depend on the order of the operations that made it)."""
    ok = (bits(got) == bits(want)) | (got.isnan() & want.isnan())
    assert bool(ok.all()), (what, int((~ok).sum()))


def kwargs_of(kind, M, d_out, seed, bias=True):
    output, masked, valued = kind
    kw = dict(output=output)
    if output == "sample":
        kw["seed"] = seed
    if masked:
        kw["mask"] = random_legal(M, d_out, seed + 1)
    if valued:
        kw["value"] = critic(seed + 2, bias)
    return kw


def forward(obs, w, b, **kw):
    return mlp.mlp_forward(obs, *w, biases=b, **kw)


def as_tuple(r):
    return r if isinstance(r, tuple) else (r,)


def single_categorical(got, output):
    """The outputs of a grouped call with nvec = (d_out,) laid out as the single categorical's: actions [M]."""
    got = list(as_tuple(got))
    k = 1 if output == "both" else 0
    assert got[k].dim() == 2 and got[k].shape[1] == 1
    got[k] = got[k][:, 0]
    return tuple(got)


# ---- 1. nvec = (d_out,) is the single categorical in every form -----------------------------------------------------------
@pytest.mark.parametrize("bias", [True, False], ids=["biased", "bias_free"])
@pytest.mark.parametrize("d_out", WIDTHS)
def test_one_group_is_the_single_categorical_in_every_form(K, d_out, bias):
    """nvec = (d_out,): every multi-discrete entry gives the bits of its single-categorical counterpart (actions as
    [M, 1], log-probabilities, logits, masked logits, values), and the plain form at the shipped and 256-row chunks,
    the staged form (pull kernel and copy engine), row splits with row_offset and the package's pushed form on ranks
    [0, 0, 0] all give the same bits."""
    M, seed = 3 * 1408, 2**36 + 5 * d_out
    w, b = config(3000 + d_out, d_out, bias)
    obs = randn((M, 256), 3010 + d_out)
    nvec = (d_out,)
    for kind in KINDS:
        output, masked, valued = kind
        if valued and d_out == 256:
            continue
        kw = kwargs_of(kind, M, d_out, seed, bias)
        want = as_tuple(forward(obs, w, b, **kw))
        got = as_tuple(forward(obs, w, b, nvec=nvec, **kw))
        same(single_categorical(got, output), want, (kind, "counterpart"))
        for chunk in (256, SHIPPED_CHUNK):
            for ce in (None, 0, 1):
                with tuning(chunk, ce):
                    same(as_tuple(forward(obs, w, b, nvec=nvec, staged=ce is not None, **kw)), got, (kind, chunk, ce))
        for split in (1, 1000, 2 * 1408 + 5):
            lo_kw, hi_kw = dict(kw), dict(kw)
            if masked:
                lo_kw["mask"], hi_kw["mask"] = kw["mask"][:split], kw["mask"][split:]
            offset = dict(row_offset=split) if output == "sample" else {}
            lo = as_tuple(forward(obs[:split], w, b, nvec=nvec, **lo_kw))
            hi = as_tuple(forward(obs[split:], w, b, nvec=nvec, **hi_kw, **offset))
            same([torch.cat([p, q]) for p, q in zip(lo, hi)], got, (kind, "split", split))
        same(pushed_call(K, obs, w, b, kw, nvec), got, (kind, "pushed"))


def pushed_call(K, obs, w, b, kw, nvec):
    """The package's pushed form on ranks [0, 0, 0] (one device, so every flag wait is already satisfied in order)."""
    M, d_out = obs.shape[0], w[2].shape[0]
    output = kw["output"]
    w3, b3 = w[2], b[2]
    values = None
    if "value" in kw:
        w3, b3 = mlp._stacked_head(w3, b3, *kw["value"])
        values = torch.full((M,), -1.0, device="cuda")
    logits = torch.zeros(M, d_out, dtype=torch.bfloat16, device="cuda") if output == "both" else None
    actions = torch.full((M, len(nvec)), -1, dtype=torch.int64, device="cuda")
    log_probs = torch.full((M,), -1.0, device="cuda") if output == "sample" else None
    bounds = [K.shard_bounds(M, 3, r) for r in range(3)]
    weights = {0: (w[0], w[1], w3, b[0], b[1], b3)}
    mlp._mlp_scatter_gather_pushed(obs, [0, 0, 0], bounds, weights, output, logits, actions, log_probs,
                                   kw.get("seed"), None, kw.get("mask"), values, nvec)
    torch.cuda.synchronize()
    return tuple(t for t in (logits, actions, log_probs, values) if t is not None)


# ---- 2. every group is the masked single categorical ----------------------------------------------------------------------
NVECS = [(3, 1, 2), (1,) * 7, (5, 8, 3, 2), (3,) * 6, (6, 4, 4, 4, 4, 7, 49), (2,) * 32, (127, 1), (129, 70),
         (100, 1, 155), (1,) * 256, (2,) * 128]


def nvec_id(nvec):
    return "-".join(map(str, nvec)) if len(nvec) <= 8 else f"{nvec[0]}x{len(nvec)}"


@pytest.mark.parametrize("masked", [True, False], ids=["masked", "unmasked"])
@pytest.mark.parametrize("nvec", NVECS, ids=nvec_id)
def test_each_group_is_the_masked_single_categorical(K, nvec, masked):
    """Group g's sampled action is ktb_mlp_bf16_policy_sample_masked's action minus lo_g under the mask legal ∧
    (column in group g), and its log-probability that entry's, bit for bit (the same noise, ranked values and
    per-thread order); the row's log-probability is the fp32 sum of those in group order; greedy actions likewise
    against ktb_mlp_bf16_policy_masked, and the logits of "both" are the masked greedy entry's.  A group with no legal
    column takes relative action 0 with a NaN log-probability.  Boundaries inside and on column pairs, groups of one
    and G = d_out."""
    d_out, G, M, seed = sum(nvec), len(nvec), 1408, 2**37 + len(nvec)
    w, b = config(3100 + d_out, d_out)
    obs = randn((M, 256), 3101 + G)
    legal = random_legal(M, d_out, seed) if masked else torch.ones(M, d_out, dtype=torch.bool, device="cuda")
    if masked:
        legal[::7, :nvec[0]] = False   # group 0 without a legal column
    mask = dict(mask=legal) if masked else {}
    acts, lps = mlp.mlp_forward(obs, *w, biases=b, output="sample", seed=seed, nvec=nvec, **mask)
    logits, greedy = mlp.mlp_forward(obs, *w, biases=b, output="both", nvec=nvec, **mask)
    assert acts.shape == greedy.shape == (M, G)
    want_logits, _ = mlp.mlp_forward(obs, *w, biases=b, output="both", mask=legal)
    same([logits], [want_logits], "logits")
    lo, terms = 0, []
    for g, n in enumerate(nvec):
        in_group = torch.zeros(d_out, dtype=torch.bool, device="cuda")
        in_group[lo:lo + n] = True
        sub = legal & in_group
        a, lp = mlp.mlp_forward(obs, *w, biases=b, output="sample", seed=seed, mask=sub)
        ag = mlp.mlp_forward(obs, *w, biases=b, output="actions", mask=sub)
        empty = ~sub.any(-1)
        for got, want in ((acts[:, g], a), (greedy[:, g], ag)):
            want = torch.where(empty, 0, want - lo)
            assert bool(((want >= 0) & (want < n)).all()), g
            assert torch.equal(got, want), (g, int((got != want).sum()))
        assert bool(lp[empty].isnan().all())
        terms.append(lp)
        lo += n
    total = terms[0]
    for t in terms[1:]:
        total = total + t
    same_or_nan(lps, total, "log_probs")
    if masked:
        assert bool(lps[::7].isnan().all())
    else:
        assert not bool(lps.isnan().any())


# ---- 3. the distribution ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
def test_joint_counts_of_two_groups_follow_the_product_of_their_softmaxes(K, masked):
    """2^20 rows of one logit vector, nvec = (3, 5, 8): the joint counts of the actions of groups 0 and 1 pass a
    chi-square test against the product of the two groups' softmaxes (p > 1e-4); under a mask the illegal columns of
    every group are never drawn."""
    from scipy.stats import chisquare

    nvec, M, seed = (3, 5, 8), 1 << 20, 2**38 + 11
    w, b = config(3200, 16)
    w = (w[0], w[1], randn((16, 1024), 3201, 0.05))
    obs = randn((1, 256), 3202).expand(M, 256).contiguous()
    legal = torch.ones(M, 16, dtype=torch.bool, device="cuda")
    if masked:
        legal[:, [1, 4, 6, 9, 10, 15]] = False
    mask = dict(mask=legal) if masked else {}
    y = mlp.mlp_forward(obs[:128], *w, biases=b, output="logits")
    assert bool((y == y[0]).all())
    y = y[0].double().masked_fill(~legal[0], float("-inf"))
    acts, _ = mlp.mlp_forward(obs, *w, biases=b, output="sample", seed=seed, nvec=nvec, **mask)
    lo = 0
    for g, n in enumerate(nvec):
        counts = torch.bincount(acts[:, g], minlength=n).cpu()
        assert counts.shape == (n,) and int(counts.sum()) == M
        assert bool((counts[~legal[0, lo:lo + n].cpu()] == 0).all()), g
        lo += n
    p0, p1 = torch.softmax(y[:3], 0).cpu(), torch.softmax(y[3:8], 0).cpu()
    joint = torch.bincount(acts[:, 0] * 5 + acts[:, 1], minlength=15).cpu().double()
    expected = (p0[:, None] * p1[None, :]).reshape(-1) * M
    live = expected > 0
    assert bool((joint[~live] == 0).all())
    p = chisquare(joint[live].numpy(), expected[live].numpy()).pvalue
    print(f"chi-square p = {p:.4g} over {int(live.sum())} cells")
    assert p > 1e-4, p


# ---- 4. guard bands -----------------------------------------------------------------------------------------------------
def md_head(kind, nvec=None):
    """The multi-discrete Head of kind (output, masked, valued); with nvec its arguments carry that nvec, else the
    named arguments nvec and n_groups."""
    output, masked, valued = kind
    sample = output == "sample"
    name = ("ktb_mlp_bf16_policy_sample_multidiscrete" if sample else "ktb_mlp_bf16_policy_multidiscrete") + \
        ("_masked" if masked else "") + ("_value" if valued else "")
    G = None if nvec is None else len(nvec)
    arr = None if nvec is None else L.arr(ctypes.c_int32, nvec)

    def groups(a):
        return (arr, G) if nvec is not None else (a["nvec"], a["n_groups"])

    mk = (lambda a: (a["mask"],)) if masked else (lambda a: ())
    if sample:
        outputs = {"actions": lambda d: 8 * (G or 1), "log_probs": lambda d: 4}
        if valued:
            outputs["values"] = lambda d: 4
        vl = (lambda a: (a["values"],)) if valued else (lambda a: ())
        args = lambda a: (*groups(a), *mk(a), a["seed"], a["row_base"], a["actions"], a["log_probs"], *vl(a))  # noqa
    else:
        outputs = {"logits": lambda d: 2 * d, "actions": lambda d: 8 * (G or 1)}
        args = lambda a: (*groups(a), *mk(a), a["logits"], a["actions"])   # noqa: E731
    return Head(name, name, name + "_pushed", True, 0, outputs, args)


@pytest.mark.parametrize("output", ["both", "sample"])
@pytest.mark.parametrize("form,M,chunk,nvec", [
    ("plain", 1000, SHIPPED_CHUNK, (3, 1, 2, 1)), ("plain", 1000, 256, (6, 4, 4, 4, 4, 7, 49)),
    ("plain", 1000, 256, (1,) * 256), ("staged", 1408, 256, (2,) * 32), ("staged", 1408, 256, (63,)),
    ("pushed", 3 * 1408, 256, (3, 4)), ("pushed", 3 * 1408, 256, (100, 1, 155)),
], ids=lambda v: nvec_id(v) if isinstance(v, tuple) else str(v))
def test_writes_stay_inside_the_outputs(K, output, form, M, chunk, nvec):
    """Every output (actions [M, G]), the scratch and the stage between guard bands, at odd and even d_out; the
    results equal mlp_forward's bit for bit."""
    seed, d_out = 9, sum(nvec)
    w, b = config(3300 + d_out, d_out)
    obs = randn((M, 256), 3301)
    want = as_tuple(forward(obs, w, b, output=output, nvec=nvec, **(dict(seed=seed) if output == "sample" else {})))
    bufs = run_guarded(form, md_head((output, False, False), nvec), K, chunk, obs, w, b, seed)
    for name, buf in bufs.items():
        buf.check(f"{form} M={M} chunk={chunk} nvec={nvec_id(nvec)}: {name}")
    names = ("logits", "actions") if output == "both" else ("actions", "log_probs")
    dtypes = {"logits": torch.int16, "actions": torch.int64, "log_probs": torch.int32}
    for name, h in zip(names, want):
        assert torch.equal(bufs[name].view(dtypes[name]).view(h.shape), bits(h)), (form, name)


# ---- 5. status codes ----------------------------------------------------------------------------------------------------
_BUFS = {}


def _buf(name, n, dtype=torch.float32):
    if name not in _BUFS:
        _BUFS[name] = torch.zeros(n, dtype=dtype, device="cuda")
    return _BUFS[name].data_ptr()


ROWS_BYTES = 256 * 256 * 2      # the status cases' M * d_in * 2: where a pushed mask may begin
NVEC_CASES = {
    "null_nvec": (dict(nvec=None), L.ERR_ARG),
    "no_groups": (dict(n_groups=0), L.ERR_ARG),
    "negative_groups": (dict(n_groups=-1), L.ERR_ARG),
    "more_groups_than_d_out": (dict(nvec=[1] * 19, n_groups=19), L.ERR_ARG),
    "empty_group": (dict(nvec=[9, 0, 9], n_groups=3), L.ERR_ARG),
    "negative_group": (dict(nvec=[19, -1], n_groups=2), L.ERR_ARG),
    "sum_below_d_out": (dict(nvec=[9, 8], n_groups=2), L.ERR_ARG),
    "sum_above_d_out": (dict(nvec=[9, 10], n_groups=2), L.ERR_ARG),
    "huge_group": (dict(nvec=[2**31 - 1, 2**31 - 1, 20], n_groups=3), L.ERR_ARG),
    "inherited_d_out_first": (dict(nvec=None, d_out=257), L.ERR_UNSUPPORTED),
    "inherited_d_in_first": (dict(n_groups=0, d_in=100), L.ERR_ARG),
}
VALUE_CASES = {"inherited_value_width_first": (dict(nvec=None, d_out=256), L.ERR_UNSUPPORTED)}
STATUS_KINDS = {kind_id(k): k for k in KINDS if k[0] != "both"}


def _status_overrides(kind, form, overrides):
    o = dict(nvec=[9, 9], n_groups=2, values=_buf("values", 4096))
    o.update(overrides)
    o["nvec"] = None if o["nvec"] is None else L.arr(ctypes.c_int32, o["nvec"])
    if kind[1]:
        o["mask"] = ROWS_BYTES if form is pushed else _buf("mask", 2048 * 512, torch.uint8)
    return o


@pytest.mark.parametrize("form", [plain, pushed], ids=["plain", "pushed"])
@pytest.mark.parametrize("kind,name", [(k, n) for k in STATUS_KINDS for n in NVEC_CASES] +
                         [(k, n) for k in STATUS_KINDS if STATUS_KINDS[k][2] for n in VALUE_CASES])
def test_bad_nvec_gets_the_documented_status_after_every_other_check(K, kind, name, form):
    overrides, status = {**NVEC_CASES, **VALUE_CASES}[name]
    k = STATUS_KINDS[kind]
    expect_status(form(md_head(k), **_status_overrides(k, form, overrides)), status)


@pytest.mark.parametrize("kind", list(STATUS_KINDS))
def test_empty_pushed_shard_runs_its_checks_and_acks(K, kind):
    """An empty shard (M = 0) with null outputs and a null nvec publishes ack[rank] = seq in the root's control block;
    with a bad argument it returns the status of the entry without groups."""
    k = STATUS_KINDS[kind]
    ctrl_root = torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda")
    empty = dict(M=0, logits=0, actions=0, log_probs=0, values=0, nvec=None, n_groups=0, mask=0)
    L.call(*pushed(md_head(k), ctrl_root=ctrl_root.data_ptr(), seq=3, rank=2, **empty))
    torch.cuda.synchronize()
    assert int(ctrl_root[512 + 8 * 2:512 + 8 * 3].view(torch.int64)) == 3
    expect_status(pushed(md_head(k), seq=0, **empty), L.ERR_ARG)


# ---- 6. Python checks ---------------------------------------------------------------------------------------------------
def test_python_checks_name_the_output_in_mlp_forward_and_scatter_gather(K):
    (w1, w2, w3), b = config(3400, 18)
    obs = randn((256, 256), 3401)
    bad = [
        ("logits", {}, (9, 9), 'nvec is not an argument of output="logits"'),
        ("gaussian", dict(seed=1, log_std=torch.zeros(18, device="cuda")), (9, 9),
         'nvec is not an argument of output="gaussian"'),
        ("actions", {}, (9.0, 9), "tuple of ints"),
        ("both", {}, (True, 17), "tuple of ints"),
        ("sample", dict(seed=1), "99", "tuple of ints"),
        ("sample", dict(seed=1), (), "empty"),
        ("actions", {}, (9, 0, 9), ">= 1"),
        ("sample", dict(seed=1), (9, 8), "sums to 17"),
        ("actions", {}, (9, 10), "sums to 19"),
    ]
    for output, kw, nvec, reason in bad:
        with pytest.raises(ValueError, match=reason):
            mlp.mlp_forward(obs, w1, w2, w3, biases=b, output=output, nvec=nvec, **kw)
        with pytest.raises(ValueError, match=reason):
            mlp.mlp_scatter_gather(obs, w1, w2, w3, devices=[0], biases=b, output=output, nvec=nvec, **kw)
    wrong = torch.zeros(256, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError, match=r"actions must have shape \(256, 2\)"):
        mlp.mlp_forward(obs, w1, w2, w3, biases=b, output="actions", nvec=(9, 9), actions=wrong)
    with pytest.raises(ValueError, match=r"actions must have shape \(256, 2\)"):
        mlp.mlp_scatter_gather(obs, w1, w2, w3, devices=[0], biases=b, output="sample", seed=1, nvec=(9, 9),
                               actions_root=wrong)
    given = torch.full((256, 2), -1, dtype=torch.int64, device="cuda")
    got = mlp.mlp_forward(obs, w1, w2, w3, biases=b, output="actions", nvec=(9, 9), actions=given)
    assert got is given and bool((given >= 0).all() and (given < 9).all())


# ---- 7. the public API ----------------------------------------------------------------------------------------------------
PUBLIC = {
    "actions": (cases.mlp_policy_multidiscrete_actions, dict(output="actions"), ()),
    "both": (cases.mlp_policy_multidiscrete_both, dict(output="both"), ()),
    "sample": (cases.mlp_policy_multidiscrete_sample, dict(output="sample", seed="seed"), ("seed",)),
    "masked_actions": (cases.mlp_policy_multidiscrete_masked_actions, dict(output="actions", mask="legal"),
                       ("legal",)),
    "masked_sample": (cases.mlp_policy_multidiscrete_masked_sample, dict(output="sample", seed="seed", mask="legal"),
                      ("legal", "seed")),
    "sample_value": (cases.mlp_policy_multidiscrete_sample_value,
                     dict(output="sample", seed="seed", value=("wv", "bv")), ("wv", "bv", "seed")),
}


def _public_case(golden, kind):
    obs = torch.randn(1000, 256, generator=torch.Generator().manual_seed(1001)).bfloat16()
    p = policy_weights(golden, sum(cases.NVEC))
    g = torch.Generator().manual_seed(78)
    body, extra, names = PUBLIC[kind]
    more = dict(seed=2**35 + 29, legal=torch.rand(obs.shape[0], 6, generator=g) < 0.5,
                wv=(torch.randn(1, 1024, generator=g) * 0.02).bfloat16(),
                bv=(torch.randn(1, generator=g) * 0.1).bfloat16())
    more["legal"][::50] = False
    more["legal"][::9, :3] = False
    policy = mapped_copy(body, "mlp", bias=True, nvec=cases.NVEC, **extra)
    return obs, p, [more[n] for n in names], body, policy, extra


def _cuda(t):
    return t.cuda() if isinstance(t, torch.Tensor) else t


def _mine(obs, p, args, kind, extra):
    """mlp_forward over all rows on cuda:0."""
    pc = [t.cuda() for t in p]
    named = dict(zip(PUBLIC[kind][2], args))
    kw = dict(output=extra["output"], nvec=cases.NVEC)
    if "seed" in named:
        kw["seed"] = named["seed"]
    if "legal" in named:
        kw["mask"] = named["legal"].cuda()
    if "wv" in named:
        kw["value"] = (named["wv"].cuda(), named["bv"].cuda())
    return as_tuple(mlp.mlp_forward(obs.cuda(), pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]), **kw))


@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["1_rank", "3_ranks"])
@pytest.mark.parametrize("kind", list(PUBLIC))
def test_mapped_multidiscrete_through_public_api(K, golden, kind, devices):
    """@kt.mapped("mlp", bias=True, output=..., nvec=NVEC) on Compute(gpus=1): each rank returns the bits of
    mlp_forward over its rows, and against the oracle's run of the body the actions of every group agree on at least
    99 % of the rows (the logits differ from the CPU's in the last bit now and then)."""
    obs, p, args, body, policy, extra = _public_case(golden, kind)
    n = len(devices)
    want = ref_dispatch.spmd_call(body, obs, *p, *args, num_proc=n, serialization="pickle")
    mine = _mine(obs, p, args, kind, extra)
    with deployed(policy, f"t-md-{kind}-{n}", devices) as remote:
        got = remote(obs.cuda(), *[t.cuda() for t in p], *[_cuda(t) for t in args], serialization="pickle")
        torch.cuda.synchronize()
    assert len(got) == len(want) == n
    k = 1 if kind == "both" else 0
    agree, total = 0, 0
    for r, (g, h) in enumerate(zip(got, want)):
        lo, hi = K.shard_bounds(obs.shape[0], n, r)
        g, h = as_tuple(g), as_tuple(h)
        same([t.cpu() for t in g], [t[lo:hi].cpu() for t in mine], (kind, r))
        assert g[k].shape == (hi - lo, len(cases.NVEC)) and h[k].shape == g[k].shape, (kind, r)
        agree += int((g[k].cpu() == h[k]).all(-1).sum())
        total += hi - lo
    assert agree >= 0.99 * total, (agree, total)


def test_mapped_multidiscrete_on_a_workers_subset(K, golden):
    """Two workers of one rank each on cuda:0; a call with workers=[1] returns rank 1's (actions, log_probs) only,
    with the bits of mlp_forward over its rows."""
    import kubetorch_b200 as kt

    obs, p, args, body, policy, extra = _public_case(golden, "masked_sample")
    mine = _mine(obs, p, args, "masked_sample", extra)
    remote = kt.fn(policy, name="t-md-workers").to(
        kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute("b200", workers=2, num_proc=1,
                                                                                 devices=[0, 0]))
    try:
        got = remote(obs.cuda(), *[t.cuda() for t in p], *[_cuda(t) for t in args], serialization="pickle",
                     workers=[1])
        torch.cuda.synchronize()
    finally:
        remote.teardown()
    lo, hi = K.shard_bounds(obs.shape[0], 2, 1)
    assert len(got) == 1
    same([t.cpu() for t in got[0]], [t[lo:hi].cpu() for t in mine], "workers=[1]")


# ---- 8. two GPUs ----------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("transfer", ["pull", "push"])
@pytest.mark.parametrize("kind", ["both", "masked_sample", "sample_value"])
def test_mapped_multidiscrete_on_two_gpus(K, golden, kind, transfer):
    """Two ranks on two GPUs, staged pull and pushed form, two back-to-back calls with fresh observations: the bits of
    one plain call."""
    obs, p, args, body, policy, extra = _public_case(golden, kind)
    with deployed(policy, f"t-md-2gpu-{kind}-{transfer}", [0, 1], transfer=transfer) as remote:
        pc = [t.cuda(0) for t in p]
        for it in range(2):
            x = torch.randn(2 * 1408, 256, generator=torch.Generator().manual_seed(15 + it)).bfloat16()
            a = list(args)
            if "legal" in PUBLIC[kind][2]:
                a[0] = torch.rand(x.shape[0], 6, generator=torch.Generator().manual_seed(19 + it)) < 0.5
            got = remote(x.cuda(0), *pc, *[t.cuda(0) if isinstance(t, torch.Tensor) else t for t in a],
                         serialization="pickle")
            torch.cuda.synchronize(0)
            torch.cuda.synchronize(1)
            want = _mine(x, p, a, kind, extra)
            got = [as_tuple(g) for g in got]
            same([torch.cat([g[k].cpu() for g in got]) for k in range(len(want))], [t.cpu() for t in want], (kind, it))

