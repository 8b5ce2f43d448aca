"""-m gpu: per-row legal-action masks on the categorical heads of the bf16 MLP policy (ktb_mlp_bf16_policy_masked*,
ktb_mlp_bf16_policy_sample_masked*, mask= of mlp_forward and kt.mapped) — masked logits and greedy actions bit for bit
against the unmasked kernel's logits filled with -inf, sampled actions and log-probabilities against fp64 restatements
over the legal columns, their distribution by a chi-square test, edge rows, all-legal masks against the unmasked
entries, every form, chunking and row split, guard bands, status codes, the public API and two GPUs."""
import ctypes

import pytest
import torch

from conftest import mapped_copy
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp
from mlp_rig import (SHIPPED_CHUNK, Guarded, Head, K, PushRig, config, deployed, entry_args,  # noqa: F401
                     expect_status, from_row, named_args, plain, policy_weights, pushed, randn, stream, tuning)

pytestmark = pytest.mark.gpu

import policy_masked_cases  # noqa: E402
from oracle import ref_dispatch  # noqa: E402

from kubetorch_b200.sampling import gumbel_uniform  # noqa: E402

WIDTHS = [1, 2, 18, 63, 64, 65, 128, 129, 255, 256]
MASKED_GREEDY = Head("ktb_mlp_bf16_policy_masked", "ktb_mlp_bf16_policy_masked",
                     "ktb_mlp_bf16_policy_masked_pushed", True, 0, {"logits": lambda d: 2 * d, "actions": lambda d: 8},
                     lambda a: (a["mask"], a["logits"], a["actions"]))
MASKED_SAMPLE = Head("ktb_mlp_bf16_policy_sample_masked", "ktb_mlp_bf16_policy_sample_masked",
                     "ktb_mlp_bf16_policy_sample_masked_pushed", True, 0,
                     {"actions": lambda d: 8, "log_probs": lambda d: 4},
                     lambda a: (a["mask"], a["seed"], a["row_base"], a["actions"], a["log_probs"]))


# ---- inputs and bars -------------------------------------------------------------------------------------------------
def random_legal(M, d_out, seed, p=0.5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(M, d_out, generator=g, device="cuda") < p


def fill(y, legal):
    return y.masked_fill(~legal, float("-inf"))


def bits(t):
    """The bit patterns of a 16- or 32-bit float tensor, for comparisons that see NaNs and signed zeros."""
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def forward(obs, w, b, output, **kw):
    return mlp.mlp_forward(obs, *w, biases=b, output=output, **kw)


def check_masked_sample(y, legal, seed, row0, actions, log_probs, what, row_ids=None):
    """y: the kernel's own UNMASKED bf16 logits of global rows row0, ... (finite); legal: their mask.  Rows with no legal
    action get action 0 and a NaN log-probability.  On the others, with s64 = masked(y) + g64 and ε = 2^-18·(1 + max
    finite |s64|): the action is legal, s64[a] >= max s64 - ε, a = argmax s64 wherever the top-2 gap exceeds ε (at
    least 99.9 % of rows), and |log_prob - (y_a - logsumexp64(masked y))| <= (d_out + 8)·2^-22·(1 + |ref|).  With
    row_ids the rows are those global rows instead."""
    M, d_out = y.shape
    assert actions.dtype == torch.int64 and actions.shape == (M,), what
    assert log_probs.dtype == torch.float32 and log_probs.shape == (M,), what
    a = actions.to(y.device)
    lp = log_probs.to(y.device)
    none = ~legal.any(dim=1)
    assert bool((a[none] == 0).all()) and bool(torch.isnan(lp[none]).all()), what
    rows = ~none
    y, legal, a, lp = y[rows], legal[rows], a[rows], lp[rows]
    assert bool(legal.gather(1, a[:, None]).all()), (what, "an illegal action on a row with a legal one")
    if row_ids is None:
        u = gumbel_uniform(seed, row0, M, d_out, device=y.device).double()[rows]
    else:
        u = gumbel_uniform(seed, 0, int(row_ids.max()) + 1, d_out, device=y.device).double()[row_ids][rows]
    s64 = fill(y.double(), legal) - torch.log(-torch.log(u))
    eps = 2.0 ** -18 * (1 + s64.masked_fill(~legal, 0).abs().amax(dim=1))
    top = s64.amax(dim=1)
    chosen = s64.gather(1, a[:, None]).squeeze(1)
    assert not bool((chosen < top - eps).any()), what
    if d_out > 1:
        top2 = s64.topk(2, dim=1).values
        clear = (top2[:, 0] - top2[:, 1]) > eps
    else:
        clear = torch.ones(a.shape[0], dtype=torch.bool, device=y.device)
    assert float(clear.double().mean()) >= 0.999, (what, float(clear.double().mean()))
    assert torch.equal(a[clear], s64.argmax(dim=1)[clear]), what
    ym = fill(y.double(), legal)
    ref = ym.gather(1, a[:, None]).squeeze(1) - torch.logsumexp(ym, dim=-1)
    tol = (d_out + 8) * 2.0 ** -22 * (1 + ref.abs())
    assert bool(((lp.double() - ref).abs() <= tol).all()), what
    one = legal.sum(dim=1) == 1
    assert bool((lp[one] == 0).all()), what


# ---- 1. exact against the unmasked kernel ----------------------------------------------------------------------------
@pytest.mark.parametrize("d_out", WIDTHS)
@pytest.mark.parametrize("chunk", [256, SHIPPED_CHUNK])
def test_masked_logits_and_actions_equal_the_filled_unmasked_logits(K, d_out, chunk):
    """About half the columns legal, plus rows with none and rows with one: masked logits are the unmasked kernel's
    logits filled with bf16 -inf bit for bit, and masked actions (with and without logits) their torch.argmax."""
    M = SHIPPED_CHUNK + 1005
    w, b = config(900 + d_out, d_out)
    w = (w[0], w[1], w[2] * 50)
    obs = randn((M, 256), 910 + d_out)
    legal = random_legal(M, d_out, 920 + d_out)
    legal[::97] = False
    legal[1::97] = torch.arange(d_out, device="cuda") == (d_out // 2)
    keep = legal.clone()
    with tuning(chunk):
        y = forward(obs, w, b, "logits")
        logits, actions = forward(obs, w, b, "both", mask=legal)
        only = forward(obs, w, b, "actions", mask=legal)
        masked_logits = forward(obs, w, b, "logits", mask=legal)
    want = fill(y, legal)
    assert torch.equal(bits(logits), bits(want)) and torch.equal(bits(masked_logits), bits(want)), (d_out, chunk)
    assert torch.equal(actions, want.argmax(-1)) and torch.equal(only, actions), (d_out, chunk)
    assert torch.equal(legal, keep)


# ---- 2. sampled ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d_out", WIDTHS)
@pytest.mark.parametrize("chunk", [256, SHIPPED_CHUNK])
def test_masked_sample_bars_at_every_head_width(K, d_out, chunk):
    M, seed = SHIPPED_CHUNK + 1005, 2**33 + 11 * d_out
    w, b = config(1000 + d_out, d_out)
    w = (w[0], w[1], w[2] * 50)
    obs = randn((M, 256), 1010 + d_out)
    legal = random_legal(M, d_out, 1020 + d_out)
    legal[::89] = False
    legal[1::89] = torch.arange(d_out, device="cuda") == (d_out - 1)
    with tuning(chunk):
        y = forward(obs, w, b, "logits")
        actions, log_probs = forward(obs, w, b, "sample", seed=seed, mask=legal)
    check_masked_sample(y, legal, seed, 0, actions, log_probs, f"d_out={d_out} chunk={chunk}")


# ---- 3. the distribution -----------------------------------------------------------------------------------------------
def test_masked_draws_follow_softmax_over_each_legal_set(K):
    """W3 = 0 and b3 a fixed logit vector; four mask patterns cycled over 2^20 rows.  For each pattern its illegal
    columns get no draws and a chi-square test against softmax(b3) renormalised over its legal set gives p > 1e-4."""
    from scipy.stats import chisquare

    b3v = [1.0, 0.5, -0.5, 0.0, 2.0, -1.0, 0.75, 0.25, -3.0, 1.5]
    d_out, M = len(b3v), 1 << 20
    patterns = torch.tensor([[1, 1, 1, 1, 1, 1, 1, 1, 1, 1], [1, 0, 1, 0, 1, 0, 1, 0, 1, 0],
                             [0, 0, 0, 1, 1, 1, 0, 0, 0, 1], [0, 1, 1, 0, 0, 0, 0, 1, 0, 0]],
                            dtype=torch.bool, device="cuda")
    legal = patterns[torch.arange(M, device="cuda") % 4].contiguous()
    (w1, w2, _), (b1, b2, _) = config(1100, d_out)
    w3 = torch.zeros(d_out, 1024, dtype=torch.bfloat16, device="cuda")
    b3 = torch.tensor(b3v, dtype=torch.bfloat16, device="cuda")
    obs = randn((M, 256), 1101)
    actions, log_probs = forward(obs, (w1, w2, w3), (b1, b2, b3), "sample", seed=20261017, mask=legal)
    for k in range(4):
        a = actions[k::4]
        counts = torch.bincount(a, minlength=d_out).cpu()
        live = patterns[k].cpu()
        assert int(counts[~live].sum()) == 0, (k, counts.tolist())
        p = torch.softmax(fill(b3.double().cpu(), live), -1)
        stat = chisquare(counts[live].double().numpy(), (p[live] * a.numel()).numpy())
        print(f"pattern {k}: chi-square over {int(live.sum())} columns: stat={stat.statistic:.2f} p={stat.pvalue:.4f}")
        assert stat.pvalue > 1e-4, (k, stat, counts.tolist())
        ref = torch.log_softmax(fill(b3.double(), patterns[k]), -1)[a]
        tol = (d_out + 8) * 2.0 ** -22 * (1 + ref.abs())
        assert bool(((log_probs[k::4].double() - ref).abs() <= tol).all()), k


# ---- 4. edge rows ----------------------------------------------------------------------------------------------------------
def test_edge_rows_in_one_call(K):
    """b3 plants NaN at column 3 and +inf at column 5 of every row.  Rows cycle through: no legal action (action 0, NaN
    log-probability, all -inf logits); one legal finite column (that action, log-probability 0.0); NaN and +inf columns
    illegal (no effect: the bars over the finite legal columns); the NaN column legal (action 3, the first NaN, and a
    NaN log-probability); the +inf column legal and the NaN one not (action 5, NaN log-probability, as torch)."""
    d_out, M, seed = 18, 5 * 1024, 4321
    w, b = config(1200, d_out)
    b3 = b[2].clone()
    b3[3], b3[5] = float("nan"), float("inf")
    b = (b[0], b[1], b3)
    obs = randn((M, 256), 1201)
    kind = torch.arange(M, device="cuda") % 5
    legal = random_legal(M, d_out, 1202)
    cols = torch.arange(d_out, device="cuda")
    legal[kind == 0] = False
    one_col = (torch.arange(M, device="cuda") // 5) % d_out
    one_col = torch.where((one_col == 3) | (one_col == 5), one_col + 1, one_col)
    legal[kind == 1] = cols[None, :] == one_col[kind == 1][:, None]
    legal[kind == 2, 3] = False
    legal[kind == 2, 5] = False
    legal[kind == 2, 0] = True
    legal[kind == 3, 3] = True
    legal[kind == 4, 3] = False
    legal[kind == 4, 5] = True
    y = forward(obs, w, b, "logits")
    logits, actions = forward(obs, w, b, "both", mask=legal)
    sa, slp = forward(obs, w, b, "sample", seed=seed, mask=legal)
    want = fill(y, legal)
    assert torch.equal(bits(logits), bits(want))
    assert torch.equal(actions, want.argmax(-1))
    assert bool(torch.isneginf(logits[kind == 0].float()).all())
    assert bool((actions[kind == 0] == 0).all()) and bool((sa[kind == 0] == 0).all())
    assert bool(torch.isnan(slp[kind == 0]).all())
    assert torch.equal(sa[kind == 1], one_col[kind == 1]) and torch.equal(actions[kind == 1], one_col[kind == 1])
    assert bool((slp[kind == 1] == 0).all())
    assert bool((actions[kind == 3] == 3).all()) and bool((sa[kind == 3] == 3).all())
    assert bool(torch.isnan(slp[kind == 3]).all())
    assert bool((actions[kind == 4] == 5).all()) and bool((sa[kind == 4] == 5).all())
    assert bool(torch.isnan(slp[kind == 4]).all())
    ref = torch.log_softmax(want.float(), -1).gather(1, sa[:, None]).squeeze(1)
    assert torch.equal(torch.isnan(slp), torch.isnan(ref))
    rows = kind == 2
    check_masked_sample(y[rows], legal[rows], seed, 0, sa[rows], slp[rows], "NaN and +inf illegal",
                        row_ids=rows.nonzero()[:, 0])


# ---- 5. all-true masks ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d_out", [1, 18, 64, 129, 256])
def test_all_true_mask_gives_the_unmasked_bits(K, d_out):
    M, seed = 3000, 99
    w, b = config(1300 + d_out, d_out)
    obs = randn((M, 256), 1301)
    legal = torch.ones(M, d_out, dtype=torch.bool, device="cuda")
    for output in ("logits", "actions", "both", "sample"):
        kw = dict(seed=seed) if output == "sample" else {}
        want = forward(obs, w, b, output, **kw)
        got = forward(obs, w, b, output, mask=legal, **kw)
        want, got = (want, got) if isinstance(want, tuple) else ((want,), (got,))
        for g, h in zip(got, want):
            assert torch.equal(bits(g) if g.is_floating_point() else g, bits(h) if h.is_floating_point() else h), \
                (output, d_out)


# ---- 6. forms --------------------------------------------------------------------------------------------------------------
def _outputs(head, M, d_out):
    if head is MASKED_GREEDY:
        return {"logits": torch.full((M, d_out), -1, dtype=torch.int16, device="cuda"),
                "actions": torch.full((M,), -1, dtype=torch.int64, device="cuda")}
    return {"actions": torch.full((M,), -1, dtype=torch.int64, device="cuda"),
            "log_probs": torch.full((M,), -1, dtype=torch.int32, device="cuda")}


def _want(head, obs, w, b, legal, seed, **kw):
    if head is MASKED_GREEDY:
        logits, actions = forward(obs, w, b, "both", mask=legal, **kw)
        return {"logits": bits(logits), "actions": actions}
    actions, log_probs = forward(obs, w, b, "sample", seed=seed, mask=legal, **kw)
    return {"actions": actions, "log_probs": bits(log_probs)}


def _same(got, want, what):
    for name in want:
        assert torch.equal(got[name], want[name]), (what, name)


@pytest.mark.parametrize("head", [MASKED_GREEDY, MASKED_SAMPLE], ids=["greedy", "sample"])
@pytest.mark.parametrize("d_out", [18, 129])
def test_every_form_chunking_and_row_split_gives_identical_bits(K, head, d_out):
    """Repeat calls, chunk sizes 256 / 512 / shipped, plain and staged (pull kernel and copy engine), pushed through the
    rig (three back-to-back calls with fresh observations and masks), and [0, s) + [s, M) with row_offset = s: the bits
    of one plain call.  The mask is unchanged after every call."""
    w, b = config(1400 + d_out, d_out)
    M, seed = SHIPPED_CHUNK + 1000, 77
    obs = randn((M, 256), 1401)
    legal = random_legal(M, d_out, 1402)
    keep = legal.clone()
    want = _want(head, obs, w, b, legal, seed)
    _same(_want(head, obs, w, b, legal, seed), want, "repeat")
    for chunk in (256, 512, SHIPPED_CHUNK):
        for ce in (None, 0, 1):
            with tuning(chunk, ce):
                _same(_want(head, obs, w, b, legal, seed, staged=ce is not None), want, (chunk, ce))
    for split in (1, 1000, 16896, 16900):
        lo = _want(head, obs[:split], w, b, legal[:split], seed)
        hi = _want(head, obs[split:], w, b, legal[split:], seed, row_offset=split)
        _same({k: torch.cat([lo[k], hi[k]]) for k in want}, want, split)
    assert torch.equal(legal, keep)
    Mp = 3 * 1408
    rig = PushRig(K, Mp, 256, 1024, 512, "ce", head, sides=[("mask", d_out)])
    for it in range(3):
        obs_p = randn((Mp, 256), 1410 + it)
        legal_p = random_legal(Mp, d_out, 1420 + it)
        keep_p = legal_p.clone()
        want_p = _want(head, obs_p, w, b, legal_p, seed)
        out = _outputs(head, Mp, d_out)
        rig.call(obs_p, w, b, {k: t.data_ptr() for k, t in out.items()}, seed, sides={"mask": legal_p})
        torch.cuda.synchronize()
        _same(out, want_p, ("pushed", it))
        assert torch.equal(legal_p, keep_p)
    assert rig.statuses() == [0] * rig.n


@pytest.mark.parametrize("output", ["both", "sample"])
def test_package_push_path_on_one_gpu_matches_plain_bits(K, output):
    """mlp_scatter_gather's pushed form with a mask (a cached PushSession grown for the mask rows, the masked copy-engine
    scatter, the root's shard on the side stream) with ranks [0, 0, 0] on cuda:0, back to back with fresh inputs and one
    unmasked call between: equal to one plain call over all rows."""
    devs, rows, d_out, seed = [0, 0, 0], 35072, 64, 9
    M = 3 * rows
    bounds = [K.shard_bounds(M, 3, r) for r in range(3)]
    w, b = config(1500, d_out)
    weights = {0: (*w, *b)}
    for it in range(3):
        obs = randn((M, 256), 1501 + it)
        legal = random_legal(M, d_out, 1511 + it) if it != 1 else None
        kw = dict(seed=seed) if output == "sample" else {}
        want = forward(obs, w, b, output, mask=legal, **kw)
        logits = torch.full((M, d_out), -1, dtype=torch.bfloat16, device="cuda") if output == "both" else None
        actions = torch.full((M,), -1, dtype=torch.int64, device="cuda")
        log_probs = torch.full((M,), -1, dtype=torch.float32, device="cuda") if output == "sample" else None
        mlp._mlp_scatter_gather_pushed(obs, devs, bounds, weights, output, logits, actions, log_probs,
                                       seed if output == "sample" else None, None, legal)
        torch.cuda.synchronize()
        got = (logits, actions) if output == "both" else (actions, log_probs)
        for g, h in zip(got, want):
            assert torch.equal(bits(g) if g.is_floating_point() else g, bits(h) if h.is_floating_point() else h), it
    mlp._push_sessions[tuple(devs)].check()


# ---- 7. guard bands ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("head", [MASKED_GREEDY, MASKED_SAMPLE], ids=["greedy", "sample"])
@pytest.mark.parametrize("form,M,chunk,d_out", [
    ("plain", 1000, SHIPPED_CHUNK, 7), ("plain", 1000, 256, 129), ("staged", 1408, 256, 18), ("pushed", 3 * 1408, 256, 7),
])
def test_writes_stay_inside_the_outputs(K, head, form, M, chunk, d_out):
    """Every output, the scratch and the stage between guard bands (the logits at a 2-byte offset); the mask itself in
    a guarded buffer is unchanged; the results equal mlp_forward's bit for bit."""
    seed = 5
    w, b = config(1600, d_out)
    obs = randn((M, 256), 1601)
    legal = random_legal(M, d_out, 1602)
    want = _want(head, obs, w, b, legal, seed)
    gmask = Guarded(M * d_out, 3)
    gmask.view().copy_(legal.view(torch.uint8).flatten())
    bufs = {name: Guarded(M * row_bytes(d_out), 2 if name == "logits" else 0) for name, row_bytes in head.outputs.items()}
    out = {name: buf.ptr() for name, buf in bufs.items()}
    with tuning(chunk):
        if form == "pushed":
            rig = PushRig(K, M, 256, 1024, 512, "ce", head, sides=[("mask", d_out)])
            for _ in range(3):
                rig.call(obs, w, b, out, seed, sides={"mask": gmask.view()})
            torch.cuda.synchronize()
            assert rig.statuses() == [0] * rig.n
            bufs.update({f"stage[{r}]": rig.stage[r] for r in range(1, rig.n)})
            bufs.update({f"scratch[{r}]": rig.scratch[r] for r in range(1, rig.n)})
        else:
            bufs["scratch"] = Guarded(L.load().ktb_mlp_scratch_bytes(M, 1024))
            if form == "staged":
                bufs["stage"] = Guarded(L.load().ktb_mlp_stage_bytes(M, 256))
            L.call(*entry_args(head, named_args(obs, w, b, out, seed, mask=gmask.ptr(), scratch=bufs["scratch"].ptr(),
                                                stage=bufs["stage"].ptr() if form == "staged" else None)))
    bufs["mask"] = gmask
    for name, buf in bufs.items():
        buf.check(f"{form} M={M} chunk={chunk} d_out={d_out}: {name}")
    assert torch.equal(gmask.view(), legal.view(torch.uint8).flatten())
    dtypes = {"logits": torch.int16, "actions": torch.int64, "log_probs": torch.int32}
    _same({name: bufs[name].view(dtypes[name]).view(want[name].shape) for name in want}, want, form)


# ---- 8. status codes -------------------------------------------------------------------------------------------------------
_MASK = {}


def _mask_ptr():
    if "t" not in _MASK:
        _MASK["t"] = torch.ones(2048 * 512, dtype=torch.uint8, device="cuda")
    return _MASK["t"].data_ptr()


ROWS_BYTES = 256 * 256 * 2      # the status cases' M * d_in * 2: where a pushed mask may begin
STATUS_CASES = {
    "null_mask": (plain, dict(mask=0), L.ERR_ARG),
    "staged_null_mask": (plain, dict(mask=0, stage_off=0), L.ERR_ARG),
    "inherited_checks_first": (plain, dict(mask=0, d_out=257), L.ERR_UNSUPPORTED),
    "pushed_mask_offset_over_the_rows": (pushed, dict(mask=ROWS_BYTES - 1), L.ERR_ARG),
    "pushed_mask_offset_zero": (pushed, dict(mask=0), L.ERR_ARG),
    "pushed_mask_past_stage_stride": (pushed, dict(mask=(1 << 20) - 256 * 18 + 1), L.ERR_ARG),
    "pushed_mask_offset_past_stage_stride": (pushed, dict(mask=(1 << 21)), L.ERR_ARG),
    "pushed_inherited_checks_first": (pushed, dict(mask=0, d_out=257), L.ERR_UNSUPPORTED),
}


@pytest.mark.parametrize("head", [MASKED_GREEDY, MASKED_SAMPLE], ids=["greedy", "sample"])
@pytest.mark.parametrize("name", list(STATUS_CASES))
def test_bad_arguments_get_the_documented_status(K, head, name):
    form, overrides, status = STATUS_CASES[name]
    overrides = dict(overrides)
    if form is plain and "stage_off" in overrides:
        overrides.pop("stage_off")
        overrides["stage"] = _zero_stage()
    expect_status(form(head, **{"mask": _mask_ptr(), **overrides}), status)


def _zero_stage():
    if "stage" not in _MASK:
        _MASK["stage"] = torch.zeros(1 << 24, dtype=torch.uint8, device="cuda")
    return _MASK["stage"].data_ptr()


def _scatter_args(**overrides):
    """ktb_push_scatter_ce_masked over 3 × 256 rows of d_in 256 for ranks [0, 0, 0], call 1, stage_stride 1 MiB."""
    if "bufs" not in _MASK:
        _MASK["bufs"] = dict(obs=torch.zeros(768 * 256, dtype=torch.bfloat16, device="cuda"),
                             stage=torch.zeros(2 << 20, dtype=torch.uint8, device="cuda"),
                             ctrl=torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda"))
    z = _MASK["bufs"]
    a = dict(root_dev=0, obs=z["obs"].data_ptr(), n_elems=768 * 256, granule=256, dtype=L.BF16, n=3, root_rank=0,
             stride=1 << 20, chunk_elems=256 * 256, mask=_mask_ptr(), row_bytes=18, mask_offset=ROWS_BYTES, seq=1)
    a.update(overrides)
    stages = L.arr(ctypes.c_void_p, [0] + [z["stage"].data_ptr()] * 2)
    ctrls = L.arr(ctypes.c_void_p, [z["ctrl"].data_ptr()] * 3)
    return ("ktb_push_scatter_ce_masked", a["root_dev"], a["obs"], a["n_elems"], a["granule"], a["dtype"], a["n"],
            a["root_rank"], L.arr(ctypes.c_int, [0, 0, 0]), stages, a["stride"], ctrls, z["ctrl"].data_ptr(),
            a["chunk_elems"], a["mask"], a["row_bytes"], a["mask_offset"], a["seq"], stream())


SCATTER_CASES = {
    "null_mask": (dict(mask=0), L.ERR_ARG),
    "zero_row_bytes": (dict(row_bytes=0), L.ERR_ARG),
    "chunk_not_whole_rows": (dict(chunk_elems=256 * 256 + 1), L.ERR_ARG),
    "mask_offset_over_the_rows": (dict(mask_offset=ROWS_BYTES - 1), L.ERR_ARG),
    "mask_past_stage_stride": (dict(mask_offset=(1 << 20) - 256 * 18 + 1), L.ERR_ARG),
    "mask_offset_past_stage_stride": (dict(mask_offset=1 << 21), L.ERR_ARG),
    "inherited_checks_first": (dict(mask=0, root_dev=15), L.ERR_STATE),
}


@pytest.mark.parametrize("name", list(SCATTER_CASES))
def test_masked_scatter_bad_arguments_get_the_documented_status(K, name):
    overrides, status = SCATTER_CASES[name]
    expect_status(_scatter_args(**overrides), status)


def test_python_checks_reach_mlp_forward_and_scatter_gather(K):
    """A mask of the wrong dtype, shape, device or layout, or one given with output="gaussian", is a ValueError."""
    (w1, w2, w3), b = config(1700, 18)
    obs = randn((256, 256), 1701)
    good = torch.ones(256, 18, dtype=torch.bool, device="cuda")
    bad = [good.to(torch.uint8), good[:, :17].contiguous(), good[:255].contiguous(), good.cpu(),
           torch.ones(18, 256, dtype=torch.bool, device="cuda").t()]
    for m in bad:
        for output, kw in (("actions", {}), ("both", {}), ("logits", {}), ("sample", dict(seed=1))):
            with pytest.raises(ValueError, match="mask"):
                mlp.mlp_forward(obs, w1, w2, w3, biases=b, output=output, mask=m, **kw)
            with pytest.raises(ValueError, match="mask"):
                mlp.mlp_scatter_gather(obs, w1, w2, w3, devices=[0], biases=b, output=output, mask=m, **kw)
    log_std = torch.zeros(18, dtype=torch.float32, device="cuda")
    with pytest.raises(ValueError, match="gaussian"):
        mlp.mlp_forward(obs, w1, w2, w3, biases=b, output="gaussian", seed=1, log_std=log_std, mask=good)
    assert mlp.mlp_forward(obs, w1, w2, w3, biases=b, output="actions", mask=good).shape == (256,)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_mask_on_another_gpu_than_obs_is_refused(K):
    (w1, w2, w3), b = config(1710, 18)
    obs = randn((256, 256), 1711)
    other = torch.ones(256, 18, dtype=torch.bool, device="cuda:1")
    with pytest.raises(ValueError, match="device of obs"):
        mlp.mlp_forward(obs, w1, w2, w3, biases=b, output="actions", mask=other)
    with pytest.raises(ValueError, match="device of obs"):
        mlp.mlp_scatter_gather(obs, w1, w2, w3, devices=[0, 1], biases=b, output="actions", mask=other)


# ---- 9. the public API -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("output", ["actions", "sample"])
@pytest.mark.parametrize("case", ["recorded", "ragged_1000_rows_3_ranks"])
def test_mapped_mask_through_public_api(K, golden, output, case):
    """@kt.mapped("mlp", bias=True, output=..., mask="legal") on Compute(gpus=1) with three ranks on cuda:0: each rank's
    result equals the masked kernel's over its rows bit for bit, never picks an illegal action where its row has a
    legal one, and agrees with the oracle's run of the body on at least 99 % of the rows."""
    if case == "recorded":
        obs, d_out = golden["all_inputs"]["mlp_obs"], 64
    else:
        obs, d_out = torch.randn(1000, 256, generator=torch.Generator().manual_seed(1000)).bfloat16(), 6
    p = policy_weights(golden, d_out)
    legal = torch.rand(obs.shape[0], d_out, generator=torch.Generator().manual_seed(3)) < 0.5
    legal[::50] = False
    n_ranks, seed = 3, 2**35 + 19
    if output == "sample":
        body, extra, args = policy_masked_cases.mlp_policy_masked_sample, dict(seed="seed"), (seed,)
    else:
        body, extra, args = policy_masked_cases.mlp_policy_masked_actions, {}, ()
    want = ref_dispatch.spmd_call(body, obs, *p, legal, *args, num_proc=n_ranks, serialization="pickle")
    policy = mapped_copy(body, "mlp", bias=True, output=output, mask="legal", **extra)
    with deployed(policy, f"t-masked-{output}-{case}", [0] * n_ranks) as remote:
        pc = [t.cuda() for t in p]
        lc = legal.cuda()
        got = remote(obs.cuda(), *pc, lc, *args, serialization="pickle")
        torch.cuda.synchronize()
        kw = dict(seed=seed) if output == "sample" else {}
        mine = mlp.mlp_forward(obs.cuda(), pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]), output=output, mask=lc,
                               **kw)
        assert len(got) == len(want) == n_ranks
        agree, total = 0, 0
        for r, (g, h) in enumerate(zip(got, want)):
            lo, hi = K.shard_bounds(obs.shape[0], n_ranks, r)
            ga = g[0] if output == "sample" else g
            ha = h[0] if output == "sample" else h
            ma = mine[0] if output == "sample" else mine
            assert torch.equal(ga.cpu(), ma[lo:hi].cpu()), (case, r)
            if output == "sample":
                assert torch.equal(bits(g[1].cpu()), bits(mine[1][lo:hi].cpu())), (case, r)
            has = legal[lo:hi].any(-1)
            assert bool(legal[lo:hi][has].gather(1, ga.cpu()[has][:, None]).all())
            agree += int((ga.cpu() == ha).sum())
            total += hi - lo
        assert agree >= 0.99 * total, (agree, total)


# ---- 10. two GPUs ----------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("output", ["actions", "sample"])
@pytest.mark.parametrize("transfer", ["pull", "push"])
def test_mapped_mask_on_two_gpus(K, golden, output, transfer):
    """Two ranks on two GPUs, staged pull and pushed form, three back-to-back calls with fresh observations and masks (the
    push form reuses staging half seq & 1 while the call before may still run): the bits of one plain call."""
    p = policy_weights(golden, 18)
    seed = 4242
    if output == "sample":
        body, extra, args = policy_masked_cases.mlp_policy_masked_sample, dict(seed="seed"), (seed,)
    else:
        body, extra, args = policy_masked_cases.mlp_policy_masked_actions, {}, ()
    policy = mapped_copy(body, "mlp", bias=True, output=output, mask="legal", **extra)
    with deployed(policy, f"t-masked-2gpu-{output}-{transfer}", [0, 1], transfer=transfer) as remote:
        pc = [t.cuda(0) for t in p]
        for it in range(3):
            obs = torch.randn(2 * 1408, 256, generator=torch.Generator().manual_seed(5 + it)).bfloat16().cuda(0)
            legal = (torch.rand(obs.shape[0], 18, generator=torch.Generator().manual_seed(9 + it)) < 0.5).cuda(0)
            got = remote(obs, *pc, legal, *args, serialization="pickle")
            torch.cuda.synchronize(0)
            torch.cuda.synchronize(1)
            kw = dict(seed=seed) if output == "sample" else {}
            want = mlp.mlp_forward(obs, pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]), output=output, mask=legal,
                                   **kw)
            if output == "sample":
                assert torch.equal(torch.cat([g[0].cpu() for g in got]), want[0].cpu()), it
                assert torch.equal(bits(torch.cat([g[1].cpu() for g in got])), bits(want[1].cpu())), it
            else:
                assert torch.equal(torch.cat([g.cpu() for g in got]), want.cpu()), it
