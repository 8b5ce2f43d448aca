"""-m gpu: the ε-greedy Q-network head of the bf16 MLP policy (ktb_mlp_bf16_policy_epsilon_greedy*, output=
"epsilon_greedy" of mlp_forward and kt.mapped) — tied bit for bit to the greedy entries (themselves checked against
fp64) and to the host's exploration streams: ε = 0 and ε = 1 at every head width, mixed per-row ε and its IEEE edges,
the explore frequency and the uniformity of exploratory actions over 2^20 rows, edge rows, every form, chunking and
row split, guard bands, status codes, the push scatter with two side sources, the public API and two GPUs."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import mapped_copy
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp
from mlp_rig import (SHIPPED_CHUNK, Guarded, Head, K, PushRig, config, deployed, entry_args,  # noqa: F401
                     expect_status, from_row, named_args, plain, pushed, randn, stream, tuning)

pytestmark = pytest.mark.gpu

import policy_epsilon_cases as cases  # noqa: E402
from oracle import ref_dispatch  # noqa: E402

from kubetorch_b200.sampling import explore_noise  # noqa: E402

WIDTHS = [1, 2, 3, 18, 63, 64, 65, 128, 129, 255, 256]
_OUT = {"actions": lambda d: 8, "q": lambda d: 4, "q_max": lambda d: 4}
EPS = Head("ktb_mlp_bf16_policy_epsilon_greedy", "ktb_mlp_bf16_policy_epsilon_greedy",
           "ktb_mlp_bf16_policy_epsilon_greedy_pushed", True, 0, _OUT,
           lambda a: (a["epsilon"], a["seed"], a["row_base"], a["actions"], a["q"], a["q_max"]))
EPS_MASKED = Head("ktb_mlp_bf16_policy_epsilon_greedy_masked", "ktb_mlp_bf16_policy_epsilon_greedy_masked",
                  "ktb_mlp_bf16_policy_epsilon_greedy_masked_pushed", True, 0, _OUT,
                  lambda a: (a["mask"], a["epsilon"], a["seed"], a["row_base"], a["actions"], a["q"], a["q_max"]))


# ---- helpers -----------------------------------------------------------------------------------------------------------
def random_legal(M, d_out, seed, p=0.5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(M, d_out, generator=g, device="cuda") < p


def bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def run(obs, w, b, eps, seed, legal=None, **kw):
    """(actions, q, q_max) of mlp_forward's ε-greedy head."""
    return mlp.mlp_forward(obs, *w, biases=b, output="epsilon_greedy", seed=seed, epsilon=eps, mask=legal, **kw)


def greedy(obs, w, b, legal=None):
    """(masked bf16 logits, greedy actions) of the greedy entry: the reference every output is tied to."""
    return mlp.mlp_forward(obs, *w, biases=b, output="both", mask=legal)


def gathered(logits, actions):
    return logits.float().gather(1, actions[:, None])[:, 0]


def explore_actions(seed, row0, rows, d_out, legal):
    """The host's exploratory action of each row: the legal column with the largest word, ties to the lower column."""
    _, w = explore_noise(seed, row0, rows, d_out, device="cuda")
    if legal is not None:
        w = w.masked_fill(~legal, -1)
    return w.argmax(-1)


def coin(seed, row0, rows, eps):
    u, _ = explore_noise(seed, row0, rows, 1, device="cuda")
    return u < eps


def same(got, want, what):
    for g, h in zip(got, want):
        if g.is_floating_point():
            g, h = bits(g), bits(h)
        assert torch.equal(g, h), what


# ---- 1. ε = 0: the greedy entry ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("biased", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("d_out", WIDTHS)
def test_epsilon_zero_is_the_greedy_entry(K, d_out, biased, masked):
    """ε = 0 (a tensor of zeros, and the float 0.0): actions are ktb_mlp_bf16_policy(_masked)'s greedy actions and
    q == q_max == its (masked) logits at the action, widened exactly."""
    w, b = config(100 + d_out, d_out, biased)
    M = 1000
    obs = randn((M, 256), 101 + d_out)
    legal = random_legal(M, d_out, 102 + d_out) if masked else None
    logits, g = greedy(obs, w, b, legal)
    want = (g, gathered(logits, g), gathered(logits, g))
    same(run(obs, w, b, torch.zeros(M, device="cuda"), 7, legal), want, "tensor")
    same(run(obs, w, b, 0.0, 7, legal), want, "float")


# ---- 2. ε = 1: the exploration stream ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("d_out", WIDTHS)
def test_epsilon_one_takes_the_host_exploration(K, d_out, masked):
    """ε = 1: every row explores; actions are the host's explore_noise ranking over the legal columns, q is the greedy
    entry's (masked) logits at those actions and q_max at its greedy action."""
    w, b = config(200 + d_out, d_out)
    M, seed, row0 = 1000, 2**33 + 5, 2**32 - 300
    obs = randn((M, 256), 201 + d_out)
    legal = random_legal(M, d_out, 202 + d_out) if masked else None
    logits, g = greedy(obs, w, b, legal)
    e = explore_actions(seed, row0, M, d_out, legal)
    same(run(obs, w, b, 1.0, seed, legal, row_offset=row0), (e, gathered(logits, e), gathered(logits, g)), d_out)


# ---- 3. mixed per-row ε ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("d_out", [1, 18, 64, 200])
def test_mixed_epsilon_follows_the_host_coin(K, d_out, masked):
    """Random per-row ε with 0, 1, -1, +inf, -inf, NaN and the smallest and largest grid points mixed in: each row is
    greedy or exploratory exactly as the host's coin u < ε says."""
    w, b = config(300 + d_out, d_out)
    M, seed = 4096, 31
    obs = randn((M, 256), 301)
    legal = random_legal(M, d_out, 302) if masked else None
    eps = torch.rand(M, generator=torch.Generator(device="cuda").manual_seed(303), device="cuda")
    special = torch.tensor([0.0, 1.0, -1.0, float("inf"), float("-inf"), float("nan"), 2.0 ** -24, 1 - 2.0 ** -24],
                           device="cuda")
    eps[::7] = special.repeat(M // 7 // 8 + 1)[:len(eps[::7])]
    logits, g = greedy(obs, w, b, legal)
    e = explore_actions(seed, 0, M, d_out, legal)
    a = torch.where(coin(seed, 0, M, eps), e, g)
    same(run(obs, w, b, eps, seed, legal), (a, gathered(logits, a), gathered(logits, g)), d_out)


# ---- 4. statistics over 2^20 rows ------------------------------------------------------------------------------------------
def _grid_probability(eps):
    """P(u < ε) for u = (2k + 1)·2^-24, k uniform in [0, 2^23): the count of grid points below fp32 ε over 2^23."""
    t = float(torch.tensor(eps, dtype=torch.float32)) * 2**24   # exact in fp64: 2k + 1 < t
    return min(2**23, max(0, math.ceil((t - 1) / 2))) / 2**23


@pytest.mark.parametrize("eps", [0.01, 0.05, 0.5])
def test_explore_frequency_is_the_grid_probability(K, eps):
    """Over 2^20 rows of a head whose greedy action is column 0 in every row (b3 puts +8 there): the actions are the
    host's exploratory ones on the rows its coin names and 0 elsewhere, and those rows' frequency is within 5 sigma of
    the exact grid probability."""
    M, d_out, seed = 1 << 20, 6, 41
    w, b = config(400, d_out)
    b3 = b[2].clone()
    b3[0] = 8.0
    obs = randn((M, 256), 401)
    actions, _, _ = run(obs, w, (b[0], b[1], b3), eps, seed)
    explored = coin(seed, 0, M, torch.tensor(eps, dtype=torch.float32, device="cuda"))
    assert torch.equal(actions, torch.where(explored, explore_actions(seed, 0, M, d_out, None), 0))
    p = _grid_probability(eps)
    n = int(explored.sum())
    sigma = (M * p * (1 - p)) ** 0.5
    assert abs(n - M * p) <= 5 * sigma, (n, M * p, sigma)


def test_exploratory_actions_are_uniform_over_the_legal_columns(K):
    """ε = 1 over 2^20 rows, four mask patterns cycled by row: per pattern, the counts of exploratory actions pass a
    chi-square test against uniform over its legal columns (p > 1e-4), and no illegal column is ever taken."""
    from scipy.stats import chisquare

    M, d_out, seed = 1 << 20, 18, 43
    w, b = config(500, d_out)
    obs = randn((M, 256), 501)
    patterns = torch.zeros(4, d_out, dtype=torch.bool, device="cuda")
    patterns[0] = True
    patterns[1, ::2] = True
    patterns[2, 5:8] = True
    patterns[3, 17] = True
    legal = patterns[torch.arange(M, device="cuda") % 4]
    actions, _, _ = run(obs, w, b, 1.0, seed, legal)
    assert bool(legal.gather(1, actions[:, None]).all())
    for k in range(4):
        cols = patterns[k].nonzero()[:, 0]
        counts = torch.bincount(actions[k::4], minlength=d_out)[cols].cpu().double()
        if len(cols) > 1:
            assert chisquare(counts.numpy()).pvalue > 1e-4, (k, counts)
        else:
            assert int(counts[0]) == M // 4


# ---- 5. edge rows ------------------------------------------------------------------------------------------------------------
def test_edge_rows(K):
    """No legal action: action 0 and q = q_max = -inf, greedy or exploring.  A NaN Q-value in a legal column is the
    greedy action and q_max, and does not change an exploring row's action; NaN and +inf in illegal columns change
    nothing; an all-true mask gives the unmasked bits."""
    M, d_out, seed = 512, 12, 51
    w, b = config(600, d_out)
    obs = randn((M, 256), 601)
    legal = random_legal(M, d_out, 602)
    legal[::5] = False
    for eps in (0.0, 1.0, 0.5):
        a, q, qm = run(obs, w, b, eps, seed, legal)
        none = ~legal.any(1)
        assert bool((a[none] == 0).all()) and bool((q[none] == float("-inf")).all())
        assert bool((qm[none] == float("-inf")).all())
    # a NaN Q-value in legal column 4 of every row (through b3)
    b3 = b[2].clone()
    b3[4] = float("nan")
    ones = torch.ones(M, d_out, dtype=torch.bool, device="cuda")
    a0, q0, m0 = run(obs, w, (b[0], b[1], b3), 0.0, seed, ones)
    assert bool((a0 == 4).all()) and bool(q0.isnan().all()) and bool(m0.isnan().all())
    a1, _, m1 = run(obs, w, (b[0], b[1], b3), 1.0, seed, ones)
    assert torch.equal(a1, explore_actions(seed, 0, M, d_out, None)) and bool(m1.isnan().all())
    # NaN and +inf in illegal columns 4 and 7: the bits of finite values there
    b3[7] = float("inf")
    illegal = legal.clone()
    illegal[:, 4] = illegal[:, 7] = False
    b3f = b[2].clone()
    for eps in (0.0, 0.3, 1.0):
        same(run(obs, w, (b[0], b[1], b3), eps, seed, illegal), run(obs, w, (b[0], b[1], b3f), eps, seed, illegal), eps)
        same(run(obs, w, b, eps, seed, ones), run(obs, w, b, eps, seed), ("all-true", eps))


# ---- 6. forms -----------------------------------------------------------------------------------------------------------------
def _fresh(M):
    return {"actions": torch.full((M,), -1, dtype=torch.int64, device="cuda"),
            "q": torch.full((M,), -1, dtype=torch.int32, device="cuda"),
            "q_max": torch.full((M,), -1, dtype=torch.int32, device="cuda")}


def _mixed_eps(M, seed):
    return torch.rand(M, generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda") * 0.6


@pytest.mark.parametrize("head", [EPS, EPS_MASKED], ids=["unmasked", "masked"])
@pytest.mark.parametrize("d_out", [18, 129])
def test_every_form_chunking_and_row_split_gives_identical_bits(K, head, d_out):
    """Repeat calls, chunk sizes 256 / 512 / shipped, plain and staged (pull kernel and copy engine), pushed through the
    rig with mask and ε side payloads (three calls with fresh inputs), and [0, s) + [s, M) with row_offset = s: the
    bits of one plain call.  ε and the mask are unchanged after every call."""
    w, b = config(700 + d_out, d_out)
    M, seed = SHIPPED_CHUNK + 1000, 77
    obs = randn((M, 256), 701)
    legal = random_legal(M, d_out, 702) if head is EPS_MASKED else None
    eps = _mixed_eps(M, 703)
    keep = eps.clone()
    want = run(obs, w, b, eps, seed, legal)
    same(run(obs, w, b, eps, seed, legal), want, "repeat")
    for chunk in (256, 512, SHIPPED_CHUNK):
        for ce in (None, 0, 1):
            with tuning(chunk, ce):
                same(run(obs, w, b, eps, seed, legal, staged=ce is not None), want, (chunk, ce))
    for split in (1, 1000, 16896, 16900):
        lo = run(obs[:split], w, b, eps[:split], seed, None if legal is None else legal[:split])
        hi = run(obs[split:], w, b, eps[split:], seed, None if legal is None else legal[split:], row_offset=split)
        same([torch.cat([x, y]) for x, y in zip(lo, hi)], want, split)
    assert torch.equal(eps, keep)
    Mp = 3 * 1408
    masked = [("mask", d_out)] if head is EPS_MASKED else []
    rig = PushRig(K, Mp, 256, 1024, 512, "ce", head, sides=masked + [("epsilon", 4)])
    for it in range(3):
        obs_p = randn((Mp, 256), 710 + it)
        legal_p = random_legal(Mp, d_out, 720 + it) if head is EPS_MASKED else None
        eps_p = _mixed_eps(Mp, 730 + it)
        want_p = run(obs_p, w, b, eps_p, seed, legal_p)
        out = _fresh(Mp)
        rig.call(obs_p, w, b, {k: t.data_ptr() for k, t in out.items()}, seed,
                 sides=dict(epsilon=eps_p, **({} if legal_p is None else dict(mask=legal_p))))
        torch.cuda.synchronize()
        same([out["actions"], out["q"].view(torch.float32), out["q_max"].view(torch.float32)], want_p, ("pushed", it))
    assert rig.statuses() == [0] * rig.n


@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
def test_package_push_path_on_one_gpu_matches_plain_bits(K, masked):
    """mlp_scatter_gather's pushed form (rows | mask | ε in each staging half, ktb_push_scatter_ce_sides, the root's shard
    on the side stream) with ranks [0, 0, 0] on cuda:0, back to back with fresh inputs, ε as a tensor and as a float:
    equal to one plain call over all rows."""
    devs, rows, d_out, seed = [0, 0, 0], 35072, 64, 9
    M = 3 * rows
    bounds = [K.shard_bounds(M, 3, r) for r in range(3)]
    w, b = config(800, d_out)
    weights = {0: (*w, *b)}
    for it, eps in enumerate((_mixed_eps(M, 801), 0.25, _mixed_eps(M, 802))):
        obs = randn((M, 256), 810 + it)
        legal = random_legal(M, d_out, 820 + it) if masked else None
        want = run(obs, w, b, eps, seed, legal)
        got = _fresh(M)
        eps_t = eps if isinstance(eps, torch.Tensor) else torch.full((M,), eps, device="cuda")
        mlp._mlp_scatter_gather_pushed(obs, devs, bounds, weights, "epsilon_greedy", None, got["actions"],
                                       got["q"].view(torch.float32), seed, None, legal,
                                       got["q_max"].view(torch.float32), None, None, eps_t)
        torch.cuda.synchronize()
        same([got["actions"], got["q"].view(torch.float32), got["q_max"].view(torch.float32)], want, it)
        pull = mlp.mlp_scatter_gather(obs, *w, devices=devs, transfer="pull", biases=b, output="epsilon_greedy",
                                      seed=seed, mask=legal, epsilon=eps)
        torch.cuda.synchronize()
        same([torch.cat([g[k] for g in pull]) for k in range(3)], want, ("pull", it))
    mlp._push_sessions[tuple(devs)].check()


# ---- 7. guard bands --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("head", [EPS, EPS_MASKED], ids=["unmasked", "masked"])
@pytest.mark.parametrize("form,M,chunk,d_out", [
    ("plain", 1000, SHIPPED_CHUNK, 7), ("plain", 1000, 256, 129), ("staged", 1408, 256, 18), ("pushed", 3 * 1408, 256, 7),
])
def test_writes_stay_inside_the_outputs(K, head, form, M, chunk, d_out):
    """actions, q, q_max, the scratch and the stage between guard bands; ε and the mask in guarded buffers are unchanged;
    the results equal mlp_forward's bit for bit."""
    seed = 5
    w, b = config(900, d_out)
    obs = randn((M, 256), 901)
    legal = random_legal(M, d_out, 902) if head is EPS_MASKED else None
    eps = _mixed_eps(M, 903)
    want = run(obs, w, b, eps, seed, legal)
    geps = Guarded(M * 4, 4)
    geps.view(torch.float32).copy_(eps)
    gmask = Guarded(M * d_out, 3)
    if legal is not None:
        gmask.view().copy_(legal.view(torch.uint8).flatten())
    bufs = {name: Guarded(M * row_bytes(d_out)) for name, row_bytes in head.outputs.items()}
    out = {name: buf.ptr() for name, buf in bufs.items()}
    with tuning(chunk):
        if form == "pushed":
            masked = [("mask", d_out)] if legal is not None else []
            rig = PushRig(K, M, 256, 1024, 512, "ce", head, sides=masked + [("epsilon", 4)])
            sides = dict(epsilon=geps.view(torch.float32), **({} if legal is None else dict(mask=gmask.view())))
            for _ in range(3):
                rig.call(obs, w, b, out, seed, sides=sides)
            torch.cuda.synchronize()
            assert rig.statuses() == [0] * rig.n
            bufs.update({f"stage[{r}]": rig.stage[r] for r in range(1, rig.n)})
            bufs.update({f"scratch[{r}]": rig.scratch[r] for r in range(1, rig.n)})
        else:
            bufs["scratch"] = Guarded(L.load().ktb_mlp_scratch_bytes(M, 1024))
            if form == "staged":
                bufs["stage"] = Guarded(L.load().ktb_mlp_stage_bytes(M, 256))
            L.call(*entry_args(head, named_args(obs, w, b, out, seed, mask=gmask.ptr(), epsilon=geps.ptr(),
                                                scratch=bufs["scratch"].ptr(),
                                                stage=bufs["stage"].ptr() if form == "staged" else None)))
    bufs["mask"], bufs["epsilon"] = gmask, geps
    for name, buf in bufs.items():
        buf.check(f"{form} M={M} chunk={chunk} d_out={d_out}: {name}")
    assert torch.equal(geps.view(torch.float32), eps)
    if legal is not None:
        assert torch.equal(gmask.view(), legal.view(torch.uint8).flatten())
    same([bufs["actions"].view(torch.int64), bufs["q"].view(torch.float32), bufs["q_max"].view(torch.float32)], want,
         form)


# ---- 8. status codes -------------------------------------------------------------------------------------------------------
_Z = {}


def _z(name, n, dtype=torch.float32):
    if name not in _Z:
        _Z[name] = torch.zeros(n, dtype=dtype, device="cuda")
    return _Z[name].data_ptr()


def _io():
    """ε, q and q_max of the status cases, and an all-legal mask, as large as any case uses."""
    return dict(epsilon=_z("epsilon", 4096), q=_z("q", 4096), q_max=_z("q_max", 4096),
                mask=_z("mask", 2048 * 512, torch.uint8) if "mask" in _Z else _ones_mask())


def _ones_mask():
    _Z["mask"] = torch.ones(2048 * 512, dtype=torch.uint8, device="cuda")
    return _Z["mask"].data_ptr()


ROWS_BYTES = 256 * 256 * 2      # the status cases' M * d_in * 2: where a pushed side region may begin
MASK_END = ROWS_BYTES + 256 * 18
STATUS_CASES = {
    "null_epsilon": (plain, dict(epsilon=0), L.ERR_ARG),
    "null_actions": (plain, dict(actions=0), L.ERR_ARG),
    "null_q": (plain, dict(q=0), L.ERR_ARG),
    "null_q_max": (plain, dict(q_max=0), L.ERR_ARG),
    "unaligned_epsilon": (plain, dict(epsilon_off=2), L.ERR_ARG),
    "unaligned_actions": (plain, dict(actions_off=4), L.ERR_ARG),
    "unaligned_q": (plain, dict(q_off=1), L.ERR_ARG),
    "unaligned_q_max": (plain, dict(q_max_off=2), L.ERR_ARG),
    "staged_null_epsilon": (plain, dict(epsilon=0, stage="zero"), L.ERR_ARG),
    "d_out_257": (plain, dict(d_out=257), L.ERR_UNSUPPORTED),
    "inherited_checks_first": (plain, dict(epsilon=0, q=0, d_out=257), L.ERR_UNSUPPORTED),
    "empty_call_takes_null_outputs": (plain, dict(M=0, epsilon=0, actions=0, q=0, q_max=0), None),
    "pushed_epsilon_over_the_rows": (pushed, dict(epsilon=ROWS_BYTES - 4), L.ERR_ARG),
    "pushed_epsilon_past_stage_stride": (pushed, dict(epsilon=(1 << 20) - 256 * 4 + 4), L.ERR_ARG),
    "pushed_epsilon_offset_past_stage_stride": (pushed, dict(epsilon=1 << 21), L.ERR_ARG),
    "pushed_epsilon_unaligned": (pushed, dict(epsilon=MASK_END + 258), L.ERR_ARG),
    "pushed_null_q": (pushed, dict(epsilon=MASK_END + 256, q=0), L.ERR_ARG),
    "pushed_d_out_257": (pushed, dict(epsilon=MASK_END + 256, d_out=257), L.ERR_UNSUPPORTED),
}
MASKED_ONLY = {
    "null_mask_first": (plain, dict(mask=0, epsilon=0), L.ERR_ARG),
    "pushed_epsilon_over_the_mask": (pushed, dict(mask=ROWS_BYTES, epsilon=ROWS_BYTES + 256), L.ERR_ARG),
    "pushed_epsilon_ends_in_the_mask": (pushed, dict(mask=ROWS_BYTES + 1020, epsilon=ROWS_BYTES), L.ERR_ARG),
    "pushed_mask_checks_first": (pushed, dict(mask=0, epsilon=0), L.ERR_ARG),
}


@pytest.mark.parametrize("head", [EPS, EPS_MASKED], ids=["unmasked", "masked"])
@pytest.mark.parametrize("name", list(STATUS_CASES) + list(MASKED_ONLY))
def test_bad_arguments_get_the_documented_status(K, head, name):
    if name in MASKED_ONLY and head is EPS:
        pytest.skip("a masked entry's case")
    form, overrides, status = {**STATUS_CASES, **MASKED_ONLY}[name]
    args = dict(_io(), **({"mask": MASK_END - 256 * 18} if form is pushed else {}))
    if form is pushed:
        args["epsilon"] = MASK_END + 256
    args.update(overrides)
    if args.get("stage") == "zero":
        args["stage"] = _z("stage", 1 << 24, torch.uint8)
    for name_off in [k for k in args if k.endswith("_off") and k[:-4] in ("epsilon", "q", "q_max")]:
        args[name_off[:-4]] = _io()[name_off[:-4]] + args.pop(name_off)
    call = form(head, **args)
    if status is None:
        L.call(*call)
        torch.cuda.synchronize()
    else:
        expect_status(call, status)


def _sides_args(n_sides=2, **overrides):
    """ktb_push_scatter_ce_sides over 3 × 256 rows of d_in 256 for ranks [0, 0, 0], call 1, stage_stride 1 MiB: a mask
    side (18 B per row) after the rows and an ε side (4 B per row) after it."""
    if "bufs" not in _Z:
        _Z["bufs"] = dict(obs=torch.zeros(768 * 256, dtype=torch.bfloat16, device="cuda"),
                          stage=torch.zeros(2 << 20, dtype=torch.uint8, device="cuda"),
                          ctrl=torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda"))
    z = _Z["bufs"]
    io = _io()
    a = dict(root_dev=0, n_elems=768 * 256, granule=256, n=3, chunk_elems=256 * 256, n_sides=n_sides,
             src=[io["mask"], io["epsilon"]], row_bytes=[18, 4], offsets=[ROWS_BYTES, MASK_END + 256], seq=1)
    a.update(overrides)
    stages = L.arr(ctypes.c_void_p, [0] + [z["stage"].data_ptr()] * 2)
    ctrls = L.arr(ctypes.c_void_p, [z["ctrl"].data_ptr()] * 3)
    arrays = (L.arr(ctypes.c_void_p, a["src"]), L.arr(ctypes.c_size_t, a["row_bytes"]),
              L.arr(ctypes.c_size_t, a["offsets"])) if a["src"] is not None else (None, None, None)
    return ("ktb_push_scatter_ce_sides", a["root_dev"], z["obs"].data_ptr(), a["n_elems"], a["granule"], L.BF16, a["n"],
            0, L.arr(ctypes.c_int, [0, 0, 0]), stages, 1 << 20, ctrls, z["ctrl"].data_ptr(), a["chunk_elems"],
            a["n_sides"], *arrays, a["seq"], stream())


SIDES_CASES = {
    "zero_sides": (dict(n_sides=0), L.ERR_ARG),
    "three_sides": (dict(n_sides=3), L.ERR_ARG),
    "null_arrays": (dict(src=None), L.ERR_ARG),
    "null_second_source": (dict(null_second=True), L.ERR_ARG),
    "zero_row_bytes": (dict(row_bytes=[18, 0]), L.ERR_ARG),
    "chunk_not_whole_rows": (dict(chunk_elems=256 * 256 + 1), L.ERR_ARG),
    "side_over_the_rows": (dict(offsets=[ROWS_BYTES, ROWS_BYTES - 4]), L.ERR_ARG),
    "side_past_stage_stride": (dict(offsets=[ROWS_BYTES, (1 << 20) - 256 * 4 + 4]), L.ERR_ARG),
    "sides_overlap": (dict(offsets=[ROWS_BYTES, MASK_END - 4]), L.ERR_ARG),
    "sides_overlap_reversed": (dict(offsets=[ROWS_BYTES + 1020, ROWS_BYTES]), L.ERR_ARG),
    "inherited_checks_first": (dict(n_sides=0, root_dev=15), L.ERR_STATE),
}


@pytest.mark.parametrize("name", list(SIDES_CASES))
def test_sides_scatter_bad_arguments_get_the_documented_status(K, name):
    overrides, status = SIDES_CASES[name]
    if overrides.get("null_second"):
        overrides = dict(src=[_io()["mask"], 0])
    expect_status(_sides_args(**overrides), status)


def test_masked_scatter_is_the_one_side_case(K):
    """ktb_push_scatter_ce_masked and ktb_push_scatter_ce_sides with the same one side land the same staging bytes."""
    M, d_in, d_out = 3 * 256, 256, 18
    obs = randn((M, d_in), 950)
    legal = random_legal(M, d_out, 951).view(torch.uint8)
    stride = 1 << 20
    got = []
    for entry in ("masked", "sides"):
        stage = torch.zeros(2 * stride, dtype=torch.uint8, device="cuda")
        ctrl = [torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda") for _ in range(3)]
        stages = L.arr(ctypes.c_void_p, [0, stage.data_ptr(), stage.data_ptr() + stride // 2])
        ctrls = L.arr(ctypes.c_void_p, [c.data_ptr() for c in ctrl])
        head = (0, obs.data_ptr(), obs.numel(), d_in, L.BF16, 3, 0, L.arr(ctypes.c_int, [0, 0, 0]), stages,
                stride // 2, ctrls, ctrl[0].data_ptr(), 256 * d_in)
        if entry == "masked":
            L.call("ktb_push_scatter_ce_masked", *head, legal.data_ptr(), d_out, ROWS_BYTES, 1, stream())
        else:
            L.call("ktb_push_scatter_ce_sides", *head, 1, L.arr(ctypes.c_void_p, [legal.data_ptr()]),
                   L.arr(ctypes.c_size_t, [d_out]), L.arr(ctypes.c_size_t, [ROWS_BYTES]), 1, stream())
        torch.cuda.synchronize()
        got.append(stage)
    assert torch.equal(got[0], got[1])
    base = stride // 2 + ROWS_BYTES   # rank 1's half 1 (call 1), mask after its 256 rows
    assert torch.equal(got[0][base:base + 256 * d_out], legal[256:512].flatten())


# ---- 9. the public API -------------------------------------------------------------------------------------------------------
def _public_case(masked, eps_kind):
    g = torch.Generator().manual_seed(91)
    d_out, M = 18, 2 * 1408 + 100
    p = [(torch.randn(1024, 256, generator=g) * 0.05).bfloat16(), (torch.randn(1024, generator=g) * 0.1).bfloat16(),
         (torch.randn(1024, 1024, generator=g) * 0.03).bfloat16(), (torch.randn(1024, generator=g) * 0.1).bfloat16(),
         (torch.randn(d_out, 1024, generator=g) * 0.05).bfloat16(), (torch.randn(d_out, generator=g) * 0.1).bfloat16()]
    obs = torch.randn(M, 256, generator=g).bfloat16()
    legal = torch.rand(M, d_out, generator=g) < 0.6 if masked else None
    eps = 0.2 if eps_kind == "float" else torch.rand(M, generator=g) * 0.4
    body = cases.mlp_policy_epsilon_greedy_masked if masked else cases.mlp_policy_epsilon_greedy
    policy = mapped_copy(body, "mlp", bias=True, output="epsilon_greedy", seed="seed", epsilon="eps",
                         **({"mask": "legal"} if masked else {}))
    return obs, p, legal, eps, 2**34 + 3, body, policy


def _args(obs, p, legal, eps, seed, cuda):
    c = (lambda t: t.cuda()) if cuda else (lambda t: t)   # noqa: E731
    tail = ((c(legal),) if legal is not None else ()) + (c(eps) if isinstance(eps, torch.Tensor) else eps,)
    return (c(obs), *[c(t) for t in p], *tail, seed)


def _against_body(K, obs, p, legal, eps, seed, got, want, n):
    """Each rank's outputs against the oracle's run of the body: exploring rows' actions are equal everywhere, greedy
    rows' actions wherever the body's fp32 top-2 gap exceeds 2^-6, and q and q_max agree at rtol 2^-7, atol 1e-2."""
    M = obs.shape[0]
    e = torch.full((M,), eps) if not isinstance(eps, torch.Tensor) else eps
    explored = (explore_noise(seed, 0, M, 1)[0] < e)
    for r, (g, h) in enumerate(zip(got, want)):
        lo, hi = K.shard_bounds(M, n, r)
        g, h = [t.cpu() for t in g], [t.cpu() for t in h]
        ex = explored[lo:hi]
        assert torch.equal(g[0][ex], h[0][ex]), r
        hb = torch.relu(F.linear(torch.relu(F.linear(obs[lo:hi], p[0], p[1])), p[2], p[3]))
        y = F.linear(hb, p[4], p[5]).float()
        if legal is not None:
            y = y.masked_fill(~legal[lo:hi], float("-inf"))
        top2 = y.topk(2, dim=1).values
        clear = ~ex & ((top2[:, 0] - top2[:, 1]) > 2.0 ** -6)
        assert torch.equal(g[0][clear], h[0][clear]), r
        for k in (1, 2):
            assert torch.allclose(g[k], h[k], rtol=2.0 ** -7, atol=1e-2, equal_nan=True), (r, k)


def _mine(obs, p, legal, eps, seed):
    pc = [t.cuda() for t in p]
    return mlp.mlp_forward(obs.cuda(), pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]), output="epsilon_greedy",
                           seed=seed, epsilon=eps.cuda() if isinstance(eps, torch.Tensor) else eps,
                           mask=None if legal is None else legal.cuda())


@pytest.mark.parametrize("eps_kind", ["float", "tensor"])
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["1_rank", "3_ranks"])
def test_mapped_epsilon_head_through_public_api(K, devices, masked, eps_kind):
    """@kt.mapped("mlp", bias=True, output="epsilon_greedy", seed="seed", epsilon="eps"[, mask="legal"]) on
    Compute(gpus=1): each rank returns the bits of mlp_forward over its rows, and agrees with the oracle's run of the
    body as _against_body states."""
    obs, p, legal, eps, seed, body, policy = _public_case(masked, eps_kind)
    n = len(devices)
    want = ref_dispatch.spmd_call(body, *_args(obs, p, legal, eps, seed, False), num_proc=n, serialization="pickle")
    mine = _mine(obs, p, legal, eps, seed)
    with deployed(policy, f"t-eps-{int(masked)}-{eps_kind}-{n}", devices) as remote:
        got = remote(*_args(obs, p, legal, eps, seed, True), serialization="pickle")
        torch.cuda.synchronize()
    assert len(got) == len(want) == n
    for r, g in enumerate(got):
        lo, hi = K.shard_bounds(obs.shape[0], n, r)
        assert isinstance(g, tuple) and len(g) == 3, r
        same([t.cpu() for t in g], [t[lo:hi].cpu() for t in mine], r)
    _against_body(K, obs, p, legal, eps, seed, got, want, n)


def test_mapped_epsilon_head_on_a_workers_subset(K):
    """Two workers of one rank each on cuda:0; a call with workers=[1] returns rank 1's outputs only, with the bits of
    mlp_forward over its rows."""
    import kubetorch_b200 as kt

    obs, p, legal, eps, seed, body, policy = _public_case(True, "tensor")
    mine = _mine(obs, p, legal, eps, seed)
    remote = kt.fn(policy, name="t-eps-workers").to(
        kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute("b200", workers=2, num_proc=1,
                                                                                 devices=[0, 0]))
    try:
        got = remote(*_args(obs, p, legal, eps, seed, True), serialization="pickle", workers=[1])
        torch.cuda.synchronize()
    finally:
        remote.teardown()
    lo, hi = K.shard_bounds(obs.shape[0], 2, 1)
    assert len(got) == 1
    same([t.cpu() for t in got[0]], [t[lo:hi].cpu() for t in mine], "workers=[1]")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("transfer", ["pull", "push"])
def test_mapped_epsilon_head_on_two_gpus(K, transfer):
    """Two ranks on two GPUs, staged pull and pushed form, three calls with fresh observations: the bits of one plain
    call."""
    obs, p, legal, eps, seed, body, policy = _public_case(True, "tensor")
    with deployed(policy, f"t-eps-2gpu-{transfer}", [0, 1], transfer=transfer) as remote:
        for it in range(3):
            x = torch.randn(2 * 1408, 256, generator=torch.Generator().manual_seed(5 + it)).bfloat16()
            lg = torch.rand(x.shape[0], 18, generator=torch.Generator().manual_seed(6 + it)) < 0.6
            e = torch.rand(x.shape[0], generator=torch.Generator().manual_seed(7 + it)) * 0.5
            got = remote(*_args(x, p, lg, e, seed, True), serialization="pickle")
            torch.cuda.synchronize(0)
            torch.cuda.synchronize(1)
            want = _mine(x, p, lg, e, seed)
            same([torch.cat([g[k].cpu() for g in got]) for k in range(3)], [t.cpu() for t in want], it)
