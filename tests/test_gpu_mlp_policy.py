"""-m gpu: the nn.Linear policy form of the bf16 MLP (ktb_mlp_bf16_policy*, mlp_layer_wgmma_kernel) against an fp64
reference layer by layer with biases, at every head width class from 1 to 256; its greedy actions against torch.argmax
of its own logits, with planted ties, NaN and infinities; bit identity with the 64-wide entries and across every
form; guard bands around every buffer it writes; the mapped op through the public API; and its status codes."""
import pytest
import torch

from conftest import mapped_copy
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp
from mlp_rig import (BIAS_FREE_64, GREEDY, NO_BIAS, SHIPPED_CHUNK, Guarded, K, PushRig, check_layer,  # noqa: F401
                     chunk_rows, config, deployed, entry_args, exact_h1, expect_status, hidden_through_head, identity,
                     layer_cases, named_args, plain, policy_weights, pushed, randn, run_guarded, scaled_copies,
                     tuning)

pytestmark = pytest.mark.gpu

import policy_cases  # noqa: E402
from oracle import ref_dispatch  # noqa: E402


# ---- 1. per-layer bias bar --------------------------------------------------------------------------------------------
LAYER_SHAPES = [(64, 256, 128), (128, 256, 1000), (192, 1024, 1000), (256, 1024, 128), (512, 1024, 1000),
                (64, 1280, 1000), (256, 768, 17024)]


@pytest.mark.parametrize("layer", ["layer1", "layer2", "head"])
@pytest.mark.parametrize("d_in,d_hidden,M,chunk_rows", layer_cases(LAYER_SHAPES), indirect=["chunk_rows"])
def test_biased_layer_matches_fp64_within_one_rounding(K, layer, d_in, d_hidden, M, chunk_rows):
    """Each layer with a random bias, the others exact pass-throughs (identity W2, selection head, no bias).  Biases are
    drawn like the weights (σ = 0.1); far larger biases cancel the products more often, which leaves more results
    within accumulation error of a bf16 rounding boundary (the bound then still holds, the 99.9 % share need not)."""
    seed = d_in * 100_003 + d_hidden * 101 + M + 7
    what = f"{layer} d_in={d_in} d_hidden={d_hidden} M={M} chunk={chunk_rows or SHIPPED_CHUNK}"
    if layer == "layer1":
        obs = randn((M, d_in), seed)
        w1, b1 = randn((d_hidden, d_in), seed + 1, 0.1), randn((d_hidden,), seed + 4, 0.1)
        got = hidden_through_head(obs, w1, identity(d_hidden), 256, b1=b1)
        check_layer(got, obs, w1, b1, True, what)
        return
    obs = randn((M, d_in), seed).abs()
    w1 = scaled_copies(d_in, d_hidden)
    h1 = exact_h1(obs, d_in, d_hidden)
    if layer == "layer2":
        w2, b2 = randn((d_hidden, d_hidden), seed + 2, 0.1), randn((d_hidden,), seed + 5, 0.1)
        got = hidden_through_head(obs, w1, w2, 256, b2=b2)
        check_layer(got, h1, w2, b2, True, what)
    else:
        w3, b3 = randn((256, d_hidden), seed + 3, 0.1), randn((256,), seed + 6, 0.1)   # a 256-wide head
        got = mlp.mlp_forward(obs, w1, identity(d_hidden), w3, biases=(None, None, b3))
        check_layer(got, h1, w3, b3, False, what)


# ---- 2. head widths, 3. actions -------------------------------------------------------------------------------------
HEAD_WIDTHS = [1, 2, 6, 18, 63, 64, 65, 100, 128, 129, 255, 256]


@pytest.mark.parametrize("d_out", HEAD_WIDTHS)
def test_head_width_bar_and_exact_actions(K, d_out):
    """The head at every tile class (64 / 128 / 256 wide, full and ragged): logits within the bias bar, actions equal
    torch.argmax of the kernel's own logits on every row, and the three output modes agree bit for bit.  At least
    64 000 outputs per width, so that the 99.9 % share is a statistic and not one or two outputs."""
    d_in, d_hidden, M = 256, 1024, max(1000, -(-64000 // d_out))
    obs = randn((M, d_in), 41 + d_out).abs()
    w1 = scaled_copies(d_in, d_hidden)
    h1 = exact_h1(obs, d_in, d_hidden)
    w3, b3 = randn((d_out, d_hidden), 43 + d_out, 0.1), randn((d_out,), 45 + d_out, 0.1)
    w2 = identity(d_hidden)
    logits, actions = mlp.mlp_forward(obs, w1, w2, w3, biases=(None, None, b3), output="both")
    check_layer(logits, h1, w3, b3, False, f"head d_out={d_out}")
    assert actions.dtype == torch.int64 and actions.shape == (M,)
    assert torch.equal(actions, torch.argmax(logits, dim=-1))
    assert torch.equal(mlp.mlp_forward(obs, w1, w2, w3, biases=(None, None, b3), output="actions"), actions)
    assert torch.equal(mlp.mlp_forward(obs, w1, w2, w3, biases=(None, None, b3)), logits)


@pytest.mark.parametrize("cols", [(3, 5), (2, 10), (60, 130), (1, 7, 200), (0, 255)],
                         ids=["quad-lanes", "same-lane-other-j", "across-64", "three-way", "first-last"])
def test_planted_ties_go_to_the_lowest_index(K, cols):
    """Duplicate W3 rows and biases, lifted above every other logit: an exact tie on every row, resolved to the
    lowest of the tied columns whether they sit in different lanes of a quad, in different register pairs of a
    lane, or across 64-column boundaries."""
    d_out, M = 256, 1000
    (w1, w2, w3), (b1, b2, b3) = config(51, d_out)
    w3, b3 = w3.clone(), b3.clone()
    for c in cols:
        w3[c] = w3[cols[0]]
        b3[c] = 8.0
    obs = randn((M, 256), 53)
    logits, actions = mlp.mlp_forward(obs, w1, w2, w3, biases=(b1, b2, b3), output="both")
    assert bool((logits[:, list(cols)] == logits[:, [cols[0]]]).all())       # the tie is exact
    assert torch.equal(actions, torch.argmax(logits, dim=-1))
    assert bool((actions == min(cols)).all()), actions.unique()


@pytest.mark.parametrize("case", ["nan", "inf", "all_negative"])
def test_nan_inf_and_padding_never_mislead_the_argmax(K, case):
    """NaN in b3 at columns 5 and 9 → action 5 on every row (the first NaN wins); +inf at 7 and 100 → 7; and with
    b3 = -100 on a head of 18 (a 64-wide tile of which 46 columns are TMA zero fill) no padded column is ever chosen."""
    d_out = 18 if case == "all_negative" else 128
    (w1, w2, w3), (b1, b2, b3) = config(61, d_out)
    b3 = b3.clone()
    if case == "nan":
        b3[5] = b3[9] = float("nan")
        want = 5
    elif case == "inf":
        b3[7] = b3[100] = float("inf")
        want = 7
    else:
        b3.fill_(-100.0)
        want = None
    obs = randn((1000, 256), 63)
    logits, actions = mlp.mlp_forward(obs, w1, w2, w3, biases=(b1, b2, b3), output="both")
    only = mlp.mlp_forward(obs, w1, w2, w3, biases=(b1, b2, b3), output="actions")
    assert torch.equal(only, actions)
    assert torch.equal(actions, torch.argmax(logits, dim=-1))
    if want is not None:
        assert bool((actions == want).all()), actions.unique()
    else:
        assert bool((logits < 0).all()) and int(actions.max()) < d_out


# ---- 4. bit identity --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1000, 16896 + 128])
def test_bias_free_64_wide_logits_equal_the_original_entry(K, M):
    """ktb_mlp_bf16_policy with no biases, d_out = 64 and logits only equals ktb_mlp_bf16 bit for bit."""
    w, _ = config(71, 64, bias=False)
    obs = randn((M, 256), 73)
    want = torch.empty(M, 64, dtype=torch.bfloat16, device="cuda")
    got = torch.empty_like(want)
    scratch = mlp._scratch_for(0, M, 1024)
    for head, logits in ((BIAS_FREE_64, want), (GREEDY, got)):
        L.call(*entry_args(head, named_args(obs, w, NO_BIAS, {"logits": logits.data_ptr()},
                                            scratch=scratch.data_ptr())))
    assert torch.equal(got, want)


@pytest.mark.parametrize("d_out", [18, 64, 200])
def test_every_chunking_and_pull_gives_identical_bits(K, d_out):
    """With biases and both outputs: the plain and staged forms (pulled by kernel or copy engine) at every chunk size."""
    w, b = config(81 + d_out, d_out)
    obs = randn((16896 + 128 + 1000, 256), 83)
    want_l, want_a = mlp.mlp_forward(obs, *w, biases=b, output="both")
    for chunk in (128, 256, 4096, SHIPPED_CHUNK):
        for ce in (None, 0, 1):      # plain, then staged pulled by kernel and by copy engine
            with tuning(chunk, ce):
                got_l, got_a = mlp.mlp_forward(obs, *w, biases=b, output="both", staged=ce is not None)
            assert torch.equal(got_l, want_l) and torch.equal(got_a, want_a), (chunk, ce)


@pytest.mark.parametrize("engine", ["sm", "ce"])
@pytest.mark.parametrize("chunk_rows", [256, 512])
def test_pushed_form_on_one_gpu_matches_plain_bits(K, engine, chunk_rows):
    """ktb_mlp_bf16_policy_pushed fed by either scatter engine, three consecutive calls: logits and actions equal the
    plain form's bit for bit, and every control block's status stays 0."""
    M, d_out = 3 * 1408, 18
    w, b = config(91, d_out)
    rig = PushRig(K, M, 256, 1024, chunk_rows, engine, GREEDY)
    for it in range(3):
        obs = randn((M, 256), 93 + it)
        want_l, want_a = mlp.mlp_forward(obs, *w, biases=b, output="both")
        logits = torch.full((M, d_out), float("nan"), dtype=torch.bfloat16, device="cuda")
        actions = torch.full((M,), -1, dtype=torch.int64, device="cuda")
        rig.call(obs, w, b, {"logits": logits.data_ptr(), "actions": actions.data_ptr()})
        torch.cuda.synchronize()
        assert torch.equal(logits, want_l) and torch.equal(actions, want_a), (engine, chunk_rows, it)
    assert rig.statuses() == [0] * rig.n


@pytest.mark.parametrize("output", ["logits", "actions", "both"])
def test_package_push_path_on_one_gpu_matches_plain_bits(K, output):
    """The package's pushed form (what mlp_scatter_gather(transfer="push") runs: a cached PushSession, copy-engine
    scatter, the root's shard on the session's side stream) with ranks [0, 0, 0] on cuda:0.  35 072 rows per rank = two
    full 16 896-row push chunks and a 1 280-row tail; biases; three consecutive calls (both staging halves, ack
    back-pressure).  Ranks 1 and 2 run beside the root's shard on one device, so each needs its own scratch.  The
    results equal mlp_forward over all rows bit for bit, and the session's status stays clean."""
    devs, rows, d_out = [0, 0, 0], 35072, 18
    M = 3 * rows
    bounds = [K.shard_bounds(M, 3, r) for r in range(3)]
    assert [e - b for b, e in bounds] == [rows] * 3 and rows == 2 * mlp.PUSH_CHUNK_ROWS + 1280
    w, b = config(131, d_out)
    weights = {0: (*w, *b)}
    for it in range(3):
        obs = randn((M, 256), 133 + it)
        want_l, want_a = mlp.mlp_forward(obs, *w, biases=b, output="both")
        logits = None if output == "actions" else \
            torch.full((M, d_out), float("nan"), dtype=torch.bfloat16, device="cuda")
        actions = None if output == "logits" else torch.full((M,), -1, dtype=torch.int64, device="cuda")
        mlp._mlp_scatter_gather_pushed(obs, devs, bounds, weights, output, logits, actions)
        torch.cuda.synchronize()
        if logits is not None:
            assert torch.equal(logits, want_l), (output, it)
        if actions is not None:
            assert torch.equal(actions, want_a), (output, it)
    mlp._push_sessions[tuple(devs)].check()


# ---- 5. guard bands -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form,M,chunk,d_out,misalign", [
    ("plain", 1000, SHIPPED_CHUNK, 7, 0), ("plain", 1000, 256, 7, 0), ("plain", 1000, 256, 18, 2),
    ("staged", 1000, SHIPPED_CHUNK, 7, 0), ("staged", 1000, 256, 129, 0), ("staged", 1408, 256, 18, 2),
    ("pushed", 3 * 1408, 256, 7, 0), ("pushed", 3 * 1408, 256, 18, 2),
])
def test_writes_stay_inside_the_documented_buffers(K, form, M, chunk, d_out, misalign):
    """logits (M·d_out·2 bytes, also at a 2-byte-aligned base), actions (M·8), scratch and stage sized as the header
    documents, each between two bands of a byte pattern, with odd head widths and ragged M; the results also equal
    mlp_forward bit for bit."""
    w, b = config(101, d_out)
    obs = randn((M, 256), 103)
    want_l, want_a = mlp.mlp_forward(obs, *w, biases=b, output="both")
    bufs = run_guarded(form, GREEDY, K, chunk, obs, w, b, offsets={"logits": misalign})
    for name, buf in bufs.items():
        buf.check(f"{form} M={M} chunk={chunk} d_out={d_out}: {name}")
    assert torch.equal(bufs["logits"].view(torch.bfloat16).view(M, d_out), want_l)
    assert torch.equal(bufs["actions"].view(torch.int64), want_a)


def test_actions_only_writes_no_logits(K):
    """output="actions": the logits buffer of the policy entry may be NULL and nothing else is written."""
    M, d_out = 1000, 18
    w, b = config(111, d_out)
    obs = randn((M, 256), 113)
    want = mlp.mlp_forward(obs, *w, biases=b, output="actions")
    actions, scratch = Guarded(M * 8), Guarded(L.load().ktb_mlp_scratch_bytes(M, 1024))
    L.call(*entry_args(GREEDY, named_args(obs, w, b, {"actions": actions.ptr()}, scratch=scratch.ptr())))
    actions.check("actions only: actions")
    scratch.check("actions only: scratch")
    assert torch.equal(actions.view(torch.int64), want)


# ---- 6. the public API ----------------------------------------------------------------------------------------------
def _fp32_logits(obs, w1, b1, w2, b2, w3, b3):
    h = torch.relu(obs.float() @ w1.float().t() + b1.float()).bfloat16()
    h = torch.relu(h.float() @ w2.float().t() + b2.float()).bfloat16()
    return h.float() @ w3.float().t() + b3.float()


_CASE_FN = {"logits": policy_cases.mlp_policy_biased, "actions": policy_cases.mlp_policy_actions,
            "both": policy_cases.mlp_policy_both}


def _check_rank(g, want, ref32, output, what):
    """One rank's result against the oracle's: logits at the bf16 tolerance, actions wherever the fp32 top-2 gap
    exceeds 2^-6 (elsewhere bf16 rounding may legitimately pick another column)."""
    logits = g[0] if output == "both" else g if output == "logits" else None
    actions = g[1] if output == "both" else g if output == "actions" else None
    want_l = want[0] if output == "both" else want if output == "logits" else None
    if logits is not None:
        assert logits.dtype == torch.bfloat16 and tuple(logits.shape) == tuple(want_l.shape), what
        torch.testing.assert_close(logits.cpu().float(), want_l.float(), rtol=2**-7, atol=1e-2)
    if actions is not None:
        assert actions.dtype == torch.int64 and tuple(actions.shape) == (ref32.shape[0],), what
        if ref32.shape[0]:
            top2 = ref32.topk(2, dim=1).values
            clear = (top2[:, 0] - top2[:, 1]) > 2**-6
            assert torch.equal(actions.cpu()[clear], ref32.argmax(1)[clear]), what
        if logits is not None:
            assert torch.equal(actions, torch.argmax(logits, dim=-1)), what


@pytest.mark.parametrize("output", ["logits", "actions", "both"])
@pytest.mark.parametrize("case", ["recorded", "ragged_1000_rows_3_ranks", "2_rows_3_ranks"])
def test_mapped_policy_through_public_api(K, golden, case, output):
    """@kt.mapped("mlp", bias=True, output=...) on Compute(gpus=1) with three ranks on cuda:0, against the oracle's
    restatement of the reference call: unaligned shard offsets (1000 rows at d_out = 6), empty shards, and the
    recorded observations."""
    if case == "recorded":
        obs, d_out = golden["all_inputs"]["mlp_obs"], 64
    else:
        rows = 1000 if case.startswith("ragged") else 2
        obs, d_out = torch.randn(rows, 256, generator=torch.Generator().manual_seed(rows)).bfloat16(), 6
    p = policy_weights(golden, d_out)
    n_ranks = 3
    want = ref_dispatch.spmd_call(_CASE_FN[output], obs, *p, num_proc=n_ranks, serialization="pickle")
    policy = mapped_copy(_CASE_FN[output], "mlp", bias=True, output=output)
    with deployed(policy, f"t-policy-{case}-{output}", [0] * n_ranks) as remote:
        got = remote(obs.cuda(), *[t.cuda() for t in p], serialization="pickle")
        torch.cuda.synchronize()
        assert len(got) == len(want) == n_ranks
        ref32 = _fp32_logits(obs, *p)
        for r, (g, h) in enumerate(zip(got, want)):
            lo, hi = K.shard_bounds(obs.shape[0], n_ranks, r)
            _check_rank(g, h, ref32[lo:hi], output, (case, output, r))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("transfer", ["pull", "push"])
def test_mapped_policy_on_two_gpus(K, golden, transfer):
    """Two ranks on two GPUs: the staged pull and the pushed form (peer-stored logits and actions)."""
    obs = torch.randn(2 * 1408, 256, generator=torch.Generator().manual_seed(5)).bfloat16()
    p = policy_weights(golden, 18)
    want = ref_dispatch.spmd_call(policy_cases.mlp_policy_both, obs, *p, num_proc=2, serialization="pickle")
    policy = mapped_copy(policy_cases.mlp_policy_both, "mlp", bias=True, output="both")
    with deployed(policy, f"t-policy-2gpu-{transfer}", [0, 1], transfer=transfer) as remote:
        got = remote(obs.cuda(0), *[t.cuda(0) for t in p], serialization="pickle")
        torch.cuda.synchronize(0)
        torch.cuda.synchronize(1)
        ref32 = _fp32_logits(obs, *p)
        for r, (g, h) in enumerate(zip(got, want)):
            lo, hi = K.shard_bounds(obs.shape[0], 2, r)
            _check_rank(g, h, ref32[lo:hi], "both", (transfer, r))


# ---- 7. argument statuses -------------------------------------------------------------------------------------------
STATUS_CASES = {
    "d_out_0": (plain, dict(d_out=0), L.ERR_ARG),
    "d_out_257": (plain, dict(d_out=257), L.ERR_UNSUPPORTED),
    "both_outputs_null": (plain, dict(logits=0, actions=0), L.ERR_ARG),
    "misaligned_actions": (plain, dict(actions_off=4), L.ERR_ARG),
    "odd_logits": (plain, dict(logits_off=1), L.ERR_ARG),
    "odd_bias": (plain, dict(b3_off=1), L.ERR_ARG),
    "misaligned_obs": (plain, dict(obs_off=2), L.ERR_ARG),
    "misaligned_stage": (plain, dict(stage_off=8), L.ERR_ARG),
    "d_in_not_multiple_of_64": (plain, dict(d_in=96), L.ERR_ARG),
    "pushed_d_out_0": (pushed, dict(d_out=0), L.ERR_ARG),
    "pushed_d_out_257": (pushed, dict(d_out=257), L.ERR_UNSUPPORTED),
    "pushed_both_outputs_null": (pushed, dict(logits=0, actions=0), L.ERR_ARG),
    "pushed_misaligned_actions": (pushed, dict(actions_off=4), L.ERR_ARG),
    "pushed_misaligned_w2": (pushed, dict(w2_off=2), L.ERR_ARG),
    "pushed_stride_not_multiple_of_16": (pushed, dict(stride=(1 << 20) + 8), L.ERR_ARG),
    "pushed_stride_not_multiple_of_16_even_seq": (pushed, dict(stride=(1 << 20) + 8, seq=2), L.ERR_ARG),
}


@pytest.mark.parametrize("name", list(STATUS_CASES))
def test_bad_arguments_get_the_documented_status(K, name):
    form, overrides, status = STATUS_CASES[name]
    expect_status(form(GREEDY, **overrides), status)


def test_python_checks_reach_the_public_api_as_value_errors(K):
    """Bias of the wrong length, or a head wider than 256: ValueError before any launch."""
    (w1, w2, w3), (b1, b2, b3) = config(121, 18)
    obs = randn((256, 256), 123)
    with pytest.raises(ValueError):
        mlp.mlp_forward(obs, w1, w2, w3, biases=(b1, b2, b1))
    with pytest.raises(ValueError):
        mlp.mlp_forward(obs, w1, w2, randn((257, 1024), 125), biases=(b1, b2, None))
    with pytest.raises(ValueError):
        mlp.mlp_scatter_gather(obs, w1, w2, w3, devices=[0, 0], biases=(b1.float(), b2, b3))
