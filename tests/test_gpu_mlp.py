"""-m gpu: the bf16 policy MLP (ktb_mlp.cu, config C4) against an fp64 reference, layer by layer, at every shape class
the ABI accepts, on every entry point (plain, staged, pushed, the mapped op of the public API), with guard bands around
every buffer the kernels write and a check of every status code the ABI documents."""
import pytest
import torch

from conftest import mapped_copy
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp
from mlp_rig import (BIAS_FREE_64, NO_BIAS, SHIPPED_CHUNK, Guarded, K, PushRig, check_layer, chunk_rows,  # noqa: F401
                     config, deployed, exact_h1, expect_status, hidden_through_head, identity, layer_cases, plain,
                     pushed, randn, run_guarded, scaled_copies, tuning)

pytestmark = pytest.mark.gpu

from oracle import cases, ref_dispatch  # noqa: E402

D_OUT = 64


# ---- 1. layer-isolated checks with an exact criterion ---------------------------------------------------------------
# (d_in, d_hidden, M), a pairwise set: d_in 64..512 = 1..8 layer-1 K blocks against the 4-stage ring, each with d_hidden
# 256 and 1024; d_hidden 256..1280 = 1..5 N tiles and 4..20 K blocks, each with d_in 64 and 256; M from one row block to
# more than the shipped chunk, ragged (1000) included
SHAPES = [
    (64, 256, 128), (64, 1024, 384), (128, 256, 1000), (128, 1024, 17024), (192, 256, 384), (192, 1024, 1000),
    (256, 256, 17024), (256, 1024, 128), (320, 256, 1000), (320, 1024, 384), (512, 256, 128), (512, 1024, 1000),
    (64, 512, 17024), (64, 768, 128), (64, 1280, 1000), (256, 512, 384), (256, 768, 17024), (256, 1280, 384),
]


@pytest.mark.parametrize("layer", ["layer1", "layer2", "head"])
@pytest.mark.parametrize("d_in,d_hidden,M,chunk_rows", layer_cases(SHAPES), indirect=["chunk_rows"])
def test_layer_matches_fp64_within_one_rounding(K, layer, d_in, d_hidden, M, chunk_rows):
    seed = d_in * 100_003 + d_hidden * 101 + M
    what = f"{layer} d_in={d_in} d_hidden={d_hidden} M={M} chunk={chunk_rows or SHIPPED_CHUNK}"
    if layer == "layer1":            # W2 = I and a selection W3 pass h1 through exactly
        obs = randn((M, d_in), seed)
        w1 = randn((d_hidden, d_in), seed + 1, 0.1)
        got = hidden_through_head(obs, w1, identity(d_hidden), D_OUT)
        check_layer(got, obs, w1, None, True, what)
        return
    obs = randn((M, d_in), seed).abs()
    w1 = scaled_copies(d_in, d_hidden)
    h1 = exact_h1(obs, d_in, d_hidden)
    if layer == "layer2":            # h1 is known exactly; a selection W3 passes h2 through
        w2 = randn((d_hidden, d_hidden), seed + 2, 0.1)
        got = hidden_through_head(obs, w1, w2, D_OUT)
        check_layer(got, h1, w2, None, True, what)
    else:                            # W2 = I: h2 = h1 exactly; the head has no ReLU
        w3 = randn((D_OUT, d_hidden), seed + 3, 0.1)
        got = mlp.mlp_forward(obs, w1, identity(d_hidden), w3)
        check_layer(got, h1, w3, None, False, what)


# ---- end to end at the config's scale ---------------------------------------------------------------------------------
def _mlp_ref(obs, w1, w2, w3):
    """fp32 evaluation of the bf16 module with bf16 rounding between layers (what ATen does)."""
    h = torch.relu(obs.float() @ w1.float().t()).bfloat16()
    h = torch.relu(h.float() @ w2.float().t()).bfloat16()
    return (h.float() @ w3.float().t()).bfloat16()


def test_mlp_wgmma_matches_recorded_reference_and_fp32(K, golden):
    """bf16 MLP policy (config C4): tolerance rtol=2^-7, atol=1e-2 vs the reference runtime's CPU bf16 result and vs
    an fp32 evaluation (BASELINE.md §3); top-1 action equal wherever the fp32 top-2 gap exceeds 2^-6."""
    inp = golden["all_inputs"]
    obs, w1, w2, w3 = (inp[k].cuda() for k in ("mlp_obs", "mlp_w1", "mlp_w2", "mlp_w3"))
    got = mlp.mlp_forward(obs, w1, w2, w3).cpu().float()
    want_ref = torch.cat(golden["cases"]["mlp_bf16_256_x2"]["result"]).float()
    want_f32 = _mlp_ref(inp["mlp_obs"], inp["mlp_w1"], inp["mlp_w2"], inp["mlp_w3"]).float()
    torch.testing.assert_close(got, want_f32, rtol=2**-7, atol=1e-2)
    torch.testing.assert_close(got, want_ref, rtol=2**-7, atol=1e-2)
    # larger M (three row chunks, many tiles), random observations at the config's scale
    g = torch.Generator().manual_seed(7)
    obs2 = torch.randn(128 * 300, 256, generator=g).bfloat16()
    want2 = _mlp_ref(obs2, inp["mlp_w1"], inp["mlp_w2"], inp["mlp_w3"]).float()
    got2 = mlp.mlp_forward(obs2.cuda(), w1, w2, w3).cpu().float()
    torch.testing.assert_close(got2, want2, rtol=2**-7, atol=1e-2)
    top2 = want2.topk(2, dim=1).values
    clear = (top2[:, 0] - top2[:, 1]) > 2**-6
    assert torch.equal(got2.argmax(1)[clear], want2.argmax(1)[clear])


# ---- 3. one answer whatever the path --------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [16896 + 128, 1000])
def test_every_chunking_and_pull_gives_identical_bits(K, M):
    """Every 128 x N tile is computed the same way whatever the chunking, so the plain and staged forms (pulled by kernel
    or by copy engine, ktb_set_tuning 22) agree bit for bit at every chunk size."""
    w, _ = config(11, D_OUT, bias=False)
    obs = randn((M, 256), 13)
    want = mlp.mlp_forward(obs, *w)
    for chunk in (128, 256, 4096, SHIPPED_CHUNK):
        for ce in (None, 0, 1):      # plain, then staged pulled by kernel and by copy engine
            with tuning(chunk, ce):
                assert torch.equal(mlp.mlp_forward(obs, *w, staged=ce is not None), want), (chunk, ce)


# ---- 4. the pushed form on one GPU ------------------------------------------------------------------------------------
# 1408 rows per rank = five 256-row chunks and a 128-row tail
@pytest.mark.parametrize("engine", ["sm", "ce"])
def test_pushed_form_on_one_gpu_matches_plain_bits(K, engine):
    """ktb_mlp_bf16_pushed fed by ktb_push_scatter_chunked / ktb_push_scatter_ce, three consecutive calls (both
    staging halves, ack back-pressure): the logits equal mlp_forward over all rows bit for bit."""
    M, d_in, d_hidden = 3 * 1408, 256, 1024
    w, _ = config(21, D_OUT, bias=False)
    rig = PushRig(K, M, d_in, d_hidden, 256, engine, BIAS_FREE_64)
    for it in range(3):
        obs = randn((M, d_in), 100 + it)
        want = mlp.mlp_forward(obs, *w)
        logits = Guarded(M * D_OUT * 2)
        rig.call(obs, w, NO_BIAS, {"logits": logits.ptr()})
        torch.cuda.synchronize()
        assert torch.equal(logits.view(torch.bfloat16).view(M, D_OUT), want), (engine, it)
    assert rig.statuses() == [0] * rig.n


# ---- 5. guard bands -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form,M,chunk", [
    ("plain", 1000, SHIPPED_CHUNK), ("plain", 1408, 256), ("plain", 1000, 256),
    ("staged", 1000, SHIPPED_CHUNK), ("staged", 1408, 256), ("staged", 1000, 256),
    ("pushed", 3 * 1408, 256),
])
def test_writes_stay_inside_the_documented_buffers(K, form, M, chunk):
    """logits, scratch and stage sized exactly as include/ktb200.h documents, each between two bands of a byte pattern;
    the result also equals mlp_forward bit for bit.  The pushed case runs with ktb_set_tuning(8, 256) below its
    chunk_rows = 512, so a scratch sized by the tuning chunk would be too small for it."""
    w, _ = config(31, D_OUT, bias=False)
    obs = randn((M, 256), 33)
    want = mlp.mlp_forward(obs, *w)
    bufs = run_guarded(form, BIAS_FREE_64, K, chunk, obs, w, NO_BIAS)
    for name, buf in bufs.items():
        buf.check(f"{form} M={M} chunk={chunk}: {name}")
    assert torch.equal(bufs["logits"].view(torch.bfloat16).view(M, D_OUT), want)


# ---- 6. the public API ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["recorded", "ragged_1000_rows_3_ranks", "2_rows_3_ranks"])
def test_mapped_mlp_through_public_api(K, golden, case):
    """@kt.mapped("mlp") deployed on Compute(gpus=1) with its ranks on cuda:0, against the oracle's restatement of the
    reference call at the documented bf16 tolerance: shards of any row count, and empty shards."""
    inp = golden["all_inputs"]
    w = [inp[k] for k in ("mlp_w1", "mlp_w2", "mlp_w3")]
    if case == "recorded":
        obs, n_ranks = inp["mlp_obs"], 2
    else:
        rows, n_ranks = (1000, 3) if case.startswith("ragged") else (2, 3)
        obs = torch.randn(rows, 256, generator=torch.Generator().manual_seed(rows)).bfloat16()
    want = ref_dispatch.spmd_call(cases.mlp_policy, obs, *w, num_proc=n_ranks, serialization="pickle")
    with deployed(mapped_copy(cases.mlp_policy, "mlp"), f"t-mlp-{case}", [0] * n_ranks) as remote:
        got = remote(obs.cuda(), *[t.cuda() for t in w], serialization="pickle")
        torch.cuda.synchronize()
        assert len(got) == len(want) == n_ranks
        for r, (g, h) in enumerate(zip(got, want)):
            assert g.dtype == h.dtype and tuple(g.shape) == tuple(h.shape), (case, r)
            torch.testing.assert_close(g.cpu().float(), h.float(), rtol=2**-7, atol=1e-2)
        if case == "recorded":
            for g, h in zip(got, golden["cases"]["mlp_bf16_256_x2"]["result"]):
                torch.testing.assert_close(g.cpu().float(), h.float(), rtol=2**-7, atol=1e-2)


# ---- 7. argument checks ---------------------------------------------------------------------------------------------
STATUS_CASES = {
    "d_in_not_multiple_of_64": (plain, dict(d_in=96), L.ERR_ARG),
    "d_hidden_not_multiple_of_256": (plain, dict(d_hidden=384), L.ERR_ARG),
    "d_out_not_64": (plain, dict(d_out=128), L.ERR_UNSUPPORTED),
    "misaligned_obs": (plain, dict(obs_off=2), L.ERR_ARG),
    "misaligned_logits": (plain, dict(logits_off=8), L.ERR_ARG),
    "staged_null_stage": (plain, dict(stage=0), L.ERR_ARG),
    "staged_misaligned_stage": (plain, dict(stage_off=4), L.ERR_ARG),
    "pushed_more_than_64_chunks": (pushed, dict(M=65 * 128, chunk_rows=128, stride=1 << 24), L.ERR_ARG),
    "pushed_shard_exceeds_stage_stride": (pushed, dict(M=256, stride=256 * 256 * 2 - 256), L.ERR_ARG),
    "pushed_rows_not_multiple_of_128": (pushed, dict(M=200), L.ERR_ARG),
    "pushed_d_out_not_64": (pushed, dict(d_out=128), L.ERR_UNSUPPORTED),
    "pushed_stride_not_multiple_of_16": (pushed, dict(stride=(1 << 20) + 8), L.ERR_ARG),
    "pushed_stride_not_multiple_of_16_even_seq": (pushed, dict(stride=(1 << 20) + 8, seq=2), L.ERR_ARG),
}


@pytest.mark.parametrize("name", list(STATUS_CASES))
def test_bad_arguments_get_the_documented_status(K, name):
    form, overrides, status = STATUS_CASES[name]
    expect_status(form(BIAS_FREE_64, **overrides), status)
