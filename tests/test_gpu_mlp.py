"""-m gpu: the bf16 policy MLP (ktb_mlp.cu, config C4) against an fp64 reference, layer by layer, at every shape class
the ABI accepts, on every entry point (plain, staged, pushed, the mapped op of the public API), with guard bands around
every buffer the kernels write and a check of every status code the ABI documents."""
import ctypes

import pytest
import torch

from conftest import mapped_copy

pytestmark = pytest.mark.gpu

from oracle import cases, ref_dispatch  # noqa: E402

D_OUT = 64
SHIPPED_CHUNK = 16896          # ktb_set_tuning key 8 as the library ships it


@pytest.fixture(scope="module")
def K():
    assert torch.cuda.is_available()
    from kubetorch_b200.device import lib as L
    from kubetorch_b200.device import ops

    L.load()
    ops.ensure_init([0])
    return ops


def _L():
    from kubetorch_b200.device import lib as L

    return L


def _mlp():
    from kubetorch_b200.device import mlp

    return mlp


def _randn(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).bfloat16()


def _stream():
    return int(torch.cuda.current_stream(0).cuda_stream)


# ---- 1. layer-isolated checks with an exact criterion ---------------------------------------------------------------
def _bf16(t):
    """fp64 → fp32 → bf16, each step round-to-nearest-even: a monotone rounding to bf16 (identical to direct RNE except
    where the fp64 value lies within fp32 rounding distance of a bf16 tie)."""
    return t.float().bfloat16().float()


def _check_gemm(got, a, b, relu, what):
    """got[M, N] (bf16, from the kernel) must be act(a · bᵀ) rounded to bf16 from SOME value that fp32 accumulation of
    the exact bf16 × bf16 products could produce.  r = the exact result (fp64: every product is exact, the sum's error
    is far below the bound), e = K·2^-23·Σ|a_k·b_k| a deliberately generous bound on the fp32 accumulation error, and
    rounding is monotonic, so   bf16(act(r − e)) <= got <= bf16(act(r + e)).  For almost every element that admits
    exactly one bf16 value: at least 99.9 % must equal bf16(act(r))."""
    a64, b64 = a.double(), b.double()
    r = a64 @ b64.t()
    e = (a.shape[1] * 2.0 ** -23) * (a64.abs() @ b64.abs().t())
    act = (lambda t: t.clamp_min(0)) if relu else (lambda t: t)
    g = got.float()
    lo, hi = _bf16(act(r - e)), _bf16(act(r + e))
    bad = ~((lo <= g) & (g <= hi))          # NaN fails too
    if bool(bad.any()):
        idx = bad.nonzero()[:6].tolist()
        rows = [(i, j, float(g[i, j]), float(lo[i, j]), float(hi[i, j]), float(r[i, j])) for i, j in idx]
        pytest.fail(f"{what}: {int(bad.sum())} of {g.numel()} outputs outside [bf16(act(r-e)), bf16(act(r+e))]; "
                    f"(row, col, got, lo, hi, r): {rows}")
    exact = float((g == _bf16(act(r))).double().mean())
    print(f"{what}: {exact:.6f} of {g.numel()} outputs are the bf16 rounding of the fp64 result")
    assert exact >= 0.999, (what, exact)


def _identity(n):
    return torch.eye(n, device="cuda").bfloat16()


def _select(d_hidden, cols):
    """W3 that copies the hidden units `cols` (64 of them) to the logits: one product with 1.0, exact zeros."""
    w = torch.zeros(D_OUT, d_hidden, device="cuda")
    w[torch.arange(D_OUT, device="cuda"), cols] = 1.0
    return w.bfloat16()


def _copy_scales(d_in, d_hidden):
    """2^-(n // d_in) for every hidden unit n, exact (Python floats: a device pow need not be exact)."""
    return torch.tensor([2.0 ** -(n // d_in) for n in range(d_hidden)], dtype=torch.float64, device="cuda")


def _scaled_copies(d_in, d_hidden):
    """W1[n, n mod d_in] = 2^-(n // d_in): h1 = exactly scaled copies of (non-negative) obs, distinct per K block."""
    n = torch.arange(d_hidden, device="cuda")
    w = torch.zeros(d_hidden, d_in, dtype=torch.float64, device="cuda")
    w[n, n % d_in] = _copy_scales(d_in, d_hidden)
    return w.bfloat16()


def _hidden_through_head(obs, w1, w2):
    """The full hidden activation that the last layer sees, read out 64 units per call through a selection W3: every
    column of every 256-wide tile (every epilogue register pair and lane group) is observed."""
    d_hidden = w1.shape[0]
    mlp = _mlp()
    parts = [mlp.mlp_forward(obs, w1, w2, _select(d_hidden, torch.arange(t * 64, t * 64 + 64, device="cuda")))
             for t in range(d_hidden // 64)]
    return torch.cat(parts, dim=1)


# (d_in, d_hidden, M), a pairwise set: d_in 64..512 = 1..8 layer-1 K blocks against the 4-stage ring, each with d_hidden
# 256 and 1024; d_hidden 256..1280 = 1..5 N tiles and 4..20 K blocks, each with d_in 64 and 256; M from one row block to
# more than the shipped chunk, ragged (1000) included
SHAPES = [
    (64, 256, 128), (64, 1024, 384), (128, 256, 1000), (128, 1024, 17024), (192, 256, 384), (192, 1024, 1000),
    (256, 256, 17024), (256, 1024, 128), (320, 256, 1000), (320, 1024, 384), (512, 256, 128), (512, 1024, 1000),
    (64, 512, 17024), (64, 768, 128), (64, 1280, 1000), (256, 512, 384), (256, 768, 17024), (256, 1280, 384),
]
CHUNKED = (256, 1024, 5 * 256 + 128)   # with ktb_set_tuning(8, 256): five whole chunks and a 128-row last chunk


def _layer_cases():
    out = [pytest.param(*s, None, id=f"din{s[0]}-dh{s[1]}-M{s[2]}") for s in SHAPES]
    out.append(pytest.param(*CHUNKED, 256, id=f"din{CHUNKED[0]}-dh{CHUNKED[1]}-M{CHUNKED[2]}-chunk256"))
    return out


@pytest.fixture
def chunk_rows(K, request):
    chunk = request.param
    if chunk is not None:
        K.set_tuning(8, chunk)
    try:
        yield chunk
    finally:
        K.set_tuning(8, SHIPPED_CHUNK)


@pytest.mark.parametrize("layer", ["layer1", "layer2", "head"])
@pytest.mark.parametrize("d_in,d_hidden,M,chunk_rows", _layer_cases(), indirect=["chunk_rows"])
def test_layer_matches_fp64_within_one_rounding(K, layer, d_in, d_hidden, M, chunk_rows):
    seed = d_in * 100_003 + d_hidden * 101 + M
    what = f"{layer} d_in={d_in} d_hidden={d_hidden} M={M} chunk={chunk_rows or SHIPPED_CHUNK}"
    if layer == "layer1":            # W2 = I and a selection W3 pass h1 through exactly
        obs = _randn((M, d_in), seed)
        w1 = _randn((d_hidden, d_in), seed + 1, 0.1)
        got = _hidden_through_head(obs, w1, _identity(d_hidden))
        _check_gemm(got, obs, w1, True, what)
        return
    obs = _randn((M, d_in), seed).abs()
    w1 = _scaled_copies(d_in, d_hidden)
    h1_exact = obs.double()[:, torch.arange(d_hidden, device="cuda") % d_in] * _copy_scales(d_in, d_hidden)
    h1 = h1_exact.bfloat16()
    assert torch.equal(h1.double(), h1_exact)      # power-of-two scaling of bf16 values is exact
    if layer == "layer2":            # h1 is known exactly; a selection W3 passes h2 through
        w2 = _randn((d_hidden, d_hidden), seed + 2, 0.1)
        got = _hidden_through_head(obs, w1, w2)
        _check_gemm(got, h1, w2, True, what)
    else:                            # W2 = I: h2 = h1 exactly; the head has no ReLU
        w3 = _randn((D_OUT, d_hidden), seed + 3, 0.1)
        got = _mlp().mlp_forward(obs, w1, _identity(d_hidden), w3)
        _check_gemm(got, h1, w3, False, what)


# ---- end to end at the config's scale ---------------------------------------------------------------------------------
def _mlp_ref(obs, w1, w2, w3):
    """fp32 evaluation of the bf16 module with bf16 rounding between layers (what ATen does)."""
    h = torch.relu(obs.float() @ w1.float().t()).bfloat16()
    h = torch.relu(h.float() @ w2.float().t()).bfloat16()
    return (h.float() @ w3.float().t()).bfloat16()


def test_mlp_wgmma_matches_recorded_reference_and_fp32(K, golden):
    """bf16 MLP policy (config C4): tolerance rtol=2^-7, atol=1e-2 vs the reference runtime's CPU bf16 result and vs
    an fp32 evaluation (BASELINE.md §3); top-1 action equal wherever the fp32 top-2 gap exceeds 2^-6."""
    mlp = _mlp()
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
def _config_weights(seed):
    return (_randn((1024, 256), seed, 0.02), _randn((1024, 1024), seed + 1, 0.02), _randn((D_OUT, 1024), seed + 2, 0.02))


@pytest.mark.parametrize("M", [16896 + 128, 1000])
def test_every_chunking_and_pull_gives_identical_bits(K, M):
    """Every 128 x N tile is computed the same way whatever the chunking, so the plain and staged forms (pulled by kernel
    or by copy engine, ktb_set_tuning 22) agree bit for bit at every chunk size."""
    mlp = _mlp()
    w = _config_weights(11)
    obs = _randn((M, 256), 13)
    want = mlp.mlp_forward(obs, *w)
    try:
        for chunk in (128, 256, 4096, SHIPPED_CHUNK):
            K.set_tuning(8, chunk)
            assert torch.equal(mlp.mlp_forward(obs, *w), want), ("plain", chunk)
            for ce in (0, 1):
                K.set_tuning(22, ce)
                assert torch.equal(mlp.mlp_forward(obs, *w, staged=True), want), ("staged", chunk, ce)
    finally:
        K.set_tuning(8, SHIPPED_CHUNK)
        K.set_tuning(22, 0)


# ---- 4. the pushed form on one GPU ------------------------------------------------------------------------------------
class _Guarded:
    """An `nbytes` buffer inside a larger allocation whose bands before and after hold a byte pattern: a write past
    the buffer lands in memory the test owns and shows up as a changed band.  Each band is at least as large as the
    buffer (and 256-byte aligned), so even an overrun by a whole buffer stays inside memory the test owns."""

    FILL = 0xA5

    def __init__(self, nbytes):
        self.nbytes = int(nbytes)
        self.band = max(1 << 16, (self.nbytes + 255) // 256 * 256)
        self.raw = torch.full((self.nbytes + 2 * self.band,), self.FILL, dtype=torch.uint8, device="cuda")

    def ptr(self):
        return self.raw.data_ptr() + self.band

    def view(self, dtype=torch.uint8):
        return self.raw[self.band:self.band + self.nbytes].view(dtype)

    def check(self, what):
        torch.cuda.synchronize()
        for name, band in (("before", self.raw[:self.band]), ("after", self.raw[self.band + self.nbytes:])):
            changed = (band != self.FILL).nonzero()
            assert changed.numel() == 0, f"{what}: {changed.numel()} bytes changed in the band {name} the " \
                                         f"{self.nbytes}-byte buffer (first at band offset {int(changed[0])})"


class _PushRig:
    """What PushSession does for the map, for the MLP: ranks [0, 0, 0] on cuda:0 and ONE stream.  Every flag a kernel
    waits on is published by work enqueued before it on that stream (or on library streams that stream already waits
    for), so no wait can block.  Staging and scratch are guarded buffers of the documented sizes."""

    def __init__(self, K, M, d_in, d_hidden, chunk_rows, engine, n_ranks=3):
        L = _L()
        self.K, self.M, self.d_in, self.d_hidden, self.chunk_rows, self.engine = K, M, d_in, d_hidden, chunk_rows, engine
        self.n = n_ranks
        self.bounds = [K.shard_bounds(M, n_ranks, r) for r in range(n_ranks)]
        shard = max(e - b for b, e in self.bounds)
        self.stride = (shard * d_in * 2 + 255) // 256 * 256
        self.ctrl = [torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda")
                     for _ in range(n_ranks)]
        self.stage = [None] + [_Guarded(2 * self.stride) for _ in range(1, n_ranks)]
        self.scratch = [None] + [_Guarded(_mlp().pushed_scratch_bytes(e - b, d_hidden, chunk_rows))
                                 for b, e in self.bounds[1:]]
        torch.cuda.synchronize()
        self.seq = 0

    def call(self, obs, w, logits):
        L, mlp = _L(), _mlp()
        self.seq += 1
        seq, n, d_in, st = self.seq, self.n, self.d_in, _stream()
        stage_ptrs = L.arr(ctypes.c_void_p, [0] + [s.ptr() for s in self.stage[1:]])
        ctrl_ptrs = L.arr(ctypes.c_void_p, [c.data_ptr() for c in self.ctrl])
        if self.engine == "sm":
            L.call("ktb_push_scatter_chunked", 0, obs.data_ptr(), obs.numel(), d_in, L.BF16, n, 0, stage_ptrs,
                   self.stride, ctrl_ptrs, self.ctrl[0].data_ptr(), self.chunk_rows * d_in, 0, seq, st)
        else:
            L.call("ktb_push_scatter_ce", 0, obs.data_ptr(), obs.numel(), d_in, L.BF16, n, 0,
                   L.arr(ctypes.c_int, [0] * n), stage_ptrs, self.stride, ctrl_ptrs, self.ctrl[0].data_ptr(),
                   self.chunk_rows * d_in, seq, st)
        y = logits.ptr()
        for r in range(1, n):
            b, e = self.bounds[r]
            L.call("ktb_mlp_bf16_pushed", 0, self.stage[r].ptr(), self.stride, e - b, d_in, self.d_hidden, D_OUT,
                   w[0].data_ptr(), w[1].data_ptr(), w[2].data_ptr(), y + b * D_OUT * 2, self.scratch[r].ptr(),
                   self.ctrl[r].data_ptr(), self.ctrl[0].data_ptr(), r, self.chunk_rows, seq, st)
        b, e = self.bounds[0]
        mlp.mlp_forward(obs[b:e], *w, out=logits.view(torch.bfloat16).view(self.M, D_OUT)[b:e],
                        stream=torch.cuda.current_stream(0))
        L.call("ktb_push_wait", 0, self.ctrl[0].data_ptr(), n, 0, seq, st)

    def statuses(self):
        L = _L()
        out = []
        for c in self.ctrl:
            s = ctypes.c_uint(0)
            L.call("ktb_push_status", 0, c.data_ptr(), ctypes.byref(s))
            out.append(s.value)
        return out


# 1408 rows per rank = five 256-row chunks and a 128-row tail
@pytest.mark.parametrize("engine", ["sm", "ce"])
def test_pushed_form_on_one_gpu_matches_plain_bits(K, engine):
    """ktb_mlp_bf16_pushed fed by ktb_push_scatter_chunked / ktb_push_scatter_ce, three consecutive calls (both
    staging halves, ack back-pressure): the logits equal mlp_forward over all rows bit for bit."""
    M, d_in, d_hidden = 3 * 1408, 256, 1024
    w = _config_weights(21)
    rig = _PushRig(K, M, d_in, d_hidden, 256, engine)
    for it in range(3):
        obs = _randn((M, d_in), 100 + it)
        want = _mlp().mlp_forward(obs, *w)
        logits = _Guarded(M * D_OUT * 2)
        rig.call(obs, w, logits)
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
    L, mlp = _L(), _mlp()
    d_in, d_hidden = 256, 1024
    w = _config_weights(31)
    obs = _randn((M, d_in), 33)
    want = mlp.mlp_forward(obs, *w)
    K.set_tuning(8, chunk)
    try:
        logits = _Guarded(M * D_OUT * 2)
        buffers = {"logits": logits}
        if form == "pushed":
            rig = _PushRig(K, M, d_in, d_hidden, 512, "sm")
            for it in range(3):
                rig.call(obs, w, logits)
            torch.cuda.synchronize()
            assert rig.statuses() == [0] * rig.n
            buffers.update({f"stage[{r}]": rig.stage[r] for r in range(1, rig.n)})
            buffers.update({f"scratch[{r}]": rig.scratch[r] for r in range(1, rig.n)})
        else:
            scratch = _Guarded(L.load().ktb_mlp_scratch_bytes(M, d_hidden))
            buffers["scratch"] = scratch
            args = [0, obs.data_ptr(), M, d_in, d_hidden, D_OUT, w[0].data_ptr(), w[1].data_ptr(), w[2].data_ptr(),
                    logits.ptr(), scratch.ptr()]
            if form == "plain":
                L.call("ktb_mlp_bf16", *args, _stream())
            else:
                stage = _Guarded(L.load().ktb_mlp_stage_bytes(M, d_in))
                buffers["stage"] = stage
                L.call("ktb_mlp_bf16_staged", *args, stage.ptr(), _stream())
        for name, buf in buffers.items():
            buf.check(f"{form} M={M} chunk={chunk}: {name}")
        assert torch.equal(logits.view(torch.bfloat16).view(M, D_OUT), want)
    finally:
        K.set_tuning(8, SHIPPED_CHUNK)


# ---- 6. the public API ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["recorded", "ragged_1000_rows_3_ranks", "2_rows_3_ranks"])
def test_mapped_mlp_through_public_api(K, golden, case):
    """@kt.mapped("mlp") deployed on Compute(gpus=1) with its ranks on cuda:0, against the oracle's restatement of the
    reference call at the documented bf16 tolerance: shards of any row count, and empty shards."""
    import kubetorch_b200 as kt

    inp = golden["all_inputs"]
    w = [inp[k] for k in ("mlp_w1", "mlp_w2", "mlp_w3")]
    if case == "recorded":
        obs, n_ranks = inp["mlp_obs"], 2
    else:
        rows, n_ranks = (1000, 3) if case.startswith("ragged") else (2, 3)
        obs = torch.randn(rows, 256, generator=torch.Generator().manual_seed(rows)).bfloat16()
    want = ref_dispatch.spmd_call(cases.mlp_policy, obs, *w, num_proc=n_ranks, serialization="pickle")
    policy = mapped_copy(cases.mlp_policy, "mlp")
    remote = kt.fn(policy, name=f"t-mlp-{case}").to(
        kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute(
            "b200", workers=1, num_proc=n_ranks, devices=[0] * n_ranks))
    try:
        got = remote(obs.cuda(), *[t.cuda() for t in w], serialization="pickle")
        torch.cuda.synchronize()
        assert len(got) == len(want) == n_ranks
        for r, (g, h) in enumerate(zip(got, want)):
            assert g.dtype == h.dtype and tuple(g.shape) == tuple(h.shape), (case, r)
            torch.testing.assert_close(g.cpu().float(), h.float(), rtol=2**-7, atol=1e-2)
        if case == "recorded":
            for g, h in zip(got, golden["cases"]["mlp_bf16_256_x2"]["result"]):
                torch.testing.assert_close(g.cpu().float(), h.float(), rtol=2**-7, atol=1e-2)
    finally:
        remote.teardown()


# ---- 7. argument checks ---------------------------------------------------------------------------------------------
def _arg_case(K, name):
    L = _L()
    w1, w2, w3 = (torch.zeros(s, dtype=torch.bfloat16, device="cuda") for s in ((1024, 512), (1024, 1024), (128, 1024)))
    obs = torch.zeros(2048, 512, dtype=torch.bfloat16, device="cuda")
    out = torch.zeros(2048, 128, dtype=torch.bfloat16, device="cuda")
    scratch = torch.zeros(1 << 24, dtype=torch.uint8, device="cuda")
    ctrl = torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda")
    p = lambda t, off=0: t.data_ptr() + off   # noqa: E731

    def plain(M=256, d_in=256, d_hidden=1024, d_out=64, obs_off=0, out_off=0):
        return ("ktb_mlp_bf16", 0, p(obs, obs_off), M, d_in, d_hidden, d_out, p(w1), p(w2), p(w3), p(out, out_off),
                p(scratch), _stream())

    def pushed(M=256, chunk_rows=256, stride=1 << 20, d_out=64):
        return ("ktb_mlp_bf16_pushed", 0, p(scratch), stride, M, 256, 1024, d_out, p(w1), p(w2), p(w3), p(out),
                p(scratch), p(ctrl), p(ctrl), 1, chunk_rows, 1, _stream())

    table = {
        "d_in_not_multiple_of_64": (plain(d_in=96), L.ERR_ARG),
        "d_hidden_not_multiple_of_256": (plain(d_hidden=384), L.ERR_ARG),
        "d_out_not_64": (plain(d_out=128), L.ERR_UNSUPPORTED),
        "misaligned_obs": (plain(obs_off=2), L.ERR_ARG),
        "misaligned_logits": (plain(out_off=8), L.ERR_ARG),
        "staged_null_stage": (("ktb_mlp_bf16_staged",) + plain()[1:-1] + (0, _stream()), L.ERR_ARG),
        "staged_misaligned_stage": (("ktb_mlp_bf16_staged",) + plain()[1:-1] + (p(scratch, 4), _stream()), L.ERR_ARG),
        "pushed_more_than_64_chunks": (pushed(M=65 * 128, chunk_rows=128, stride=1 << 24), L.ERR_ARG),
        "pushed_shard_exceeds_stage_stride": (pushed(M=256, stride=256 * 256 * 2 - 256), L.ERR_ARG),
        "pushed_rows_not_multiple_of_128": (pushed(M=200), L.ERR_ARG),
        "pushed_d_out_not_64": (pushed(d_out=128), L.ERR_UNSUPPORTED),
    }
    return table[name]


@pytest.mark.parametrize("name", [
    "d_in_not_multiple_of_64", "d_hidden_not_multiple_of_256", "d_out_not_64", "misaligned_obs", "misaligned_logits",
    "staged_null_stage", "staged_misaligned_stage", "pushed_more_than_64_chunks", "pushed_shard_exceeds_stage_stride",
    "pushed_rows_not_multiple_of_128", "pushed_d_out_not_64",
])
def test_bad_arguments_get_the_documented_status(K, name):
    L = _L()
    args, status = _arg_case(K, name)
    with pytest.raises(L.KtbError) as ei:
        L.call(*args)
    assert ei.value.status == status, (name, str(ei.value))
    torch.cuda.synchronize()    # nothing was launched; the device stays healthy
