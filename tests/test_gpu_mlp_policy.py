"""-m gpu: the nn.Linear policy form of the bf16 MLP (ktb_mlp_bf16_policy*, mlp_layer_wgmma_kernel) against an fp64
reference layer by layer with biases, at every head width class from 1 to 256; its greedy actions against torch.argmax
of its own logits, with planted ties, NaN and infinities; bit identity with the 64-wide entries and across every
form; guard bands around every buffer it writes; the mapped op through the public API; and its status codes."""
import ctypes

import pytest
import torch

from conftest import mapped_copy
from test_gpu_mlp import CHUNKED, SHIPPED_CHUNK, _bf16, _copy_scales, _Guarded, _identity, _scaled_copies

pytestmark = pytest.mark.gpu

import policy_cases  # noqa: E402
from oracle import ref_dispatch  # noqa: E402


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


def _ptr(t):
    return 0 if t is None else t.data_ptr()


# ---- 1. per-layer bias bar --------------------------------------------------------------------------------------------
def _check_layer(got, a, b, bias, relu, what):
    """got[M, N] must be act(a · bᵀ + bias) rounded to bf16 from SOME value that fp32 accumulation of the exact products
    and the bias could produce: with r the fp64 result and e = (K+1)·2^-23·(Σ|a·b| + |bias|),
    bf16(act(r − e)) <= got <= bf16(act(r + e)), and at least 99.9 % of outputs equal bf16(act(r))."""
    a64, b64 = a.double(), b.double()
    r = a64 @ b64.t()
    s = a64.abs() @ b64.abs().t()
    if bias is not None:
        r = r + bias.double()
        s = s + bias.double().abs()
    e = ((a.shape[1] + 1) * 2.0 ** -23) * s
    act = (lambda t: t.clamp_min(0)) if relu else (lambda t: t)
    g = got.float()
    lo, hi = _bf16(act(r - e)), _bf16(act(r + e))
    bad = ~((lo <= g) & (g <= hi))
    if bool(bad.any()):
        idx = bad.nonzero()[:6].tolist()
        rows = [(i, j, float(g[i, j]), float(lo[i, j]), float(hi[i, j]), float(r[i, j])) for i, j in idx]
        pytest.fail(f"{what}: {int(bad.sum())} of {g.numel()} outputs outside [bf16(act(r-e)), bf16(act(r+e))]; "
                    f"(row, col, got, lo, hi, r): {rows}")
    exact = float((g == _bf16(act(r))).double().mean())
    print(f"{what}: {exact:.6f} of {g.numel()} outputs are the bf16 rounding of the fp64 result")
    assert exact >= 0.999, (what, exact)


def _select(d_hidden, cols):
    """A head that copies hidden units `cols` to the logits: one product with 1.0, exact zeros elsewhere."""
    w = torch.zeros(len(cols), d_hidden, device="cuda")
    w[torch.arange(len(cols), device="cuda"), cols] = 1.0
    return w.bfloat16()


def _hidden_through_head(obs, w1, b1, w2, b2):
    """The full second hidden activation, read out 256 units per call through a selection head of width 256."""
    d_hidden = w1.shape[0]
    parts = [_mlp().mlp_forward(obs, w1, w2, _select(d_hidden, torch.arange(t * 256, t * 256 + 256, device="cuda")),
                                biases=(b1, b2, None))
             for t in range(d_hidden // 256)]
    return torch.cat(parts, dim=1)


def _exact_h1(obs, d_in, d_hidden):
    """Non-negative obs through _scaled_copies: h1 known exactly (power-of-two scaling of bf16 values)."""
    h1_exact = obs.double()[:, torch.arange(d_hidden, device="cuda") % d_in] * _copy_scales(d_in, d_hidden)
    h1 = h1_exact.bfloat16()
    assert torch.equal(h1.double(), h1_exact)
    return h1


LAYER_SHAPES = [(64, 256, 128), (128, 256, 1000), (192, 1024, 1000), (256, 1024, 128), (512, 1024, 1000),
                (64, 1280, 1000), (256, 768, 17024)]


def _layer_cases():
    out = [pytest.param(*s, None, id=f"din{s[0]}-dh{s[1]}-M{s[2]}") for s in LAYER_SHAPES]
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
def test_biased_layer_matches_fp64_within_one_rounding(K, layer, d_in, d_hidden, M, chunk_rows):
    """Each layer with a random bias, the others exact pass-throughs (identity W2, selection head, no bias).  Biases are
    drawn like the weights (σ = 0.1); far larger biases cancel the products more often, which leaves more results
    within accumulation error of a bf16 rounding boundary (the bound then still holds, the 99.9 % share need not)."""
    seed = d_in * 100_003 + d_hidden * 101 + M + 7
    what = f"{layer} d_in={d_in} d_hidden={d_hidden} M={M} chunk={chunk_rows or SHIPPED_CHUNK}"
    if layer == "layer1":
        obs = _randn((M, d_in), seed)
        w1, b1 = _randn((d_hidden, d_in), seed + 1, 0.1), _randn((d_hidden,), seed + 4, 0.1)
        got = _hidden_through_head(obs, w1, b1, _identity(d_hidden), None)
        _check_layer(got, obs, w1, b1, True, what)
        return
    obs = _randn((M, d_in), seed).abs()
    w1 = _scaled_copies(d_in, d_hidden)
    h1 = _exact_h1(obs, d_in, d_hidden)
    if layer == "layer2":
        w2, b2 = _randn((d_hidden, d_hidden), seed + 2, 0.1), _randn((d_hidden,), seed + 5, 0.1)
        got = _hidden_through_head(obs, w1, None, w2, b2)
        _check_layer(got, h1, w2, b2, True, what)
    else:
        w3, b3 = _randn((256, d_hidden), seed + 3, 0.1), _randn((256,), seed + 6, 0.1)   # a 256-wide head
        got = _mlp().mlp_forward(obs, w1, _identity(d_hidden), w3, biases=(None, None, b3))
        _check_layer(got, h1, w3, b3, False, what)


# ---- 2. head widths, 3. actions -------------------------------------------------------------------------------------
HEAD_WIDTHS = [1, 2, 6, 18, 63, 64, 65, 100, 128, 129, 255, 256]


@pytest.mark.parametrize("d_out", HEAD_WIDTHS)
def test_head_width_bar_and_exact_actions(K, d_out):
    """The head at every tile class (64 / 128 / 256 wide, full and ragged): logits within the bias bar, actions equal
    torch.argmax of the kernel's own logits on every row, and the three output modes agree bit for bit.  At least
    64 000 outputs per width, so that the 99.9 % share is a statistic and not one or two outputs."""
    d_in, d_hidden, M = 256, 1024, max(1000, -(-64000 // d_out))
    obs = _randn((M, d_in), 41 + d_out).abs()
    w1 = _scaled_copies(d_in, d_hidden)
    h1 = _exact_h1(obs, d_in, d_hidden)
    w3, b3 = _randn((d_out, d_hidden), 43 + d_out, 0.1), _randn((d_out,), 45 + d_out, 0.1)
    mlp, w2 = _mlp(), _identity(d_hidden)
    logits, actions = mlp.mlp_forward(obs, w1, w2, w3, biases=(None, None, b3), output="both")
    _check_layer(logits, h1, w3, b3, False, f"head d_out={d_out}")
    assert actions.dtype == torch.int64 and actions.shape == (M,)
    assert torch.equal(actions, torch.argmax(logits, dim=-1))
    assert torch.equal(mlp.mlp_forward(obs, w1, w2, w3, biases=(None, None, b3), output="actions"), actions)
    assert torch.equal(mlp.mlp_forward(obs, w1, w2, w3, biases=(None, None, b3)), logits)


def _config(seed, d_out, bias=True):
    w = (_randn((1024, 256), seed, 0.02), _randn((1024, 1024), seed + 1, 0.02), _randn((d_out, 1024), seed + 2, 0.02))
    b = (_randn((1024,), seed + 3, 0.1), _randn((1024,), seed + 4, 0.1), _randn((d_out,), seed + 5, 0.1)) if bias \
        else (None, None, None)
    return w, b


@pytest.mark.parametrize("cols", [(3, 5), (2, 10), (60, 130), (1, 7, 200), (0, 255)],
                         ids=["quad-lanes", "same-lane-other-j", "across-64", "three-way", "first-last"])
def test_planted_ties_go_to_the_lowest_index(K, cols):
    """Duplicate W3 rows and biases, lifted above every other logit: an exact tie on every row, resolved to the
    lowest of the tied columns whether they sit in different lanes of a quad, in different register pairs of a
    lane, or across 64-column boundaries."""
    d_out, M = 256, 1000
    (w1, w2, w3), (b1, b2, b3) = _config(51, d_out)
    w3, b3 = w3.clone(), b3.clone()
    for c in cols:
        w3[c] = w3[cols[0]]
        b3[c] = 8.0
    obs = _randn((M, 256), 53)
    logits, actions = _mlp().mlp_forward(obs, w1, w2, w3, biases=(b1, b2, b3), output="both")
    assert bool((logits[:, list(cols)] == logits[:, [cols[0]]]).all())       # the tie is exact
    assert torch.equal(actions, torch.argmax(logits, dim=-1))
    assert bool((actions == min(cols)).all()), actions.unique()


@pytest.mark.parametrize("case", ["nan", "inf", "all_negative"])
def test_nan_inf_and_padding_never_mislead_the_argmax(K, case):
    """NaN in b3 at columns 5 and 9 → action 5 on every row (the first NaN wins); +inf at 7 and 100 → 7; and with
    b3 = -100 on a head of 18 (a 64-wide tile of which 46 columns are TMA zero fill) no padded column is ever chosen."""
    d_out = 18 if case == "all_negative" else 128
    (w1, w2, w3), (b1, b2, b3) = _config(61, d_out)
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
    obs = _randn((1000, 256), 63)
    mlp = _mlp()
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
    L, mlp = _L(), _mlp()
    (w1, w2, w3), _ = _config(71, 64, bias=False)
    obs = _randn((M, 256), 73)
    want = torch.empty(M, 64, dtype=torch.bfloat16, device="cuda")
    got = torch.empty_like(want)
    scratch = mlp._scratch_for(0, M, 1024)
    L.call("ktb_mlp_bf16", 0, obs.data_ptr(), M, 256, 1024, 64, w1.data_ptr(), w2.data_ptr(), w3.data_ptr(),
           want.data_ptr(), scratch.data_ptr(), _stream())
    L.call("ktb_mlp_bf16_policy", 0, obs.data_ptr(), M, 256, 1024, 64, w1.data_ptr(), 0, w2.data_ptr(), 0,
           w3.data_ptr(), 0, got.data_ptr(), 0, scratch.data_ptr(), 0, _stream())
    assert torch.equal(got, want)


@pytest.mark.parametrize("d_out", [18, 64, 200])
def test_every_chunking_and_pull_gives_identical_bits(K, d_out):
    """With biases and both outputs: the plain and staged forms (pulled by kernel or copy engine) at every chunk size."""
    mlp = _mlp()
    w, b = _config(81 + d_out, d_out)
    obs = _randn((16896 + 128 + 1000, 256), 83)
    want_l, want_a = mlp.mlp_forward(obs, *w, biases=b, output="both")
    try:
        for chunk in (128, 256, 4096, SHIPPED_CHUNK):
            K.set_tuning(8, chunk)
            got_l, got_a = mlp.mlp_forward(obs, *w, biases=b, output="both")
            assert torch.equal(got_l, want_l) and torch.equal(got_a, want_a), ("plain", chunk)
            for ce in (0, 1):
                K.set_tuning(22, ce)
                got_l, got_a = mlp.mlp_forward(obs, *w, biases=b, output="both", staged=True)
                assert torch.equal(got_l, want_l) and torch.equal(got_a, want_a), ("staged", chunk, ce)
    finally:
        K.set_tuning(8, SHIPPED_CHUNK)
        K.set_tuning(22, 0)


class _PolicyPushRig:
    """Ranks [0, 0, 0] on cuda:0 and one stream, as in test_gpu_mlp._PushRig, for ktb_mlp_bf16_policy_pushed: every
    flag a kernel waits on is published by work enqueued before it, so no wait can block."""

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

    def call(self, obs, w, b, d_out, logits_ptr, actions_ptr):
        """logits_ptr / actions_ptr: base addresses of the M-row results (0 = not wanted)."""
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
        for r in range(1, n):
            lo, hi = self.bounds[r]
            L.call("ktb_mlp_bf16_policy_pushed", 0, self.stage[r].ptr(), self.stride, hi - lo, d_in, self.d_hidden,
                   d_out, w[0].data_ptr(), _ptr(b[0]), w[1].data_ptr(), _ptr(b[1]), w[2].data_ptr(), _ptr(b[2]),
                   logits_ptr + lo * d_out * 2 if logits_ptr else 0, actions_ptr + lo * 8 if actions_ptr else 0,
                   self.scratch[r].ptr(), self.ctrl[r].data_ptr(), self.ctrl[0].data_ptr(), r, self.chunk_rows, seq, st)
        lo, hi = self.bounds[0]
        scratch = mlp._scratch_for(0, hi - lo, self.d_hidden)
        L.call("ktb_mlp_bf16_policy", 0, obs.data_ptr() + lo * d_in * 2, hi - lo, d_in, self.d_hidden, d_out,
               w[0].data_ptr(), _ptr(b[0]), w[1].data_ptr(), _ptr(b[1]), w[2].data_ptr(), _ptr(b[2]),
               logits_ptr + lo * d_out * 2 if logits_ptr else 0, actions_ptr + lo * 8 if actions_ptr else 0,
               scratch.data_ptr(), 0, st)
        L.call("ktb_push_wait", 0, self.ctrl[0].data_ptr(), n, 0, seq, st)

    def statuses(self):
        L = _L()
        out = []
        for c in self.ctrl:
            s = ctypes.c_uint(0)
            L.call("ktb_push_status", 0, c.data_ptr(), ctypes.byref(s))
            out.append(s.value)
        return out


@pytest.mark.parametrize("engine", ["sm", "ce"])
@pytest.mark.parametrize("chunk_rows", [256, 512])
def test_pushed_form_on_one_gpu_matches_plain_bits(K, engine, chunk_rows):
    """ktb_mlp_bf16_policy_pushed fed by either scatter engine, three consecutive calls: logits and actions equal the
    plain form's bit for bit, and every control block's status stays 0."""
    M, d_out = 3 * 1408, 18
    w, b = _config(91, d_out)
    rig = _PolicyPushRig(K, M, 256, 1024, chunk_rows, engine)
    for it in range(3):
        obs = _randn((M, 256), 93 + it)
        want_l, want_a = _mlp().mlp_forward(obs, *w, biases=b, output="both")
        logits = torch.full((M, d_out), float("nan"), dtype=torch.bfloat16, device="cuda")
        actions = torch.full((M,), -1, dtype=torch.int64, device="cuda")
        rig.call(obs, w, b, d_out, logits.data_ptr(), actions.data_ptr())
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
    mlp = _mlp()
    devs, rows, d_out = [0, 0, 0], 35072, 18
    M = 3 * rows
    bounds = [K.shard_bounds(M, 3, r) for r in range(3)]
    assert [e - b for b, e in bounds] == [rows] * 3 and rows == 2 * mlp.PUSH_CHUNK_ROWS + 1280
    w, b = _config(131, d_out)
    weights = {0: (*w, *b)}
    for it in range(3):
        obs = _randn((M, 256), 133 + it)
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
def _guarded(nbytes, misalign=0):
    """A _Guarded buffer whose start is moved `misalign` bytes past a 256-byte boundary."""
    g = _Guarded(nbytes)
    g.band += misalign
    return g


@pytest.mark.parametrize("form,M,chunk,d_out,misalign", [
    ("plain", 1000, SHIPPED_CHUNK, 7, 0), ("plain", 1000, 256, 7, 0), ("plain", 1000, 256, 18, 2),
    ("staged", 1000, SHIPPED_CHUNK, 7, 0), ("staged", 1000, 256, 129, 0), ("staged", 1408, 256, 18, 2),
    ("pushed", 3 * 1408, 256, 7, 0), ("pushed", 3 * 1408, 256, 18, 2),
])
def test_writes_stay_inside_the_documented_buffers(K, form, M, chunk, d_out, misalign):
    """logits (M·d_out·2 bytes, also at a 2-byte-aligned base), actions (M·8), scratch and stage sized as the header
    documents, each between two bands of a byte pattern, with odd head widths and ragged M; the results also equal
    mlp_forward bit for bit."""
    L, mlp = _L(), _mlp()
    d_in, d_hidden = 256, 1024
    w, b = _config(101, d_out)
    obs = _randn((M, d_in), 103)
    want_l, want_a = mlp.mlp_forward(obs, *w, biases=b, output="both")
    K.set_tuning(8, chunk)
    try:
        logits, actions = _guarded(M * d_out * 2, misalign), _Guarded(M * 8)
        buffers = {"logits": logits, "actions": actions}
        if form == "pushed":
            rig = _PolicyPushRig(K, M, d_in, d_hidden, 512, "sm")
            for _ in range(3):
                rig.call(obs, w, b, d_out, logits.ptr(), actions.ptr())
            torch.cuda.synchronize()
            assert rig.statuses() == [0] * rig.n
            buffers.update({f"stage[{r}]": rig.stage[r] for r in range(1, rig.n)})
            buffers.update({f"scratch[{r}]": rig.scratch[r] for r in range(1, rig.n)})
        else:
            scratch = _Guarded(L.load().ktb_mlp_scratch_bytes(M, d_hidden))
            buffers["scratch"] = scratch
            stage = 0
            if form == "staged":
                buffers["stage"] = _Guarded(L.load().ktb_mlp_stage_bytes(M, d_in))
                stage = buffers["stage"].ptr()
            L.call("ktb_mlp_bf16_policy", 0, obs.data_ptr(), M, d_in, d_hidden, d_out, w[0].data_ptr(), b[0].data_ptr(),
                   w[1].data_ptr(), b[1].data_ptr(), w[2].data_ptr(), b[2].data_ptr(), logits.ptr(), actions.ptr(),
                   scratch.ptr(), stage, _stream())
        for name, buf in buffers.items():
            buf.check(f"{form} M={M} chunk={chunk} d_out={d_out}: {name}")
        assert torch.equal(logits.view().view(torch.bfloat16).view(M, d_out), want_l)
        assert torch.equal(actions.view(torch.int64), want_a)
    finally:
        K.set_tuning(8, SHIPPED_CHUNK)


def test_actions_only_writes_no_logits(K):
    """output="actions": the logits buffer of the policy entry may be NULL and nothing else is written."""
    L, mlp = _L(), _mlp()
    M, d_out = 1000, 18
    w, b = _config(111, d_out)
    obs = _randn((M, 256), 113)
    want = mlp.mlp_forward(obs, *w, biases=b, output="actions")
    actions, scratch = _Guarded(M * 8), _Guarded(L.load().ktb_mlp_scratch_bytes(M, 1024))
    L.call("ktb_mlp_bf16_policy", 0, obs.data_ptr(), M, 256, 1024, d_out, w[0].data_ptr(), b[0].data_ptr(),
           w[1].data_ptr(), b[1].data_ptr(), w[2].data_ptr(), b[2].data_ptr(), 0, actions.ptr(), scratch.ptr(), 0,
           _stream())
    actions.check("actions only: actions")
    scratch.check("actions only: scratch")
    assert torch.equal(actions.view(torch.int64), want)


# ---- 6. the public API ----------------------------------------------------------------------------------------------
def _policy_weights(golden, d_out):
    """The recorded policy weights with random biases; heads other than 64 wide are random too."""
    inp = golden["all_inputs"]
    g = torch.Generator().manual_seed(d_out)
    w1, w2 = inp["mlp_w1"], inp["mlp_w2"]
    w3 = inp["mlp_w3"] if d_out == 64 else (torch.randn(d_out, 1024, generator=g) * 0.02).bfloat16()
    b1, b2, b3 = ((torch.randn(n, generator=g) * 0.1).bfloat16() for n in (1024, 1024, d_out))
    return w1, b1, w2, b2, w3, b3


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
    import kubetorch_b200 as kt

    if case == "recorded":
        obs, d_out = golden["all_inputs"]["mlp_obs"], 64
    else:
        rows = 1000 if case.startswith("ragged") else 2
        obs, d_out = torch.randn(rows, 256, generator=torch.Generator().manual_seed(rows)).bfloat16(), 6
    p = _policy_weights(golden, d_out)
    n_ranks = 3
    want = ref_dispatch.spmd_call(_CASE_FN[output], obs, *p, num_proc=n_ranks, serialization="pickle")
    policy = mapped_copy(_CASE_FN[output], "mlp", bias=True, output=output)
    remote = kt.fn(policy, name=f"t-policy-{case}-{output}").to(
        kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute(
            "b200", workers=1, num_proc=n_ranks, devices=[0] * n_ranks))
    try:
        got = remote(obs.cuda(), *[t.cuda() for t in p], serialization="pickle")
        torch.cuda.synchronize()
        assert len(got) == len(want) == n_ranks
        ref32 = _fp32_logits(obs, *p)
        for r, (g, h) in enumerate(zip(got, want)):
            lo, hi = K.shard_bounds(obs.shape[0], n_ranks, r)
            _check_rank(g, h, ref32[lo:hi], output, (case, output, r))
    finally:
        remote.teardown()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("transfer", ["pull", "push"])
def test_mapped_policy_on_two_gpus(K, golden, transfer):
    """Two ranks on two GPUs: the staged pull and the pushed form (peer-stored logits and actions)."""
    import kubetorch_b200 as kt

    obs = torch.randn(2 * 1408, 256, generator=torch.Generator().manual_seed(5)).bfloat16()
    p = _policy_weights(golden, 18)
    want = ref_dispatch.spmd_call(policy_cases.mlp_policy_both, obs, *p, num_proc=2, serialization="pickle")
    policy = mapped_copy(policy_cases.mlp_policy_both, "mlp", bias=True, output="both")
    remote = kt.fn(policy, name=f"t-policy-2gpu-{transfer}").to(
        kt.Compute(gpus=2, allowed_serialization=["json", "pickle"]).distribute(
            "b200", workers=1, num_proc=2, devices=[0, 1], transfer=transfer))
    try:
        got = remote(obs.cuda(0), *[t.cuda(0) for t in p], serialization="pickle")
        torch.cuda.synchronize(0)
        torch.cuda.synchronize(1)
        ref32 = _fp32_logits(obs, *p)
        for r, (g, h) in enumerate(zip(got, want)):
            lo, hi = K.shard_bounds(obs.shape[0], 2, r)
            _check_rank(g, h, ref32[lo:hi], "both", (transfer, r))
    finally:
        remote.teardown()


# ---- 7. argument statuses -------------------------------------------------------------------------------------------
def _arg_case(K, name):
    L = _L()
    w1, w2, w3 = (torch.zeros(s, dtype=torch.bfloat16, device="cuda") for s in ((1024, 256), (1024, 1024), (512, 1024)))
    bias = torch.zeros(1024, dtype=torch.bfloat16, device="cuda")
    obs = torch.zeros(2048, 256, dtype=torch.bfloat16, device="cuda")
    out = torch.zeros(2048, 512, dtype=torch.bfloat16, device="cuda")
    act = torch.zeros(2048, dtype=torch.int64, device="cuda")
    scratch = torch.zeros(1 << 24, dtype=torch.uint8, device="cuda")
    ctrl = torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda")
    p = lambda t, off=0: t.data_ptr() + off   # noqa: E731

    def plain(d_out=18, logits=None, actions=None, obs_off=0, b3_off=0, d_in=256, stage=0):
        return ("ktb_mlp_bf16_policy", 0, p(obs, obs_off), 256, d_in, 1024, d_out, p(w1), p(bias), p(w2), p(bias),
                p(w3), p(bias, b3_off), p(out) if logits is None else logits, p(act) if actions is None else actions,
                p(scratch), stage, _stream())

    def pushed(d_out=18, logits=None, actions=None, w2_off=0):
        return ("ktb_mlp_bf16_policy_pushed", 0, p(scratch), 1 << 20, 256, 256, 1024, d_out, p(w1), p(bias),
                p(w2, w2_off), p(bias), p(w3), p(bias), p(out) if logits is None else logits,
                p(act) if actions is None else actions, p(scratch), p(ctrl), p(ctrl), 1, 256, 1, _stream())

    table = {
        "d_out_0": (plain(d_out=0), L.ERR_ARG),
        "d_out_257": (plain(d_out=257), L.ERR_UNSUPPORTED),
        "both_outputs_null": (plain(logits=0, actions=0), L.ERR_ARG),
        "misaligned_actions": (plain(actions=p(act, 4)), L.ERR_ARG),
        "odd_logits": (plain(logits=p(out, 1)), L.ERR_ARG),
        "odd_bias": (plain(b3_off=1), L.ERR_ARG),
        "misaligned_obs": (plain(obs_off=2), L.ERR_ARG),
        "misaligned_stage": (plain(stage=p(scratch, 8)), L.ERR_ARG),
        "d_in_not_multiple_of_64": (plain(d_in=96), L.ERR_ARG),
        "pushed_d_out_0": (pushed(d_out=0), L.ERR_ARG),
        "pushed_d_out_257": (pushed(d_out=257), L.ERR_UNSUPPORTED),
        "pushed_both_outputs_null": (pushed(logits=0, actions=0), L.ERR_ARG),
        "pushed_misaligned_actions": (pushed(actions=p(act, 4)), L.ERR_ARG),
        "pushed_misaligned_w2": (pushed(w2_off=2), L.ERR_ARG),
    }
    return table[name]


@pytest.mark.parametrize("name", [
    "d_out_0", "d_out_257", "both_outputs_null", "misaligned_actions", "odd_logits", "odd_bias", "misaligned_obs",
    "misaligned_stage", "d_in_not_multiple_of_64", "pushed_d_out_0", "pushed_d_out_257", "pushed_both_outputs_null",
    "pushed_misaligned_actions", "pushed_misaligned_w2",
])
def test_bad_arguments_get_the_documented_status(K, name):
    L = _L()
    args, status = _arg_case(K, name)
    with pytest.raises(L.KtbError) as ei:
        L.call(*args)
    assert ei.value.status == status, (name, str(ei.value))
    torch.cuda.synchronize()    # nothing was launched; the device stays healthy


def test_python_checks_reach_the_public_api_as_value_errors(K):
    """Bias of the wrong length, or a head wider than 256: ValueError before any launch."""
    mlp = _mlp()
    (w1, w2, w3), (b1, b2, b3) = _config(121, 18)
    obs = _randn((256, 256), 123)
    with pytest.raises(ValueError):
        mlp.mlp_forward(obs, w1, w2, w3, biases=(b1, b2, b1))
    with pytest.raises(ValueError):
        mlp.mlp_forward(obs, w1, w2, _randn((257, 1024), 125), biases=(b1, b2, None))
    with pytest.raises(ValueError):
        mlp.mlp_scatter_gather(obs, w1, w2, w3, devices=[0, 0], biases=(b1.float(), b2, b3))
