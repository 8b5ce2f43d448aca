"""-m gpu: the sampling head of the bf16 MLP policy (ktb_mlp_bf16_policy_sample*, output="sample") — its Gumbel-max
actions and log-probabilities against fp64 restatements built from the kernel's own logits, its distribution against
softmax by a chi-square test, bit identity across chunkings, forms, row offsets and repeat calls, seeds, planted NaN /
infinite / masked rows, guard bands, status codes, and the mapped op through the public API."""
import ctypes

import pytest
import torch

from conftest import mapped_copy
from test_gpu_mlp import SHIPPED_CHUNK, _Guarded, _identity
from test_gpu_mlp_policy import _PolicyPushRig, _config, _policy_weights, _randn, _stream

pytestmark = pytest.mark.gpu

import policy_sample_cases  # noqa: E402
from oracle import ref_dispatch  # noqa: E402

from kubetorch_b200.sampling import gumbel_uniform  # noqa: E402


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


def _ptr(t):
    return 0 if t is None else t.data_ptr()


# ---- the bars ----------------------------------------------------------------------------------------------------------
def _lse64(y):
    return torch.logsumexp(y.double(), dim=-1)


def _check_sample(y, seed, row0, actions, log_probs, what, row_ids=None):
    """y: the kernel's own bf16 logits of global rows row0, row0 + 1, ... (or of global rows `row_ids`), all finite.
    With s64 = y + g64 (g64 in fp64 from the exact u) and ε = 2^-18·(1 + max|s64|) per row: s64[a] >= max s64 - ε
    on every row; a = argmax s64 wherever the top-2 gap exceeds ε, on at least 99.9 % of the rows; and
    |log_prob - (y_a - logsumexp64(y))| <= (d_out + 8)·2^-22·(1 + |ref|)."""
    M, d_out = y.shape
    assert actions.dtype == torch.int64 and actions.shape == (M,), what
    assert log_probs.dtype == torch.float32 and log_probs.shape == (M,), what
    assert bool(torch.isfinite(y.float()).all()), what
    a = actions.to(y.device)
    assert bool(((a >= 0) & (a < d_out)).all()), (what, a.min(), a.max())
    if row_ids is None:
        u = gumbel_uniform(seed, row0, M, d_out, device=y.device).double()
    else:
        u = gumbel_uniform(seed, 0, int(row_ids.max()) + 1, d_out, device=y.device).double()[row_ids]
    s64 = y.double() - torch.log(-torch.log(u))
    eps = 2.0 ** -18 * (1 + s64.abs().amax(dim=1))
    top = s64.amax(dim=1)
    chosen = s64.gather(1, a[:, None]).squeeze(1)
    bad = chosen < top - eps
    assert not bool(bad.any()), (what, int(bad.sum()), bad.nonzero()[:4].tolist())
    if d_out > 1:
        top2 = s64.topk(2, dim=1).values
        clear = (top2[:, 0] - top2[:, 1]) > eps
    else:
        clear = torch.ones(M, dtype=torch.bool, device=y.device)
    assert float(clear.double().mean()) >= 0.999, (what, float(clear.double().mean()))
    assert torch.equal(a[clear], s64.argmax(dim=1)[clear]), what
    ref = y.double().gather(1, a[:, None]).squeeze(1) - _lse64(y)
    err = (log_probs.to(y.device).double() - ref).abs()
    tol = (d_out + 8) * 2.0 ** -22 * (1 + ref.abs())
    assert bool((err <= tol).all()), (what, float((err / tol).max()))


def _sample(obs, w, b, seed, **kw):
    return _mlp().mlp_forward(obs, *w, biases=b, output="sample", seed=seed, **kw)


def _logits(obs, w, b):
    return _mlp().mlp_forward(obs, *w, biases=b, output="logits")


# ---- 1. the bars at every head width -----------------------------------------------------------------------------------
@pytest.mark.parametrize("d_out", [1, 6, 18, 64, 129, 200, 256])
@pytest.mark.parametrize("chunk", [256, SHIPPED_CHUNK])
def test_sample_bars_at_every_head_width(K, d_out, chunk):
    """17 901 rows: more than one chunk at either chunk size, and a partial last tile; a seed past 2^32; logits of a
    few units so that the draws are far from uniform."""
    M, seed = SHIPPED_CHUNK + 1005, 2**33 + 7 * d_out
    w, b = _config(200 + d_out, d_out)
    w = (w[0], w[1], w[2] * 50)
    obs = _randn((M, 256), 210 + d_out)
    K.set_tuning(8, chunk)
    try:
        y = _logits(obs, w, b)
        actions, log_probs = _sample(obs, w, b, seed)
    finally:
        K.set_tuning(8, SHIPPED_CHUNK)
    _check_sample(y, seed, 0, actions, log_probs, f"d_out={d_out} chunk={chunk}")


# ---- 2. the distribution -----------------------------------------------------------------------------------------------
def test_draws_follow_softmax_and_never_pick_masked_columns(K):
    """W3 = 0 and b3 a fixed logit vector with two -inf (masked) columns: every row has the distribution softmax(b3).
    2^20 rows at a fixed seed: the masked columns get no draws and a chi-square goodness-of-fit test over the others
    gives p > 1e-4; every log-probability equals log_softmax(b3)[a] within the bar."""
    from scipy.stats import chisquare

    b3v = [1.0, 0.5, float("-inf"), 0.0, 2.0, -1.0, float("-inf"), 0.25, -3.0, 1.5]
    d_out, M = len(b3v), 1 << 20
    (w1, w2, _), (b1, b2, _) = _config(300, d_out)
    w3 = torch.zeros(d_out, 1024, dtype=torch.bfloat16, device="cuda")
    b3 = torch.tensor(b3v, dtype=torch.bfloat16, device="cuda")
    obs = _randn((M, 256), 301)
    actions, log_probs = _sample(obs, (w1, w2, w3), (b1, b2, b3), 20240611)
    counts = torch.bincount(actions, minlength=d_out).cpu()
    assert counts.numel() == d_out and int(counts[2]) == 0 and int(counts[6]) == 0, counts.tolist()
    p = torch.softmax(b3.double().cpu(), -1)
    live = p > 0
    stat = chisquare(counts[live].double().numpy(), (p[live] * M).numpy())
    print(f"chi-square over {int(live.sum())} columns: stat={stat.statistic:.2f} p={stat.pvalue:.4f}")
    assert stat.pvalue > 1e-4, (stat, counts.tolist())
    ref = torch.log_softmax(b3.double(), -1)[actions]
    tol = (d_out + 8) * 2.0 ** -22 * (1 + ref.abs())
    assert bool(((log_probs.double() - ref).abs() <= tol).all())


# ---- 3. identical bits ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d_out", [18, 200])
def test_every_chunking_form_and_row_split_gives_identical_bits(K, d_out):
    """Repeat calls, chunk sizes 256 / 512 / shipped, plain and staged (kernel or copy-engine pull), and one call over
    M rows against two calls over [0, b) and [b, M) with row_offset = b."""
    w, b = _config(400 + d_out, d_out)
    M, seed = SHIPPED_CHUNK + 1000, 77
    obs = _randn((M, 256), 401)
    want_a, want_lp = _sample(obs, w, b, seed)
    again = _sample(obs, w, b, seed)
    assert torch.equal(again[0], want_a) and torch.equal(again[1], want_lp)
    try:
        for chunk in (256, 512, SHIPPED_CHUNK):
            K.set_tuning(8, chunk)
            a, lp = _sample(obs, w, b, seed)
            assert torch.equal(a, want_a) and torch.equal(lp, want_lp), ("plain", chunk)
            for ce in (0, 1):
                K.set_tuning(22, ce)
                a, lp = _sample(obs, w, b, seed, staged=True)
                assert torch.equal(a, want_a) and torch.equal(lp, want_lp), ("staged", chunk, ce)
    finally:
        K.set_tuning(8, SHIPPED_CHUNK)
        K.set_tuning(22, 0)
    for split in (1, 1000, 16896, 16900):
        a0, lp0 = _sample(obs[:split], w, b, seed)
        a1, lp1 = _sample(obs[split:], w, b, seed, row_offset=split)
        assert torch.equal(torch.cat([a0, a1]), want_a) and torch.equal(torch.cat([lp0, lp1]), want_lp), split
    shifted = _sample(obs, w, b, seed, row_offset=5)
    assert not torch.equal(shifted[0], want_a)


class _SamplePushRig(_PolicyPushRig):
    """_PolicyPushRig driving ktb_mlp_bf16_policy_sample_pushed; rank r's row_base is its shard's begin."""

    def call(self, obs, w, b, d_out, seed, actions_ptr, log_probs_ptr):
        L = _L()
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
            L.call("ktb_mlp_bf16_policy_sample_pushed", 0, self.stage[r].ptr(), self.stride, hi - lo, d_in,
                   self.d_hidden, d_out, w[0].data_ptr(), _ptr(b[0]), w[1].data_ptr(), _ptr(b[1]), w[2].data_ptr(),
                   _ptr(b[2]), seed, lo, actions_ptr + lo * 8, log_probs_ptr + lo * 4, self.scratch[r].ptr(),
                   self.ctrl[r].data_ptr(), self.ctrl[0].data_ptr(), r, self.chunk_rows, seq, st)
        lo, hi = self.bounds[0]
        scratch = _mlp()._scratch_for(0, hi - lo, self.d_hidden)
        L.call("ktb_mlp_bf16_policy_sample", 0, obs.data_ptr() + lo * d_in * 2, hi - lo, d_in, self.d_hidden, d_out,
               w[0].data_ptr(), _ptr(b[0]), w[1].data_ptr(), _ptr(b[1]), w[2].data_ptr(), _ptr(b[2]), seed, lo,
               actions_ptr + lo * 8, log_probs_ptr + lo * 4, scratch.data_ptr(), 0, st)
        L.call("ktb_push_wait", 0, self.ctrl[0].data_ptr(), n, 0, seq, st)


@pytest.mark.parametrize("engine", ["sm", "ce"])
def test_pushed_form_on_one_gpu_matches_plain_bits(K, engine):
    """ktb_mlp_bf16_policy_sample_pushed fed by either scatter engine with ranks [0, 0, 0] on cuda:0, three consecutive
    calls with fresh observations: the actions and log-probabilities equal one plain call over all rows, bit for bit."""
    M, d_out, seed = 3 * 1408, 18, 2**40 + 3
    w, b = _config(500, d_out)
    rig = _SamplePushRig(K, M, 256, 1024, 512, engine)
    for it in range(3):
        obs = _randn((M, 256), 501 + it)
        want_a, want_lp = _sample(obs, w, b, seed)
        actions = torch.full((M,), -1, dtype=torch.int64, device="cuda")
        log_probs = torch.full((M,), float("nan"), dtype=torch.float32, device="cuda")
        rig.call(obs, w, b, d_out, seed, actions.data_ptr(), log_probs.data_ptr())
        torch.cuda.synchronize()
        assert torch.equal(actions, want_a) and torch.equal(log_probs, want_lp), (engine, it)
    assert rig.statuses() == [0] * rig.n


def test_package_push_path_on_one_gpu_matches_plain_bits(K):
    """mlp_scatter_gather's pushed form (a cached PushSession, copy-engine scatter, the root's shard on the side
    stream) with ranks [0, 0, 0] on cuda:0 and output="sample": equal to one plain call over all rows."""
    mlp = _mlp()
    devs, rows, d_out, seed = [0, 0, 0], 35072, 64, 9
    M = 3 * rows
    bounds = [K.shard_bounds(M, 3, r) for r in range(3)]
    w, b = _config(510, d_out)
    weights = {0: (*w, *b)}
    for it in range(2):
        obs = _randn((M, 256), 511 + it)
        want_a, want_lp = _sample(obs, w, b, seed)
        actions = torch.full((M,), -1, dtype=torch.int64, device="cuda")
        log_probs = torch.full((M,), float("nan"), dtype=torch.float32, device="cuda")
        mlp._mlp_scatter_gather_pushed(obs, devs, bounds, weights, "sample", None, actions, log_probs, seed)
        torch.cuda.synchronize()
        assert torch.equal(actions, want_a) and torch.equal(log_probs, want_lp), it
    mlp._push_sessions[tuple(devs)].check()


# ---- 4. seeds ------------------------------------------------------------------------------------------------------------
def test_nearby_seeds_draw_different_actions(K):
    """On a near-uniform 64-wide head, seeds s, s + 1 and s + 2^32 agree on about 1/64 of the rows only."""
    (w1, w2, _), (b1, b2, _) = _config(600, 64)
    w3 = torch.zeros(64, 1024, dtype=torch.bfloat16, device="cuda")
    b3 = torch.zeros(64, dtype=torch.bfloat16, device="cuda")
    obs = _randn((8192, 256), 601)
    s = 123456789
    draws = [_sample(obs, (w1, w2, w3), (b1, b2, b3), seed)[0] for seed in (s, s + 1, s + 2**32)]
    for i in range(3):
        for j in range(i + 1, 3):
            same = float((draws[i] == draws[j]).double().mean())
            assert same < 0.05, (i, j, same)


# ---- 5. planted rows -----------------------------------------------------------------------------------------------------
def test_planted_nan_inf_and_masked_rows(K):
    """Identity hidden layers pass non-negative observations through exactly, so trigger units of 2^100 reach the
    head, where products of 2^200 overflow: +inf at columns 1 and 5 (action 1), every column -inf (action 0, as
    torch.argmax), -inf at columns 0 and 2 only (never drawn), and an all-zero row (±0 logits).  NaN logits come from
    b3 (NaN at columns 3 and 6: action 3, the first NaN, on every row; an inf - inf inside the GEMM is not a reliable
    way to plant one).  log_prob is NaN exactly where torch's log_softmax is."""
    d, d_out, M, big = 256, 8, 4096, 2.0 ** 100
    obs = (torch.rand(M, d, generator=torch.Generator(device="cuda").manual_seed(7), device="cuda") * 0.5)
    obs[:, 176:] = 0
    w3 = torch.randn(d_out, d, generator=torch.Generator(device="cuda").manual_seed(8), device="cuda") * 0.5
    w3[:, 176:] = 0
    w3[1, 255] = w3[5, 255] = big                       # +inf trigger
    w3[:, 252] = -big                                   # all -inf trigger
    w3[0, 251] = w3[2, 251] = -big                      # masked columns trigger
    kinds = {"inf": [255], "all_neg_inf": [252], "masked": [251]}
    rows = {}
    for k, (kind, units) in enumerate(kinds.items()):
        idx = torch.arange(k, M, 8, device="cuda")
        rows[kind] = idx
        for u in units:
            obs[idx, u] = big
    zero = torch.arange(7, M, 8, device="cuda")
    obs[zero] = 0
    obs, w3 = obs.bfloat16(), w3.bfloat16()
    w = (_identity(d), _identity(d), w3)
    b = (None, None, None)
    y = _logits(obs, w, b)
    actions, log_probs = _sample(obs, w, b, 31)
    yf = y.float()
    assert bool(torch.isposinf(yf[rows["inf"]][:, [1, 5]]).all())
    assert bool(torch.isneginf(yf[rows["all_neg_inf"]]).all())
    assert bool(torch.isneginf(yf[rows["masked"]][:, [0, 2]]).all())
    assert bool((yf[zero] == 0).all())
    assert bool((actions[rows["inf"]] == 1).all()), actions[rows["inf"]].unique()
    assert bool((actions[rows["all_neg_inf"]] == 0).all()), actions[rows["all_neg_inf"]].unique()
    assert not bool(((actions[rows["masked"]] == 0) | (actions[rows["masked"]] == 2)).any())
    want = torch.log_softmax(yf, -1).gather(1, actions[:, None]).squeeze(1)
    assert torch.equal(torch.isnan(log_probs), torch.isnan(want))
    special = torch.cat([rows["inf"], rows["all_neg_inf"]])
    assert bool(torch.isnan(log_probs[special]).all())
    finite = torch.ones(M, dtype=torch.bool, device="cuda")
    finite[special] = False
    finite[rows["masked"]] = False
    _check_sample(y[finite], 31, 0, actions[finite], log_probs[finite], "finite rows", row_ids=finite.nonzero()[:, 0])
    masked = rows["masked"]
    ref = torch.log_softmax(yf[masked].double(), -1).gather(1, actions[masked][:, None]).squeeze(1)
    assert bool(((log_probs[masked].double() - ref).abs() <= 16 * 2.0 ** -22 * (1 + ref.abs())).all())
    assert bool(((log_probs[zero].double() + torch.log(torch.tensor(8.0, dtype=torch.float64))).abs() < 1e-6).all())
    b3 = torch.zeros(d_out, dtype=torch.bfloat16, device="cuda")
    b3[3] = b3[6] = float("nan")
    y = _logits(obs, w, (None, None, b3))
    actions, log_probs = _sample(obs, w, (None, None, b3), 31)
    assert bool(torch.isnan(y[:, [3, 6]]).all())
    assert bool((actions == 3).all()), actions.unique()
    want = torch.log_softmax(y.float(), -1).gather(1, actions[:, None]).squeeze(1)
    assert bool(torch.isnan(want).all()) and bool(torch.isnan(log_probs).all())


# ---- 6. guard bands --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form,M,chunk,d_out", [
    ("plain", 1000, SHIPPED_CHUNK, 7), ("plain", 1000, 256, 129), ("staged", 1408, 256, 18), ("pushed", 3 * 1408, 256, 7),
])
def test_writes_stay_inside_actions_and_log_probs(K, form, M, chunk, d_out):
    """actions (M·8 bytes), log_probs (M·4), scratch and stage between guard bands; a logits buffer passed to no one
    stays untouched; the results equal mlp_forward's bit for bit."""
    L, mlp = _L(), _mlp()
    d_in, d_hidden, seed = 256, 1024, 5
    w, b = _config(700, d_out)
    obs = _randn((M, d_in), 701)
    want_a, want_lp = _sample(obs, w, b, seed)
    K.set_tuning(8, chunk)
    try:
        actions, log_probs, logits = _Guarded(M * 8), _Guarded(M * 4), _Guarded(M * d_out * 2)
        buffers = {"actions": actions, "log_probs": log_probs}
        if form == "pushed":
            rig = _SamplePushRig(K, M, d_in, d_hidden, 512, "sm")
            for _ in range(3):
                rig.call(obs, w, b, d_out, seed, actions.ptr(), log_probs.ptr())
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
            L.call("ktb_mlp_bf16_policy_sample", 0, obs.data_ptr(), M, d_in, d_hidden, d_out, w[0].data_ptr(),
                   b[0].data_ptr(), w[1].data_ptr(), b[1].data_ptr(), w[2].data_ptr(), b[2].data_ptr(), seed, 0,
                   actions.ptr(), log_probs.ptr(), scratch.ptr(), stage, _stream())
        for name, buf in buffers.items():
            buf.check(f"{form} M={M} chunk={chunk} d_out={d_out}: {name}")
        assert bool((logits.view() == _Guarded.FILL).all()), "a logits buffer nobody was given changed"
        assert torch.equal(actions.view(torch.int64), want_a)
        assert torch.equal(log_probs.view(torch.float32), want_lp)
    finally:
        K.set_tuning(8, SHIPPED_CHUNK)


# ---- 7. status codes -------------------------------------------------------------------------------------------------
def _arg_case(name):
    L = _L()
    w1, w2, w3 = (torch.zeros(s, dtype=torch.bfloat16, device="cuda") for s in ((1024, 256), (1024, 1024), (512, 1024)))
    bias = torch.zeros(1024, dtype=torch.bfloat16, device="cuda")
    obs = torch.zeros(2048, 256, dtype=torch.bfloat16, device="cuda")
    act = torch.zeros(2048, dtype=torch.int64, device="cuda")
    lp = torch.zeros(2048, dtype=torch.float32, device="cuda")
    scratch = torch.zeros(1 << 24, dtype=torch.uint8, device="cuda")
    ctrl = torch.zeros(L.load().ktb_push_control_bytes(), dtype=torch.uint8, device="cuda")
    p = lambda t, off=0: t.data_ptr() + off   # noqa: E731

    def plain(d_out=18, actions=None, log_probs=None):
        return ("ktb_mlp_bf16_policy_sample", 0, p(obs), 256, 256, 1024, d_out, p(w1), p(bias), p(w2), p(bias), p(w3),
                p(bias), 1, 0, p(act) if actions is None else actions, p(lp) if log_probs is None else log_probs,
                p(scratch), 0, _stream())

    def pushed(d_out=18, actions=None, log_probs=None):
        return ("ktb_mlp_bf16_policy_sample_pushed", 0, p(scratch), 1 << 20, 256, 256, 1024, d_out, p(w1), p(bias),
                p(w2), p(bias), p(w3), p(bias), 1, 0, p(act) if actions is None else actions,
                p(lp) if log_probs is None else log_probs, p(scratch), p(ctrl), p(ctrl), 1, 256, 1, _stream())

    table = {
        "null_actions": (plain(actions=0), L.ERR_ARG),
        "null_log_probs": (plain(log_probs=0), L.ERR_ARG),
        "misaligned_actions": (plain(actions=p(act, 4)), L.ERR_ARG),
        "misaligned_log_probs": (plain(log_probs=p(lp, 2)), L.ERR_ARG),
        "d_out_257": (plain(d_out=257), L.ERR_UNSUPPORTED),
        "pushed_null_actions": (pushed(actions=0), L.ERR_ARG),
        "pushed_null_log_probs": (pushed(log_probs=0), L.ERR_ARG),
        "pushed_misaligned_log_probs": (pushed(log_probs=p(lp, 1)), L.ERR_ARG),
        "pushed_d_out_257": (pushed(d_out=257), L.ERR_UNSUPPORTED),
    }
    return table[name]


@pytest.mark.parametrize("name", [
    "null_actions", "null_log_probs", "misaligned_actions", "misaligned_log_probs", "d_out_257", "pushed_null_actions",
    "pushed_null_log_probs", "pushed_misaligned_log_probs", "pushed_d_out_257",
])
def test_bad_arguments_get_the_documented_status(K, name):
    L = _L()
    args, status = _arg_case(name)
    with pytest.raises(L.KtbError) as ei:
        L.call(*args)
    assert ei.value.status == status, (name, str(ei.value))
    torch.cuda.synchronize()    # nothing was launched; the device stays healthy


def test_python_checks_reach_mlp_forward(K):
    (w1, w2, w3), b = _config(800, 18)
    obs = _randn((256, 256), 801)
    for bad in (None, -1, 2**64, True, 1.0):
        with pytest.raises(ValueError):
            _mlp().mlp_forward(obs, w1, w2, w3, biases=b, output="sample", seed=bad)
    with pytest.raises(ValueError):
        _mlp().mlp_forward(obs, w1, w2, w3, biases=b, output="sample", seed=1, row_offset=-1)


# ---- 8. the public API ---------------------------------------------------------------------------------------------------
def _check_rank(got, want, y, seed, row0, what):
    """One rank's (actions, log_probs) under the bars, from the kernel's own logits y of the rank's rows; the oracle's
    body must agree wherever its fp32 restatement is clear (the two sides' logits may differ by bf16 roundings)."""
    a, lp = got
    assert isinstance(got, tuple) and len(got) == 2, what
    assert a.shape == want[0].shape and lp.shape == want[1].shape, what
    if a.shape[0] == 0:
        return
    _check_sample(y, seed, row0, a.cuda(), lp.cuda(), what)


@pytest.mark.parametrize("case", ["recorded", "ragged_1000_rows_3_ranks", "2_rows_3_ranks"])
def test_mapped_sample_through_public_api(K, golden, case):
    """@kt.mapped("mlp", bias=True, output="sample", seed="seed") on Compute(gpus=1) with three ranks on cuda:0,
    against the oracle's run of the body: each rank's draws satisfy the bars over its rows' global indices, and agree
    with the body's actions on at least 99 % of the rows."""
    import kubetorch_b200 as kt

    if case == "recorded":
        obs, d_out = golden["all_inputs"]["mlp_obs"], 64
    else:
        rows = 1000 if case.startswith("ragged") else 2
        obs, d_out = torch.randn(rows, 256, generator=torch.Generator().manual_seed(rows)).bfloat16(), 6
    p = _policy_weights(golden, d_out)
    n_ranks, seed = 3, 2**35 + 17
    want = ref_dispatch.spmd_call(policy_sample_cases.mlp_policy_sample, obs, *p, seed, num_proc=n_ranks,
                                  serialization="pickle")
    policy = mapped_copy(policy_sample_cases.mlp_policy_sample, "mlp", bias=True, output="sample", seed="seed")
    remote = kt.fn(policy, name=f"t-sample-{case}").to(
        kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute(
            "b200", workers=1, num_proc=n_ranks, devices=[0] * n_ranks))
    try:
        pc = [t.cuda() for t in p]
        got = remote(obs.cuda(), *pc, seed, serialization="pickle")
        torch.cuda.synchronize()
        assert len(got) == len(want) == n_ranks
        y = _mlp().mlp_forward(obs.cuda(), pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]))
        agree, total = 0, 0
        for r, (g, h) in enumerate(zip(got, want)):
            lo, hi = K.shard_bounds(obs.shape[0], n_ranks, r)
            _check_rank(g, h, y[lo:hi], seed, lo, (case, r))
            agree += int((g[0].cpu() == h[0]).sum())
            total += hi - lo
        assert agree >= 0.99 * total, (agree, total)
    finally:
        remote.teardown()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("transfer", ["pull", "push"])
def test_mapped_sample_on_two_gpus(K, golden, transfer):
    """Two ranks on two GPUs, staged pull and pushed form: the same bits as one plain call over all rows."""
    import kubetorch_b200 as kt

    obs = torch.randn(2 * 1408, 256, generator=torch.Generator().manual_seed(5)).bfloat16()
    p = _policy_weights(golden, 18)
    seed = 4242
    policy = mapped_copy(policy_sample_cases.mlp_policy_sample, "mlp", bias=True, output="sample", seed="seed")
    remote = kt.fn(policy, name=f"t-sample-2gpu-{transfer}").to(
        kt.Compute(gpus=2, allowed_serialization=["json", "pickle"]).distribute(
            "b200", workers=1, num_proc=2, devices=[0, 1], transfer=transfer))
    try:
        pc = [t.cuda(0) for t in p]
        got = remote(obs.cuda(0), *pc, seed, serialization="pickle")
        torch.cuda.synchronize(0)
        torch.cuda.synchronize(1)
        want_a, want_lp = _mlp().mlp_forward(obs.cuda(0), pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]),
                                             output="sample", seed=seed)
        assert torch.equal(torch.cat([g[0].cpu() for g in got]), want_a.cpu())
        assert torch.equal(torch.cat([g[1].cpu() for g in got]), want_lp.cpu())
    finally:
        remote.teardown()
