"""-m gpu: the sum reduction (`map_reduce_kernel` and the partials fold in csrc/ktb_reduce.cu, reached through
`ktb_map_reduce_sum` and `ktb_scatter_map_reduce`) against exact references.

Most inputs are drawn so that every mapped value y_i = op(x_i) is a multiple of 2^-k and every partial sum the
kernel can form stays below 2^(24-k) in fp32 and below 2^(53-k) in fp64. Then no order of fp32 and fp64 additions
can round, and the kernel must return float32(S) bit for bit, S = sum(y_i) in fp64 (exact too). Integer sums must
equal the int64 sum, which wraps modulo 2^64 like `torch.sum`. Sizes and start addresses are chosen from the
launch geometry (tests/reduce_geometry.py) so that every loop and branch of the kernel runs."""
import contextlib
import ctypes

import pytest
import torch

from conftest import resolve_args
from reduce_geometry import reduce_geometry

pytestmark = pytest.mark.gpu

from oracle import cases, ref_dispatch  # noqa: E402

T = 64 * 1024                      # bytes of one LOADS-8 tile, the default grid unit
U = 2.0 ** -24                     # unit roundoff of fp32
FLOATS = (torch.float32, torch.bfloat16, torch.float16)
ES = {torch.float32: 4, torch.bfloat16: 2, torch.float16: 2, torch.int32: 4, torch.int64: 8}
INT_VIEW = {4: torch.int32, 8: torch.int64}


@pytest.fixture(scope="module")
def K():
    assert torch.cuda.is_available()
    from kubetorch_b200.device import lib as L
    from kubetorch_b200.device import ops

    L.load()
    ops.ensure_init([0])
    return ops


@contextlib.contextmanager
def _tuning(K, loads=8, cap=4):
    """ktb_set_tuning key 13 (256-bit loads per thread and tile) and key 6 (grid cap in units of 1024 CTAs)."""
    K.set_tuning(13, loads)
    K.set_tuning(6, cap)
    try:
        yield
    finally:
        K.set_tuning(13, 8)
        K.set_tuning(6, 4)


TUNINGS = {"default": (8, 4), "loads4": (4, 4), "cap1024": (8, 1)}


# ---- exact inputs ---------------------------------------------------------------------------------------------
# dtype -> (largest |x|, [(op, alpha, beta, k)]): every mapped value is a multiple of 2^-k
EXACT = {
    torch.float32: (2**11, [("identity", 1, 0, 0), ("scale", 2, 0, 0), ("scale", -0.5, 0, 1), ("affine", 0.5, 0.25, 2),
                            ("affine", 3, -7, 0)]),
    torch.bfloat16: (127, [("identity", 1, 0, 0), ("scale", 2, 0, 0), ("affine", 0.5, 0.25, 2), ("affine", -1, 1, 0)]),
    torch.float16: (1023, [("identity", 1, 0, 0), ("scale", 2, 0, 0), ("affine", 0.5, 0.25, 2), ("affine", -1, 1, 0)]),
    torch.int32: (None, [("identity", 1, 0, 0), ("scale", 65537, 0, 0), ("affine", 3, -7, 0)]),
    torch.int64: (None, [("identity", 1, 0, 0), ("scale", -5, 0, 0), ("affine", -5, 11, 0)]),
}


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _exact_input(dtype, n, seed):
    """n values on cuda:0. Floats: integers 2 <= |x| <= bound with random signs, so no mapped value of EXACT is 0
    and a dropped or doubled element always moves the sum. Integers: the whole range of the dtype."""
    g = _gen(seed)
    if dtype == torch.int32:
        return torch.randint(-(2**31), 2**31, (n,), dtype=torch.int32, device="cuda", generator=g)
    if dtype == torch.int64:
        return torch.randint(-(2**31), 2**31, (2 * n,), dtype=torch.int32, device="cuda", generator=g).view(torch.int64)
    bound = EXACT[dtype][0]
    mag = torch.randint(2, bound + 1, (n,), dtype=torch.int32, device="cuda", generator=g)
    sign = torch.randint(0, 2, (n,), dtype=torch.int32, device="cuda", generator=g) * 2 - 1
    return (mag * sign).to(dtype)


def _op(x, op, a, b):
    """The op's own definition (oracle/cases.py), evaluated by torch in the tensor's dtype."""
    if op == "identity":
        return x
    if op == "scale":
        return x * a
    return x * a + b


def _exact_sum(y):
    """float32(sum) from an exact fp64 sum for floats; the int64 sum, modulo 2^64, for integers."""
    if y.dtype.is_floating_point:
        return y.double().sum().float()
    return y.to(torch.int64).sum()


def _assert_exact(y, k, geos):
    """The precondition of a bit-exact float sum: y·2^k is integral and the largest partial sum any thread (m values)
    or the whole input can form stays within 2^(24-k) in fp32 and 2^(53-k) in fp64."""
    if not y.dtype.is_floating_point or y.numel() == 0:
        return
    scaled = y.double() * 2.0**k
    assert bool((scaled == scaled.round()).all()), "inputs are not multiples of 2^-k"
    top = float(scaled.abs().max())
    for g in geos:
        assert g.m * top <= 2**24, g
    assert y.numel() * top <= 2**53


def _bits(t):
    t = t.reshape(-1)
    return t.view(INT_VIEW[t.element_size()])


class _Results:
    """Kernel outputs and references, compared bit for bit after one synchronise."""

    def __init__(self):
        self.rows = []

    def add(self, label, got, want):
        assert got.dtype == want.dtype, (label, got.dtype, want.dtype)
        self.rows.append((label, got.reshape(1), want.reshape(1)))

    def check(self):
        if not self.rows:
            return
        got = torch.cat([r[1] for r in self.rows])
        want = torch.cat([r[2] for r in self.rows])
        bad = (_bits(got) != _bits(want)).nonzero().flatten().tolist()
        msgs = [f"{self.rows[i][0]}: got {got[i].item()!r}, want {want[i].item()!r}" for i in bad[:12]]
        assert not bad, f"{len(bad)} of {len(self.rows)} sums differ:\n" + "\n".join(msgs)


def _geometry_sizes(es):
    """(label, n): n·es bytes at every branch of the launch geometry. With 64 KiB tiles these are 1, 2, 511, 512,
    513, 4095 and 4096 CTAs (odd and even partial counts, one and two fold load rounds), and finally more tiles
    than CTAs, followed by remainder packets and an element tail."""
    spec = [("0", 0), ("ES", es), ("32-ES", 32 - es), ("32", 32), ("32+ES", 32 + es), ("T-32", T - 32),
            ("T-ES", T - es), ("T", T), ("T+ES", T + es), ("T+32", T + 32), ("2T", 2 * T), ("511T+ES", 511 * T + es),
            ("512T", 512 * T), ("513T+32", 513 * T + 32), ("4095T", 4095 * T), ("4096T", 4096 * T),
            ("4097T+3x8KiB+7ES", 4097 * T + 3 * 32 * 256 + 7 * es)]
    return [(label, nbytes // es) for label, nbytes in spec]


MISALIGNED_SIZES = [("32+ES", 32), ("T+ES", T), ("2T", 2 * T), ("96T", 96 * T)]


def _sweep(K, res, x_full, dtype, op, a, b, k, loads, cap, sizes, offsets=(0,)):
    y_full = _op(x_full, op, a, b)
    es = ES[dtype]
    for label, n in sizes:
        for off in offsets:
            x, y = x_full[off:off + n], y_full[off:off + n]
            g = reduce_geometry(n, es, x.data_ptr(), loads, cap)
            if off:
                assert x.data_ptr() % 32 == off * es and g.n_vec == 0
            _assert_exact(y, k, [g])
            got = K.map_reduce_sum(x, op, a, b)
            res.add(f"{dtype} {op}({a},{b}) n={label} start+{off}", got, _exact_sum(y))


@pytest.mark.parametrize("tuning", list(TUNINGS))
@pytest.mark.parametrize("dtype", list(EXACT))
def test_exact_sums_over_the_launch_geometry(K, dtype, tuning):
    """Every op of EXACT, at every size of the geometry, and at starts 1 … 32/ES−1 elements past a 32-byte boundary
    (no packets: the whole input takes the element loop); under LOADS 8 and 4 and a grid cap of 4096 and 1024."""
    loads, cap = TUNINGS[tuning]
    es = ES[dtype]
    sizes = _geometry_sizes(es)
    x_full = _exact_input(dtype, sizes[-1][1] + 32 // es, seed=11 + es)
    assert x_full.data_ptr() % 32 == 0
    res = _Results()
    with _tuning(K, loads, cap):
        for op, a, b, k in EXACT[dtype][1]:
            _sweep(K, res, x_full, dtype, op, a, b, k, loads, cap, sizes)
            _sweep(K, res, x_full, dtype, op, a, b, k, loads, cap,
                   [(label, nbytes // es) for label, nbytes in MISALIGNED_SIZES], offsets=range(1, 32 // es))
        res.check()


@pytest.mark.parametrize("tuning", ["default", "loads4"])
def test_exact_in_fp64_but_not_in_fp32(K, tuning):
    """x = 2^12 + j, 1 <= j <= 7: each thread's fp32 partial (at most 137 values) stays exact, each CTA's partial
    (8192 or 16384 values) passes 2^24, and the total has more than 24 significant bits. Per-CTA partials and the
    fold in fp64 round the total once; demoting either to fp32 rounds it more than once.

    The same values with the sign flipped every 16384 elements: the CTA partials pass 2^24 with alternating signs
    and cancel, so the total is small and exact in fp32, and a CTA partial rounded to fp32 shows in the result."""
    loads, cap = TUNINGS[tuning]
    sizes = [(label, n) for label, n in _geometry_sizes(4) if n >= 511 * T // 4 or label in ("2T", "T+32")]
    n_max = sizes[-1][1]
    x_pos = (2**12 + torch.randint(1, 8, (n_max,), dtype=torch.int32, device="cuda", generator=_gen(5))).float()
    sign = 1 - 2 * ((torch.arange(n_max, device="cuda") // (T // 4)) % 2)
    x_alt = x_pos * sign
    res = _Results()
    with _tuning(K, loads, cap):
        for x_full in (x_pos, x_alt):
            _sweep(K, res, x_full, torch.float32, "identity", 1, 0, 0, loads, cap, sizes)
            _sweep(K, res, x_full, torch.float32, "affine", 3, -7, 0, loads, cap, sizes)
        res.check()
    # the premises: CTA partials past 2^24, a positive total past 2^24 · 64, an alternating total below 2^24
    s = x_pos[:4096 * T // 4].double()
    assert float(s[:T // 8].sum()) > 2**24 and float(s.sum()) > 2**30
    assert abs(float(x_alt[:4096 * T // 4].double().sum())) < 2**24


def _sizes_and_starts(es):
    """A few sizes of every path, each aligned and one element past a 32-byte boundary."""
    return [(label, nbytes // es) for label, nbytes in
            (("1", es), ("7", 7 * es), ("T+ES", T + es), ("2T+3x8KiB+7ES", 2 * T + 3 * 32 * 256 + 7 * es),
             ("513T+32", 513 * T + 32))]


@pytest.mark.parametrize("dtype,x0,op,a,b", [
    (torch.bfloat16, 3.0, "scale", 1.7, 0),        # bf16(3 * 1.7f) = 5.09375, not 5.1000004
    (torch.bfloat16, 3.0, "affine", 1.7, -0.3),    # and beta rounded to bf16 before the add, the sum rounded again
    (torch.float16, 3.0, "scale", 1.7, 0),
    (torch.float16, 3.0, "affine", 1.7, -0.3),
    (torch.float16, 60000.0, "scale", 2, 0),       # 120000 overflows fp16: every y is +inf, so is the sum
])
def test_each_element_is_rounded_to_the_tensor_dtype(K, dtype, x0, op, a, b):
    """A constant input at an alpha and beta the dtype cannot represent. The op's definition is torch on the CPU,
    like the reference's ranks; every y is the same dyadic y0, so the exact sum is n·y0. A kernel that skipped one
    rounding step would be off by n times a fixed amount."""
    y0 = _op(torch.full((1,), x0, dtype=dtype), op, a, b)
    unrounded = torch.tensor([x0], dtype=torch.float32) * a + b
    assert float(y0) != float(unrounded)
    es = ES[dtype]
    sizes = _sizes_and_starts(es)
    x_full = torch.full((sizes[-1][1] + 1,), x0, dtype=dtype, device="cuda")
    res = _Results()
    for label, n in sizes:
        for off in (0, 1):
            x = x_full[off:off + n]
            y = y0.cuda().expand(n)
            if torch.isfinite(y0).all():
                _assert_exact(y, 10, [reduce_geometry(n, es, x.data_ptr())])
            res.add(f"{dtype} {x0} {op}({a},{b}) n={label} start+{off}", K.map_reduce_sum(x, op, a, b), _exact_sum(y))
    res.check()


@pytest.mark.parametrize("dtype,scale", [(torch.float32, 2.0**-149), (torch.bfloat16, 2.0**-133)])
def test_subnormal_inputs_are_not_flushed(K, dtype, scale):
    """x = j·2^-149 (f32) or j·2^-133 (bf16), 1 <= |j| <= 7: the smallest subnormals of the dtype. Any flush to zero
    on the path, in the load, the op or an fp32 add, changes the sum."""
    es = ES[dtype]
    sizes = _sizes_and_starts(es)
    g = _gen(3)
    j = torch.randint(1, 8, (sizes[-1][1] + 1,), device="cuda", generator=g)
    j = j * (torch.randint(0, 2, j.shape, device="cuda", generator=g) * 2 - 1)
    x_full = (j.double() * scale).to(dtype)
    k = 149 if dtype == torch.float32 else 133
    res = _Results()
    for op, a in (("identity", 1), ("scale", 2)):
        y_full = _op(x_full, op, a, 0)
        assert bool((y_full != 0).all())
        for label, n in sizes:
            for off in (0, 1):
                x, y = x_full[off:off + n], y_full[off:off + n]
                _assert_exact(y, k, [reduce_geometry(n, es, x.data_ptr())])
                res.add(f"{dtype} subnormal {op} n={label} start+{off}", K.map_reduce_sum(x, op, a), _exact_sum(y))
    res.check()


# ---- random data under a bound derived from the kernel -----------------------------------------------------------
def _gamma(k):
    return k * U / (1 - k * U)


@pytest.mark.parametrize("tuning", ["default", "loads4"])
@pytest.mark.parametrize("dtype", FLOATS)
def test_random_sums_within_the_derived_bound(K, dtype, tuning):
    """|got − S| <= γ(m+3)·Σ|y_i| + 2^-24·|S|, S = Σ y_i and Σ|y_i| in fp64, y = the kernel's own map of x.

    Derivation. Each thread adds its values in fp32: 8 or 16 values of a packet in a chain, that partial into one of
    four accumulators once per tile round or remainder packet, tail elements one by one, then (acc0 + acc1) +
    (acc2 + acc3). A value that reaches the thread's result passes through at most m − 1 + 2 fp32 additions (m from
    the geometry: a chain of c values repeated r times takes c − 1 + r <= c·r additions). By the standard bound for
    a summation tree of depth d, the thread's fp32 result is within γ(m+1)·Σ|y_i| of its exact sum (Higham,
    Accuracy and Stability of Numerical Algorithms, §4.2). Everything after that (the block reduction, the per-CTA
    partials and the fold) is fp64: at most ~40 additions of relative error 2^-53, far below 2^-24·Σ|y_i|. So the
    fp64 total s is within E = γ(m+2)·Σ|y_i| of S, and the final rounding to fp32 adds at most 2^-24·|s| <=
    2^-24·(|S| + E); (1 + 2^-24)·γ(m+2) <= γ(m+3)."""
    loads, cap = TUNINGS[tuning]
    es = ES[dtype]
    sizes = [(label, n) for label, n in _geometry_sizes(es) if n] + [("96T", 96 * T // es)]
    g = _gen(17)
    x_full = torch.randn(max(n for _, n in sizes) + 1, device="cuda", generator=g)
    x_full = (x_full * 8).to(dtype) if dtype == torch.float16 else x_full.to(dtype)
    failures = []
    with _tuning(K, loads, cap):
        for op, a, b in (("identity", 1, 0), ("scale", 1.7, 0), ("affine", 1.7, -0.3)):
            y_full = K.map_tensor(x_full, op, a, b)
            for label, n in sizes:
                for off in ((0, 1) if label in ("T+ES", "96T") else (0,)):
                    x, y = x_full[off:off + n], y_full[off:off + n].double()
                    m = reduce_geometry(n, es, x.data_ptr(), loads, cap).m
                    got = float(K.map_reduce_sum(x, op, a, b))
                    s, s_abs = float(y.sum()), float(y.abs().sum())
                    bound = _gamma(m + 3) * s_abs + U * abs(s)
                    if not abs(got - s) <= bound:
                        failures.append(f"{dtype} {op} n={label} start+{off}: |{got} - {s}| > {bound} (m={m})")
    assert not failures, "\n".join(failures)


def _rand(dtype, n, seed=0):
    g = torch.Generator().manual_seed(seed)
    if dtype == torch.float32:
        return torch.randn(n, generator=g)
    if dtype == torch.bfloat16:
        return torch.randn(n, generator=g).bfloat16()
    if dtype == torch.float16:
        return (torch.randn(n, generator=g) * 8).half()
    if dtype == torch.int32:
        return torch.randint(-(2**31), 2**31 - 1, (n,), dtype=torch.int32, generator=g)
    return torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, generator=g)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16, torch.int32, torch.int64])
def test_reduce_sizes(K, dtype):
    """Regression bar on fixed seeded data: float sums within 8·eps·Σ|x| of the fp64 sum, integer sums exact."""
    for n in [0, 1, 33, 1000, 70_001, (1 << 21) + 5]:
        x = _rand(dtype, n, seed=n + 1)
        if dtype == torch.int64:
            x = x >> 24  # keep the true sum inside int64
        got = K.map_reduce_sum(x.cuda(), "identity").cpu()
        if dtype.is_floating_point:
            ref = float(x.double().sum())
            tol = 8 * torch.finfo(torch.float32).eps * float(x.double().abs().sum()) + 1e-30
            assert abs(float(got) - ref) <= tol, (dtype, n)
        else:
            assert int(got) == int(x.sum()), (dtype, n)
    # workspace is left clean: a second call gives the same answer
    x = _rand(torch.int32, 5000).cuda()
    assert int(K.map_reduce_sum(x, "affine", 3, 1)) == int(K.map_reduce_sum(x, "affine", 3, 1))


def test_golden_sums(K, golden):
    for name in ("sum_i64_130_x4", "sum_i32_515_x4", "sum_f32_1001_x4"):
        rec = golden["cases"][name]
        args = resolve_args(golden, rec["args"])
        x = args[0]
        a, b = (args[1], args[2]) if len(args) == 3 else (1, 0)
        op = "affine" if len(args) == 3 else "identity"
        total, partials = K.scatter_map_reduce(x.cuda(), op, a, b, devices=[0] * 4)
        if x.dtype.is_floating_point:
            # fp32 sums: order differs from torch's pairwise sum; tolerance = 8 ulp of sum(|x|)
            tol = 8 * torch.finfo(torch.float32).eps * float(x.abs().sum())
            for g, w in zip(partials.tolist(), rec["result"]):
                assert abs(g - w) <= tol, name
        else:
            assert partials.tolist() == rec["result"], name
            assert int(total.item()) == sum(rec["result"])


# ---- special values, determinism, workspaces ---------------------------------------------------------------------
@pytest.mark.parametrize("dtype", FLOATS)
def test_special_values(K, dtype):
    """+inf gives +inf, NaN gives NaN, +inf and −inf give NaN, planted inside a tile, in the remainder packets, in
    the element tail, and in an input that starts one element past a 32-byte boundary."""
    es = ES[dtype]
    n = (2 * T + 3 * 32 * 256 + 7 * es) // es
    g = reduce_geometry(n, es)
    assert (g.n_tiles, g.rem, g.tail) == (2, 3 * 256, 7)
    where = {"tile": (100, 101), "remainder": ((2 * T + 32 * 300) // es, (2 * T + 32 * 700) // es + 3),
             "tail": (n - 3, n - 1), "misaligned": (5000, n - 2)}
    base = _exact_input(dtype, n + 1, seed=23)
    inf, nan = float("inf"), float("nan")

    def kind(t):  # 0 finite, ±1 ±inf, 2 NaN (NaN payloads are not compared)
        return torch.where(torch.isnan(t), 2.0, torch.where(torch.isinf(t), t.sign(), 0.0))

    res = _Results()
    for region, (i, j) in where.items():
        for planted, want in (((inf,), inf), ((-inf,), -inf), ((nan,), nan), ((inf, -inf), nan)):
            xb = base.clone()
            for pos, v in zip((i, j), planted):
                xb[pos + (region == "misaligned")] = v
            x = xb[1:n + 1] if region == "misaligned" else xb[:n]
            for op, a in (("identity", 1), ("scale", 2)):
                got = K.map_reduce_sum(x, op, a)
                res.add(f"{dtype} {planted} in {region} {op}", kind(got), kind(torch.tensor([want], device="cuda")))
    res.check()


def test_deterministic_across_calls_streams_and_forms(K):
    """The fold runs in a fixed order: repeated calls, a call with another stream current (its own workspace) and a
    one-rank scatter_map_reduce give identical bits on the same 64 MiB of random data."""
    x = torch.randn(16 << 20, device="cuda", generator=_gen(29))
    runs = [K.map_reduce_sum(x, "affine", 1.7, -0.3) for _ in range(3)]
    s2 = torch.cuda.Stream()
    s2.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s2):
        other = K.map_reduce_sum(x, "affine", 1.7, -0.3)
    torch.cuda.current_stream().wait_stream(s2)
    total, partials = K.scatter_map_reduce(x, "affine", 1.7, -0.3, devices=[0])
    got = torch.cat(runs + [other, total, partials])
    assert bool(torch.isfinite(got).all())
    assert bool((_bits(got) == _bits(got[:1])).all()), got.tolist()


def test_workspace_is_reset_between_launches(K):
    """About 40 reductions of different sizes, from n = 0 to more than 4096 tiles, back to back on one stream into
    slots of one output tensor. Each launch relies on the last CTA of the previous one to have reset the ticket
    counter; every slot must be exact."""
    n_max = (4097 * T + 3 * 32 * 256 + 7 * 4) // 4
    x = _exact_input(torch.float32, n_max, seed=31)
    sizes = [0, 1, 7, 8, 9, 2047, 16384, 16385, 3 * 16384 + 5, 0, 511 * 16384 + 1, 1, 2 * 16384, n_max, 4096 * 16384,
             255, 256, 257, 513 * 16384 + 8, 5, 0, 4095 * 16384, 12345, 100_000, n_max - 1, 3, 16383, 1 << 20, 33,
             (1 << 22) + 1, 999, 2, 4097 * 16384, 77, 40_000, 1000, 0, 64, n_max, 6]
    out = torch.full((len(sizes),), float("nan"), device="cuda")
    for i, n in enumerate(sizes):
        K.map_reduce_sum(x[:n], "affine", 3, -7, out=out[i:i + 1])
    torch.cuda.synchronize()
    y = _op(x, "affine", 3, -7)
    res = _Results()
    for i, n in enumerate(sizes):
        _assert_exact(y[:n], 0, [reduce_geometry(n, 4)])
        res.add(f"slot {i} n={n}", out[i], _exact_sum(y[:n]))
    res.check()


def test_stream_argument_selects_that_streams_workspace(K):
    """map_reduce_sum(x, stream=s) launches on s and must use s's workspace, not the current stream's: the workspace
    holds the ticket counter and the per-CTA partials, and two streams sharing one would mix their partials."""
    cur = torch.cuda.current_stream()
    s = torch.cuda.Stream()
    a = torch.full((1000,), 7.0, device="cuda")
    b = torch.full((1000,), 5.0, device="cuda")
    K.map_reduce_sum(a, "identity")                      # one CTA: partials[0] of the current workspace = 7000
    torch.cuda.synchronize()
    ws_cur = K._workspace(0).clone()
    got = K.map_reduce_sum(b, "identity", stream=s)      # one CTA on s: partials[0] = 5000
    torch.cuda.synchronize()
    assert float(got) == 5000.0
    ws_s = K._workspace(0, s.cuda_stream)
    assert ws_s.data_ptr() != K._workspace(0).data_ptr()
    assert torch.equal(K._workspace(0), ws_cur)          # the current stream's workspace was not touched
    assert float(ws_cur[64:72].view(torch.float64)) == 7000.0
    assert float(ws_s[64:72].view(torch.float64)) == 5000.0
    assert cur == torch.cuda.current_stream()


def test_reductions_on_two_streams_at_once(K):
    """Large exact reductions alternating between the current stream and stream=s with no synchronisation between
    them, so they overlap on the GPU; every result must be exact. Run once: a shared workspace shows as wrong sums
    (the kernel never waits on the counter, so it cannot hang)."""
    n = 8192 * 2048 + 3                                  # 64 MiB of f32: 1025 CTAs, a fold with an odd count
    xs = [_exact_input(torch.float32, n, seed=40 + i) for i in range(2)]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    out = torch.full((16,), float("nan"), device="cuda")
    for i in range(16):
        K.map_reduce_sum(xs[i % 2], "scale", 2, out=out[i:i + 1], stream=s if i % 2 else None)
    torch.cuda.synchronize()
    res = _Results()
    for i in range(16):
        y = _op(xs[i % 2], "scale", 2, 0)
        _assert_exact(y, 0, [reduce_geometry(n, 4)])
        res.add(f"call {i} on {'s' if i % 2 else 'current'}", out[i], _exact_sum(y))
    res.check()


# ---- the scatter form and the C-ABI ------------------------------------------------------------------------------
@pytest.mark.parametrize("ranks", [1, 3, 4, 16])
@pytest.mark.parametrize("dtype", list(EXACT))
def test_scatter_map_reduce_shards(K, dtype, ranks):
    """ops.scatter_map_reduce with every rank time-sliced on cuda:0: row shards of x.chunk(ranks), ragged, starting
    at any element (so misaligned), and empty past the data. partials[r] is the exact sum of shard r; total is
    float32(Σ float64(partials)) for floats and the int64 sum for integers, which also match the oracle."""
    es = ES[dtype]
    op, a, b, k = EXACT[dtype][1][-1]
    res = _Results()
    checked = 0
    for cols in (1, 5, 37):
        for rows in (ranks - 1, 3 * ranks + 2, 4099):
            x = _exact_input(dtype, rows * cols, seed=rows * 100 + cols).reshape(rows, cols)
            total, partials = K.scatter_map_reduce(x, op, a, b, devices=[0] * ranks)
            y = _op(x, op, a, b)
            chunks = y.chunk(ranks) if rows else ()
            for r in range(ranks):
                yr = chunks[r].reshape(-1) if r < len(chunks) else y.reshape(-1)[:0]
                start = x.data_ptr() + K.shard_bounds(rows, ranks, r)[0] * cols * es
                _assert_exact(yr, k, [reduce_geometry(yr.numel(), es, start)])
                res.add(f"{dtype} {rows}x{cols} rank {r}/{ranks}", partials[r], _exact_sum(yr))
            want_total = partials.double().sum().float() if dtype.is_floating_point else partials.sum()
            res.add(f"{dtype} {rows}x{cols} total/{ranks}", total, want_total)
            if not dtype.is_floating_point and rows * cols < 20_000:
                oracle = ref_dispatch.spmd_call(cases.shard_sum, x.cpu(), a, b, num_proc=ranks)
                assert partials.tolist() == oracle, (dtype, rows, cols, ranks)
                checked += 1
    res.check()
    assert checked or dtype.is_floating_point


def test_status_codes(K):
    from kubetorch_b200.device import lib as L

    x = torch.zeros(64, device="cuda")
    out = torch.zeros(1, dtype=torch.int64, device="cuda")
    ws = K._workspace(0)
    st = torch.cuda.current_stream().cuda_stream

    def status(name, *args):
        with pytest.raises(L.KtbError) as ei:
            L.call(name, *args)
        return ei.value.status

    red = lambda op, dt, src, n, o, w: status("ktb_map_reduce_sum", 0, op, dt, src, n, 1.0, 0.0, o, w, st)  # noqa: E731
    assert red(L.OP_IDENTITY, L.U8, x.data_ptr(), 64, out.data_ptr(), ws.data_ptr()) == L.ERR_ARG
    assert red(7, L.F32, x.data_ptr(), 64, out.data_ptr(), ws.data_ptr()) == L.ERR_ARG
    assert red(L.OP_IDENTITY, L.F32, x.data_ptr(), 64, None, ws.data_ptr()) == L.ERR_ARG
    assert red(L.OP_IDENTITY, L.F32, x.data_ptr(), 64, out.data_ptr(), None) == L.ERR_ARG
    assert red(L.OP_IDENTITY, L.F32, None, 64, out.data_ptr(), ws.data_ptr()) == L.ERR_ARG
    assert red(L.OP_IDENTITY, L.F32, x.data_ptr() + 2, 60, out.data_ptr(), ws.data_ptr()) == L.ERR_ARG
    assert status("ktb_map_reduce_sum", 9, L.OP_IDENTITY, L.F32, x.data_ptr(), 64, 1.0, 0.0, out.data_ptr(),
                  ws.data_ptr(), st) == L.ERR_STATE
    # n = 0 with a null src is a valid empty sum: 0 lands in a garbage-filled out
    for dt, o in ((L.F32, torch.full((1,), float("nan"), device="cuda")),
                  (L.I64, torch.full((1,), -0x5A5A5A5A5A5A5A5B, dtype=torch.int64, device="cuda"))):
        L.call("ktb_map_reduce_sum", 0, L.OP_AFFINE, dt, None, 0, 3.0, 1.0, o.data_ptr(), ws.data_ptr(), st)
        torch.cuda.synchronize()
        assert o.item() == 0 and not bool(o.isnan().any()), dt

    assert status("ktb_reduce_partials", 0, L.F32, x.data_ptr(), 0, out.data_ptr(), st) == L.ERR_ARG
    assert status("ktb_reduce_partials", 0, L.U8, x.data_ptr(), 4, out.data_ptr(), st) == L.ERR_ARG

    devs = L.arr(ctypes.c_int, [0] * 17)
    wss = L.arr(ctypes.c_void_p, [ws.data_ptr()] * 17)
    wss_null = L.arr(ctypes.c_void_p, [None, ws.data_ptr()])
    sts = L.arr(L.c_uintptr, [st] * 17)
    parts = torch.zeros(17, dtype=torch.int64, device="cuda")

    def smr(dt, n, granule, n_ranks, root, workspaces=wss):
        return status("ktb_scatter_map_reduce", L.OP_IDENTITY, dt, x.data_ptr(), n, granule, 1.0, 0.0, n_ranks, devs,
                      root, parts.data_ptr(), out.data_ptr(), workspaces, sts)

    assert smr(L.U8, 64, 1, 2, 0) == L.ERR_ARG
    assert smr(L.F32, 64, 0, 2, 0) == L.ERR_ARG
    assert smr(L.F32, 64, 5, 2, 0) == L.ERR_ARG
    assert smr(L.F32, 64, 1, 2, 0, wss_null) == L.ERR_ARG
    assert smr(L.F32, 64, 1, 0, 0) == L.ERR_ARG
    assert smr(L.F32, 64, 1, 17, 0) == L.ERR_ARG
    assert smr(L.F32, 64, 1, 2, 2) == L.ERR_ARG
    assert smr(L.F32, 64, 1, 2, -1) == L.ERR_ARG
    torch.cuda.synchronize()
