"""-m gpu: every element-wise path against the exact reference of tests/elementwise_ref.py, at every 16-bit input, the
f32 / integer edge values, every row of the scalar tables, independent src/dst alignments, tile and stage edges, and
with every destination between guard bands that must come back untouched.

The rule (DESIGN.md §1): a scale/affine result of f32/bf16/f16 equals the reference bit for bit wherever the reference
is not NaN and is NaN exactly where it is NaN; identity and every u8 / integer result are byte-exact.  All paths share
apply_words / apply_elem, so every path also gives the same bytes as ktb_map's VEC path, NaN payloads included.

Which case reaches which branch:
  * map_tma_kernel's ring wrap: test_map_tma_ring_wraps — 48 MiB + 3 bf16 elements, 1536 stages of 32 KiB over a grid
    of sm_count (132) CTAs, so every CTA loops at least 11 tiles (> STAGES = 4; the mbarrier parity flips twice).
  * seg_map_kernel's 256-bit / 128-bit / element branches: test_map_batch_exact, segments whose src/dst offsets are
    (32, 32) / (16, 32), (32, 16), (16, 16) / any pair with an element-aligned side.
  * push_consume_kernel's 256-bit / element branches: test_push_session_exact, the `aligned` shape (shards start at
    multiples of 8192 elements) / the `rows` shape (7-element rows: every rank's shard starts misaligned).
  * ktb_map's fallbacks TMA -> VEC -> SCALAR: test_map_offsets, src and dst offsets 0..32 bytes chosen independently.
"""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

import elementwise_ref as R
from mlp_rig import Guarded

pytestmark = pytest.mark.gpu

import kubetorch_b200 as kt  # noqa: E402
from kubetorch_b200.device import lib as L  # noqa: E402
from oracle import cases, ref_dispatch  # noqa: E402

VEC, TMA, SCALAR, AUTO = L.VARIANT_VEC, L.VARIANT_TMA, L.VARIANT_SCALAR, L.VARIANT_AUTO
VEC_TILE = 16384         # map_vec_kernel: 256 threads x 4 x 16 bytes per CTA iteration
TMA_STAGE = 32768        # map_tma_kernel: bytes per ring stage
SEG_TILE = 32768         # seg_map_kernel: bytes per CTA work item
CASES = [(dt, op) for dt in R.DTYPES for op in R.ops_of(dt)]
CASE_IDS = [f"{str(d)[6:]}-{o}" for d, o in CASES]
# one scalar row per dtype whose results include NaN, infinities, rounding ties and wrap-around
ROW = {torch.uint8: (1, 0), torch.float32: (1.7, -0.3), torch.bfloat16: (1.7, -0.3), torch.float16: (1.7, 65520.0),
       torch.int32: (2 ** 53 + 1, -2 ** 31), torch.int64: (2 ** 31 - 1, -2 ** 53)}
SECOND_ROW = {torch.uint8: (1, 0), torch.float32: (3e38, 1e-8), torch.bfloat16: (0.1, 1 + 2 ** -8),
              torch.float16: (-1.0, 0.25), torch.int32: (-2 ** 63, 2 ** 32 + 3), torch.int64: (-2 ** 63, 65537)}


@pytest.fixture(scope="module")
def K():
    assert torch.cuda.is_available()
    from kubetorch_b200.device import ops

    L.load()
    ops.ensure_init([0])
    return ops


def _sm_count():
    return L.load().ktb_sm_count(0)


def patterns(dtype, n, phase=0):
    """n elements of the dtype's generator, tiled (every 16-bit pattern appears once per 65 536 elements)."""
    base = R.inputs(dtype)
    return np.resize(np.roll(base, -phase), n)


def to_dev(u):
    """numpy bit patterns -> a CUDA uint8 tensor of their bytes."""
    return torch.from_numpy(np.ascontiguousarray(u).view(np.uint8)).cuda()


def got_bits(t, dtype):
    return R.bits_of(t.reshape(-1).view(torch.uint8)).view(R.UINT[dtype])


def expect(dtype, op, got, x, a, b, what, same_as=None):
    """got (bit patterns) against the reference of x under the rule; and byte-equal to `same_as` when given."""
    want = R.reference(dtype, op, x, a, b)
    bad = R.mismatches(dtype, op, got, want)
    assert bad.size == 0, f"{what}: {bad.size} of {len(want)} wrong; (i, x, got, want): " \
                          f"{R.describe(dtype, x, got, want, bad)}"
    if same_as is not None:
        diff = np.nonzero(np.asarray(got) != np.asarray(same_as))[0]
        assert diff.size == 0, f"{what}: {diff.size} bytes differ from the VEC path, first at {diff[:4].tolist()}"


def exact_scalars(dtype, a, b):
    """Whether the entries take (a, b) for `dtype` (an int64 scalar a double does not hold is refused)."""
    return dtype != torch.int64 or (R.int64_exact(a) and R.int64_exact(b))


def run_map(K, dtype, op, x, a, b, variant, src_off=0, dst_off=0, inplace=False, what=""):
    """ktb_map of the bit patterns x from a buffer src_off bytes past a 256-byte boundary into a guarded destination
    dst_off bytes past one (in place: the guarded buffer is both); returns the result's bit patterns."""
    es, n = R.ES[dtype], len(x)
    nbytes = n * es
    g = Guarded(nbytes, dst_off)
    if inplace:
        g.view().copy_(to_dev(x))
        src = g.ptr()
    else:
        raw = torch.empty(nbytes + 256, dtype=torch.uint8, device="cuda")
        raw[src_off:src_off + nbytes].copy_(to_dev(x))
        src = raw.data_ptr() + src_off
    A, B = K.scalar_args(dtype, a, b)
    L.call("ktb_map", 0, K.OPS[op], K.dtype_code(dtype), src, g.ptr(), n, A, B, variant, K.current_stream_handle(0))
    g.check(what)
    return got_bits(g.view(), dtype)


# ---- ktb_map ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,op", CASES, ids=CASE_IDS)
def test_map_scalar_table(K, dtype, op):
    """Every row of the scalar table on every generator value (each 16-bit pattern twice plus a 5-element tail), through
    VEC, TMA and SCALAR; an int64 row a double cannot carry raises TypeError before any launch."""
    x = patterns(dtype, 2 * len(R.inputs(dtype)) + 5)
    for a, b in R.scalar_rows(dtype, op):
        what = f"{dtype} {op} a={a!r} b={b!r}"
        if not exact_scalars(dtype, a, b):
            try:
                y = K.map_tensor(R.to_torch(x, dtype).cuda(), op, a, b)
            except TypeError as e:
                assert "exactly representable" in str(e), e
                continue
            got, want = R.bits_of(y), R.reference(dtype, op, x, a, b)
            bad = R.mismatches(dtype, op, got, want)
            pytest.fail(f"{what}: no TypeError, and {bad.size} of {len(x)} results differ from the exact ones; "
                        f"(i, x, got, want): {R.describe(dtype, x, got, want, bad)}")
        vec = run_map(K, dtype, op, x, a, b, VEC, what=what)
        expect(dtype, op, vec, x, a, b, what + " VEC")
        for variant in (TMA, SCALAR):
            got = run_map(K, dtype, op, x, a, b, variant, what=what)
            expect(dtype, op, got, x, a, b, f"{what} variant {variant}", same_as=vec)


OFFSET_CASES = [(dt, "identity" if dt == torch.uint8 else "affine") for dt in R.DTYPES]


@pytest.mark.parametrize("variant", [VEC, TMA, SCALAR])
@pytest.mark.parametrize("dtype,op", OFFSET_CASES, ids=[f"{str(d)[6:]}-{o}" for d, o in OFFSET_CASES])
def test_map_offsets(K, dtype, op, variant):
    """src and dst at every element offset 0..32 bytes, independently, and in place: misaligned pointers fall back
    TMA -> VEC -> SCALAR and must give the same bytes.  2 x 16 KiB + 16 B - es: two VEC tiles, one 16-byte vector and
    all but one element of the next."""
    es = R.ES[dtype]
    n = (2 * VEC_TILE + 16 - es) // es
    a, b = ROW[dtype]
    x = patterns(dtype, n, phase=1234)
    vec = run_map(K, dtype, op, x, a, b, VEC, what="aligned VEC")
    for so in range(0, 33, es):
        for do in range(0, 33, es):
            got = run_map(K, dtype, op, x, a, b, variant, so, do, what=f"src+{so} dst+{do}")
            expect(dtype, op, got, x, a, b, f"{dtype} variant {variant} src+{so} dst+{do}", same_as=vec)
        got = run_map(K, dtype, op, x, a, b, variant, so, so, inplace=True, what=f"in place +{so}")
        expect(dtype, op, got, x, a, b, f"{dtype} variant {variant} in place +{so}", same_as=vec)


def _edge_sizes(es, sm):
    vec = [VEC_TILE // es + d for d in (-1, 0, 1)] + [(k * VEC_TILE + 16 - es) // es for k in (1, 3)]
    tma = [TMA_STAGE // es + d for d in (-1, 0, 1)] + [(TMA_STAGE + t) // es for t in range(es, 16, es)]
    return [1, 2, 3] + vec + tma + [sm * 8 * 256 * 2 + 3]     # the last: SCALAR's grid-stride loop iterates


@pytest.mark.parametrize("dtype,op", CASES, ids=CASE_IDS)
def test_map_edge_sizes(K, dtype, op):
    """Sizes at the VEC tile edges, the TMA stage edges with every 16-byte tail (1..15 bytes), and past SCALAR's grid
    (sm_count x 8 CTAs x 256 threads elements), through every variant, under two scalar rows."""
    for n in _edge_sizes(R.ES[dtype], _sm_count()):
        x = patterns(dtype, n, phase=n)
        for a, b in {ROW[dtype], SECOND_ROW[dtype]}:
            what = f"{dtype} {op} n={n} a={a!r} b={b!r}"
            vec = run_map(K, dtype, op, x, a, b, VEC, what=what)
            expect(dtype, op, vec, x, a, b, what + " VEC")
            for variant in (TMA, SCALAR, AUTO):
                expect(dtype, op, run_map(K, dtype, op, x, a, b, variant, what=what), x, a, b,
                       f"{what} variant {variant}", same_as=vec)


def test_map_tma_ring_wraps(K):
    """48 MiB + 3 bf16 elements (every pattern 384 times, then 3): 1536 full stages over sm_count CTAs, so every CTA
    re-arms each of its 4 stages at least twice (bulk_wait_read, a new load into a used stage, parity flips); CTA 0
    maps the 6-byte tail."""
    dtype, op, (a, b) = torch.bfloat16, "affine", ROW[torch.bfloat16]
    n = (48 << 20) // 2 + 3
    sm = _sm_count()
    tiles = (n * 2 & ~15) // TMA_STAGE
    assert tiles // sm >= 2 * 4, (tiles, sm)
    base = R.all_16bit()
    want = R.reference(dtype, op, base, a, b)
    reps = n // len(base)
    src = to_dev(np.resize(base, n))
    outs = {}
    for variant in (TMA, VEC):
        g = Guarded(n * 2)
        A, B = K.scalar_args(dtype, a, b)
        L.call("ktb_map", 0, K.OPS[op], K.dtype_code(dtype), src.data_ptr(), g.ptr(), n, A, B, variant,
               K.current_stream_handle(0))
        g.check(f"variant {variant}")
        outs[variant] = g
    got = outs[TMA].view(torch.int16)
    w = torch.from_numpy(want.view(np.int16)).cuda()
    body = got[:reps * len(base)].view(reps, len(base))

    def nan(t):
        return (t.int() & 0x7FFF) > 0x7F80

    nb, nw = nan(body), nan(w)
    bad = (nb != nw) | (~nw & (body != w))
    del nb
    assert not bool(bad.any()), f"{int(bad.sum())} wrong elements, first at {bad.nonzero()[:4].tolist()}"
    expect(dtype, op, got_bits(got[reps * len(base):], dtype), base[:3], a, b, "tail")
    assert torch.equal(outs[TMA].view(), outs[VEC].view()), "TMA and VEC differ"


# ---- ktb_map_batch ----------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def seg_large(value):
    from kubetorch_b200.device import ops

    try:
        ops.set_tuning(12, value)
        yield
    finally:
        ops.set_tuning(12, 1)


def _segment_plan(dtype, count):
    """(length, src_align, dst_align) per segment: alignment classes 32 / 16 / element cycle independently for src and
    dst; the first segments are 1 element, one tile - es, one tile, one tile + es and 3 tiles + a tail, the rest short."""
    es = R.ES[dtype]
    t = SEG_TILE // es
    big = [1, t - 1, t, t + 1, 3 * t + 7]
    classes = (32, 16, es)
    plan = []
    for i in range(count):
        n = big[i % len(big)] if i < 3 * len(big) else 1 + (i * 37) % 300
        plan.append((n, classes[i % 3], classes[(i // 3) % 3]))
    return plan


def _place(sizes_aligns, es):
    """Byte offsets in one arena: each segment `align` bytes past a 256-byte boundary (32 -> 0), 64+ bytes apart."""
    offs, cur = [], 0
    for n, align in sizes_aligns:
        o = (cur + 255) // 256 * 256 + (0 if align == 32 else align)
        offs.append(o)
        cur = o + n * es + 64
    return offs, cur


@pytest.mark.parametrize("large", [1, 0])
@pytest.mark.parametrize("count", [96, 97, 1025])
@pytest.mark.parametrize("dtype,op", CASES, ids=CASE_IDS)
def test_map_batch_exact(K, dtype, op, count, large):
    es = R.ES[dtype]
    a, b = ROW[dtype]
    plan = _segment_plan(dtype, count)
    x = patterns(dtype, sum(n for n, _, _ in plan), phase=count)
    bounds = np.cumsum([0] + [n for n, _, _ in plan])
    src_offs, src_len = _place([(n, s) for n, s, _ in plan], es)
    dst_offs, dst_len = _place([(n, d) for n, _, d in plan], es)
    src = torch.zeros(src_len, dtype=torch.uint8)
    xb = np.ascontiguousarray(x).view(np.uint8)
    for i, (n, _, _) in enumerate(plan):
        src[src_offs[i]:src_offs[i] + n * es] = torch.from_numpy(xb[bounds[i] * es:bounds[i + 1] * es])
    src = src.cuda()
    dst = Guarded(dst_len)
    A, B = K.scalar_args(dtype, a, b)
    with seg_large(large):
        L.call("ktb_map_batch", 0, K.OPS[op], K.dtype_code(dtype),
               L.arr(ctypes.c_void_p, [src.data_ptr() + o for o in src_offs]),
               L.arr(ctypes.c_void_p, [dst.ptr() + o for o in dst_offs]),
               L.arr(ctypes.c_size_t, [n for n, _, _ in plan]), count, A, B, K.current_stream_handle(0))
        dst.check(f"{count} segments")
    out = R.bits_of(dst.view())
    want = R.reference(dtype, op, x, a, b)
    untouched = np.ones(dst_len, dtype=bool)
    for i, (n, sa, da) in enumerate(plan):
        o = dst_offs[i]
        got = out[o:o + n * es].view(R.UINT[dtype])
        bad = R.mismatches(dtype, op, got, want[bounds[i]:bounds[i + 1]])
        assert bad.size == 0, f"segment {i} ({n} elements, src align {sa}, dst align {da}): {bad.size} wrong, " \
                              f"first at {bad[:4].tolist()}"
        untouched[o:o + n * es] = False
    gaps = np.nonzero(untouched & (out != Guarded.FILL))[0]
    assert gaps.size == 0, f"{gaps.size} bytes written between segments, first at arena offset {gaps[:4].tolist()}"
    # the batch gives the bytes ktb_map gives
    vec = run_map(K, dtype, op, x, a, b, VEC)
    got_all = np.concatenate([out[o:o + n * es] for o, (n, _, _) in zip(dst_offs, plan)]).view(R.UINT[dtype])
    assert np.array_equal(got_all, vec)


# ---- scatter_map_gather -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_ranks", [2, 3, 8])
@pytest.mark.parametrize("dtype,op", CASES, ids=CASE_IDS)
def test_scatter_map_gather_exact(K, dtype, op, n_ranks):
    """Every rank time-sliced on cuda:0; 2-D inputs with odd row lengths (the ranks' shard pointers are misaligned) and
    fewer rows than ranks."""
    es = R.ES[dtype]
    for shape in ((37, 1001), (n_ranks - 1, 999), (1, 13)):
        n = shape[0] * shape[1]
        x = patterns(dtype, n, phase=n)
        xt = R.to_torch(x, dtype).cuda().reshape(shape)
        for a, b in {ROW[dtype], SECOND_ROW[dtype]}:
            g = Guarded(n * es)
            out = g.view(dtype).reshape(shape)
            K.scatter_map_gather(xt, op, a, b, devices=[0] * n_ranks, out_root=out)
            g.check(f"{shape} over {n_ranks} ranks")
            vec = run_map(K, dtype, op, x, a, b, VEC)
            expect(dtype, op, got_bits(out, dtype), x, a, b, f"{dtype} {op} {shape} x{n_ranks}", same_as=vec)


# ---- PushSession ------------------------------------------------------------------------------------------------------
PUSH_SHAPES = {"aligned": (3 * 8192 - 2,), "rows": (20001, 7)}


@pytest.mark.parametrize("shape", list(PUSH_SHAPES))
@pytest.mark.parametrize("n_chunks", [1, 3, 32])
@pytest.mark.parametrize("dtype,op", CASES, ids=CASE_IDS)
def test_push_session_exact(K, dtype, op, n_chunks, shape):
    """Three ranks time-sliced on cuda:0, three consecutive calls (both staging halves, one reused) under different
    scalar rows, then the sticky status must be clean.  `aligned`: ragged 1-D shards that start at multiples of 8192
    elements (32-byte aligned: the 256-bit branch); `rows`: 7-element rows, so every rank's shard starts misaligned
    (the element branch)."""
    es = R.ES[dtype]
    shp = PUSH_SHAPES[shape]
    n = int(np.prod(shp))
    x = patterns(dtype, n, phase=n_chunks)
    xt = R.to_torch(x, dtype).cuda().reshape(shp)
    gran = K.row_elems(xt)
    sess = K.PushSession([0, 0, 0], K.shard_bounds(shp[0], 3, 0)[1] * gran * es, n_chunks=n_chunks)
    rows = [ROW[dtype], SECOND_ROW[dtype], ROW[dtype]]
    for it, (a, b) in enumerate(rows):
        g = Guarded(n * es)
        out = g.view(dtype).reshape(shp)
        sess.call(xt, out, op, a, b)
        g.check(f"call {it}")
        expect(dtype, op, got_bits(out, dtype), x, a, b, f"{dtype} {op} {shape} chunks={n_chunks} call {it}",
               same_as=run_map(K, dtype, op, x, a, b, VEC))
    sess.check()


# ---- host-resident pipelines ------------------------------------------------------------------------------------------
class HostGuarded:
    """A pinned host buffer `offset` bytes into a larger pinned allocation whose bands hold a byte pattern."""

    def __init__(self, nbytes, offset):
        self.nbytes, self.start = nbytes, 4096 + offset
        self.raw = torch.full((self.start + nbytes + 4096,), Guarded.FILL, dtype=torch.uint8).pin_memory()

    def view(self, dtype):
        return self.raw[self.start:self.start + self.nbytes].view(dtype)

    def check(self, what):
        bands = torch.cat([self.raw[:self.start], self.raw[self.start + self.nbytes:]])
        assert bool((bands == Guarded.FILL).all()), f"{what}: a band around the host buffer changed"


@pytest.mark.parametrize("dtype,op", CASES, ids=CASE_IDS)
def test_map_host_exact(K, dtype, op):
    """map_host with 4096-byte chunks (the smallest the entry takes; a shard spans several and the last is a few
    bytes), pinned src and dst views at element offsets: one rank on [0]; three ranks of 3-element rows on [0, 0, 0];
    and ranks 0 and 2 of those three, which leave rank 1's shard of dst as it was."""
    es = R.ES[dtype]
    n = 5 * 4096 // es + 3
    x = patterns(dtype, n, phase=7)
    rows = n // 3
    lo, hi = (3 * i for i in K.shard_bounds(rows, 3, 1))   # rank 1's elements
    skipped = np.zeros(rows * 3, dtype=bool)
    skipped[lo:hi] = True
    for a, b in {ROW[dtype], SECOND_ROW[dtype]}:
        for src_off, dst_off in ((es, 3 * es), (0, es)):
            src = HostGuarded(n * es, src_off)
            src.view(torch.uint8).copy_(torch.from_numpy(np.ascontiguousarray(x).view(np.uint8)))
            dst = HostGuarded(n * es, dst_off)
            K.map_host(src.view(dtype), op, a, b, out_host=dst.view(dtype), devices=[0], chunk_bytes=4096)
            dst.check("one rank")
            vec = run_map(K, dtype, op, x, a, b, VEC)
            expect(dtype, op, got_bits(dst.view(dtype), dtype), x, a, b, f"one rank {dtype} {op}", same_as=vec)
            for ranks in (None, [0, 2]):
                what = f"ranks {ranks} of [0, 0, 0] {dtype} {op}"
                dst = HostGuarded(rows * 3 * es, dst_off)
                K.map_host(src.view(dtype)[:rows * 3].view(rows, 3), op, a, b,
                           out_host=dst.view(dtype).view(rows, 3), devices=[0, 0, 0], ranks=ranks, chunk_bytes=4096)
                dst.check(what)
                done = ~skipped if ranks else np.ones(rows * 3, dtype=bool)
                expect(dtype, op, got_bits(dst.view(dtype), dtype)[done], x[:rows * 3][done], a, b, what,
                       same_as=vec[:rows * 3][done])
                if ranks:
                    assert bool((dst.view(torch.uint8)[lo * es:hi * es] == Guarded.FILL).all()), \
                        f"{what}: rank 1's shard was written"


# ---- the public API ---------------------------------------------------------------------------------------------------
def _affine_const(a, b):
    def affine_const(x):
        return cases._shard(x) * a + b
    return affine_const


def _deploy(fn, name, n_ranks, **dist):
    comp = kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute(
        "b200", workers=1, num_proc=n_ranks, devices=[0] * n_ranks, **dist)
    return kt.fn(fn, name=name).to(comp)


def _int_inputs(dtype, n, seed):
    return R.to_torch(patterns(dtype, n, phase=seed), dtype)


def _assert_ranks_equal(got, want, what):
    assert isinstance(got, list) and len(got) == len(want), what
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and tuple(g.shape) == tuple(w.shape), what
        assert torch.equal(g.cpu().reshape(-1).view(torch.uint8), w.reshape(-1).view(torch.uint8)), what


CONST_ROWS = [(a, -7) for a in R.INT_SCALARS] + [(3, b) for b in R.INT_SCALARS if b != -7]


@pytest.mark.parametrize("a,b", CONST_ROWS, ids=[f"a{a}-b{b}" for a, b in CONST_ROWS])
def test_api_declared_integer_constants(a, b):
    """kt.mapped("affine", alpha=a, beta=b): the deploy-time self-check (it runs an int64 tensor) refuses a constant an
    int64 tensor cannot take exactly with TypeError; otherwise the small-call lane and remote.map give the body's
    results on int32 and int64.  Without the self-check, the int32 lane takes every constant and an int64 call of a
    refused one raises TypeError."""
    n_ranks = 3
    body = _affine_const(a, b)
    fn = kt.mapped("affine", alpha=a, beta=b)(body)
    ok64 = R.int64_exact(a) and R.int64_exact(b)
    if not ok64:
        with pytest.raises(TypeError, match="exactly representable"):
            _deploy(fn, "t-ew-const", n_ranks, placement="auto")
    for self_check in ((True, False) if ok64 else (False,)):
        remote = _deploy(fn, "t-ew-const", n_ranks, placement="auto", self_check=self_check)
        try:
            assert remote._fast is not None and remote._batch is not None
            for dtype in R.INTS:
                xs = [_int_inputs(dtype, n, seed=n) for n in (1, 5, 263, 1003)]
                if dtype == torch.int64 and not ok64:
                    with pytest.raises(TypeError, match="exactly representable"):
                        remote(xs[-1].cuda(), serialization="pickle")
                    with pytest.raises(TypeError, match="exactly representable"):
                        remote.map([x.cuda() for x in xs], serialization="pickle")
                    continue
                wants = [ref_dispatch.spmd_call(body, x, num_proc=n_ranks, serialization="pickle") for x in xs]
                for x, want in zip(xs, wants):
                    _assert_ranks_equal(remote(x.cuda(), serialization="pickle"), want, (dtype, a, b, "lane"))
                for got, want in zip(remote.map([x.cuda() for x in xs], serialization="pickle"), wants):
                    _assert_ranks_equal(got, want, (dtype, a, b, "map"))
        finally:
            remote.teardown()


def test_api_integer_call_arguments():
    """affine(x, alpha, beta) with the scalars as call arguments, on the general device route (placement="ranks": one
    launch per rank) and the host route: every integer row equals the body's result or, for an int64 row a double
    cannot carry, raises TypeError; a Python float on an integer tensor raises TypeError even when integral."""
    n_ranks = 3
    fn = kt.mapped("affine", alpha="alpha", beta="beta")(_affine_args)
    remote = _deploy(fn, "t-ew-args", n_ranks, placement="ranks")
    try:
        for dtype in R.INTS:
            x = _int_inputs(dtype, 1003, seed=3).reshape(17, 59)
            for a, b in CONST_ROWS:
                for resident in ("device", "host"):
                    arg = x.cuda() if resident == "device" else x
                    if dtype == torch.int64 and not (R.int64_exact(a) and R.int64_exact(b)):
                        with pytest.raises(TypeError, match="exactly representable"):
                            remote(arg, a, b, serialization="pickle")
                        continue
                    want = ref_dispatch.spmd_call(_affine_args, x, a, b, num_proc=n_ranks, serialization="pickle")
                    _assert_ranks_equal(remote(arg, a, b, serialization="pickle"), want, (dtype, a, b, resident))
            for a, b in ((2.0, 1), (3, -1.0)):
                with pytest.raises(TypeError, match="not an integer"):
                    remote(x.cuda(), a, b, serialization="pickle")
    finally:
        remote.teardown()


def _affine_args(x, alpha, beta):
    return cases._shard(x) * alpha + beta
