"""-m gpu: the CUDA kernels, called through the C-ABI, against the oracle (the reference's SPMD
semantics evaluated on CPU) — bit-exact for every dtype/op. The sum reduction has its own file, test_gpu_reduce.py."""
import ctypes
import os

import pytest
import torch

from conftest import resolve_args

pytestmark = pytest.mark.gpu

from oracle import cases, ref_dispatch  # noqa: E402


@pytest.fixture(scope="module")
def K():
    assert torch.cuda.is_available()
    from kubetorch_b200.device import lib as L
    from kubetorch_b200.device import ops

    L.load()
    ops.ensure_init([0])
    return ops


def _rand(dtype, n, seed=0):
    g = torch.Generator().manual_seed(seed)
    if dtype == torch.float32:
        return torch.randn(n, generator=g)
    if dtype == torch.bfloat16:
        return torch.randn(n, generator=g).bfloat16()
    if dtype == torch.float16:
        return (torch.randn(n, generator=g) * 8).half()
    if dtype == torch.uint8:
        return torch.randint(0, 256, (n,), dtype=torch.uint8, generator=g)
    if dtype == torch.int32:
        return torch.randint(-(2**31), 2**31 - 1, (n,), dtype=torch.int32, generator=g)
    return torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, generator=g)


def _cpu_op(x, op, a, b):
    if op == "identity":
        return x.clone()
    if op == "scale":
        return x * a
    return x * a + b


SIZES = [0, 1, 7, 31, 255, 1000, 4097, 65536 + 3, (1 << 20) + 17]
VARIANTS = [1, 2, 3]  # VEC, TMA, SCALAR


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("dtype,op,a,b", [
    (torch.uint8, "identity", 1, 0),
    (torch.float32, "identity", 1, 0),
    (torch.float32, "scale", 2.0, 0),
    (torch.float32, "scale", 0.1, 0),
    (torch.float32, "affine", 0.1, 0.3),
    (torch.bfloat16, "scale", 2.0, 0),
    (torch.bfloat16, "scale", 1.7, 0),
    (torch.bfloat16, "affine", 1.5, 0.25),
    (torch.bfloat16, "affine", 1.7, -0.3),   # beta is rounded to bf16 before the add (torch CPU scalar semantics)
    (torch.float16, "scale", 1.7, 0),
    (torch.float16, "affine", 1.5, 0.25),
    (torch.float16, "affine", 1.7, -0.3),
    (torch.float16, "identity", 1, 0),
    (torch.int32, "scale", 65537, 0),
    (torch.int32, "affine", 3, -7),
    (torch.int64, "scale", -5, 0),
    (torch.int64, "affine", -5, 11),
])
def test_map_matches_torch_cpu_bit_exact(K, dtype, op, a, b, variant):
    for n in SIZES:
        x = _rand(dtype, n, seed=n)
        want = _cpu_op(x, op, a, b)
        got = K.map_tensor(x.cuda(), op, a, b, variant=variant).cpu()
        assert got.dtype == want.dtype
        assert torch.equal(got.view(torch.uint8), want.view(torch.uint8)), (dtype, op, n, variant)


@pytest.mark.parametrize("variant", [1, 3])
def test_map_misaligned_and_inplace(K, variant):
    base = _rand(torch.float32, 10_000).cuda()
    for off in (1, 3, 5):  # 4-byte aligned only → scalar path, still exact
        x = base[off:off + 5000]
        out = torch.empty(5003, device="cuda")[off % 3:off % 3 + 5000]
        K.map_tensor(x, "affine", 0.5, 1.25, out=out, variant=variant)
        assert torch.equal(out.cpu(), x.cpu() * 0.5 + 1.25)
    y = base.clone()
    K.map_tensor(y, "scale", 3.0, out=y, variant=variant)  # src == dst
    assert torch.equal(y.cpu(), base.cpu() * 3.0)


def test_map_rejects_bad_arguments(K):
    from kubetorch_b200.device import lib as L

    x = torch.zeros(64, device="cuda")
    with pytest.raises(L.KtbError) as ei:
        L.call("ktb_map", 0, 7, L.F32, x.data_ptr(), x.data_ptr(), 64, 1.0, 0.0, 0, 0)
    assert ei.value.status == L.ERR_ARG
    with pytest.raises(L.KtbError):
        L.call("ktb_map", 0, L.OP_SCALE, L.U8, x.data_ptr(), x.data_ptr(), 64, 1.0, 0.0, 0, 0)
    with pytest.raises(L.KtbError):  # partial overlap
        L.call("ktb_map", 0, L.OP_SCALE, L.F32, x.data_ptr(), x.data_ptr() + 16, 32, 1.0, 0.0, 0, 0)
    with pytest.raises(L.KtbError) as ei:
        L.call("ktb_map", 9, L.OP_SCALE, L.F32, x.data_ptr(), x.data_ptr(), 64, 1.0, 0.0, 0, 0)
    assert ei.value.status == L.ERR_STATE


def test_golden_reference_runtime_cases(K, golden):
    """Every tensor case recorded from the UNMODIFIED reference runtime, reproduced by the kernels with
    n_ranks time-sliced on cuda:0 (same shard arithmetic, same kernels)."""
    table = {"double": ("scale", 2.0, 0.0), "identity": ("identity", 1.0, 0.0)}
    checked = 0
    for name, rec in golden["cases"].items():
        fn = rec["callable"]
        if rec["status_code"] != 200 or fn not in ("double", "identity", "scale", "affine"):
            continue
        if (rec.get("kwargs") or {}).get("workers"):
            continue  # `workers=` sub-selections are host logic, covered on the CPU backends
        args = resolve_args(golden, rec["args"])
        x = args[0]
        if fn in table:
            op, a, b = table[fn]
        elif fn == "scale":
            op, a, b = "scale", args[1], 0
        else:
            op, a, b = "affine", args[1], args[2]
        # records taken on K real pods x P ranks have world size K*P
        n_ranks = rec["distributed_config"]["num_proc"] * len(rec.get("pods") or [None])
        out = K.scatter_map_gather(x.cuda(), op, a, b, devices=[0] * n_ranks).cpu()
        want = torch.cat([w.reshape(-1) for w in rec["result"]])
        assert torch.equal(out.view(torch.uint8), want.view(torch.uint8)), name
        # shard boundaries = the reference's per-rank result lengths
        for r, w in enumerate(rec["result"]):
            b0, e0 = K.shard_bounds(x.numel(), n_ranks, r)
            assert e0 - b0 == w.numel(), (name, r)
        checked += 1
    assert checked >= 10


def test_pack_unpack_roundtrip(K):
    g = torch.Generator().manual_seed(3)
    shapes = [(1,), (3, 5), (0,), (257,), (64, 64), (1000, 33), (7,), (2, 3, 4)]
    dtypes = [torch.float32, torch.bfloat16, torch.uint8, torch.int64, torch.float32, torch.bfloat16, torch.int32,
              torch.float32]
    srcs = []
    for s, d in zip(shapes, dtypes):
        t = torch.randint(0, 200, s, generator=g).to(d)
        srcs.append(t.cuda())
    # add many tiny tensors (> one launch worth of segment descriptors) and one misaligned view
    big = torch.arange(5000, dtype=torch.float32).cuda()
    srcs += [big[i * 10 + 1:i * 10 + 8].clone() for i in range(300)]
    srcs.append(big[1:1001])  # 4-byte aligned source pointer
    arena, offsets = K.pack(srcs)
    torch.cuda.synchronize()
    assert all(o % 256 == 0 for o in offsets)
    specs = [(t.dtype, tuple(t.shape)) for t in srcs]
    for v, t in zip(K.arena_views(arena, offsets, specs), srcs):
        assert torch.equal(v.cpu().view(torch.uint8), t.cpu().contiguous().view(torch.uint8))
    outs = [torch.empty_like(t, memory_format=torch.contiguous_format) for t in srcs]
    K.unpack(arena, offsets, outs)
    for o, t in zip(outs, srcs):
        assert torch.equal(o.cpu().view(torch.uint8), t.cpu().contiguous().view(torch.uint8))
    # the codec the arena replaces: reference pickles+base64s the same leaves; payload must survive
    body = ref_dispatch.serialize_body(ref_dispatch.build_call_body(*[t.cpu() for t in srcs[:8]]), "pickle")
    back, _ = ref_dispatch.parse_callable_params(dict(body), "pickle")
    for v, t in zip(K.arena_views(arena, offsets, specs)[:8], back):
        assert torch.equal(v.cpu().view(torch.uint8), t.contiguous().view(torch.uint8))


@pytest.mark.parametrize("count", [96, 97, 1024, 1025, 2500])
@pytest.mark.parametrize("large", [1, 0])
def test_pack_many_segments_descriptor_batches(K, count, large):
    """> 96 segments ride in large kernel parameters (one launch per 1024); tuning 12 = 0 forces 96 per launch."""
    g = torch.Generator().manual_seed(count)
    sizes = torch.randint(1, 9000, (count,), generator=g).tolist()
    sizes[count // 2] = 300_001          # one segment spanning many 32 KiB tiles
    flat = torch.randint(0, 255, (sum(sizes) + 64,), generator=g, dtype=torch.uint8).cuda()
    srcs, off = [], 0
    for i, n in enumerate(sizes):
        srcs.append(flat[off + (i % 3):off + (i % 3) + n])      # mixed 1/2/16/32-byte alignment
        off += n
    K.set_tuning(12, large)
    try:
        arena, offsets = K.pack(srcs)
        outs = [torch.empty(n, dtype=torch.uint8, device="cuda") for n in sizes]
        K.unpack(arena, offsets, outs)
        torch.cuda.synchronize()
    finally:
        K.set_tuning(12, 1)
    a = arena.cpu()
    for t, o, dst in zip(srcs, offsets, outs):
        assert torch.equal(a[o:o + t.numel()], t.cpu())
        assert torch.equal(dst.cpu(), t.cpu())


def test_map_batch(K):
    xs = [_rand(torch.float32, n, seed=n).cuda() for n in [1, 5, 256, 1000, 4096, 100_003] + [64] * 200]
    outs = K.map_batch(xs, "affine", 0.5, 2.0)
    for x, o in zip(xs, outs):
        assert torch.equal(o.cpu(), x.cpu() * 0.5 + 2.0)


def test_broadcast_same_device(K):
    x = _rand(torch.uint8, 1_000_003).cuda()
    dsts = [torch.zeros_like(x) for _ in range(3)]
    K.broadcast(x, dsts)
    for d in dsts:
        assert torch.equal(d.cpu(), x.cpu())
    xm = x[1:70_001]  # misaligned → byte kernel
    dm = [torch.zeros(70_000, dtype=torch.uint8, device="cuda") for _ in range(2)]
    K.broadcast(xm, dm)
    assert all(torch.equal(d.cpu(), xm.cpu()) for d in dm)


def test_map_host_pipeline(K):
    for n in [1, 1000, (1 << 22) + 13]:
        x = _rand(torch.float32, n, seed=5).pin_memory()
        out = K.map_host(x, "affine", 0.25, -1.0, chunk_bytes=1 << 20)
        assert torch.equal(out, x * 0.25 + -1.0)


def test_map_host_multi_single_thread_pipeline(K):
    for n in [3, 70_001, (1 << 22) + 5]:
        x = _rand(torch.float32, n, seed=9).pin_memory()
        out = K.map_host_multi(x, "affine", 1.5, 0.5, devices=[0], chunk_bytes=1 << 20)
        assert torch.equal(out, x * 1.5 + 0.5)
    x2 = _rand(torch.int32, 40_000).reshape(100, 400).pin_memory()
    assert torch.equal(K.map_host_multi(x2, "scale", 3, devices=[0]), x2 * 3)


def test_zero_copy_host_pointers(K):
    """Mapped pinned host memory is a valid src/dst for the kernels (UVA)."""
    x = _rand(torch.float32, 100_000).pin_memory()
    out = torch.empty_like(x).pin_memory()
    from kubetorch_b200.device import lib as L

    L.call("ktb_map", 0, L.OP_SCALE, L.F32, x.data_ptr(), out.data_ptr(), x.numel(), 2.0, 0.0, L.VARIANT_VEC,
           torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(out, x * 2)


def test_full_size_properties(K):
    """BASELINE configs[1] at full size (64 Mi fp32): linearity and index checks instead of a CPU pass."""
    n = 1 << 26
    x = (torch.arange(n, dtype=torch.int32, device="cuda") % (1 << 20)).float()  # exact in fp32
    y = K.scatter_map_gather(x, "scale", 2.0, devices=[0] * 8)
    idx = torch.randint(0, n, (1 << 16,), device="cuda")
    assert torch.equal(y[idx], ((idx % (1 << 20)) * 2).float())
    assert torch.equal(y[-5:].cpu(), x[-5:].cpu() * 2)
    # checksum of checksums: sum(2x) == 2 sum(x), exactly, in int64
    xi = torch.arange(n, dtype=torch.int64, device="cuda")
    t2, p2 = K.scatter_map_reduce(xi, "scale", 2, devices=[0] * 8)
    assert int(t2) == n * (n - 1) and sum(p2.tolist()) == n * (n - 1)
    # identity round trip is idempotent
    z = K.map_tensor(K.map_tensor(x, "identity"), "identity")
    assert torch.equal(z, x)


def test_push_pipeline_emulated_on_one_gpu(K):
    """push/push flag pipeline with all ranks time-sliced on cuda:0 (same stream → root first): same results
    as the oracle, across consecutive calls (staging parity + ack back-pressure) and ragged shards."""
    for n_ranks, n in ((4, 1 << 20), (3, 1003), (8, (1 << 22) + 77), (2, 5)):
        x = _rand(torch.float32, n, seed=n).cuda()
        sess = K.PushSession([0] * n_ranks, K.shard_bounds(n, n_ranks, 0)[1] * 4, n_chunks=4)
        for it in range(5):
            a, b = 0.5 + it, 1.0 - it
            y = torch.zeros_like(x)
            sess.call(x, y, "affine", a, b)
            torch.cuda.synchronize()
            assert torch.equal(y.cpu(), x.cpu() * a + b), (n_ranks, n, it)
        sess.check()
    xi = _rand(torch.int64, 70_001).cuda()
    sess = K.PushSession([0, 0, 0], K.shard_bounds(70_001, 3, 0)[1] * 8, n_chunks=8)
    yi = torch.zeros_like(xi)
    sess.call(xi, yi, "scale", -3)
    torch.cuda.synchronize()
    assert torch.equal(yi.cpu(), xi.cpu() * -3)


def test_numa_sharded_pinned_buffers_are_pinned_pooled_and_correct(K):
    """kt.pinned_empty / ktb_host_alloc_sharded: page-locked (torch sees it as pinned), usable by the host pipeline,
    returned to the pool when the last view dies and handed out again without a new allocation."""
    import gc

    import kubetorch_b200 as kt

    n = (8 << 20) // 4 + 12345                       # > 4 MiB: the sharded allocator, ragged size
    x = kt.pinned_empty((n,), torch.float32, gpus=1)
    assert x.is_pinned() and not x.is_cuda and x.numel() == n
    x.copy_(torch.arange(n, dtype=torch.float32))
    y = K.map_host(x, "scale", 2.0, device=0)
    assert torch.equal(y, x * 2)
    ptr = x.data_ptr()
    view = x[10:20]
    del x
    gc.collect()
    assert view.data_ptr() == ptr + 40                # a living view keeps the block out of the pool
    z = kt.pinned_empty((n,), torch.float32, gpus=1)
    zptr = z.data_ptr()
    assert zptr != ptr
    del view, z
    gc.collect()
    again = kt.pinned_empty((n,), torch.float32, gpus=1)
    assert again.data_ptr() in (ptr, zptr) and again.is_pinned()   # a pooled block is reused, nothing new is allocated
    small = kt.pinned_empty((16,), torch.float32, gpus=1)          # small tensors come from torch's pinned allocator
    assert small.is_pinned()
    assert K.device_numa_node(0) >= -1
