"""-m gpu: the argument statuses of the element-wise entry points of the C-ABI.  Every entry rejects an unknown op, an
unknown dtype and an (op, dtype) pair it has no kernel for with KTB_ERR_ARG, before any kernel runs; empty calls keep
their documented statuses.  One GPU; the multi-rank entries run with every rank on device 0."""
from ctypes import c_int, c_size_t, c_void_p

import pytest
import torch

from kubetorch_b200.device import lib as L

pytestmark = pytest.mark.gpu

N = 4096                 # elements of every non-empty call
ES_MAX = 8               # the widest element (I64): buffers hold N of them
CHUNK = 1 << 16          # chunk_bytes of the host-resident entries
BAD_OPS = (-1, 3, 7)
BAD_DTYPES = (-1, 6, 99)
# ktb_map_host_multi_subset: ktb_map_host_multi with two ranks on device 0, rank 1 left out (NULL staging)
MAP = ("ktb_map", "ktb_map_batch", "ktb_push_consume", "ktb_scatter_map_gather", "ktb_map_host_multi",
       "ktb_map_host_multi_subset")
REDUCE = ("ktb_map_reduce_sum", "ktb_scatter_map_reduce")
SCATTER = ("ktb_push_scatter", "ktb_push_scatter_chunked", "ktb_push_scatter_ce")   # take no op


@pytest.fixture(scope="module")
def call():
    """call(entry, op, dtype, n) -> the raw status of `entry` on n elements, with real buffers of the documented sizes."""
    from kubetorch_b200.device import ops

    lib = L.load()
    ops.ensure_init([0])

    def dev(nbytes):
        return torch.zeros(nbytes, dtype=torch.uint8, device="cuda")

    src, dst = dev(N * ES_MAX), dev(N * ES_MAX)
    out, partials, ws = dev(8), dev(8), dev(lib.ktb_reduce_workspace_bytes())
    src_h = torch.zeros(N * ES_MAX, dtype=torch.uint8).pin_memory()
    dst_h = torch.zeros(N * ES_MAX, dtype=torch.uint8).pin_memory()
    stage_in, stage_out = dev(2 * CHUNK), dev(2 * CHUNK)      # double-buffered chunk staging
    stride = N * ES_MAX
    stage = dev(2 * stride)                                  # push staging: two halves of stage_stride
    ctrl_root, ctrl_rank = dev(lib.ktb_push_control_bytes()), dev(lib.ktb_push_control_bytes())
    one, two = L.arr(c_int, [0]), L.arr(c_int, [0, 0])      # devs of one rank, of two ranks

    def ptr(t):
        return t.data_ptr()

    def vp(*ts):   # pointer array; None is a null entry
        return L.arr(c_void_p, [None if t is None else t.data_ptr() for t in ts])

    entries = {
        "ktb_map": lambda op, dt, n: lib.ktb_map(0, op, dt, ptr(src), ptr(dst), n, 2.0, 1.0, L.VARIANT_AUTO, 0),
        "ktb_map_batch": lambda op, dt, n: lib.ktb_map_batch(0, op, dt, vp(src), vp(dst), L.arr(c_size_t, [n]), 1,
                                                             2.0, 1.0, 0),
        "ktb_push_consume": lambda op, dt, n: lib.ktb_push_consume(0, op, dt, ptr(stage), stride, ptr(dst), n, 2.0, 1.0,
                                                                   ptr(ctrl_rank), ptr(ctrl_root), 1, 4, 1, 0),
        "ktb_scatter_map_gather": lambda op, dt, n: lib.ktb_scatter_map_gather(op, dt, ptr(src), ptr(dst), n, 1, 2.0,
                                                                               1.0, 1, one, 0, L.VARIANT_AUTO, None),
        "ktb_map_host_multi": lambda op, dt, n: lib.ktb_map_host_multi(op, dt, ptr(src_h), ptr(dst_h), n, 1, 2.0, 1.0,
                                                                       1, one, CHUNK, vp(stage_in), vp(stage_out)),
        "ktb_map_host_multi_subset": lambda op, dt, n: lib.ktb_map_host_multi(
            op, dt, ptr(src_h), ptr(dst_h), n, 1, 2.0, 1.0, 2, two, CHUNK, vp(stage_in, None), vp(stage_out, None)),
        "ktb_map_reduce_sum": lambda op, dt, n: lib.ktb_map_reduce_sum(0, op, dt, ptr(src), n, 2.0, 1.0, ptr(out),
                                                                       ptr(ws), 0),
        "ktb_scatter_map_reduce": lambda op, dt, n: lib.ktb_scatter_map_reduce(op, dt, ptr(src), n, 1, 2.0, 1.0, 1, one,
                                                                               0, ptr(partials), ptr(out), vp(ws), None),
        # root 0 pushes to rank 1, both on device 0
        "ktb_push_scatter": lambda op, dt, n: lib.ktb_push_scatter(0, ptr(src), n, 1, dt, 2, 0, vp(None, stage), stride,
                                                                   vp(ctrl_root, ctrl_rank), ptr(ctrl_root), 4, 1, 0),
        "ktb_push_scatter_chunked": lambda op, dt, n: lib.ktb_push_scatter_chunked(
            0, ptr(src), n, 1, dt, 2, 0, vp(None, stage), stride, vp(ctrl_root, ctrl_rank), ptr(ctrl_root), 1024, 0, 1, 0),
        "ktb_push_scatter_ce": lambda op, dt, n: lib.ktb_push_scatter_ce(
            0, ptr(src), n, 1, dt, 2, 0, two, vp(None, stage), stride, vp(ctrl_root, ctrl_rank), ptr(ctrl_root), 1024, 1,
            0),
    }

    def run(entry, op, dtype, n):
        status = entries[entry](op, dtype, n)
        torch.cuda.synchronize()   # a rejected call leaves the device healthy
        return status

    return run


ROWS = (
    [(e, op, L.F32) for e in MAP + REDUCE for op in BAD_OPS]
    + [(e, L.OP_IDENTITY, dt) for e in MAP + REDUCE + SCATTER for dt in BAD_DTYPES]
    + [(e, op, L.U8) for e in MAP for op in (L.OP_SCALE, L.OP_AFFINE)]
    + [(e, op, L.U8) for e in REDUCE for op in (L.OP_IDENTITY, L.OP_SCALE, L.OP_AFFINE)]
)


@pytest.mark.parametrize("entry,op,dtype", ROWS, ids=[f"{e}-op{o}-dtype{d}" for e, o, d in ROWS])
def test_bad_op_or_dtype_is_rejected(call, entry, op, dtype):
    assert call(entry, op, dtype, N) == L.ERR_ARG


# An empty call with a bad op: the entries that check the op on entry reject it (ktb_map_batch when it has segments,
# even empty ones); the entries whose empty call returns before any work return KTB_OK.
EMPTY = [("ktb_map", L.ERR_ARG), ("ktb_map_batch", L.ERR_ARG), ("ktb_map_reduce_sum", L.ERR_ARG),
         ("ktb_scatter_map_reduce", L.ERR_ARG), ("ktb_push_consume", L.ERR_ARG),
         ("ktb_map_host_multi", L.OK), ("ktb_map_host_multi_subset", L.OK), ("ktb_scatter_map_gather", L.OK)]


@pytest.mark.parametrize("op", BAD_OPS)
@pytest.mark.parametrize("entry,want", EMPTY, ids=[e for e, _ in EMPTY])
def test_empty_call_with_bad_op(call, entry, want, op):
    assert call(entry, op, L.F32, 0) == want


@pytest.mark.parametrize("op", BAD_OPS)
def test_map_batch_without_segments_is_ok_whatever_the_op(call, op):
    lib = L.load()
    assert lib.ktb_map_batch(0, op, L.F32, None, None, None, 0, 2.0, 1.0, 0) == L.OK
    torch.cuda.synchronize()


# ktb_map_host_multi's rank rules, two ranks on device 0: a rank whose two staging buffers are NULL is not part of the
# call, one NULL of a pair is an error, and a device may carry several ranks (a bad op or dtype on a rank subset: the
# ktb_map_host_multi_subset rows above).  case: (op, stage_in, stage_out, status)
HOST_RANKS = {
    "one_null_stage": (L.OP_SCALE, ("in", "in"), ("out", None), L.ERR_ARG),
    "all_ranks_null": (L.OP_SCALE, (None, None), (None, None), L.OK),
    "shared_device": (L.OP_SCALE, ("in", "in"), ("out", "out"), L.OK),
}


@pytest.mark.parametrize("case", list(HOST_RANKS))
def test_map_host_multi_rank_rules(case):
    from kubetorch_b200.device import ops

    lib = L.load()
    ops.ensure_init([0])
    op, ins, outs, want = HOST_RANKS[case]
    stage = {"in": torch.zeros(2 * CHUNK, dtype=torch.uint8, device="cuda"),
             "out": torch.zeros(2 * CHUNK, dtype=torch.uint8, device="cuda")}
    src = torch.arange(N, dtype=torch.float32).pin_memory()
    dst = torch.full((N,), -1.0).pin_memory()

    def stages(keys):
        return L.arr(c_void_p, [stage[k].data_ptr() if k else None for k in keys])

    status = lib.ktb_map_host_multi(op, L.F32, src.data_ptr(), dst.data_ptr(), N, 1, 2.0, 1.0, 2, L.arr(c_int, [0, 0]),
                                    CHUNK, stages(ins), stages(outs))
    torch.cuda.synchronize()
    assert status == want
    # a rejected call and a call without ranks leave dst untouched; two ranks sharing the device compute all of it
    assert torch.equal(dst, src * 2.0 if case == "shared_device" else torch.full((N,), -1.0))
