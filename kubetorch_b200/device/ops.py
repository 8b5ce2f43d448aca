"""Tensor-facing wrappers over the C-ABI (torch.Tensor is the arg/result currency).

Everything here enqueues hand-written sm_90a kernels from libktb200.so on the caller's current
CUDA stream; nothing computes with torch ops.  Reference rows replaced (SURVEY.md §8(a)):
a3/a11/a12 (pack/unpack codecs), a7-a9 (fan-out / fan-in), a11 (callable execution for the
registered ops).
"""
from __future__ import annotations

import ctypes
import threading
from typing import List, Optional, Sequence, Tuple

import torch

from . import lib as L

_DTYPE_CODES = {
    torch.uint8: L.U8,
    torch.float32: L.F32,
    torch.bfloat16: L.BF16,
    torch.int32: L.I32,
    torch.int64: L.I64,
    torch.float16: L.F16,
}
OPS = {"identity": L.OP_IDENTITY, "scale": L.OP_SCALE, "affine": L.OP_AFFINE}

_init_lock = threading.Lock()
_registered: set = set()


def require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError(
            "kubetorch_b200 device path needs a CUDA device (H100, sm_90a); no CPU fallback exists. "
            "Use kt.Compute(cpus=...) for the in-process CPU backend."
        )


def device_count() -> int:
    return torch.cuda.device_count()


def synchronize(device: int) -> None:
    torch.cuda.synchronize(device)


def is_pinned(t: torch.Tensor) -> bool:
    return (not t.is_cuda) and t.is_pinned()


def join_devices(root: int, devices: Sequence[int]) -> None:
    """Order the root's current stream after everything enqueued so far on the current streams of `devices`."""
    root_stream = torch.cuda.current_stream(root)
    for d in set(int(d) for d in devices):
        if d == root:
            continue
        ev = torch.cuda.Event()
        with torch.cuda.device(d):
            ev.record(torch.cuda.current_stream(d))
        with torch.cuda.device(root):
            root_stream.wait_event(ev)


def ensure_init(devices: Sequence[int]) -> None:
    """Register devices with the library (enables NVLink peer access between all registered)."""
    if _registered.issuperset(devices):  # per-call fast path: nothing to register
        return
    require_cuda()
    devs = [int(d) for d in devices]
    with _init_lock:
        new = [d for d in devs if d not in _registered]
        if not new:
            return
        L.call("ktb_init", len(new), L.arr(ctypes.c_int, new))
        _registered.update(new)


def dtype_code(dtype: torch.dtype) -> int:
    try:
        return _DTYPE_CODES[dtype]
    except KeyError:
        raise TypeError(f"kubetorch_b200 mapped ops support {sorted(str(k) for k in _DTYPE_CODES)}, got {dtype}")


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def current_stream_handle(device: int) -> int:
    """cudaStream_t of torch's current stream on `device` (the raw getter skips building a Stream object)."""
    if _raw_stream is not None:
        return int(_raw_stream(device))
    return int(torch.cuda.current_stream(device).cuda_stream)


def _stream(device: int, stream: Optional[torch.cuda.Stream]) -> int:
    return int(stream.cuda_stream) if stream is not None else current_stream_handle(device)


def _check_dev_tensor(t: torch.Tensor, name: str) -> int:
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    return t.device.index


def row_elems(t: torch.Tensor) -> int:
    """Elements per dim-0 row (the indivisible unit of `x.chunk(world)`)."""
    if t.dim() == 0 or t.shape[0] == 0:
        return 1
    return max(1, t.numel() // t.shape[0])


def shard_bounds(n: int, world: int, rank: int) -> Tuple[int, int]:
    """Python twin of ktb_shard_bounds (tests/test_abi.py checks they agree): `x.chunk(world)[rank]` bounds."""
    if world <= 0 or rank < 0 or rank >= world:
        raise ValueError(f"bad world/rank {world}/{rank}")
    chunk = -(-n // world)
    b = min(n, chunk * rank)
    return b, min(n, b + chunk)


def shard_bounds_c(n: int, world: int, rank: int) -> Tuple[int, int]:
    b, e = ctypes.c_size_t(), ctypes.c_size_t()
    L.call("ktb_shard_bounds", n, world, rank, ctypes.byref(b), ctypes.byref(e))
    return b.value, e.value


# ---- element-wise map ------------------------------------------------------------------------------
def map_tensor(
    x: torch.Tensor,
    op: str = "identity",
    alpha: float = 1.0,
    beta: float = 0.0,
    out: Optional[torch.Tensor] = None,
    variant: int = L.VARIANT_AUTO,
    stream: Optional[torch.cuda.Stream] = None,
    device: Optional[int] = None,
) -> torch.Tensor:
    """out = op(x) on `device` (default: x's device). x/out may live on a peer GPU."""
    xd = _check_dev_tensor(x, "x")
    dev = xd if device is None else int(device)
    ensure_init({dev, xd})
    if out is None:
        with torch.cuda.device(dev):
            out = torch.empty_like(x, device=f"cuda:{dev}")
    else:
        od = _check_dev_tensor(out, "out")
        ensure_init({od})
        if out.dtype != x.dtype or out.numel() != x.numel():
            raise ValueError("out must match x in dtype and numel")
    L.call(
        "ktb_map", dev, OPS[op], dtype_code(x.dtype), x.data_ptr(), out.data_ptr(), x.numel(),
        float(alpha), float(beta), int(variant), _stream(dev, stream),
    )
    return out


def fast_dtype_codes(integral_params: bool) -> dict:
    """dtype -> code for the small-call lane; integer dtypes only when alpha/beta are integral (torch would promote)."""
    codes = dict(_DTYPE_CODES)
    if not integral_params:
        codes.pop(torch.int32, None)
        codes.pop(torch.int64, None)
    return codes


def fast_map(device: int, op: str, alpha: float, beta: float):
    """launch(dtype_code, src_ptr, dst_ptr, n_elems): ONE ctypes hop into ktb_map on torch's current stream of
    `device`, everything else pre-bound (no per-call marshalling of constants, no Python-level checks)."""
    ensure_init({device})
    fn = L.load().ktb_map
    op_code, dev = OPS[op], int(device)
    raw = _raw_stream if _raw_stream is not None else (lambda d: torch.cuda.current_stream(d).cuda_stream)
    check = L.check

    def launch(code, src, dst, n):
        rc = fn(dev, op_code, code, src, dst, n, alpha, beta, 0, raw(dev))
        if rc:
            check(rc)

    return launch


def batch_map(device: int, op: str, alpha: float, beta: float):
    """run(dtype_code, dtype, xs, sizes) -> tuple of outputs: n small calls out_i = op(x_i) in ONE segmented launch
    (ktb_map_batch), the outputs carved out of one fresh arena (256-byte aligned, so every output is a valid vector
    target)."""
    ensure_init({device})
    fn = L.load().ktb_map_batch
    op_code, dev = OPS[op], int(device)
    raw = _raw_stream if _raw_stream is not None else (lambda d: torch.cuda.current_stream(d).cuda_stream)

    def run(code, dtype, xs, sizes):
        n = len(xs)
        es = xs[0].element_size()
        align = 256 // es
        padded = [(s + align - 1) // align * align for s in sizes]
        arena = torch.empty(sum(padded), dtype=dtype, device=f"cuda:{dev}")
        base = arena.data_ptr()
        outs, dst, off = [], [], 0
        pieces = arena.split(padded)
        for i in range(n):
            outs.append(pieces[i][:sizes[i]] if padded[i] != sizes[i] else pieces[i])
            dst.append(base + off * es)
            off += padded[i]
        rc = fn(dev, op_code, code, (ctypes.c_void_p * n)(*[x.data_ptr() for x in xs]), (ctypes.c_void_p * n)(*dst),
                (ctypes.c_size_t * n)(*sizes), n, alpha, beta, raw(dev))
        if rc:
            L.check(rc)
        return outs

    return run


_ws_cache = {}


def _workspace(dev: int, stream: Optional[int] = None) -> torch.Tensor:
    """Reduce workspace (ticket counter + per-CTA partials) of one stream on `dev`, default torch's current one.
    Reductions on one stream run in order and may share it; two streams must never share one."""
    current = current_stream_handle(dev)
    key = (dev, current if stream is None else int(stream))
    ws = _ws_cache.get(key)
    if ws is None:
        nbytes = L.load().ktb_reduce_workspace_bytes()
        ws = torch.zeros(nbytes, dtype=torch.uint8, device=f"cuda:{dev}")
        if key[1] != current:  # the zero fill runs on the current stream: finish it before another stream uses ws
            torch.cuda.current_stream(dev).synchronize()
        _ws_cache[key] = ws
    return ws


def acc_dtype(dtype: torch.dtype) -> torch.dtype:
    return torch.float32 if dtype in (torch.float32, torch.bfloat16, torch.float16) else torch.int64


def map_reduce_sum(
    x: torch.Tensor,
    op: str = "identity",
    alpha: float = 1.0,
    beta: float = 0.0,
    out: Optional[torch.Tensor] = None,
    stream: Optional[torch.cuda.Stream] = None,
    device: Optional[int] = None,
) -> torch.Tensor:
    """out[0] = sum(op(x)); fp32 accumulator for f32/bf16, int64 for integer dtypes."""
    xd = _check_dev_tensor(x, "x")
    dev = xd if device is None else int(device)
    ensure_init({dev, xd})
    if x.dtype == torch.uint8:
        raise TypeError("uint8 is not reducible")
    if out is None:
        out = torch.empty(1, dtype=acc_dtype(x.dtype), device=f"cuda:{dev}")
    st = _stream(dev, stream)
    L.call(
        "ktb_map_reduce_sum", dev, OPS[op], dtype_code(x.dtype), x.data_ptr(), x.numel(), float(alpha),
        float(beta), out.data_ptr(), _workspace(dev, st).data_ptr(), st,
    )
    return out


# ---- pack / unpack ---------------------------------------------------------------------------------
def pack_layout(nbytes: Sequence[int]) -> Tuple[List[int], int]:
    n = len(nbytes)
    offs = (ctypes.c_size_t * max(n, 1))()
    total = ctypes.c_size_t()
    L.call("ktb_pack_layout", L.arr(ctypes.c_size_t, list(nbytes)) if n else None, n, offs, ctypes.byref(total))
    return [offs[i] for i in range(n)], total.value


def pack(
    tensors: Sequence[torch.Tensor],
    arena: Optional[torch.Tensor] = None,
    stream: Optional[torch.cuda.Stream] = None,
) -> Tuple[torch.Tensor, List[int]]:
    """Gather tensor leaves into one uint8 arena at 256-byte aligned offsets. Returns (arena, offsets)."""
    if not tensors:
        return (arena if arena is not None else torch.empty(0, dtype=torch.uint8)), []
    dev = _check_dev_tensor(tensors[0], "tensors[0]")
    for i, t in enumerate(tensors):
        if _check_dev_tensor(t, f"tensors[{i}]") != dev:
            raise ValueError("all tensors to pack must be on the same device")
    ensure_init({dev})
    nbytes = [t.numel() * t.element_size() for t in tensors]
    offsets, total = pack_layout(nbytes)
    if arena is None:
        arena = torch.empty(max(total, 1), dtype=torch.uint8, device=f"cuda:{dev}")
    elif arena.numel() * arena.element_size() < total:
        raise ValueError(f"arena too small: need {total} bytes")
    n = len(tensors)
    c_offs = L.arr(ctypes.c_size_t, offsets)
    L.call(
        "ktb_pack", dev, L.arr(ctypes.c_void_p, [t.data_ptr() for t in tensors]), L.arr(ctypes.c_size_t, nbytes), n,
        arena.data_ptr(), arena.numel() * arena.element_size(), c_offs, 0, _stream(dev, stream),
    )
    return arena, offsets


class PackPlan:
    """A pack (or unpack) of a fixed set of tensors into a fixed arena with the ctypes descriptor
    arrays built once: `run()` is one C call (no per-tensor Python work), graph-capturable."""

    def __init__(self, tensors: Sequence[torch.Tensor], arena: Optional[torch.Tensor] = None):
        self.dev = _check_dev_tensor(tensors[0], "tensors[0]")
        ensure_init({self.dev})
        self.tensors = list(tensors)
        self.nbytes = [t.numel() * t.element_size() for t in tensors]
        self.offsets, self.total = pack_layout(self.nbytes)
        self.arena = arena if arena is not None else torch.empty(max(self.total, 1), dtype=torch.uint8,
                                                                   device=f"cuda:{self.dev}")
        n = len(tensors)
        self._n = n
        self._ptrs = L.arr(ctypes.c_void_p, [t.data_ptr() for t in tensors])
        self._nb = L.arr(ctypes.c_size_t, self.nbytes)
        self._offs = L.arr(ctypes.c_size_t, self.offsets)
        self._arena_bytes = self.arena.numel() * self.arena.element_size()

    def run(self, stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        L.call("ktb_pack", self.dev, self._ptrs, self._nb, self._n, self.arena.data_ptr(), self._arena_bytes,
               self._offs, 0, _stream(self.dev, stream))
        return self.arena

    def run_unpack(self, stream: Optional[torch.cuda.Stream] = None):
        L.call("ktb_unpack", self.dev, self.arena.data_ptr(), self._offs, self._nb, self._n, self._ptrs,
               _stream(self.dev, stream))
        return self.tensors


class BatchPlan:
    """n independent small calls out_i = op(x_i) with prebuilt descriptor arrays."""

    def __init__(self, xs: Sequence[torch.Tensor], outs: Sequence[torch.Tensor], op: str, alpha=1.0, beta=0.0):
        self.dev = _check_dev_tensor(xs[0], "xs[0]")
        ensure_init({self.dev})
        self.xs, self.outs = list(xs), list(outs)
        self._src = L.arr(ctypes.c_void_p, [t.data_ptr() for t in xs])
        self._dst = L.arr(ctypes.c_void_p, [t.data_ptr() for t in outs])
        self._n_elems = L.arr(ctypes.c_size_t, [t.numel() for t in xs])
        self._args = (OPS[op], dtype_code(xs[0].dtype), float(alpha), float(beta))

    def run(self, stream: Optional[torch.cuda.Stream] = None):
        op, dt, a, b = self._args
        L.call("ktb_map_batch", self.dev, op, dt, self._src, self._dst, self._n_elems, len(self.xs), a, b,
               _stream(self.dev, stream))
        return self.outs


def unpack(
    arena: torch.Tensor,
    offsets: Sequence[int],
    outs: Sequence[torch.Tensor],
    stream: Optional[torch.cuda.Stream] = None,
) -> Sequence[torch.Tensor]:
    """Scatter arena segments back into the destination tensors `outs` (same device as arena)."""
    if not outs:
        return outs
    dev = _check_dev_tensor(arena, "arena")
    ensure_init({dev})
    nbytes = [t.numel() * t.element_size() for t in outs]
    for i, t in enumerate(outs):
        _check_dev_tensor(t, f"outs[{i}]")
    L.call(
        "ktb_unpack", dev, arena.data_ptr(), L.arr(ctypes.c_size_t, list(offsets)), L.arr(ctypes.c_size_t, nbytes),
        len(outs), L.arr(ctypes.c_void_p, [t.data_ptr() for t in outs]), _stream(dev, stream),
    )
    return outs


def arena_views(arena: torch.Tensor, offsets: Sequence[int], specs: Sequence[Tuple[torch.dtype, Tuple[int, ...]]]):
    """Zero-copy typed views of packed segments (offsets are 256-byte aligned)."""
    flat = arena.view(torch.uint8).reshape(-1)
    views = []
    for off, (dtype, shape) in zip(offsets, specs):
        n = 1
        for s in shape:
            n *= s
        nb = n * torch.empty((), dtype=dtype).element_size()
        views.append(flat[off : off + nb].view(dtype).reshape(shape))
    return views


def map_batch(
    xs: Sequence[torch.Tensor],
    op: str = "identity",
    alpha: float = 1.0,
    beta: float = 0.0,
    outs: Optional[Sequence[torch.Tensor]] = None,
    stream: Optional[torch.cuda.Stream] = None,
    device: Optional[int] = None,
) -> Sequence[torch.Tensor]:
    """n independent small calls out_i = op(x_i) coalesced into one segmented launch (on `device`,
    default xs[0]'s; sources/destinations may be peer-mapped)."""
    if not xs:
        return []
    dev = _check_dev_tensor(xs[0], "xs[0]") if device is None else int(device)
    ensure_init({dev})
    dt = xs[0].dtype
    for i, t in enumerate(xs):
        _check_dev_tensor(t, f"xs[{i}]")
        if t.dtype != dt:
            raise ValueError("map_batch needs one dtype per batch")
    if outs is None:
        outs = [torch.empty_like(t) for t in xs]
    L.call(
        "ktb_map_batch", dev, OPS[op], dtype_code(dt), L.arr(ctypes.c_void_p, [t.data_ptr() for t in xs]),
        L.arr(ctypes.c_void_p, [t.data_ptr() for t in outs]), L.arr(ctypes.c_size_t, [t.numel() for t in xs]),
        len(xs), float(alpha), float(beta), _stream(dev, stream),
    )
    return outs


# ---- multi-GPU ---------------------------------------------------------------------------------------
def broadcast(src: torch.Tensor, dsts: Sequence[torch.Tensor], stream: Optional[torch.cuda.Stream] = None):
    """One kernel on src's device reads src once and peer-stores it to every dst."""
    root = _check_dev_tensor(src, "src")
    devs = {root}
    nbytes = src.numel() * src.element_size()
    for i, d in enumerate(dsts):
        devs.add(_check_dev_tensor(d, f"dsts[{i}]"))
        if d.numel() * d.element_size() < nbytes:
            raise ValueError(f"dsts[{i}] is smaller than src")
    ensure_init(devs)
    L.call(
        "ktb_broadcast", root, src.data_ptr(), L.arr(ctypes.c_void_p, [d.data_ptr() for d in dsts]), len(dsts),
        nbytes, _stream(root, stream),
    )
    return dsts


def _scatter_devices(x_root: torch.Tensor, devices: Sequence[int], root_rank: int) -> List[int]:
    """The ranks' devices of a scatter form, registered, with devices[root_rank] checked to hold x_root."""
    root = _check_dev_tensor(x_root, "x_root")
    devs = [int(d) for d in devices]
    if devs[root_rank] != root:
        raise ValueError(f"x_root lives on cuda:{root} but devices[{root_rank}] is {devs[root_rank]}")
    ensure_init(set(devs))
    return devs


def scatter_map_gather(
    x_root: torch.Tensor,
    op: str,
    alpha: float = 1.0,
    beta: float = 0.0,
    devices: Sequence[int] = (0,),
    out_root: Optional[torch.Tensor] = None,
    root_rank: int = 0,
    variant: int = L.VARIANT_AUTO,
    granule: Optional[int] = None,
) -> torch.Tensor:
    """Fused scatter → map → gather: rank r's kernel pulls shard r of x_root (`x.chunk(world)` along
    dim 0; `granule` = elements per row, default from x_root's shape) from the root GPU over NVLink,
    applies op, and pushes it into out_root."""
    devs = _scatter_devices(x_root, devices, root_rank)
    if out_root is None:
        out_root = torch.empty_like(x_root)
    streams = [current_stream_handle(d) for d in devs]
    L.call(
        "ktb_scatter_map_gather", OPS[op], dtype_code(x_root.dtype), x_root.data_ptr(), out_root.data_ptr(),
        x_root.numel(), int(granule or row_elems(x_root)), float(alpha), float(beta), len(devs), L.arr(ctypes.c_int, devs), root_rank, int(variant),
        L.arr(L.c_uintptr, streams),
    )
    return out_root


def scatter_map_reduce(
    x_root: torch.Tensor,
    op: str,
    alpha: float = 1.0,
    beta: float = 0.0,
    devices: Sequence[int] = (0,),
    root_rank: int = 0,
    granule: Optional[int] = None,
) -> Tuple[torch.Tensor, torch.Tensor]:
    """Gather-reduce variant. Returns (total[1], partials[n_ranks]) on the root GPU."""
    devs = _scatter_devices(x_root, devices, root_rank)
    adt = acc_dtype(x_root.dtype)
    partials = torch.zeros(len(devs), dtype=adt, device=x_root.device)
    total = torch.empty(1, dtype=adt, device=x_root.device)
    wss = [_workspace(d) for d in devs]
    streams = [int(torch.cuda.current_stream(d).cuda_stream) for d in devs]
    L.call(
        "ktb_scatter_map_reduce", OPS[op], dtype_code(x_root.dtype), x_root.data_ptr(), x_root.numel(),
        int(granule or row_elems(x_root)), float(alpha),
        float(beta), len(devs), L.arr(ctypes.c_int, devs), root_rank, partials.data_ptr(), total.data_ptr(),
        L.arr(ctypes.c_void_p, [w.data_ptr() for w in wss]), L.arr(L.c_uintptr, streams),
    )
    return total, partials


class Arena:
    """A library-owned device allocation (ktb_arena_alloc): IPC-exportable, viewable as a torch tensor."""

    def __init__(self, device: int, nbytes: int, zero: bool = False):
        ensure_init({device})
        self.device, self.nbytes = int(device), int(nbytes)
        p = ctypes.c_void_p()
        L.call("ktb_arena_alloc", self.device, self.nbytes, ctypes.byref(p))
        self.ptr = p.value
        self._owned = True
        if zero:
            self.tensor(torch.uint8).zero_()
            torch.cuda.synchronize(self.device)

    def tensor(self, dtype: torch.dtype = torch.uint8, numel: Optional[int] = None, offset: int = 0) -> torch.Tensor:
        es = torch.empty((), dtype=dtype).element_size()
        n = (self.nbytes - offset) // es if numel is None else int(numel)
        typestr = {torch.uint8: "|u1", torch.float32: "<f4", torch.int32: "<i4", torch.int64: "<i8",
                   torch.bfloat16: "<u2"}[dtype]
        holder = type("_CAI", (), {})()
        holder.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (self.ptr + offset, False),
                                           "version": 3}
        t = torch.as_tensor(holder, device=f"cuda:{self.device}")
        return t.view(torch.bfloat16) if dtype == torch.bfloat16 else t

    def export(self) -> bytes:
        h = (ctypes.c_ubyte * L.IPC_HANDLE_BYTES)()
        L.call("ktb_ipc_export", self.device, ctypes.c_void_p(self.ptr), h)
        return bytes(h)

    def free(self):
        if self._owned and self.ptr:
            L.call("ktb_arena_free", self.device, ctypes.c_void_p(self.ptr))
            self.ptr = 0


def ipc_open(device: int, handle: bytes) -> int:
    """Map another process's arena on `device`; returns the device pointer."""
    ensure_init({device})
    h = (ctypes.c_ubyte * L.IPC_HANDLE_BYTES).from_buffer_copy(handle)
    p = ctypes.c_void_p()
    L.call("ktb_ipc_open", int(device), h, ctypes.byref(p))
    return p.value


def ipc_close(device: int, ptr: int) -> None:
    """Unmap an arena opened with ipc_open (must happen before its owner frees it)."""
    L.call("ktb_ipc_close", int(device), ctypes.c_void_p(ptr))


class PushTimeout(RuntimeError):
    """An in-kernel flag wait of the push/push pipeline timed out (a rank's GPU stalled or died)."""


# Control-block fields the host reads or writes (KTB_CTRL_STATUS / KTB_CTRL_TIMEOUT_NS in csrc/ktb_common.cuh).
_CTRL_STATUS = 1032       # u32 sticky status word: nonzero once an in-kernel wait timed out
_CTRL_TIMEOUT_NS = 1040   # u64 spin limit of the in-kernel waits in ns, 0 = the 10 s default


class PushSession:
    """Push/push scatter → exec → gather driven by ONE controller process over distinct GPUs
    (ktb_push_*): the root's kernel pushes shard pieces into each rank's staging buffer, each rank's
    kernel waits in-kernel for its piece, maps it and pushes the result into the root's result
    buffer. No events between devices: flags in device memory order everything.

    `call()` is the element-wise form.  Other forms (the MLP's) put their own launches between the same steps:
    `begin()`, the root's own shard on the stream `fork()` returns, the scatter and the ranks' consumers, `finish()`."""

    def __init__(self, devices: Sequence[int], max_shard_bytes: int, n_chunks: int = 32):
        self.devices = [int(d) for d in devices]
        ensure_init(set(self.devices))
        self.root = self.devices[0]
        self.n_chunks = int(n_chunks)
        self.stride = (int(max_shard_bytes) + 255) // 256 * 256
        cb = L.load().ktb_push_control_bytes()
        self.ctrl = [torch.zeros(cb, dtype=torch.uint8, device=f"cuda:{d}") for d in self.devices]
        self.stage = [None if r == 0 else torch.empty(2 * self.stride, dtype=torch.uint8, device=f"cuda:{d}")
                      for r, d in enumerate(self.devices)]
        for d in set(self.devices):
            torch.cuda.synchronize(d)
        self.seq = 0
        # host mirror of every control block's sticky status word, refreshed by an async D2H copy behind each call:
        # a timed-out in-kernel wait is seen at the NEXT call without a host sync on the data path
        self._side = torch.cuda.Stream(self.root)       # the root's own shard runs beside the scatter, not behind it
        self._ev_fork, self._ev_join = torch.cuda.Event(), torch.cuda.Event()
        self._status_host = torch.zeros(len(self.devices), dtype=torch.int32).pin_memory()
        self._status_dev = [c[_CTRL_STATUS:_CTRL_STATUS + 4].view(torch.int32) for c in self.ctrl]
        self.stage_ptrs = L.arr(ctypes.c_void_p, [0 if s is None else s.data_ptr() for s in self.stage])
        self.ctrl_ptrs = L.arr(ctypes.c_void_p, [c.data_ptr() for c in self.ctrl])

    def begin(self) -> int:
        """Start a call: raise PushTimeout if an in-kernel wait of an earlier call timed out, else return the new seq."""
        if bool(self._status_host.any()):
            bad = [self.devices[i] for i in self._status_host.nonzero().flatten().tolist()]
            raise PushTimeout(f"push pipeline: an in-kernel wait timed out on cuda:{bad} during an earlier call")
        self.seq += 1
        return self.seq

    def fork(self) -> torch.cuda.Stream:
        """The side stream, ordered after the root's current stream, for the root's own shard; finish(joined=True)
        joins it.  Fork BEFORE the scatter launch and launch the shard before it: the other order lets the two grids
        interleave on the SMs and costs 0.3 ms at 1 GiB; shard-first costs the shard's own time (41 us for the map at
        N = 2, 256 MiB)."""
        with torch.cuda.device(self.root):
            self._ev_fork.record(torch.cuda.current_stream(self.root))
            self._side.wait_event(self._ev_fork)
        return self._side

    def finish(self, seq: int, joined: bool) -> None:
        """End call `seq` on the root's current stream: wait for every rank's results (ktb_push_wait), join the side
        stream if the call forked it, and queue each control block's status mirror behind the call on its device."""
        L.call("ktb_push_wait", self.root, self.ctrl[0].data_ptr(), len(self.devices), 0, seq,
               current_stream_handle(self.root))
        if joined:
            with torch.cuda.device(self.root):
                self._ev_join.record(self._side)
                torch.cuda.current_stream(self.root).wait_event(self._ev_join)
        for r, d in enumerate(self.devices):
            with torch.cuda.device(d):
                self._status_host[r:r + 1].copy_(self._status_dev[r], non_blocking=True)

    def call(self, x_root: torch.Tensor, out_root: torch.Tensor, op: str, alpha: float = 1.0, beta: float = 0.0):
        seq = self.begin()
        n, es = len(self.devices), x_root.element_size()
        gran = row_elems(x_root)
        rows = x_root.numel() // gran
        dt = dtype_code(x_root.dtype)
        b, e = shard_bounds(rows, n, 0)   # the root's own shard maps on the root's HBM
        own = e > b
        if own:
            side = self.fork()
            L.call("ktb_map", self.root, OPS[op], dt, x_root.data_ptr() + b * gran * es,
                   out_root.data_ptr() + b * gran * es, (e - b) * gran, float(alpha), float(beta), L.VARIANT_AUTO,
                   int(side.cuda_stream))
        L.call("ktb_push_scatter", self.root, x_root.data_ptr(), x_root.numel(), gran, dt, n, 0, self.stage_ptrs,
               self.stride, self.ctrl_ptrs, self.ctrl[0].data_ptr(), self.n_chunks, seq,
               current_stream_handle(self.root))
        for r in range(1, n):
            b, e = shard_bounds(rows, n, r)
            if (e - b) * gran * es > self.stride:
                raise ValueError("shard larger than the session's staging buffers")
            L.call("ktb_push_consume", self.devices[r], OPS[op], dt, self.stage[r].data_ptr(), self.stride,
                   out_root.data_ptr() + b * gran * es, (e - b) * gran, float(alpha), float(beta),
                   self.ctrl[r].data_ptr(), self.ctrl[0].data_ptr(), r, self.n_chunks, seq,
                   current_stream_handle(self.devices[r]))
        self.finish(seq, joined=own)
        return out_root

    def set_spin_timeout(self, seconds: float) -> None:
        """In-kernel flag waits give up after `seconds` (default 10 s) and raise the sticky status word."""
        ns = torch.tensor([int(seconds * 1e9)], dtype=torch.int64)
        for d, c in zip(self.devices, self.ctrl):
            c[_CTRL_TIMEOUT_NS:_CTRL_TIMEOUT_NS + 8].view(torch.int64).copy_(ns.to(f"cuda:{d}"))
            torch.cuda.synchronize(d)

    def check(self):
        for d, c in zip(self.devices, self.ctrl):
            st = ctypes.c_uint(0)
            L.call("ktb_push_status", d, c.data_ptr(), ctypes.byref(st))
            if st.value:
                raise PushTimeout(f"push pipeline: an in-kernel wait timed out on cuda:{d}")


# ---- NUMA-sharded pinned host tensors ------------------------------------------------------------------
class _PinnedPool:
    """Recycles ktb_host_alloc_sharded blocks (page-faulting + page-locking 256 MiB costs ~100 ms; a call must not).
    A block returns to the pool when the last tensor view of it dies (weakref.finalize on the exporting buffer)."""

    MAX_CACHED_BYTES = 8 << 30

    def __init__(self):
        self._free = {}
        self._cached = 0
        self._lock = threading.Lock()

    def take(self, key):
        with self._lock:
            lst = self._free.get(key)
            if lst:
                self._cached -= key[0]
                return lst.pop()
        return None

    def give(self, key, ptr):
        with self._lock:
            if self._cached + key[0] <= self.MAX_CACHED_BYTES:
                self._free.setdefault(key, []).append(ptr)
                self._cached += key[0]
                return
        try:
            L.call("ktb_host_free_sharded", ctypes.c_void_p(ptr))
        except Exception:  # noqa: BLE001 - interpreter shutdown / library already closed
            pass


_pinned_pool = _PinnedPool()
_PINNED_POOL_MIN_BYTES = 4 << 20


def pinned_empty(shape, dtype: torch.dtype, devices: Optional[Sequence[int]] = None) -> torch.Tensor:
    """Uninitialised pinned host tensor.  With `devices` (distinct GPU ids, rank order) and at least 4 MiB, the
    pages of `x.chunk(len(devices))[r]` sit on the NUMA node of devices[r] (ktb_host_alloc_sharded), so every GPU
    of a sharded host-resident call moves its shard over its own socket's memory controllers."""
    import weakref

    shape = tuple(int(s) for s in shape)
    numel = 1
    for d in shape:
        numel *= d
    es = torch.empty((), dtype=dtype).element_size()
    nbytes = numel * es
    devs = [int(d) for d in (devices or [])]
    if nbytes < _PINNED_POOL_MIN_BYTES or not devs:
        return torch.empty(shape, dtype=dtype, pin_memory=True)
    ensure_init(set(devs))
    if len(set(devs)) != len(devs) or len(devs) == 1:
        devs, part_end = devs[:1], [nbytes]
    else:
        rows = shape[0] if shape else 1
        gran = numel // max(rows, 1)
        part_end = [shard_bounds(rows, len(devs), r)[1] * gran * es for r in range(len(devs))]
    key = (nbytes, tuple(devs), tuple(part_end))
    ptr = _pinned_pool.take(key)
    if ptr is None:
        out = ctypes.c_void_p()
        L.call("ktb_host_alloc_sharded", nbytes, len(devs), L.arr(ctypes.c_size_t, part_end), L.arr(ctypes.c_int, devs),
               ctypes.byref(out))
        ptr = out.value
    buf = (ctypes.c_uint8 * nbytes).from_address(ptr)
    weakref.finalize(buf, _pinned_pool.give, key, ptr)
    return torch.frombuffer(buf, dtype=torch.uint8).view(dtype).reshape(shape)


def device_numa_node(device: int) -> int:
    ensure_init({device})
    return L.load().ktb_device_numa_node(int(device))


# ---- host-resident args ------------------------------------------------------------------------------
_stage_cache = {}
_host_locks = {}


def map_host(
    x_host: torch.Tensor,
    op: str = "identity",
    alpha: float = 1.0,
    beta: float = 0.0,
    out_host: Optional[torch.Tensor] = None,
    device: int = 0,
    chunk_bytes: int = 16 << 20,
) -> torch.Tensor:
    """out_host = op(x_host), both pinned host tensors; H2D, kernel and D2H of successive chunks overlap."""
    require_cuda()
    if x_host.is_cuda or not x_host.is_pinned():
        raise ValueError("x_host must be a pinned host tensor")
    if out_host is None:
        out_host = torch.empty_like(x_host).pin_memory()
    elif out_host.is_cuda or not out_host.is_pinned():
        raise ValueError("out_host must be a pinned host tensor")
    ensure_init({device})
    key = (device, chunk_bytes)
    # one host-path call at a time per device: the staging buffers and the library's three copy/exec
    # streams are per-device (the PCIe link serialises them anyway)
    with _init_lock:
        lock = _host_locks.setdefault(device, threading.Lock())
    with lock:
        st = _stage_cache.get(key)
        if st is None:
            st = (
                torch.empty(2 * chunk_bytes, dtype=torch.uint8, device=f"cuda:{device}"),
                torch.empty(2 * chunk_bytes, dtype=torch.uint8, device=f"cuda:{device}"),
            )
            _stage_cache[key] = st
        L.call(
            "ktb_map_host", device, OPS[op], dtype_code(x_host.dtype), x_host.data_ptr(), out_host.data_ptr(),
            x_host.numel(), float(alpha), float(beta), chunk_bytes, st[0].data_ptr(), st[1].data_ptr(),
        )
    return out_host


_multi_lock = threading.Lock()


def host_chunk_bytes(shard_bytes: int) -> int:
    """Chunk size of the host pipeline: ~8 chunks per shard, between 1 MiB and 8 MiB, 256-byte multiple."""
    c = max(1 << 20, min(8 << 20, shard_bytes // 8))
    return (c + 255) // 256 * 256


def map_host_multi(
    x_host: torch.Tensor,
    op: str,
    alpha: float = 1.0,
    beta: float = 0.0,
    out_host: Optional[torch.Tensor] = None,
    devices: Sequence[int] = (0,),
    chunk_bytes: Optional[int] = None,
) -> torch.Tensor:
    """Sharded host-resident call on distinct GPUs from ONE host thread (ktb_map_host_multi)."""
    require_cuda()
    if x_host.is_cuda or not x_host.is_pinned():
        raise ValueError("x_host must be a pinned host tensor")
    if out_host is None:
        out_host = torch.empty_like(x_host).pin_memory()
    devs = [int(d) for d in devices]
    ensure_init(set(devs))
    gran = row_elems(x_host)
    rows = x_host.numel() // gran
    shard_bytes = shard_bounds(rows, len(devs), 0)[1] * gran * x_host.element_size()
    cb = int(chunk_bytes or host_chunk_bytes(shard_bytes))
    with _multi_lock:
        stages = []
        for d in devs:
            key = (d, cb)
            st = _stage_cache.get(key)
            if st is None:
                st = (torch.empty(2 * cb, dtype=torch.uint8, device=f"cuda:{d}"),
                      torch.empty(2 * cb, dtype=torch.uint8, device=f"cuda:{d}"))
                torch.cuda.synchronize(d)
                _stage_cache[key] = st
            stages.append(st)
        L.call(
            "ktb_map_host_multi", OPS[op], dtype_code(x_host.dtype), x_host.data_ptr(), out_host.data_ptr(),
            x_host.numel(), gran, float(alpha), float(beta), len(devs), L.arr(ctypes.c_int, devs), cb,
            L.arr(ctypes.c_void_p, [s[0].data_ptr() for s in stages]),
            L.arr(ctypes.c_void_p, [s[1].data_ptr() for s in stages]),
        )
    return out_host


def set_tuning(key: int, value: int) -> None:
    L.call("ktb_set_tuning", key, value)
