"""ctypes binding of libktb200.so (include/ktb200.h) — the only way the package reaches the GPU.

There is no CPU fallback: if the library is missing or a call fails, this raises.  The binding
is what a kubetorch maintainer would add behind the supervisor seam
(kt/serving/supervisor_factory.py:11-58); see INTEGRATION.md.
"""
from __future__ import annotations

import ctypes
import os
import threading
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_size_t, c_void_p

_LIB_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "lib", "libktb200.so")

# enums (include/ktb200.h)
OP_IDENTITY, OP_SCALE, OP_AFFINE = 0, 1, 2
U8, F32, BF16, I32, I64, F16 = 0, 1, 2, 3, 4, 5
VARIANT_AUTO, VARIANT_VEC, VARIANT_TMA, VARIANT_SCALAR = 0, 1, 2, 3
OK, ERR_CUDA, ERR_ARG, ERR_STATE, ERR_UNSUPPORTED = 0, -1, -2, -3, -4
PACK_ALIGN = 256
IPC_HANDLE_BYTES = 64

c_uintptr = ctypes.c_size_t  # uintptr_t


class KtbError(RuntimeError):
    """A libktb200 call failed. ``status`` is the ktb_status code."""

    def __init__(self, status: int, message: str):
        super().__init__(f"libktb200 error {status}: {message}")
        self.status = status


class KtbLibraryMissing(ImportError):
    pass


_SIGNATURES = {
    "ktb_init": (c_int, [c_int, POINTER(c_int)]),
    "ktb_shutdown": (c_int, []),
    "ktb_last_error": (c_char_p, []),
    "ktb_version": (c_int, []),
    "ktb_sm_count": (c_int, [c_int]),
    "ktb_peer_enabled": (c_int, [c_int, c_int]),
    "ktb_arena_alloc": (c_int, [c_int, c_size_t, POINTER(c_void_p)]),
    "ktb_arena_free": (c_int, [c_int, c_void_p]),
    "ktb_host_alloc": (c_int, [c_size_t, POINTER(c_void_p)]),
    "ktb_host_free": (c_int, [c_void_p]),
    "ktb_device_numa_node": (c_int, [c_int]),
    "ktb_host_alloc_sharded": (c_int, [c_size_t, c_int, POINTER(c_size_t), POINTER(c_int), POINTER(c_void_p)]),
    "ktb_host_free_sharded": (c_int, [c_void_p]),
    "ktb_ipc_export": (c_int, [c_int, c_void_p, c_void_p]),
    "ktb_ipc_open": (c_int, [c_int, c_void_p, POINTER(c_void_p)]),
    "ktb_ipc_close": (c_int, [c_int, c_void_p]),
    "ktb_shard_bounds": (c_int, [c_size_t, c_int, c_int, POINTER(c_size_t), POINTER(c_size_t)]),
    "ktb_map": (c_int, [c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_double, c_double, c_int, c_uintptr]),
    "ktb_map_identity_u8": (c_int, [c_int, c_void_p, c_void_p, c_size_t, c_uintptr]),
    "ktb_map_scale_f32": (c_int, [c_int, c_void_p, c_void_p, c_size_t, c_float, c_uintptr]),
    "ktb_map_affine_f32": (c_int, [c_int, c_void_p, c_void_p, c_size_t, c_float, c_float, c_uintptr]),
    "ktb_map_scale_bf16": (c_int, [c_int, c_void_p, c_void_p, c_size_t, c_float, c_uintptr]),
    "ktb_map_affine_bf16": (c_int, [c_int, c_void_p, c_void_p, c_size_t, c_float, c_float, c_uintptr]),
    "ktb_reduce_workspace_bytes": (c_size_t, []),
    "ktb_map_reduce_sum": (c_int, [c_int, c_int, c_int, c_void_p, c_size_t, c_double, c_double, c_void_p, c_void_p, c_uintptr]),
    "ktb_reduce_partials": (c_int, [c_int, c_int, c_void_p, c_int, c_void_p, c_uintptr]),
    "ktb_pack_layout": (c_int, [POINTER(c_size_t), c_int, POINTER(c_size_t), POINTER(c_size_t)]),
    "ktb_pack": (c_int, [c_int, POINTER(c_void_p), POINTER(c_size_t), c_int, c_void_p, c_size_t, POINTER(c_size_t), c_int, c_uintptr]),
    "ktb_unpack": (c_int, [c_int, c_void_p, POINTER(c_size_t), POINTER(c_size_t), c_int, POINTER(c_void_p), c_uintptr]),
    "ktb_map_batch": (c_int, [c_int, c_int, c_int, POINTER(c_void_p), POINTER(c_void_p), POINTER(c_size_t), c_int, c_double, c_double, c_uintptr]),
    "ktb_broadcast": (c_int, [c_int, c_void_p, POINTER(c_void_p), c_int, c_size_t, c_uintptr]),
    "ktb_scatter_map_gather": (c_int, [c_int, c_int, c_void_p, c_void_p, c_size_t, c_size_t, c_double, c_double, c_int, POINTER(c_int), c_int, c_int, POINTER(c_uintptr)]),
    "ktb_scatter_map_reduce": (c_int, [c_int, c_int, c_void_p, c_size_t, c_size_t, c_double, c_double, c_int, POINTER(c_int), c_int, c_void_p, c_void_p, POINTER(c_void_p), POINTER(c_uintptr)]),
    "ktb_push_control_bytes": (c_size_t, []),
    "ktb_push_scatter": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int, POINTER(c_void_p), c_size_t,
                                 POINTER(c_void_p), c_void_p, c_int, ctypes.c_ulonglong, c_uintptr]),
    "ktb_push_scatter_chunked": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int, POINTER(c_void_p),
                                         c_size_t, POINTER(c_void_p), c_void_p, c_size_t, c_int, ctypes.c_ulonglong,
                                         c_uintptr]),
    "ktb_push_scatter_ce": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int, POINTER(c_int), POINTER(c_void_p),
                                    c_size_t, POINTER(c_void_p), c_void_p, c_size_t, ctypes.c_ulonglong, c_uintptr]),
    "ktb_push_consume": (c_int, [c_int, c_int, c_int, c_void_p, c_size_t, c_void_p, c_size_t, c_double, c_double,
                                 c_void_p, c_void_p, c_int, c_int, ctypes.c_ulonglong, c_uintptr]),
    "ktb_push_wait": (c_int, [c_int, c_void_p, c_int, c_int, ctypes.c_ulonglong, c_uintptr]),
    "ktb_push_status": (c_int, [c_int, c_void_p, POINTER(ctypes.c_uint)]),
    "ktb_map_host": (c_int, [c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_double, c_double, c_size_t, c_void_p, c_void_p]),
    "ktb_map_host_multi": (c_int, [c_int, c_int, c_void_p, c_void_p, c_size_t, c_size_t, c_double, c_double, c_int,
                                   POINTER(c_int), c_size_t, POINTER(c_void_p), POINTER(c_void_p)]),
    "ktb_mlp_scratch_bytes": (c_size_t, [c_size_t, c_int]),
    "ktb_mlp_bf16": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uintptr]),
    "ktb_mlp_stage_bytes": (c_size_t, [c_size_t, c_int]),
    "ktb_mlp_bf16_staged": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_uintptr]),
    "ktb_mlp_bf16_pushed": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_size_t, ctypes.c_ulonglong,
                                    c_uintptr]),
    "ktb_mlp_bf16_policy": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uintptr]),
    "ktb_mlp_bf16_policy_pushed": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_int, c_size_t, ctypes.c_ulonglong, c_uintptr]),
    "ktb_mlp_bf16_policy_sample": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_uint64, ctypes.c_uint64,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_uintptr]),
    "ktb_mlp_bf16_policy_sample_pushed": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int, c_void_p,
                                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_uint64,
                                                  ctypes.c_uint64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                  c_int, c_size_t, ctypes.c_ulonglong, c_uintptr]),
    "ktb_mlp_bf16_policy_gaussian": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p,
                                             c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_uint64,
                                             ctypes.c_uint64, c_void_p, c_void_p, c_void_p, c_void_p, c_uintptr]),
    "ktb_mlp_bf16_policy_gaussian_pushed": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int,
                                                    c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                    c_void_p, ctypes.c_uint64, ctypes.c_uint64, c_void_p, c_void_p,
                                                    c_void_p, c_void_p, c_void_p, c_int, c_size_t, ctypes.c_ulonglong,
                                                    c_uintptr]),
    # experiment knob, not in the stable header
    "ktb_set_tuning": (c_int, [c_int, c_int]),
}

_lib = None
_lock = threading.Lock()


def lib_path() -> str:
    return _LIB_PATH


def map_kernel_source_sha256() -> str:
    """sha256 of the SOURCE of the dominant kernel (the "VEC" section of csrc/ktb_map.cu = map_vec_kernel and its
    load/store helpers, plus the per-element op math and the streaming PTX helpers of ktb_common.cuh).  Stamped into
    profiles/roofline_traffic.json at ncu-capture time; bench.py reports `traffic: null` ("stale") when it differs."""
    import hashlib

    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "csrc")

    def section(name, start, stop):
        text = open(os.path.join(csrc, name)).read()
        a = text.index(start)
        return text[a:text.index(stop, a)]

    h = hashlib.sha256()
    h.update(section("ktb_map.cu", "// ---- VEC ---", "// ---- SCALAR ---").encode())
    h.update(section("ktb_common.cuh", "// ---- per-element op math", "// ---- PTX: mbarrier").encode())
    return h.hexdigest()


def load() -> ctypes.CDLL:
    """Load libktb200.so (once) and declare every prototype. Raises KtbLibraryMissing if absent."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(_LIB_PATH):
            raise KtbLibraryMissing(
                f"{_LIB_PATH} not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "or `make -C kubetorch_b200/csrc`. kubetorch_b200 has no CPU fallback for the device path."
            )
        lib = ctypes.CDLL(_LIB_PATH, mode=ctypes.RTLD_GLOBAL)
        for name, (restype, argtypes) in _SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
        return lib


def last_error() -> str:
    msg = load().ktb_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def check(status: int) -> int:
    if status < 0:
        raise KtbError(status, last_error())
    return status


def call(name: str, *args):
    """Call a status-returning entry point and raise KtbError on failure."""
    return check(getattr(load(), name)(*args))


def arr(ctype, values):
    return (ctype * len(values))(*values)
