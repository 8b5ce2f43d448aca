"""ctypes binding of libktb200.so (include/ktb200.h) — the only way the package reaches the GPU.

There is no CPU fallback: if the library is missing or a call fails, this raises.  The binding
is what a kubetorch maintainer would add behind the supervisor seam
(kt/serving/supervisor_factory.py:11-58); see INTEGRATION.md.
"""
from __future__ import annotations

import ctypes
import os
import re
import threading
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_size_t, c_void_p

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB_PATH = os.path.join(_PKG, "lib", "libktb200.so")
_HEADER = os.path.join(os.path.dirname(_PKG), "include", "ktb200.h")   # the Makefile builds the library from it

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


# ctypes of the C types the header's entries take.  Scalars pass by value.  A pointer to a buffer type is a device or
# raw buffer, passed as a data_ptr() int; a pointer to a host scalar is a host array or an out-parameter.
_SCALARS = {"int": c_int, "size_t": c_size_t, "uintptr_t": c_uintptr, "float": c_float, "double": c_double,
            "uint64_t": ctypes.c_uint64, "unsigned long long": ctypes.c_ulonglong}
_HOST_SCALARS = {"int": c_int, "int32_t": ctypes.c_int32, "size_t": c_size_t, "uintptr_t": c_uintptr,
                 "unsigned int": ctypes.c_uint}
_BUFFERS = ("void", "float", "int64_t", "uint8_t", "unsigned char")
_RESTYPES = {"int": c_int, "size_t": c_size_t, "const char*": c_char_p}


def _argtype(param: str):
    """ctypes class of one parameter declaration (`const` ignored, `T x[N]` read as `T* x`), None if it has no rule."""
    base = " ".join(re.sub(r"\bconst\b|\[\w*\]", " ", param).replace("*", " ").split()[:-1])   # the name dropped
    stars = param.count("*") + param.count("[")
    if stars == 0:
        return _SCALARS.get(base)
    if stars == 1 and base in _BUFFERS:
        return c_void_p
    if stars == 1 and base in _HOST_SCALARS:
        return POINTER(_HOST_SCALARS[base])
    if stars == 2 and base == "void":
        return POINTER(c_void_p)
    return None


def _parse_header(text: str) -> dict:
    """name -> (restype, argtypes) of every `ktb_*(...)` declaration in the text of include/ktb200.h.  A type without
    a rule above raises: a guessed ctypes class would shift every later argument without an error."""
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    signatures = {}
    for ret, name, params in re.findall(r"^(\w[\w ]*\**)\s*\b(ktb_\w+)\s*\(([^)]*)\)\s*;", text, flags=re.M):
        params = [" ".join(p.split()) for p in params.split(",")] if params.strip() not in ("", "void") else []
        restype, argtypes = _RESTYPES.get(" ".join(ret.split())), [_argtype(p) for p in params]
        if restype is None:
            raise TypeError(f"ktb200.h: {name}: no ctypes rule for the return type {ret.strip()!r}")
        for p, t in zip(params, argtypes):
            if t is None:
                raise TypeError(f"ktb200.h: {name}: no ctypes rule for the parameter {p!r}")
        signatures[name] = (restype, argtypes)
    return signatures


with open(_HEADER) as _f:
    _SIGNATURES = _parse_header(_f.read())
_SIGNATURES["ktb_set_tuning"] = (c_int, [c_int, c_int])   # experiment knob, not in the stable header

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
