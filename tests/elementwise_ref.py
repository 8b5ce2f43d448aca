"""An exact, torch-independent restatement of the element-wise op math (DESIGN.md §1) on the bit patterns of the
inputs, with the input generators and scalar tables the element-wise suites share (tests/test_elementwise_ref_cpu.py
pins it to torch CPU; tests/test_gpu_elementwise_exact.py checks the kernels against it).  Not a test module.

    f32   y = (x * a) + b in float32, two separately rounded IEEE operations (no FMA); a, b = float32(python value)
    bf16  x widened exactly to f32, the product rounded to bf16 (RNE), beta rounded to bf16, the f32 sum rounded again
    f16   the same through float16
    i32 / i64  arithmetic modulo 2^32 / 2^64 with the exact scalars (Python ints reduced modulo 2^bits)
    u8 and every identity   a copy of the bytes
"""
import math

import numpy as np
import torch

DTYPES = (torch.uint8, torch.float32, torch.bfloat16, torch.float16, torch.int32, torch.int64)
FLOATS = (torch.float32, torch.bfloat16, torch.float16)
INTS = (torch.int32, torch.int64)
UINT = {torch.uint8: np.uint8, torch.float32: np.uint32, torch.bfloat16: np.uint16, torch.float16: np.uint16,
        torch.int32: np.uint32, torch.int64: np.uint64}
_NP_SIGNED = {np.uint8: np.uint8, np.uint16: np.int16, np.uint32: np.int32, np.uint64: np.int64}
_TORCH_SIGNED = {np.uint8: torch.uint8, np.uint16: torch.int16, np.uint32: torch.int32, np.uint64: torch.int64}
ES = {dt: np.dtype(u).itemsize for dt, u in UINT.items()}


def ops_of(dtype):
    """The ops the kernels take for `dtype` (u8 is identity only)."""
    return ("identity",) if dtype == torch.uint8 else ("identity", "scale", "affine")


# ---- scalar tables ----------------------------------------------------------------------------------------------------
FLOAT_ALPHAS = (1.0, -1.0, 2.0, 0.5, 1.7, 0.1, 0.0, -0.0, 3e38, 1e39, math.inf, -math.inf, math.nan, 1e-45)
FLOAT_BETAS = (0.0, -0.0, 0.25, -0.3, 1 + 2 ** -8, 65520.0, 1e-8, math.inf, math.nan)
INT_SCALARS = (0, 1, -1, 65537, 2 ** 31 - 1, -2 ** 31, 2 ** 32 + 3, 2 ** 53 + 1, 2 ** 62 + 7, 2 ** 63 - 1, -2 ** 63)


def scalar_rows(dtype, op):
    """Every (alpha, beta) of the tables for (dtype, op): each alpha for scale, alpha x beta for affine."""
    if op == "identity":
        return [(1, 0)]
    alphas, betas = (FLOAT_ALPHAS, FLOAT_BETAS) if dtype in FLOATS else (INT_SCALARS, INT_SCALARS)
    if op == "scale":
        return [(a, 0) for a in alphas]
    return [(a, b) for a in alphas for b in betas]


def int64_exact(v):
    """Whether an int64 scalar reaches the kernels exactly (its signed 64-bit reduction is a double)."""
    r = (int(v) + 2 ** 63) % 2 ** 64 - 2 ** 63
    return int(float(r)) == r


# ---- input generators (uint bit patterns) -----------------------------------------------------------------------------
def all_u8():
    return np.arange(256, dtype=np.uint8)


def all_16bit():
    """Every one of the 65 536 bf16 / f16 bit patterns."""
    return np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)


F32_MANTISSAS = (0, 1, 0x400000, 0x7FFFFF, 0x8000, 0x7FFF, 0x18000)   # 0x8000 / 0x18000: bf16 rounding ties


def f32_set(seed=0):
    """Every (sign, exponent) with the mantissas above and two random ones (zeros, subnormals, the bf16 tie cases, the
    largest finite values, ±inf, quiet and signalling NaNs of both signs)."""
    rng = np.random.default_rng(seed)
    sign_exp = (np.arange(512, dtype=np.uint32) << 23)                  # sign bit = bit 8 of the index << 23 = bit 31
    mant = np.array(F32_MANTISSAS, dtype=np.uint32)
    fixed = (sign_exp[:, None] | mant[None, :]).reshape(-1)
    rand = (sign_exp[:, None] | rng.integers(1, 1 << 23, (512, 2), dtype=np.uint32)).reshape(-1)
    nans = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF800001, 0x7FA00000, 0xFFC00001], dtype=np.uint32)
    return np.concatenate([fixed, rand, nans])


def int_set(dtype, seed=0, n_random=256):
    """0, ±1, MIN, MAX, MIN+1, MAX-1 and random values of int32 / int64, as uint bit patterns."""
    bits = 8 * ES[dtype]
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    special = [0, 1, -1, lo, hi, lo + 1, hi - 1]
    rng = np.random.default_rng(seed)
    rand = rng.integers(lo, hi, n_random, dtype=np.int64 if bits == 64 else np.int32, endpoint=True).tolist()
    return np.array([v % (1 << bits) for v in special + rand], dtype=UINT[dtype])


def inputs(dtype):
    """The generator of `dtype`: bit patterns as a numpy uint array."""
    if dtype == torch.uint8:
        return all_u8()
    if dtype in (torch.bfloat16, torch.float16):
        return all_16bit()
    if dtype == torch.float32:
        return f32_set()
    return int_set(dtype)


# ---- torch <-> bit patterns -------------------------------------------------------------------------------------------
def to_torch(u, dtype):
    """numpy uint bit patterns -> a CPU tensor of `dtype` with exactly those bits."""
    u = np.ascontiguousarray(u, dtype=UINT[dtype])
    return torch.from_numpy(u.view(_NP_SIGNED[u.dtype.type])).view(dtype)


def bits_of(t):
    """The bit patterns of a tensor as a numpy uint array (a copy on the host)."""
    t = t.detach().contiguous().cpu().reshape(-1)
    u = UINT[t.dtype]
    return t.view(_TORCH_SIGNED[u]).numpy().view(u)


# ---- the op math ------------------------------------------------------------------------------------------------------
def _f32(v):
    with np.errstate(over="ignore"):
        return np.float32(v)


def bf16_rne(u32):
    """float32 bit patterns -> bf16 bit patterns, round to nearest even; a NaN stays a NaN (quiet, sign kept)."""
    u = u32.astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    nan = (u32 & 0x7FFFFFFF) > 0x7F800000
    r[nan] = ((u32[nan] >> 16) | 0x40).astype(np.uint16)
    return r


def _widen_bf16(u16):
    return (u16.astype(np.uint32) << 16).view(np.float32)


def reference(dtype, op, x, alpha=1, beta=0):
    """op(x) of the bit patterns `x` (numpy uint array of UINT[dtype]) as bit patterns."""
    x = np.ascontiguousarray(x, dtype=UINT[dtype])
    if op == "identity" or dtype == torch.uint8:
        return x.copy()
    affine = op == "affine"
    if dtype in INTS:
        bits = 8 * ES[dtype]
        u = UINT[dtype]
        a, b = u(int(alpha) % (1 << bits)), u(int(beta) % (1 << bits))
        with np.errstate(over="ignore"):
            y = x * a
            return (y + b) if affine else y
    a = _f32(alpha)
    with np.errstate(all="ignore"):
        if dtype == torch.float32:
            y = x.view(np.float32) * a
            if affine:
                y = y + _f32(beta)
            return y.view(np.uint32)
        if dtype == torch.bfloat16:
            y = bf16_rne((_widen_bf16(x) * a).view(np.uint32))
            if affine:
                b = _widen_bf16(bf16_rne(np.array([_f32(beta)]).view(np.uint32)))[0]
                y = bf16_rne((_widen_bf16(y) + b).view(np.uint32))
            return y
        y = (x.view(np.float16).astype(np.float32) * a).astype(np.float16)
        if affine:
            b = np.float32(_f32(beta).astype(np.float16))
            y = (y.astype(np.float32) + b).astype(np.float16)
        return y.view(np.uint16)


def is_nan(dtype, u):
    """NaN mask of bit patterns (all False for the non-float dtypes)."""
    if dtype == torch.float32:
        return (u & 0x7FFFFFFF) > 0x7F800000
    if dtype == torch.bfloat16:
        return (u & 0x7FFF) > 0x7F80
    if dtype == torch.float16:
        return (u & 0x7FFF) > 0x7C00
    return np.zeros(u.shape, dtype=bool)


def mismatches(dtype, op, got, want):
    """Indices where `got` breaks the comparison rule against `want` (both uint bit patterns): a scale/affine result of
    a float dtype equals `want` bit for bit wherever `want` is not NaN and is NaN exactly where `want` is NaN (the NaN
    payload is unspecified); identity and every u8 / integer result are byte-exact."""
    got, want = np.asarray(got).reshape(-1), np.asarray(want).reshape(-1)
    assert got.shape == want.shape, (got.shape, want.shape)
    if op == "identity" or dtype not in FLOATS:
        return np.nonzero(got != want)[0]
    nw, ng = is_nan(dtype, want), is_nan(dtype, got)
    return np.nonzero((nw != ng) | (~nw & (got != want)))[0]


def describe(dtype, x, got, want, idx, k=6):
    """The first k mismatches as (index, input, got, want) hex strings."""
    return [(int(i), hex(int(x[i % len(x)])) if x is not None else None, hex(int(got[i])), hex(int(want[i])))
            for i in idx[:k]]
