"""The exact element-wise reference (tests/elementwise_ref.py) against its semantic definition, torch CPU eager `x * a` /
`x * a + b`, on every input generator and every scalar row; and the host-side scalar rules of the element-wise entries
(kubetorch_b200.device.ops.scalar_args, the call-argument check of the b200 backend).  No GPU needed."""
import math

import numpy as np
import pytest
import torch

import elementwise_ref as R
from kubetorch_b200.device import ops
from kubetorch_b200.mapped import MappedSpec
from oracle import cases


def _torch_op(x, op, a, b):
    if op == "identity":
        return x.clone()
    return x * a if op == "scale" else x * a + b


CASES = [(dt, op) for dt in R.DTYPES for op in R.ops_of(dt)]


@pytest.mark.parametrize("dtype,op", CASES, ids=[f"{str(d)[6:]}-{o}" for d, o in CASES])
def test_reference_equals_torch_cpu(dtype, op):
    """Bit for bit on every output torch does not make NaN, NaN exactly where torch does (torch's own NaN payloads
    depend on its code path), for every generator value and every row of the scalar table."""
    x_bits = R.inputs(dtype)
    x = R.to_torch(x_bits, dtype)
    assert np.array_equal(R.bits_of(x), x_bits)
    rows = R.scalar_rows(dtype, op)
    for a, b in rows:
        want = R.bits_of(_torch_op(x, op, a, b))
        got = R.reference(dtype, op, x_bits, a, b)
        bad = R.mismatches(dtype, op, got, want)
        assert bad.size == 0, (dtype, op, a, b, R.describe(dtype, x_bits, got, want, bad))
    assert len(rows) == {"identity": 1, "scale": 14 if dtype in R.FLOATS else 11,
                         "affine": 14 * 9 if dtype in R.FLOATS else 11 * 11}[op]


def test_generators_cover_their_edges():
    f = R.f32_set()
    assert f.dtype == np.uint32 and len(np.unique(f)) >= 2 * 256 * len(R.F32_MANTISSAS)
    v = f.view(np.float32)
    assert np.isinf(v).sum() == 2 and np.isnan(v).sum() >= 2 * (len(R.F32_MANTISSAS) + 1)
    assert ((f & 0x7F800000) == 0).sum() >= 2 * 9          # zeros and subnormals of both signs
    for pattern in (0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF800001, 0x80000000, 0x7F7FFFFF, 0x3F808000, 0x3F818000):
        assert pattern in f, hex(pattern)
    assert len(np.unique(R.all_16bit())) == 1 << 16 and len(np.unique(R.all_u8())) == 256
    for dt, lo in ((torch.int32, -2 ** 31), (torch.int64, -2 ** 63)):
        s = set(R.bits_of(R.to_torch(R.int_set(dt), dt).view(dt)).tolist())
        for v in (0, 1, -1, lo, -lo - 1, lo + 1, -lo - 2):
            assert v % (-2 * lo) in s, (dt, v)


def test_bf16_rounding_routine_equals_torch():
    u = np.concatenate([R.f32_set(), np.random.default_rng(1).integers(0, 1 << 32, 1 << 16, dtype=np.uint32)])
    got = R.bf16_rne(u)
    want = R.bits_of(R.to_torch(u, torch.float32).bfloat16())
    assert R.mismatches(torch.bfloat16, "scale", got, want).size == 0


# ---- the host-side scalar rules ---------------------------------------------------------------------------------------
def test_scalar_args_reduces_int32_scalars_exactly():
    for v in R.INT_SCALARS:
        a, b = ops.scalar_args(torch.int32, v, -v)
        assert a == (v + 2 ** 31) % 2 ** 32 - 2 ** 31 and b == (-v + 2 ** 31) % 2 ** 32 - 2 ** 31
    assert ops.scalar_args(torch.int32, 2 ** 53 + 1, 0) == (1.0, 0.0)      # rounding through a double gave 0


def test_scalar_args_refuses_int64_scalars_a_double_does_not_hold():
    for v in R.INT_SCALARS:
        if R.int64_exact(v):
            assert ops.scalar_args(torch.int64, v, v) == (float(v), float(v))
        else:
            with pytest.raises(TypeError, match="exactly representable"):
                ops.scalar_args(torch.int64, v, 0)
            with pytest.raises(TypeError, match="exactly representable"):
                ops.scalar_args(torch.int64, 1, v)
    assert R.int64_exact(-2 ** 63) and R.int64_exact(2 ** 53) and not R.int64_exact(2 ** 53 + 1)
    assert ops.scalar_args(torch.int64, 2 ** 64 + 3, 2.0) == (3.0, 2.0)   # reduced modulo 2^64 first
    with pytest.raises(TypeError, match="not an integer"):
        ops.scalar_args(torch.int64, 0.5, 0)
    with pytest.raises(TypeError, match="not an integer"):
        ops.scalar_args(torch.int32, 1, math.inf)


def test_scalar_args_keeps_float_scalars():
    assert ops.scalar_args(torch.float32, 2 ** 53 + 1, 0.1) == (float(2 ** 53 + 1), 0.1)
    assert ops.scalar_args(torch.bfloat16, 1e39, -0.0)[0] == 1e39
    assert math.isnan(ops.scalar_args(torch.float16, math.nan, 0)[0])


def test_lane_dtype_codes_follow_scalar_args():
    assert torch.int32 in ops.fast_dtype_codes(2 ** 53 + 1, -7) and torch.int64 not in ops.fast_dtype_codes(2 ** 53 + 1, -7)
    assert torch.int64 in ops.fast_dtype_codes(-2 ** 63, 2 ** 53)
    codes = ops.fast_dtype_codes(0.5, 0)
    assert torch.int32 not in codes and torch.int64 not in codes and torch.float32 in codes


def test_float_call_argument_on_an_integer_tensor_is_refused():
    """torch promotes `x_int * 2.0` to float32, which the integer kernels do not do: a Python float passed as a call
    argument is refused on an int32/int64 tensor, integral or not, before anything runs."""
    from kubetorch_b200.serving.b200_supervisor import B200Supervisor

    sup = B200Supervisor(devices=[0])
    for dtype in (torch.int32, torch.int64):
        x = torch.arange(6, dtype=dtype)
        for a, b in ((2.0, 1), (3, -1.0), (0.5, 0)):
            with pytest.raises(TypeError, match="not an integer"):
                sup._run_mapped(MappedSpec("affine", alpha="alpha", beta="beta"), cases.affine, [x, a, b], {}, [0])
        with pytest.raises(TypeError, match="not an integer"):
            sup._run_mapped(MappedSpec("scale", alpha="alpha"), cases.scale, [x, 2.0], {}, [0])
        with pytest.raises(TypeError, match="not an integer"):   # a declared constant that is not integral
            sup._run_mapped(MappedSpec("scale", alpha=0.5), cases.double, [x], {}, [0])
