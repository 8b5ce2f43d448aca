"""The reference and the constructed inputs of the MLP IEEE suites (tests/test_gpu_mlp_ieee.py on the device,
tests/test_mlp_ieee_cpu.py pinning this module on CPU).  Not a test module.

The trunk's reference is the definition of tests/policy_cases.py evaluated in torch on CPU: fp32 F.linear over the
bf16 values, torch.relu (which keeps NaN), one bf16 rounding per layer.  Whether an output is NaN, +inf, -inf or finite
does not depend on the order of the sum unless a finite partial sum overflows, and the overflow cases below are built
from exact single products, so the classes are compared exactly and only finite values get a tolerance."""
import torch
import torch.nn.functional as F

D_IN, D_HIDDEN, D_OUT = 64, 256, 64      # the constructed cases: one K block, one N tile per layer

BF16_MAX = (2 - 2 ** -7) * 2.0 ** 127
TIE = (2 - 2 ** -8) * 2.0 ** 127         # halfway between BF16_MAX and 2^128: round-to-nearest-even gives +inf
FP32_ULP_AT_TIE = 2.0 ** 104
TIE_A, TIE_B = 146 * 2.0 ** 56, 224 * 2.0 ** 57   # 146 · 224 = 511 · 64: a bf16 pair whose product is TIE
BIG = 1.5 * 2.0 ** 64                    # BIG · 2^63 = 1.5 · 2^127 > FLT_MAX / 2: two such products overflow fp32
SUB = 2.0 ** -133                        # the smallest bf16 subnormal; m · SUB for m < 128 are all of them

FINITE, NAN, POS_INF, NEG_INF = 0, 1, 2, 3


def trunk(obs, w1, b1, w2, b2, w3, b3):
    """bf16 logits of the policy  Linear → ReLU → Linear → ReLU → Linear  in torch on CPU (any bias may be None)."""
    f = lambda t: None if t is None else t.cpu().float()   # noqa: E731
    h = torch.relu(F.linear(f(obs), f(w1), f(b1))).bfloat16()
    h = torch.relu(F.linear(h.float(), f(w2), f(b2))).bfloat16()
    return F.linear(h.float(), f(w3), f(b3)).bfloat16()


def trunk64(obs, w1, b1, w2, b2, w3, b3):
    """The same network restated in fp64: each layer's exact sum (fp64 is exact for the constructed cases), rounded to
    fp32 (where an overflowing sum becomes ±inf) and then to bf16, with ReLU as `x < 0 ? 0 : x`."""
    d = lambda t: None if t is None else t.cpu().double()   # noqa: E731

    def layer(x, w, b, relu):
        y = x @ w.t() + (0 if b is None else b)
        y = y.float()
        if relu:
            y = torch.where(y < 0, torch.zeros_like(y), y)
        return y.bfloat16().double()

    h = layer(d(obs), d(w1), d(b1), True)
    h = layer(h, d(w2), d(b2), True)
    return layer(h, d(w3), d(b3), False).bfloat16()


def classes(t):
    """Each element's IEEE class: FINITE, NAN, POS_INF or NEG_INF (int8, the shape of t)."""
    t = t.float()
    c = torch.full(t.shape, FINITE, dtype=torch.int8, device=t.device)
    c[t.isnan()] = NAN
    c[t == float("inf")] = POS_INF
    c[t == float("-inf")] = NEG_INF
    return c


def assert_matches(got, want, what, rtol=0.0, atol=0.0):
    """got and want have the same class everywhere, and agree within rtol, atol on the elements finite in both (bit
    for bit with the defaults)."""
    got, want = got.cpu(), want.cpu()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    cg, cw = classes(got), classes(want)
    bad = cg != cw
    if bool(bad.any()):
        idx = bad.nonzero()[:6].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} elements of another class; (index, got, "
                             f"want): {[(i, float(got[tuple(i)]), float(want[tuple(i)])) for i in idx]}")
    fin = cw == FINITE
    torch.testing.assert_close(got[fin].float(), want[fin].float(), rtol=rtol, atol=atol, msg=lambda m: f"{what}: {m}")


def same_bits(got, want, what):
    """Bit for bit, with any NaN equal to any NaN."""
    got, want = got.cpu(), want.cpu()
    assert got.dtype == want.dtype and got.shape == want.shape, what
    if not got.is_floating_point():
        assert torch.equal(got, want), (what, int((got != want).sum()))
        return
    nan = want.isnan()
    assert torch.equal(got.isnan(), nan), (what, int((got.isnan() != nan).sum()))
    assert torch.equal(got[~nan], want[~nan]) and torch.equal(torch.signbit(got[~nan]), torch.signbit(want[~nan])), \
        (what, int((got[~nan] != want[~nan]).sum()))


def _bf16(t):
    b = t.bfloat16()
    assert torch.equal(b.double(), t), "a constructed value is not a bf16 value"
    return b


def _net(obs, w1, b1, w2, b2, w3, b3):
    return tuple(None if t is None else _bf16(t) for t in (obs, w1, b1, w2, b2, w3, b3))


def overflow_case(layer, M=256):
    """(obs, w1, b1, w2, b2, w3, b3) bias-free, built of exact products; row i of kind i % 4 puts in `layer` ("hidden":
    layer 1, unit 0 or 1; "head": logits 0 to 3, through a copying trunk):
      0: TIE_A · TIE_B = TIE, which rounds to +inf in bf16 (-inf in the negated head column)
      1: the same minus one fp32 ulp (a second product, -2^104): rounds to BF16_MAX
      2: two products of 1.5 · 2^127: the fp32 accumulator overflows to +inf (-inf negated)
      3: one such product: 1.5 · 2^127, finite.
    In "hidden" W2 and W3 have no zero (2^-8, W3's rows alternating in sign), so an infinite unit reaches every logit as
    +inf or -inf instead of turning into NaN (inf · 0) on the way."""
    z = lambda *s: torch.zeros(*s, dtype=torch.float64)   # noqa: E731
    obs, w1, w2, w3 = z(M, D_IN), z(D_HIDDEN, D_IN), z(D_HIDDEN, D_HIDDEN), z(D_OUT, D_HIDDEN)
    kind = torch.arange(M) % 4
    obs[kind <= 1, 0] = TIE_A
    obs[kind == 1, 1] = 2.0 ** 52
    obs[kind >= 2, 2] = BIG
    obs[kind == 2, 3] = BIG
    if layer == "hidden":
        w1[0, 0], w1[0, 1] = TIE_B, -2.0 ** 52
        w1[1, 2] = w1[1, 3] = 2.0 ** 63
        w2.fill_(2.0 ** -8)
        w3.fill_(2.0 ** -8)
        w3[1::2] = -2.0 ** -8
    else:
        w1[torch.arange(D_IN), torch.arange(D_IN)] = 1.0       # units 0..63 copy the (non-negative) observations
        w2 = torch.eye(D_HIDDEN, dtype=torch.float64)
        for s, j in ((1.0, 0), (-1.0, 1)):
            w3[j, 0], w3[j, 1] = s * TIE_B, -s * 2.0 ** 52
            w3[j + 2, 2] = w3[j + 2, 3] = s * 2.0 ** 63
    return _net(obs, w1, None, w2, None, w3, None)


def subnormal_case(bias, M=256):
    """(obs, w1, b1, w2, b2, w3, b3) whose exact results are known; rows differ in m = 1 + i % 127, so every bf16
    subnormal m · SUB takes part:
      unit 0 = obs[:, 4] · 2^100 = m · 2^-33: a subnormal observation times a large weight, a normal product
      unit 1 = 2^100 · w1[1, 5] with w1[1, 5] = 5 · SUB: a subnormal weight
      unit 2 = obs[:, 6] · 2^-66 = m · SUB with obs[:, 6] = m · 2^-67: normal inputs, a subnormal result
      units 3..10 (with `bias`) = 2^-125 + b1[u] = u' · SUB with b1[u] = -(256 - u') · SUB normal, u' = 3, 17, .., 127
    W2 is the identity (the subnormal hidden units are layer 2's inputs) and the head copies units 0..63, with logit
    63 = -unit 2, a negative subnormal without a ReLU after it."""
    z = lambda *s: torch.zeros(*s, dtype=torch.float64)   # noqa: E731
    obs, w1, w3 = z(M, D_IN), z(D_HIDDEN, D_IN), z(D_OUT, D_HIDDEN)
    m = (1 + torch.arange(M) % 127).double()
    obs[:, 4] = m * SUB
    obs[:, 5] = 2.0 ** 100
    obs[:, 6] = m * 2.0 ** -67
    obs[:, 7] = 2.0 ** -62
    w1[0, 4], w1[1, 5], w1[2, 6] = 2.0 ** 100, 5 * SUB, 2.0 ** -66
    b1 = None
    if bias:
        b1 = z(D_HIDDEN)
        for u, keep in zip(range(3, 11), (3, 17, 33, 64, 65, 100, 126, 127)):
            w1[u, 7] = 2.0 ** -63
            b1[u] = -(256 - keep) * SUB
    w3[torch.arange(D_OUT - 1), torch.arange(D_OUT - 1)] = 1.0
    w3[D_OUT - 1, 2] = -1.0
    return _net(obs, w1, b1, torch.eye(D_HIDDEN, dtype=torch.float64), None, w3, None)


def random_net(seed, d_in=256, d_hidden=1024, d_out=64, bias=True):
    """The rig's policy shape with random bf16 weights (σ 0.02) and biases (σ 0.1) on CPU."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale: (torch.randn(*s, generator=g) * scale).bfloat16()   # noqa: E731
    w1, w2, w3 = r(d_hidden, d_in, scale=0.02), r(d_hidden, d_hidden, scale=0.02), r(d_out, d_hidden, scale=0.02)
    b = (r(d_hidden, scale=0.1), r(d_hidden, scale=0.1), r(d_out, scale=0.1)) if bias else (None, None, None)
    return w1, b[0], w2, b[1], w3, b[2]


# Where a poisoned weight or bias goes: (tensor index in (w1, b1, w2, b2, w3, b3), the indices).  W1 columns 5 and 250
# sit in the first and the last 64-wide K block of d_in = 256; the rows and bias entries one in each 256-wide N tile.
TILE_UNITS = (17, 256 + 100, 512 + 201, 768 + 255)
POISON_SITES = {
    "w1_first_k_block": (0, [(u, 5) for u in (3, 700)]),
    "w1_last_k_block": (0, [(u, 250) for u in (3, 700)]),
    "w1_row_per_tile": (0, [(u, (7 * u) % 256) for u in TILE_UNITS]),
    "w2": (2, [(u, (3 * u + 11) % 1024) for u in TILE_UNITS]),
    "b1_per_tile": (1, [(u,) for u in TILE_UNITS]),
    "b2_per_tile": (3, [(u,) for u in TILE_UNITS]),
}


def poisoned(net, site, value):
    """net with `value` written at every index of POISON_SITES[site] (the other tensors shared, not copied)."""
    which, idx = POISON_SITES[site]
    t = net[which].clone()
    for i in idx:
        t[i] = value
    return net[:which] + (t,) + net[which + 1:]
