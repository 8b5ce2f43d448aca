"""The returns kernels of ktb_returns.cu and the PER sampler and update of ktb_replay.cu at the top of the sizes their C
entries accept, bit for bit (NaN against NaN) against the torch bodies of tests/policy_*_cases.py run on the same GPU
and the header's restatements: n-step spans past the grid's y limit, more than 65 535 blocks in x, long rows through
the staged tile walk, planes of more than 2^31 elements, and PER capacities from 2^24 to 2^30.

Rows are independent in every returns kernel, so where a body or a restatement over the whole array would be too slow
or too large the reference runs on row slices (n-step: on column windows, since its output depends on n + 1 steps);
the kernel always runs on the whole array.  tests/test_returns_limits_cpu.py restates the launch arithmetic and checks
that every shape below reaches the regime its test names.  The peaks in the docstrings are torch.cuda's
max_memory_allocated measured on an H100 80GB HBM3."""
import math

import numpy as np
import pytest
import torch

from kubetorch_b200.device import lib as L
from kubetorch_b200.device import ops, replay, returns
from policy_gae_cases import gae, header_gae
from policy_nstep_cases import header_nstep, nstep
from policy_per_cases import per_sample, per_update, sum_tree
from policy_retrace_cases import header_retrace, retrace
from policy_vtrace_cases import header_vtrace, vtrace
from test_gpu_gae import GUARD, SENTINEL, guarded, guards_untouched, same
from test_gpu_nstep import GAMMAS
from test_gpu_per import LONG_SENTINEL, guarded_long

pytestmark = pytest.mark.gpu

CUDA = "cuda:0"
SPECIAL = [0.0, -0.0, 1.0, -1.5, 1e30, -1e30, 3e38, 1e-40, -1e-45, math.inf, -math.inf, math.nan]
DONES = [1.0, 0.5, math.nan, 0.0]

# n-step across the span boundary: span 1 with grid.y = 65535 exactly, span 2 ending in a one-step tile, span 3
NSTEP_SPAN_TS = [65535 * 32, 65535 * 32 + 1, 65535 * 32 * 2 + 33]
NSTEP_NS = [1, 5, 31, 32]
# more than 65535 blocks in x: 65537 blocks of 32 rows, the last one holding a single row
GRID_N = 65535 * 32 + 33
GRID_TS = [1, 3, 33]
# long rows: thousands of trips around each kernel's ring of stages and a last tile of 3 steps
LONG_N, LONG_T = 33, 100003
# planes of 2^31 + 31 elements: [N, 33] for the recurrences, [33, T] for n-step (span 32)
BIG = 65075263
BIG_SHAPES = {"gae": (BIG, 33), "vtrace": (BIG, 33), "retrace": (BIG, 33), "nstep": (33, BIG)}
# PER capacities around 2^24, where (float)C stops being exact, up to the ABI's 2^30 (2^19 tree blocks)
PER_CASES = [(1 << 24, "sparse"), (1 << 24, "dense"), ((1 << 24) + 1, "sparse"), ((1 << 24) + 1, "dense"),
             ((1 << 24) + 3, "overflow"), ((1 << 24) + 3, "dense"), ((1 << 27) + 5, "sparse"),
             ((1 << 27) + 5, "dense"), ((1 << 30) - 1, "last"), ((1 << 30) - 1, "dense"), (1 << 30, "sparse"),
             (1 << 30, "dense")]
PER_BATCHES = [7, 8192]
PER_BETAS = [0.4, 1.0, 0.5, 2.0]   # every one of torch's pow paths but the fill of β = 0, which hides (float)C


@pytest.fixture(scope="module")
def dev():
    ops.ensure_init([0])
    return 0


@pytest.fixture(autouse=True)
def peak_memory(request):
    """Every test starts from an empty cache and leaves one; its peak allocation is recorded as a user property."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    torch.cuda.synchronize()
    request.node.user_properties.append(("peak_bytes", torch.cuda.max_memory_allocated()))
    torch.cuda.empty_cache()


# ---- helpers ---------------------------------------------------------------------------------------------------------
def same_on_device(got, want, what="", chunk=1 << 26):
    """same() without the trip to the host, for planes too large to copy: NaN against NaN, every other element bit for
    bit, a chunk of 2^26 elements at a time.  Names the first differing element."""
    got, want = got.reshape(-1), want.reshape(-1)
    assert got.numel() == want.numel(), (what, got.numel(), want.numel())
    for a in range(0, got.numel(), chunk):
        g, w = got[a:a + chunk], want[a:a + chunk]
        nan = w.isnan()
        bad = (g.isnan() != nan) | (~nan & (g.view(torch.int32) != w.view(torch.int32)))
        if bool(bad.any()):
            i = int(bad.nonzero()[0, 0])
            pytest.fail(f"{what}: element {a + i} is {float(g[i])!r}, want {float(w[i])!r}")


def guards_and_all_written(buf, offset, n, chunk=1 << 26):
    """guards_untouched() on the guard words alone (the buffer can be gigabytes), and no sentinel left inside: every
    output element was written."""
    lo = GUARD + offset
    guards_untouched(torch.cat([buf[:lo], buf[lo + n:]]), offset, 0)
    bits = buf[lo:lo + n].view(torch.int32)
    for a in range(0, n, chunk):
        assert not bool((bits[a:a + chunk] == SENTINEL).any()), f"an element in [{a}, {a + chunk}) was not written"


def outputs(N, T, offsets=(1, 3)):
    """Two guarded [N, T] outputs: ((buffer, view), (buffer, view))."""
    return [(buf, view.view(N, T)) for buf, view in (guarded(N * T, o) for o in offsets)]


def check_guards(outs, offsets=(1, 3)):
    for (buf, view), o in zip(outs, offsets):
        guards_and_all_written(buf, o, view.numel())


# The [N, T] planes and the [N] vector of each op, in the C entry's order, and its scalars.
PLANES = {"gae": ("rewards", "values", "dones"), "vtrace": ("log_rhos", "rewards", "values", "dones"),
          "retrace": ("log_rhos", "rewards", "q", "values", "dones", "baseline"),
          "nstep": ("rewards", "values", "dones", "baseline")}
PARAMS = {"gae": dict(gamma=0.99, lam=0.95), "vtrace": dict(gamma=0.99, lam=0.95, rho_bar=1.0, c_bar=0.9,
                                                            pg_rho_bar=1.5),
          "retrace": dict(gamma=0.997, lam=0.9), "nstep": dict(n=5, gamma=0.99)}


def kernel(op, ins, outs, p):
    """The op's wrapper (one C call on the current stream) into the given [N, T] outputs."""
    o = dict(zip({"gae": ("adv", "ret"), "vtrace": ("vs", "pg_adv"), "retrace": ("ret", "td"),
                  "nstep": ("ret", "td")}[op], (view for _, view in outs)))
    if op == "gae":
        got = returns.gae(*ins, p["gamma"], p["lam"], **o)
    elif op == "vtrace":
        got = returns.vtrace(*ins, p["gamma"], p["lam"], p["rho_bar"], p["c_bar"], p["pg_rho_bar"], **o)
    elif op == "retrace":
        got = returns.retrace(*ins, p["gamma"], p["lam"], **o)
    else:
        got = returns.nstep(*ins, p["n"], p["gamma"], **o)
    torch.cuda.synchronize()
    return got


def body(op, ins, p):
    if op == "gae":
        return gae(*ins, p["gamma"], p["lam"])
    if op == "vtrace":
        return vtrace(*ins, p["gamma"], p["lam"], p["rho_bar"], p["c_bar"], p["pg_rho_bar"])
    if op == "retrace":
        return retrace(*ins, p["gamma"], p["lam"])
    return nstep(*ins, p["n"], p["gamma"])


def header(op, ins, p):
    if op == "gae":
        return header_gae(*(x.cpu() for x in ins), p["gamma"], p["lam"])
    if op == "vtrace":
        return header_vtrace(*ins, p["gamma"], p["lam"], p["rho_bar"], p["c_bar"], p["pg_rho_bar"])
    if op == "retrace":
        return header_retrace(*ins, p["gamma"], p["lam"])
    return header_nstep(*ins, p["n"], p["gamma"])


def device_rollouts(op, N, T, seed, special_rate=0.01, special_cols=None):
    """Seeded inputs generated on the GPU: random planes, episode ends (done = 1) at 5 % of the steps, and at
    `special_rate` of the elements of columns [0, special_cols) the special values, done = 0.5 and done = NaN.  A NaN
    runs back along a recurrence's row to its start, so long rows keep them near the start of the row."""
    g = torch.Generator(device=CUDA).manual_seed(seed)
    ins = []
    for name in PLANES[op]:
        if name == "dones":
            ins.append((torch.rand(N, T, generator=g, device=CUDA) < 0.05).float())
        else:
            ins.append(torch.randn(N, T, generator=g, device=CUDA) * (0.5 if name == "log_rhos" else 2.0))
    ins.append(torch.randn(N, generator=g, device=CUDA) * 5)
    s, dn = torch.tensor(SPECIAL, device=CUDA), torch.tensor(DONES, device=CUDA)
    for name, x in zip(PLANES[op] + ("vector",), ins):
        y = x[..., :special_cols] if special_cols is not None and x.dim() == 2 else x
        hit = torch.rand(y.shape, generator=g, device=CUDA) < special_rate
        pool = dn if name == "dones" else s
        y[hit] = pool[torch.randint(0, len(pool), (int(hit.sum()),), generator=g, device=CUDA)]
    return ins


# ---- 1. n-step across the span boundary ------------------------------------------------------------------------------
def nstep_span(T):
    """ktb_nstep_f32's span: ceil(n_tiles / 65535), at least kNstepSpan (1)."""
    n_tiles = (T + 31) // 32
    return max(1, (n_tiles + 65534) // 65535)


def span_boundaries(T):
    """The first tile k1 past the spans of blocks 0, 1, 2, a middle one, the last but one and the last (capped at
    the row's tile count)."""
    span, n_tiles = nstep_span(T), (T + 31) // 32
    grid_y = -(-n_tiles // span)
    blocks = sorted({0, 1, 2, grid_y // 2, grid_y - 2, grid_y - 1})
    return [min((y + 1) * span, n_tiles) for y in blocks]


def mark_span_boundaries(ins, T):
    """At steps 32·k1 - 1, 32·k1, 32·k1 + n - 1 and 32·k1 + n of every n in NSTEP_NS, around each span boundary
    k1: row i at boundary j takes, by (i + j) mod 3, special values and an episode end, an episode end alone
    (done 1, 0.5 or NaN), or its random values."""
    r, v, d, b, lv = ins
    steps = sorted({32 * k1 + o for k1 in span_boundaries(T) for o in [-1, 0] + NSTEP_NS + [n - 1 for n in NSTEP_NS]})
    steps = [t for t in steps if 0 <= t < T]
    for j, t in enumerate(steps):
        for i in range(r.shape[0]):
            mode = (i + j) % 3
            if mode == 0:
                r[i, t] = SPECIAL[(i + 2 * j) % len(SPECIAL)]
                v[i, t] = SPECIAL[(i + 3 * j + 1) % len(SPECIAL)]
                b[i, t] = SPECIAL[(i + 5 * j + 2) % len(SPECIAL)]
            if mode < 2:
                d[i, t] = DONES[(i + j) % 3]
    lv[::3] = torch.tensor(SPECIAL, device=CUDA).repeat(lv[::3].numel() // len(SPECIAL) + 1)[:lv[::3].numel()]
    return steps


def header_window(ins, ret, td, a, e, n, gamma):
    """header_nstep over steps [a, e) of every row against the kernel's outputs there: all of them when e is the
    row's end (last_values then bootstraps), else the first e - a - n, whose windows lie inside [a, e)."""
    r, v, d, b, lv = ins
    T = r.shape[1]
    last = lv if e == T else torch.zeros_like(lv)
    hr, ht = header_nstep(r[:, a:e], v[:, a:e], d[:, a:e], b[:, a:e], last, n, gamma)
    m = e - a if e == T else e - a - n
    same(ret[:, a:a + m], hr[:, :m], ("header ret", a, e, n))
    same(td[:, a:a + m], ht[:, :m], ("header td", a, e, n))


@pytest.mark.parametrize("T", NSTEP_SPAN_TS, ids=["span1", "span2", "span3"])
@pytest.mark.parametrize("N", [1, 33])
def test_nstep_across_span_boundaries(dev, N, T):
    """Every row and step of ktb_nstep_f32 against the body nstep() (vectorised over T, so it runs on the whole
    array), for n = 1, 5, 31 and 32: T = 65535·32 is span 1 with grid.y = 65535 exactly, 65535·32 + 1 span 2 whose
    last block ends in a tile of one step, 65535·64 + 33 span 3.  Episode ends, special values and done 0.5 / NaN
    sit at the span boundaries of the first three blocks, a middle one and the last two, where each block's last
    halo is cut to n steps and every other halo is a whole tile copied once.  header_nstep checks the 128 steps
    around the first, the last but one and the last boundary of every row.  The guard bands around ret and td stay
    untouched and every element is written.  Peak: 7.8 GB at N = 33, span 3."""
    ins = device_rollouts("nstep", N, T, seed=N * 7 + T % 1000, special_rate=0.0005)
    mark_span_boundaries(ins, T)
    k1s = span_boundaries(T)
    for i, n in enumerate(NSTEP_NS):
        gamma = GAMMAS[(i + NSTEP_SPAN_TS.index(T)) % len(GAMMAS)]
        outs = outputs(N, T)
        ret, td = kernel("nstep", ins, outs, dict(n=n, gamma=gamma))
        check_guards(outs)
        want = nstep(*ins, n, gamma)
        same_on_device(ret, want[0], ("torch ret", N, T, n))
        same_on_device(td, want[1], ("torch td", N, T, n))
        del want
        for k1 in (k1s[0], k1s[-2], k1s[-1]):
            a = max(0, 32 * k1 - 64)
            header_window(ins, ret, td, a, min(T, 32 * k1 + 64 + n), n, gamma)
        del outs, ret, td


# ---- 2. grid x beyond 65 535 blocks ----------------------------------------------------------------------------------
GRID_ROWS = [(0, 64), (65534 * 32, GRID_N)]   # blocks 0-1, and blocks 65534, 65535 and the last (one row)


@pytest.mark.parametrize("T", GRID_TS)
@pytest.mark.parametrize("op", ["gae", "vtrace", "retrace", "nstep"])
def test_more_than_65535_blocks_in_x(dev, op, T):
    """N = 65535·32 + 33 rows: 65537 blocks in grid.x, the last one a single row.  The body runs on the whole array
    (T <= 33 steps of its loop) and must equal the kernel at every element; the header's restatement checks rows
    [0, 64) (blocks 0 and 1) and [65534·32, N) (blocks 65534, 65535 and the partial last one).  Guards and every
    element written are checked.  Peak: 5.0 GB, V-trace at T = 33."""
    p = PARAMS[op]
    ins = device_rollouts(op, GRID_N, T, seed=T + len(op))
    outs = outputs(GRID_N, T)
    got = kernel(op, ins, outs, p)
    check_guards(outs)
    want = body(op, ins, p)
    for k in range(2):
        same_on_device(got[k], want[k], (op, T, "torch", k))
    del want
    for a, e in GRID_ROWS:
        h = header(op, [x[a:e] for x in ins], p)
        for k in range(2):
            same(got[k][a:e], h[k], (op, T, a, "header", k))


# ---- 3. long rows through the staged tile walk -----------------------------------------------------------------------
@pytest.mark.parametrize("op", ["gae", "vtrace", "retrace"])
def test_long_rows(dev, op):
    """N = 33 rows of T = 100 003 steps: 3126 tiles per warp, so thousands of trips around the kStages ring, and a
    last tile of 3 steps, which is the first one each warp scans.  Every element against the body's per-step torch
    loop and the header's restatement.  Special values and done 0.5 / NaN are kept in the first 64 steps of each row,
    since a NaN makes every earlier step of its row NaN; episode ends run over the whole row.  Peak: 0.24 GB."""
    p = PARAMS[op]
    ins = device_rollouts(op, LONG_N, LONG_T, seed=len(op), special_rate=0.05, special_cols=64)
    outs = outputs(LONG_N, LONG_T)
    got = kernel(op, ins, outs, p)
    check_guards(outs)
    want = body(op, ins, p)
    h = header(op, ins, p)
    for k in range(2):
        same_on_device(got[k], want[k], (op, "torch", k))
        same(got[k], h[k], (op, "header", k))


# ---- 4. planes of more than 2^31 elements ----------------------------------------------------------------------------
BIG_NEED = 3 * BIG * 33 * 4 + (1 << 30)   # one input plane, two outputs and 1 GiB for the references and guards


def big_row_slices():
    """The [N, 33] ops' checked rows: the first 64, 64 around element 2^30, and the last 64, the last row holding
    elements 2^31 - 2 to 2^31 + 30."""
    mid = (1 << 30) // 33
    return [(0, 64), (mid - 32, mid + 32), (BIG - 64, BIG)]


def big_windows():
    """n-step's checked steps of all 33 rows: the first 256, 256 around the span boundary at step 1024·31744 (span
    32), and the last 256, row 32's last 31 steps being elements 2^31 to 2^31 + 30."""
    mid = 1024 * 31744
    return [(0, 256), (mid - 128, mid + 128 + 32), (BIG - 256, BIG)]


def fill_pattern(x, seed):
    """Small finite values, episode ends (1.0) at every 7th element and a block of special values near the start:
    the pattern of the checked parts of the one aliased input plane."""
    g = torch.Generator().manual_seed(seed)
    y = torch.rand(x.shape, generator=g) * 0.5 - 0.25
    y.view(-1)[::7] = 1.0
    y.view(-1)[3:3 + 2 * len(SPECIAL):2] = torch.tensor(SPECIAL)
    x.copy_(y)


@pytest.mark.parametrize("op", ["gae", "vtrace", "retrace", "nstep"])
def test_planes_past_2_31_elements(dev, op):
    """N·T = 2^31 + 31 elements per plane: [65 075 263, 33] for GAE, V-trace and Retrace (2 033 602 blocks in
    grid.x), [33, 65 075 263] for n-step (span 32).  Every input is one aliased plane (the header allows it for
    n-step and Retrace, check_buffers for all four; the [N] vector is the plane's first N elements), zero except the
    checked parts, which hold fill_pattern().  The reference runs on those parts: rows big_row_slices() of the
    recurrences, column windows big_windows() of every n-step row at n = 5 and 32; in both the last part holds
    finite elements past index 2^31 - 1.  The guard bands stay untouched and no output element is left unwritten.
    Skipped only when the GPU has less free memory than BIG_NEED (26.8 GB).  Peak: 25.8 GB, three 8.6 GB planes."""
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < BIG_NEED:
        pytest.skip(f"needs {BIG_NEED / 1e9:.1f} GB of free GPU memory for three planes of 2^31 + 31 fp32 elements, "
                    f"{free / 1e9:.1f} GB free")
    N, T = BIG_SHAPES[op]
    plane = torch.zeros(N, T, device=CUDA)
    parts = big_windows() if op == "nstep" else big_row_slices()
    for k, (a, e) in enumerate(parts):
        fill_pattern(plane[:, a:e] if op == "nstep" else plane[a:e], seed=k)
    vec = plane.view(-1)[:N]
    ins = [plane] * len(PLANES[op]) + [vec]
    last_flat = (N - 1) * T + T - 1
    assert last_flat > (1 << 31) - 1
    for n in ([5, 32] if op == "nstep" else [None]):
        p = dict(PARAMS[op], n=n) if n else PARAMS[op]
        outs = outputs(N, T)
        got = kernel(op, ins, outs, p)
        check_guards(outs)
        past = 0   # checked elements past index 2^31 - 1 whose reference is finite
        for a, e in parts:
            if op == "nstep":
                last = vec if e == T else torch.zeros_like(vec)
                want = nstep(*(x[:, a:e] for x in ins[:-1]), last, n, p["gamma"])
                m = e - a if e == T else e - a - n
                for k in range(2):
                    same_on_device(got[k][:, a:a + m], want[k][:, :m], (op, n, a, k))
                flat = torch.arange(N, device=CUDA)[:, None] * T + torch.arange(a, a + m, device=CUDA)
                past += int(((flat > (1 << 31) - 1) & want[0][:, :m].isfinite()).sum())
            else:
                want = body(op, [x[a:e] for x in ins], p)
                for k in range(2):
                    same_on_device(got[k][a:e], want[k], (op, a, k))
                flat = torch.arange(a * T, e * T, device=CUDA).view(e - a, T)
                past += int(((flat > (1 << 31) - 1) & want[0].isfinite()).sum())
        assert past > 0, "no finite reference element past index 2^31 - 1"
        del outs, got, want
        torch.cuda.empty_cache()


# ---- 5. PER at large C -----------------------------------------------------------------------------------------------
def device_priorities(c, kind, seed, offset):
    """(buffer, priorities) generated on the GPU with a seeded generator, at `offset` words into the buffer:
      sparse    uniform [0, 2) with 30 % zeros and one dominant item (1 + C/8) at a random leaf;
      last      sparse with the dominant item at leaf C - 1;
      dense     uniform [0.01, 2.01): no zero, so min p > 0 and the weights are finite;
      overflow  3e38 at every nonzero of sparse: the total overflows to inf."""
    g = torch.Generator(device=CUDA).manual_seed(seed)
    buf = torch.empty(c + offset + 1, device=CUDA)
    p = buf[offset:offset + c]
    p.uniform_(0.0, 2.0, generator=g)
    if kind == "dense":
        p.add_(0.01)
    else:
        for a in range(0, c, 1 << 26):
            x = p[a:a + (1 << 26)]
            x.masked_fill_(torch.rand(x.numel(), generator=g, device=CUDA) < 0.3, 0.0)
        at = c - 1 if kind == "last" else int(torch.randint(0, c, (1,), generator=g, device=CUDA))
        p[at] = 1.0 + c / 8
        if kind == "overflow":
            p.masked_fill_(p > 0, 3e38)
    return buf, p


def tree_equals_body(tree, p, what):
    """The kernel's tree against the body's levels in the header's layout, level by level on the device (body_tree()
    builds a second tree and compares on the host, which at 2^30 leaves is two more 4 GiB copies)."""
    levels = sum_tree(p)
    for lv in levels[1:]:
        same_on_device(tree[lv.numel():2 * lv.numel()], lv, (what, "level of", lv.numel()))   # the root is tree[1]
    same_on_device(tree[0:1], p.min().view(1), (what, "min"))
    return bool(levels[-1][0].isfinite())


def sample(dev, p, seed, batch, beta):
    """ktb_per_sample_f32 on p into guarded outputs, guards checked on the device: (tree, indices, weights)."""
    c = p.numel()
    tn = replay.tree_size(c)
    (tbuf, tree), (wbuf, w) = guarded(tn, 3), guarded(batch, 2)
    ibuf, idx = guarded_long(batch)
    rc = L.load().ktb_per_sample_f32(dev, p.data_ptr(), c, batch, 0, batch, seed, replay.per_scalars(beta=beta)[0],
                                     tree.data_ptr(), idx.data_ptr(), w.data_ptr(), ops.current_stream_handle(0))
    assert rc == L.OK, L.last_error()
    torch.cuda.synchronize()
    guards_and_all_written(tbuf, 3, tn)
    guards_untouched(wbuf, 2, batch)
    bits = ibuf.cpu()
    assert (bits[:GUARD] == LONG_SENTINEL).all() and (bits[GUARD + batch:] == LONG_SENTINEL).all()
    return tree, idx, w


@pytest.mark.parametrize("c,kind", PER_CASES, ids=[f"{c}-{k}" for c, k in PER_CASES])
def test_per_sample_at_large_capacity(dev, c, kind):
    """ktb_per_sample_f32 at C from 2^24 to 2^30, batches 7 and 8192: the tree equals the body's levels, the indices
    and weights equal per_sample() on the GPU, every index lies in [0, C), indices never decrease, and with a finite
    total no zero priority is drawn.  (float)C is inexact at 2^24 + 1, 2^24 + 3, 2^27 + 5 and 2^30 - 1; the dense
    priorities have min p > 0, so their weights are finite and show (float)C's bits.  C > 2^29 has 2^19 tree blocks
    for the top kernel and a 30-level descent.  The priorities sit at word offset 0 (float4 loads) or 1 (scalar
    loads) of their buffer.  Peak: 17.6 GB at C = 2^30 - 1 and 2^30: priorities, tree and the body's levels."""
    i = PER_CASES.index((c, kind))
    buf, p = device_priorities(c, kind, seed=i, offset=i % 2)
    for k, batch in enumerate(PER_BATCHES):
        beta = PER_BETAS[(i + k) % len(PER_BETAS)]
        seed = 1000 * i + batch
        tree, idx, w = sample(dev, p, seed, batch, beta)
        finite = tree_equals_body(tree, p, (c, kind, batch))
        assert finite == (kind != "overflow")
        del tree
        torch.cuda.empty_cache()
        want_idx, want_w = per_sample(p, seed, batch, beta)
        assert torch.equal(idx, want_idx), (c, kind, batch)
        same_on_device(w, want_w, (c, kind, batch, beta, "weights"))
        assert bool(((idx >= 0) & (idx < c)).all()) and bool((idx[1:] >= idx[:-1]).all())
        if finite:
            assert bool((p[idx] > 0).all()), "a zero-priority item was drawn"
        if kind == "last" and batch == 8192:
            assert bool((idx == c - 1).any()), "the dominant item at leaf C - 1 was never drawn"
        if kind == "dense":
            assert bool((w > 0).all()) and bool(w.isfinite().all())


# ---- the update at C = 2^30 ------------------------------------------------------------------------------------------
UPDATE_SLOTS = 14   # log2 of the update's hash slots at B = 8192: the least power of two >= 2·B


def update_slot(k, log2_slots=UPDATE_SLOTS):
    """per_update_kernel's home slot of index k: the top log2_slots bits of k·0x9E3779B1 mod 2^32."""
    return ((np.asarray(k, dtype=np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)) >> np.uint64(
        32 - log2_slots)


def colliding_indices(c=1 << 30, count=8192, log2_slots=UPDATE_SLOTS):
    """`count` distinct indices below c, the largest ones there are, that share one home slot of the update's hash
    table: found on the host by inverting the multiplier over the 2^(32 - log2_slots) products of the slot whose
    preimages reach closest to c."""
    inv = pow(0x9E3779B1, -1, 1 << 32)
    best = None
    for h in range(64):
        x = np.arange(h << (32 - log2_slots), (h + 1) << (32 - log2_slots), dtype=np.uint64)
        k = (x * np.uint64(inv)) & np.uint64(0xFFFFFFFF)
        k = np.sort(k[k < c])[-count:]
        if best is None or k[0] > best[0]:
            best = k
    return best.astype(np.int64)


def body_on_positions(want, indices, td, alpha, eps):
    """per_update() on the positions the indices name, in place in `want`: the in-range indices (the body raises on
    the others) renumbered onto a compact copy of those priorities, so the body runs at size B rather than C."""
    keep = (indices >= 0) & (indices < want.numel())
    uniq, inv = torch.unique(indices[keep], return_inverse=True)
    sub = want[uniq]
    per_update(sub, inv, td[keep], alpha, eps)
    want[uniq] = sub


def test_per_update_at_the_largest_capacity(dev):
    """ktb_per_update_f32 on C = 2^30 priorities between guard bands: indices C - 1, C, 2^31, -1 and 2^32 + 5 among
    in-range ones (the out-of-range ones write nothing), 8192 copies of C - 1 (the last occurrence wins), and 8192
    distinct indices near 2^30 that share one home slot of the 2^14-slot hash table, so every key probes past the
    others.  After each call the whole buffer equals per_update() applied to the named positions, and the guards
    are untouched.  Peak: 9.0 GB."""
    c = 1 << 30
    buf, p = guarded(c, 1)
    g = torch.Generator(device=CUDA).manual_seed(5)
    p.uniform_(0.0, 2.0, generator=g)
    want = p.clone()
    collide = colliding_indices()
    assert len(set(update_slot(collide).tolist())) == 1 and len(set(collide.tolist())) == 8192
    cases = [
        (torch.tensor([c - 1, c, 1 << 31, -1, (1 << 32) + 5, 0, c - 1, 12345, c, c - 2]), 0.6),
        (torch.full((8192,), c - 1), 1.0),
        (torch.from_numpy(collide[np.random.default_rng(0).permutation(8192)]), 0.5),
    ]
    for indices, alpha in cases:
        indices = indices.to(CUDA)
        td = torch.randn(len(indices), generator=g, device=CUDA) * 3
        td[::97] = torch.tensor([0.0, -0.0, math.inf, math.nan, 1e-40], device=CUDA)[
            torch.arange(len(td[::97]), device=CUDA) % 5]
        assert replay.per_update(p, indices, td, alpha, 1e-6) is p
        torch.cuda.synchronize()
        body_on_positions(want, indices, td, alpha, 1e-6)
        same_on_device(p, want, (len(indices), alpha))
        guards_and_all_written(buf, 1, c)
