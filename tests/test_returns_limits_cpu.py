"""The launch plan behind tests/test_gpu_returns_limits.py, without a GPU: the grid arithmetic of ktb_returns.cu's and
ktb_replay.cu's C entries restated in Python from their sources, and every shape of the GPU file checked to reach the
regime its test names.  A retuned kNstepSpan, tile or tree size fails here rather than leaving the GPU tests quietly
short of the code paths they were written for."""
import os
import re

import numpy as np

import test_gpu_returns_limits as G

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "kubetorch_b200", "csrc")
RETURNS = open(os.path.join(CSRC, "ktb_returns.cu")).read()
REPLAY = open(os.path.join(CSRC, "ktb_replay.cu")).read()
INT31 = (1 << 31) - 1


def constant(src, name):
    """The value of `constexpr int|size_t name = <expression>;` in src, its k-constants resolved the same way."""
    m = re.search(r"constexpr (?:int|size_t) %s = ([^;]+);" % name, src)
    assert m, name
    expr = m.group(1).replace("size_t(1)", "1")
    assert re.fullmatch(r"[\w\s*+<()-]+", expr), expr   # integer arithmetic only
    return int(eval(expr, {"__builtins__": {}}, {k: constant(src, k) for k in re.findall(r"\bk[A-Z]\w*", expr)}))


def code(src):
    return " ".join(src.split())


# ---- the launch arithmetic, as the C entries compute it --------------------------------------------------------------
K_NSTEP_SPAN = constant(RETURNS, "kNstepSpan")
K_TREE_SPAN = constant(REPLAY, "kTreeSpan")
ROWS_PER_BLOCK = 32   # one warp per 32 rows in every returns kernel
STEPS_PER_TILE = 32


def test_the_sources_launch_as_restated():
    r = code(RETURNS)
    # gae, vtrace and retrace: one block per 32 rows
    assert r.count("<<<(unsigned)((N + 31) / 32), 32,") == 3
    assert "size_t span = (n_tiles + 65534) / 65535;" in r
    assert "span = span > (size_t)kNstepSpan ? span : (size_t)kNstepSpan;" in r
    assert "const dim3 grid((unsigned)((N + 31) / 32), (unsigned)((n_tiles + span - 1) / span));" in r
    assert r.count("const size_t n_tiles = (T + 31) / 32;") == 3
    p = code(REPLAY)
    assert "const size_t blocks = P > (size_t)kTreeSpan ? P / kTreeSpan : 1;" in p
    assert "if (blocks > 1) per_tree_top_kernel<<<1, kTopThreads, 0, s>>>(tree, blocks);" in p
    assert "while ((size_t(1) << log2_slots) < 2 * B) ++log2_slots;" in p
    assert "uint32_t h = (k * 0x9E3779B1u) >> (32 - log2_slots);" in p
    assert "1.0f / (float)batch, (float)C, -beta" in p
    assert constant(REPLAY, "kPerMaxC") == 1 << 30 and constant(REPLAY, "kPerMaxBatch") == 8192


def nstep_grid(N, T):
    """(grid.x, grid.y, span) of ktb_nstep_f32."""
    n_tiles = (T + STEPS_PER_TILE - 1) // STEPS_PER_TILE
    span = max((n_tiles + 65534) // 65535, K_NSTEP_SPAN)
    return (N + ROWS_PER_BLOCK - 1) // ROWS_PER_BLOCK, (n_tiles + span - 1) // span, span


def grid_x(N):
    return (N + ROWS_PER_BLOCK - 1) // ROWS_PER_BLOCK


def per_plan(C):
    """(P, tree blocks, descent levels) of ktb_per_sample_f32."""
    P = 1
    while P < C:
        P <<= 1
    return P, P // K_TREE_SPAN if P > K_TREE_SPAN else 1, P.bit_length() - 1


def log2_slots(B):
    s = 1
    while (1 << s) < 2 * B:
        s += 1
    return s


# ---- every GPU shape reaches its regime ------------------------------------------------------------------------------
def test_nstep_shapes_reach_spans_1_2_3_and_32():
    plans = [nstep_grid(1, t) for t in G.NSTEP_SPAN_TS]
    assert [span for _, _, span in plans] == [1, 2, 3]
    assert plans[0][1] == 65535                       # span 1 fills grid.y exactly
    _, y, span = plans[1]
    last_block_tiles = (G.NSTEP_SPAN_TS[1] + 31) // 32 - (y - 1) * span
    assert last_block_tiles == 2 and G.NSTEP_SPAN_TS[1] % 32 == 1   # span 2's last block: a whole tile, then one step
    assert nstep_grid(33, G.NSTEP_SPAN_TS[0])[0] == 2
    for T in G.NSTEP_SPAN_TS:   # the GPU file's own span, and its boundaries inside the row
        assert G.nstep_span(T) == nstep_grid(1, T)[2]
        k1s = G.span_boundaries(T)   # blocks 0 and the last among them; the last one ends the row
        assert k1s[0] == G.nstep_span(T) and k1s[-1] == (T + 31) // 32 and all(32 * k1 < T for k1 in k1s[:-1])
    _, y, span = nstep_grid(*G.BIG_SHAPES["nstep"])
    assert span >= 16 and y <= 65535 and span == 32
    assert all(n <= 32 for n in G.NSTEP_NS) and max(G.NSTEP_NS) == 32


def test_grid_x_shapes_pass_65535_blocks():
    assert grid_x(G.GRID_N) == 65537 and G.GRID_N % 32 == 1    # the last block holds one row
    lo, hi = G.GRID_ROWS[-1]
    assert lo // 32 <= 65534 and hi == G.GRID_N                # the header sees blocks 65534 to the last
    for op, (N, T) in G.BIG_SHAPES.items():
        if op != "nstep":
            assert grid_x(N) > 65535


def test_long_rows_circle_the_ring():
    n_tiles = (G.LONG_T + 31) // 32
    stages = [constant(RETURNS, k) for k in ("kGaeStages", "kVtraceStages", "kRetraceStages")]
    assert all(n_tiles > 1000 * s for s in stages) and G.LONG_T % 32 != 0


def test_big_planes_put_checked_elements_past_2_31():
    for op, (N, T) in G.BIG_SHAPES.items():
        assert N * T == (1 << 31) + 31
        if op == "nstep":
            a, e = G.big_windows()[-1]
            assert e == T and (N - 1) * T + e - 1 > INT31   # the last window reaches row 32's elements past 2^31 - 1
        else:
            a, e = G.big_row_slices()[-1]
            assert e == N and (N - 1) * T + T - 1 > INT31 and (N - 1) * T <= INT31   # the last row straddles 2^31
    assert G.BIG_NEED < 27e9


def test_per_capacities_reach_inexact_float_c_and_2_19_blocks():
    cs = sorted({c for c, _ in G.PER_CASES})
    assert cs == [1 << 24, (1 << 24) + 1, (1 << 24) + 3, (1 << 27) + 5, (1 << 30) - 1, 1 << 30]
    inexact = [c for c in cs if float(np.float32(c)) != c]
    assert inexact == [(1 << 24) + 1, (1 << 24) + 3, (1 << 27) + 5, (1 << 30) - 1]
    assert all((c, "dense") in G.PER_CASES for c in inexact)   # min p > 0: weights that show (float)C
    assert 0.0 not in G.PER_BETAS                              # β = 0 makes every weight 1
    assert per_plan(1 << 30) == (1 << 30, 1 << 19, 30) and per_plan((1 << 30) - 1)[1] == 1 << 19
    assert per_plan((1 << 24) + 1)[1] > 1024                    # past the 1024 threads of the top kernel
    kinds = {k for _, k in G.PER_CASES}
    assert {"overflow", "last"} <= kinds and G.PER_BATCHES == [7, 8192]


def test_update_keys_share_one_slot_near_2_30():
    assert log2_slots(8192) == G.UPDATE_SLOTS
    keys = G.colliding_indices()
    assert len(keys) == 8192 and len(set(keys.tolist())) == 8192
    assert keys.max() < 1 << 30 and keys.min() > (1 << 30) * 7 // 8
    slots = ((keys.astype(np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)) >> np.uint64(32 - 14)
    assert len(set(slots.tolist())) == 1
