"""Prioritized replay without a GPU: the header's fp32 restatement equals the body of tests/policy_per_cases.py bit for
bit (tree, indices, weights); the body's properties over capacities around powers of two and the usual β (indices in
range whatever the priorities hold, no zero-priority draw, indices that never decrease, the same bits under every split
of the strata); draw frequencies that match p_i / Σp; the replay noise stream; the update's last-occurrence rule;
kt.mapped("per")'s options; the wrapper's scalars; the ctypes prototypes and the first status of each entry."""
import ctypes
import math
import os
import re
from unittest import mock

import numpy as np
import pytest
import torch
from scipy import stats

import kubetorch_b200 as kt
from kubetorch_b200.device import lib as L
from kubetorch_b200.mapped import MLP_FORMS
from kubetorch_b200.sampling import gumbel_uniform, replay_noise
from oracle import ref_dispatch
from policy_per_cases import (BETA, header_per_sample, mapped_per, mapped_per_beta, per_sample, per_update,
                              sum_tree)
from test_gae_cpu import same

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "ktb200.h")
CS = [1, 2, 3, 31, 32, 33, 1000, 4097]
BETAS = [0.0, 0.4, 0.5, 1.0]


def priorities(c, seed, zeros=0.3):
    """Seeded priorities p^α: uniform in (0, 2) with a share of exact zeros."""
    g = torch.Generator().manual_seed(seed)
    p = torch.rand(c, generator=g) * 2
    p[torch.rand(c, generator=g) < zeros] = 0.0
    if not (p > 0).any():
        p[c // 2] = 1.0
    return p


def tree_of(levels):
    """The body's levels in the header's layout: [min, total, internal nodes 2 .. P - 1] (no leaves)."""
    p = levels[0].numel()
    out = torch.zeros(max(p, 2))
    for lv in levels[1:]:
        out[lv.numel():2 * lv.numel()] = lv
    out[1] = levels[-1][0]
    return out


# ---- the header restatement -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("c", CS)
def test_header_restatement_equals_the_body(c, beta):
    p = priorities(c, seed=c)
    batch = 64
    tree, idx, w = header_per_sample(p, 11 + c, batch, beta)
    want_idx, want_w = per_sample(p, 11 + c, batch, beta)
    want_tree = tree_of(sum_tree(p))
    want_tree[0] = p.min()
    same(tree, want_tree, c)
    assert np.array_equal(idx, want_idx.numpy()), c
    same(w, want_w, (c, beta))


def test_header_restatement_on_special_values():
    s = torch.tensor([0.0, 1e-45, 1e-40, 3e38, math.inf, math.nan, 1.0, 0.25])
    for c in (8, 33, 1000):
        p = s.repeat(c // 8 + 1)[:c][torch.randperm(c, generator=torch.Generator().manual_seed(c))].contiguous()
        for beta in BETAS:
            tree, idx, w = header_per_sample(p, c, 128, beta)
            want_idx, want_w = per_sample(p, c, 128, beta)
            assert np.array_equal(idx, want_idx.numpy()), (c, beta)
            same(w, want_w, (c, beta))


# ---- properties -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("beta", BETAS)
@pytest.mark.parametrize("c", CS)
def test_properties(c, beta):
    p = priorities(c, seed=100 + c)
    for seed in range(3):
        idx, w = per_sample(p, seed, 256, beta)
        assert idx.dtype == torch.int64 and w.dtype == torch.float32
        assert ((idx >= 0) & (idx < c)).all()
        assert (p[idx] > 0).all(), "a zero-priority item was drawn"
        assert (idx[1:] >= idx[:-1]).all(), "indices decrease between strata"
        if beta == 0.0:
            assert (w == 1.0).all()
        elif p.min() == 0:   # the largest weight, of a zero priority, is inf
            assert (w == 0).all()
        else:
            assert (w > 0).all() and (w <= 1.0 + 1e-6).all()
        # every split of the strata into calls draws the same bits
        for cuts in ([0, 100, 256], [0, 1, 2, 255, 256], [0, 37, 38, 200, 256]):
            parts = [per_sample(p, seed, 256, beta, a, b - a) for a, b in zip(cuts, cuts[1:])]
            assert torch.equal(torch.cat([x[0] for x in parts]), idx)
            same(torch.cat([x[1] for x in parts]), w)


def test_indices_stay_in_range_whatever_the_priorities_hold():
    g = torch.Generator().manual_seed(5)
    for c in CS:
        for fill in (math.nan, math.inf, -math.inf, -1.0, 0.0, 3e38):
            p = torch.rand(c, generator=g)
            p[torch.rand(c, generator=g) < 0.3] = fill
            idx, _ = per_sample(p, c, 512, 0.4)
            assert ((idx >= 0) & (idx < c)).all(), (c, fill)
            tree, h_idx, _ = header_per_sample(p, c, 512, 0.4)
            assert np.array_equal(h_idx, idx.numpy()), (c, fill)


def test_all_zero_priorities_draw_index_zero():
    idx, w = per_sample(torch.zeros(33), 1, 16, 0.4)
    assert (idx == 0).all() and w.isnan().all()


def test_draw_frequencies_match_the_priorities():
    """χ² over 400 batches of 64: each item's count against 400·64·p_i / Σp (stratified draws vary less than a
    multinomial, so the multinomial's χ² is a loose bound)."""
    p = priorities(33, seed=3)
    counts = torch.zeros(33)
    for seed in range(400):
        idx, _ = per_sample(p, seed, 64, 0.4)
        counts += torch.bincount(idx, minlength=33).float()
    expected = p / p.sum() * counts.sum()
    live = expected > 0
    assert counts[~live].sum() == 0
    assert stats.chisquare(counts[live].numpy(), expected[live].double().numpy() * (
        counts.sum().item() / expected[live].double().sum().item())).pvalue > 1e-3
    # 1 : 2 : 3 : 4 over 2000 seeds
    freq = torch.zeros(4)
    for seed in range(2000):
        freq += torch.bincount(per_sample(torch.tensor([1.0, 2.0, 3.0, 4.0]), seed, 1, 0.4)[0], minlength=4).float()
    assert torch.allclose(freq / 2000, torch.tensor([0.1, 0.2, 0.3, 0.4]), atol=0.03)


# ---- the body on any number of ranks ----------------------------------------------------------------------------------
@pytest.mark.parametrize("ranks", [1, 2, 3, 5])
def test_body_through_the_oracle_is_independent_of_the_rank_count(ranks):
    p = priorities(1000, seed=9)
    with mock.patch.dict(os.environ, {"RANK": "0", "WORLD_SIZE": "1"}):
        want = mapped_per(p, 21)
    got = ref_dispatch.spmd_call(mapped_per, p, 21, num_proc=ranks, serialization="pickle")
    assert len(got) == ranks
    assert torch.equal(torch.cat([g[0] for g in got]), want[0])
    same(torch.cat([g[1] for g in got]), want[1])
    named = ref_dispatch.spmd_call(mapped_per_beta, p, 21, BETA, num_proc=ranks, serialization="pickle")
    assert torch.equal(torch.cat([g[0] for g in named]), want[0])


# ---- the noise stream -------------------------------------------------------------------------------------------------
def test_replay_noise_shards_and_is_its_own_stream():
    whole = replay_noise(77, 0, 8192)
    assert whole.dtype == torch.float32 and ((whole > 0) & (whole < 1)).all()
    assert torch.equal(torch.cat([replay_noise(77, a, b - a) for a, b in [(0, 5), (5, 4000), (4000, 8192)]]), whole)
    assert torch.equal(replay_noise(77, 3, 1), whole[3:4])
    for word3 in range(4):
        other = gumbel_uniform(77, 0, 8192, 2, word3=word3)
        assert not (other == whole[:, None]).any(dim=1).any(), word3
    assert not torch.equal(replay_noise(78, 0, 8192), whole)
    assert kt.replay_noise is replay_noise


# ---- the update -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alpha", [0.5, 0.6, 1.0])
def test_update_takes_the_last_occurrence(alpha):
    g = torch.Generator().manual_seed(int(alpha * 10))
    c = 1000
    for indices in (torch.full((64,), 17), torch.randint(0, 50, (512,), generator=g), torch.randperm(c)[:300]):
        td = torch.randn(len(indices), generator=g)
        p = torch.rand(c, generator=g)
        want, new = p.clone(), (td.abs() + 1e-6) ** alpha
        for b in range(len(indices)):   # in order: the last write wins
            want[indices[b]] = new[b]
        per_update(p, indices, td, alpha, 1e-6)
        same(p, want, alpha)


# ---- kt.mapped("per") -------------------------------------------------------------------------------------------------
def _body(*params):
    ns = {}
    exec(f"def body({', '.join(params)}):\n    pass", ns)
    return ns["body"]


def test_mapped_takes_constants_and_names():
    spec = kt.mapped("per", batch=512, beta=0.4, seed="seed")(_body("prio", "seed")).__ktb_mapped__
    assert spec.op == "per" and spec.extra == dict(batch=512, seed="seed", beta=0.4)
    spec = kt.mapped("per", batch=1, beta="b", seed=7, self_check=False)(_body("prio", "b")).__ktb_mapped__
    assert spec.extra == dict(batch=1, seed=7, self_check=False, beta="b")
    assert kt.mapped("per", batch=8192, beta=0, seed=0)(_body("p")).__ktb_mapped__.extra["beta"] == 0


REFUSED = dict(alpha=2.0, reduce="sum", arg="prio", bias=True, output="logits", n=5, gamma=0.99, lam=0.95,
               **{k: "x" for k in MLP_FORMS if k not in ("seed", "gamma", "alpha")})


@pytest.mark.parametrize("option", sorted(REFUSED))
def test_mapped_refuses_every_other_option(option):
    with pytest.raises(ValueError, match=f"^{option}= is not an option of the 'per' op, which takes batch=, beta=, "
                                         f"seed= and self_check=: its callable is \\(priorities, ...\\)"):
        kt.mapped("per", batch=512, beta=0.4, seed="seed", **{option: REFUSED[option]})


@pytest.mark.parametrize("kw,match", [
    (dict(beta=0.4, seed=1), "batch= is required with the 'per' op"),
    (dict(batch=512, seed=1), "beta= is required with the 'per' op"),
    (dict(batch=512, beta=0.4), "seed= is required with the 'per' op"),
    (dict(batch=0, beta=0.4, seed=1), "batch must be an int constant in \\[1, 8192\\]"),
    (dict(batch=8193, beta=0.4, seed=1), "batch must be an int constant"),
    (dict(batch="batch", beta=0.4, seed=1), "batch must be an int constant"),
    (dict(batch=True, beta=0.4, seed=1), "batch must be an int constant"),
    (dict(batch=512, beta=-0.1, seed=1), "beta must be >= 0"),
    (dict(batch=512, beta=math.nan, seed=1), "beta must be a finite number"),
    (dict(batch=512, beta=0.4, seed=-1), "seed must be an int in \\[0, 2\\*\\*64\\)"),
    (dict(batch=512, beta=0.4, seed=1.0), "seed must be an int"),
    (dict(batch=512, beta=0.4, seed=1, self_check=1), "self_check must be True or False"),
])
def test_mapped_refuses_missing_or_bad_parameters(kw, match):
    with pytest.raises(ValueError, match=match):
        kt.mapped("per", **kw)


def test_mapped_refuses_a_name_that_is_not_an_argument_and_a_callable_without_parameters():
    with pytest.raises(ValueError, match="'seed' is not an argument"):
        kt.mapped("per", batch=512, beta=0.4, seed="seed")(_body("prio", "s"))
    with pytest.raises(ValueError, match="'beta' is not an argument"):
        kt.mapped("per", batch=512, beta="beta", seed=1)(_body("prio"))
    with pytest.raises(ValueError, match="takes \\(priorities, ...\\) positionally"):
        kt.mapped("per", batch=512, beta=0.4, seed=1)(_body())


def test_wrapper_scalars_follow_torch():
    from kubetorch_b200.device.replay import per_scalars

    for v in BETAS + [0.6, 1 / 3, 2.0, 7]:
        assert per_scalars(beta=v) == ((torch.ones(1) * v).item(),), v
    assert per_scalars(alpha=0.6, eps=1e-6) == ((torch.ones(1) * 0.6).item(), (torch.ones(1) * 1e-6).item())
    with pytest.raises(ValueError, match="^beta must be >= 0"):
        per_scalars(beta=-1e-3)
    with pytest.raises(ValueError, match="^alpha must be a finite number"):
        per_scalars(alpha=math.inf)
    with pytest.raises(ValueError, match="^eps=1e\\+39 must be finite in float32"):
        per_scalars(eps=1e39)
    with pytest.raises(ValueError, match="rounds to 0.5 in float32, where torch's pow takes a special path"):
        per_scalars(beta=0.5 + 1e-12)
    with pytest.raises(ValueError, match="rounds to 2.0 in float32"):
        per_scalars(alpha=2 - 1e-12)
    assert per_scalars(eps=1 + 1e-12) == (1.0,)   # eps is no exponent


# ---- the C ABI --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("entry,names", [
    ("ktb_per_sample_f32", ["dev", "priorities", "C", "batch", "j0", "rows", "seed", "beta", "tree", "indices",
                            "weights", "stream"]),
    ("ktb_per_update_f32", ["dev", "priorities", "C", "indices", "td", "B", "alpha", "eps", "stream"]),
])
def test_ctypes_prototype_matches_the_header(entry, names):
    text = open(HEADER).read()
    m = re.search(rf"\bint {entry}\(([^)]*)\);", text)
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    assert [p.split()[-1].lstrip("*") for p in params] == names
    restype, argtypes = L._SIGNATURES[entry]
    assert restype is ctypes.c_int and len(argtypes) == len(params)
    for p, t in zip(params, argtypes):
        want = ctypes.c_void_p if "*" in p else {"int": ctypes.c_int, "size_t": ctypes.c_size_t, "float": ctypes.c_float,
                                                  "uint64_t": ctypes.c_uint64, "uintptr_t": L.c_uintptr}[p.split()[0]]
        assert t is want, (p, t)


def test_an_unregistered_device_comes_first():
    lib = L.load()
    assert lib.ktb_per_sample_f32(15, 0, 0, 0, 0, 0, 0, math.nan, 0, 0, 0, 0) == L.ERR_STATE
    assert lib.ktb_per_update_f32(15, 0, 0, 0, 0, 0, math.nan, math.nan, 0) == L.ERR_STATE
