"""User callables of prioritized experience replay's proportional sampler (Schaul et al. 2016: Ape-X, R2D2, Rainbow),
written as a kubetorch user writes SPMD functions: rank r draws its strata `torch.arange(batch).chunk(WORLD_SIZE)[RANK]`
of one stratified batch from the priorities of a replay buffer.

TEST INFRASTRUCTURE.  per_sample() is the semantic definition of @kt.mapped("per", batch=..., beta=..., seed=...): the
sampler is stateless, so each call builds the sum tree of the priorities (the stored p_i^α, as OpenAI baselines stores
them) and draws from it.  Every node is ONE fp32 add of its two children over the leaves padded with +0 to a power of
two; stratum j descends from the mass (j + u_j)·(total / batch), u_j = kubetorch_b200.sampling.replay_noise(seed, j, 1),
stepping right where mass >= left and the right child holds mass (> 0), so no subtree of zero mass is ever entered and
every index lies in [0, C) whatever the priorities hold.  The importance weights are (C·p_i / total)^-β over the largest
one, (C·min p / total)^-β.  per_update() is the definition of kubetorch_b200.device.replay.per_update: the new
priorities (|td| + eps)^α, a repeated index taking its last occurrence.  include/ktb200.h restates the draw as fp32
operations (header_per_sample below), and the CUDA path must reproduce its bits.
"""
import os

import numpy as np

from kubetorch_b200.sampling import gumbel_uniform, replay_noise

BATCH, BETA = 512, 0.4


def sum_tree(priorities):
    """The levels of the sum tree, leaves first: each level is one fp32 add of the pairs of the level below."""
    import torch

    c = priorities.numel()
    p = 1 << (c - 1).bit_length()   # leaves padded with +0 to a power of two
    lv = torch.zeros(p, dtype=torch.float32, device=priorities.device)
    lv[:c] = priorities
    levels = [lv]
    while levels[-1].numel() > 1:
        levels.append(levels[-1][0::2] + levels[-1][1::2])
    return levels


def descend(levels, mass, strict=False):
    """The leaf each mass lands on, from the root down; `strict` is the wrong rule mass > left."""
    import torch

    node = torch.zeros(mass.shape, dtype=torch.int64, device=mass.device)
    for lv in reversed(levels[:-1]):
        left, right = lv[2 * node], lv[2 * node + 1]
        go = ((mass > left) if strict else (mass >= left)) & (right > 0)   # never enter a subtree of zero mass
        mass = torch.where(go, mass - left, mass)
        node = 2 * node + go.long()
    return node


def importance_weights(priorities, node, total, beta, normalise=True):
    c = priorities.numel()
    w = (priorities[node] / total * c) ** -beta
    return w / (priorities.min() / total * c) ** -beta if normalise else w


def per_sample(priorities, seed, batch, beta, j0=0, rows=None):
    """(int64 indices, fp32 weights) of strata j0 .. j0 + rows - 1 of `batch`."""
    import torch

    rows = batch - j0 if rows is None else rows
    levels = sum_tree(priorities)
    total = levels[-1]
    j = torch.arange(j0, j0 + rows, device=priorities.device)
    u = replay_noise(seed, j0, rows, priorities.device)
    mass = (j.to(torch.float32) + u) * (total / batch)
    node = descend(levels, mass)
    return node, importance_weights(priorities, node, total, beta)


def per_update(priorities, indices, td, alpha, eps):
    """In place; a repeated index takes its LAST occurrence."""
    import torch

    new = (td.abs() + eps) ** alpha
    pos = torch.arange(len(indices), device=td.device)
    last = torch.full_like(priorities, -1, dtype=torch.int64).scatter_reduce_(0, indices, pos, "amax")
    keep = last[indices] == pos
    priorities[indices[keep]] = new[keep]


def strata(batch):
    """(j0, rows): this rank's strata torch.arange(batch).chunk(WORLD_SIZE)[RANK] (none for ranks past them)."""
    r, w = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    chunk = -(-batch // w)
    j0 = min(batch, chunk * r)
    return j0, min(batch, j0 + chunk) - j0


def mapped_per(priorities, seed):
    """@kt.mapped("per", batch=BATCH, beta=BETA, seed="seed")."""
    return per_sample(priorities, seed, BATCH, BETA, *strata(BATCH))


def mapped_per_beta(priorities, seed, beta):
    """β as a call argument: @kt.mapped("per", batch=BATCH, beta="beta", seed="seed")."""
    return per_sample(priorities, seed, BATCH, beta, *strata(BATCH))


def mapped_per_seeded(priorities):
    """A constant seed: @kt.mapped("per", batch=BATCH, beta=BETA, seed=7)."""
    return per_sample(priorities, 7, BATCH, BETA, *strata(BATCH))


def _wrong(priorities, seed, mass_of=None, strict=False, normalise=True):
    import torch

    j0, rows = strata(BATCH)
    levels = sum_tree(priorities)
    total = levels[-1]
    j = torch.arange(j0, j0 + rows, device=priorities.device)
    mass = mass_of(j, total) if mass_of else (j.to(torch.float32) + replay_noise(seed, j0, rows, j.device)) * (
        total / BATCH)
    node = descend(levels, mass, strict)
    return node, importance_weights(priorities, node, total, BETA, normalise)


def mapped_per_uniform(priorities, seed):
    """Uniform draws over the whole total, not one per stratum: not the op's body."""
    return _wrong(priorities, seed, lambda j, total: replay_noise(seed, int(j[0]) if len(j) else 0, len(j), j.device)
                  * total)


def mapped_per_local(priorities, seed):
    """Strata numbered from 0 on every rank, not by their global j: not the op's body."""
    import torch

    return _wrong(priorities, seed, lambda j, total: (torch.arange(len(j), device=j.device).float()
                                                      + replay_noise(seed, 0, len(j), j.device)) * (total / BATCH))


def mapped_per_strict(priorities, seed):
    """mass > left in place of mass >= left: not the op's body."""
    return _wrong(priorities, seed, strict=True)


def mapped_per_unnormalised(priorities, seed):
    """Weights not divided by the largest weight: not the op's body."""
    return _wrong(priorities, seed, normalise=False)


def mapped_per_other_stream(priorities, seed):
    """The Gumbel stream's uniforms (counter word 3 = 0) in place of the replay stream's: not the op's body."""
    return _wrong(priorities, seed, lambda j, total: (
        j.float() + gumbel_uniform(seed, int(j[0]) if len(j) else 0, len(j), 1, j.device)[:, 0]) * (total / BATCH))


def header_per_sample(priorities, seed, batch, beta, j0=0, rows=None):
    """include/ktb200.h's restatement in numpy fp32, one rounding per operation: (tree, indices, weights) as numpy
    arrays, tree in the header's layout (min, total, internal nodes 2 .. P - 1).  pw is torch's pow on the device of
    priorities (CUDA's on a GPU), so only the arithmetic around it is restated here."""
    import torch

    f = np.float32
    rows = batch - j0 if rows is None else rows
    p = priorities.cpu().numpy().astype(f)
    c = p.size
    n_leaves = 1 << (c - 1).bit_length()
    heap = np.zeros(2 * n_leaves, dtype=f)   # heap[n] is node n; leaves at n_leaves ..
    heap[n_leaves:n_leaves + c] = p
    with np.errstate(all="ignore"):
        k = n_leaves
        while k > 1:
            heap[k // 2:k] = heap[k:2 * k:2] + heap[k + 1:2 * k:2]
            k //= 2
        tree = np.zeros(max(n_leaves, 2), dtype=f)
        tree[1:n_leaves] = heap[1:n_leaves]
        tree[1] = heap[1]
        tree[0] = p.min()
        total = heap[1]
        u = replay_noise(seed, j0, rows).numpy()
        mass = (np.arange(j0, j0 + rows).astype(f) + u) * (total * (f(1) / f(batch)))
        n = np.ones(rows, dtype=np.int64)
        for _ in range(n_leaves.bit_length() - 1):
            left, right = heap[2 * n], heap[2 * n + 1]
            go = (mass >= left) & (right > f(0))
            mass = np.where(go, mass - left, mass).astype(f)
            n = 2 * n + go
        idx = n - n_leaves

        def pw(x):
            return (torch.from_numpy(np.ascontiguousarray(x, dtype=f)).to(priorities.device) ** -beta).cpu().numpy()

        weights = pw(p[idx] / total * f(c)) / pw(np.array([tree[0] / total * f(c)], dtype=f))
    return tree, idx, weights.astype(f)
