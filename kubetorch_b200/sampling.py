"""The Gumbel noise of @kt.mapped("mlp", output="sample"), the Gaussian noise of output="gaussian", the exploration
draws of output="epsilon_greedy" and the stratum offsets of @kt.mapped("per"), in plain torch (no GPU, no library).

A sampled policy body adds ``gumbel_noise(seed, row0, rows, d_out)`` to its fp32 logits, takes the argmax and gathers
the log_softmax; a Gaussian policy body adds ``exp(log_std)·normal_noise(seed, row0, rows, d_out)`` to its mean; an
ε-greedy body takes ``u, w = explore_noise(seed, row0, rows, d_out)``, explores where ``u < ε`` and then takes the
legal column with the largest word ``w``.  The device kernel draws the very same numbers in its head epilogue
(include/ktb200.h).  For global row i (the row's index in the whole observation batch) and column j:

    x = Philox4x32-10(counter = (i mod 2^32, i >> 32, j >> 1, s), key = (seed mod 2^32, seed >> 32)), word j & 1
    u = (2·(x >> 9) + 1)·2^-24          exact in fp32, strictly inside (0, 1), never 0.5

    stream  s   use
    Gumbel  0   g = -log(-log(u)) in fp32, added to the logits of output="sample"
    Gaussian 1  z = Φ⁻¹(u) in fp32, within ±5.29471 and never 0, the noise of output="gaussian" (and of
                "deterministic", scaled by σ and clipped)
    explore 2   the word x itself (a uint32): ranks the legal columns of an exploring row of output="epsilon_greedy"
    coin    3   u of column 0 only (one draw per row): the row explores iff u < ε in fp32
    replay  4   u of column 0 only, with i the global stratum of a prioritized replay batch (replay_noise): the
                stratum's draw lands at mass (i + u)·(total / batch) of the sum tree

The noise depends on (seed, i, j) only, so every sharding of the rows draws the same noise for the same row.
"""
from __future__ import annotations

import torch

_M0, _M1 = 0xD2511F53, 0xCD9E8D57
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_U32 = 0xFFFFFFFF


def _mul_hi_lo(m: int, x: torch.Tensor):
    """(m·x >> 32, m·x mod 2^32) for a 32-bit constant m and int64 x < 2^32: x in 16-bit limbs, each product < 2^48."""
    t = m * (x & 0xFFFF)
    u = m * (x >> 16)
    hi = (u + (t >> 16)) >> 16
    lo = (t + ((u & 0xFFFF) << 16)) & _U32
    return hi, lo


def philox4x32_10(counter: torch.Tensor, key: torch.Tensor) -> torch.Tensor:
    """Philox4x32-10 (Random123) on int64 tensors of 32-bit words: counter [..., 4] and key [..., 2] (broadcast
    against each other) give the four output words [..., 4]."""
    c = [counter[..., q].to(torch.int64) for q in range(4)]
    k0, k1 = key[..., 0].to(torch.int64), key[..., 1].to(torch.int64)
    for _ in range(10):
        hi0, lo0 = _mul_hi_lo(_M0, c[0])
        hi1, lo1 = _mul_hi_lo(_M1, c[2])
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0, k1 = (k0 + _W0) & _U32, (k1 + _W1) & _U32
    return torch.stack(torch.broadcast_tensors(*c), dim=-1)


def _check_seed(seed) -> int:
    if isinstance(seed, bool) or not isinstance(seed, int) or not 0 <= seed < 1 << 64:
        raise ValueError(f"seed must be an int in [0, 2**64), got {seed!r}")
    return seed


def random_words(seed: int, row_offset: int, rows: int, cols: int, device="cpu", word3: int = 0) -> torch.Tensor:
    """int64 [rows, cols]: the 32-bit Philox word of global row row_offset + r and column j.  `word3` is the fourth
    counter word: 0 for the Gumbel noise, 1 for the Gaussian noise, 2 for the exploration words, 3 for the coin, 4 for
    the replay strata."""
    seed = _check_seed(seed)
    if row_offset < 0 or rows < 0 or cols < 0:
        raise ValueError("row_offset, rows and cols must be non-negative")
    if isinstance(word3, bool) or not isinstance(word3, int) or not 0 <= word3 <= _U32:
        raise ValueError(f"word3 must be an int in [0, 2**32), got {word3!r}")
    i = torch.arange(rows, dtype=torch.int64, device=device) + int(row_offset)
    pairs = torch.arange((cols + 1) // 2, dtype=torch.int64, device=device)
    counter = torch.stack(torch.broadcast_tensors(i[:, None] & _U32, i[:, None] >> 32, pairs[None, :],
                                                  torch.full_like(pairs, word3)[None, :]), dim=-1)
    key = torch.tensor([seed & _U32, seed >> 32], dtype=torch.int64, device=device)
    x = philox4x32_10(counter, key)                       # [rows, pairs, 4]: words 0 and 1 serve columns 2p, 2p + 1
    return x[..., :2].reshape(rows, 2 * pairs.numel())[:, :cols]


def gumbel_uniform(seed: int, row_offset: int, rows: int, cols: int, device="cpu", word3: int = 0) -> torch.Tensor:
    """float32 [rows, cols]: u = (2·(x >> 9) + 1)·2^-24, exact and strictly inside (0, 1)."""
    x = random_words(seed, row_offset, rows, cols, device, word3=word3)
    return (2 * (x >> 9) + 1).to(torch.float32) * 2.0 ** -24


def normal_noise(seed: int, row_offset: int, rows: int, cols: int, device="cpu") -> torch.Tensor:
    """float32 [rows, cols]: the Gaussian noise z = Φ⁻¹(u) of global rows row_offset .. row_offset + rows - 1, where u
    is the exact uniform of the Philox words with counter word 3 = 1 (never the Gumbel stream's).  Computed as fp64
    ndtri of the exact u rounded to fp32; the device's fp32 normcdfinvf is within 2^-20·(1 + |z|) of it.  u is never
    0.5, so z is never 0; |z| <= 5.29471, the probability mass beyond (about 1.2e-7) is never drawn."""
    u = gumbel_uniform(seed, row_offset, rows, cols, device, word3=1)
    return torch.special.ndtri(u.double()).to(torch.float32)


def gumbel_noise(seed: int, row_offset: int, rows: int, cols: int, device="cpu") -> torch.Tensor:
    """float32 [rows, cols]: the Gumbel noise g = -log(-log(u)) of global rows row_offset .. row_offset + rows - 1."""
    u = gumbel_uniform(seed, row_offset, rows, cols, device)
    return -torch.log(-torch.log(u))


def explore_noise(seed: int, row_offset: int, rows: int, cols: int, device="cpu"):
    """(u, words) of output="epsilon_greedy" for global rows row_offset .. row_offset + rows - 1: u float32 [rows], the
    exact uniform of word 0 of counter (i, 0, 3) (a row explores iff u < ε in fp32), and words int64 [rows, cols], the
    uint32 Philox word j & 1 of counter (i, j >> 1, 2) (an exploring row takes the legal column with the largest word,
    ties to the lower column).  Neither stream reuses the Gumbel (0) or Gaussian (1) draws of the same seed."""
    u = gumbel_uniform(seed, row_offset, rows, 1, device, word3=3)[:, 0]
    return u, random_words(seed, row_offset, rows, cols, device, word3=2)


def replay_noise(seed: int, row0: int, rows: int, device="cpu") -> torch.Tensor:
    """float32 [rows]: the offsets u of strata row0 .. row0 + rows - 1 of @kt.mapped("per"), the exact uniform of word 0
    of counter (j, 0, 4), strictly inside (0, 1).  Stratum j draws at mass (j + u)·(total / batch) of the sum tree.  The
    stream reuses none of the Gumbel (0), Gaussian (1), exploration (2) or coin (3) draws of the same seed."""
    return gumbel_uniform(seed, row0, rows, 1, device, word3=4)[:, 0]
