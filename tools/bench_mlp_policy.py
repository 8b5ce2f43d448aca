#!/usr/bin/env python
"""The nn.Linear policy form of the bf16 MLP on one GPU, at the scale of BASELINE config C4: 4096 x 512 observation
rows through 256 -> 1024 -> 1024 -> d_out, device-resident on cuda:0.

Variants, timed alternately (one sample = the mean of --calls back-to-back calls between CUDA events; the median of
--samples samples is reported):
  a  the C entry ktb_mlp_bf16 (no bias, d_out 64, logits), called directly
  b  the C entry ktb_mlp_bf16_policy, no bias, d_out 64, logits (its logits must equal a's bit for bit)
  c  mlp_forward (ktb_mlp_bf16_policy) with biases, d_out 64, logits
  d  policy with biases, d_out 64, actions only
  e  policy with biases, d_out 64, logits and actions
  f  policy with biases, d_out 18 and d_out 256, logits and actions
  g  policy with biases, d_out 18, 64 and 256, sampled actions and log-probabilities (output="sample"), timed in the
     same alternation as d (actions only), which has the same GEMMs and no noise
  h  policy with biases, d_out 6, 18 and 64, Gaussian actions and log-probabilities (output="gaussian", log_std over
     [-2, 0.5]), timed in the same alternation beside the logits-only call and output="sample" at the same d_out
  i  policy with biases, d_out 18, 64 and 256, a random legal-action mask (about 50 % legal): masked actions right
     after the same unmasked call, and masked sampled actions right after the unmasked output="sample" call
  j  policy with biases and a value head (a critic nn.Linear(1024, 1) on the same trunk, value=(wv, bv)), d_out 6, 18,
     63, 64 and 255: output="sample", output="sample" with a random legal-action mask and output="gaussian", each
     right after the same call without a value head; and the eager critic, what a user pays without the fused value:
     the unfused output="sample" call plus the trunk and the value head recomputed with F.linear in torch
  k  multi-discrete heads (nvec=), nvec (3,)*6, (2,)*32, (6, 4, 4, 4, 4, 7, 49) and (2,)*128 (d_out 18, 64, 78 and
     256): greedy actions and output="sample", each unmasked and under a random legal-action mask, each beside the
     single-categorical call of the same d_out and output; and the eager arm, what a user pays without the grouped
     head: the logits entry (masked in torch under a mask), then split, Gumbel noise, argmax and log_softmax in torch.
     (2,)*128 shows the cost of 128 per-group quad reductions.
  l  state-dependent Gaussian heads (log_std=(w_ls, b_ls), SAC's actor), d_out 6, 17, 64 and 128, unsquashed and
     squashed (squash=True), each beside output="gaussian" at the same d_out; and the eager arm, what a user pays
     without the fused head: the logits entry over the stacked head [w3; w_ls], then clamp, exp, noise, tanh and the
     log-density in torch.  The interleaved head doubles the head's columns: d_out 64 runs in the 128-wide tile and 128
     in the 256-wide one.
  m  ε-greedy Q-network heads (output="epsilon_greedy"), d_out 6, 18 and 64, ε 0.01, 0.05 and 1.0 (the worst case:
     every row draws a Philox call per column pair), unmasked and under a random legal-action mask, each beside
     output="actions" and output="sample" at the same d_out and mask; and the eager arm, what a user pays without the
     fused head: the logits entry (masked in torch under a mask), then argmax, the exploration draws of explore_noise,
     where and two gathers in torch.
  n  evaluating given actions (output="evaluate" and "gaussian_evaluate"): the categorical head at d_out 18, 64 and
     256, the masked MicroRTS nvec (6, 4, 4, 4, 4, 7, 49) with a value head, and the Gaussian head at d_out 6 and 17,
     each scoring the actions of the matching sampling call and timed beside it; and the eager arm, what a user pays
     without the evaluating head: the logits entry, then mask, split, log_softmax, gather, softmax and entr (or
     Normal.log_prob and entropy) in torch.
  o  deterministic actors (output="deterministic", DDPG's and TD3's), d_out 6, 17 and 64: the noise-free squashed
     actor beside output="logits", exploration (σ = 0.1) beside output="gaussian", and TD3's target policy smoothing
     (σ = 0.2, noise_clip = 0.5), at the same d_out; and the eager arm, what a user pays without the fused head: the
     logits entry, then tanh, normal_noise on the device and the two clamps in torch.
  p  Q(s, a) critics (output="critic", SAC's and TD3's), the C4 trunk with the actions fed into layer 1 (256 + d_act ->
     1024 -> 1024 -> 1), d_act 6, 17 and 64, single and twin, each beside output="logits" at d_out 1 on the same
     observations (the difference is the action block and the head); and the eager twin, what a user pays without
     the feature: torch.cat of the rows and the bf16 actions padded to d_in + 64, w1 padded likewise, the logits entry
     per critic, .float() and torch.minimum.
  q  TD targets (output="td_target") over the twin critics of p and a 256 -> 1024 -> 1024 -> d_act actor, d_act 6, 17
     and 64: TD3's (σ 0.2, clip 0.5) and SAC's (squashed, α 0.2), each beside the two-call arm (the actor entry, the
     twin critic entry, then reward + 0.99 * (1 - done) * t in eager torch) and the eager arm (the logits entries, the
     actor's head, the padded concatenation and the minimum in torch).  Before timing, the fused y equals the two-call
     arm's bit for bit on every row, and is within rtol 2^-7, atol 1e-2 of the eager arm's on at least 99 % of the rows
     (the eager arm's tanh and log rounding move some bf16 actions by an ulp).
  r  DQN targets (output="dqn_target") over the C4 trunk, d_out 6, 18 and 64 and d_out 18 under a random legal-action
     mask, DQN (the target network selects) and Double DQN (an online network of its own selects), each beside the
     two-call arm (output="actions" on the selector, output="logits" on the target, then the gather and reward + 0.99 *
     (1 - done) * q in eager torch) and the eager arm (the logits entry on each network, then the mask, argmax, gather
     and the target in torch).  Before timing, the fused y equals both arms' bit for bit on every row.
Parity: 2048 sampled rows against an fp32 evaluation (rtol 2^-7, atol 1e-2; actions wherever the fp32 top-2 gap
exceeds 2^-6), and the actions equal torch.argmax of the kernel's logits on every row.  Sampled rows: on 2048
consecutive rows, the action is the argmax of the kernel's logits plus the fp64 Gumbel noise wherever the top-2 gap
exceeds 2^-18·(1 + max|s|), and the log-probability is within (d_out + 8)·2^-22·(1 + |ref|) of the fp64 log_softmax.
Masked rows: the masked actions equal torch.argmax of the kernel's logits filled with -inf on every row, and every
sampled action on a row with a legal action is legal.  Value rows: every valued call's actions and log-probabilities
equal those of the same call without a value head on every row, bit for bit, the masked call's values equal the
unmasked call's, and the values are within rtol 2^-7, atol 1e-2 of the eager critic's.  Multi-discrete rows: the
greedy actions equal the per-group argmax of the kernel's (masked) logits on every row; the sampled actions equal the
eager arm's on at least 99.9 % of the rows (its noise comes from torch's log, not the kernel's logf), its
log-probabilities within 2^-16·(1 + |ref|) on those rows, and every masked sample in a group with a legal action is
legal.  State-dependent rows: on 2048 consecutive rows, the unsquashed actions are within 2^-19·σ·(1 + |z|) +
2^-23·|μ| of μ + σ·z (μ and ℓ the kernel's logits over the interleaved head, σ = exp(clamp(ℓ))), the squashed actions
within 2 ulp of tanh of the unsquashed ones, and on every row both the actions and log-probabilities are within rtol
1e-4, atol 1e-4 of the eager arm's.  ε-greedy rows: actions, q and q_max equal the eager arm's on every row, bit for
bit.  Evaluating rows: the categorical log-probabilities of the sampled actions equal the sampling call's on every row,
bit for bit (NaN in the same rows), its values too; log-probabilities and entropies are within rtol 1e-4, atol 1e-4 of
the eager arm's (the Gaussian's log-probabilities within rtol 1e-4, atol 1e-3 of the sampling call's), and the values
within rtol 2^-7, atol 1e-2 of the eager critic's.  Deterministic rows: on 2048 consecutive rows, the noise-free
actions are within tanhf's 2 ulp of fp64 tanh(y) (y the kernel's logits) and the noisy ones within
σ·2^-19·(1 + |z|) + 2^-22·|t| + 2^-23·(|t| + |n|) of clamp(tanh(y) + clamp(σ·z, ±c), ±1) in fp64; on every row
the smoothing actions are within rtol 1e-5, atol 1e-5 of the eager arm's.  Critic rows: q equals the logits entry
over [obs | bf16(act) | 0] and the padded w1 on every row, bit for bit; the twin's q1 and q2 equal the single critics'
and its q_min the eager arm's torch.minimum (bit for bit off ties of signed zeros); q is within rtol 2^-7, atol 1e-2 of
an fp32 evaluation on 2048 rows.  Gaussian rows: on 2048 consecutive rows, the actions are within 2^-19·σ·(1 + |z|) + 2^-23·|y| of y + σ·z (y the
kernel's logits, σ and z = ndtri(u) in fp64) and the log-probabilities within the bar of tests/test_gpu_mlp_gaussian.py.
The card name and its power limit are read in the same run.  Prints one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from kubetorch_b200.device import lib as L  # noqa: E402
from kubetorch_b200.device import mlp  # noqa: E402
from kubetorch_b200.device import ops  # noqa: E402
from kubetorch_b200.sampling import explore_noise, gumbel_noise, gumbel_uniform, normal_noise  # noqa: E402

HALF_LOG_2PI = 0.9189385332046727
LN2 = 0.6931471805599453

SEED = 0x5EED


def _power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:  # noqa: BLE001
        return None


def _fp32(obs, w, b):
    h = obs.float() @ w[0].float().t()
    h = torch.relu(h + b[0].float() if b[0] is not None else h).bfloat16()
    h2 = h.float() @ w[1].float().t()
    h = torch.relu(h2 + b[1].float() if b[1] is not None else h2).bfloat16()
    y = h.float() @ w[2].float().t()
    return y + b[2].float() if b[2] is not None else y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=7)
    ap.add_argument("--calls", type=int, default=3)
    args = ap.parse_args()
    L.load()
    ops.ensure_init([0])
    M, d_in, d_hidden = 4096 * 512, 256, 1024
    g = torch.Generator(device="cuda:0").manual_seed(0)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, device="cuda:0", generator=g) * scale).bfloat16()   # noqa: E731
    obs = rnd(M, d_in)
    w1, w2 = rnd(d_hidden, d_in, scale=0.02), rnd(d_hidden, d_hidden, scale=0.02)
    b1, b2 = rnd(d_hidden, scale=0.1), rnd(d_hidden, scale=0.1)
    heads = {d: (rnd(d, d_hidden, scale=0.02), rnd(d, scale=0.1)) for d in (18, 64, 256)}
    scratch = mlp._scratch_for(0, M, d_hidden)
    stream = int(torch.cuda.current_stream(0).cuda_stream)

    def original_a(out):
        L.call("ktb_mlp_bf16", 0, obs.data_ptr(), M, d_in, d_hidden, 64, w1.data_ptr(), w2.data_ptr(),
               heads[64][0].data_ptr(), out.data_ptr(), scratch.data_ptr(), stream)
        return out

    def policy_b(out):
        L.call("ktb_mlp_bf16_policy", 0, obs.data_ptr(), M, d_in, d_hidden, 64, w1.data_ptr(), 0, w2.data_ptr(), 0,
               heads[64][0].data_ptr(), 0, out.data_ptr(), 0, scratch.data_ptr(), 0, stream)
        return out

    parity = {}
    out_a = torch.empty(M, 64, dtype=torch.bfloat16, device="cuda:0")
    out_b = torch.empty(M, 64, dtype=torch.bfloat16, device="cuda:0")
    variants = {
        "a_original_d64": (64, lambda: original_a(out_a)),
        "b_policy_nobias_d64": (64, lambda: policy_b(out_b)),
        "c_bias_logits_d64": (64, lambda: mlp.mlp_forward(obs, w1, w2, heads[64][0], biases=(b1, b2, heads[64][1]))),
        "d_bias_actions_d64": (64, lambda: mlp.mlp_forward(obs, w1, w2, heads[64][0], biases=(b1, b2, heads[64][1]),
                                                           output="actions")),
        "e_bias_both_d64": (64, lambda: mlp.mlp_forward(obs, w1, w2, heads[64][0], biases=(b1, b2, heads[64][1]),
                                                        output="both")),
        "f_bias_both_d18": (18, lambda: mlp.mlp_forward(obs, w1, w2, heads[18][0], biases=(b1, b2, heads[18][1]),
                                                        output="both")),
        "f_bias_both_d256": (256, lambda: mlp.mlp_forward(obs, w1, w2, heads[256][0], biases=(b1, b2, heads[256][1]),
                                                          output="both")),
    }
    for d in (18, 64, 256):
        variants[f"g_bias_sample_d{d}"] = (d, lambda d=d: mlp.mlp_forward(
            obs, w1, w2, heads[d][0], biases=(b1, b2, heads[d][1]), output="sample", seed=SEED))
    g6 = torch.Generator(device="cuda:0").manual_seed(6)   # its own generator: the other heads and rows stay as they were
    heads[6] = ((torch.randn(6, d_hidden, device="cuda:0", generator=g6) * 0.02).bfloat16(),
                (torch.randn(6, device="cuda:0", generator=g6) * 0.1).bfloat16())
    log_stds = {d: torch.linspace(-2.0, 0.5, d, device="cuda:0") for d in (6, 18, 64)}
    for d in (6, 18):
        variants[f"h_bias_logits_d{d}"] = (d, lambda d=d: mlp.mlp_forward(obs, w1, w2, heads[d][0],
                                                                          biases=(b1, b2, heads[d][1])))
    variants["h_bias_sample_d6"] = (6, lambda: mlp.mlp_forward(obs, w1, w2, heads[6][0], biases=(b1, b2, heads[6][1]),
                                                               output="sample", seed=SEED))
    for d in (6, 18, 64):
        variants[f"h_bias_gaussian_d{d}"] = (d, lambda d=d: mlp.mlp_forward(
            obs, w1, w2, heads[d][0], biases=(b1, b2, heads[d][1]), output="gaussian", seed=SEED,
            log_std=log_stds[d]))
    gm = torch.Generator(device="cuda:0").manual_seed(7)
    legal = {d: torch.rand(M, d, device="cuda:0", generator=gm) < 0.5 for d in (18, 64, 256)}
    for d in (18, 64, 256):
        bs = (b1, b2, heads[d][1])
        variants[f"i_bias_actions_d{d}"] = (d, lambda d=d, bs=bs: mlp.mlp_forward(
            obs, w1, w2, heads[d][0], biases=bs, output="actions"))
        variants[f"i_bias_masked_actions_d{d}"] = (d, lambda d=d, bs=bs: mlp.mlp_forward(
            obs, w1, w2, heads[d][0], biases=bs, output="actions", mask=legal[d]))
        variants[f"i_bias_sample_d{d}"] = (d, lambda d=d, bs=bs: mlp.mlp_forward(
            obs, w1, w2, heads[d][0], biases=bs, output="sample", seed=SEED))
        variants[f"i_bias_masked_sample_d{d}"] = (d, lambda d=d, bs=bs: mlp.mlp_forward(
            obs, w1, w2, heads[d][0], biases=bs, output="sample", seed=SEED, mask=legal[d]))
    gj = torch.Generator(device="cuda:0").manual_seed(8)   # its own generator again
    for d in (63, 255):
        heads[d] = ((torch.randn(d, d_hidden, device="cuda:0", generator=gj) * 0.02).bfloat16(),
                    (torch.randn(d, device="cuda:0", generator=gj) * 0.1).bfloat16())
    critic = ((torch.randn(1, d_hidden, device="cuda:0", generator=gj) * 0.02).bfloat16(),
              (torch.randn(1, device="cuda:0", generator=gj) * 0.1).bfloat16())
    for d in (6, 18, 63, 64, 255):
        legal.setdefault(d, torch.rand(M, d, device="cuda:0", generator=gj) < 0.5)
        log_stds.setdefault(d, torch.linspace(-2.0, 0.5, d, device="cuda:0"))
    value_widths = (6, 18, 63, 64, 255)
    for d in value_widths:
        bs = (b1, b2, heads[d][1])
        for kind, kw in (("sample", dict(output="sample", seed=SEED)),
                         ("masked_sample", dict(output="sample", seed=SEED, mask=legal[d])),
                         ("gaussian", dict(output="gaussian", seed=SEED, log_std=log_stds[d]))):
            variants[f"j_bias_{kind}_d{d}"] = (d, lambda d=d, bs=bs, kw=kw: mlp.mlp_forward(
                obs, w1, w2, heads[d][0], biases=bs, **kw))
            variants[f"j_bias_{kind}_value_d{d}"] = (d, lambda d=d, bs=bs, kw=kw: mlp.mlp_forward(
                obs, w1, w2, heads[d][0], biases=bs, value=critic, **kw))

        def eager_critic(d=d, bs=bs):
            actions, log_probs = mlp.mlp_forward(obs, w1, w2, heads[d][0], biases=bs, output="sample", seed=SEED)
            h = torch.relu(F.linear(torch.relu(F.linear(obs, w1, b1)), w2, b2))
            return actions, log_probs, F.linear(h, *critic).float().squeeze(-1)

        variants[f"j_bias_eager_critic_d{d}"] = (d, eager_critic)
    gk = torch.Generator(device="cuda:0").manual_seed(9)   # its own generator again
    heads[78] = ((torch.randn(78, d_hidden, device="cuda:0", generator=gk) * 0.02).bfloat16(),
                 (torch.randn(78, device="cuda:0", generator=gk) * 0.1).bfloat16())
    legal[78] = torch.rand(M, 78, device="cuda:0", generator=gk) < 0.5
    nvecs = {18: (3,) * 6, 64: (2,) * 32, 78: (6, 4, 4, 4, 4, 7, 49), 256: (2,) * 128}

    def eager_groups(d, mask, sample):
        """The logits entry, then the grouped head in torch: what a user pays without nvec=."""
        y = mlp.mlp_forward(obs, w1, w2, heads[d][0], biases=(b1, b2, heads[d][1]))
        if mask:
            y = y.masked_fill(~legal[d], float("-inf"))
        y = y.float()
        z = y + gumbel_noise(SEED, 0, M, d, device="cuda:0") if sample else y
        acts = torch.stack([p.argmax(-1) for p in z.split(nvecs[d], -1)], -1)
        if not sample:
            return acts
        lp = None
        for i, p in enumerate(y.split(nvecs[d], -1)):
            t = torch.log_softmax(p, -1).gather(-1, acts[:, i:i + 1]).squeeze(-1)
            lp = t if lp is None else lp + t
        return acts, lp

    for d, nvec in nvecs.items():
        bs = (b1, b2, heads[d][1])
        for mask in (False, True):
            m = dict(mask=legal[d]) if mask else {}
            tag = "masked_" if mask else ""
            for out, kw in (("actions", dict(output="actions")), ("sample", dict(output="sample", seed=SEED))):
                variants[f"k_bias_{tag}{out}_d{d}"] = (d, lambda d=d, bs=bs, kw=kw, m=m: mlp.mlp_forward(
                    obs, w1, w2, heads[d][0], biases=bs, **kw, **m))
                variants[f"k_bias_{tag}{out}_nvec_d{d}"] = (d, lambda d=d, bs=bs, kw=kw, m=m, nvec=nvec: mlp.mlp_forward(
                    obs, w1, w2, heads[d][0], biases=bs, nvec=nvec, **kw, **m))
                variants[f"k_bias_{tag}{out}_eager_d{d}"] = (d, lambda d=d, mask=mask, out=out: eager_groups(
                    d, mask, out == "sample"))
    gl = torch.Generator(device="cuda:0").manual_seed(10)   # its own generator again
    state_widths = (6, 17, 64, 128)
    for d in state_widths:
        if d not in heads:
            heads[d] = ((torch.randn(d, d_hidden, device="cuda:0", generator=gl) * 0.02).bfloat16(),
                        (torch.randn(d, device="cuda:0", generator=gl) * 0.1).bfloat16())
        log_stds.setdefault(d, torch.linspace(-2.0, 0.5, d, device="cuda:0"))
    ls_heads = {d: ((torch.randn(d, d_hidden, device="cuda:0", generator=gl) * 0.02).bfloat16(),
                    torch.linspace(-2.0, 0.5, d, device="cuda:0").bfloat16()) for d in state_widths}
    stacked_ls = {d: (torch.cat((heads[d][0], ls_heads[d][0])), torch.cat((heads[d][1], ls_heads[d][1])))
                  for d in state_widths}

    def eager_state(d, squash):
        """The logits entry over [w3; w_ls], then the state-dependent head in torch: what a user pays without it."""
        y = mlp.mlp_forward(obs, w1, w2, stacked_ls[d][0], biases=(b1, b2, stacked_ls[d][1])).float()
        mu, ls = y[:, :d], y[:, d:].clamp(-20.0, 2.0)
        z = normal_noise(SEED, 0, M, d, device="cuda:0")
        u = mu + torch.exp(ls) * z
        lp = (-0.5 * z * z - ls - HALF_LOG_2PI).sum(-1)
        if not squash:
            return u, lp
        au = u.abs()
        return torch.tanh(u), lp - (2 * (LN2 - au - torch.log1p(torch.exp(-2 * au)))).sum(-1)

    for d in state_widths:
        bs = (b1, b2, heads[d][1])
        variants[f"l_bias_gaussian_d{d}"] = (d, lambda d=d, bs=bs: mlp.mlp_forward(
            obs, w1, w2, heads[d][0], biases=bs, output="gaussian", seed=SEED, log_std=log_stds[d]))
        for squash in (False, True):
            tag = "squashed" if squash else "unsquashed"
            variants[f"l_bias_state_{tag}_d{d}"] = (d, lambda d=d, bs=bs, squash=squash: mlp.mlp_forward(
                obs, w1, w2, heads[d][0], biases=bs, output="gaussian", seed=SEED, log_std=ls_heads[d],
                squash=squash))
            variants[f"l_bias_state_{tag}_eager_d{d}"] = (d, lambda d=d, squash=squash: eager_state(d, squash))
    eps_widths, eps_values = (6, 18, 64), (0.01, 0.05, 1.0)

    def eager_epsilon(d, mask, eps):
        """The logits entry, then the ε-greedy head in torch: what a user pays without output="epsilon_greedy"."""
        q = mlp.mlp_forward(obs, w1, w2, heads[d][0], biases=(b1, b2, heads[d][1]))
        if mask:
            q = q.masked_fill(~legal[d], float("-inf"))
        u, w = explore_noise(SEED, 0, M, d, device="cuda:0")
        greedy = q.argmax(-1)
        explore_a = w.masked_fill(~legal[d], -1).argmax(-1) if mask else w.argmax(-1)
        actions = torch.where(u < eps, explore_a, greedy)
        qf = q.float()
        return actions, qf.gather(1, actions[:, None])[:, 0], qf.gather(1, greedy[:, None])[:, 0]

    for d in eps_widths:
        bs = (b1, b2, heads[d][1])
        for mask in (False, True):
            m = dict(mask=legal[d]) if mask else {}
            tag = "masked_" if mask else ""
            variants[f"m_bias_{tag}actions_d{d}"] = (d, lambda d=d, bs=bs, m=m: mlp.mlp_forward(
                obs, w1, w2, heads[d][0], biases=bs, output="actions", **m))
            variants[f"m_bias_{tag}sample_d{d}"] = (d, lambda d=d, bs=bs, m=m: mlp.mlp_forward(
                obs, w1, w2, heads[d][0], biases=bs, output="sample", seed=SEED, **m))
            for eps in eps_values:
                variants[f"m_bias_{tag}epsilon{eps}_d{d}"] = (d, lambda d=d, bs=bs, m=m, eps=eps: mlp.mlp_forward(
                    obs, w1, w2, heads[d][0], biases=bs, output="epsilon_greedy", seed=SEED, epsilon=eps, **m))
                variants[f"m_bias_{tag}epsilon{eps}_eager_d{d}"] = (
                    d, lambda d=d, mask=mask, eps=eps: eager_epsilon(d, mask, eps))
    def eager_evaluate(d, taken, mask=None, nvec=None, value=None):
        """The logits entry, then the evaluation in torch: what a user pays without output="evaluate"."""
        y = mlp.mlp_forward(obs, w1, w2, heads[d][0], biases=(b1, b2, heads[d][1]))
        if mask is not None:
            y = y.masked_fill(~mask, float("-inf"))
        parts = y.float().split(list(nvec or (d,)), -1)
        a = taken if nvec else taken[:, None]
        lp = sum(q.log_softmax(-1).gather(-1, a[:, g:g + 1])[:, 0] for g, q in enumerate(parts))
        ent = sum(torch.special.entr(q.softmax(-1)).sum(-1) for q in parts)
        if value is None:
            return lp, ent
        h = torch.relu(F.linear(torch.relu(F.linear(obs, w1, b1)), w2, b2))
        return lp, ent, F.linear(h, *value).float().squeeze(-1)

    def eager_gaussian_evaluate(d, taken):
        mu = mlp.mlp_forward(obs, w1, w2, heads[d][0], biases=(b1, b2, heads[d][1])).float()
        dist = torch.distributions.Normal(mu, log_stds[d].exp())
        return dist.log_prob(taken).sum(-1), dist.entropy().sum(-1)

    evaluate_cases = {}
    for d in (18, 64, 256):
        bs = (b1, b2, heads[d][1])
        taken = mlp.mlp_forward(obs, w1, w2, heads[d][0], biases=bs, output="sample", seed=SEED)[0]
        evaluate_cases[f"d{d}"] = (d, "sample", dict(output="sample", seed=SEED),
                                   dict(output="evaluate", taken=taken), lambda d=d, t=taken: eager_evaluate(d, t))
    nv = nvecs[78]
    kw78 = dict(mask=legal[78], nvec=nv, value=critic)
    taken = mlp.mlp_forward(obs, w1, w2, heads[78][0], biases=(b1, b2, heads[78][1]), output="sample", seed=SEED,
                            **kw78)[0]
    evaluate_cases["masked_nvec_value_d78"] = (78, "sample", dict(output="sample", seed=SEED, **kw78),
                                               dict(output="evaluate", taken=taken, **kw78),
                                               lambda t=taken: eager_evaluate(78, t, legal[78], nv, critic))
    for d in (6, 17):
        log_stds.setdefault(d, torch.linspace(-2.0, 0.5, d, device="cuda:0"))
        bs = (b1, b2, heads[d][1])
        taken = mlp.mlp_forward(obs, w1, w2, heads[d][0], biases=bs, output="gaussian", seed=SEED,
                                log_std=log_stds[d])[0]
        evaluate_cases[f"gaussian_d{d}"] = (d, "gaussian", dict(output="gaussian", seed=SEED, log_std=log_stds[d]),
                                            dict(output="gaussian_evaluate", taken=taken, log_std=log_stds[d]),
                                            lambda d=d, t=taken: eager_gaussian_evaluate(d, t))
    for tag, (d, sampled, kw_s, kw_e, eager) in evaluate_cases.items():
        bs = (b1, b2, heads[d][1])
        variants[f"n_bias_{sampled}_{tag}"] = (d, lambda d=d, bs=bs, kw=kw_s: mlp.mlp_forward(
            obs, w1, w2, heads[d][0], biases=bs, **kw))
        variants[f"n_bias_evaluate_{tag}"] = (d, lambda d=d, bs=bs, kw=kw_e: mlp.mlp_forward(
            obs, w1, w2, heads[d][0], biases=bs, **kw))
        variants[f"n_bias_evaluate_eager_{tag}"] = (d, eager)
    det_opts = {"deterministic": {}, "explore": dict(noise=0.1, seed=SEED),
                "smooth": dict(noise=0.2, noise_clip=0.5, seed=SEED)}

    def eager_deterministic(d, noise=0.2, clip=0.5):
        """The logits entry, then tanh, the noise and the clamps in torch: what a user pays without the fused head."""
        y = mlp.mlp_forward(obs, w1, w2, heads[d][0], biases=(b1, b2, heads[d][1]))
        z = normal_noise(SEED, 0, M, d, device="cuda:0")
        return (y.float().tanh() + (noise * z).clamp(-clip, clip)).clamp(-1.0, 1.0)

    for d in (6, 17, 64):
        bs = (b1, b2, heads[d][1])
        log_stds.setdefault(d, torch.linspace(-2.0, 0.5, d, device="cuda:0"))
        variants[f"o_bias_logits_d{d}"] = (d, lambda d=d, bs=bs: mlp.mlp_forward(obs, w1, w2, heads[d][0], biases=bs))
        variants[f"o_bias_gaussian_d{d}"] = (d, lambda d=d, bs=bs: mlp.mlp_forward(
            obs, w1, w2, heads[d][0], biases=bs, output="gaussian", seed=SEED, log_std=log_stds[d]))
        for tag, kw in det_opts.items():
            variants[f"o_bias_{tag}_d{d}"] = (d, lambda d=d, bs=bs, kw=kw: mlp.mlp_forward(
                obs, w1, w2, heads[d][0], biases=bs, output="deterministic", **kw))
        variants[f"o_bias_smooth_eager_d{d}"] = (d, lambda d=d: eager_deterministic(d))
    gp = torch.Generator(device="cuda:0").manual_seed(12)   # its own generator again
    critic_widths = (6, 17, 64)
    critic_acts = {a: torch.rand(M, a, device="cuda:0", generator=gp) * 2 - 1 for a in critic_widths}
    critics = {(a, i): ((torch.randn(d_hidden, d_in + a, device="cuda:0", generator=gp) * 0.02).bfloat16(),
                        (torch.randn(d_hidden, device="cuda:0", generator=gp) * 0.1).bfloat16(),
                        (torch.randn(d_hidden, d_hidden, device="cuda:0", generator=gp) * 0.02).bfloat16(),
                        (torch.randn(d_hidden, device="cuda:0", generator=gp) * 0.1).bfloat16(),
                        (torch.randn(1, d_hidden, device="cuda:0", generator=gp) * 0.02).bfloat16(),
                        (torch.randn(1, device="cuda:0", generator=gp) * 0.1).bfloat16())
               for a in critic_widths for i in (0, 1)}

    def critic_call(a, twin):
        c = critics[(a, 0)]
        return mlp.mlp_forward(obs, c[0], c[2], c[4], biases=(c[1], c[3], c[5]), output="critic",
                               action=critic_acts[a], twin=critics[(a, 1)] if twin else None)

    def eager_twin(a):
        """torch.cat and padding, the logits entry per critic, .float() and torch.minimum: what a user pays without
        output="critic"."""
        x = torch.cat([obs, critic_acts[a].to(torch.bfloat16), obs.new_zeros(M, 64 - a)], -1)
        qs = []
        for i in (0, 1):
            c = critics[(a, i)]
            qs.append(mlp.mlp_forward(x, F.pad(c[0], (0, 64 - a)), c[2], c[4], biases=(c[1], c[3], c[5])).float()
                      .squeeze(-1))
        return qs[0], qs[1], torch.minimum(qs[0], qs[1])

    for a in critic_widths:
        c = critics[(a, 0)]
        w1_obs = c[0][:, :d_in].contiguous()   # the observation columns of w1, sliced once outside the timed calls
        variants[f"p_bias_logits_d1_a{a}"] = (1, lambda c=c, w=w1_obs: mlp.mlp_forward(obs, w, c[2], c[4],
                                                                                       biases=(c[1], c[3], c[5])))
        variants[f"p_bias_critic_a{a}"] = (1, lambda a=a: critic_call(a, False))
        variants[f"p_bias_critic_twin_a{a}"] = (1, lambda a=a: critic_call(a, True))
        variants[f"p_bias_critic_twin_eager_a{a}"] = (1, lambda a=a: eager_twin(a))
    # q: TD targets over the twin critics of p, with a 256 -> 1024 -> 1024 -> d_act actor (its own weights)
    gq = torch.Generator(device="cuda:0").manual_seed(13)
    qr = lambda *s, scale=1.0: (torch.randn(*s, device="cuda:0", generator=gq) * scale).bfloat16()   # noqa: E731
    actors = {a: (qr(d_hidden, d_in, scale=0.02), qr(d_hidden, scale=0.1), qr(d_hidden, d_hidden, scale=0.02),
                  qr(d_hidden, scale=0.1), qr(a, d_hidden, scale=0.02), qr(a, scale=0.1)) for a in critic_widths}
    actor_ls = {a: (qr(a, d_hidden, scale=0.02), torch.linspace(-2.0, 0.5, a, device="cuda:0").bfloat16())
                for a in critic_widths}
    reward = torch.randn(M, device="cuda:0", generator=gq)
    done = (torch.rand(M, device="cuda:0", generator=gq) < 0.05).float()
    td_opts = {"td3": dict(policy="deterministic", noise=0.2, noise_clip=0.5, seed=SEED),
               "sac": dict(policy="gaussian", squash=True, seed=SEED, alpha=0.2)}

    def td_fused(a, tag):
        c, kw = critics[(a, 0)], dict(td_opts[tag])
        if tag == "sac":
            kw["log_std"] = actor_ls[a]
        return mlp.mlp_forward(obs, c[0], c[2], c[4], biases=(c[1], c[3], c[5]), output="td_target",
                               twin=critics[(a, 1)], actor=actors[a], reward=reward, done=done, gamma=0.99, **kw)

    def td_two_call(a, tag):
        """The actor entry, the twin critic entry, then the target in eager torch."""
        ac, c, kw = actors[a], critics[(a, 0)], dict(td_opts[tag])
        if tag == "td3":
            kw.pop("policy")
            act = mlp.mlp_forward(obs, ac[0], ac[2], ac[4], biases=(ac[1], ac[3], ac[5]), output="deterministic", **kw)
        else:
            act, logp = mlp.mlp_forward(obs, ac[0], ac[2], ac[4], biases=(ac[1], ac[3], ac[5]), output="gaussian",
                                        seed=SEED, log_std=actor_ls[a], squash=True)
        t = mlp.mlp_forward(obs, c[0], c[2], c[4], biases=(c[1], c[3], c[5]), output="critic", action=act,
                            twin=critics[(a, 1)])[2]
        if tag == "sac":
            t = t - 0.2 * logp
        return reward + 0.99 * (1 - done) * t

    def td_eager(a, tag):
        """Logits entries and torch: the actor's logits (over [w3; w_ls] for SAC), its head in torch, then the eager
        twin of p over those actions and the target in torch."""
        ac = actors[a]
        z = normal_noise(SEED, 0, M, a, device="cuda:0")
        if tag == "td3":
            y = mlp.mlp_forward(obs, ac[0], ac[2], ac[4], biases=(ac[1], ac[3], ac[5])).float()
            act = (y.tanh() + (0.2 * z).clamp(-0.5, 0.5)).clamp(-1.0, 1.0)
        else:
            y = mlp.mlp_forward(obs, ac[0], ac[2], torch.cat((ac[4], actor_ls[a][0])),
                                biases=(ac[1], ac[3], torch.cat((ac[5], actor_ls[a][1])))).float()
            mu, ls = y[:, :a], y[:, a:].clamp(-20.0, 2.0)
            u = mu + torch.exp(ls) * z
            au = u.abs()
            logp = (-0.5 * z * z - ls - HALF_LOG_2PI).sum(-1) - (2 * (LN2 - au - torch.log1p(torch.exp(-2 * au)))).sum(-1)
            act = torch.tanh(u)
        x = torch.cat([obs, act.to(torch.bfloat16), obs.new_zeros(M, 64 - a)], -1)
        qs = [mlp.mlp_forward(x, F.pad(critics[(a, i)][0], (0, 64 - a)), critics[(a, i)][2], critics[(a, i)][4],
                              biases=critics[(a, i)][1::2]).float().squeeze(-1) for i in (0, 1)]
        t = torch.minimum(qs[0], qs[1])
        if tag == "sac":
            t = t - 0.2 * logp
        return reward + 0.99 * (1 - done) * t

    for a in critic_widths:
        for tag in td_opts:
            variants[f"q_bias_{tag}_target_a{a}"] = (1, lambda a=a, tag=tag: td_fused(a, tag))
            variants[f"q_bias_{tag}_two_call_a{a}"] = (1, lambda a=a, tag=tag: td_two_call(a, tag))
            variants[f"q_bias_{tag}_eager_a{a}"] = (1, lambda a=a, tag=tag: td_eager(a, tag))
    for a in critic_widths:   # parity before timing: the fused target equals the two-call arm bit for bit
        for tag in td_opts:
            got, two = td_fused(a, tag), td_two_call(a, tag)
            assert torch.equal(got.view(torch.int32), two.view(torch.int32)), (tag, a)
            eager = td_eager(a, tag)
            close = torch.isclose(got, eager, rtol=2.0 ** -7, atol=1e-2)
            assert float(close.float().mean()) > 0.99, (tag, a)
            parity[f"q_bias_{tag}_a{a}"] = {"target_eq_two_call_all_rows": "ok",
                                            "target_vs_eager_frac_close": round(float(close.float().mean()), 6),
                                            "target_eq_eager_bits_frac": round(float(
                                                (got.view(torch.int32) == eager.view(torch.int32)).float().mean()), 6)}
            del got, two, eager
    # r: DQN targets; the online network has weights of its own
    gr = torch.Generator(device="cuda:0").manual_seed(17)
    rr = lambda *s, scale=1.0: (torch.randn(*s, device="cuda:0", generator=gr) * scale).bfloat16()   # noqa: E731
    q_nets = {(d, k): (rr(d_hidden, d_in, scale=0.02), rr(d_hidden, scale=0.1), rr(d_hidden, d_hidden, scale=0.02),
                       rr(d_hidden, scale=0.1), rr(d, d_hidden, scale=0.02), rr(d, scale=0.1))
              for d in (6, 18, 64) for k in ("target", "online")}
    q_legal = torch.rand(M, 18, device="cuda:0", generator=gr) < 0.5

    def dqn_fused(d, double, mask):
        t = q_nets[(d, "target")]
        return mlp.mlp_forward(obs, t[0], t[2], t[4], biases=t[1::2], output="dqn_target", reward=reward, done=done,
                               gamma=0.99, online=q_nets[(d, "online")] if double else None, mask=mask)

    def dqn_two_call(d, double, mask):
        """The actions entry on the selector, the logits entry on the target, then the gather and y in eager torch."""
        t, s = q_nets[(d, "target")], q_nets[(d, "online" if double else "target")]
        a = mlp.mlp_forward(obs, s[0], s[2], s[4], biases=s[1::2], output="actions", mask=mask)
        qt = mlp.mlp_forward(obs, t[0], t[2], t[4], biases=t[1::2], output="logits")
        return reward + 0.99 * (1 - done) * qt.float().gather(1, a[:, None]).squeeze(1)

    def dqn_eager(d, double, mask):
        """The logits entry on each network, then the mask, argmax, gather and y in torch."""
        t, s = q_nets[(d, "target")], q_nets[(d, "online")]
        qt = mlp.mlp_forward(obs, t[0], t[2], t[4], biases=t[1::2])
        sel = mlp.mlp_forward(obs, s[0], s[2], s[4], biases=s[1::2]) if double else qt
        if mask is not None:
            sel = sel.masked_fill(~mask, float("-inf"))
        return reward + 0.99 * (1 - done) * qt.float().gather(1, sel.argmax(-1, keepdim=True)).squeeze(1)

    dqn_cases = [(6, None), (18, None), (18, q_legal), (64, None)]
    for d, mask in dqn_cases:
        for double in (False, True):
            tag = ("double" if double else "dqn") + ("_masked" if mask is not None else "")
            for arm, fn in (("target", dqn_fused), ("two_call", dqn_two_call), ("eager", dqn_eager)):
                variants[f"r_bias_{tag}_{arm}_d{d}"] = (d, lambda d=d, double=double, mask=mask, fn=fn: fn(d, double,
                                                                                                         mask))
    for d, mask in dqn_cases:   # parity before timing: the fused target equals both arms bit for bit
        for double in (False, True):
            tag = ("double" if double else "dqn") + ("_masked" if mask is not None else "")
            got = dqn_fused(d, double, mask)
            for arm in (dqn_two_call, dqn_eager):
                assert torch.equal(got.view(torch.int32), arm(d, double, mask).view(torch.int32)), (tag, d, arm)
            parity[f"r_bias_{tag}_d{d}"] = {"target_eq_two_call_all_rows": "ok", "target_eq_eager_all_rows": "ok"}
            del got
    for _, fn in variants.values():   # warm-up: tensor maps, smem attributes, allocations
        fn()
        fn()
    torch.cuda.synchronize(0)
    samples = {k: [] for k in variants}
    for _ in range(args.samples):
        for name, (_, fn) in variants.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.calls):
                fn()
            e1.record()
            torch.cuda.synchronize(0)
            samples[name].append(e0.elapsed_time(e1) / args.calls)

    # parity
    a = variants["a_original_d64"][1]()
    b = variants["b_policy_nobias_d64"][1]()
    torch.cuda.synchronize(0)
    parity["b_equals_a_bitwise"] = bool(torch.equal(a, b))
    idx = torch.randint(0, M, (2048,), device="cuda:0", generator=g)
    for name, d, bias in (("a_original_d64", 64, False), ("e_bias_both_d64", 64, True), ("f_bias_both_d18", 18, True),
                          ("f_bias_both_d256", 256, True)):
        res = variants[name][1]()
        logits, actions = res if isinstance(res, tuple) else (res, None)
        w = (w1, w2, heads[d][0])
        bs = (b1, b2, heads[d][1]) if bias else (None, None, None)
        ref = _fp32(obs[idx], w, bs)
        torch.testing.assert_close(logits[idx].float(), ref.bfloat16().float(), rtol=2**-7, atol=1e-2)
        entry = {"logits_2048_rows": "ok"}
        if actions is not None:
            assert torch.equal(actions, torch.argmax(logits, dim=-1))
            top2 = ref.topk(2, dim=1).values
            clear = (top2[:, 0] - top2[:, 1]) > 2**-6
            assert torch.equal(actions[idx][clear], ref.argmax(1)[clear])
            only = mlp.mlp_forward(obs, *w, biases=bs, output="actions")
            assert torch.equal(only, actions)
            entry.update({"actions_eq_argmax_all_rows": "ok", "actions_vs_fp32_clear_rows": int(clear.sum()),
                          "actions_only_eq_both": "ok"})
        parity[name] = entry
    assert parity["b_equals_a_bitwise"]
    r0 = M - 2048 - 77
    for d in (18, 64, 256):
        actions, log_probs = variants[f"g_bias_sample_d{d}"][1]()
        w, bs = (w1, w2, heads[d][0]), (b1, b2, heads[d][1])
        y = mlp.mlp_forward(obs[r0:r0 + 2048], *w, biases=bs).double()
        s64 = y - torch.log(-torch.log(gumbel_uniform(SEED, r0, 2048, d, device="cuda:0").double()))
        a = actions[r0:r0 + 2048]
        eps = 2.0 ** -18 * (1 + s64.abs().amax(1))
        top2 = s64.topk(2, dim=1).values
        clear = (top2[:, 0] - top2[:, 1]) > eps
        assert bool((s64.gather(1, a[:, None]).squeeze(1) >= top2[:, 0] - eps).all())
        assert torch.equal(a[clear], s64.argmax(1)[clear])
        ref = y.gather(1, a[:, None]).squeeze(1) - torch.logsumexp(y, -1)
        assert bool(((log_probs[r0:r0 + 2048].double() - ref).abs() <= (d + 8) * 2.0 ** -22 * (1 + ref.abs())).all())
        parity[f"g_bias_sample_d{d}"] = {"sample_bars_2048_rows": "ok", "clear_rows": int(clear.sum())}
    for d in (6, 18, 64):
        actions, log_probs = variants[f"h_bias_gaussian_d{d}"][1]()
        w, bs = (w1, w2, heads[d][0]), (b1, b2, heads[d][1])
        y = mlp.mlp_forward(obs[r0:r0 + 2048], *w, biases=bs).double()
        z = torch.special.ndtri(gumbel_uniform(SEED, r0, 2048, d, device="cuda:0", word3=1).double())
        ls = log_stds[d].double()
        sigma = ls.exp()
        err = (actions[r0:r0 + 2048].double() - (y + sigma * z)).abs()
        assert bool((err <= 2.0 ** -19 * sigma * (1 + z.abs()) + 2.0 ** -23 * y.abs()).all())
        t = 0.5 * z * z + ls
        ref = -t.sum(-1) - d * HALF_LOG_2PI
        tol = 2.0 ** -20 * ((1 + z.abs()) ** 2).sum(-1) + (d + 8) * 2.0 ** -23 * (t.abs().sum(-1) + d * 0.92)
        assert bool(((log_probs[r0:r0 + 2048].double() - ref).abs() <= tol).all())
        parity[f"h_bias_gaussian_d{d}"] = {"gaussian_bars_2048_rows": "ok"}

    for d in (18, 64, 256):
        logits = mlp.mlp_forward(obs, w1, w2, heads[d][0], biases=(b1, b2, heads[d][1]))
        actions = variants[f"i_bias_masked_actions_d{d}"][1]()
        assert torch.equal(actions, logits.masked_fill(~legal[d], float("-inf")).argmax(-1))
        del logits
        sampled, _ = variants[f"i_bias_masked_sample_d{d}"][1]()
        has = legal[d].any(-1)
        assert bool(legal[d][has].gather(1, sampled[has][:, None]).all())
        parity[f"i_bias_masked_d{d}"] = {"masked_actions_eq_masked_argmax_all_rows": "ok",
                                         "sampled_actions_legal_all_rows": "ok"}

    for d in value_widths:
        entry = {}
        _, _, eager = variants[f"j_bias_eager_critic_d{d}"][1]()
        values = {}
        for kind in ("sample", "masked_sample", "gaussian"):
            want = variants[f"j_bias_{kind}_d{d}"][1]()
            got = variants[f"j_bias_{kind}_value_d{d}"][1]()
            for g_, w_ in zip(got[:2], want):
                assert torch.equal(g_.view(torch.int32) if g_.dtype == torch.float32 else g_,
                                   w_.view(torch.int32) if w_.dtype == torch.float32 else w_), (kind, d)
            values[kind] = got[2]
            torch.testing.assert_close(got[2], eager, rtol=2**-7, atol=1e-2)
            entry[f"{kind}_draws_eq_unvalued_all_rows"] = "ok"
            del want, got
        assert torch.equal(values["masked_sample"].view(torch.int32), values["sample"].view(torch.int32))
        entry["masked_values_eq_unmasked"] = "ok"
        entry["values_vs_eager_critic"] = "ok"
        parity[f"j_bias_value_d{d}"] = entry
        del eager, values

    for d, nvec in nvecs.items():
        entry = {}
        for tag in ("", "masked_"):
            logits = mlp.mlp_forward(obs, w1, w2, heads[d][0], biases=(b1, b2, heads[d][1]))
            if tag:
                logits = logits.masked_fill(~legal[d], float("-inf"))
            greedy = variants[f"k_bias_{tag}actions_nvec_d{d}"][1]()
            assert torch.equal(greedy, torch.stack([p.argmax(-1) for p in logits.split(nvec, -1)], -1)), (tag, d)
            assert torch.equal(greedy, variants[f"k_bias_{tag}actions_eager_d{d}"][1]()), (tag, d)
            del logits, greedy
            acts, lp = variants[f"k_bias_{tag}sample_nvec_d{d}"][1]()
            want_a, want_lp = variants[f"k_bias_{tag}sample_eager_d{d}"][1]()
            rows = (acts == want_a).all(-1)
            assert float(rows.double().mean()) >= 0.999, (tag, d, float(rows.double().mean()))
            a_lp, b_lp = lp[rows], want_lp[rows]
            fin = b_lp.isfinite()
            assert torch.equal(fin, a_lp.isfinite()), (tag, d)
            assert bool(((a_lp[fin] - b_lp[fin]).abs() <= 2.0 ** -16 * (1 + b_lp[fin].abs())).all()), (tag, d)
            entry[f"{tag}greedy_eq_group_argmax_all_rows"] = "ok"
            entry[f"{tag}sample_rows_eq_eager"] = round(float(rows.double().mean()), 6)
            if tag:
                lo = 0
                for i, n in enumerate(nvec):
                    part = legal[d][:, lo:lo + n]
                    has = part.any(-1)
                    assert bool(part[has].gather(1, acts[has][:, i:i + 1]).all()), (d, i)
                    lo += n
                entry["masked_samples_legal_all_rows"] = "ok"
            del acts, lp, want_a, want_lp
        parity[f"k_bias_nvec_d{d}"] = entry

    for d in state_widths:
        entry = {}
        w3s, b3s = mlp._stacked_head(heads[d][0], heads[d][1], None, None, *ls_heads[d])
        y = mlp.mlp_forward(obs[r0:r0 + 2048], w1, w2, w3s, biases=(b1, b2, b3s)).double()
        mu, sigma = y[:, 0::2], y[:, 1::2].clamp(-20.0, 2.0).exp()
        z = torch.special.ndtri(gumbel_uniform(SEED, r0, 2048, d, device="cuda:0", word3=1).double())
        u, lp = variants[f"l_bias_state_unsquashed_d{d}"][1]()
        a, lp_sq = variants[f"l_bias_state_squashed_d{d}"][1]()
        err = (u[r0:r0 + 2048].double() - (mu + sigma * z)).abs()
        assert bool((err <= 2.0 ** -19 * sigma * (1 + z.abs()) + 2.0 ** -23 * mu.abs()).all()), d
        t = torch.tanh(u[r0:r0 + 2048].double())
        assert bool(((a[r0:r0 + 2048].double() - t).abs() <= 2.0 ** -22 * t.abs() + 2.0 ** -126).all()), d
        entry["state_bars_2048_rows"] = "ok"
        for tag, got in (("unsquashed", (u, lp)), ("squashed", (a, lp_sq))):
            want = variants[f"l_bias_state_{tag}_eager_d{d}"][1]()
            for g_, w_ in zip(got, want):
                torch.testing.assert_close(g_, w_, rtol=1e-4, atol=1e-4)
            entry[f"{tag}_vs_eager_all_rows"] = "ok"
            del want
        parity[f"l_bias_state_d{d}"] = entry
        del u, lp, a, lp_sq

    for d in eps_widths:
        entry = {}
        for tag in ("", "masked_"):
            for eps in eps_values:
                got = variants[f"m_bias_{tag}epsilon{eps}_d{d}"][1]()
                want = variants[f"m_bias_{tag}epsilon{eps}_eager_d{d}"][1]()
                for g_, w_ in zip(got, want):
                    assert torch.equal(g_.view(torch.int32) if g_.dtype == torch.float32 else g_,
                                       w_.view(torch.int32) if w_.dtype == torch.float32 else w_), (tag, eps, d)
                entry[f"{tag}epsilon{eps}_eq_eager_all_rows"] = "ok"
                del got, want
        parity[f"m_bias_epsilon_d{d}"] = entry

    for tag, (d, sampled, _, _, _) in evaluate_cases.items():
        drawn = variants[f"n_bias_{sampled}_{tag}"][1]()
        got = variants[f"n_bias_evaluate_{tag}"][1]()
        want = variants[f"n_bias_evaluate_eager_{tag}"][1]()
        if sampled == "sample":
            lp, ref = got[0], drawn[1]
            nan = lp.isnan()
            assert torch.equal(nan, ref.isnan()) and torch.equal(lp[~nan].view(torch.int32),
                                                                 ref[~nan].view(torch.int32)), tag
            if len(got) == 3:
                assert torch.equal(got[2].view(torch.int32), drawn[2].view(torch.int32)), tag
        else:
            assert torch.allclose(got[0], drawn[1], rtol=1e-4, atol=1e-3), tag
        for g_, w_ in zip(got[:2], want[:2]):
            assert torch.allclose(g_, w_, rtol=1e-4, atol=1e-4, equal_nan=True), tag
        if len(got) == 3:   # the eager critic is a different GEMM: the value rows' bar
            assert torch.allclose(got[2], want[2], rtol=2.0 ** -7, atol=1e-2), tag
        parity[f"n_bias_evaluate_{tag}"] = "ok"
        del drawn, got, want

    r0 = int(torch.randint(0, M - 2048, (1,), device="cuda:0", generator=g))
    for d in (6, 17, 64):
        y = variants[f"o_bias_logits_d{d}"][1]()[r0:r0 + 2048].double()
        t64 = y.tanh()
        z64 = torch.special.ndtri(gumbel_uniform(SEED, r0, 2048, d, device="cuda:0", word3=1).double())
        for tag, kw in det_opts.items():
            got = variants[f"o_bias_{tag}_d{d}"][1]()[r0:r0 + 2048].double()
            sigma, clip = kw.get("noise", 0.0), kw.get("noise_clip", float("inf"))
            n64 = (sigma * z64).clamp(-clip, clip)
            ref = (t64 + n64).clamp(-1, 1)
            tol = 2.0 ** -22 * t64.abs() + 2.0 ** -148
            if sigma:
                tol = tol + sigma * 2.0 ** -19 * (1 + z64.abs()) + 2.0 ** -23 * (t64.abs() + n64.abs())
            assert bool(((got - ref).abs() <= tol).all()), (tag, d)
        got = variants[f"o_bias_smooth_d{d}"][1]()
        want = variants[f"o_bias_smooth_eager_d{d}"][1]()
        assert torch.allclose(got, want, rtol=1e-5, atol=1e-5), d
        parity[f"o_bias_deterministic_d{d}"] = "ok"
        del y, got, want

    for a in critic_widths:
        q = variants[f"p_bias_critic_a{a}"][1]()
        q1, q2, qm = variants[f"p_bias_critic_twin_a{a}"][1]()
        e1, e2, em = variants[f"p_bias_critic_twin_eager_a{a}"][1]()
        assert torch.equal(q.view(torch.int32), e1.view(torch.int32)), a
        assert torch.equal(q1.view(torch.int32), q.view(torch.int32)), a
        assert torch.equal(q2.view(torch.int32), e2.view(torch.int32)), a
        off_ties = ~((q1 == 0) & (q2 == 0))
        assert torch.equal(qm[off_ties].view(torch.int32), em[off_ties].view(torch.int32)), a
        c = critics[(a, 0)]
        x = torch.cat([obs[idx], critic_acts[a][idx].to(torch.bfloat16)], -1)
        ref = _fp32(x, (c[0], c[2], c[4]), (c[1], c[3], c[5])).squeeze(-1)
        torch.testing.assert_close(q[idx], ref.bfloat16().float(), rtol=2**-7, atol=1e-2)
        parity[f"p_bias_critic_a{a}"] = {"q_eq_logits_entry_all_rows": "ok", "twin_eq_eager_all_rows": "ok",
                                         "q_vs_fp32_2048_rows": "ok"}
        del q, q1, q2, qm, e1, e2, em

    result = {"what": "mlp_policy_c4_scale", "rows": M, "shape": f"{d_in}->{d_hidden}->{d_hidden}->d_out",
              "device": torch.cuda.get_device_name(0), "power_limit_w": _power_limit_w(),
              "samples": args.samples, "calls_per_sample": args.calls, "variants": {}, "parity": parity}
    for name, (d, _) in variants.items():
        ms = statistics.median(samples[name])
        flop = 2 * M * (d_in * d_hidden + d_hidden * d_hidden + d_hidden * d)
        result["variants"][name] = {"d_out": d, "ms_median": round(ms, 3), "ms_min": round(min(samples[name]), 3),
                                    "ms_max": round(max(samples[name]), 3), "tflops": round(flop / ms / 1e9, 1)}
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
