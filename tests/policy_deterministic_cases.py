"""User callables of the deterministic actor (DDPG, TD3), written as a kubetorch user writes SPMD functions: rank r runs
the trunk  Linear → ReLU → Linear → ReLU  on its `obs.chunk(WORLD_SIZE)[RANK]` rows and a head nn.Linear(d_hidden,
d_out) (w3, b3) on it, squashes the mean with tanh, adds σ times the Gaussian noise of its rows' GLOBAL indices,
clipped to [-c, c], and clamps the action to [-1, 1].

TEST INFRASTRUCTURE.  These functions are the semantic definition of @kt.mapped("mlp", output="deterministic",
noise=σ, noise_clip=c, seed="seed", squash=...) (with bias=True): with μ the bf16 logits, t = tanh(μ.float()) (μ.float()
unsquashed), t + (σ·z).clamp(-c, c) when σ != 0, and t.clamp(-1, 1) when squashed.  The oracle restatement
(oracle/ref_dispatch.spmd_call) executes them on CPU; the CUDA path must reproduce their results.
"""
import math

from policy_value_cases import _row0, _trunk


def deterministic(mu, seed, row0, noise=0.0, noise_clip=math.inf, squash=True):
    """fp32 actions [rows, d_out] of the bf16 head outputs mu of global rows row0, ...: the header's definition."""
    from kubetorch_b200.sampling import normal_noise

    t = mu.float().tanh() if squash else mu.float()
    if noise != 0:
        z = normal_noise(seed, row0, mu.shape[0], mu.shape[1], device=mu.device)
        t = t + (noise * z).clamp(-noise_clip, noise_clip)   # fp32 multiply, then one fp32 add
    return t.clamp(-1.0, 1.0) if squash else t


def mlp_policy_deterministic(obs, w1, b1, w2, b2, w3, b3):
    """The noise-free squashed actor: tanh(μ), a DDPG / TD3 actor's action at evaluation time (and SAC's
    predict(deterministic=True) over the SAC actor's mean rows)."""
    import torch.nn.functional as F

    return deterministic(F.linear(_trunk(obs, w1, b1, w2, b2), w3, b3), None, _row0(obs))


def mlp_policy_deterministic_explore(obs, w1, b1, w2, b2, w3, b3, seed):
    """Exploration at rollout time: clip(tanh(μ) + N(0, 0.1), -1, 1)."""
    import torch.nn.functional as F

    return deterministic(F.linear(_trunk(obs, w1, b1, w2, b2), w3, b3), seed, _row0(obs), noise=0.1)


def mlp_policy_deterministic_smoothing(obs, w1, b1, w2, b2, w3, b3, seed):
    """TD3's target policy smoothing: clip(tanh(μ) + clip(N(0, 0.2), -0.5, 0.5), -1, 1)."""
    import torch.nn.functional as F

    return deterministic(F.linear(_trunk(obs, w1, b1, w2, b2), w3, b3), seed, _row0(obs), noise=0.2, noise_clip=0.5)


def mlp_policy_deterministic_unsquashed(obs, w1, b1, w2, b2, w3, b3, sigma, seed):
    """An unsquashed actor with the noise σ of a call argument, unclipped: μ + σ·z."""
    import torch.nn.functional as F

    return deterministic(F.linear(_trunk(obs, w1, b1, w2, b2), w3, b3), seed, _row0(obs), noise=sigma, squash=False)
