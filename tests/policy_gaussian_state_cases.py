"""User callables of the state-dependent Gaussian policy (SAC's actor), written as a kubetorch user writes SPMD
functions: rank r runs the trunk  Linear → ReLU → Linear → ReLU  on its `obs.chunk(WORLD_SIZE)[RANK]` rows, a mean head
nn.Linear(d_hidden, d_out) (w3, b3) and a log-std head nn.Linear(d_hidden, d_out) (w_ls, b_ls) on it, clamps the
log-std, draws u = μ + exp(log_std)·z with the Gaussian noise of its rows' GLOBAL indices, optionally squashes the
action with tanh, and returns (actions, log_probs), or (actions, log_probs, values) with a critic (wv, bv) beside it.

TEST INFRASTRUCTURE.  These functions are the semantic definition of @kt.mapped("mlp", bias=True, output="gaussian",
seed="seed", log_std=("w_ls", "b_ls"), log_std_bounds=(lo, hi), squash=...[, value=("wv", "bv")]).  The tanh
correction is the exact log(1 - tanh²u) = 2·(log 2 - |u| - softplus(-2|u|)), finite for finite u, not SB3's
log(1 - tanh²u + 1e-6).  The oracle restatement (oracle/ref_dispatch.spmd_call) executes them on CPU; the CUDA path
must reproduce their results.
"""
import math

from policy_value_cases import _row0, _trunk, _value

LOG_STD_BOUNDS = (-20.0, 2.0)


def gaussian_state(h, w3, b3, w_ls, b_ls, seed, row0, bounds=LOG_STD_BOUNDS, squash=False):
    """(float32 actions [rows, d_out], float32 log_probs [rows]) of the trunk output h of global rows row0, ...."""
    import torch
    import torch.nn.functional as F

    from kubetorch_b200.sampling import normal_noise

    mu = F.linear(h, w3, b3).float()
    ls = F.linear(h, w_ls, b_ls).float().clamp(bounds[0], bounds[1])   # torch.clamp: a NaN stays NaN
    z = normal_noise(seed, row0, mu.shape[0], mu.shape[1], device=mu.device)
    u = mu + torch.exp(ls) * z
    log_probs = (-0.5 * z * z - ls - 0.5 * math.log(2 * math.pi)).sum(-1)
    if not squash:
        return u, log_probs
    au = u.abs()   # softplus(-2|u|) as log1p(exp(-2|u|)): F.softplus's CPU kernel rounds by the batch's shape
    return torch.tanh(u), log_probs - (2 * (math.log(2) - au - torch.log1p(torch.exp(-2 * au)))).sum(-1)


def mlp_policy_gaussian_state(obs, w1, b1, w2, b2, w3, b3, w_ls, b_ls, seed):
    """Unsquashed actions with the log-std clamped to (-20, 2)."""
    return gaussian_state(_trunk(obs, w1, b1, w2, b2), w3, b3, w_ls, b_ls, seed, _row0(obs))


def mlp_policy_gaussian_state_squashed(obs, w1, b1, w2, b2, w3, b3, w_ls, b_ls, seed):
    """SAC's actor: tanh-squashed actions with the log-std clamped to (-20, 2)."""
    return gaussian_state(_trunk(obs, w1, b1, w2, b2), w3, b3, w_ls, b_ls, seed, _row0(obs), squash=True)


def mlp_policy_gaussian_state_squashed_value(obs, w1, b1, w2, b2, w3, b3, w_ls, b_ls, wv, bv, seed):
    """SAC's actor as above, with the state value of a critic on the same trunk."""
    h = _trunk(obs, w1, b1, w2, b2)
    return (*gaussian_state(h, w3, b3, w_ls, b_ls, seed, _row0(obs), squash=True), _value(h, wv, bv))
