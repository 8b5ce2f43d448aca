"""bf16 MLP policy (BASELINE config C4) on wgmma tensor cores — tensor-facing wrapper of
ktb_mlp_bf16_policy (biases, heads of 1 to 256 outputs, greedy actions), ktb_mlp_bf16_policy_sample (seeded
Gumbel-max actions with their log-probabilities, kubetorch_b200.sampling), ktb_mlp_bf16_policy_gaussian (seeded
diagonal-Gaussian actions with their log-probabilities), the _masked forms of the first two (a per-row legal-action
mask), the _value forms of the sampled heads (a critic's state value on the same trunk), the _multidiscrete forms of
the greedy and sampled heads (one categorical per group of columns), the _gaussian_state forms (a per-row log-std
head, optionally tanh-squashed actions), the _epsilon_greedy forms (a Q-network's ε-greedy actor), the _evaluate
and _gaussian_evaluate forms (the log-probability and entropy of given actions), the _deterministic forms (DDPG's and
TD3's actor: tanh actions with clipped Gaussian noise), the _critic forms (Q(s, a) critics with the actions fed into
layer 1, single or twin), the _td_target forms (TD3's, DDPG's and SAC's Bellman target: the actor, the target critics
and the target in one call), the _dqn_target forms (DQN's and Double DQN's Bellman target: the greedy next action, the
target network's Q at it and the target in one call) and their scatter→exec→gather form."""
from __future__ import annotations

import ctypes
import math
import weakref
from typing import List, Optional, Sequence, Tuple

import torch

from . import lib as L
from . import ops
from ..mapped import MLP_OUTPUTS as OUTPUTS
from ..mapped import CONSTANT_CHECKS, EVALUATE_OUTPUTS, TD_OPTIONS, check_mlp_options, check_mlp_rules, check_nvec

_scratch = {}
_stage = {}
_weight_cache = {}
_stacked_heads = {}   # (device, id(w3)) -> [weakref to w3, stamp of w3 / b3 / wv / bv / w_ls / b_ls, W3, b3]
_padded_w1s = {}      # (device, id(w1)) -> [weakref to w1, stamp of w1 and d_in, W1p]
_pool = None


def pushed_scratch_bytes(M: int, d_hidden: int, chunk_rows: int, critic: bool = False) -> int:
    """Scratch of ktb_mlp_bf16_policy_pushed: two hidden activations of min(chunk_rows, M) rows, and with `critic` the
    action tile [rows, 64] bf16 of the _critic entries.  It follows the pushed form's own chunk_rows, not the tuning
    chunk that ktb_mlp_scratch_bytes uses for the pull forms."""
    rows = min(int(chunk_rows), int(M))
    return 2 * rows * int(d_hidden) * 2 + (rows * 64 * 2 if critic else 0)


def pushed_td_scratch_bytes(M: int, d_hidden_actor: int, d_hidden: int, d_act: int, chunk_rows: int) -> int:
    """Scratch of the _td_target _pushed entries: ktb_mlp_td_target_scratch_bytes at the pushed form's chunk_rows."""
    rows = min(int(chunk_rows), int(M))
    return pushed_scratch_bytes(M, max(d_hidden_actor, d_hidden), chunk_rows, True) + rows * (4 * int(d_act) + 8)


def _cached_buffer(cache: dict, key, dev: int, nbytes: int) -> torch.Tensor:
    """cache[key]: a uint8 buffer on `dev` of at least `nbytes`, replaced by a larger one when a call needs more."""
    buf = cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = cache[key] = torch.empty(nbytes, dtype=torch.uint8, device=f"cuda:{dev}")
    return buf


def _scratch_for(dev: int, M: int, d_hidden: int, critic: bool = False) -> torch.Tensor:
    lib = L.load()
    nbytes = lib.ktb_mlp_critic_scratch_bytes(M, d_hidden) if critic else lib.ktb_mlp_scratch_bytes(M, d_hidden)
    return _cached_buffer(_scratch, dev, dev, nbytes)


def _stage_for(dev: int, M: int, d_in: int) -> torch.Tensor:
    return _cached_buffer(_stage, dev, dev, L.load().ktb_mlp_stage_bytes(M, d_in))


def _thread_pool():
    """Threads that issue the ranks' launches in parallel (ctypes releases the GIL)."""
    global _pool
    if _pool is None:
        from concurrent.futures import ThreadPoolExecutor

        _pool = ThreadPoolExecutor(max_workers=16, thread_name_prefix="ktb-mlp")
    return _pool


MAX_D_OUT = 256
LOG_STD_BOUNDS = (-20.0, 2.0)   # SB3's and Spinning Up's clamp of a SAC actor's log-std


def _check_value(value, w3, b3, d_hidden, d_out) -> None:
    """_check_policy's checks of a value head (wv, bv), in this order: the pair, the head width, bv given exactly when
    b3 is, then wv's dtype and shape, layout and device, then bv."""
    if not isinstance(value, (tuple, list)) or len(value) != 2:
        raise ValueError("value must be (wv, bv): the critic's weight [1, d_hidden] and its bias [1] or None")
    wv, bv = value
    if d_out == MAX_D_OUT:
        raise ValueError(f"d_out={d_out}: with a value head the policy is 1 to {MAX_D_OUT - 1} wide (its "
                         f"columns and the value's must fit one {MAX_D_OUT}-wide tile)")
    if (bv is None) != (b3 is None):
        raise ValueError("value: bv is given exactly when b3 is (a zero bias in the policy's columns would turn -0.0 "
                         "logits into +0.0)")
    if not isinstance(wv, torch.Tensor) or wv.dtype != torch.bfloat16 or tuple(wv.shape) != (1, d_hidden):
        raise ValueError(f"value: wv must be a bfloat16 tensor of shape (1, {d_hidden})")
    if not wv.is_contiguous():
        raise ValueError("value: wv must be contiguous")
    if not wv.is_cuda or wv.device != w3.device:
        raise ValueError(f"value: wv must be a CUDA tensor on the device of w3 ({w3.device}), got {wv.device}")
    if bv is not None and (not isinstance(bv, torch.Tensor) or bv.dtype != torch.bfloat16 or tuple(bv.shape) != (1,)
                           or not bv.is_contiguous() or bv.device != w3.device):
        raise ValueError(f"value: bv must be a contiguous bfloat16 tensor of shape (1,) on the device of w3 "
                         f"({w3.device})")


def _check_state_std(log_std, w3, b3, d_hidden, d_out, valued) -> None:
    """_check_policy's checks of a state-dependent log-std head log_std = (w_ls, b_ls), in this order: the pair, the
    head width (2·d_out columns, one more with a value head, in one 256-wide tile), b_ls given exactly when b3 is,
    w_ls's dtype and shape, layout and device, then b_ls."""
    if len(log_std) != 2:
        raise ValueError("log_std must be a tensor or (w_ls, b_ls): the log-std head's weight [d_out, d_hidden] and "
                         "its bias [d_out] or None")
    w_ls, b_ls = log_std
    limit = (MAX_D_OUT - valued) // 2
    if d_out > limit:
        raise ValueError(f"d_out={d_out}: a log-std head allows 1 to {limit} actions (the interleaved mean and "
                         f"log-std{' and the value column' if valued else ''} must fit one {MAX_D_OUT}-wide tile)")
    if (b_ls is None) != (b3 is None):
        raise ValueError("log_std: b_ls is given exactly when b3 is (a zero bias in the mean's columns would turn -0.0 "
                         "means into +0.0)")
    if not isinstance(w_ls, torch.Tensor) or w_ls.dtype != torch.bfloat16 or tuple(w_ls.shape) != (d_out, d_hidden):
        raise ValueError(f"log_std: w_ls must be a bfloat16 tensor of shape ({d_out}, {d_hidden})")
    if not w_ls.is_contiguous():
        raise ValueError("log_std: w_ls must be contiguous")
    if not w_ls.is_cuda or w_ls.device != w3.device:
        raise ValueError(f"log_std: w_ls must be a CUDA tensor on the device of w3 ({w3.device}), got {w_ls.device}")
    if b_ls is not None and (not isinstance(b_ls, torch.Tensor) or b_ls.dtype != torch.bfloat16
                             or tuple(b_ls.shape) != (d_out,) or not b_ls.is_contiguous() or b_ls.device != w3.device):
        raise ValueError(f"log_std: b_ls must be a contiguous bfloat16 tensor of shape ({d_out},) on the device of w3 "
                         f"({w3.device})")


def _check_epsilon(epsilon, obs) -> None:
    """_check_policy's checks of an epsilon tensor: a contiguous CUDA float32 tensor [M] on the device of obs [M,
    d_in]."""
    if not isinstance(obs, torch.Tensor):
        raise ValueError("an epsilon tensor is checked against obs: pass the obs [M, d_in] it goes with")
    if epsilon.dtype != torch.float32 or tuple(epsilon.shape) != (obs.shape[0],):
        raise ValueError(f"epsilon must be a float32 tensor of shape ({obs.shape[0]},), got {epsilon.dtype} "
                         f"{tuple(epsilon.shape)}")
    if not epsilon.is_contiguous():
        raise ValueError("epsilon must be contiguous")
    if not epsilon.is_cuda or epsilon.device != obs.device:
        raise ValueError(f"epsilon must be a CUDA tensor on the device of obs ({obs.device}), got {epsilon.device}")


def _check_taken(taken, output, obs, d_out, nvec) -> None:
    """_check_policy's checks of an evaluate output's given actions `taken`, in this order: a tensor; the dtype and
    shape (int64 [M], [M, len(nvec)] with nvec, for "evaluate"; float32 [M, d_out] for "gaussian_evaluate"; obs [M,
    d_in]); contiguous; a CUDA tensor on the device of obs."""
    if not isinstance(taken, torch.Tensor):
        raise ValueError(f"taken must be a tensor, got {type(taken).__name__}")
    if not isinstance(obs, torch.Tensor):
        raise ValueError("taken is checked against obs: pass the obs [M, d_in] it goes with")
    M = obs.shape[0]
    if output == "gaussian_evaluate":
        dtype, shape = torch.float32, (M, d_out)
    else:
        dtype, shape = torch.int64, (M,) if nvec is None else (M, len(nvec))
    if taken.dtype != dtype or tuple(taken.shape) != shape:
        raise ValueError(f"taken must be a {str(dtype).replace('torch.', '')} tensor of shape {shape}, got "
                         f"{str(taken.dtype).replace('torch.', '')} {tuple(taken.shape)}")
    if not taken.is_contiguous():
        raise ValueError("taken must be contiguous")
    if not taken.is_cuda or taken.device != obs.device:
        raise ValueError(f"taken must be a CUDA tensor on the device of obs ({obs.device}), got {taken.device}")


MAX_D_ACT = 64   # a critic's actions fill one 64-wide K block of layer 1


def _check_critic(w1, w2, w3, biases, obs, action, twin) -> None:
    """_check_policy's checks of output="critic", in this order: w3 one row; action an fp32 [M, d_act] CUDA tensor,
    contiguous, on the device of obs [M, d_in], with 1 <= d_act <= 64; w1 [d_hidden, d_in + d_act]; then twin = (w1,
    b1, w2, b2, w3, b3) of the second critic (_check_twin)."""
    if w3.shape[0] != 1:
        raise ValueError(f"d_out={w3.shape[0]}: a critic's w3 is [1, d_hidden] (one Q-value per row)")
    if not isinstance(action, torch.Tensor) or action.dtype != torch.float32 or action.dim() != 2:
        raise ValueError("action must be a 2-D float32 tensor [M, d_act]")
    if not isinstance(obs, torch.Tensor):
        raise ValueError("action is checked against obs: pass the obs [M, d_in] it goes with")
    M, d_in = obs.shape
    d_act = action.shape[1]
    if action.shape[0] != M:
        raise ValueError(f"action must have {M} rows (one per observation), got {tuple(action.shape)}")
    if not 1 <= d_act <= MAX_D_ACT:
        raise ValueError(f"d_act={d_act}: a critic takes 1 to {MAX_D_ACT} action columns (one K block of layer 1)")
    if not action.is_contiguous():
        raise ValueError("action must be contiguous")
    if not action.is_cuda or action.device != obs.device:
        raise ValueError(f"action must be a CUDA tensor on the device of obs ({obs.device}), got {action.device}")
    d_hidden = w1.shape[0]
    if tuple(w1.shape) != (d_hidden, d_in + d_act):
        raise ValueError(f"w1 must be [d_hidden, d_in + d_act] = [{d_hidden}, {d_in + d_act}] (the critic's layer 1 "
                         f"over torch.cat([obs, action], -1)), got {tuple(w1.shape)}")
    if twin is not None:
        _check_twin(twin, w1, w2, w3, biases)


def _padded_w1(w1: torch.Tensor, d_in: int) -> torch.Tensor:
    """W1p = [w1 | 0] [d_hidden, d_in + 64] of a critic's layer-1 weight w1 [d_hidden, d_in + d_act], on the device of
    w1: the action columns padded with zero columns to one 64-wide K block.  One entry per (device, w1) is kept, and
    rewritten in place when w1 has a new data_ptr or _version: target critics are Polyak-updated in place every step.
    Rewriting in place bumps W1p's own _version, so _weights_on copies the new weight to other devices."""
    stamp = (w1.data_ptr(), w1._version, d_in)
    key = (w1.device.index, id(w1))
    entry = _padded_w1s.get(key)
    if entry is None or entry[0]() is not w1:
        for k, e in list(_padded_w1s.items()):   # weights that are gone, or a new w1 that reuses an old id
            if e[0]() is None or k == key:
                del _padded_w1s[k]
        entry = _padded_w1s[key] = [weakref.ref(w1), None, None]
    if entry[1] != stamp:
        shape = (w1.shape[0], d_in + MAX_D_ACT)
        if entry[2] is None or tuple(entry[2].shape) != shape:
            entry[2] = torch.zeros(shape, dtype=w1.dtype, device=w1.device)
        entry[2][:, :w1.shape[1]].copy_(w1)
        entry[2][:, w1.shape[1]:].zero_()
        entry[1] = stamp
    return entry[2]


def _check_twin(twin, w1, w2, w3, biases, what="twin", of=("the second critic", "the first critic's")) -> None:
    """_check_critic's checks of twin = (w1, b1, w2, b2, w3, b3) of a second critic (or of a Double DQN target's online
    network, `what` naming the option and `of` the networks in the messages): six entries, biases given exactly as the
    first critic's, each weight a contiguous CUDA bfloat16 tensor of the first's shape on the device of w1."""
    if not isinstance(twin, (tuple, list)) or len(twin) != 6:
        raise ValueError(f"{what} must be (w1, b1, w2, b2, w3, b3) of {of[0]} (biases None without biases)")
    for name, t, mine in zip(("b1", "b2", "b3"), twin[1::2], biases):
        if (t is None) != (mine is None):
            raise ValueError(f"{what}: {name} is given exactly when {of[1]} is")
    for name, t, like in zip(("w1", "w2", "w3", "b1", "b2", "b3"), (*twin[0::2], *twin[1::2]), (w1, w2, w3, *biases)):
        if t is None:
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != torch.bfloat16 or tuple(t.shape) != tuple(like.shape) \
                or not t.is_contiguous() or not t.is_cuda or t.device != w1.device:
            raise ValueError(f"{what}: {name} must be a contiguous CUDA bfloat16 tensor of shape {tuple(like.shape)} "
                             f"on the device of w1 ({w1.device})")


def _check_td_target(w1, w2, w3, biases, obs, twin, log_std, actor, reward, done) -> None:
    """_check_policy's checks of output="td_target"'s tensors, in this order: actor = (w1, b1, w2, b2, w3, b3): six
    entries, biases given exactly as the critic's, contiguous CUDA bfloat16 on the device of w1, w1 [d_ha, d_in], w2
    [d_ha, d_ha], w3 [d_act, d_ha] with 1 <= d_act <= 64; the critic's w3 one row and w1 [d_hidden, d_in + d_act]; the
    twin; with a log_std = (w_ls, b_ls) pair the log-std head against the actor; reward and done fp32 [M] or [M, 1] of
    one shape, contiguous, on the device of obs [M, d_in]."""
    if not isinstance(actor, (tuple, list)) or len(actor) != 6:
        raise ValueError("actor must be (w1, b1, w2, b2, w3, b3) of the actor (biases None without biases)")
    for name, t, mine in zip(("b1", "b2", "b3"), actor[1::2], biases):
        if (t is None) != (mine is None):
            raise ValueError(f"actor: {name} is given exactly when the critic's is")
    for name, t in zip(("w1", "w2", "w3"), actor[0::2]):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.bfloat16 or t.dim() != 2 or not t.is_contiguous() \
                or not t.is_cuda or t.device != w1.device:
            raise ValueError(f"actor: {name} must be a 2-D contiguous CUDA bfloat16 tensor on the device of w1 "
                             f"({w1.device})")
    if not isinstance(obs, torch.Tensor):
        raise ValueError("a TD target is checked against obs: pass the next observations [M, d_in] it goes with")
    d_in = obs.shape[1]
    aw1, _, aw2, _, aw3, _ = actor
    d_ha, d_act = aw1.shape[0], aw3.shape[0]
    if tuple(aw1.shape) != (d_ha, d_in) or tuple(aw2.shape) != (d_ha, d_ha) or aw3.shape[1] != d_ha:
        raise ValueError(f"actor: weight shapes must be w1 [d_h, {d_in}], w2 [d_h, d_h], w3 [d_act, d_h] (nn.Linear "
                         f"layout), got {tuple(aw1.shape)}, {tuple(aw2.shape)}, {tuple(aw3.shape)}")
    if not 1 <= d_act <= MAX_D_ACT:
        raise ValueError(f"d_act={d_act}: a TD target's actor takes 1 to {MAX_D_ACT} actions (one K block of the "
                         f"critic's layer 1)")
    _check_biases(actor[1::2], d_ha, d_act, "actor: ")
    if w3.shape[0] != 1:
        raise ValueError(f"d_out={w3.shape[0]}: a critic's w3 is [1, d_hidden] (one Q-value per row)")
    if tuple(w1.shape) != (w1.shape[0], d_in + d_act):
        raise ValueError(f"w1 must be [d_hidden, d_in + d_act] = [{w1.shape[0]}, {d_in + d_act}] (the critic's layer "
                         f"1 over torch.cat([next_obs, actor(next_obs)], -1)), got {tuple(w1.shape)}")
    if twin is not None:
        _check_twin(twin, w1, w2, w3, biases)
    if log_std is not None:
        _check_state_std(log_std, aw3, actor[5], d_ha, d_act, False)
    _check_reward_done(reward, done, obs)


def _check_reward_done(reward, done, obs) -> None:
    """A TD or DQN target's reward and done: fp32 [M] or [M, 1] of one shape, contiguous, on the device of obs [M,
    d_in]."""
    M = obs.shape[0]
    for name, t in (("reward", reward), ("done", done)):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or tuple(t.shape) not in ((M,), (M, 1)):
            raise ValueError(f"{name} must be a float32 tensor of shape ({M},) or ({M}, 1), got "
                             f"{getattr(t, 'dtype', type(t).__name__)} {tuple(getattr(t, 'shape', ()))}")
        if not t.is_contiguous():
            raise ValueError(f"{name} must be contiguous")
        if not t.is_cuda or t.device != obs.device:
            raise ValueError(f"{name} must be a CUDA tensor on the device of obs ({obs.device}), got {t.device}")
    if reward.shape != done.shape:
        raise ValueError(f"reward and done must have one shape, got {tuple(reward.shape)} and {tuple(done.shape)}")


_ARGUMENTS = ("seed", "log_std", "mask", "value", "nvec", "log_std_bounds", "squash", "epsilon", "taken", "noise",
              "noise_clip", "action", "twin") + TD_OPTIONS + ("online",)   # _check_policy's options, td's, online


def _check_policy(w1, w3, biases, output, seed=None, log_std=None, mask=None, obs=None, value=None,
                  nvec=None, log_std_bounds=None, squash=None, epsilon=None, taken=None, noise=None,
                  noise_clip=None, action=None, twin=None, w2=None, td=(None,) * 6, online=None) -> None:
    """Raise ValueError for a call the kernels do not take, td = (actor, policy, reward, done, gamma, alpha) (a DQN
    target's reward, done and gamma there too) and None an option not given.  The options each output takes and
    requires are those of the table mapped.MLP_TAKES (check_mlp_options, check_mlp_rules), and a constant's value is
    checked as mapped() checks it (CONSTANT_CHECKS).  Then the tensors: a TD target's (_check_td_target), a critic's
    (_check_critic) and a DQN target's (its online network as a twin, _check_twin, then reward and done); a head 1 to 256
    wide; nvec
    summing to d_out; taken (_check_taken); an epsilon tensor (_check_epsilon); log_std, a 1-D contiguous CUDA float32
    tensor of length d_out or a state-dependent head (w_ls, b_ls) (_check_state_std); a mask, a contiguous CUDA
    torch.bool tensor [M, d_out] on the device of obs [M, d_in]; a value head (_check_value); the biases."""
    if output not in OUTPUTS:
        raise ValueError(f"output must be one of {OUTPUTS}, got {output!r}")
    values = (seed, log_std, mask, value, nvec, log_std_bounds, squash, epsilon, taken, noise, noise_clip, action, twin,
              *td, online)
    given = {name: v for name, v in zip(_ARGUMENTS, values) if v is not None}
    actor, policy, reward, done = td[:4]
    row = check_mlp_options(output, policy, given, argument=True)
    check_mlp_rules(row, output, policy, log_std, given, argument=True)
    for name, v in given.items():   # an epsilon may also be a per-row tensor (_check_epsilon)
        if name in CONSTANT_CHECKS and not (name == "epsilon" and isinstance(v, torch.Tensor)):
            CONSTANT_CHECKS[name](v)
    if output == "td_target":
        _check_td_target(w1, w2, w3, biases, obs, twin, log_std, actor, reward, done)
        _check_biases(biases, w1.shape[0], w3.shape[0])
        return
    if output == "critic":
        _check_critic(w1, w2, w3, biases, obs, action, twin)
    if output == "dqn_target":
        if online is not None:
            _check_twin(online, w1, w2, w3, biases, "online", ("the online network", "the target network's"))
        if not isinstance(obs, torch.Tensor):
            raise ValueError("a DQN target is checked against obs: pass the next observations [M, d_in] it goes with")
        _check_reward_done(reward, done, obs)
    if len(biases) != 3:
        raise ValueError("biases must be (b1, b2, b3), each a tensor or None")
    d_hidden, d_out = w1.shape[0], w3.shape[0]
    if not 1 <= d_out <= MAX_D_OUT:
        raise ValueError(f"d_out={d_out}: the policy head is 1 to {MAX_D_OUT} wide")
    if nvec is not None:
        check_nvec(nvec, d_out)
    if taken is not None:
        _check_taken(taken, output, obs, d_out, nvec)
    if isinstance(epsilon, torch.Tensor):
        _check_epsilon(epsilon, obs)
    if isinstance(log_std, (tuple, list)):
        _check_state_std(log_std, w3, biases[2], d_hidden, d_out, value is not None)
    elif log_std is not None and (not isinstance(log_std, torch.Tensor) or log_std.dtype != torch.float32
                                  or not log_std.is_cuda or not log_std.is_contiguous() or log_std.dim() != 1
                                  or log_std.shape[0] != d_out):
        raise ValueError(f"log_std must be a 1-D contiguous CUDA float32 tensor of length {d_out}")
    if mask is not None:
        if not isinstance(obs, torch.Tensor):
            raise ValueError("a mask is checked against obs: pass the obs [M, d_in] it goes with")
        if not isinstance(mask, torch.Tensor) or mask.dtype != torch.bool:
            raise ValueError("mask must be a torch.bool tensor")
        if tuple(mask.shape) != (obs.shape[0], d_out):
            raise ValueError(f"mask must have shape ({obs.shape[0]}, {d_out}), got {tuple(mask.shape)}")
        if not mask.is_contiguous():
            raise ValueError("mask must be contiguous")
        if not mask.is_cuda or mask.device != obs.device:
            raise ValueError(f"mask must be a CUDA tensor on the device of obs ({obs.device}), got {mask.device}")
    if value is not None:
        _check_value(value, w3, biases[2], d_hidden, d_out)
    _check_biases(biases, d_hidden, d_out)


def _check_biases(biases, d_hidden, d_out, what="") -> None:
    """Each bias given is a 1-D contiguous CUDA bfloat16 tensor of its layer's width."""
    for name, b, n in zip(("b1", "b2", "b3"), biases, (d_hidden, d_hidden, d_out)):
        if b is None:
            continue
        if not isinstance(b, torch.Tensor) or b.dtype != torch.bfloat16 or not b.is_cuda or not b.is_contiguous() \
                or b.dim() != 1 or b.shape[0] != n:
            raise ValueError(f"{what}{name} must be a 1-D contiguous CUDA bfloat16 tensor of length {n}")


def _stacked_head(w3, b3, wv=None, bv=None, w_ls=None, b_ls=None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """(W3, b3) of the head a C entry runs, on the device of w3: with a log-std head (w_ls, b_ls) the rows of w3 and
    w_ls interleaved, W3s = [w3_0; w_ls_0; w3_1; w_ls_1; ...] [2·d_out, d_hidden]; with a value head the critic's wv
    under them (W3v = [w3; wv] or W3sv = [W3s; wv]); the biases likewise (None without biases).  One entry per
    (device, head) is kept, and rewritten in place when any part has a new data_ptr or _version: PPO and SAC loops
    update their weights in place between rollout steps.  Rewriting in place bumps the head's own _version, so
    _weights_on copies the new head to other devices."""
    stamp = tuple(None if t is None else (t.data_ptr(), t._version) for t in (w3, b3, wv, bv, w_ls, b_ls))
    key = (w3.device.index, id(w3))
    entry = _stacked_heads.get(key)
    if entry is None or entry[0]() is not w3:
        for k, e in list(_stacked_heads.items()):   # heads whose w3 is gone, or a new w3 that reuses an old id
            if e[0]() is None or k == key:
                del _stacked_heads[k]
        entry = _stacked_heads[key] = [weakref.ref(w3), None, None, None]
    if entry[1] != stamp:
        for i, (mean, ls, v) in ((2, (w3, w_ls, wv)), (3, (b3, b_ls, bv))):
            if mean is None:
                entry[i] = None
                continue
            d = mean.shape[0]
            shape = ((2 * d if ls is not None else d) + (v is not None),) + tuple(mean.shape[1:])
            if entry[i] is None or tuple(entry[i].shape) != shape:
                entry[i] = torch.empty(shape, dtype=mean.dtype, device=mean.device)
            if ls is None:
                entry[i][:d].copy_(mean)
            else:
                entry[i][0:2 * d:2].copy_(mean)
                entry[i][1:2 * d:2].copy_(ls)
            if v is not None:
                entry[i][shape[0] - 1:].copy_(v)
        entry[1] = stamp
    return entry[2], entry[3]


def _outputs(output, M, d_out, device, logits, actions, log_probs, values=None, valued=False, nvec=None, twin=False):
    """(logits, actions, log_probs, values) of `M` rows as `output` writes them: bf16 logits [M, d_out]; int64 actions
    [M], [M, len(nvec)] with nvec, or fp32 [M, d_out] with "gaussian"; fp32 log_probs [M]; with `valued`, fp32 values
    [M].  "deterministic" writes fp32 actions [M, d_out] only.  With "epsilon_greedy" the last two slots hold its fp32
    q [M] and q_max [M]; with "evaluate" and
    "gaussian_evaluate" the actions slot holds the fp32 entropy [M].  With "critic" the logits slot holds the fp32 q
    [M] (q1 of a `twin`), and a twin's q2 and q_min ride in the actions and log_probs slots.  A buffer the mode does not
    write is None, a missing one is allocated on `device` and a given one is
    registered with the library (ops.ensure_init); given multi-discrete actions must be [M, len(nvec)]."""
    def buf(t, shape, dtype):
        if t is None:
            return torch.empty(shape, dtype=dtype, device=device)
        ops.ensure_init({t.device.index})
        return t

    gaussian = output in ("gaussian", "deterministic")
    if output == "critic":
        return buf(logits, (M,), torch.float32), buf(actions, (M,), torch.float32) if twin else None, \
            buf(log_probs, (M,), torch.float32) if twin else None, None
    if output in EVALUATE_OUTPUTS:
        return None, buf(actions, (M,), torch.float32), buf(log_probs, (M,), torch.float32), \
            buf(values, (M,), torch.float32) if valued else None
    if nvec is not None and actions is not None and tuple(actions.shape) != (M, len(nvec)):
        raise ValueError(f"actions must have shape ({M}, {len(nvec)}) with nvec of {len(nvec)} groups, got "
                         f"{tuple(actions.shape)}")
    return (buf(logits, (M, d_out), torch.bfloat16) if output in ("logits", "both") else None,
            None if output == "logits" else
            buf(actions, (M, d_out), torch.float32) if gaussian else
            buf(actions, (M,) if nvec is None else (M, len(nvec)), torch.int64),
            buf(log_probs, (M,), torch.float32) if output in ("sample", "gaussian", "epsilon_greedy") else None,
            buf(values, (M,), torch.float32) if valued or output == "epsilon_greedy" else None)


def _head(output, logits, actions, log_probs, seed, row_base, log_std, ptr, pushed=False, mask=None, values=None,
          nvec=None, std=None, epsilon=None, taken=None, det=None, act=None, twin=None):
    """The C entry that computes `output` (its _pushed form with `pushed`) and the head's arguments of that entry, the
    pointers as ptr(tensor) gives them.  `mask`, unless None, picks the _masked entry and is its mask argument: the
    mask's address in the pull forms, its offset in the staging half in the pushed forms.  `values`, unless None,
    picks the _value entry (whose W3 and b3 are the stacked head) and is its values buffer.  `nvec`, unless None,
    picks the _multidiscrete entry and is its group sizes.  `std` = (log_std_min, log_std_max, squash), unless None,
    picks the _gaussian_state entry (whose W3 and b3 are the interleaved head) in place of log_std.  With
    "epsilon_greedy", `epsilon` is ε's address (pull forms) or its offset in the staging half (pushed forms), and
    log_probs and values are its q and q_max buffers.  With "evaluate" and "gaussian_evaluate", `taken` is the given
    actions' address or offset likewise, and `actions` is the entropy buffer.  With "deterministic", `det` is the
    entry's (noise, noise_clip, squash) (_det); a noise-free call passes seed 0, which draws nothing.  With "critic",
    `act` is the actions' address or offset likewise, `twin` (unless None) the six weight and bias pointers of the
    second critic, which pick the _twin entry, and logits (q1), actions (q2) and log_probs (q_min) its outputs."""
    valued = () if values is None else (ptr(values),)
    pushed_suffix = "_pushed" if pushed else ""
    if output == "critic":
        pair = twin is not None
        return "ktb_mlp_bf16_critic" + ("_twin" if pair else "") + pushed_suffix, \
            (*(twin or ()), act, ptr(logits), *((ptr(actions), ptr(log_probs)) if pair else ()))
    if output == "deterministic":
        return "ktb_mlp_bf16_policy_deterministic" + pushed_suffix, (*det, seed or 0, row_base, ptr(actions))
    if output == "gaussian_evaluate":
        return "ktb_mlp_bf16_policy_gaussian_evaluate" + ("" if values is None else "_value") + pushed_suffix, \
            (ptr(log_std), taken, ptr(log_probs), ptr(actions), *valued)
    if output == "evaluate":
        groups = (None, 0) if nvec is None else (L.arr(ctypes.c_int32, nvec), len(nvec))
        return "ktb_mlp_bf16_policy_evaluate" + ("" if mask is None else "_masked") + \
            ("" if values is None else "_value") + pushed_suffix, \
            (*groups, *(() if mask is None else (mask,)), taken, ptr(log_probs), ptr(actions), *valued)
    eps = output == "epsilon_greedy"
    suffix = ("" if nvec is None else "_multidiscrete") + ("" if mask is None else "_masked") + \
        ("" if values is None or eps else "_value") + ("_pushed" if pushed else "")
    grouped = () if nvec is None else (L.arr(ctypes.c_int32, nvec), len(nvec))
    masked = () if mask is None else (mask,)
    valued = () if values is None else (ptr(values),)
    if output == "gaussian" and std is not None:
        return "ktb_mlp_bf16_policy_gaussian_state" + suffix, (*std, seed, row_base, ptr(actions), ptr(log_probs),
                                                               *valued)
    if output == "gaussian":
        return "ktb_mlp_bf16_policy_gaussian" + suffix, (ptr(log_std), seed, row_base, ptr(actions), ptr(log_probs),
                                                         *valued)
    if eps:
        return "ktb_mlp_bf16_policy_epsilon_greedy" + suffix, (*masked, epsilon, seed, row_base, ptr(actions),
                                                               ptr(log_probs), ptr(values))
    if output == "sample":
        return "ktb_mlp_bf16_policy_sample" + suffix, (*grouped, *masked, seed, row_base, ptr(actions), ptr(log_probs),
                                                       *valued)
    return "ktb_mlp_bf16_policy" + suffix, (*grouped, *masked, ptr(logits), ptr(actions))


def _std(log_std, log_std_bounds, squash):
    """The (log_std_min, log_std_max, squash) arguments of a _gaussian_state entry, or None for any other log_std."""
    if not isinstance(log_std, (tuple, list)):
        return None
    lo, hi = LOG_STD_BOUNDS if log_std_bounds is None else log_std_bounds
    return float(lo), float(hi), int(bool(squash))


def _det(noise, noise_clip, squash):
    """The (noise, noise_clip, squash) arguments of a _deterministic entry: no noise is σ = 0, no clip is +inf and
    squash defaults to True."""
    return (0.0 if noise is None else float(noise), math.inf if noise_clip is None else float(noise_clip),
            int(squash is None or squash))


def _rows(bufs, b, e):
    """Rows b .. e - 1 of each buffer; None stays None."""
    return [None if t is None else t[b:e] for t in bufs]


def _result(output, logits, actions, log_probs, values=None):
    """What a call with `output` returns, from its buffers."""
    if output == "logits":
        return logits
    if output == "actions":
        return actions
    if output == "both":
        return logits, actions
    if output in EVALUATE_OUTPUTS:   # the entropy rides in the actions slot
        return (log_probs, actions) if values is None else (log_probs, actions, values)
    if output == "deterministic":
        return actions
    if output == "critic":   # q, or (q1, q2, q_min) of a twin
        return logits if actions is None else (logits, actions, log_probs)
    return (actions, log_probs) if values is None else (actions, log_probs, values)


def mlp_forward(obs: torch.Tensor, w1: torch.Tensor, w2: torch.Tensor, w3: torch.Tensor,
                out: Optional[torch.Tensor] = None, device: Optional[int] = None,
                stream: Optional[torch.cuda.Stream] = None, staged: Optional[bool] = None,
                biases: Sequence[Optional[torch.Tensor]] = (None, None, None), output: str = "logits",
                actions: Optional[torch.Tensor] = None, seed: Optional[int] = None, row_offset: int = 0,
                log_probs: Optional[torch.Tensor] = None, log_std: Optional[torch.Tensor] = None,
                mask: Optional[torch.Tensor] = None, value: Optional[Sequence[Optional[torch.Tensor]]] = None,
                values: Optional[torch.Tensor] = None, nvec: Optional[Sequence[int]] = None,
                log_std_bounds: Optional[Tuple[float, float]] = None, squash: Optional[bool] = None,
                epsilon=None, q: Optional[torch.Tensor] = None, q_max: Optional[torch.Tensor] = None,
                taken: Optional[torch.Tensor] = None, entropy: Optional[torch.Tensor] = None,
                noise: Optional[float] = None, noise_clip: Optional[float] = None,
                action: Optional[torch.Tensor] = None, twin: Optional[Sequence[Optional[torch.Tensor]]] = None,
                q2: Optional[torch.Tensor] = None, q_min: Optional[torch.Tensor] = None,
                actor: Optional[Sequence[Optional[torch.Tensor]]] = None, policy: Optional[str] = None,
                reward: Optional[torch.Tensor] = None, done: Optional[torch.Tensor] = None,
                gamma: Optional[float] = None, alpha: Optional[float] = None, target: Optional[torch.Tensor] = None,
                online: Optional[Sequence[Optional[torch.Tensor]]] = None, _stacked: bool = False):
    """logits[M, d_out] = W3·relu(W2·relu(W1·obsᵀ + b1) + b2) + b3; bf16 storage, fp32 accumulation in registers,
    each bias added to the fp32 accumulator (nn.Linear).  `biases` = (b1, b2, b3), each optional.  `output` is
    "logits" (returns the logits), "actions" (returns int64 argmax actions[M]; no logits are written), "both"
    (returns (logits, actions)), "sample" (returns (actions, log_probs): int64 actions drawn from
    softmax(logits) by Gumbel-max with the noise of kubetorch_b200.sampling.gumbel_noise(seed, row_offset, M, d_out),
    and the fp32 log_softmax(logits)[action] of each row; no logits are written) or "gaussian" (returns (actions,
    log_probs): fp32 actions[M, d_out] = logits + exp(log_std)·normal_noise(seed, row_offset, M, d_out) and the fp32
    log-density of each row's action under Normal(logits, exp(log_std)); no logits are written).  `obs` / `out` /
    `actions` / `log_probs` may be peer-mapped (pull the observations / push the results over NVLink).  Without
    biases, at d_out == 64 and with logits only the logits equal ktb_mlp_bf16's.  `mask`, a bool [M, d_out] tensor on
    the device of obs (True: legal), applies a per-row legal-action mask to every output but "gaussian": the head
    computes logits.masked_fill(~mask, -inf) and stores, ranks and samples those masked logits; an all-True mask gives
    the unmasked bits.  `value` = (wv, bv), with output="sample" or "gaussian" (masked or not), adds the state value of
    a critic nn.Linear(d_hidden, 1) on the same trunk (wv its bf16 weight [1, d_hidden], bv its bf16 bias [1], given
    exactly when b3 is): the call returns (actions, log_probs, values) with fp32 values[M] = F.linear(h, wv, bv), the
    bf16 result widened exactly, into `values` when given; the actions and log-probabilities keep their bits.  The
    head then runs over W3v = [w3; wv], stacked once per device and head (_stacked_head).  `nvec` = (n_0, ...,
    n_{G-1}), ints >= 1 summing to d_out, with output="actions", "both" or "sample" (masked or not, and with a value
    head where "sample" takes one), makes the head multi-discrete: group g is the columns [lo_g, lo_g + n_g) with lo_g
    = n_0 + ... + n_{g-1}, actions are int64 [M, G] of group-relative indices (the greedy or sampled action of each
    group's logits alone, with the noise of "sample"), and log_probs[i] is the fp32 sum of the groups'
    log_softmax(group)[a_g] in group order; a group with no legal action takes action 0 with a NaN log-probability.
    The logits of "both" and nvec = (d_out,) keep the bits of the call without nvec.  With output="gaussian",
    `log_std` = (w_ls, b_ls) makes the log-std state-dependent (SAC's actor): w_ls a bf16 [d_out, d_hidden] and b_ls a
    bf16 [d_out] (given exactly when b3 is), so ls = F.linear(h, w_ls, b_ls).float() clamped to `log_std_bounds`
    (default (-20.0, 2.0); a NaN stays NaN), u = logits + exp(ls)·normal_noise(seed, row_offset, M, d_out), actions
    are tanh(u) with `squash=True` and u otherwise, and log_probs the Normal log-density of u minus, when squashed,
    sum_j log(1 - tanh(u_j)^2), taken exactly as 2·(log 2 - |u| - softplus(-2|u|)) (not SB3's
    log(1 - tanh^2 + 1e-6), which differs where |u| > about 7).  The head then runs over the interleaved rows of w3 and
    w_ls (_stacked_head), at most 128 actions (127 with a value head).  log_std_bounds and squash are refused with a
    tensor log_std.  output="epsilon_greedy" (a Q-network's actor; masked or not, with `seed`) returns (actions, q,
    q_max): with u, w = kubetorch_b200.sampling.explore_noise(seed, row_offset, M, d_out), row i explores iff u[i] <
    epsilon[i] in fp32 and then takes the legal column with the largest w (ties to the lower column), and otherwise
    the argmax of its (masked) logits; q is the fp32 (masked) logit of the action taken and q_max that of the argmax,
    into `q` and `q_max` when given; no logits are written.  `epsilon` is a CUDA float32 tensor [M] on the device of
    obs or a number broadcast to every row (rounded to fp32; NaN refused).  output="evaluate" (masked, multi-discrete
    and with a value head as "sample" takes them) and "gaussian_evaluate" (with a tensor log_std, and a value head)
    score the actions `taken` on the device of obs (int64 [M], [M, len(nvec)] with nvec, of group-relative indices; fp32
    [M, d_out] for the Gaussian) and return (log_probs, entropy), or (log_probs, entropy, values) with a value head,
    into `log_probs`, `entropy` and `values` when given: fp32 log_probs[i] = sum_g log_softmax(group_g)[a_g] of the
    (masked) logits and entropy[i] = sum_g entr(softmax(group_g)).sum(), or Normal(logits, exp(log_std))'s
    log_prob(taken).sum(-1) and entropy().sum(-1); an action out of range gives a NaN row (it is not checked, which
    would need a host synchronisation), an illegal one -inf.  No noise is drawn and no logits are written.
    output="deterministic" (DDPG's and TD3's actor) returns fp32 actions[M, d_out], into `actions` when given:
    t = tanh(logits.float()) with `squash` True or None, logits.float() with squash=False; with `noise` σ >= 0 (and then
    `seed`) t + (σ·normal_noise(seed, row_offset, M, d_out)).clamp(-noise_clip, noise_clip), noise_clip >= 0 defaulting
    to +inf; then clamp(-1, 1) when squashed (NaN stays NaN).  σ = 0.1 is exploration, σ = 0.2 with noise_clip = 0.5
    TD3's target policy smoothing, no noise the deterministic mode of a tanh-squashed or an unsquashed policy.
    output="critic" (SAC's and TD3's Q(s, a), forward only) returns fp32 q[M], into `q` when given: with `action` an
    fp32 [M, d_act] tensor on the device of obs (1 <= d_act <= 64), w1 the critic's [d_hidden, d_in + d_act] and w3
    its [1, d_hidden], q = F.linear(h2, w3, b3).float() over x = torch.cat([obs, action.to(torch.bfloat16)], -1), every
    layer rounded as above.  With `twin` = (w1, b1, w2, b2, w3, b3) of a second critic (biases given exactly as the
    first's) it returns (q1, q2, q_min), into `q`, `q2` and `q_min` when given: q_min = torch.minimum(q1, q2) (NaN
    when either is, q1 on ties).  Layer 1 runs over w1 padded with zero columns to d_in + 64 (_padded_w1, kept per
    device and weight) and reads the actions, packed to bf16 once per row chunk, as its last K block; the
    observations are never copied.  output="td_target" (the Bellman target of TD3, DDPG and SAC, forward only)
    returns fp32 y of the shape of `reward`, into `target` when given: obs are the next observations, w1, w2, w3 and
    biases the (target) critic's and `twin` an optional second one, as with "critic"; `actor` = (w1, b1, w2, b2, w3,
    b3) is the (target) actor, biases given exactly when the critic's are, w3 [d_act, d_ha] with its own d_ha.  With
    policy="deterministic" (TD3, DDPG) the next actions are output="deterministic"'s with `noise`, `noise_clip`,
    `seed` and `squash`; with policy="gaussian" (SAC) they and their log-probabilities are output="gaussian"'s with
    log_std = (w_ls, b_ls), `log_std_bounds`, `squash` and `seed`, the noise of global rows row_offset, ....  Then
    t = q (q_min with a twin), less alpha * logp with "gaussian", and y = reward + gamma * (1 - done) * t evaluated in
    fp32 as torch evaluates that expression; `reward` and `done` are fp32 [M] or [M, 1] on the device of obs, and gamma
    and alpha finite numbers (alpha required with "gaussian" and refused with "deterministic").  Per row chunk the
    actor's actions stay in scratch and feed the critics' action tile; nothing M-sized but y is written.
    output="dqn_target" (the Bellman target of DQN and Double DQN, forward only) returns fp32 y of the shape of
    `reward`, into `target` when given: obs are the next observations, w1, w2, w3 and biases the target Q-network's and
    `online` = (w1, b1, w2, b2, w3, b3) an optional online Q-network of the same shapes (biases given exactly when the
    target's are).  The next action a* is the argmax of the online network's logits (Double DQN) or of the target's
    (DQN), masked with `mask` (bool [M, d_out] legal actions of the next states) when given, with output="actions"'s
    rules; q = the target's logit at a*, UNMASKED, widened to fp32; and y = reward + gamma * (1 - done) * q evaluated
    as torch evaluates it (so a terminal row with no legal action gives y = reward at done = 1).  `reward`, `done` and
    `gamma` as with "td_target".  Per row chunk a* stays in scratch; nothing M-sized but y is written.
    `_stacked` (internal, from
    mlp_scatter_gather, which checked the call): w3 and biases[2] are
    already the head the C entry takes (stacked with a value head, interleaved with a log-std head), and a critic's
    w1 (and its twin's) is already W1p; a TD target's actor w3 and b3 are already interleaved with its log-std head."""
    for name, t in (("obs", obs), ("w1", w1), ("w2", w2), ("w3", w3)):
        if t.dtype != torch.bfloat16 or not t.is_cuda or not t.is_contiguous():
            raise ValueError(f"{name} must be a contiguous CUDA bfloat16 tensor")
    dev = w1.device.index if device is None else int(device)
    ops.ensure_init({dev, obs.device.index})
    M, d_in = obs.shape
    d_hidden, d_out = w1.shape[0], w3.shape[0]
    critic = output == "critic"
    td = (actor, policy, reward, done, gamma, alpha)
    # a critic's layer 1 also reads the actions: checked by _check_critic and _check_td_target
    d_w1 = w1.shape[1] if critic or output == "td_target" else d_in
    if w1.shape != (d_hidden, d_w1) or w2.shape != (d_hidden, d_hidden) or w3.shape != (d_out, d_hidden):
        raise ValueError("weight shapes must be W1[d_h,d_in], W2[d_h,d_h], W3[d_out,d_h] (nn.Linear layout)")
    if not _stacked:
        _check_policy(w1, w3, biases, output, seed, log_std, mask, obs, value, nvec, log_std_bounds, squash, epsilon,
                      taken, noise, noise_clip, action, twin, w2, td, online)
    if output == "td_target":
        return _td_target(obs, w1, w2, w3, biases, twin, td, seed, log_std, log_std_bounds, squash, noise, noise_clip,
                          row_offset, target, dev, stream if stream is not None else torch.cuda.current_stream(dev),
                          staged, _stacked)
    if output == "dqn_target":
        return _dqn_target(obs, w1, w2, w3, biases, online, mask, reward, done, gamma, target, dev,
                           stream if stream is not None else torch.cuda.current_stream(dev), staged)
    std = _std(log_std, log_std_bounds, squash) if output == "gaussian" else None
    valued = value is not None or (_stacked and values is not None)
    if _stacked:
        d_out = (d_out - valued) // (2 if std is not None else 1)
    if output in ("sample", "gaussian", "epsilon_greedy", "deterministic") and \
            (isinstance(row_offset, bool) or not isinstance(row_offset, int) or row_offset < 0):
        raise ValueError(f"row_offset must be a non-negative int, got {row_offset!r}")
    eps = output == "epsilon_greedy"
    if eps:   # q and q_max ride in the log_probs and values slots
        log_probs, values = q, q_max
    if output in EVALUATE_OUTPUTS:   # the entropy rides in the actions slot
        actions = entropy
    if critic:   # q (or q1), q2 and q_min ride in the logits, actions and log_probs slots
        out, actions, log_probs = q, q2, q_min
        d_out = action.shape[1]   # the C entry's d_act
    out, actions, log_probs, values = _outputs(output, M, d_out, f"cuda:{dev}", out, actions, log_probs, values, valued,
                                               nvec, twin is not None)
    s = stream if stream is not None else torch.cuda.current_stream(dev)
    if critic and not _stacked:
        with torch.cuda.stream(s):   # a rewrite of W1p is ordered after earlier calls on s
            w1 = _padded_w1(w1, d_in)
            if twin is not None:
                twin = (_padded_w1(twin[0], d_in), *twin[1:])
    if eps and not isinstance(epsilon, torch.Tensor):
        with torch.cuda.stream(s):   # freed after the call, its memory is reused in s's order, after the kernel
            epsilon = torch.full((M,), float(epsilon), dtype=torch.float32, device=f"cuda:{dev}")
    if not _stacked and (value is not None or std is not None):
        with torch.cuda.stream(s):   # a rewrite of the stacked head is ordered after earlier calls on s
            w3, b3 = _stacked_head(w3, biases[2], *(value or (None, None)), *(log_std if std is not None else ()))
        biases = (biases[0], biases[1], b3)
    if staged is None:
        staged = obs.device.index != dev   # observations on another GPU: pull each row chunk over NVLink once
    ptr = lambda t: 0 if t is None else t.data_ptr()   # noqa: E731
    entry, head = _head(output, out, actions, log_probs, seed, row_offset, log_std, ptr,
                        mask=None if mask is None else ptr(mask), values=values, nvec=nvec, std=std,
                        epsilon=ptr(epsilon) if eps else None, taken=ptr(taken),
                        det=_det(noise, noise_clip, squash) if output == "deterministic" else None,
                        act=ptr(action), twin=None if twin is None else tuple(ptr(t) for t in twin))
    L.call(entry, dev, obs.data_ptr(), M, d_in, d_hidden, d_out, w1.data_ptr(), ptr(biases[0]), w2.data_ptr(),
           ptr(biases[1]), w3.data_ptr(), ptr(biases[2]), *head, _scratch_for(dev, M, d_hidden, critic).data_ptr(),
           _stage_for(dev, M, d_in).data_ptr() if staged else 0, int(s.cuda_stream))
    return _result(output, out, actions, log_probs, values)


def _td_args(policy, seed, log_std, log_std_bounds, squash, noise, noise_clip, row_offset):
    """The policy's arguments of a _td_target entry: those of the standalone _deterministic or _gaussian_state entry,
    (noise, noise_clip, squash) or (log_std_min, log_std_max, squash), then seed (0 for a noise-free actor, which draws
    nothing) and row_base."""
    if policy == "deterministic":
        return (*_det(noise, noise_clip, squash), seed or 0, row_offset)
    return (*_std(log_std, log_std_bounds, squash), seed, row_offset)


def _td_target(obs, w1, w2, w3, biases, twin, td, seed, log_std, log_std_bounds, squash, noise, noise_clip,
               row_offset, target, dev, s, staged, stacked):
    """mlp_forward's output="td_target" on `dev` and stream `s`: y of the shape of reward, into `target` when given."""
    actor, policy, reward, done, gamma, alpha = td
    if isinstance(row_offset, bool) or not isinstance(row_offset, int) or row_offset < 0:
        raise ValueError(f"row_offset must be a non-negative int, got {row_offset!r}")
    M, d_in = obs.shape
    gaussian = policy == "gaussian"
    aw1, ab1, aw2, ab2, aw3, ab3 = actor
    if target is None:
        target = torch.empty(reward.shape, dtype=torch.float32, device=f"cuda:{dev}")
    else:
        ops.ensure_init({target.device.index})
    if not stacked:
        with torch.cuda.stream(s):   # a rewrite of W1p or of the interleaved head is ordered after earlier calls on s
            w1 = _padded_w1(w1, d_in)
            if twin is not None:
                twin = (_padded_w1(twin[0], d_in), *twin[1:])
            if gaussian:
                aw3, ab3 = _stacked_head(aw3, ab3, None, None, *log_std)
    d_act = aw3.shape[0] // (2 if gaussian else 1)
    if staged is None:
        staged = obs.device.index != dev
    ptr = lambda t: 0 if t is None else t.data_ptr()   # noqa: E731
    lib = L.load()
    scratch = _cached_buffer(_scratch, dev, dev,
                             lib.ktb_mlp_td_target_scratch_bytes(M, aw1.shape[0], w1.shape[0], d_act))
    L.call("ktb_mlp_bf16_td_target_" + policy, dev, obs.data_ptr(), M, d_in, w1.shape[0], d_act, w1.data_ptr(),
           ptr(biases[0]), w2.data_ptr(), ptr(biases[1]), w3.data_ptr(), ptr(biases[2]),
           *(ptr(t) for t in (twin or (None,) * 6)), aw1.shape[0], *(ptr(t) for t in (aw1, ab1, aw2, ab2, aw3, ab3)),
           *_td_args(policy, seed, log_std, log_std_bounds, squash, noise, noise_clip, row_offset), reward.data_ptr(),
           done.data_ptr(), float(gamma), *((float(alpha),) if gaussian else ()), target.data_ptr(),
           scratch.data_ptr(), _stage_for(dev, M, d_in).data_ptr() if staged else 0, int(s.cuda_stream))
    return target


def _dqn_target(obs, w1, w2, w3, biases, online, mask, reward, done, gamma, target, dev, s, staged):
    """mlp_forward's output="dqn_target" on `dev` and stream `s`: y of the shape of reward, into `target` when given."""
    M, d_in = obs.shape
    if target is None:
        target = torch.empty(reward.shape, dtype=torch.float32, device=f"cuda:{dev}")
    else:
        ops.ensure_init({target.device.index})
    if staged is None:
        staged = obs.device.index != dev
    ptr = lambda t: 0 if t is None else t.data_ptr()   # noqa: E731
    scratch = _cached_buffer(_scratch, dev, dev, L.load().ktb_mlp_dqn_target_scratch_bytes(M, w1.shape[0]))
    L.call("ktb_mlp_bf16_dqn_target" + ("" if mask is None else "_masked"), dev, obs.data_ptr(), M, d_in, w1.shape[0],
           w3.shape[0], w1.data_ptr(), ptr(biases[0]), w2.data_ptr(), ptr(biases[1]), w3.data_ptr(), ptr(biases[2]),
           *(ptr(t) for t in (online or (None,) * 6)), *(() if mask is None else (mask.data_ptr(),)), reward.data_ptr(),
           done.data_ptr(), float(gamma), target.data_ptr(), scratch.data_ptr(),
           _stage_for(dev, M, d_in).data_ptr() if staged else 0, int(s.cuda_stream))
    return target


def _weights_on(dev: int, ws: Sequence[torch.Tensor]) -> List[torch.Tensor]:
    """Weights are shared by all ranks: broadcast once per (weights, device) and kept resident
    (excluded from per-call bytes, SURVEY.md §8(d) C4)."""
    out = []
    for w in ws:
        if w is None or w.device.index == dev:
            out.append(w)
            continue
        key = (w.data_ptr(), w._version, dev)
        c = _weight_cache.get(key)
        if c is None:
            c = torch.empty_like(w, device=f"cuda:{dev}")
            ops.broadcast(w, [c])
            torch.cuda.synchronize(w.device)
            _weight_cache[key] = c
        out.append(c)
    return out


PUSH_CHUNK_ROWS = 16896      # 132 SMs x 128 rows: each 256-wide layer of a chunk is whole waves of 128 x 256 tiles


def _use_push(devs, bounds, transfer) -> bool:
    """Whether a scatter→exec→gather call takes the push form: distinct devices, shards of whole 128-row blocks and at
    most 64 chunks each, unless transfer="pull"; transfer="push" without them is a ValueError."""
    distinct = len(set(devs)) == len(devs) and len(devs) > 1
    pushable = distinct and all((e - b) % 128 == 0 for b, e in bounds) and \
        -(-max(e - b for b, e in bounds) // PUSH_CHUNK_ROWS) <= 64
    if transfer == "push" and not pushable:
        raise ValueError("push transfer needs distinct devices and shards of a multiple of 128 rows")
    return pushable and transfer != "pull"
_push_sessions = {}          # device tuple -> ops.PushSession
_push_scratch = {}           # (device tuple, rank) -> scratch of that rank's pushed GEMMs


def _stage_layout(rows: int, d_in: int, sides) -> Tuple[dict, int]:
    """The staging half of a pushed call whose largest shard has `rows` rows of d_in bf16 observations: the rows, then
    each side input (name, bytes per row) of `sides` in order, 256-byte aligned after the previous region.  Returns the
    sides' offsets by name and the half's bytes."""
    offsets, end = {}, rows * d_in * 2
    for name, row_bytes in sides:
        offsets[name] = (end + 255) // 256 * 256
        end = offsets[name] + rows * row_bytes
    return offsets, end


def _forward_rows(obs_root, b, e, dev, stream, staged, ws, bufs, output, seed, log_std, mask, nvec, std, epsilon,
                  taken, det, action, twin, td) -> None:
    """mlp_forward of rows b .. e - 1 of a scatter→exec→gather call on `dev` and `stream`, into those rows of `bufs`:
    the arguments of _mlp_scatter_gather_pushed, with ws, log_std and twin those on `dev`."""
    logits, actions, log_probs, values = _rows(bufs, b, e)
    valued = values is not None and epsilon is None   # an ε-greedy head's values slot is its q_max
    target = {}   # a TD or DQN target's options, its y in the logits slot
    if td is not None:
        target = dict(reward=td[2][b:e], done=td[3][b:e], gamma=td[4], target=logits)
        target.update(dict(online=None if td[0] is None else td[0][dev]) if output == "dqn_target" else
                      dict(actor=td[0][dev], policy=td[1], alpha=td[5], twin=twin))
    mlp_forward(obs_root[b:e], ws[0], ws[1], ws[2], out=logits, device=dev, stream=stream, staged=staged,
                biases=ws[3:], output=output, actions=actions, seed=seed, row_offset=b, log_probs=log_probs,
                log_std=log_std, mask=None if mask is None else mask[b:e], values=values, nvec=nvec,
                log_std_bounds=None if std is None else std[:2],
                **(det or dict(squash=None if std is None else bool(std[2]))),
                **({} if epsilon is None else dict(epsilon=epsilon[b:e], q=log_probs, q_max=values)),
                **({} if taken is None else dict(taken=taken[b:e], entropy=actions)),
                **({} if output != "critic" else dict(action=action[b:e], twin=twin, q=logits, q2=actions,
                                                       q_min=log_probs)),
                **target,
                _stacked=valued or std is not None or output == "critic" or td is not None)


def _mlp_scatter_gather_pushed(obs_root, devs, bounds, weights, output, out_root, actions_root, log_probs_root=None,
                               seed=None, log_std=None, mask=None, values_root=None, nvec=None, std=None,
                               epsilon=None, taken=None, det=None, action=None, twin=None, td=None) -> None:
    """The root PUSHES each rank's observation rows in GEMM-sized chunks (copy engines, posted NVLink writes, flags in
    device memory); every rank's GEMM chain consumes chunk c as soon as it has landed and stores its logits (and/or
    actions) straight into the root's result; the root's own shard runs on the session's side stream beside the scatter.
    No host synchronisation, no events between devices.  weights[dev] = (w1, w2, w3, b1, b2, b3) on that device (biases
    may be None); out_root / actions_root / log_probs_root are None when `output` does not want them (with "gaussian",
    actions_root holds the fp32 actions [M, d_out]).  log_std[dev] is the Gaussian head's log_std on that device.  With
    output="sample" or "gaussian" rank r draws the noise of global rows b_r .. e_r - 1 (its shard's place in obs_root).
    A legal-action `mask` [M, d_out] on the root travels with its rows: the copy engines push each rank's mask rows into
    the same staging half (_stage_layout), so no rank reads the root's memory; every other per-row input below travels
    the same way.  With `values_root` (fp32 [M]) weights[dev] holds the stacked W3v and b3v in place of w3 and b3, and
    each rank stores its values there too.  `nvec` picks every rank's multi-discrete entry.  `std` (_std) picks every
    rank's _gaussian_state entry, weights[dev] then holding the interleaved head.  With output="epsilon_greedy",
    `epsilon` is the fp32 [M] on the root, pushed with the rows like the mask, and log_probs_root / values_root are its
    q and q_max.  With output="evaluate" or "gaussian_evaluate", `taken` (on the root) is pushed with the rows, and
    actions_root is the entropy.  With output="deterministic", `det` is the call's dict(noise=, noise_clip=, squash=),
    and each staging half holds the rows only.  With output="critic", `action` (fp32 [M, d_act] on the root) is pushed
    with the rows, weights[dev] holds W1p in place of w1, twin[dev] (unless None) the second critic's (W1p, b1, W2, b2,
    W3, b3), and out_root / actions_root / log_probs_root are q (q1), q2 and q_min.  With output="td_target", td =
    (actors, policy, reward, done, gamma, alpha): actors[dev] is the actor's six weights and biases on that device (its
    head interleaved with the log-std head for policy="gaussian", picked by `std`; "deterministic" by `det`), reward and
    done (on the root) are pushed with the rows, weights[dev] and twin[dev] are the target critics as with "critic", and
    out_root is y.  With output="dqn_target", td = (onlines, None, reward, done, gamma, None): onlines[dev] (None for
    DQN) is the online network's six weights and biases on that device, the mask (unless None) and one side of
    interleaved (reward, done) pairs, stacked on the root, are pushed with the rows, and out_root is y."""
    root, n, key = devs[0], len(devs), tuple(devs)
    critic = output == "critic"
    valued = values_root is not None and epsilon is None   # an ε-greedy head's values_root is its q_max
    d_in, d_hidden = obs_root.shape[1], weights[root][0].shape[0]
    actors, policy, reward, done, gamma, alpha = td or (None,) * 6
    dqn = output == "dqn_target"
    rd = None
    if dqn:   # one side of (reward, done) pairs: the pushed entries take at most two sides, the mask one of them
        rd, reward, done = torch.stack((reward.reshape(-1), done.reshape(-1)), 1), None, None
    if td is not None and not dqn:   # the entry's d_act
        d_out = actors[root][4].shape[0] // (2 if std is not None else 1)
    else:
        d_out = action.shape[1] if critic else (weights[root][2].shape[0] - valued) // (2 if std is not None else 1)
    rows = max(e - b for b, e in bounds)
    taken_row = None if taken is None else taken[0].numel() * taken.element_size() if taken.dim() > 1 else \
        taken.element_size()
    sides = [(name, t, row_bytes) for name, t, row_bytes in
             (("mask", mask, d_out), ("epsilon", epsilon, 4), ("taken", taken, taken_row), ("act", action, 4 * d_out),
              ("reward", reward, 4), ("done", done, 4), ("rd", rd, 8)) if t is not None]
    offsets, stage_bytes = _stage_layout(rows, d_in, [(name, row_bytes) for name, _, row_bytes in sides])
    sess = _push_sessions.get(key)
    if sess is None or sess.stride < stage_bytes:
        sess = _push_sessions[key] = ops.PushSession(devs, stage_bytes)
    try:
        seq = sess.begin()
    except ops.PushTimeout:
        del _push_sessions[key]
        raise
    # scratch per rank, not per device: ranks sharing a device must not share one, nor the root's own shard on the
    # side stream
    if dqn:   # the chunk's int64 actions after the hidden activations
        scratch_bytes = pushed_scratch_bytes(rows, d_hidden, PUSH_CHUNK_ROWS) + min(PUSH_CHUNK_ROWS, rows) * 8
    elif td is not None:
        scratch_bytes = pushed_td_scratch_bytes(rows, actors[root][0].shape[0], d_hidden, d_out, PUSH_CHUNK_ROWS)
    else:
        scratch_bytes = pushed_scratch_bytes(rows, d_hidden, PUSH_CHUNK_ROWS, critic)
    scratch = [None] + [_cached_buffer(_push_scratch, (key, r), devs[r], scratch_bytes) for r in range(1, n)]
    streams = [ops.current_stream_handle(d) for d in devs]
    bufs = (out_root, actions_root, log_probs_root, values_root)
    b0, e0 = bounds[0]
    own = e0 > b0
    if own:
        _forward_rows(obs_root, b0, e0, root, sess.fork(), False, weights[root], bufs, output, seed,
                      None if log_std is None else log_std[root], mask, nvec, std, epsilon, taken, det, action,
                      None if twin is None else twin[root], td)
    scatter = (L.arr(ctypes.c_int, devs), sess.stage_ptrs, sess.stride, sess.ctrl_ptrs, sess.ctrl[0].data_ptr(),
               PUSH_CHUNK_ROWS * d_in)
    if sides:
        L.call("ktb_push_scatter_ce_sides", root, obs_root.data_ptr(), obs_root.numel(), d_in, L.BF16, n, 0, *scatter,
               len(sides), L.arr(ctypes.c_void_p, [t.data_ptr() for _, t, _ in sides]),
               L.arr(ctypes.c_size_t, [row_bytes for _, _, row_bytes in sides]),
               L.arr(ctypes.c_size_t, [offsets[name] for name, _, _ in sides]), seq, streams[0])
    else:
        L.call("ktb_push_scatter_ce", root, obs_root.data_ptr(), obs_root.numel(), d_in, L.BF16, n, 0, *scatter, seq,
               streams[0])

    # a TD target's actor options as mlp_forward takes them
    pol = det or dict(log_std_bounds=None if std is None else std[:2], squash=None if std is None else std[2])

    def issue(r):
        b, e = bounds[r]
        ws = weights[devs[r]]
        ptr = lambda t: 0 if t is None or e == b else t.data_ptr()   # noqa: E731
        logits, actions, log_probs, values = _rows(bufs, b, e)
        wptr = lambda t: 0 if t is None else t.data_ptr()   # noqa: E731
        if dqn:   # y rides in the logits slot
            entry = "ktb_mlp_bf16_dqn_target" + ("" if mask is None else "_masked") + "_pushed"
            head = (*(wptr(t) for t in (actors[devs[r]] if actors is not None else (None,) * 6)),
                    *(() if mask is None else (offsets["mask"],)), offsets["rd"], float(gamma), ptr(logits))
        elif td is not None:   # y rides in the logits slot
            entry = "ktb_mlp_bf16_td_target_" + policy + "_pushed"
            head = (*(wptr(t) for t in (twin[devs[r]] if twin is not None else (None,) * 6)),
                    actors[root][0].shape[0], *(wptr(t) for t in actors[devs[r]]),
                    *_td_args(policy, seed, None if log_std is None else log_std[devs[r]], pol.get("log_std_bounds"),
                              pol["squash"], pol.get("noise"), pol.get("noise_clip"), b),
                    offsets["reward"], offsets["done"], float(gamma), *((float(alpha),) if policy == "gaussian" else ()),
                    ptr(logits))
        else:
            entry, head = _head(output, logits, actions, log_probs, seed, b,
                                None if log_std is None else log_std[devs[r]], ptr, pushed=True,
                                mask=offsets.get("mask"), values=values, nvec=nvec, std=std,
                                epsilon=offsets.get("epsilon"), taken=offsets.get("taken"),
                                det=None if det is None else _det(**det), act=offsets.get("act"),
                                twin=None if twin is None else tuple(ptr(t) for t in twin[devs[r]]))
        L.call(entry, devs[r], sess.stage[r].data_ptr(), sess.stride, e - b, d_in, d_hidden, d_out, ws[0].data_ptr(),
               ptr(ws[3]), ws[1].data_ptr(), ptr(ws[4]), ws[2].data_ptr(), ptr(ws[5]), *head, scratch[r].data_ptr(),
               sess.ctrl[r].data_ptr(), sess.ctrl[0].data_ptr(), r, PUSH_CHUNK_ROWS, seq, streams[r])

    list(_thread_pool().map(issue, range(1, n)))
    sess.finish(seq, joined=own)


def mlp_scatter_gather(obs_root: torch.Tensor, w1, w2, w3, devices: Sequence[int],
                       out_root: Optional[torch.Tensor] = None, transfer: str = "auto",
                       biases: Sequence[Optional[torch.Tensor]] = (None, None, None), output: str = "logits",
                       actions_root: Optional[torch.Tensor] = None, seed: Optional[int] = None,
                       log_probs_root: Optional[torch.Tensor] = None, log_std: Optional[torch.Tensor] = None,
                       mask: Optional[torch.Tensor] = None, value: Optional[Sequence[Optional[torch.Tensor]]] = None,
                       values_root: Optional[torch.Tensor] = None, nvec: Optional[Sequence[int]] = None,
                       log_std_bounds: Optional[Tuple[float, float]] = None, squash: Optional[bool] = None,
                       epsilon=None, taken: Optional[torch.Tensor] = None,
                       entropy_root: Optional[torch.Tensor] = None, noise: Optional[float] = None,
                       noise_clip: Optional[float] = None, action: Optional[torch.Tensor] = None,
                       twin: Optional[Sequence[Optional[torch.Tensor]]] = None,
                       q_root: Optional[torch.Tensor] = None, q2_root: Optional[torch.Tensor] = None,
                       q_min_root: Optional[torch.Tensor] = None,
                       actor: Optional[Sequence[Optional[torch.Tensor]]] = None, policy: Optional[str] = None,
                       reward: Optional[torch.Tensor] = None, done: Optional[torch.Tensor] = None,
                       gamma: Optional[float] = None, alpha: Optional[float] = None,
                       target_root: Optional[torch.Tensor] = None,
                       online: Optional[Sequence[Optional[torch.Tensor]]] = None) -> list:
    """Rank r runs the MLP on `obs.chunk(world)[r]`: its first GEMM's TMA loads read the rows straight
    from the root GPU (scatter) and its last epilogue stores the logits straight into the root's
    result buffer (gather). Returns rank-ordered views of the root result: logits views for output="logits",
    int64 actions views for "actions", (logits, actions) pairs for "both", (actions, log_probs) pairs for "sample"
    and "gaussian" (fp32 actions [rows, d_out] with the latter), (actions, log_probs, values) triples with a value head.
    With "sample" or "gaussian" rank r draws the noise of the global rows of its shard (row_offset = its shard's begin),
    so the result does not depend on the number of ranks or their devices.  `biases`, `seed`, `log_std`, `mask` and
    `value` as in mlp_forward; the mask lives on the root GPU and each rank applies its rows of it (read in place by
    the pull form, pushed with the rows by the push form); the head with the value head stacked under it is built on
    the root and copied to the other devices like the other weights, and every rank stores its values into
    `values_root` (allocated on the root when None).  `nvec` as in mlp_forward: actions are [rows, G] views.
    A state-dependent log_std = (w_ls, b_ls), with `log_std_bounds` and `squash`, as in mlp_forward: the interleaved
    head is built on the root and copied to the other devices like the other weights.  output="epsilon_greedy" with
    `epsilon` (a float, or an fp32 [M] on the root) as in mlp_forward returns (actions, q, q_max) triples; each rank
    reads its rows of ε in place on the pull form, and the push form pushes them with the rows.  output="evaluate" and
    "gaussian_evaluate" with `taken` on the root as in mlp_forward return (log_probs, entropy) pairs, or triples with
    a value head, into `log_probs_root`, `entropy_root` and `values_root` when given; each rank reads its rows of taken
    in place on the pull form, and the push form pushes them with the rows.  output="deterministic" with `noise`,
    `noise_clip`, `seed` and `squash` as in mlp_forward returns fp32 actions [rows, d_out] views of `actions_root`;
    each rank draws the noise of its shard's global rows.  output="critic" with `action` (fp32 [M, d_act] on the root)
    and `twin` as in mlp_forward returns fp32 q [rows] views of `q_root`, or (q1, q2, q_min) triples of views of
    `q_root`, `q2_root` and `q_min_root` with a twin; each rank reads its rows of action in place on the pull form, and
    the push form pushes them with the rows.  W1p (and the twin's) is built on the root and copied to the other devices
    like the other weights, again after an in-place update of w1.  output="td_target" with `actor`, `policy`, its
    options, `twin`, `reward`, `done` (on the root), `gamma` and `alpha` as in mlp_forward returns fp32 y views of
    `target_root` (of reward's shape, allocated on the root when None); each rank draws the noise of its shard's global
    rows, reads its rows of reward and done in place on the pull form, and the push form pushes them with the rows.
    output="dqn_target" with `online`, `mask`, `reward`, `done` (on the root) and `gamma` as in mlp_forward returns fp32
    y views of `target_root` likewise; the online network is copied to the other devices like the other weights, each
    rank reads its rows of mask, reward and done in place on the pull form, and the push form pushes them with the
    rows, reward and done as one side of interleaved pairs."""
    root = obs_root.device.index
    devs = [int(d) for d in devices]
    if devs[0] != root:
        raise ValueError("obs must live on the root GPU (devices[0])")
    td = (actor, policy, reward, done, gamma, alpha)
    _check_policy(w1, w3, biases, output, seed, log_std, mask, obs_root, value, nvec, log_std_bounds, squash, epsilon,
                  taken, noise, noise_clip, action, twin, w2, td, online)
    if transfer not in ("auto", "pull", "push"):
        raise ValueError("transfer must be 'auto', 'pull' or 'push'")
    critic, target, dqn = output == "critic", output == "td_target", output == "dqn_target"
    if critic:   # q (or q1), q2 and q_min ride in the logits, actions and log_probs slots
        out_root, actions_root, log_probs_root = q_root, q2_root, q_min_root
    det = dict(noise=noise, noise_clip=noise_clip, squash=squash) \
        if output == "deterministic" or target and policy == "deterministic" else None
    ops.ensure_init(set(devs))
    M = obs_root.shape[0]
    if output == "epsilon_greedy" and not isinstance(epsilon, torch.Tensor):   # before `ready`: every rank reads it
        epsilon = torch.full((M,), float(epsilon), dtype=torch.float32, device=obs_root.device)
    valued = value is not None
    if taken is not None:   # the entropy rides in the actions slot
        actions_root = entropy_root
    if target or dqn:   # y, of reward's shape, rides in the logits slot
        if target_root is None:
            target_root = torch.empty(reward.shape, dtype=torch.float32, device=obs_root.device)
        else:
            ops.ensure_init({target_root.device.index})
        bufs = (target_root, None, None, None)
    else:
        bufs = _outputs(output, M, w3.shape[0], obs_root.device, out_root, actions_root, log_probs_root, values_root,
                        valued, nvec, twin is not None)
    std = _std(log_std, log_std_bounds, squash) if output == "gaussian" or target and policy == "gaussian" else None
    if target and std is not None:   # the SAC actor's head interleaved with its log-std head
        actor = (*actor[:4], *_stacked_head(actor[4], actor[5], None, None, *log_std))
    elif valued or std is not None:
        w3, b3 = _stacked_head(w3, biases[2], *(value or (None, None)), *(log_std if std is not None else ()))
        biases = (biases[0], biases[1], b3)
    twins = None
    if critic or target:
        w1 = _padded_w1(w1, obs_root.shape[1])
        if twin is not None:
            twin = (_padded_w1(twin[0], obs_root.shape[1]), *twin[1:])
            twins = {dev: tuple(_weights_on(dev, twin)) for dev in set(devs)}
    root_stream = torch.cuda.current_stream(root)
    ready = torch.cuda.Event()
    ready.record(root_stream)
    bounds = [ops.shard_bounds(M, len(devs), r) for r in range(len(devs))]
    views = [target_root[b:e] if target or dqn else _result(output, *_rows(bufs, b, e)) for b, e in bounds]
    weights = {dev: _weights_on(dev, (w1, w2, w3)) + _weights_on(dev, biases) for dev in set(devs)}
    if std is not None:   # the pair only marks the form on each rank: its rows are in the interleaved head
        log_stds = {dev: log_std for dev in set(devs)}
    else:
        log_stds = None if log_std is None else {dev: _weights_on(dev, (log_std,))[0] for dev in set(devs)}
    if target:
        td = ({dev: tuple(_weights_on(dev, actor)) for dev in set(devs)}, *td[1:])
    if dqn:   # the online network where td holds a TD target's actors
        td = (None if online is None else {dev: tuple(_weights_on(dev, online)) for dev in set(devs)}, *td[1:])
    if _use_push(devs, bounds, transfer):
        _mlp_scatter_gather_pushed(obs_root, devs, bounds, weights, output, *bufs[:3], seed, log_stds, mask, bufs[3],
                                   nvec, std, epsilon, taken, det, action, twins, td if target or dqn else None)
        return views
    rows = max(e - b for b, e in bounds)
    for dev in set(devs):       # allocate scratch/staging on the calling thread (allocator + first use)
        if target:
            d_act = actor[4].shape[0] // (2 if std is not None else 1)
            _cached_buffer(_scratch, dev, dev,
                           L.load().ktb_mlp_td_target_scratch_bytes(rows, actor[0].shape[0], w1.shape[0], d_act))
        elif dqn:
            _cached_buffer(_scratch, dev, dev, L.load().ktb_mlp_dqn_target_scratch_bytes(rows, w1.shape[0]))
        else:
            _scratch_for(dev, rows, w1.shape[0], critic)
        if dev != root:
            _stage_for(dev, rows, obs_root.shape[1])
    streams = {dev: torch.cuda.current_stream(dev) for dev in set(devs)}

    def issue(r):
        """Enqueue rank r's whole pipeline (≈50 launches); ctypes releases the GIL, so ranks issue in parallel."""
        dev = devs[r]
        b, e = bounds[r]
        if e == b:
            return None
        st = streams[dev]
        with torch.cuda.device(dev):
            if dev != root:
                st.wait_event(ready)
            _forward_rows(obs_root, b, e, dev, st, None, weights[dev], bufs, output, seed,
                          None if log_stds is None else log_stds[dev], mask, nvec, std, epsilon, taken, det, action,
                          None if twins is None else twins[dev], td if target or dqn else None)
            if dev != root:
                ev = torch.cuda.Event()
                ev.record(st)
                return ev
        return None

    if len(set(devs)) > 1:
        done_evs = list(_thread_pool().map(issue, range(len(devs))))
    else:
        done_evs = [issue(r) for r in range(len(devs))]
    for ev in done_evs:
        if ev is not None:
            root_stream.wait_event(ev)
    return views
