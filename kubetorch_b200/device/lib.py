"""ctypes binding of libktb200.so (include/ktb200.h) — the only way the package reaches the GPU.

There is no CPU fallback: if the library is missing or a call fails, this raises.  The binding
is what a kubetorch maintainer would add behind the supervisor seam
(kt/serving/supervisor_factory.py:11-58); see INTEGRATION.md.
"""
from __future__ import annotations

import ctypes
import os
import threading
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_size_t, c_void_p

_LIB_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "lib", "libktb200.so")

# enums (include/ktb200.h)
OP_IDENTITY, OP_SCALE, OP_AFFINE = 0, 1, 2
U8, F32, BF16, I32, I64, F16 = 0, 1, 2, 3, 4, 5
VARIANT_AUTO, VARIANT_VEC, VARIANT_TMA, VARIANT_SCALAR = 0, 1, 2, 3
OK, ERR_CUDA, ERR_ARG, ERR_STATE, ERR_UNSUPPORTED = 0, -1, -2, -3, -4
PACK_ALIGN = 256
IPC_HANDLE_BYTES = 64

c_uintptr = ctypes.c_size_t  # uintptr_t


class KtbError(RuntimeError):
    """A libktb200 call failed. ``status`` is the ktb_status code."""

    def __init__(self, status: int, message: str):
        super().__init__(f"libktb200 error {status}: {message}")
        self.status = status


class KtbLibraryMissing(ImportError):
    pass


_SIGNATURES = {
    "ktb_init": (c_int, [c_int, POINTER(c_int)]),
    "ktb_shutdown": (c_int, []),
    "ktb_last_error": (c_char_p, []),
    "ktb_version": (c_int, []),
    "ktb_sm_count": (c_int, [c_int]),
    "ktb_peer_enabled": (c_int, [c_int, c_int]),
    "ktb_arena_alloc": (c_int, [c_int, c_size_t, POINTER(c_void_p)]),
    "ktb_arena_free": (c_int, [c_int, c_void_p]),
    "ktb_host_alloc": (c_int, [c_size_t, POINTER(c_void_p)]),
    "ktb_host_free": (c_int, [c_void_p]),
    "ktb_device_numa_node": (c_int, [c_int]),
    "ktb_host_alloc_sharded": (c_int, [c_size_t, c_int, POINTER(c_size_t), POINTER(c_int), POINTER(c_void_p)]),
    "ktb_host_free_sharded": (c_int, [c_void_p]),
    "ktb_ipc_export": (c_int, [c_int, c_void_p, c_void_p]),
    "ktb_ipc_open": (c_int, [c_int, c_void_p, POINTER(c_void_p)]),
    "ktb_ipc_close": (c_int, [c_int, c_void_p]),
    "ktb_shard_bounds": (c_int, [c_size_t, c_int, c_int, POINTER(c_size_t), POINTER(c_size_t)]),
    "ktb_map": (c_int, [c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_double, c_double, c_int, c_uintptr]),
    "ktb_map_identity_u8": (c_int, [c_int, c_void_p, c_void_p, c_size_t, c_uintptr]),
    "ktb_map_scale_f32": (c_int, [c_int, c_void_p, c_void_p, c_size_t, c_float, c_uintptr]),
    "ktb_map_affine_f32": (c_int, [c_int, c_void_p, c_void_p, c_size_t, c_float, c_float, c_uintptr]),
    "ktb_map_scale_bf16": (c_int, [c_int, c_void_p, c_void_p, c_size_t, c_float, c_uintptr]),
    "ktb_map_affine_bf16": (c_int, [c_int, c_void_p, c_void_p, c_size_t, c_float, c_float, c_uintptr]),
    "ktb_reduce_workspace_bytes": (c_size_t, []),
    "ktb_map_reduce_sum": (c_int, [c_int, c_int, c_int, c_void_p, c_size_t, c_double, c_double, c_void_p, c_void_p, c_uintptr]),
    "ktb_reduce_partials": (c_int, [c_int, c_int, c_void_p, c_int, c_void_p, c_uintptr]),
    "ktb_pack_layout": (c_int, [POINTER(c_size_t), c_int, POINTER(c_size_t), POINTER(c_size_t)]),
    "ktb_pack": (c_int, [c_int, POINTER(c_void_p), POINTER(c_size_t), c_int, c_void_p, c_size_t, POINTER(c_size_t), c_int, c_uintptr]),
    "ktb_unpack": (c_int, [c_int, c_void_p, POINTER(c_size_t), POINTER(c_size_t), c_int, POINTER(c_void_p), c_uintptr]),
    "ktb_map_batch": (c_int, [c_int, c_int, c_int, POINTER(c_void_p), POINTER(c_void_p), POINTER(c_size_t), c_int, c_double, c_double, c_uintptr]),
    "ktb_broadcast": (c_int, [c_int, c_void_p, POINTER(c_void_p), c_int, c_size_t, c_uintptr]),
    "ktb_scatter_map_gather": (c_int, [c_int, c_int, c_void_p, c_void_p, c_size_t, c_size_t, c_double, c_double, c_int, POINTER(c_int), c_int, c_int, POINTER(c_uintptr)]),
    "ktb_scatter_map_reduce": (c_int, [c_int, c_int, c_void_p, c_size_t, c_size_t, c_double, c_double, c_int, POINTER(c_int), c_int, c_void_p, c_void_p, POINTER(c_void_p), POINTER(c_uintptr)]),
    "ktb_push_control_bytes": (c_size_t, []),
    "ktb_push_scatter": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int, POINTER(c_void_p), c_size_t,
                                 POINTER(c_void_p), c_void_p, c_int, ctypes.c_ulonglong, c_uintptr]),
    "ktb_push_scatter_chunked": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int, POINTER(c_void_p),
                                         c_size_t, POINTER(c_void_p), c_void_p, c_size_t, c_int, ctypes.c_ulonglong,
                                         c_uintptr]),
    "ktb_push_scatter_ce": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int, POINTER(c_int), POINTER(c_void_p),
                                    c_size_t, POINTER(c_void_p), c_void_p, c_size_t, ctypes.c_ulonglong, c_uintptr]),
    "ktb_push_scatter_ce_masked": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int, POINTER(c_int),
                                           POINTER(c_void_p), c_size_t, POINTER(c_void_p), c_void_p, c_size_t,
                                           c_void_p, c_size_t, c_size_t, ctypes.c_ulonglong, c_uintptr]),
    "ktb_push_consume": (c_int, [c_int, c_int, c_int, c_void_p, c_size_t, c_void_p, c_size_t, c_double, c_double,
                                 c_void_p, c_void_p, c_int, c_int, ctypes.c_ulonglong, c_uintptr]),
    "ktb_push_wait": (c_int, [c_int, c_void_p, c_int, c_int, ctypes.c_ulonglong, c_uintptr]),
    "ktb_push_status": (c_int, [c_int, c_void_p, POINTER(ctypes.c_uint)]),
    "ktb_map_host_multi": (c_int, [c_int, c_int, c_void_p, c_void_p, c_size_t, c_size_t, c_double, c_double, c_int,
                                   POINTER(c_int), c_size_t, POINTER(c_void_p), POINTER(c_void_p)]),
    "ktb_mlp_scratch_bytes": (c_size_t, [c_size_t, c_int]),
    "ktb_mlp_bf16": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uintptr]),
    "ktb_mlp_stage_bytes": (c_size_t, [c_size_t, c_int]),
    "ktb_mlp_bf16_staged": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_uintptr]),
    "ktb_mlp_bf16_pushed": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_size_t, ctypes.c_ulonglong,
                                    c_uintptr]),
    "ktb_mlp_bf16_policy": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uintptr]),
    "ktb_mlp_bf16_policy_pushed": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_int, c_size_t, ctypes.c_ulonglong, c_uintptr]),
    "ktb_mlp_bf16_policy_sample": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_uint64, ctypes.c_uint64,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_uintptr]),
    "ktb_mlp_bf16_policy_sample_pushed": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int, c_void_p,
                                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_uint64,
                                                  ctypes.c_uint64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                  c_int, c_size_t, ctypes.c_ulonglong, c_uintptr]),
    "ktb_mlp_bf16_policy_gaussian": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p,
                                             c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_uint64,
                                             ctypes.c_uint64, c_void_p, c_void_p, c_void_p, c_void_p, c_uintptr]),
    "ktb_mlp_bf16_policy_gaussian_pushed": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int,
                                                    c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                    c_void_p, ctypes.c_uint64, ctypes.c_uint64, c_void_p, c_void_p,
                                                    c_void_p, c_void_p, c_void_p, c_int, c_size_t, ctypes.c_ulonglong,
                                                    c_uintptr]),
    "ktb_mlp_bf16_policy_masked": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_uintptr]),
    "ktb_mlp_bf16_policy_masked_pushed": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int,
                                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                  c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                                  c_size_t, ctypes.c_ulonglong, c_uintptr]),
    "ktb_mlp_bf16_policy_sample_masked": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p,
                                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                  ctypes.c_uint64, ctypes.c_uint64, c_void_p, c_void_p, c_void_p,
                                                  c_void_p, c_uintptr]),
    "ktb_mlp_bf16_policy_sample_masked_pushed": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int,
                                                         c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                         c_size_t, ctypes.c_uint64, ctypes.c_uint64, c_void_p,
                                                         c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_size_t,
                                                         ctypes.c_ulonglong, c_uintptr]),
    "ktb_mlp_bf16_policy_sample_value": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p,
                                                 c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_uint64,
                                                 ctypes.c_uint64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                 c_uintptr]),
    "ktb_mlp_bf16_policy_sample_value_pushed": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int,
                                                        c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                        ctypes.c_uint64, ctypes.c_uint64, c_void_p, c_void_p, c_void_p,
                                                        c_void_p, c_void_p, c_void_p, c_int, c_size_t,
                                                        ctypes.c_ulonglong, c_uintptr]),
    "ktb_mlp_bf16_policy_sample_masked_value": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p,
                                                        c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                        ctypes.c_uint64, ctypes.c_uint64, c_void_p, c_void_p, c_void_p,
                                                        c_void_p, c_void_p, c_uintptr]),
    "ktb_mlp_bf16_policy_sample_masked_value_pushed": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int,
                                                               c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                               c_void_p, c_size_t, ctypes.c_uint64, ctypes.c_uint64,
                                                               c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                               c_void_p, c_int, c_size_t, ctypes.c_ulonglong,
                                                               c_uintptr]),
    "ktb_mlp_bf16_policy_gaussian_value": (c_int, [c_int, c_void_p, c_size_t, c_int, c_int, c_int, c_void_p, c_void_p,
                                                   c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_uint64,
                                                   ctypes.c_uint64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                   c_uintptr]),
    "ktb_mlp_bf16_policy_gaussian_value_pushed": (c_int, [c_int, c_void_p, c_size_t, c_size_t, c_int, c_int, c_int,
                                                          c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                          c_void_p, ctypes.c_uint64, ctypes.c_uint64, c_void_p,
                                                          c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                                          c_size_t, ctypes.c_ulonglong, c_uintptr]),
    # experiment knob, not in the stable header
    "ktb_set_tuning": (c_int, [c_int, c_int]),
}
# The _multidiscrete entries: each takes its categorical counterpart's arguments with (nvec, n_groups) after b3 (or
# b3v), the 12th argument of the plain and staged forms and the 13th of the pushed ones.
for _head, _suffixes in (("ktb_mlp_bf16_policy", ("", "_masked")),
                         ("ktb_mlp_bf16_policy_sample", ("", "_masked", "_value", "_masked_value"))):
    for _suffix in _suffixes:
        for _form, _at in (("", 12), ("_pushed", 13)):
            _restype, _args = _SIGNATURES[_head + _suffix + _form]
            _SIGNATURES[_head + "_multidiscrete" + _suffix + _form] = (
                _restype, _args[:_at] + [POINTER(ctypes.c_int32), c_int] + _args[_at:])
# The _gaussian_state entries: each takes its _gaussian counterpart's arguments with (log_std_min, log_std_max, squash)
# in place of log_std, the 13th argument of the plain and staged forms and the 14th of the pushed ones.
for _suffix in ("", "_value"):
    for _form, _at in (("", 12), ("_pushed", 13)):
        _restype, _args = _SIGNATURES["ktb_mlp_bf16_policy_gaussian" + _suffix + _form]
        _SIGNATURES["ktb_mlp_bf16_policy_gaussian_state" + _suffix + _form] = (
            _restype, _args[:_at] + [ctypes.c_float, ctypes.c_float, c_int] + _args[_at + 1:])
# The _epsilon_greedy entries: the sample entries' arguments with (epsilon, seed, row_base, actions, q, q_max) in place
# of (seed, row_base, actions, log_probs); the masked ones with the mask before epsilon, and the pushed ones with
# (mask_offset and) epsilon_offset in place of the pointers.
# seed is the 13th argument of the plain and staged forms and the 14th of the pushed ones, one later when masked.
for _masked in ("", "_masked"):
    for _form, _eps, _at in (("", c_void_p, 12), ("_pushed", c_size_t, 13)):
        _restype, _args = _SIGNATURES["ktb_mlp_bf16_policy_sample" + _masked + _form]
        _at += bool(_masked)
        _SIGNATURES["ktb_mlp_bf16_policy_epsilon_greedy" + _masked + _form] = (
            _restype, _args[:_at] + [_eps] + _args[_at:_at + 4] + [c_void_p] + _args[_at + 4:])
# The _evaluate entries: ktb_mlp_bf16_policy's arguments up to b3 (the first 12 of the plain and staged forms, 13 of
# the pushed ones), then (nvec, n_groups, [mask,] taken, log_probs, entropy, [values,]) with (mask_offset,) taken_offset
# in the pushed forms; the _gaussian_evaluate ones take log_std in place of (nvec, n_groups, [mask,]).
for _masked in ("", "_masked"):
    for _valued in ("", "_value"):
        for _form, _in, _at in (("", c_void_p, 12), ("_pushed", c_size_t, 13)):
            _args = _SIGNATURES["ktb_mlp_bf16_policy" + _form][1]
            _head_args = [POINTER(ctypes.c_int32), c_int] + [_in] * (1 + bool(_masked)) + [c_void_p] * (2 + bool(_valued))
            _SIGNATURES["ktb_mlp_bf16_policy_evaluate" + _masked + _valued + _form] = (
                c_int, _args[:_at] + _head_args + _args[_at + 2:])
            if not _masked:
                _SIGNATURES["ktb_mlp_bf16_policy_gaussian_evaluate" + _valued + _form] = (
                    c_int, _args[:_at] + [c_void_p, _in] + [c_void_p] * (2 + bool(_valued)) + _args[_at + 2:])
# The _deterministic entries: the _gaussian_state entries' arguments with (noise, noise_clip, squash) in place of
# (log_std_min, log_std_max, squash) and without log_probs, the 19th argument of the plain and staged forms and the 20th
# of the pushed ones.
for _form, _at in (("", 18), ("_pushed", 19)):
    _restype, _args = _SIGNATURES["ktb_mlp_bf16_policy_gaussian_state" + _form]
    _SIGNATURES["ktb_mlp_bf16_policy_deterministic" + _form] = (_restype, _args[:_at] + _args[_at + 1:])
# The _critic entries: ktb_mlp_bf16_policy's arguments up to b3 (d_act in place of d_out, W1p for W1), the second
# critic's six after them in the _twin forms, then act (act_offset in the pushed forms) and q, or q1, q2 and q_min.
_SIGNATURES["ktb_mlp_critic_scratch_bytes"] = (c_size_t, [c_size_t, c_int])
for _twin in ("", "_twin"):
    for _form, _act, _at in (("", c_void_p, 12), ("_pushed", c_size_t, 13)):
        _args = _SIGNATURES["ktb_mlp_bf16_policy" + _form][1]
        _head_args = [c_void_p] * (6 if _twin else 0) + [_act] + [c_void_p] * (3 if _twin else 1)
        _SIGNATURES["ktb_mlp_bf16_critic" + _twin + _form] = (c_int, _args[:_at] + _head_args + _args[_at + 2:])
# The _td_target entries: the _critic_twin entries' arguments up to the second critic's b3, then d_hidden_actor and the
# actor's six pointers, the policy's five arguments, then reward and done (their offsets in the pushed forms), gamma,
# alpha (_gaussian only) and y, then the rest of the _critic_twin entries' arguments from scratch on.
_SIGNATURES["ktb_mlp_td_target_scratch_bytes"] = (c_size_t, [c_size_t, c_int, c_int, c_int])
for _policy, _alpha in (("_deterministic", []), ("_gaussian", [c_float])):
    for _form, _side, _at in (("", c_void_p, 18), ("_pushed", c_size_t, 19)):
        _args = _SIGNATURES["ktb_mlp_bf16_critic_twin" + _form][1]
        _SIGNATURES["ktb_mlp_bf16_td_target" + _policy + _form] = (
            c_int, _args[:_at] + [c_int] + [c_void_p] * 6 + [c_float, c_float, c_int, ctypes.c_uint64, ctypes.c_uint64]
            + [_side, _side, c_float] + _alpha + [c_void_p] + _args[_at + 4:])
# The _dqn_target entries: ktb_mlp_bf16_policy's arguments up to b3 (the target network), the online network's six
# pointers, ([mask,] reward, done, gamma, y) with (mask_offset,) rd_offset in place of (mask, reward, done) in the pushed
# forms, then ktb_mlp_bf16_policy's arguments from scratch on.
_SIGNATURES["ktb_mlp_dqn_target_scratch_bytes"] = (c_size_t, [c_size_t, c_int])
for _masked in ("", "_masked"):
    for _form, _in, _rd, _at in (("", c_void_p, [c_void_p, c_void_p], 12), ("_pushed", c_size_t, [c_size_t], 13)):
        _args = _SIGNATURES["ktb_mlp_bf16_policy" + _form][1]
        _SIGNATURES["ktb_mlp_bf16_dqn_target" + _masked + _form] = (
            c_int, _args[:_at] + [c_void_p] * 6 + [_in] * bool(_masked) + _rd + [c_float, c_void_p] + _args[_at + 2:])
_SIGNATURES["ktb_gae_f32"] = (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_size_t, c_float, c_float,
                                      c_void_p, c_void_p, c_uintptr])
_SIGNATURES["ktb_push_scatter_ce_sides"] = (
    c_int, _SIGNATURES["ktb_push_scatter_ce"][1][:13] + [c_int, POINTER(c_void_p), POINTER(c_size_t), POINTER(c_size_t),
                                                         ctypes.c_ulonglong, c_uintptr])

_lib = None
_lock = threading.Lock()


def lib_path() -> str:
    return _LIB_PATH


def map_kernel_source_sha256() -> str:
    """sha256 of the SOURCE of the dominant kernel (the "VEC" section of csrc/ktb_map.cu = map_vec_kernel and its
    load/store helpers, plus the per-element op math and the streaming PTX helpers of ktb_common.cuh).  Stamped into
    profiles/roofline_traffic.json at ncu-capture time; bench.py reports `traffic: null` ("stale") when it differs."""
    import hashlib

    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "csrc")

    def section(name, start, stop):
        text = open(os.path.join(csrc, name)).read()
        a = text.index(start)
        return text[a:text.index(stop, a)]

    h = hashlib.sha256()
    h.update(section("ktb_map.cu", "// ---- VEC ---", "// ---- SCALAR ---").encode())
    h.update(section("ktb_common.cuh", "// ---- per-element op math", "// ---- PTX: mbarrier").encode())
    return h.hexdigest()


def load() -> ctypes.CDLL:
    """Load libktb200.so (once) and declare every prototype. Raises KtbLibraryMissing if absent."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(_LIB_PATH):
            raise KtbLibraryMissing(
                f"{_LIB_PATH} not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "or `make -C kubetorch_b200/csrc`. kubetorch_b200 has no CPU fallback for the device path."
            )
        lib = ctypes.CDLL(_LIB_PATH, mode=ctypes.RTLD_GLOBAL)
        for name, (restype, argtypes) in _SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
        return lib


def last_error() -> str:
    msg = load().ktb_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def check(status: int) -> int:
    if status < 0:
        raise KtbError(status, last_error())
    return status


def call(name: str, *args):
    """Call a status-returning entry point and raise KtbError on failure."""
    return check(getattr(load(), name)(*args))


def arr(ctype, values):
    return (ctype * len(values))(*values)
