"""bf16 MLP policy (BASELINE config C4) on wgmma tensor cores — tensor-facing wrapper of
ktb_mlp_bf16_policy (biases, heads of 1 to 256 outputs, greedy actions), ktb_mlp_bf16_policy_sample (seeded
Gumbel-max actions with their log-probabilities, kubetorch_b200.sampling), ktb_mlp_bf16_policy_gaussian (seeded
diagonal-Gaussian actions with their log-probabilities) and their scatter→exec→gather form."""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence

import torch

from . import lib as L
from . import ops
from ..mapped import MLP_OUTPUTS as OUTPUTS
from ..sampling import _check_seed

_scratch = {}
_stage = {}
_weight_cache = {}
_pool = None


def pushed_scratch_bytes(M: int, d_hidden: int, chunk_rows: int) -> int:
    """Scratch of ktb_mlp_bf16_policy_pushed: two hidden activations of min(chunk_rows, M) rows.  It follows the pushed form's
    own chunk_rows, not the tuning chunk that ktb_mlp_scratch_bytes uses for the pull forms."""
    return 2 * min(int(chunk_rows), int(M)) * int(d_hidden) * 2


def _cached_buffer(cache: dict, key, dev: int, nbytes: int) -> torch.Tensor:
    """cache[key]: a uint8 buffer on `dev` of at least `nbytes`, replaced by a larger one when a call needs more."""
    buf = cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = cache[key] = torch.empty(nbytes, dtype=torch.uint8, device=f"cuda:{dev}")
    return buf


def _scratch_for(dev: int, M: int, d_hidden: int) -> torch.Tensor:
    return _cached_buffer(_scratch, dev, dev, L.load().ktb_mlp_scratch_bytes(M, d_hidden))


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


def _check_policy(w1, w3, biases, output, seed=None, log_std=None) -> None:
    """Raise ValueError for an output mode, a head width, a bias, (output="sample" or "gaussian") a seed or
    (output="gaussian") a log_std the kernels do not take.  A seed is an int (not a bool) in [0, 2**64); log_std is
    a 1-D contiguous CUDA float32 tensor of length d_out, given with output="gaussian" only."""
    if output not in OUTPUTS:
        raise ValueError(f"output must be one of {OUTPUTS}, got {output!r}")
    if output in ("sample", "gaussian"):
        _check_seed(seed)
    if len(biases) != 3:
        raise ValueError("biases must be (b1, b2, b3), each a tensor or None")
    d_hidden, d_out = w1.shape[0], w3.shape[0]
    if not 1 <= d_out <= MAX_D_OUT:
        raise ValueError(f"d_out={d_out}: the policy head is 1 to {MAX_D_OUT} wide")
    if output != "gaussian":
        if log_std is not None:
            raise ValueError('log_std is an argument of output="gaussian" only')
    elif not isinstance(log_std, torch.Tensor) or log_std.dtype != torch.float32 or not log_std.is_cuda \
            or not log_std.is_contiguous() or log_std.dim() != 1 or log_std.shape[0] != d_out:
        raise ValueError(f"log_std must be a 1-D contiguous CUDA float32 tensor of length {d_out}")
    for name, b, n in zip(("b1", "b2", "b3"), biases, (d_hidden, d_hidden, d_out)):
        if b is None:
            continue
        if not isinstance(b, torch.Tensor) or b.dtype != torch.bfloat16 or not b.is_cuda or not b.is_contiguous() \
                or b.dim() != 1 or b.shape[0] != n:
            raise ValueError(f"{name} must be a 1-D contiguous CUDA bfloat16 tensor of length {n}")


def _outputs(output, M, d_out, device, logits, actions, log_probs):
    """(logits, actions, log_probs) of `M` rows as `output` writes them: bf16 logits [M, d_out]; int64 actions [M], or
    fp32 [M, d_out] with "gaussian"; fp32 log_probs [M].  A buffer the mode does not write is None, a missing one is
    allocated on `device` and a given one is registered with the library (ops.ensure_init)."""
    def buf(t, shape, dtype):
        if t is None:
            return torch.empty(shape, dtype=dtype, device=device)
        ops.ensure_init({t.device.index})
        return t

    gaussian = output == "gaussian"
    return (buf(logits, (M, d_out), torch.bfloat16) if output in ("logits", "both") else None,
            None if output == "logits" else
            buf(actions, (M, d_out), torch.float32) if gaussian else buf(actions, (M,), torch.int64),
            buf(log_probs, (M,), torch.float32) if output in ("sample", "gaussian") else None)


def _head(output, logits, actions, log_probs, seed, row_base, log_std, ptr, pushed=False):
    """The C entry that computes `output` (its _pushed form with `pushed`) and the head's arguments of that entry, the
    pointers as ptr(tensor) gives them."""
    suffix = "_pushed" if pushed else ""
    if output == "gaussian":
        return "ktb_mlp_bf16_policy_gaussian" + suffix, (ptr(log_std), seed, row_base, ptr(actions), ptr(log_probs))
    if output == "sample":
        return "ktb_mlp_bf16_policy_sample" + suffix, (seed, row_base, ptr(actions), ptr(log_probs))
    return "ktb_mlp_bf16_policy" + suffix, (ptr(logits), ptr(actions))


def _rows(bufs, b, e):
    """Rows b .. e - 1 of each buffer; None stays None."""
    return [None if t is None else t[b:e] for t in bufs]


def _result(output, logits, actions, log_probs):
    """What a call with `output` returns, from its buffers."""
    if output == "logits":
        return logits
    if output == "actions":
        return actions
    if output == "both":
        return logits, actions
    return actions, log_probs


def mlp_forward(obs: torch.Tensor, w1: torch.Tensor, w2: torch.Tensor, w3: torch.Tensor,
                out: Optional[torch.Tensor] = None, device: Optional[int] = None,
                stream: Optional[torch.cuda.Stream] = None, staged: Optional[bool] = None,
                biases: Sequence[Optional[torch.Tensor]] = (None, None, None), output: str = "logits",
                actions: Optional[torch.Tensor] = None, seed: Optional[int] = None, row_offset: int = 0,
                log_probs: Optional[torch.Tensor] = None, log_std: Optional[torch.Tensor] = None):
    """logits[M, d_out] = W3·relu(W2·relu(W1·obsᵀ + b1) + b2) + b3; bf16 storage, fp32 accumulation in registers,
    each bias added to the fp32 accumulator (nn.Linear).  `biases` = (b1, b2, b3), each optional.  `output` is
    "logits" (returns the logits), "actions" (returns int64 argmax actions[M]; no logits are written), "both"
    (returns (logits, actions)), "sample" (returns (actions, log_probs): int64 actions drawn from
    softmax(logits) by Gumbel-max with the noise of kubetorch_b200.sampling.gumbel_noise(seed, row_offset, M, d_out),
    and the fp32 log_softmax(logits)[action] of each row; no logits are written) or "gaussian" (returns (actions,
    log_probs): fp32 actions[M, d_out] = logits + exp(log_std)·normal_noise(seed, row_offset, M, d_out) and the fp32
    log-density of each row's action under Normal(logits, exp(log_std)); no logits are written).  `obs` / `out` /
    `actions` / `log_probs` may be peer-mapped (pull the observations / push the results over NVLink).  Without
    biases, at d_out == 64 and with logits only the logits equal ktb_mlp_bf16's."""
    for name, t in (("obs", obs), ("w1", w1), ("w2", w2), ("w3", w3)):
        if t.dtype != torch.bfloat16 or not t.is_cuda or not t.is_contiguous():
            raise ValueError(f"{name} must be a contiguous CUDA bfloat16 tensor")
    dev = w1.device.index if device is None else int(device)
    ops.ensure_init({dev, obs.device.index})
    M, d_in = obs.shape
    d_hidden, d_out = w1.shape[0], w3.shape[0]
    if w1.shape != (d_hidden, d_in) or w2.shape != (d_hidden, d_hidden) or w3.shape != (d_out, d_hidden):
        raise ValueError("weight shapes must be W1[d_h,d_in], W2[d_h,d_h], W3[d_out,d_h] (nn.Linear layout)")
    _check_policy(w1, w3, biases, output, seed, log_std)
    if output in ("sample", "gaussian") and \
            (isinstance(row_offset, bool) or not isinstance(row_offset, int) or row_offset < 0):
        raise ValueError(f"row_offset must be a non-negative int, got {row_offset!r}")
    out, actions, log_probs = _outputs(output, M, d_out, f"cuda:{dev}", out, actions, log_probs)
    s = stream if stream is not None else torch.cuda.current_stream(dev)
    if staged is None:
        staged = obs.device.index != dev   # observations on another GPU: pull each row chunk over NVLink once
    ptr = lambda t: 0 if t is None else t.data_ptr()   # noqa: E731
    entry, head = _head(output, out, actions, log_probs, seed, row_offset, log_std, ptr)
    L.call(entry, dev, obs.data_ptr(), M, d_in, d_hidden, d_out, w1.data_ptr(), ptr(biases[0]), w2.data_ptr(),
           ptr(biases[1]), w3.data_ptr(), ptr(biases[2]), *head, _scratch_for(dev, M, d_hidden).data_ptr(),
           _stage_for(dev, M, d_in).data_ptr() if staged else 0, int(s.cuda_stream))
    return _result(output, out, actions, log_probs)


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
_push_sessions = {}          # device tuple -> ops.PushSession
_push_scratch = {}           # (device tuple, rank) -> scratch of that rank's pushed GEMMs


def _mlp_scatter_gather_pushed(obs_root, devs, bounds, weights, output, out_root, actions_root, log_probs_root=None,
                               seed=None, log_std=None) -> None:
    """The root PUSHES each rank's observation rows in GEMM-sized chunks (copy engines, posted NVLink writes, flags in
    device memory); every rank's GEMM chain consumes chunk c as soon as it has landed and stores its logits (and/or
    actions) straight into the root's result; the root's own shard runs on the session's side stream beside the
    scatter.  No host synchronisation, no events between devices.  weights[dev] = (w1, w2, w3, b1, b2, b3) on that
    device (biases may be None); out_root / actions_root / log_probs_root are None when `output` does not want them
    (with "gaussian", actions_root holds the fp32 actions [M, d_out]).  log_std[dev] is the Gaussian head's log_std on
    that device.  With output="sample" or "gaussian" rank r draws the noise of global rows b_r .. e_r - 1 (its shard's
    place in obs_root)."""
    root, n, key = devs[0], len(devs), tuple(devs)
    d_in, d_hidden, d_out = obs_root.shape[1], weights[root][0].shape[0], weights[root][2].shape[0]
    rows = max(e - b for b, e in bounds)
    sess = _push_sessions.get(key)
    if sess is None or sess.stride < rows * d_in * 2:
        sess = _push_sessions[key] = ops.PushSession(devs, rows * d_in * 2)
    try:
        seq = sess.begin()
    except ops.PushTimeout:
        del _push_sessions[key]
        raise
    # scratch per rank, not per device: ranks sharing a device must not share one, nor the root's own shard on the
    # side stream
    scratch_bytes = pushed_scratch_bytes(rows, d_hidden, PUSH_CHUNK_ROWS)
    scratch = [None] + [_cached_buffer(_push_scratch, (key, r), devs[r], scratch_bytes) for r in range(1, n)]
    streams = [ops.current_stream_handle(d) for d in devs]
    bufs = (out_root, actions_root, log_probs_root)
    b0, e0 = bounds[0]
    own = e0 > b0
    if own:
        ws = weights[root]
        logits, actions, log_probs = _rows(bufs, b0, e0)
        mlp_forward(obs_root[b0:e0], ws[0], ws[1], ws[2], out=logits, device=root, stream=sess.fork(), staged=False,
                    biases=ws[3:], output=output, actions=actions, seed=seed, row_offset=b0, log_probs=log_probs,
                    log_std=None if log_std is None else log_std[root])
    L.call("ktb_push_scatter_ce", root, obs_root.data_ptr(), obs_root.numel(), d_in, L.BF16, n, 0,
           L.arr(ctypes.c_int, devs), sess.stage_ptrs, sess.stride, sess.ctrl_ptrs, sess.ctrl[0].data_ptr(),
           PUSH_CHUNK_ROWS * d_in, seq, streams[0])

    def issue(r):
        b, e = bounds[r]
        ws = weights[devs[r]]
        ptr = lambda t: 0 if t is None or e == b else t.data_ptr()   # noqa: E731
        entry, head = _head(output, *_rows(bufs, b, e), seed, b, None if log_std is None else log_std[devs[r]], ptr,
                            pushed=True)
        L.call(entry, devs[r], sess.stage[r].data_ptr(), sess.stride, e - b, d_in, d_hidden, d_out, ws[0].data_ptr(),
               ptr(ws[3]), ws[1].data_ptr(), ptr(ws[4]), ws[2].data_ptr(), ptr(ws[5]), *head, scratch[r].data_ptr(),
               sess.ctrl[r].data_ptr(), sess.ctrl[0].data_ptr(), r, PUSH_CHUNK_ROWS, seq, streams[r])

    list(_thread_pool().map(issue, range(1, n)))
    sess.finish(seq, joined=own)


def mlp_scatter_gather(obs_root: torch.Tensor, w1, w2, w3, devices: Sequence[int],
                       out_root: Optional[torch.Tensor] = None, transfer: str = "auto",
                       biases: Sequence[Optional[torch.Tensor]] = (None, None, None), output: str = "logits",
                       actions_root: Optional[torch.Tensor] = None, seed: Optional[int] = None,
                       log_probs_root: Optional[torch.Tensor] = None, log_std: Optional[torch.Tensor] = None) -> list:
    """Rank r runs the MLP on `obs.chunk(world)[r]`: its first GEMM's TMA loads read the rows straight
    from the root GPU (scatter) and its last epilogue stores the logits straight into the root's
    result buffer (gather). Returns rank-ordered views of the root result: logits views for output="logits",
    int64 actions views for "actions", (logits, actions) pairs for "both", (actions, log_probs) pairs for "sample"
    and "gaussian" (fp32 actions [rows, d_out] with the latter).  With "sample" or "gaussian" rank r draws the noise of
    the global rows of its shard (row_offset = its shard's begin), so the result does not depend on the number of
    ranks or their devices.  `biases`, `seed` and `log_std` as in mlp_forward."""
    root = obs_root.device.index
    devs = [int(d) for d in devices]
    if devs[0] != root:
        raise ValueError("obs must live on the root GPU (devices[0])")
    _check_policy(w1, w3, biases, output, seed, log_std)
    ops.ensure_init(set(devs))
    M = obs_root.shape[0]
    bufs = _outputs(output, M, w3.shape[0], obs_root.device, out_root, actions_root, log_probs_root)
    root_stream = torch.cuda.current_stream(root)
    ready = torch.cuda.Event()
    ready.record(root_stream)
    bounds = [ops.shard_bounds(M, len(devs), r) for r in range(len(devs))]
    views = [_result(output, *_rows(bufs, b, e)) for b, e in bounds]
    weights = {dev: _weights_on(dev, (w1, w2, w3)) + _weights_on(dev, biases) for dev in set(devs)}
    log_stds = None if log_std is None else {dev: _weights_on(dev, (log_std,))[0] for dev in set(devs)}
    distinct = len(set(devs)) == len(devs) and len(devs) > 1
    pushable = distinct and all((e - b) % 128 == 0 for b, e in bounds) and \
        -(-max(e - b for b, e in bounds) // PUSH_CHUNK_ROWS) <= 64
    if transfer not in ("auto", "pull", "push"):
        raise ValueError("transfer must be 'auto', 'pull' or 'push'")
    if transfer == "push" and not pushable:
        raise ValueError("push transfer needs distinct devices and shards of a multiple of 128 rows")
    if pushable and transfer != "pull":
        _mlp_scatter_gather_pushed(obs_root, devs, bounds, weights, output, *bufs, seed, log_stds)
        return views
    for dev in set(devs):       # allocate scratch/staging on the calling thread (allocator + first use)
        _scratch_for(dev, max(e - b for b, e in bounds), w1.shape[0])
        if dev != root:
            _stage_for(dev, max(e - b for b, e in bounds), obs_root.shape[1])
    streams = {dev: torch.cuda.current_stream(dev) for dev in set(devs)}

    def issue(r):
        """Enqueue rank r's whole pipeline (≈50 launches); ctypes releases the GIL, so ranks issue in parallel."""
        dev = devs[r]
        b, e = bounds[r]
        if e == b:
            return None
        ws = weights[dev]
        st = streams[dev]
        with torch.cuda.device(dev):
            if dev != root:
                st.wait_event(ready)
            logits, actions, log_probs = _rows(bufs, b, e)
            mlp_forward(obs_root[b:e], ws[0], ws[1], ws[2], out=logits, device=dev, stream=st, biases=ws[3:],
                        output=output, actions=actions, seed=seed, row_offset=b, log_probs=log_probs,
                        log_std=None if log_stds is None else log_stds[dev])
            if dev != root:
                ev = torch.cuda.Event()
                ev.record(st)
                return ev
        return None

    if len(set(devs)) > 1:
        done = list(_thread_pool().map(issue, range(len(devs))))
    else:
        done = [issue(r) for r in range(len(devs))]
    for ev in done:
        if ev is not None:
            root_stream.wait_event(ev)
    return views
