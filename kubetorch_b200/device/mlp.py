"""bf16 MLP policy (BASELINE config C4) on wgmma tensor cores — tensor-facing wrapper of
ktb_mlp_bf16_policy (biases, heads of 1 to 256 outputs, greedy actions) and its scatter→exec→gather form."""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence

import torch

from . import lib as L
from . import ops

_scratch = {}
_stage = {}
_weight_cache = {}
_pool = None


def pushed_scratch_bytes(M: int, d_hidden: int, chunk_rows: int) -> int:
    """Scratch of ktb_mlp_bf16_policy_pushed: two hidden activations of min(chunk_rows, M) rows.  It follows the pushed form's
    own chunk_rows, not the tuning chunk that ktb_mlp_scratch_bytes uses for the pull forms."""
    return 2 * min(int(chunk_rows), int(M)) * int(d_hidden) * 2


def _scratch_for(dev: int, M: int, d_hidden: int, chunk_rows: Optional[int] = None) -> torch.Tensor:
    if chunk_rows is None:
        nbytes = L.load().ktb_mlp_scratch_bytes(M, d_hidden)
    else:
        nbytes = pushed_scratch_bytes(M, d_hidden, chunk_rows)
    buf = _scratch.get(dev)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(nbytes, dtype=torch.uint8, device=f"cuda:{dev}")
        _scratch[dev] = buf
    return buf


def _stage_for(dev: int, M: int, d_in: int) -> torch.Tensor:
    nbytes = L.load().ktb_mlp_stage_bytes(M, d_in)
    buf = _stage.get(dev)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(nbytes, dtype=torch.uint8, device=f"cuda:{dev}")
        _stage[dev] = buf
    return buf


OUTPUTS = ("logits", "actions", "both")
MAX_D_OUT = 256


def _check_policy(w1, w3, biases, output) -> None:
    """Raise ValueError for an output mode, a head width or a bias the kernels do not take."""
    if output not in OUTPUTS:
        raise ValueError(f"output must be one of {OUTPUTS}, got {output!r}")
    if len(biases) != 3:
        raise ValueError("biases must be (b1, b2, b3), each a tensor or None")
    d_hidden, d_out = w1.shape[0], w3.shape[0]
    if not 1 <= d_out <= MAX_D_OUT:
        raise ValueError(f"d_out={d_out}: the policy head is 1 to {MAX_D_OUT} wide")
    for name, b, n in zip(("b1", "b2", "b3"), biases, (d_hidden, d_hidden, d_out)):
        if b is None:
            continue
        if not isinstance(b, torch.Tensor) or b.dtype != torch.bfloat16 or not b.is_cuda or not b.is_contiguous() \
                or b.dim() != 1 or b.shape[0] != n:
            raise ValueError(f"{name} must be a 1-D contiguous CUDA bfloat16 tensor of length {n}")


def mlp_forward(obs: torch.Tensor, w1: torch.Tensor, w2: torch.Tensor, w3: torch.Tensor,
                out: Optional[torch.Tensor] = None, device: Optional[int] = None,
                stream: Optional[torch.cuda.Stream] = None, staged: Optional[bool] = None,
                biases: Sequence[Optional[torch.Tensor]] = (None, None, None), output: str = "logits",
                actions: Optional[torch.Tensor] = None):
    """logits[M, d_out] = W3·relu(W2·relu(W1·obsᵀ + b1) + b2) + b3; bf16 storage, fp32 accumulation in registers,
    each bias added to the fp32 accumulator (nn.Linear).  `biases` = (b1, b2, b3), each optional.  `output` is
    "logits" (returns the logits), "actions" (returns int64 argmax actions[M]; no logits are written) or "both"
    (returns (logits, actions)).  `obs` / `out` / `actions` may be peer-mapped (pull the observations / push the
    results over NVLink).  Without biases, at d_out == 64 and with logits only the logits equal ktb_mlp_bf16's."""
    for name, t in (("obs", obs), ("w1", w1), ("w2", w2), ("w3", w3)):
        if t.dtype != torch.bfloat16 or not t.is_cuda or not t.is_contiguous():
            raise ValueError(f"{name} must be a contiguous CUDA bfloat16 tensor")
    dev = w1.device.index if device is None else int(device)
    ops.ensure_init({dev, obs.device.index})
    M, d_in = obs.shape
    d_hidden, d_out = w1.shape[0], w3.shape[0]
    if w1.shape != (d_hidden, d_in) or w2.shape != (d_hidden, d_hidden) or w3.shape != (d_out, d_hidden):
        raise ValueError("weight shapes must be W1[d_h,d_in], W2[d_h,d_h], W3[d_out,d_h] (nn.Linear layout)")
    _check_policy(w1, w3, biases, output)
    want_logits, want_actions = output != "actions", output != "logits"
    if want_logits:
        if out is None:
            out = torch.empty(M, d_out, dtype=torch.bfloat16, device=f"cuda:{dev}")
        else:
            ops.ensure_init({out.device.index})
    if want_actions:
        if actions is None:
            actions = torch.empty(M, dtype=torch.int64, device=f"cuda:{dev}")
        else:
            ops.ensure_init({actions.device.index})
    s = stream if stream is not None else torch.cuda.current_stream(dev)
    if staged is None:
        staged = obs.device.index != dev   # observations on another GPU: pull each row chunk over NVLink once
    ptr = lambda t: 0 if t is None else t.data_ptr()   # noqa: E731
    L.call("ktb_mlp_bf16_policy", dev, obs.data_ptr(), M, d_in, d_hidden, d_out, w1.data_ptr(), ptr(biases[0]),
           w2.data_ptr(), ptr(biases[1]), w3.data_ptr(), ptr(biases[2]), ptr(out) if want_logits else 0,
           ptr(actions) if want_actions else 0, _scratch_for(dev, M, d_hidden).data_ptr(),
           _stage_for(dev, M, d_in).data_ptr() if staged else 0, int(s.cuda_stream))
    return (out, actions) if output == "both" else actions if output == "actions" else out


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


SCATTER_ENGINE = "ce"        # "ce": copy engines push the observation chunks; "sm": the capped scatter kernel;
                             # "hybrid": copy engines serve the first CE_RANKS ranks, the capped scatter kernel the rest
CE_RANKS = 3
SCATTER_CTAS_PER_SM = 2
PUSH_CHUNK_ROWS = 16896      # 132 SMs x 128 rows: each 256-wide layer of a chunk is whole waves of 128 x 256 tiles
_push_states = {}


class _MlpPushState:
    """Per device set: control blocks, per-rank staging (2 call-parity halves), the root's side stream."""

    def __init__(self, devs: Sequence[int], stride: int):
        self.devs, self.stride, self.seq = list(devs), int(stride), 0
        cb = L.load().ktb_push_control_bytes()
        self.ctrl = [torch.zeros(cb, dtype=torch.uint8, device=f"cuda:{d}") for d in devs]
        self.stage = [None if r == 0 else torch.empty(2 * self.stride, dtype=torch.uint8, device=f"cuda:{d}")
                      for r, d in enumerate(devs)]
        for d in set(devs):
            torch.cuda.synchronize(d)
        self.stage_ptrs = L.arr(ctypes.c_void_p, [0 if t is None else t.data_ptr() for t in self.stage])
        self.ctrl_ptrs = L.arr(ctypes.c_void_p, [c.data_ptr() for c in self.ctrl])
        self.side = torch.cuda.Stream(devs[0])
        self.scatter = torch.cuda.Stream(devs[0])      # the SM scatter kernel of a hybrid scatter
        self.ev_fork, self.ev_join = torch.cuda.Event(), torch.cuda.Event()
        self.ev_scatter = torch.cuda.Event()
        self.status_host = torch.zeros(len(devs), dtype=torch.int32).pin_memory()
        self.status_dev = [c[1032:1036].view(torch.int32) for c in self.ctrl]


def _mlp_push_state(devs: Sequence[int], shard_bytes: int) -> _MlpPushState:
    key = tuple(devs)
    st = _push_states.get(key)
    stride = (int(shard_bytes) + 255) // 256 * 256
    if st is None or st.stride < stride:
        st = _push_states[key] = _MlpPushState(devs, stride)
    return st


def _mlp_scatter_gather_pushed(obs_root, w1, w2, w3, devs, out_root, bounds, weights, output="logits",
                               actions_root=None) -> None:
    """The root PUSHES each rank's observation rows in GEMM-sized chunks (posted NVLink writes, flags in device memory);
    every rank's GEMM chain consumes chunk c as soon as it has landed and stores its logits (and/or actions) straight
    into the root's result; the root's own shard runs on a side stream beside the scatter.  No host synchronisation, no
    events between devices.  weights[dev] = (w1, w2, w3, b1, b2, b3) on that device (biases may be None)."""
    root, n = devs[0], len(devs)
    d_in, d_hidden, d_out = obs_root.shape[1], w1.shape[0], w3.shape[0]
    st = _mlp_push_state(devs, max(e - b for b, e in bounds) * d_in * 2)
    if bool(st.status_host.any()):
        _push_states.pop(tuple(devs), None)
        raise ops.PushTimeout("MLP push pipeline: an in-kernel wait timed out during an earlier call")
    st.seq += 1
    seq = st.seq
    root_stream = torch.cuda.current_stream(root)
    with torch.cuda.device(root):
        b0, e0 = bounds[0]
        st.ev_fork.record(root_stream)          # forked BEFORE the scatter launch: the side stream must not queue behind it
        st.side.wait_event(st.ev_fork)
        if e0 > b0:
            ws = weights[root]
            mlp_forward(obs_root[b0:e0], ws[0], ws[1], ws[2], out=None if out_root is None else out_root[b0:e0],
                        device=root, stream=st.side, staged=False, biases=ws[3:], output=output,
                        actions=None if actions_root is None else actions_root[b0:e0])
        st.ev_join.record(st.side)
        engine = SCATTER_ENGINE if n > 2 or SCATTER_ENGINE != "hybrid" else "ce"
        ptrs = [0 if t is None else t.data_ptr() for t in st.stage]
        n_ce = n - 1 if engine == "ce" else (0 if engine == "sm" else min(CE_RANKS, n - 2))
        ce_ptrs = L.arr(ctypes.c_void_p, [p if 1 <= r <= n_ce else 0 for r, p in enumerate(ptrs)])
        sm_ptrs = L.arr(ctypes.c_void_p, [p if r > n_ce else 0 for r, p in enumerate(ptrs)])
        if n_ce < n - 1:             # the capped scatter kernel first: its few CTAs per SM leave room for the root's GEMMs
            st.scatter.wait_event(st.ev_fork)
            L.call("ktb_push_scatter_chunked", root, obs_root.data_ptr(), obs_root.numel(), d_in, L.BF16, n, 0, sm_ptrs,
                   st.stride, st.ctrl_ptrs, st.ctrl[0].data_ptr(), PUSH_CHUNK_ROWS * d_in, SCATTER_CTAS_PER_SM, seq,
                   int(st.scatter.cuda_stream))
            st.ev_scatter.record(st.scatter)
        if n_ce > 0:                 # copy engines move the rows of the other ranks: no SM of the root involved
            L.call("ktb_push_scatter_ce", root, obs_root.data_ptr(), obs_root.numel(), d_in, L.BF16, n, 0,
                   L.arr(ctypes.c_int, list(devs)), ce_ptrs, st.stride, st.ctrl_ptrs, st.ctrl[0].data_ptr(),
                   PUSH_CHUNK_ROWS * d_in, seq, int(root_stream.cuda_stream))
    streams = {d: torch.cuda.current_stream(d) for d in devs[1:]}
    scratch = {d: _scratch_for(d, max(e - b for b, e in bounds), d_hidden, PUSH_CHUNK_ROWS) for d in devs[1:]}

    def issue(r):
        dev = devs[r]
        b, e = bounds[r]
        ws = weights[dev]
        ptr = lambda t: 0 if t is None or e == b else t.data_ptr()   # noqa: E731
        L.call("ktb_mlp_bf16_policy_pushed", dev, st.stage[r].data_ptr(), st.stride, e - b, d_in, d_hidden, d_out,
               ws[0].data_ptr(), ptr(ws[3]), ws[1].data_ptr(), ptr(ws[4]), ws[2].data_ptr(), ptr(ws[5]),
               ptr(None if out_root is None else out_root[b:e]),
               ptr(None if actions_root is None else actions_root[b:e]), scratch[dev].data_ptr(),
               st.ctrl[r].data_ptr(), st.ctrl[0].data_ptr(), r, PUSH_CHUNK_ROWS, seq, int(streams[dev].cuda_stream))

    global _pool
    if _pool is None:
        from concurrent.futures import ThreadPoolExecutor

        _pool = ThreadPoolExecutor(max_workers=16, thread_name_prefix="ktb-mlp")
    list(_pool.map(issue, range(1, n)))
    with torch.cuda.device(root):
        L.call("ktb_push_wait", root, st.ctrl[0].data_ptr(), n, 0, seq, int(root_stream.cuda_stream))
        root_stream.wait_event(st.ev_join)
        if n_ce < n - 1:
            root_stream.wait_event(st.ev_scatter)
    for r, d in enumerate(devs):   # stream-ordered mirror of the sticky status words (seen at the next call)
        with torch.cuda.device(d):
            st.status_host[r:r + 1].copy_(st.status_dev[r], non_blocking=True)


def mlp_scatter_gather(obs_root: torch.Tensor, w1, w2, w3, devices: Sequence[int],
                       out_root: Optional[torch.Tensor] = None, transfer: str = "auto",
                       biases: Sequence[Optional[torch.Tensor]] = (None, None, None), output: str = "logits",
                       actions_root: Optional[torch.Tensor] = None) -> list:
    """Rank r runs the MLP on `obs.chunk(world)[r]`: its first GEMM's TMA loads read the rows straight
    from the root GPU (scatter) and its last epilogue stores the logits straight into the root's
    result buffer (gather). Returns rank-ordered views of the root result: logits views for output="logits",
    int64 actions views for "actions", (logits, actions) pairs for "both".  `biases` as in mlp_forward."""
    root = obs_root.device.index
    devs = [int(d) for d in devices]
    if devs[0] != root:
        raise ValueError("obs must live on the root GPU (devices[0])")
    _check_policy(w1, w3, biases, output)
    ops.ensure_init(set(devs))
    M = obs_root.shape[0]
    d_out = w3.shape[0]
    if output != "actions" and out_root is None:
        out_root = torch.empty(M, d_out, dtype=torch.bfloat16, device=obs_root.device)
    if output == "logits":
        actions_root = None
    else:
        if actions_root is None:
            actions_root = torch.empty(M, dtype=torch.int64, device=obs_root.device)
        if output == "actions":
            out_root = None
    root_stream = torch.cuda.current_stream(root)
    ready = torch.cuda.Event()
    ready.record(root_stream)
    bounds = [ops.shard_bounds(M, len(devs), r) for r in range(len(devs))]
    if output == "logits":
        views = [out_root[b:e] for b, e in bounds]
    elif output == "actions":
        views = [actions_root[b:e] for b, e in bounds]
    else:
        views = [(out_root[b:e], actions_root[b:e]) for b, e in bounds]
    weights = {dev: _weights_on(dev, (w1, w2, w3)) + _weights_on(dev, biases) for dev in set(devs)}
    distinct = len(set(devs)) == len(devs) and len(devs) > 1
    pushable = distinct and all((e - b) % 128 == 0 for b, e in bounds) and \
        -(-max(e - b for b, e in bounds) // PUSH_CHUNK_ROWS) <= 64
    if transfer not in ("auto", "pull", "push"):
        raise ValueError("transfer must be 'auto', 'pull' or 'push'")
    if transfer == "push" and not pushable:
        raise ValueError("push transfer needs distinct devices and shards of a multiple of 128 rows")
    if pushable and transfer != "pull":
        _mlp_scatter_gather_pushed(obs_root, w1, w2, w3, devs, out_root, bounds, weights, output, actions_root)
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
            mlp_forward(obs_root[b:e], ws[0], ws[1], ws[2], out=None if out_root is None else out_root[b:e],
                        device=dev, stream=st, biases=ws[3:], output=output,
                        actions=None if actions_root is None else actions_root[b:e])
            if dev != root:
                ev = torch.cuda.Event()
                ev.record(st)
                return ev
        return None

    global _pool
    if len(set(devs)) > 1:
        if _pool is None:
            from concurrent.futures import ThreadPoolExecutor

            _pool = ThreadPoolExecutor(max_workers=16, thread_name_prefix="ktb-mlp")
        done = list(_pool.map(issue, range(len(devs))))
    else:
        done = [issue(r) for r in range(len(devs))]
    for ev in done:
        if ev is not None:
            root_stream.wait_event(ev)
    return views
