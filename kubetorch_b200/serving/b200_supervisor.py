"""The B200 dispatch backend: distribution_type "b200" behind the reference's supervisor seam
(kt/serving/supervisor_factory.py:11-58 — "new distribution_type values are added here").

Contract honoured (the reference's own plugin API, exactly as its server drives it):

  construction   `supervisor_factory(**json.loads(KT_DISTRIBUTED_CONFIG))` — JSON values only, no
                 pointers, no callable object (kt/serving/http_server.py:971-1002).  The callable is
                 loaded from KT_FILE_PATH / KT_MODULE_NAME / KT_CLS_OR_FN_NAME / KT_INIT_ARGS in
                 setup() (http_server.py:1040-1101) and the serialization allow-list is read from
                 KT_ALLOWED_SERIALIZATION at call time (http_server.py:1777-1782).
  call           `sup.call(request, cls_or_fn_name, method_name, params, distributed_subcall)` with
                 the RAW request body (http_server.py:1757-1763): `{"data": "<b64 pickle>",
                 "workers": ..., "restart_procs": ...}` for X-Serialization: pickle, `{"args": [...],
                 "kwargs": {...}}` for json.  Decoding (http_server.py:1768-1822) and per-rank result
                 encoding `{"data": b64(pickle(result))}` / JSON check (http_server.py:1825-1842)
                 happen HERE, because on this route there is no worker process to do them.
  result         rank-ordered list, one entry per participating rank (spmd_supervisor.py:547-570);
                 `workers=` narrows the participating nodes with the reference's selector semantics
                 and error strings (spmd_supervisor.py:219-261); `restart_procs=True` re-creates the
                 backend state first (spmd_supervisor.py:263-268).
  errors         raised as Python exceptions; the server's generic handler (http_server.py:1478-1526)
                 or LocalClient packages them in the reference envelope.

The in-package client (serving/local_client.py) hands over LIVE objects instead of a wire body
(`params` has "args" but no "data"): then nothing is decoded and the per-rank results are returned
as live tensors (zero-copy views of the result buffer) — the wire codecs only run for wire bodies.

One controller process drives N local H100s.  For a @kt.mapped callable a remote call becomes:

    device-resident arg (CUDA tensor on the root GPU)
        ktb_scatter_map_gather: rank r's kernel pulls `x.chunk(N)[r]` from the root's HBM over
        NVLink/NVSwitch, applies the op, pushes the result into the root's result buffer —
        scatter, exec and gather are ONE kernel per rank; the caller gets N views, rank-ordered.
    host-resident arg (CPU tensor; the reference's client lives outside the GPU)
        each rank's shard goes host → its own GPU → host over that GPU's own PCIe link
        (ktb_map_host_multi: chunked H2D / kernel / D2H), ranks in parallel.
    reduce="sum"
        ktb_scatter_map_reduce: per-rank warp-shuffle reduction, scalar peer-stored to the root.
    "gae"
        ktb_gae_f32: one launch on the root GPU over every selected rank's rows.
    "vtrace"
        ktb_vtrace_f32: the same, one launch on the root GPU.
    "nstep"
        ktb_nstep_f32: the same, one launch on the root GPU.
    "retrace"
        ktb_retrace_f32: the same, one launch on the root GPU.
    "per"
        ktb_per_sample_f32: one launch on the root GPU over every selected rank's strata.

There is NO CPU fallback here: a missing library or GPU raises.
"""
from __future__ import annotations

import base64
import json
import os
import pickle
import threading
from typing import List, Optional

from ..distributed import local_pod_ips
from ..exceptions import PodTerminatedError, SerializationError
from ..mapped import (DQN_OPTIONS, ELEMENTWISE_OPS, GAE_OPTIONS, MLP_FORMS, NSTEP_ARGUMENTS, PER_ARGUMENTS,
                      RETRACE_OPTIONS, TD_OPTIONS, VTRACE_ARGUMENTS, VTRACE_OPTIONS, check_finite, mapped_spec,
                      names_arguments)
from .codec import HTTPException, check_allowed
from .process_worker import instantiate, load_callable, load_callable_from_env, resolve_method
from .supervisors import check_callable_name, select_worker_nodes

_INT_DTYPES = ("torch.int32", "torch.int64")


class B200Supervisor:
    def __init__(self, pointers=None, init_args=None, name: str = None, devices: Optional[List[int]] = None,
                 num_proc=None, workers: int = None, quorum_workers: int = None, distributed: bool = True,
                 allowed_serialization: Optional[str] = None, variant: int = 0,
                 callable_obj=None, transfer: str = "auto", placement: str = "auto",
                 quorum_timeout=None, monitor_members=None, port=None, restart_procs: bool = True,
                 max_threads_per_proc: int = 10, self_check: bool = True, **extra):
        # (pointers, init_args, name, callable_obj) are the in-package deploy path; the reference's server passes
        # none of them: the callable then comes from the KT_* environment in setup()
        self.pointers, self.init_args, self.name = pointers, init_args, name
        self.callable_obj = callable_obj
        self.devices = [int(d) for d in devices] if devices is not None else None
        self.num_proc = num_proc
        self.workers = int(workers or quorum_workers or 1)
        self.distributed = distributed
        self.allowed_serialization = allowed_serialization  # None → KT_ALLOWED_SERIALIZATION at call time
        self.variant = variant
        self.self_check = bool(self_check)
        self._callable = None
        self._pin_cache = {}
        self._lock = threading.Lock()
        self._host_lock = threading.Lock()
        self._push = None
        self._small = None  # small-call fast path state (see _device_map)
        self.ops = None
        if transfer not in ("auto", "pull", "push"):
            raise ValueError("transfer must be 'auto', 'pull' or 'push'")
        self.transfer = transfer
        # where device-resident element-wise shards execute: "ranks" = rank r on GPU r whatever the size (the sharded
        # path the benchmarks measure); "root" = every rank's shard on the root GPU (same results; for HBM-bound ops a
        # root-resident arg is served faster by the root's own HBM than through its NVLink port, profiles §2);
        # "auto" (default) = "ranks" from SMALL_CALL_BYTES up, "root" below it (launch-bound calls: one launch
        # instead of N launches plus 2N peer hops)
        if placement not in ("auto", "ranks", "root"):
            raise ValueError("placement must be 'auto', 'ranks' or 'root'")
        self.placement = placement
        self.worker_ips: List[str] = []
        self.config_hash = hash(("b200", tuple(self.devices or ()), num_proc, self.workers, distributed))

    # ---- lifecycle ------------------------------------------------------------------------------------
    def _load_device(self):
        """The device layer (ctypes binding of libktb200.so).  Fails loudly without the library or a GPU."""
        from ..device import lib as L
        from ..device import ops

        L.load()
        ops.require_cuda()
        return ops

    def setup(self):
        self.ops = ops = self._load_device()
        if self.devices is None:
            per = self.num_proc
            if per in (None, "auto", 0):  # pytorch_process.py:31-41: "auto" = one rank per visible GPU
                per = max(1, ops.device_count() // max(1, self.workers))
            self.devices = self._pick_devices(int(per) * self.workers)
        if self.devices and max(self.devices) >= ops.device_count():
            raise RuntimeError(
                f"kt.Compute asked for GPU index {max(self.devices)} ({len(self.devices)} ranks) but only "
                f"{ops.device_count()} GPUs are visible"
            )
        ops.ensure_init(self.devices)
        if len(self.devices) % self.workers:
            self.workers = 1
        self.worker_ips = local_pod_ips(self.workers)
        if self.name is None:
            self.name = os.environ.get("KT_CLS_OR_FN_NAME")
        if self.callable_obj is not None:
            self._callable = instantiate(self.callable_obj, self.init_args)
        elif self.pointers is not None:
            self._callable = load_callable(self.pointers, self.init_args)
        else:
            self._callable = load_callable_from_env()  # the reference server's path
        if self.self_check:
            self._self_check()

    def _pick_devices(self, n: int) -> List[int]:
        """N of the visible GPUs, rank order.  All of them when N covers the box; otherwise spread over the NUMA nodes
        (GPU 0 stays the root): the GPUs of one socket share that socket's host PCIe bandwidth, so spreading a partial
        deployment over both sockets raises what the host-resident path can move."""
        ops = self.ops
        total = ops.device_count()
        if n >= total or n <= 1:
            return list(range(n))
        try:
            by_node = {}
            for d in range(total):
                by_node.setdefault(ops.device_numa_node(d), []).append(d)
        except Exception:  # noqa: BLE001 - no topology information: first N devices
            return list(range(n))
        if len(by_node) < 2:
            return list(range(n))
        node_of = {d: k for k, ds in by_node.items() for d in ds}
        order, queues = [], [list(by_node[k]) for k in sorted(by_node, key=lambda k: by_node[k][0])]
        while len(order) < n:
            for q in queues:
                if q and len(order) < n:
                    order.append(q.pop(0))
        # ranks of one node stay adjacent (shards of neighbouring ranks share a socket): [0, 4, 1, 5] -> [0, 1, 4, 5]
        picked = sorted(order, key=lambda d: (node_of.get(d, 0) != node_of.get(0, 0), d))
        return picked if picked and picked[0] == 0 else list(range(n))

    def cleanup(self):
        self._callable = None
        self._pin_cache.clear()
        self._push = None
        self._small = None

    @property
    def world_size(self) -> int:
        return len(self.devices)

    @property
    def ranks_per_worker(self) -> int:
        return max(1, len(self.devices) // max(1, self.workers))

    # ---- deploy-time check: the declared op must compute what the Python body computes ---------------------
    def _self_check(self):
        """Run body vs kernel on a small seeded tensor per dtype and refuse the deployment on mismatch
        (the Python body stays the definition; @kt.mapped is a claim, checked here)."""
        import inspect

        import torch

        targets = []
        c = self._callable
        if inspect.isfunction(c) or inspect.ismethod(c):
            if mapped_spec(c) is not None:
                targets.append(c)
        else:  # a kt.cls instance: every @kt.mapped method
            for attr in dir(type(c)):
                m = None if attr.startswith("__") else getattr(c, attr, None)
                if callable(m) and mapped_spec(m) is not None:
                    targets.append(m)
        for method in targets:
            spec = mapped_spec(method)
            if spec.op == "gae" and spec.extra.get("self_check") is not False:
                self._self_check_gae(spec, method)
            if spec.op == "vtrace" and spec.extra.get("self_check") is not False:
                self._self_check_vtrace(spec, method)
            if spec.op == "nstep" and spec.extra.get("self_check") is not False:
                self._self_check_nstep(spec, method)
            if spec.op == "retrace" and spec.extra.get("self_check") is not False:
                self._self_check_retrace(spec, method)
            if spec.op == "per" and spec.extra.get("self_check") is not False:
                self._self_check_per(spec, method)
            if spec.op not in ELEMENTWISE_OPS or spec.extra.get("self_check") is False:
                continue
            if not (isinstance(spec.alpha, (int, float)) and isinstance(spec.beta, (int, float))):
                continue  # parameters are call arguments: nothing constant to check at deploy time
            names = list(inspect.signature(method).parameters)
            if len(names) != 1:
                continue
            world, dev0 = self.world_size, self.devices[0]
            gen = torch.Generator().manual_seed(1234)
            integral = float(spec.alpha).is_integer() and float(spec.beta).is_integer()
            for dtype in (torch.float32, torch.bfloat16, torch.int64):
                if dtype is torch.int64 and not integral:
                    continue
                if dtype.is_floating_point:
                    x = torch.randn(4 * world + 3, 5, generator=gen).to(dtype)
                else:
                    x = torch.randint(-1000, 1000, (4 * world + 3, 5), generator=gen, dtype=dtype)
                saved = {k: os.environ.get(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
                want = []
                try:
                    for r in range(world):
                        os.environ.update({"RANK": str(r), "WORLD_SIZE": str(world), "LOCAL_RANK": str(r)})
                        want.append(method(x.clone()))
                except Exception:  # noqa: BLE001 - a body that cannot run here (needs a GPU arg, a group, ...) is skipped
                    want = None
                finally:
                    for k, v in saved.items():
                        if v is None:
                            os.environ.pop(k, None)
                        else:
                            os.environ[k] = v
                if want is None:
                    break
                got = self._run_mapped(spec, method, [x.to(f"cuda:{dev0}")], {}, list(range(world)))
                self.ops.synchronize(dev0)
                ok = isinstance(got, list) and len(got) == len(want)
                if ok and spec.reduce == "sum":
                    tol = [8 * 2.0 ** -8 * float(x.float().abs().sum()) if dtype.is_floating_point else 0] * len(want)
                    ok = all(abs(float(g) - float(w)) <= t for g, w, t in zip(got, want, tol))
                elif ok:
                    ok = all(isinstance(w, torch.Tensor) and g.dtype == w.dtype and tuple(g.shape) == tuple(w.shape)
                             and torch.equal(g.cpu().reshape(-1).view(torch.uint8),
                                             w.contiguous().reshape(-1).view(torch.uint8))
                             for g, w in zip(got, want))
                if not ok:
                    raise ValueError(
                        f"@kt.mapped self-check failed for '{getattr(method, '__name__', method)}': the declared op "
                        f"'{spec.op}' (alpha={spec.alpha}, beta={spec.beta}, reduce={spec.reduce}) does not reproduce "
                        f"the Python body on a seeded {dtype} tensor; refusing to deploy"
                    )

    def _self_check_gae(self, spec, method):
        """A "gae" callable with a constant gamma and lam: its body on CPU, rank by rank, against the kernel on seeded
        (4·world + 3, 9) rollouts with some done = 1; refuse the deployment on any bit difference.  This catches a body
        that reads dones as episode starts (CleanRL's buffers, shifted by one step) and a γ or λ other than declared."""
        import inspect

        import torch

        if any(isinstance(spec.extra[k], str) for k in GAE_OPTIONS) or len(inspect.signature(method).parameters) != 4:
            return   # gamma or lam is a call argument: nothing constant to check at deploy time
        world, dev0 = self.world_size, self.devices[0]
        gen = torch.Generator().manual_seed(1234)
        n, t = 4 * world + 3, 9
        rewards, values = torch.randn(n, t, generator=gen), torch.randn(n, t, generator=gen)
        dones = (torch.rand(n, t, generator=gen) < 0.25).float()
        dones[::3, t // 2] = 1.0
        last_values = torch.randn(n, generator=gen)
        args = (rewards, values, dones, last_values)
        saved = {k: os.environ.get(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
        want = []
        try:
            for r in range(world):
                os.environ.update({"RANK": str(r), "WORLD_SIZE": str(world), "LOCAL_RANK": str(r)})
                want.append(method(*(a.clone() for a in args)))
        except Exception:  # noqa: BLE001 - a body that cannot run here (needs a GPU arg, a group, ...) is skipped
            return
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        got = self._run_mapped(spec, method, [a.to(f"cuda:{dev0}") for a in args], {}, list(range(world)))
        self.ops.synchronize(dev0)

        def same(g, w):
            return isinstance(w, torch.Tensor) and w.dtype == torch.float32 and tuple(g.shape) == tuple(w.shape) \
                and torch.equal(g.cpu().view(torch.int32), w.contiguous().view(torch.int32))

        if not all(isinstance(w, (tuple, list)) and len(w) == 2 and all(same(*p) for p in zip(g, w))
                   for g, w in zip(got, want)):
            raise ValueError(
                f"@kt.mapped self-check failed for '{getattr(method, '__name__', method)}': the 'gae' op (gamma="
                f"{spec.extra['gamma']}, lam={spec.extra['lam']}) does not reproduce the Python body's (advantages, "
                f"returns) bit for bit on seeded rollouts; refusing to deploy.  The op reads dones[:, t] as the done "
                f"flag of transition t (the episode ended after the action at step t): CleanRL's dones[t] marks that "
                f"observation t starts an episode, so pass torch.cat([dones[1:], next_done[None]]).T.contiguous()")

    def _self_check_vtrace(self, spec, method):
        """A "vtrace" callable with a constant gamma and lam: its body on the root GPU, rank by rank, against the kernel
        on seeded (4·world + 3, 9) rollouts whose log-ratios fall on both sides of every threshold, with some done = 1;
        refuse the deployment on any bit difference.  The body runs on the GPU because ρ = exp(log_rhos) is CUDA's expf
        there, which torch's CPU exp does not reproduce.  This catches a body that reads dones as episode starts, a γ,
        λ or threshold other than declared (TorchBeast's traces clamped at 1.0 under another c_bar=)."""
        import inspect

        import torch

        if any(isinstance(spec.extra[k], str) for k in VTRACE_ARGUMENTS) or \
                len(inspect.signature(method).parameters) != 5:
            return   # gamma or lam is a call argument: nothing constant to check at deploy time
        world, dev0 = self.world_size, self.devices[0]
        gen = torch.Generator().manual_seed(1234)
        n, t = 4 * world + 3, 9
        # log-ratios spread over ±2.3: ρ from 0.1 to 10, across any threshold a deployment would declare
        log_rhos = (torch.rand(n, t, generator=gen) * 4.6 - 2.3)
        rewards, values = torch.randn(n, t, generator=gen), torch.randn(n, t, generator=gen)
        dones = (torch.rand(n, t, generator=gen) < 0.25).float()
        dones[::3, t // 2] = 1.0
        bootstrap = torch.randn(n, generator=gen)
        args = [a.to(f"cuda:{dev0}") for a in (log_rhos, rewards, values, dones, bootstrap)]
        saved = {k: os.environ.get(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
        want = []
        try:
            with torch.cuda.device(dev0):
                for r in range(world):
                    os.environ.update({"RANK": str(r), "WORLD_SIZE": str(world), "LOCAL_RANK": str(r)})
                    want.append(method(*(a.clone() for a in args)))
        except Exception:  # noqa: BLE001 - a body that cannot run here (needs an argument, a group, ...) is skipped
            return
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        got = self._run_mapped(spec, method, args, {}, list(range(world)))
        self.ops.synchronize(dev0)

        def same(g, w):
            return isinstance(w, torch.Tensor) and w.dtype == torch.float32 and tuple(g.shape) == tuple(w.shape) \
                and torch.equal(g.cpu().view(torch.int32), w.cpu().contiguous().view(torch.int32))

        if not all(isinstance(w, (tuple, list)) and len(w) == 2 and all(same(*p) for p in zip(g, w))
                   for g, w in zip(got, want)):
            declared = ", ".join(f"{k}={spec.extra[k]}" for k in VTRACE_OPTIONS)
            raise ValueError(
                f"@kt.mapped self-check failed for '{getattr(method, '__name__', method)}': the 'vtrace' op ({declared}) "
                f"does not reproduce the Python body's (vs, pg_advantages) bit for bit on seeded rollouts; refusing to "
                f"deploy.  The op computes TorchBeast's from_importance_weights with the declared gamma, lam (seed_rl's "
                f"lambda_) and thresholds, clamping the traces at c_bar (TorchBeast clamps them at 1.0: declare "
                f"c_bar=1.0), and reads dones[:, t] as the done flag of transition t, TorchBeast's batch['done'][1:] "
                f"(not a flag that observation t starts an episode)")

    def _self_check_nstep(self, spec, method):
        """An "nstep" callable with a constant gamma: its body on CPU, rank by rank, against the kernel on seeded
        (4·world + 3, n + 8) rollouts with some done = 1, so that both full windows and the padded end are exercised;
        refuse the deployment on any bit difference (the op has no exp, so the CPU's bits are the GPU's).  This catches
        a body that reads dones as episode starts, a γ or n other than declared, and one that bootstraps 0 past the
        rollout's end instead of V(s_T)."""
        import inspect

        import torch

        if any(isinstance(spec.extra[k], str) for k in NSTEP_ARGUMENTS) or \
                len(inspect.signature(method).parameters) != 5:
            return   # gamma is a call argument: nothing constant to check at deploy time
        world, dev0 = self.world_size, self.devices[0]
        gen = torch.Generator().manual_seed(1234)
        n, t = 4 * world + 3, spec.extra["n"] + 8
        rewards, values = torch.randn(n, t, generator=gen), torch.randn(n, t, generator=gen)
        dones = (torch.rand(n, t, generator=gen) < 0.25).float()
        dones[::3, t // 2] = 1.0
        baseline, last_values = torch.randn(n, t, generator=gen), torch.randn(n, generator=gen)
        args = (rewards, values, dones, baseline, last_values)
        saved = {k: os.environ.get(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
        want = []
        try:
            for r in range(world):
                os.environ.update({"RANK": str(r), "WORLD_SIZE": str(world), "LOCAL_RANK": str(r)})
                want.append(method(*(a.clone() for a in args)))
        except Exception:  # noqa: BLE001 - a body that cannot run here (needs a GPU arg, a group, ...) is skipped
            return
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        got = self._run_mapped(spec, method, [a.to(f"cuda:{dev0}") for a in args], {}, list(range(world)))
        self.ops.synchronize(dev0)

        def same(g, w):
            return isinstance(w, torch.Tensor) and w.dtype == torch.float32 and tuple(g.shape) == tuple(w.shape) \
                and torch.equal(g.cpu().view(torch.int32), w.cpu().contiguous().view(torch.int32))

        if not all(isinstance(w, (tuple, list)) and len(w) == 2 and all(same(*p) for p in zip(g, w))
                   for g, w in zip(got, want)):
            raise ValueError(
                f"@kt.mapped self-check failed for '{getattr(method, '__name__', method)}': the 'nstep' op (n="
                f"{spec.extra['n']}, gamma={spec.extra['gamma']}) does not reproduce the Python body's (returns, td) "
                f"bit for bit on seeded rollouts; refusing to deploy.  The op sums n={spec.extra['n']} discounted "
                f"rewards with gamma={spec.extra['gamma']}, reads dones[:, t] as the done flag of transition t (not a "
                f"flag that observation t starts an episode: CleanRL's dones become torch.cat([dones[1:], "
                f"next_done[None]]).T.contiguous()), and past the rollout's end bootstraps from last_values, V(s_T), "
                f"not from 0")

    def _self_check_retrace(self, spec, method):
        """A "retrace" callable with a constant gamma and lam: its body on the root GPU, rank by rank, against the
        kernel on seeded (4·world + 3, 9) rollouts whose log-ratios fall on both sides of 0, so that the min(1, ρ) clip
        binds at some steps and not at others, with some done = 1; refuse the deployment on any bit difference.  The
        body runs on the GPU because ρ = exp(log_rhos) is CUDA's expf there, which torch's CPU exp does not reproduce.
        This catches a body that reads dones as episode starts, a γ or λ other than declared, unclipped traces λ·ρ, and
        one that reads the current step's values where the target reads the next step's."""
        import inspect

        import torch

        if any(isinstance(spec.extra[k], str) for k in RETRACE_OPTIONS) or \
                len(inspect.signature(method).parameters) != 7:
            return   # gamma or lam is a call argument: nothing constant to check at deploy time
        world, dev0 = self.world_size, self.devices[0]
        gen = torch.Generator().manual_seed(1234)
        n, t = 4 * world + 3, 9
        log_rhos = torch.rand(n, t, generator=gen) * 4.6 - 2.3   # ρ from 0.1 to 10: the clip at 1 binds about half
        rewards, q, values, baseline = (torch.randn(n, t, generator=gen) for _ in range(4))
        dones = (torch.rand(n, t, generator=gen) < 0.25).float()
        dones[::3, t // 2] = 1.0
        bootstrap = torch.randn(n, generator=gen)
        args = [a.to(f"cuda:{dev0}") for a in (log_rhos, rewards, q, values, dones, baseline, bootstrap)]
        saved = {k: os.environ.get(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
        want = []
        try:
            with torch.cuda.device(dev0):
                for r in range(world):
                    os.environ.update({"RANK": str(r), "WORLD_SIZE": str(world), "LOCAL_RANK": str(r)})
                    want.append(method(*(a.clone() for a in args)))
        except Exception:  # noqa: BLE001 - a body that cannot run here (needs an argument, a group, ...) is skipped
            return
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        got = self._run_mapped(spec, method, args, {}, list(range(world)))
        self.ops.synchronize(dev0)

        def same(g, w):
            return isinstance(w, torch.Tensor) and w.dtype == torch.float32 and tuple(g.shape) == tuple(w.shape) \
                and torch.equal(g.cpu().view(torch.int32), w.cpu().contiguous().view(torch.int32))

        if not all(isinstance(w, (tuple, list)) and len(w) == 2 and all(same(*p) for p in zip(g, w))
                   for g, w in zip(got, want)):
            raise ValueError(
                f"@kt.mapped self-check failed for '{getattr(method, '__name__', method)}': the 'retrace' op (gamma="
                f"{spec.extra['gamma']}, lam={spec.extra['lam']}) does not reproduce the Python body's (returns, td) "
                f"bit for bit on seeded rollouts; refusing to deploy.  The op computes rlax's retrace_continuous with "
                f"the declared gamma and lam: traces c = lam * min(1, exp(log_rhos)), the target r[:, t] + "
                f"gamma * (1 - dones[:, t]) * (values[:, t + 1] - c[:, t + 1] * q[:, t + 1] + c[:, t + 1] * g), "
                f"bootstrapped from bootstrap_value at the rollout's end, and td = returns - baseline.  It reads "
                f"dones[:, t] as the done flag of transition t (not a flag that observation t starts an episode: "
                f"CleanRL's dones become torch.cat([dones[1:], next_done[None]]).T.contiguous())")

    def _self_check_per(self, spec, method):
        """A "per" callable: its body on the root GPU, rank by rank, against the kernel, refusing the deployment on any
        bit difference.  The body runs on the GPU because its pow is CUDA's there.  The check passes its own seed and
        its own β where those name call arguments, and calls the body with the priorities and those arguments only (a
        body that needs more is not checked).  Two priority vectors of C = 1000, not a power of two: seeded values with
        30 % zeros, index 0 among them, and one dominant item; and the same zeros with every other item the least
        subnormal, where every mass and every partial sum is a whole number of that subnormal, so that masses equal
        left sums and `mass >= left` decides the descent.  This catches uniform in place of stratified draws, rank-local strata, `mass > left`,
        weights not divided by the largest one, and another noise stream."""
        import inspect

        import torch

        params = list(inspect.signature(method).parameters)
        given = {v: 8675309 if k == "seed" else 0.6 for k, v in spec.extra.items() if k in PER_ARGUMENTS
                 and isinstance(v, str)}
        if len(params) != 1 + len(given):
            return   # the body takes arguments the check cannot supply
        world, dev0 = self.world_size, self.devices[0]
        gen = torch.Generator().manual_seed(1234)
        c = 1000
        prio = torch.rand(c, generator=gen) * 2
        prio[torch.rand(c, generator=gen) < 0.3] = 0.0
        prio[0] = 0.0
        prio[617] = 500.0
        tiny = torch.where(prio > 0, torch.tensor(1e-45), torch.tensor(0.0))
        for p in (prio, tiny):
            p = p.to(f"cuda:{dev0}")
            kwargs = {params[0]: p, **given}
            saved = {k: os.environ.get(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK")}
            want = []
            try:
                with torch.cuda.device(dev0):
                    for r in range(world):
                        os.environ.update({"RANK": str(r), "WORLD_SIZE": str(world), "LOCAL_RANK": str(r)})
                        want.append(method(**{k: v.clone() if isinstance(v, torch.Tensor) else v
                                              for k, v in kwargs.items()}))
            except Exception:  # noqa: BLE001 - a body that cannot run here (needs a group, ...) is skipped
                return
            finally:
                for k, v in saved.items():
                    if v is None:
                        os.environ.pop(k, None)
                    else:
                        os.environ[k] = v
            got = self._run_mapped(spec, method, [], kwargs, list(range(world)))
            self.ops.synchronize(dev0)

            def same(g, w, dtype):
                return isinstance(w, torch.Tensor) and w.dtype == dtype and tuple(g.shape) == tuple(w.shape) \
                    and torch.equal(g.cpu().view(torch.int32 if dtype == torch.float32 else dtype),
                                    w.cpu().contiguous().view(torch.int32 if dtype == torch.float32 else dtype))

            if not all(isinstance(w, (tuple, list)) and len(w) == 2 and same(g[0], w[0], torch.int64)
                       and same(g[1], w[1], torch.float32) for g, w in zip(got, want)):
                raise ValueError(
                    f"@kt.mapped self-check failed for '{getattr(method, '__name__', method)}': the 'per' op (batch="
                    f"{spec.extra['batch']}, beta={spec.extra['beta']}, seed={spec.extra['seed']}) does not reproduce "
                    f"the Python body's (indices, weights) bit for bit on seeded priorities; refusing to deploy.  The "
                    f"op draws stratum j of torch.arange(batch).chunk(WORLD_SIZE)[RANK] (the global j) from the sum "
                    f"tree at mass (j + u) * (total / batch) with u = kubetorch_b200.sampling.replay_noise(seed, j, 1), "
                    f"steps right where mass >= left and the right child is > 0, and weights each draw by "
                    f"(p / total * C) ** -beta / (min p / total * C) ** -beta")

    # ---- small-call lane (the local CUDA-stream scheduler for launch-bound calls) ----------------------------
    SMALL_CALL_BYTES = 4 << 20

    def fast_path(self, serialization_ok):
        """A closure `fast(x) -> result | None` for the deployed FUNCTION, or None when there is none.

        The reference pays HTTP + pickle + queue hops per call (≈1 ms); here a small device-resident call is
        launch-bound, so the per-call host work is cut to: argument checks, one `torch.empty_like`, ONE ctypes hop
        that binds and launches the kernel on the caller's current stream, and the shard views.  For payloads under
        SMALL_CALL_BYTES every rank's shard executes on the root GPU in that one launch (the shards of an
        element-wise op are contiguous in the root's memory; sending 128-byte shards over NVLink to seven other
        GPUs and back costs more than mapping them where they are) — results are bit-identical to the spread
        placement.  Anything the lane does not cover returns None and takes the general path (same semantics,
        same errors)."""
        import inspect

        import torch

        method = self._callable
        if not (inspect.isfunction(method) or inspect.ismethod(method)) or not serialization_ok:
            return None
        spec = mapped_spec(method)
        if spec is None or spec.op not in ELEMENTWISE_OPS or spec.reduce is not None:
            return None
        if not (isinstance(spec.alpha, (int, float)) and isinstance(spec.beta, (int, float))):
            return None
        if len(inspect.signature(method).parameters) != 1 or self.ops is None or not hasattr(self.ops, "fast_map"):
            return None
        world, root, distributed = self.world_size, self.devices[0], self.distributed
        if self.placement == "ranks" and world > 1:
            return None                      # explicit spread placement: every call fans out, whatever its size
        spread_ok = self.placement == "auto" and world > 1 and len(set(self.devices)) == world
        small = self.SMALL_CALL_BYTES
        launch = self.ops.fast_map(root, spec.op, spec.alpha, spec.beta)
        codes = self.ops.fast_dtype_codes(spec.alpha, spec.beta)
        Tensor, empty_like = torch.Tensor, torch.empty_like

        def fast(x):
            if type(x) is not Tensor or not x.is_cuda:
                return None
            code = codes.get(x.dtype)
            if code is None or x.dim() == 0 or not x.is_contiguous() or x.device.index != root:
                return None
            n = x.numel()
            if n == 0 or (spread_ok and n * x.element_size() >= small) or self._callable is None:
                return None
            out = empty_like(x)
            launch(code, x.data_ptr(), out.data_ptr(), n)
            if world == 1:
                return [out] if distributed else out
            views = list(out.chunk(world))
            while len(views) < world:          # ranks past the data return an empty shard, like x.chunk(w)[r:r+1]
                views.append(out[:0])
            return views

        return fast

    def batch_path(self, serialization_ok):
        """`batch(xs) -> [result per x] | None`: MANY small calls of the deployed function coalesced into ONE segmented
        launch (ktb_map_batch: the descriptors ride in the kernel parameters), results carved out of one arena.
        Reached from the public API as `remote.map(xs)`.  Same coverage rules as fast_path(); None = not covered."""
        import inspect

        import torch

        method = self._callable
        if not (inspect.isfunction(method) or inspect.ismethod(method)) or not serialization_ok or self.ops is None:
            return None
        spec = mapped_spec(method)
        if spec is None or spec.op not in ELEMENTWISE_OPS or spec.reduce is not None or not hasattr(self.ops, "batch_map"):
            return None
        if not (isinstance(spec.alpha, (int, float)) and isinstance(spec.beta, (int, float))):
            return None
        if len(inspect.signature(method).parameters) != 1 or (self.placement == "ranks" and self.world_size > 1):
            return None
        world, root, distributed = self.world_size, self.devices[0], self.distributed
        codes = self.ops.fast_dtype_codes(spec.alpha, spec.beta)
        run = self.ops.batch_map(root, spec.op, spec.alpha, spec.beta)
        small = self.SMALL_CALL_BYTES
        Tensor = torch.Tensor

        def batch(xs):
            if not xs:
                return []
            dt = xs[0].dtype if type(xs[0]) is Tensor else None
            code = codes.get(dt)
            if code is None:
                return None
            es = xs[0].element_size()
            for x in xs:
                if type(x) is not Tensor or x.dtype is not dt or not x.is_cuda or x.device.index != root or \
                        x.dim() != 1 or not x.is_contiguous() or x.numel() == 0 or x.numel() * es >= small:
                    return None
            sizes = [x.numel() for x in xs]
            outs = run(code, dt, xs, sizes)
            if world == 1:
                return [[o] for o in outs] if distributed else list(outs)
            res = []
            for o in outs:
                v = list(o.chunk(world))
                while len(v) < world:
                    v.append(o[:0])
                res.append(v)
            return res

        return batch

    # ---- the call ---------------------------------------------------------------------------------------
    def call(self, request, cls_or_fn_name, method_name=None, params=None, distributed_subcall=False):
        serialization = request.headers.get("X-Serialization", "json")
        if self._callable is None:
            raise HTTPException(503, "Server is loading the callable. Please retry in a moment.")
        check_callable_name(cls_or_fn_name, self.name)
        check_allowed(serialization, self.allowed_serialization)
        # wire body (from the reference's server) or live objects (from LocalClient)?  http_server.py:1768-1822
        wire = isinstance(params, str) or (isinstance(params, dict) and "data" in params)
        if isinstance(params, str):
            params = pickle.loads(base64.b64decode(params.encode("utf-8"))) if serialization == "pickle" \
                else json.loads(params)
        params = dict(params or {})
        if "data" in params and serialization == "pickle":
            params.update(pickle.loads(base64.b64decode(params.pop("data").encode("utf-8"))))
        if params.get("restart_procs", False):
            self.cleanup()  # spmd_supervisor.py:263-268: fresh backend state (and a fresh kt.cls instance)
            self.setup()
        nodes = select_worker_nodes(params.get("workers"), self.worker_ips, self.worker_ips[0])
        per = self.ranks_per_worker
        ranks = [n * per + l for n in nodes for l in range(per)]
        method = resolve_method(self._callable, cls_or_fn_name, method_name)
        spec = mapped_spec(method)
        if spec is None:
            raise TypeError(
                f"'{cls_or_fn_name}' is not a @kt.mapped callable: the 'b200' backend executes registered device ops "
                "only. Use .distribute('spmd'|'pytorch', num_proc=N) to run arbitrary Python on N local ranks."
            )
        out = self._run_mapped(spec, method, params.get("args", []), params.get("kwargs", {}), ranks,
                               cls_or_fn_name=cls_or_fn_name)
        if wire or serialization == "json":
            out = [self._serialize_result(o, serialization, wire) for o in out]
        return out if self.distributed else out[0] if len(out) == 1 else out

    @staticmethod
    def _serialize_result(result, serialization: str, wire: bool):
        """_serialize_result of the reference's worker (http_server.py:1825-1842), run per rank."""
        if serialization == "pickle":
            try:
                import torch

                # a shard view would drag the whole result buffer's storage along
                if isinstance(result, torch.Tensor):
                    result = result.clone()
                elif isinstance(result, tuple):   # (logits, actions) or (actions, log_probs) of an mlp op
                    result = tuple(t.clone() if isinstance(t, torch.Tensor) else t for t in result)
                return {"data": base64.b64encode(pickle.dumps(result)).decode("utf-8")}
            except Exception as e:  # noqa: BLE001
                raise SerializationError(f"Result could not be serialized with pickle: {e}")
        if serialization == "json":
            try:
                json.dumps(result)
            except (TypeError, ValueError) as e:
                raise SerializationError(f"Result could not be serialized to JSON: {e}")
        return result

    def _run_mapped(self, spec, method, args, kwargs, ranks, cls_or_fn_name=None):
        import torch

        name = cls_or_fn_name or getattr(method, "__name__", "callable")
        x, alpha, beta, bound = spec.bind(method, args, kwargs)
        if spec.op == "mlp":
            return self._call_mlp(spec, bound, ranks)
        if spec.op == "gae":
            return self._call_gae(spec, bound, ranks)
        if spec.op == "vtrace":
            return self._call_vtrace(spec, bound, ranks)
        if spec.op == "nstep":
            return self._call_nstep(spec, bound, ranks)
        if spec.op == "retrace":
            return self._call_retrace(spec, bound, ranks)
        if spec.op == "per":
            return self._call_per(spec, bound, ranks)
        if spec.op not in ELEMENTWISE_OPS:
            raise TypeError(f"unsupported mapped op '{spec.op}'")
        if not isinstance(x, torch.Tensor):
            raise TypeError(f"mapped callable '{name}' expects a torch.Tensor argument, got {type(x).__name__}")
        if str(x.dtype) in _INT_DTYPES and spec.op != "identity":
            # the Python body (`x * 0.5`) would promote to float; the integer kernels do wrapping integer math only.  A
            # float passed as a call argument is refused even when integral (`x * 2.0` is float32 in torch); a declared
            # constant such as alpha=2.0 is checked against the body at deploy instead (_self_check)
            for label, v, declared in (("alpha", alpha, spec.alpha),
                                       ("beta", beta if spec.op == "affine" else 0, spec.beta)):
                if isinstance(v, float) and (not v.is_integer() or isinstance(declared, str)) \
                        or not isinstance(v, (int, float)):
                    raise TypeError(
                        f"mapped op '{spec.op}' on {x.dtype}: {label}={v!r} is not an integer — torch would promote "
                        "the result to floating point, which the integer kernels do not do")
        if spec.reduce == "sum":
            out = self._reduce(x, spec.op, alpha, beta, ranks)
        elif x.is_cuda:
            out = self._device_map(x, spec.op, alpha, beta, ranks)
        else:
            out = self._host_map(x, spec.op, alpha, beta, ranks)
        return out

    def _shard_views(self, flat_like, x, ranks=None):
        """Rank-ordered views of `flat_like` (same layout as x) following x.chunk(world) on dim 0."""
        rows = x.shape[0] if x.dim() > 0 else 1
        y = flat_like.view(x.shape) if x.dim() > 0 else flat_like.view(1)
        if self.world_size == 1:
            return [y]
        views = []
        for r in (range(self.world_size) if ranks is None else ranks):
            b, e = self.ops.shard_bounds(rows, self.world_size, r)
            views.append(y[b:e])
        return views

    def _all_ranks(self, ranks) -> bool:
        return ranks is None or len(ranks) == self.world_size

    def _device_map(self, x, op, alpha, beta, ranks=None):
        import torch

        ops = self.ops
        root = self.devices[0]
        if x.device.index != root:
            raise ValueError(f"device-resident args must live on the root GPU cuda:{root}, got {x.device}")
        if x.dim() == 0:
            x = x.reshape(1)
        x = x.contiguous()
        out = torch.empty_like(x)  # same device as x: the root GPU
        if not self._all_ranks(ranks):
            # `workers=` sub-selection: only the selected ranks' shards run (they keep their global RANK/WORLD_SIZE,
            # as the reference's do — recorded case mp_double_f32_1003_workers_1)
            xs, os_ = self._shard_views(x, x, ranks), self._shard_views(out, x, ranks)
            for r, xv, ov in zip(ranks, xs, os_):
                if xv.numel():
                    ops.map_tensor(xv, op, alpha, beta, out=ov, device=root if self.placement == "root" else self.devices[r])
            ops.join_devices(root, [self.devices[r] for r in ranks])
            return os_
        nbytes = x.numel() * x.element_size()
        if self.placement == "root" or (self.placement == "auto" and nbytes < self.SMALL_CALL_BYTES):
            # one launch on the root covers every rank's (contiguous) shard: see fast_path()
            ops.map_tensor(x, op, alpha, beta, out=out, variant=self.variant)
            return self._shard_views(out, x)
        distinct = len(set(self.devices)) == len(self.devices) and len(self.devices) > 1
        # the flag pipeline from 256 MiB at N >= 4 and from 1 GiB at N = 2; below that the single fused kernel per rank
        # has less fixed cost (crossover not yet re-measured on H100)
        auto_push = distinct and ((len(self.devices) >= 4 and nbytes >= (256 << 20)) or nbytes >= (1 << 30))
        if self.transfer == "push" or (self.transfer == "auto" and auto_push):
            # push/push flag pipeline: both NVLink directions carry posted writes (see ktb_push.cu)
            with self._lock:
                rows = x.shape[0]
                shard_bytes = ops.shard_bounds(rows, self.world_size, 0)[1] * ops.row_elems(x) * x.element_size()
                if self._push is None or self._push.stride < shard_bytes:
                    self._push = ops.PushSession(self.devices, shard_bytes)
                try:
                    self._push.call(x, out, op, alpha, beta)
                except ops.PushTimeout as e:
                    self._push = None
                    self._raise_device_timeout(e)
        else:
            ops.scatter_map_gather(x, op, alpha, beta, devices=self.devices, out_root=out, variant=self.variant)
        return self._shard_views(out, x)

    def _raise_device_timeout(self, e):
        """A timed-out in-kernel wait (a rank's GPU stalled or died) surfaces as the reference's
        PodTerminatedError (kt/serving/utils.py:111-190), not as silently stale results: the consume kernel skips
        its stores on a timeout, the status word is mirrored to the host behind every call."""
        import datetime

        raise PodTerminatedError(pod_name=f"{self.name}-0", reason="DeviceTimeout", status_code=503,
                                 events=[{"timestamp": datetime.datetime.now(datetime.timezone.utc).isoformat(),
                                          "reason": "DeviceTimeout", "message": str(e)}]) from None

    def check_device_health(self):
        """Synchronous form (reads every control block): used at teardown and by tests."""
        if self._push is not None:
            try:
                self._push.check()
            except self.ops.PushTimeout as e:
                self._push = None
                self._raise_device_timeout(e)

    def _pinned(self, key, like):
        buf = self._pin_cache.get(key)
        if buf is None or buf.numel() != like.numel() or buf.dtype != like.dtype:
            buf = self.ops.pinned_empty((like.numel(),), like.dtype, devices=self.devices)
            self._pin_cache[key] = buf
        return buf.view(like.shape)

    def _host_map(self, x, op, alpha, beta, ranks=None):
        if x.dim() == 0:
            x = x.reshape(1)
        x = x.contiguous()
        with self._host_lock:  # the pinned staging tensors are per deployment
            return self._host_map_locked(x, op, alpha, beta, ranks)

    def _host_map_locked(self, x, op, alpha, beta, ranks=None):
        ops = self.ops
        if not ops.is_pinned(x):
            staged = self._pinned("in", x)
            staged.copy_(x)  # page-locking copy: the caller handed us pageable memory
            x = staged
        # results are FRESH tensors every call (the reference returns new objects); the pinned allocations are
        # cached per size and laid out so that shard r's pages sit on the NUMA node of GPU r (ops.pinned_empty)
        out = ops.pinned_empty(tuple(x.shape), x.dtype, devices=self.devices)
        # one C call drives every selected rank's copy/exec/copy pipeline (persistent per-GPU issue threads in the
        # library); ranks outside a `workers=` subset are skipped
        all_ranks = self._all_ranks(ranks)
        ops.map_host(x, op, alpha, beta, out_host=out, devices=self.devices, ranks=None if all_ranks else ranks)
        o_shards = self._shard_views(out, x)
        return o_shards if all_ranks else [o_shards[r] for r in ranks]

    def _reduce(self, x, op, alpha, beta, ranks=None):
        ops = self.ops
        root = self.devices[0]
        if not x.is_cuda:
            x = x.to(f"cuda:{root}", non_blocking=True)
        elif x.device.index != root:
            raise ValueError(f"device-resident args must live on the root GPU cuda:{root}, got {x.device}")
        if x.dim() == 0:
            x = x.reshape(1)
        x = x.contiguous()
        _, partials = ops.scatter_map_reduce(x, op, alpha, beta, devices=self.devices)
        vals = partials.tolist()  # per-rank Python scalars, as the reference's ranks return
        return vals if self._all_ranks(ranks) else [vals[r] for r in ranks]

    def _call_mlp(self, spec, bound, ranks=None):
        from ..device import mlp

        names = list(bound)
        output = spec.extra.get("output", "logits")
        if spec.extra.get("bias", False):   # (obs, w1, b1, w2, b2, w3, b3): an nn.Linear policy
            obs, w1, b1, w2, b2, w3, b3 = (bound[n] for n in names[:7])
            biases = (b1, b2, b3)
        else:
            obs, w1, w2, w3 = (bound[n] for n in names[:4])
            biases = (None, None, None)
        # every option mlp_scatter_gather takes, a TD or DQN target's only with its output; None unless given
        own = {"td_target": TD_OPTIONS, "dqn_target": DQN_OPTIONS}.get(output, ())
        args = {name: None for name in MLP_FORMS if name not in TD_OPTIONS + DQN_OPTIONS or name in own}
        for option, v in spec.extra.items():
            if option not in MLP_FORMS:
                continue
            if names_arguments(option, v):   # resolved per call: mapped() checked that each names an argument
                v = bound[v] if isinstance(v, str) else tuple(bound[name] for name in v)
                if option in ("twin", "actor", "online") and len(v) == 3:   # (w1, w2, w3) of a bias-free network
                    v = (v[0], None, v[1], None, v[2], None)
                elif option == "alpha":
                    v = float(v)   # a number or a one-element tensor (on a GPU: one host synchronisation)
            args[option] = v
        try:
            out = mlp.mlp_scatter_gather(obs, w1, w2, w3, devices=self.devices, transfer=self.transfer,
                                         biases=biases, output=output, **args)
        except self.ops.PushTimeout as e:
            self._raise_device_timeout(e)
        return out if self._all_ranks(ranks) else [out[r] for r in ranks]

    def _call_gae(self, spec, bound, ranks=None):
        """(advantages, returns) per selected rank: one ktb_gae_f32 launch on the root over the rows of every run of
        consecutive selected ranks (all rows when every rank is selected).  The rows stay on the root: the op does a
        few flops per byte, and spreading them over the ranks' GPUs would move every byte over NVLink twice."""
        from ..device import returns

        return self._call_returns(spec, bound, ranks, ("rewards", "values", "dones", "last_values"), returns.gae,
                                  GAE_OPTIONS)

    def _call_vtrace(self, spec, bound, ranks=None):
        """(vs, pg_advantages) per selected rank: one ktb_vtrace_f32 launch on the root per run of consecutive selected
        ranks, as _call_gae."""
        from ..device import returns

        bars = {k: spec.extra[k] for k in ("rho_bar", "c_bar", "pg_rho_bar")}
        return self._call_returns(spec, bound, ranks, ("log_rhos", "rewards", "values", "dones", "bootstrap_value"),
                                  lambda *xs: returns.vtrace(*xs, **bars), VTRACE_ARGUMENTS)

    def _call_nstep(self, spec, bound, ranks=None):
        """(returns, td) per selected rank: one ktb_nstep_f32 launch on the root per run of consecutive selected ranks,
        as _call_gae."""
        from ..device import returns

        n = spec.extra["n"]
        return self._call_returns(spec, bound, ranks, ("rewards", "values", "dones", "baseline", "last_values"),
                                  lambda *xs: returns.nstep(*xs[:5], n, *xs[5:]), NSTEP_ARGUMENTS)

    def _call_retrace(self, spec, bound, ranks=None):
        """(returns, td) per selected rank: one ktb_retrace_f32 launch on the root per run of consecutive selected
        ranks, as _call_gae."""
        from ..device import returns

        return self._call_returns(spec, bound, ranks, ("log_rhos", "rewards", "q", "values", "dones", "baseline",
                                                       "bootstrap_value"), returns.retrace, RETRACE_OPTIONS)

    def _call_per(self, spec, bound, ranks=None):
        """(indices, weights) per selected rank: one ktb_per_sample_f32 launch on the root over the strata of every run
        of consecutive selected ranks (all `batch` strata when every rank is selected), each launch building the tree
        of the priorities, the first call argument, a CUDA tensor on the root GPU.  beta and seed are the constants
        declared or the call arguments they name."""
        import torch

        from ..device import replay

        prio = bound[next(iter(bound))]
        root = self.devices[0]
        if not isinstance(prio, torch.Tensor) or not prio.is_cuda or prio.device.index != root:
            where = prio.device if isinstance(prio, torch.Tensor) else type(prio).__name__
            raise ValueError(f"the 'per' op takes CUDA tensors on the root GPU cuda:{root}: priorities is on {where} "
                             f"(host tensors are not staged for this op)")
        batch = spec.extra["batch"]
        beta, seed = (bound[v] if isinstance(v, str) else v for v in (spec.extra[k] for k in PER_ARGUMENTS))
        ranks = list(range(self.world_size)) if ranks is None else list(ranks)
        bounds = [self.ops.shard_bounds(batch, self.world_size, r) for r in ranks]
        out = []
        i = 0
        while i < len(ranks):   # one launch per run of consecutive ranks
            j = i
            while j + 1 < len(ranks) and ranks[j + 1] == ranks[j] + 1:
                j += 1
            b, e = bounds[i][0], bounds[j][1]
            idx, w = replay.per_sample(prio, batch, seed, beta, j0=b, rows=e - b)
            out += [(idx[rb - b:re - b], w[rb - b:re - b]) for rb, re in bounds[i:j + 1]]
            i = j + 1
        return out

    def _call_returns(self, spec, bound, ranks, names, launch, arguments):
        """The first len(names) call arguments, checked to be CUDA tensors on the root GPU, and the options named in
        `arguments` (constants or call arguments, such as gamma and lam) checked to be finite: launch(*rows,
        *those options) over the rows of every run of consecutive selected ranks, its pair of [rows, T] outputs split
        into one pair of views per rank."""
        import torch

        tensors = [bound[n] for n in list(bound)[:len(names)]]
        root = self.devices[0]
        for name, t in zip(names, tensors):
            if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device.index != root:
                where = t.device if isinstance(t, torch.Tensor) else type(t).__name__
                raise ValueError(f"the '{spec.op}' op takes CUDA tensors on the root GPU cuda:{root}: {name} is on "
                                 f"{where} (host tensors are not staged for this op)")
        scalars = [bound[v] if isinstance(v, str) else v for v in (spec.extra[k] for k in arguments)]
        for name, v in zip(arguments, scalars):
            check_finite(name, v)
        rewards = tensors[names.index("rewards")]
        if rewards.dim() != 2:
            raise ValueError(f"rewards must be a 2-D [N, T] tensor, got {list(rewards.shape)}")
        ranks = list(range(self.world_size)) if ranks is None else list(ranks)
        bounds = [self.ops.shard_bounds(rewards.shape[0], self.world_size, r) for r in ranks]
        out = []
        i = 0
        while i < len(ranks):   # one launch per run of consecutive ranks
            j = i
            while j + 1 < len(ranks) and ranks[j + 1] == ranks[j] + 1:
                j += 1
            b, e = bounds[i][0], bounds[j][1]
            first, second = launch(*(x[b:e] for x in tensors), *scalars)
            out += [(first[rb - b:re - b], second[rb - b:re - b]) for rb, re in bounds[i:j + 1]]
            i = j + 1
        return out
