#!/usr/bin/env python
"""Host-resident e2e experiments on N GPUs.  JSON lines -> gpurun_out/sweep_host.jsonl

  pcie_probe   raw copy-engine bandwidth, all selected GPUs at once: H2D only, D2H only, both — from a plain pinned
               buffer (wherever torch put it) and from a NUMA-sharded one (ktb_host_alloc_sharded).  Shows what the
               box can deliver whatever our pipeline does.
  e2e_host     kt.fn(mapped).to(kt.Compute(gpus=N)) -> remote(host tensor), by input buffer kind
  raw          ops.map_host without the API layer, by chunk size
"""
import json
import os
import sys
import threading
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402


def _clone(fn):
    import types

    return types.FunctionType(fn.__code__, fn.__globals__, fn.__name__, fn.__defaults__, fn.__closure__)


import kubetorch_b200 as kt  # noqa: E402
from kubetorch_b200.device import ops  # noqa: E402
from oracle import cases  # noqa: E402

OUT = os.path.join(REPO, "gpurun_out", "sweep_host.jsonl")
os.makedirs(os.path.dirname(OUT), exist_ok=True)


def emit(**kw):
    line = json.dumps(kw)
    print(line, flush=True)
    with open(OUT, "a") as f:
        f.write(line + "\n")


def numa_maps_of(ptr):
    """N<node>=<pages> counts of the mapping that contains `ptr` (/proc/self/numa_maps), or None."""
    try:
        best = None
        for line in open("/proc/self/numa_maps"):
            parts = line.split()
            addr = int(parts[0], 16)
            if addr <= ptr:
                best = (addr, parts)
        if best is None:
            return None
        return {p.split("=")[0]: int(p.split("=")[1]) for p in best[1] if p[0] == "N" and "=" in p}
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)[:100]}


def pcie_probe(devs, n_elems, kinds):
    nb = n_elems * 4
    world = len(devs)
    dev_bufs = {}
    for d in devs:
        b, e = ops.shard_bounds(n_elems, world, devs.index(d))
        dev_bufs[d] = (torch.empty(e - b, device=f"cuda:{d}"), torch.empty(e - b, device=f"cuda:{d}"))
    for kind, (xin, xout) in kinds.items():
        for mode in ("h2d", "d2h", "both"):
            def work(d, r, reps):
                b, e = ops.shard_bounds(n_elems, world, r)
                s1, s2 = torch.cuda.Stream(d), torch.cuda.Stream(d)
                din, dout = dev_bufs[d]
                with torch.cuda.device(d):
                    for _ in range(reps):
                        if mode in ("h2d", "both"):
                            with torch.cuda.stream(s1):
                                din.copy_(xin[b:e], non_blocking=True)
                        if mode in ("d2h", "both"):
                            with torch.cuda.stream(s2):
                                xout[b:e].copy_(dout, non_blocking=True)
                    s1.synchronize()
                    s2.synchronize()

            def run(reps):
                ths = [threading.Thread(target=work, args=(d, r, reps)) for r, d in enumerate(devs)]
                [t.start() for t in ths]
                [t.join() for t in ths]

            run(2)
            t0 = time.perf_counter()
            reps = 6
            run(reps)
            dt = (time.perf_counter() - t0) / reps
            moved = nb * (2 if mode == "both" else 1)
            emit(what="pcie_probe", devs=devs, kind=kind, mode=mode, ms=dt * 1e3, gbps_total=moved / dt / 1e9,
                 gbps_per_gpu_per_dir=nb / world / dt / 1e9)


def main():
    n_gpus = int(sys.argv[1]) if len(sys.argv) > 1 else torch.cuda.device_count()
    quick = "--quick" in sys.argv
    n = 1 << 26
    devs = list(range(n_gpus))
    ops.ensure_init(devs)
    emit(what="numa", nodes={d: ops.device_numa_node(d) for d in devs}, cpus=os.cpu_count(),
         affinity=len(os.sched_getaffinity(0)))
    plain_in = torch.randn(n).pin_memory()
    plain_out = torch.empty(n).pin_memory()
    t0 = time.perf_counter()
    sh_in = ops.pinned_empty((n,), torch.float32, devices=devs)
    t_alloc = time.perf_counter() - t0
    sh_in.copy_(plain_in)
    sh_out = ops.pinned_empty((n,), torch.float32, devices=devs)
    emit(what="sharded_alloc", seconds=t_alloc, is_pinned=bool(sh_in.is_pinned()), numa_maps=numa_maps_of(sh_in.data_ptr()),
         plain_numa_maps=numa_maps_of(plain_in.data_ptr()))
    kinds = {"plain_pinned": (plain_in, plain_out), "numa_sharded": (sh_in, sh_out)}
    subsets = [devs]
    if n_gpus >= 8 and not quick:
        subsets += [[0], [0, 1], [0, 1, 2, 3], [4, 5, 6, 7], [0, 4]]
    for sub in subsets:
        k2 = kinds
        if sub != devs:   # a sharded buffer laid out for THIS subset
            a = ops.pinned_empty((n,), torch.float32, devices=sub)
            a.copy_(plain_in)
            k2 = {"plain_pinned": kinds["plain_pinned"], "numa_sharded": (a, ops.pinned_empty((n,), torch.float32, devices=sub))}
        pcie_probe(sub, n, k2)

    double = kt.mapped("scale", alpha=2.0)(_clone(cases.double))
    remote = kt.fn(double, name="host-sweep").to(
        kt.Compute(gpus=n_gpus).distribute("b200", workers=1, num_proc=n_gpus))
    for kind, (xh, _) in kinds.items():
        for _ in range(3):
            out = remote(xh, serialization="pickle")
        reps = 10
        t0 = time.perf_counter()
        for _ in range(reps):
            out = remote(xh, serialization="pickle")
        dt = (time.perf_counter() - t0) / reps
        ok = bool(torch.equal(torch.cat(out)[-4096:], xh[-4096:] * 2)) and bool(torch.equal(out[0][:4096], xh[:4096] * 2))
        emit(what="e2e_host", kind=kind, n_gpus=n_gpus, ms=dt * 1e3, gbps=2 * n * 4 / dt / 1e9, ok=ok)
    remote.teardown()
    # raw pipeline without the API layer, by chunk size
    for kind, (xh, yh) in kinds.items():
        for cb in (1 << 20, 2 << 20, 4 << 20, 8 << 20, 16 << 20):
            for _ in range(2):
                ops.map_host(xh, "scale", 2.0, out_host=yh, devices=devs, chunk_bytes=cb)
            t0 = time.perf_counter()
            for _ in range(8):
                ops.map_host(xh, "scale", 2.0, out_host=yh, devices=devs, chunk_bytes=cb)
            dt = (time.perf_counter() - t0) / 8
            emit(what="map_host_raw", kind=kind, n_gpus=n_gpus, chunk_bytes=cb, ms=dt * 1e3, gbps=2 * n * 4 / dt / 1e9,
                 ok=bool(torch.equal(yh[-4096:], xh[-4096:] * 2)))


if __name__ == "__main__":
    main()
