#!/usr/bin/env python
"""2-GPU NVLink sweep: a kernel on GPU 1 pulling from / pushing to GPU 0's memory (the per-rank
kernel of the fused scatter->exec->gather), by variant; plus the root-push broadcast.
Writes JSON lines to gpurun_out/sweep_peer.jsonl."""
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402

from kubetorch_b200.device import lib as L  # noqa: E402
from kubetorch_b200.device import ops  # noqa: E402

OUT = os.path.join(REPO, "gpurun_out", "sweep_peer.jsonl")
os.makedirs(os.path.dirname(OUT), exist_ok=True)
out_f = open(OUT, "a")


def emit(**kw):
    line = json.dumps(kw)
    print(line, flush=True)
    out_f.write(line + "\n")
    out_f.flush()


def timeit(fn, dev, iters=10, warm=2):
    with torch.cuda.device(dev):
        for _ in range(warm):
            fn()
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1) / iters


def main():
    assert torch.cuda.device_count() >= 2
    ops.ensure_init([0, 1])
    n = 1 << 25  # 128 MiB shard (half of C2 at N=2)
    nbytes = n * 4
    x0 = torch.randn(n, device="cuda:0")
    y0 = torch.empty_like(x0)
    x1 = torch.randn(n, device="cuda:1")
    y1 = torch.empty_like(x1)
    # torch / cudaMemcpyPeer reference
    ms = timeit(lambda: y1.copy_(x0), 1)
    emit(what="torch_peer_copy_0to1", ms=ms, gbps=nbytes / ms / 1e6)

    # copy-engine duplex reference: 0->1 and 1->0 at the same time (what the links give both ways at once)
    s0, s1 = torch.cuda.Stream(0), torch.cuda.Stream(1)

    def duplex():
        with torch.cuda.stream(s1):
            y1.copy_(x0, non_blocking=True)
        with torch.cuda.stream(s0):
            y0.copy_(x1, non_blocking=True)

    for _ in range(2):
        duplex()
    torch.cuda.synchronize(0); torch.cuda.synchronize(1)
    import time as _t
    t0 = _t.perf_counter()
    for _ in range(10):
        duplex()
    torch.cuda.synchronize(0); torch.cuda.synchronize(1)
    dt = (_t.perf_counter() - t0) / 10 * 1e3
    emit(what="torch_peer_copy_duplex", ms=dt, gbps_each_way=nbytes / dt / 1e6)

    modes = {"pull(0->1)": (x0, y1), "push(1->0)": (x1, y0), "pull+push(0->1->0)": (x0, y0), "local(1)": (x1, y1)}
    for mode, (src, dst) in modes.items():
        for variant, name in ((L.VARIANT_VEC, "vec"), (L.VARIANT_TMA, "tma")):
            try:
                ms = timeit(lambda: ops.map_tensor(src, "scale", 2.0, out=dst, variant=variant, device=1), 1)
                emit(what="peer_map", mode=mode, variant=name, ms=ms, gbps_each_way=nbytes / ms / 1e6)
            except Exception as e:  # noqa: BLE001
                emit(what="peer_map", mode=mode, variant=name, error=str(e)[:200])
    ok = torch.equal(y0.cpu(), x0.cpu() * 2)
    emit(what="peer_parity_last", ok=bool(ok))

    # fused call, both ranks (C2 at N=2): 256 MiB arg on GPU 0
    xr = torch.randn(1 << 26, device="cuda:0")
    yr = torch.empty_like(xr)
    for variant, name in ((L.VARIANT_VEC, "vec"), (L.VARIANT_TMA, "tma")):
        ms = timeit(lambda: ops.scatter_map_gather(xr, "scale", 2.0, devices=[0, 1], out_root=yr, variant=variant), 0)
        emit(what="scatter_map_gather_2gpu", variant=name, ms=ms, arg_plus_result_gbps=2 * xr.numel() * 4 / ms / 1e6,
             ok=bool(torch.equal(yr[-4096:].cpu(), xr[-4096:].cpu() * 2)))
    # broadcast root -> peer
    d1 = torch.empty(nbytes, dtype=torch.uint8, device="cuda:1")
    s0 = x0.view(torch.uint8)
    ms = timeit(lambda: ops.broadcast(s0, [d1]), 0)
    emit(what="broadcast_0to1", ms=ms, gbps=nbytes / ms / 1e6)
    # reduce over peer memory
    ms = timeit(lambda: ops.map_reduce_sum(x0, "identity", device=1), 1)
    emit(what="peer_reduce_pull", ms=ms, gbps=nbytes / ms / 1e6)


if __name__ == "__main__":
    main()
