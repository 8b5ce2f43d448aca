#!/usr/bin/env python
"""Device-resident x->2x on N GPUs (single controller): push/push flag pipeline by chunk count vs the fused
pull+push kernel, by payload size.  JSON lines -> gpurun_out/sweep_push.jsonl"""
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402

from kubetorch_b200.device import ops  # noqa: E402

OUT = os.path.join(REPO, "gpurun_out", "sweep_push.jsonl")
os.makedirs(os.path.dirname(OUT), exist_ok=True)


def emit(**kw):
    line = json.dumps(kw)
    print(line, flush=True)
    with open(OUT, "a") as f:
        f.write(line + "\n")


def timeit(fn, devs, iters):
    for _ in range(3):
        fn()
    for d in devs:
        torch.cuda.synchronize(d)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    for d in devs:
        torch.cuda.synchronize(d)
    return e0.elapsed_time(e1) / iters


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else torch.cuda.device_count()
    devs = list(range(n))
    ops.ensure_init(devs)
    if "--one" in sys.argv:      # a few calls of the shipped configuration, for ncu
        elems = (256 << 20) // 4
        x = torch.randn(elems, device="cuda:0")
        y = torch.empty_like(x)
        sess = ops.PushSession(devs, ops.shard_bounds(elems, n, 0)[1] * 4)
        for _ in range(3):
            sess.call(x, y, "scale", 2.0)
        for d in devs:
            torch.cuda.synchronize(d)
        return
    for mib in (64, 256, 1024):
        elems = (mib << 20) // 4
        x = torch.randn(elems, device="cuda:0")
        y = torch.empty_like(x)
        iters = 20 if mib <= 256 else 8
        ms = timeit(lambda: ops.scatter_map_gather(x, "scale", 2.0, devices=devs, out_root=y), devs, iters)
        emit(what="c2_device", n_gpus=n, mib=mib, mode="pull_push_fused", ms=ms, gbps=2 * elems * 4 / ms / 1e6,
             ok=bool(torch.equal(y[-4096:].cpu(), x[-4096:].cpu() * 2)))
        for chunks in (16, 32):
            y.zero_()
            sess = ops.PushSession(devs, ops.shard_bounds(elems, n, 0)[1] * 4, n_chunks=chunks)
            ms = timeit(lambda: sess.call(x, y, "scale", 2.0), devs, iters)
            sess.check()
            idx = torch.randint(0, elems, (65536,), device="cuda:0")
            ok = bool(torch.equal(y[idx], x[idx] * 2)) and bool(torch.equal(y[-4096:], x[-4096:] * 2))
            emit(what="c2_device", n_gpus=n, mib=mib, mode="push_push_pipeline", chunks=chunks, ms=ms,
                 gbps=2 * elems * 4 / ms / 1e6, link_gbps_per_dir=(n - 1) / n * elems * 4 / ms / 1e6, ok=ok)
            del sess
        del x, y


if __name__ == "__main__":
    main()
