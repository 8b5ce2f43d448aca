#!/usr/bin/env python
"""Kernel-level sweep on one H100: GB/s of each map variant, pack, reduce, host paths, and
calls/s for small payloads.  Writes JSON lines to gpurun_out/sweep.jsonl (copy summaries to profiles/)."""
import json
import os
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402

from kubetorch_b200.device import lib as L  # noqa: E402
from kubetorch_b200.device import ops  # noqa: E402

OUT = os.path.join(REPO, "gpurun_out", "sweep.jsonl")
os.makedirs(os.path.dirname(OUT), exist_ok=True)
out_f = open(OUT, "a")


def emit(**kw):
    line = json.dumps(kw)
    print(line, flush=True)
    out_f.write(line + "\n")
    out_f.flush()


def timeit(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters  # ms


def main():
    ops.ensure_init([0])
    n = 1 << 26
    x = torch.randn(n, device="cuda")
    y = torch.empty_like(x)
    nbytes = n * 4
    # torch copy reference (the MEASURED_PEAKS method)
    ms = timeit(lambda: y.copy_(x))
    emit(what="torch_copy_256MiB", ms=ms, gbps=2 * nbytes / ms / 1e6)
    ms = timeit(lambda: torch.mul(x, 2.0, out=y))
    emit(what="torch_mul_256MiB", ms=ms, gbps=2 * nbytes / ms / 1e6)

    for op in ("scale", "identity"):
        for variant, name in ((L.VARIANT_VEC, "map_vec"), (L.VARIANT_TMA, "map_tma")):
            ms = timeit(lambda: ops.map_tensor(x, op, 2.0, out=y, variant=variant))
            emit(what=name, op=op, ms=ms, gbps=2 * nbytes / ms / 1e6)

    # size sweep (identity over bytes, config C5) with the default variant
    for k in range(10, 31, 2):
        nb = 1 << k
        a = torch.empty(nb, dtype=torch.uint8, device="cuda")
        b = torch.empty_like(a)
        it = 200 if k <= 20 else 20
        ms = timeit(lambda: ops.map_tensor(a, "identity", out=b), iters=it)
        emit(what="identity_size", log2_bytes=k, ms=ms, gbps=2 * nb / ms / 1e6, calls_per_sec=1e3 / ms)
        del a, b

    # bf16 / int paths
    for dt in (torch.bfloat16, torch.int32, torch.int64):
        a = torch.ones(n, device="cuda").to(dt)
        b = torch.empty_like(a)
        ms = timeit(lambda: ops.map_tensor(a, "affine", 3, 1, out=b))
        emit(what="map_affine", dtype=str(dt), ms=ms, gbps=2 * a.numel() * a.element_size() / ms / 1e6)
        del a, b

    # reduce
    for cap in (1, 2, 4, 8):
        ops.set_tuning(6, cap)
        ms = timeit(lambda: ops.map_reduce_sum(x, "scale", 2.0))
        emit(what="reduce_sum_f32_256MiB", grid_cap=cap * 1024, ms=ms, gbps=nbytes / ms / 1e6)
    ops.set_tuning(6, 4)   # back to the library default

    # pack: 1024 tensors of 256 KiB, and 4096 of 4 KiB
    for cnt, sz in ((1024, 1 << 18), (4096, 1 << 12), (8, 1 << 25)):
        ts = [torch.empty(sz, dtype=torch.uint8, device="cuda") for _ in range(cnt)]
        plan = ops.PackPlan(ts)
        arena = plan.arena
        ms = timeit(lambda: plan.run(), iters=10)
        emit(what="pack_plan", count=cnt, seg_bytes=sz, ms=ms, gbps=2 * cnt * sz / ms / 1e6)
        ms = timeit(lambda: ops.pack(ts, arena=arena), iters=5)
        emit(what="pack_python_descs", count=cnt, seg_bytes=sz, ms=ms, gbps=2 * cnt * sz / ms / 1e6)
        cat_ms = timeit(lambda: torch.cat(ts), iters=10)
        emit(what="torch_cat", count=cnt, seg_bytes=sz, ms=cat_ms, gbps=2 * cnt * sz / cat_ms / 1e6)
        del ts, arena

    # batched small calls
    xs = [torch.randn(256, device="cuda") for _ in range(4096)]
    outs = [torch.empty_like(t) for t in xs]
    bplan = ops.BatchPlan(xs, outs, "scale", 2.0)
    ms = timeit(lambda: bplan.run(), iters=10)
    emit(what="map_batch_plan_4096x1KiB", ms=ms, calls_per_sec=4096 / ms * 1e3)
    # same calls, one launch each, captured in a CUDA graph
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for i in range(8):
            ops.map_tensor(xs[i], "scale", 2.0, out=outs[i])
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=s):
            for i in range(1024):
                ops.map_tensor(xs[i], "scale", 2.0, out=outs[i])
    ms = timeit(lambda: g.replay(), iters=10)
    emit(what="graph_1024_single_launches_1KiB", ms=ms, calls_per_sec=1024 / ms * 1e3)
    # python launch rate, no graph
    t0 = time.perf_counter()
    for i in range(4096):
        ops.map_tensor(xs[i], "scale", 2.0, out=outs[i])
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    emit(what="python_launch_loop_1KiB", calls_per_sec=4096 / dt)

    # host paths
    xh = torch.randn(n).pin_memory()
    yh = torch.empty_like(xh).pin_memory()
    ops.map_host(xh, "scale", 2.0, out_host=yh, chunk_bytes=8 << 20)  # warm-up (stage buffers, first touch)
    for chunk in (2 << 20, 4 << 20, 8 << 20, 16 << 20):
        ops.map_host(xh, "scale", 2.0, out_host=yh, chunk_bytes=chunk)
        t0 = time.perf_counter()
        for _ in range(3):
            ops.map_host(xh, "scale", 2.0, out_host=yh, chunk_bytes=chunk)
        dt = (time.perf_counter() - t0) / 3
        emit(what="map_host_pipelined", chunk_bytes=chunk, ms=dt * 1e3, gbps=2 * nbytes / dt / 1e9)
    st = torch.cuda.current_stream().cuda_stream
    for var in (L.VARIANT_VEC, L.VARIANT_TMA):
        try:
            def zc():
                L.call("ktb_map", 0, L.OP_SCALE, L.F32, xh.data_ptr(), yh.data_ptr(), n, 2.0, 0.0, var, st)
            ms = timeit(zc, iters=3, warm=1)
            emit(what="map_host_zero_copy", variant=var, ms=ms, gbps=2 * nbytes / ms / 1e6,
                 ok=bool(torch.equal(yh[:1000], xh[:1000] * 2)))
        except Exception as e:  # noqa: BLE001
            emit(what="map_host_zero_copy", variant=var, error=str(e)[:200])
    t0 = time.perf_counter()
    for _ in range(3):
        yh.copy_((xh.cuda(non_blocking=True) * 2), non_blocking=True)
        torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / 3
    emit(what="torch_h2d_mul_d2h_serial", ms=dt * 1e3, gbps=2 * nbytes / dt / 1e9)


if __name__ == "__main__":
    main()
