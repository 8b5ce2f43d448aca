"""Generalized advantage estimation on one GPU: ktb_gae_f32 against the per-step torch loop it replaces.

For each rollout shape (N environments, T steps), env-major fp32:
  kernel  the C entry on cuda:0, each launch between two CUDA events, queued behind a sleep kernel so that the host runs
          ahead and no launch gap is timed; median over --reps launches after --warmup.
  loop    the body of tests/policy_gae_cases.py (CleanRL's backward loop, about seven torch kernels per step) on the same
          GPU, timed with the host clock around the call and a device synchronise; median over --loop-reps calls.
Bytes are those the op must move, 20·N·T + 4·N (three inputs and two outputs of N·T fp32, and V(s_T)); GB/s is bytes
over the kernel time and the share is of NVIDIA's 3.35 TB/s H100 SXM data-sheet HBM3 bandwidth.  Each shape also checks
the kernel's bits against the loop's.  The card name and power limit are read in the same run.  Prints one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))

import torch  # noqa: E402

from kubetorch_b200.device import lib as L  # noqa: E402
from kubetorch_b200.device import ops, returns  # noqa: E402
from policy_gae_cases import GAMMA, LAM, gae  # noqa: E402

SHAPES = [(8, 2048), (64, 128), (1024, 128), (4096, 256), (16384, 128)]
HBM_BYTES_PER_S = 3.35e12


def _power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:  # noqa: BLE001
        return None


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--loop-reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gae.py measures on a GPU; none is visible")
    ops.ensure_init([0])
    lib = L.load()
    g, gl = returns.gae_scalars(GAMMA, LAM)
    result = {"what": "gae_f32", "device": torch.cuda.get_device_name(0), "power_limit_w": _power_limit_w(),
              "gamma": GAMMA, "lam": LAM, "reps": args.reps, "loop_reps": args.loop_reps, "shapes": []}
    for n, t in SHAPES:
        gen = torch.Generator().manual_seed(n * 131 + t)
        r, v = torch.randn(n, t, generator=gen), torch.randn(n, t, generator=gen)
        d = (torch.rand(n, t, generator=gen) < 0.02).float()
        lv = torch.randn(n, generator=gen)
        r, v, d, lv = (x.cuda() for x in (r, v, d, lv))
        adv, ret = torch.empty_like(r), torch.empty_like(r)
        stream = ops.current_stream_handle(0)
        ptrs = (r.data_ptr(), v.data_ptr(), d.data_ptr(), lv.data_ptr(), n, t, g, gl, adv.data_ptr(), ret.data_ptr(),
                stream)

        def launch():
            rc = lib.ktb_gae_f32(0, *ptrs)
            if rc:
                raise RuntimeError(L.last_error())

        for _ in range(args.warmup):
            launch()
        torch.cuda.synchronize()
        events = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                  for _ in range(args.reps)]
        torch.cuda._sleep(50_000_000)
        for e0, e1 in events:
            e0.record()
            launch()
            e1.record()
        torch.cuda.synchronize()
        kernel_ms = statistics.median(e0.elapsed_time(e1) for e0, e1 in events)

        want = gae(r, v, d, lv, GAMMA, LAM)   # warms the loop's kernels up, and the bits to check
        torch.cuda.synchronize()
        same = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip((adv, ret), want))
        loop = []
        for _ in range(args.loop_reps):
            t0 = time.perf_counter()
            gae(r, v, d, lv, GAMMA, LAM)
            torch.cuda.synchronize()
            loop.append((time.perf_counter() - t0) * 1e3)
        loop_ms = statistics.median(loop)
        nbytes = 20 * n * t + 4 * n
        result["shapes"].append({
            "N": n, "T": t, "bytes": nbytes, "kernel_us_median": round(kernel_ms * 1e3, 2),
            "kernel_us_min": round(min(e0.elapsed_time(e1) for e0, e1 in events) * 1e3, 2),
            "kernel_gb_per_s": round(nbytes / (kernel_ms * 1e-3) / 1e9, 1),
            "share_of_hbm_peak": round(nbytes / (kernel_ms * 1e-3) / HBM_BYTES_PER_S, 3),
            "torch_loop_ms_median": round(loop_ms, 3), "loop_over_kernel": round(loop_ms / kernel_ms, 1),
            "bits_equal_to_loop": same})
    print(json.dumps(result), flush=True)
    if not all(s["bits_equal_to_loop"] for s in result["shapes"]):
        raise SystemExit("the kernel's bits differ from the torch loop's")


if __name__ == "__main__":
    main()
