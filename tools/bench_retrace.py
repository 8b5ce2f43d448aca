"""Retrace(λ) on one GPU: ktb_retrace_f32 against the per-step torch loop it replaces, and ktb_gae_f32, ktb_vtrace_f32 and
ktb_nstep_f32 beside it.

For each rollout shape (N environments, T steps), env-major fp32:
  kernel  the C entry on cuda:0, each launch between two CUDA events, queued behind a sleep kernel so that the host runs
          ahead and no launch gap is timed; median over --reps launches after --warmup.
  loop    the body of tests/policy_retrace_cases.py (rlax's retrace_continuous, a few torch kernels per step) on the
          same GPU, timed with the host clock around the call and a device synchronise; median over --loop-reps calls
          (0 skips the arm).
  others  ktb_gae_f32, ktb_vtrace_f32 and ktb_nstep_f32 (n = 5) on the same rollouts, timed as the kernel.
Bytes are those the op must move, 32·N·T + 4·N for Retrace (six inputs and two outputs of N·T fp32, and the bootstrap
value), 20·N·T + 4·N for GAE and 24·N·T + 4·N for V-trace and n-step returns; GB/s is bytes over the kernel time and the
share is of NVIDIA's 3.35 TB/s H100 SXM data-sheet HBM3 bandwidth.  Each shape also checks the kernel's bits against
the loop's.  The card name and power limit are read in the same run.  Prints one JSON line.

--lib times the entries of another build of libktb200 (such as a parent commit's, or one built with another tile
layout) in place of the tree's; the entries a library lacks are skipped.  Alternate runs of the builds in one command to
compare them."""
import argparse
import ctypes
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
from kubetorch_b200.device import returns  # noqa: E402
from policy_retrace_cases import GAMMA, LAM, retrace  # noqa: E402

SHAPES = [(32, 80), (256, 80), (8, 2048), (1024, 128), (4096, 256), (16384, 128)]
N_STEP = 5
HBM_BYTES_PER_S = 3.35e12
ENTRIES = ("ktb_gae_f32", "ktb_vtrace_f32", "ktb_nstep_f32", "ktb_retrace_f32")


def _power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:  # noqa: BLE001
        return None


def _load(path):
    """The library at path with the prototypes of the entries timed here, cuda:0 registered with it."""
    lib = ctypes.CDLL(path, mode=ctypes.RTLD_LOCAL)
    for name in ("ktb_init", "ktb_last_error") + ENTRIES:
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = L._SIGNATURES[name]
    if lib.ktb_init(1, L.arr(ctypes.c_int, [0])) != L.OK:
        raise RuntimeError(lib.ktb_last_error())
    return lib


def _time(launch, reps, warmup):
    """(median, min) in ms of `launch()` between CUDA events."""
    for _ in range(warmup):
        launch()
    torch.cuda.synchronize()
    events = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    torch.cuda._sleep(50_000_000)
    for e0, e1 in events:
        e0.record()
        launch()
        e1.record()
    torch.cuda.synchronize()
    times = [e0.elapsed_time(e1) for e0, e1 in events]
    return statistics.median(times), min(times)


def _entry(lib, name, *args):
    fn = getattr(lib, name)

    def launch():
        if fn(0, *args):
            raise RuntimeError(f"{name}: {lib.ktb_last_error()}")

    return launch


def _row(nbytes, ms, ms_min):
    return {"bytes": nbytes, "kernel_us_median": round(ms * 1e3, 2), "kernel_us_min": round(ms_min * 1e3, 2),
            "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1),
            "share_of_hbm_peak": round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--loop-reps", type=int, default=5)
    ap.add_argument("--lib", default=L.lib_path(), help="the libktb200 build to time (default: the tree's)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_retrace.py measures on a GPU; none is visible")
    torch.cuda.init()
    lib = _load(args.lib)
    has = {name: hasattr(lib, name) for name in ENTRIES}
    gae_scalars = returns.gae_scalars(GAMMA, LAM)
    vtrace_scalars = returns.vtrace_scalars(GAMMA, LAM, 1.0, 1.0, 1.0)
    _, g = returns.nstep_scalars(N_STEP, GAMMA)
    retrace_scalars = returns.retrace_scalars(GAMMA, LAM)
    stream = torch.cuda.current_stream(0).cuda_stream
    result = {"what": "retrace_f32", "lib": os.path.relpath(os.path.abspath(args.lib), REPO),
              "device": torch.cuda.get_device_name(0), "power_limit_w": _power_limit_w(), "gamma": GAMMA, "lam": LAM,
              "nstep_n": N_STEP, "reps": args.reps, "loop_reps": args.loop_reps, "shapes": []}
    for N, T in SHAPES:
        gen = torch.Generator().manual_seed(N * 131 + T)
        lr = torch.randn(N, T, generator=gen) * 0.5   # ρ = e^(±0.5σ): both sides of the clip at 1
        r, q, v, b = (torch.randn(N, T, generator=gen) for _ in range(4))
        d = (torch.rand(N, T, generator=gen) < 0.02).float()
        bv = torch.randn(N, generator=gen)
        lr, r, q, v, d, b, bv = (x.cuda() for x in (lr, r, q, v, d, b, bv))
        out0, out1 = torch.empty_like(r), torch.empty_like(r)
        p = [x.data_ptr() for x in (lr, r, q, v, d, b, bv, out0, out1)]
        row = {"N": N, "T": T}
        if has["ktb_gae_f32"]:
            row["gae"] = _row(20 * N * T + 4 * N, *_time(
                _entry(lib, "ktb_gae_f32", p[1], p[3], p[4], p[6], N, T, *gae_scalars, p[7], p[8], stream),
                args.reps, args.warmup))
        if has["ktb_vtrace_f32"]:
            row["vtrace"] = _row(24 * N * T + 4 * N, *_time(
                _entry(lib, "ktb_vtrace_f32", p[0], p[1], p[3], p[4], p[6], N, T, *vtrace_scalars, p[7], p[8], stream),
                args.reps, args.warmup))
        if has["ktb_nstep_f32"]:
            row["nstep"] = _row(24 * N * T + 4 * N, *_time(
                _entry(lib, "ktb_nstep_f32", p[1], p[3], p[4], p[5], p[6], N, T, N_STEP, g, p[7], p[8], stream),
                args.reps, args.warmup))
        if has["ktb_retrace_f32"]:
            stats = _row(32 * N * T + 4 * N, *_time(
                _entry(lib, "ktb_retrace_f32", *p[:7], N, T, *retrace_scalars, p[7], p[8], stream),
                args.reps, args.warmup))
            want = retrace(lr, r, q, v, d, b, bv, GAMMA, LAM)   # warms the loop's kernels up, and the bits to check
            torch.cuda.synchronize()
            stats["bits_equal_to_loop"] = all(torch.equal(x.view(torch.int32), w.view(torch.int32))
                                              for x, w in zip((out0, out1), want))
            if args.loop_reps:
                loop = []
                for _ in range(args.loop_reps):
                    t0 = time.perf_counter()
                    retrace(lr, r, q, v, d, b, bv, GAMMA, LAM)
                    torch.cuda.synchronize()
                    loop.append((time.perf_counter() - t0) * 1e3)
                stats["torch_loop_ms_median"] = round(statistics.median(loop), 3)
                stats["loop_over_kernel"] = round(statistics.median(loop) * 1e3 / stats["kernel_us_median"], 1)
            row["retrace"] = stats
        result["shapes"].append(row)
    print(json.dumps(result), flush=True)
    if not all(s.get("retrace", {}).get("bits_equal_to_loop", True) for s in result["shapes"]):
        raise SystemExit("the kernel's bits differ from the torch loop's")


if __name__ == "__main__":
    main()
