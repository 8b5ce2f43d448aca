"""V-trace on one GPU: ktb_vtrace_f32 against the per-step torch loop it replaces, and ktb_gae_f32 beside it.

For each rollout shape (N environments, T steps), env-major fp32:
  kernel  the C entry on cuda:0, each launch between two CUDA events, queued behind a sleep kernel so that the host runs
          ahead and no launch gap is timed; median over --reps launches after --warmup.
  loop    the body of tests/policy_vtrace_cases.py (TorchBeast's from_importance_weights, a few torch kernels per step)
          on the same GPU, timed with the host clock around the call and a device synchronise; median over --loop-reps
          calls (0 skips the arm).
  gae     ktb_gae_f32 on the same rewards, values and dones, timed as the kernel.
Bytes are those the op must move, 24·N·T + 4·N for V-trace (four inputs and two outputs of N·T fp32, and V(s_T)) and
20·N·T + 4·N for GAE; GB/s is bytes over the kernel time and the share is of NVIDIA's 3.35 TB/s H100 SXM data-sheet HBM3
bandwidth.  Each shape also checks the kernel's bits against the loop's.  The card name and power limit are read in the
same run.  Prints one JSON line.

--lib times the entries of another build of libktb200 (such as a parent commit's, or one built with another stage
count) in place of the tree's; a library without ktb_vtrace_f32 is timed on GAE only.  Alternate runs of the two builds
in one command to compare them."""
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
from policy_vtrace_cases import GAMMA, vtrace  # noqa: E402

SHAPES = [(32, 80), (256, 80), (8, 2048), (1024, 128), (4096, 256), (16384, 128)]
LAM = 1.0
HBM_BYTES_PER_S = 3.35e12


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
    for name in ("ktb_init", "ktb_last_error", "ktb_gae_f32", "ktb_vtrace_f32"):
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = L._SIGNATURES[name]
    if lib.ktb_init(1, L.arr(ctypes.c_int, [0])) != L.OK:
        raise RuntimeError(lib.ktb_last_error())
    return lib


def _time(entry, args, reps, warmup):
    def launch():
        if entry(0, *args):
            raise RuntimeError(entry.__name__)

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


def _rates(nbytes, ms):
    return {"gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1),
            "share_of_hbm_peak": round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--loop-reps", type=int, default=5)
    ap.add_argument("--lib", default=L.lib_path(), help="the libktb200 build to time (default: the tree's)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vtrace.py measures on a GPU; none is visible")
    torch.cuda.init()
    lib = _load(args.lib)
    has_vtrace = hasattr(lib, "ktb_vtrace_f32")
    scalars = returns.vtrace_scalars(GAMMA, LAM, 1.0, 1.0, 1.0)
    g, gl = returns.gae_scalars(GAMMA, LAM)
    stream = torch.cuda.current_stream(0).cuda_stream
    result = {"what": "vtrace_f32", "lib": os.path.relpath(os.path.abspath(args.lib), REPO),
              "device": torch.cuda.get_device_name(0), "power_limit_w": _power_limit_w(), "gamma": GAMMA, "lam": LAM,
              "rho_bar": 1.0, "c_bar": 1.0, "pg_rho_bar": 1.0, "reps": args.reps, "loop_reps": args.loop_reps,
              "shapes": []}
    for n, t in SHAPES:
        gen = torch.Generator().manual_seed(n * 131 + t)
        lr = torch.randn(n, t, generator=gen) * 0.5   # ρ = e^(±0.5σ): both sides of the thresholds
        r, v = torch.randn(n, t, generator=gen), torch.randn(n, t, generator=gen)
        d = (torch.rand(n, t, generator=gen) < 0.02).float()
        bv = torch.randn(n, generator=gen)
        lr, r, v, d, bv = (x.cuda() for x in (lr, r, v, d, bv))
        out0, out1 = torch.empty_like(r), torch.empty_like(r)
        row = {"N": n, "T": t}
        gae_bytes = 20 * n * t + 4 * n
        ms, ms_min = _time(lib.ktb_gae_f32, (r.data_ptr(), v.data_ptr(), d.data_ptr(), bv.data_ptr(), n, t, g, gl,
                                             out0.data_ptr(), out1.data_ptr(), stream), args.reps, args.warmup)
        row["gae"] = {"bytes": gae_bytes, "kernel_us_median": round(ms * 1e3, 2), "kernel_us_min": round(ms_min * 1e3, 2),
                      **_rates(gae_bytes, ms)}
        if has_vtrace:
            nbytes = 24 * n * t + 4 * n
            ms, ms_min = _time(lib.ktb_vtrace_f32, (lr.data_ptr(), r.data_ptr(), v.data_ptr(), d.data_ptr(),
                                                    bv.data_ptr(), n, t, *scalars, out0.data_ptr(), out1.data_ptr(),
                                                    stream), args.reps, args.warmup)
            row["vtrace"] = {"bytes": nbytes, "kernel_us_median": round(ms * 1e3, 2),
                             "kernel_us_min": round(ms_min * 1e3, 2), **_rates(nbytes, ms)}
            want = vtrace(lr, r, v, d, bv, GAMMA, LAM)   # warms the loop's kernels up, and the bits to check
            torch.cuda.synchronize()
            row["vtrace"]["bits_equal_to_loop"] = all(torch.equal(a.view(torch.int32), b.view(torch.int32))
                                                      for a, b in zip((out0, out1), want))
            if args.loop_reps:
                loop = []
                for _ in range(args.loop_reps):
                    t0 = time.perf_counter()
                    vtrace(lr, r, v, d, bv, GAMMA, LAM)
                    torch.cuda.synchronize()
                    loop.append((time.perf_counter() - t0) * 1e3)
                row["vtrace"]["torch_loop_ms_median"] = round(statistics.median(loop), 3)
                row["vtrace"]["loop_over_kernel"] = round(statistics.median(loop) / ms, 1)
        result["shapes"].append(row)
    print(json.dumps(result), flush=True)
    if not all(s.get("vtrace", {}).get("bits_equal_to_loop", True) for s in result["shapes"]):
        raise SystemExit("the kernel's bits differ from the torch loop's")


if __name__ == "__main__":
    main()
