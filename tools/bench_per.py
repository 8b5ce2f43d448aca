"""Prioritized replay on one GPU: ktb_per_sample_f32 and ktb_per_update_f32 against the torch bodies they replace.

For each (C, B) of DRAWS, fp32 priorities with 30 % zeros:
  kernel  the C entry on cuda:0 (tree pass, top pass when C > 2048, draw pass), each call between two CUDA events,
          queued behind a sleep kernel so that the host runs ahead and no launch gap of the host is timed; median over
          --reps calls after --warmup.
  torch   the body of tests/policy_per_cases.py (a torch sum tree, about 2·log2(C) small kernels) on the same GPU, timed
          with the host clock around the call and a device synchronise; median over --torch-reps calls.
For each B of UPDATES, random indices into C = 2^21 priorities, many repeated: ktb_per_update_f32 and the body's
per_update (whose boolean mask synchronises the host once), timed the same ways.
Bytes are the model of the byte traffic each op must move, kept here: a draw reads the C priorities and writes the P - 1
internal nodes (4·C + 4·P), reads back the block roots (at most 4·P / 2048) and writes 12 bytes per stratum; the descent's
loads (B·log2 P pairs) mostly hit L2 and are not counted.  An update reads 12 bytes per position and writes at most 4.
The share is that byte count over the kernel time, of NVIDIA's 3.35 TB/s H100 SXM data-sheet HBM3 bandwidth.  Each
shape also checks the kernel's bits against the body's.  The card name and power limit are read in the same run.
Prints one JSON line."""
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
from kubetorch_b200.device import ops, replay  # noqa: E402
from policy_per_cases import per_sample, per_update  # noqa: E402

DRAWS = [(1 << 16, 32), (1 << 20, 512), (1 << 21, 512), (1 << 24, 4096)]
UPDATES = [512, 8192]
UPDATE_C = 1 << 21
BETA, ALPHA, EPS = 0.4, 0.6, 1e-6
HBM_BYTES_PER_S = 3.35e12


def _power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:  # noqa: BLE001
        return None


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


def _host_time(fn, reps):
    """Median in ms of fn() between host clocks, each call ending in a device synchronise."""
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(out)


def _entry(name, *args):
    fn = getattr(L.load(), name)

    def launch():
        if fn(0, *args):
            raise RuntimeError(f"{name}: {L.last_error()}")

    return launch


def _row(nbytes, ms, ms_min, torch_ms):
    return {"bytes": nbytes, "kernel_us_median": round(ms * 1e3, 2), "kernel_us_min": round(ms_min * 1e3, 2),
            "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1),
            "share_of_hbm_bound": round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3),
            "torch_ms_median": round(torch_ms, 3), "torch_over_kernel": round(torch_ms * 1e3 / (ms * 1e3), 1)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--torch-reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_per.py measures on a GPU; none is visible")
    torch.cuda.init()
    ops.ensure_init([0])
    stream = torch.cuda.current_stream(0).cuda_stream
    b32, = replay.per_scalars(beta=BETA)
    a32, e32 = replay.per_scalars(alpha=ALPHA, eps=EPS)
    result = {"what": "per_f32", "device": torch.cuda.get_device_name(0), "power_limit_w": _power_limit_w(),
              "beta": BETA, "alpha": ALPHA, "reps": args.reps, "torch_reps": args.torch_reps, "draws": [],
              "updates": []}
    for c, batch in DRAWS:
        gen = torch.Generator().manual_seed(c + batch)
        prio = torch.rand(c, generator=gen)
        prio[torch.rand(c, generator=gen) < 0.3] = 0.0
        prio = prio.cuda()
        n = replay.tree_size(c)
        tree = torch.empty(n, device="cuda:0")
        idx = torch.empty(batch, dtype=torch.int64, device="cuda:0")
        w = torch.empty(batch, device="cuda:0")
        launch = _entry("ktb_per_sample_f32", prio.data_ptr(), c, batch, 0, batch, 12345, b32, tree.data_ptr(),
                        idx.data_ptr(), w.data_ptr(), stream)
        ms, ms_min = _time(launch, args.reps, args.warmup)
        torch_ms = _host_time(lambda: per_sample(prio, 12345, batch, BETA), args.torch_reps)
        want = per_sample(prio, 12345, batch, BETA)
        torch.cuda.synchronize()
        row = {"C": c, "B": batch, **_row(4 * c + 4 * n + 4 * (n // 2048) + 12 * batch, ms, ms_min, torch_ms)}
        row["bits_equal_to_torch"] = torch.equal(idx, want[0]) and torch.equal(w.view(torch.int32),
                                                                               want[1].view(torch.int32))
        result["draws"].append(row)
    for batch in UPDATES:
        gen = torch.Generator().manual_seed(batch)
        prio = torch.rand(UPDATE_C, generator=gen).cuda()
        indices = torch.randint(0, UPDATE_C // 64 if batch > 512 else UPDATE_C, (batch,), generator=gen).cuda()
        td = torch.randn(batch, generator=gen).cuda()
        mine, ref = prio.clone(), prio.clone()
        launch = _entry("ktb_per_update_f32", mine.data_ptr(), UPDATE_C, indices.data_ptr(), td.data_ptr(), batch, a32,
                        e32, stream)
        ms, ms_min = _time(launch, args.reps, args.warmup)
        torch_ms = _host_time(lambda: per_update(ref, indices, td, ALPHA, EPS), args.torch_reps)
        torch.cuda.synchronize()
        row = {"C": UPDATE_C, "B": batch, "distinct": int(indices.unique().numel()),
               **_row(16 * batch, ms, ms_min, torch_ms)}
        row["bits_equal_to_torch"] = torch.equal(mine.view(torch.int32), ref.view(torch.int32))
        result["updates"].append(row)
    print(json.dumps(result), flush=True)
    if not all(r["bits_equal_to_torch"] for r in result["draws"] + result["updates"]):
        raise SystemExit("the kernels' bits differ from the torch bodies'")


if __name__ == "__main__":
    main()
