#!/usr/bin/env python
"""BASELINE config C4: RL rollout — 4096 env-state shards (512 x 256 bf16 each, 1 GiB) through the bf16 MLP
policy 256->1024->1024->64, scatter/gather across N GPUs via the public API (@kt.mapped("mlp")).
Device-resident obs on GPU 0; per call bytes = 1 GiB in + 256 MiB out; 5.77e12 flop."""
import json
import os
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402


def _clone(fn):
    """A copy of an oracle callable to decorate (the shared function object stays undecorated)."""
    import types

    return types.FunctionType(fn.__code__, fn.__globals__, fn.__name__, fn.__defaults__, fn.__closure__)

import kubetorch_b200 as kt  # noqa: E402
from oracle import cases  # noqa: E402


def main():
    n_gpus = int(sys.argv[1]) if len(sys.argv) > 1 else torch.cuda.device_count()
    transfer = sys.argv[2] if len(sys.argv) > 2 else "auto"          # auto | pull | push
    shards, rows = 4096, 512
    M = shards * rows
    g = torch.Generator(device="cuda:0").manual_seed(0)
    obs = torch.randn(M, 256, device="cuda:0", generator=g).bfloat16()
    w1 = (torch.randn(1024, 256, device="cuda:0", generator=g) * 0.02).bfloat16()
    w2 = (torch.randn(1024, 1024, device="cuda:0", generator=g) * 0.02).bfloat16()
    w3 = (torch.randn(64, 1024, device="cuda:0", generator=g) * 0.02).bfloat16()
    policy = kt.mapped("mlp")(_clone(cases.mlp_policy))
    remote = kt.fn(policy, name="c4-policy").to(kt.Compute(gpus=n_gpus).distribute("b200", workers=1, num_proc=n_gpus, transfer=transfer))
    for _ in range(3):
        out = remote(obs, w1, w2, w3, serialization="pickle")
    torch.cuda.synchronize(0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    iters = 10
    e0.record()
    t_host0 = time.perf_counter()
    for _ in range(iters):
        out = remote(obs, w1, w2, w3, serialization="pickle")
    host_issue_ms = (time.perf_counter() - t_host0) / iters * 1e3   # time to ENQUEUE one call (no device sync)
    e1.record()
    for d in range(n_gpus):
        torch.cuda.synchronize(d)
    ms = e0.elapsed_time(e1) / iters
    assert len(out) == n_gpus and sum(o.shape[0] for o in out) == M
    # parity on sampled rows vs an fp32 evaluation (rtol 2^-7, atol 1e-2)
    logits = torch.cat(out)
    idx = torch.randint(0, M, (2048,), device="cuda:0")
    h = torch.relu(obs[idx].float() @ w1.float().t()).bfloat16()
    h = torch.relu(h.float() @ w2.float().t()).bfloat16()
    ref = (h.float() @ w3.float().t()).bfloat16()
    torch.testing.assert_close(logits[idx].float(), ref.float(), rtol=2**-7, atol=1e-2)
    flop = 2 * (256 * 1024 + 1024 * 1024 + 1024 * 64) * M
    nbytes = M * 256 * 2 + M * 64 * 2
    print(json.dumps({"what": "c4_rl_rollout", "n_gpus": n_gpus, "transfer": transfer, "ms_per_call": ms, "calls_per_sec": 1e3 / ms,
                      "arg_plus_result_gbps": nbytes / ms / 1e6, "tflops": flop / ms / 1e9, "parity": "ok (2048 rows)", "host_issue_ms_per_call": host_issue_ms,
                      "root_nvlink_gbps_each_way": (n_gpus - 1) / n_gpus * (M * 256 * 2) / ms / 1e6 if n_gpus > 1 else 0}),
          flush=True)
    remote.teardown()


if __name__ == "__main__":
    main()
