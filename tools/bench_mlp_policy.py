#!/usr/bin/env python
"""The nn.Linear policy form of the bf16 MLP on one GPU, at the scale of BASELINE config C4: 4096 x 512 observation
rows through 256 -> 1024 -> 1024 -> d_out, device-resident on cuda:0.

Variants, timed alternately (one sample = the mean of --calls back-to-back calls between CUDA events; the median of
--samples samples is reported):
  a  the C entry ktb_mlp_bf16 (no bias, d_out 64, logits), called directly
  b  the C entry ktb_mlp_bf16_policy, no bias, d_out 64, logits (its logits must equal a's bit for bit)
  c  mlp_forward (ktb_mlp_bf16_policy) with biases, d_out 64, logits
  d  policy with biases, d_out 64, actions only
  e  policy with biases, d_out 64, logits and actions
  f  policy with biases, d_out 18 and d_out 256, logits and actions
  g  policy with biases, d_out 18, 64 and 256, sampled actions and log-probabilities (output="sample"), timed in the
     same alternation as d (actions only), which has the same GEMMs and no noise
  h  policy with biases, d_out 6, 18 and 64, Gaussian actions and log-probabilities (output="gaussian", log_std over
     [-2, 0.5]), timed in the same alternation beside the logits-only call and output="sample" at the same d_out
Parity: 2048 sampled rows against an fp32 evaluation (rtol 2^-7, atol 1e-2; actions wherever the fp32 top-2 gap
exceeds 2^-6), and the actions equal torch.argmax of the kernel's logits on every row.  Sampled rows: on 2048
consecutive rows, the action is the argmax of the kernel's logits plus the fp64 Gumbel noise wherever the top-2 gap
exceeds 2^-18·(1 + max|s|), and the log-probability is within (d_out + 8)·2^-22·(1 + |ref|) of the fp64 log_softmax.
Gaussian rows: on 2048 consecutive rows, the actions are within 2^-19·σ·(1 + |z|) + 2^-23·|y| of y + σ·z (y the
kernel's logits, σ and z = ndtri(u) in fp64) and the log-probabilities within the bar of tests/test_gpu_mlp_gaussian.py.
The card name and its power limit are read in the same run.  Prints one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402

from kubetorch_b200.device import lib as L  # noqa: E402
from kubetorch_b200.device import mlp  # noqa: E402
from kubetorch_b200.device import ops  # noqa: E402
from kubetorch_b200.sampling import gumbel_uniform  # noqa: E402

HALF_LOG_2PI = 0.9189385332046727

SEED = 0x5EED


def _power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:  # noqa: BLE001
        return None


def _fp32(obs, w, b):
    h = obs.float() @ w[0].float().t()
    h = torch.relu(h + b[0].float() if b[0] is not None else h).bfloat16()
    h2 = h.float() @ w[1].float().t()
    h = torch.relu(h2 + b[1].float() if b[1] is not None else h2).bfloat16()
    y = h.float() @ w[2].float().t()
    return y + b[2].float() if b[2] is not None else y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=7)
    ap.add_argument("--calls", type=int, default=3)
    args = ap.parse_args()
    L.load()
    ops.ensure_init([0])
    M, d_in, d_hidden = 4096 * 512, 256, 1024
    g = torch.Generator(device="cuda:0").manual_seed(0)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, device="cuda:0", generator=g) * scale).bfloat16()   # noqa: E731
    obs = rnd(M, d_in)
    w1, w2 = rnd(d_hidden, d_in, scale=0.02), rnd(d_hidden, d_hidden, scale=0.02)
    b1, b2 = rnd(d_hidden, scale=0.1), rnd(d_hidden, scale=0.1)
    heads = {d: (rnd(d, d_hidden, scale=0.02), rnd(d, scale=0.1)) for d in (18, 64, 256)}
    scratch = mlp._scratch_for(0, M, d_hidden)
    stream = int(torch.cuda.current_stream(0).cuda_stream)

    def original_a(out):
        L.call("ktb_mlp_bf16", 0, obs.data_ptr(), M, d_in, d_hidden, 64, w1.data_ptr(), w2.data_ptr(),
               heads[64][0].data_ptr(), out.data_ptr(), scratch.data_ptr(), stream)
        return out

    def policy_b(out):
        L.call("ktb_mlp_bf16_policy", 0, obs.data_ptr(), M, d_in, d_hidden, 64, w1.data_ptr(), 0, w2.data_ptr(), 0,
               heads[64][0].data_ptr(), 0, out.data_ptr(), 0, scratch.data_ptr(), 0, stream)
        return out

    out_a = torch.empty(M, 64, dtype=torch.bfloat16, device="cuda:0")
    out_b = torch.empty(M, 64, dtype=torch.bfloat16, device="cuda:0")
    variants = {
        "a_original_d64": (64, lambda: original_a(out_a)),
        "b_policy_nobias_d64": (64, lambda: policy_b(out_b)),
        "c_bias_logits_d64": (64, lambda: mlp.mlp_forward(obs, w1, w2, heads[64][0], biases=(b1, b2, heads[64][1]))),
        "d_bias_actions_d64": (64, lambda: mlp.mlp_forward(obs, w1, w2, heads[64][0], biases=(b1, b2, heads[64][1]),
                                                           output="actions")),
        "e_bias_both_d64": (64, lambda: mlp.mlp_forward(obs, w1, w2, heads[64][0], biases=(b1, b2, heads[64][1]),
                                                        output="both")),
        "f_bias_both_d18": (18, lambda: mlp.mlp_forward(obs, w1, w2, heads[18][0], biases=(b1, b2, heads[18][1]),
                                                        output="both")),
        "f_bias_both_d256": (256, lambda: mlp.mlp_forward(obs, w1, w2, heads[256][0], biases=(b1, b2, heads[256][1]),
                                                          output="both")),
    }
    for d in (18, 64, 256):
        variants[f"g_bias_sample_d{d}"] = (d, lambda d=d: mlp.mlp_forward(
            obs, w1, w2, heads[d][0], biases=(b1, b2, heads[d][1]), output="sample", seed=SEED))
    g6 = torch.Generator(device="cuda:0").manual_seed(6)   # its own generator: the other heads and rows stay as they were
    heads[6] = ((torch.randn(6, d_hidden, device="cuda:0", generator=g6) * 0.02).bfloat16(),
                (torch.randn(6, device="cuda:0", generator=g6) * 0.1).bfloat16())
    log_stds = {d: torch.linspace(-2.0, 0.5, d, device="cuda:0") for d in (6, 18, 64)}
    for d in (6, 18):
        variants[f"h_bias_logits_d{d}"] = (d, lambda d=d: mlp.mlp_forward(obs, w1, w2, heads[d][0],
                                                                          biases=(b1, b2, heads[d][1])))
    variants["h_bias_sample_d6"] = (6, lambda: mlp.mlp_forward(obs, w1, w2, heads[6][0], biases=(b1, b2, heads[6][1]),
                                                               output="sample", seed=SEED))
    for d in (6, 18, 64):
        variants[f"h_bias_gaussian_d{d}"] = (d, lambda d=d: mlp.mlp_forward(
            obs, w1, w2, heads[d][0], biases=(b1, b2, heads[d][1]), output="gaussian", seed=SEED,
            log_std=log_stds[d]))
    for _, fn in variants.values():   # warm-up: tensor maps, smem attributes, allocations
        fn()
        fn()
    torch.cuda.synchronize(0)
    samples = {k: [] for k in variants}
    for _ in range(args.samples):
        for name, (_, fn) in variants.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.calls):
                fn()
            e1.record()
            torch.cuda.synchronize(0)
            samples[name].append(e0.elapsed_time(e1) / args.calls)

    # parity
    a = variants["a_original_d64"][1]()
    b = variants["b_policy_nobias_d64"][1]()
    torch.cuda.synchronize(0)
    parity = {"b_equals_a_bitwise": bool(torch.equal(a, b))}
    idx = torch.randint(0, M, (2048,), device="cuda:0", generator=g)
    for name, d, bias in (("a_original_d64", 64, False), ("e_bias_both_d64", 64, True), ("f_bias_both_d18", 18, True),
                          ("f_bias_both_d256", 256, True)):
        res = variants[name][1]()
        logits, actions = res if isinstance(res, tuple) else (res, None)
        w = (w1, w2, heads[d][0])
        bs = (b1, b2, heads[d][1]) if bias else (None, None, None)
        ref = _fp32(obs[idx], w, bs)
        torch.testing.assert_close(logits[idx].float(), ref.bfloat16().float(), rtol=2**-7, atol=1e-2)
        entry = {"logits_2048_rows": "ok"}
        if actions is not None:
            assert torch.equal(actions, torch.argmax(logits, dim=-1))
            top2 = ref.topk(2, dim=1).values
            clear = (top2[:, 0] - top2[:, 1]) > 2**-6
            assert torch.equal(actions[idx][clear], ref.argmax(1)[clear])
            only = mlp.mlp_forward(obs, *w, biases=bs, output="actions")
            assert torch.equal(only, actions)
            entry.update({"actions_eq_argmax_all_rows": "ok", "actions_vs_fp32_clear_rows": int(clear.sum()),
                          "actions_only_eq_both": "ok"})
        parity[name] = entry
    assert parity["b_equals_a_bitwise"]
    r0 = M - 2048 - 77
    for d in (18, 64, 256):
        actions, log_probs = variants[f"g_bias_sample_d{d}"][1]()
        w, bs = (w1, w2, heads[d][0]), (b1, b2, heads[d][1])
        y = mlp.mlp_forward(obs[r0:r0 + 2048], *w, biases=bs).double()
        s64 = y - torch.log(-torch.log(gumbel_uniform(SEED, r0, 2048, d, device="cuda:0").double()))
        a = actions[r0:r0 + 2048]
        eps = 2.0 ** -18 * (1 + s64.abs().amax(1))
        top2 = s64.topk(2, dim=1).values
        clear = (top2[:, 0] - top2[:, 1]) > eps
        assert bool((s64.gather(1, a[:, None]).squeeze(1) >= top2[:, 0] - eps).all())
        assert torch.equal(a[clear], s64.argmax(1)[clear])
        ref = y.gather(1, a[:, None]).squeeze(1) - torch.logsumexp(y, -1)
        assert bool(((log_probs[r0:r0 + 2048].double() - ref).abs() <= (d + 8) * 2.0 ** -22 * (1 + ref.abs())).all())
        parity[f"g_bias_sample_d{d}"] = {"sample_bars_2048_rows": "ok", "clear_rows": int(clear.sum())}
    for d in (6, 18, 64):
        actions, log_probs = variants[f"h_bias_gaussian_d{d}"][1]()
        w, bs = (w1, w2, heads[d][0]), (b1, b2, heads[d][1])
        y = mlp.mlp_forward(obs[r0:r0 + 2048], *w, biases=bs).double()
        z = torch.special.ndtri(gumbel_uniform(SEED, r0, 2048, d, device="cuda:0", word3=1).double())
        ls = log_stds[d].double()
        sigma = ls.exp()
        err = (actions[r0:r0 + 2048].double() - (y + sigma * z)).abs()
        assert bool((err <= 2.0 ** -19 * sigma * (1 + z.abs()) + 2.0 ** -23 * y.abs()).all())
        t = 0.5 * z * z + ls
        ref = -t.sum(-1) - d * HALF_LOG_2PI
        tol = 2.0 ** -20 * ((1 + z.abs()) ** 2).sum(-1) + (d + 8) * 2.0 ** -23 * (t.abs().sum(-1) + d * 0.92)
        assert bool(((log_probs[r0:r0 + 2048].double() - ref).abs() <= tol).all())
        parity[f"h_bias_gaussian_d{d}"] = {"gaussian_bars_2048_rows": "ok"}

    result = {"what": "mlp_policy_c4_scale", "rows": M, "shape": f"{d_in}->{d_hidden}->{d_hidden}->d_out",
              "device": torch.cuda.get_device_name(0), "power_limit_w": _power_limit_w(),
              "samples": args.samples, "calls_per_sample": args.calls, "variants": {}, "parity": parity}
    for name, (d, _) in variants.items():
        ms = statistics.median(samples[name])
        flop = 2 * M * (d_in * d_hidden + d_hidden * d_hidden + d_hidden * d)
        result["variants"][name] = {"d_out": d, "ms_median": round(ms, 3), "ms_min": round(min(samples[name]), 3),
                                    "ms_max": round(max(samples[name]), 3), "tflops": round(flop / ms / 1e9, 1)}
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
