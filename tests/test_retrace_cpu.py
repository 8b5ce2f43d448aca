"""Retrace(λ) without a GPU: the header's fp32 restatement equals the body of tests/policy_retrace_cases.py bit for bit;
λ = 0 and cut traces give the one-step target, and on-policy Retrace at λ = 1 gives the n-step body's returns; columns 0
of log_rhos, q and values are never read; a NaN crosses an episode boundary as the body's products make it; the body
gives the same bits on any number of ranks; kt.mapped("retrace") takes its options and refuses every other; the ctypes
prototype matches the header; and every FFMA of the kernel's SASS belongs to an expf, with no local-memory traffic."""
import ctypes
import math
import os
import re
import subprocess
from unittest import mock

import numpy as np
import pytest
import torch

import kubetorch_b200 as kt
from kubetorch_b200.device import lib as L
from kubetorch_b200.mapped import MLP_FORMS
from oracle import ref_dispatch
from policy_nstep_cases import nstep
from policy_retrace_cases import GAMMA, LAM, header_retrace, mapped_retrace, mapped_retrace_args, retrace
from test_gae_cpu import same

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "ktb200.h")
# (gamma, lam): the usual pair, λ = 1 (uncut traces), λ = 0 (one-step targets), γ = 0, and γ = 1
OPTIONS = [(0.99, 0.95), (0.997, 1.0), (0.9, 0.0), (0.0, 0.5), (1.0, 0.9)]
SPECIAL = [0.0, -0.0, 1.0, -1.5, 1e30, -1e30, 1e-40, math.inf, -math.inf, math.nan]


def rollouts(n, t, seed=0, special=True, done_values=(0.0, 1.0, 0.5, math.nan)):
    """Seeded env-major (log_rhos, rewards, q, values, dones, baseline, bootstrap_value): log-ratios around 0 on both
    sides of the clip at ρ = 1, normal values with special values sprinkled into every input (log-ratios ±inf and NaN
    among them), and dones drawn from done_values (mostly 0)."""
    g = torch.Generator().manual_seed(seed)
    lr = torch.randn(n, t, generator=g)
    r, q = torch.randn(n, t, generator=g) * 2, torch.randn(n, t, generator=g) * 5
    v, b = torch.randn(n, t, generator=g) * 5, torch.randn(n, t, generator=g) * 5
    bv = torch.randn(n, generator=g) * 5
    if special:
        s = torch.tensor(SPECIAL)
        for x in (lr, r, q, v, b, bv):
            hit = torch.rand(x.shape, generator=g) < 0.03
            x[hit] = s[torch.randint(0, len(SPECIAL), (int(hit.sum()),), generator=g)]
    pick = torch.randint(0, len(done_values), (n, t), generator=g)
    d = torch.tensor(done_values)[pick] * (torch.rand(n, t, generator=g) < 0.3)
    d[torch.rand(n, t, generator=g) < 0.7] = 0.0
    if any(x != x for x in done_values):
        d[0, 0] = math.nan
    return lr, r, q, v, d, b, bv


# ---- the header restatement -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("opts", OPTIONS, ids=[str(o) for o in OPTIONS])
@pytest.mark.parametrize("t", [1, 2, 7, 33, 128])
def test_header_restatement_equals_the_body(t, opts):
    args = rollouts(64, t, seed=t)
    for a, b in zip(header_retrace(*args, *opts), retrace(*args, *opts)):
        same(a, b, (t, opts))


def test_every_special_value_meets_every_done():
    """Each special value as log-ratio, reward, q, value and bootstrap (−0 among them) against each done flag, on
    one-step rows (the first step's r + disc·bootstrap) and behind a second step (the general step)."""
    s = torch.tensor(SPECIAL)
    grid = torch.cartesian_prod(s, s, s, s, s, torch.tensor([0.0, 1.0, 0.5, math.nan]))
    lr, r, q, v, bv, d = (grid[:, i].contiguous() for i in range(6))
    b = r.flip(0).contiguous()
    for opts in OPTIONS:
        one = (lr[:, None], r[:, None], q[:, None], v[:, None], d[:, None], b[:, None], bv)
        for x, y in zip(header_retrace(*one, *opts), retrace(*one, *opts)):
            same(x, y, opts)
        two = (torch.stack([lr.flip(0), lr], 1), torch.stack([r.flip(0), r], 1), torch.stack([q.flip(0), q], 1),
               torch.stack([v.flip(0), v], 1), torch.stack([d.flip(0), d], 1), torch.stack([b, b.flip(0)], 1), bv)
        for x, y in zip(header_retrace(*two, *opts), retrace(*two, *opts)):
            same(x, y, opts)


def test_negative_zero_bootstrap_passes_the_first_step():
    """r = −0, bootstrap = −0: the body's first step is −0 + disc·−0 = −0, and the header's general step gives −0
    there because it starts from nq = nc = −0."""
    z = torch.full((2, 1), -0.0)
    args = (torch.zeros(2, 1), z, z, z, torch.zeros(2, 1), torch.zeros(2, 1), torch.full((2,), -0.0))
    ret, _ = retrace(*args, GAMMA, LAM)
    assert torch.signbit(ret).all()
    same(header_retrace(*args, GAMMA, LAM)[0], ret)


# ---- properties -------------------------------------------------------------------------------------------------------
def test_lambda_zero_is_the_one_step_target():
    """λ = 0: every trace is 0, so ret = r + (γ(1 − d))·v_next, bellman_target's order, bit for bit."""
    lr, r, q, v, d, b, bv = rollouts(64, 33, seed=3, special=False, done_values=(0.0, 1.0, 0.5))
    ret, td = retrace(lr, r, q, v, d, b, bv, GAMMA, 0.0)
    v_next = torch.cat([v[:, 1:], bv[:, None]], 1)
    want = r + (GAMMA * (1.0 - d)) * v_next
    same(ret, want)
    same(td, want - b)


def test_cut_traces_everywhere_are_lambda_zero():
    """log_rhos = −inf: ρ = 0 and c = 0 at every step, Watkins' cut at every step, the same bits as λ = 0."""
    lr, r, q, v, d, b, bv = rollouts(64, 33, seed=4, special=False, done_values=(0.0, 1.0, 0.5))
    cut = retrace(torch.full_like(lr, -math.inf), r, q, v, d, b, bv, GAMMA, LAM)
    for x, y in zip(cut, retrace(lr, r, q, v, d, b, bv, GAMMA, 0.0)):
        same(x, y)


@pytest.mark.parametrize("t", [1, 2, 7, 31, 32])
def test_on_policy_lambda_one_is_the_nstep_return(t):
    """log_rhos = 0, λ = 1 and values = q = baseline: c = 1, so (v − q) + g is +0 + g and Retrace is the discounted sum
    to the rollout's end, the n-step body at n = 32 ≥ T, bit for bit in both outputs."""
    lr, r, q, v, d, b, bv = rollouts(64, t, seed=5 + t, special=False, done_values=(0.0, 1.0))
    got = retrace(torch.zeros_like(lr), r, v, v, d, v, bv, GAMMA, 1.0)
    for x, y in zip(got, nstep(r, v, d, v, bv, 32, GAMMA)):
        same(x, y, t)


def test_columns_zero_of_log_rhos_q_and_values_are_never_read():
    args = list(rollouts(64, 33, seed=6))
    want = retrace(*args, GAMMA, LAM)
    g = torch.Generator().manual_seed(7)
    for i in (0, 2, 3):   # log_rhos, q, values
        other = [a.clone() for a in args]
        other[i][:, 0] = torch.randn(64, generator=g) * 100
        other[i][::4, 0] = math.nan
        for x, y, h in zip(retrace(*other, GAMMA, LAM), want, header_retrace(*other, GAMMA, LAM)):
            same(x, y, i)
            same(h, y, i)


def test_an_infinite_value_leaks_nan_across_a_done():
    """A done multiplies by 1 − d = 0, it does not select: values = inf after the boundary makes every target before it
    NaN, in the body and the header alike.  With finite values the boundary cuts the row."""
    lr, r, q, v, d, b, bv = rollouts(4, 12, seed=8, special=False, done_values=(0.0,))
    d[:, 5] = 1.0
    v[0, 6] = math.inf
    ret, td = retrace(lr, r, q, v, d, b, bv, GAMMA, LAM)
    for x, y in zip(header_retrace(lr, r, q, v, d, b, bv, GAMMA, LAM), (ret, td)):
        same(x, y)
    assert ret[0, :6].isnan().all() and ret[0, 6:].isfinite().all()
    cut = retrace(lr[1:, :6], r[1:, :6], q[1:, :6], v[1:, :6], d[1:, :6], b[1:, :6], torch.zeros(3), GAMMA, LAM)
    same(ret[1:, :6], cut[0])
    same(td[1:, :6], cut[1])


# ---- the body on any number of ranks ----------------------------------------------------------------------------------
@pytest.mark.parametrize("ranks", [1, 2, 3, 4])
def test_body_through_the_oracle_is_independent_of_the_rank_count(ranks):
    args = rollouts(37, 9, seed=9)
    with mock.patch.dict(os.environ, {"RANK": "0", "WORLD_SIZE": "1"}):
        want = mapped_retrace(*args)
    got = ref_dispatch.spmd_call(mapped_retrace, *args, num_proc=ranks, serialization="pickle")
    assert len(got) == ranks
    for k in range(2):
        same(torch.cat([g[k] for g in got]), want[k], (ranks, k))
    named = ref_dispatch.spmd_call(mapped_retrace_args, *args, GAMMA, LAM, num_proc=ranks, serialization="pickle")
    for k in range(2):
        same(torch.cat([g[k] for g in named]), want[k], (ranks, k))


# ---- kt.mapped("retrace") ---------------------------------------------------------------------------------------------
def _body(*params):
    ns = {}
    exec(f"def body({', '.join(params)}):\n    pass", ns)
    return ns["body"]


PARAMS = ("log_rhos", "rewards", "q", "values", "dones", "baseline", "bootstrap_value", "g", "l")


def test_mapped_takes_constants_and_names():
    spec = kt.mapped("retrace", gamma=0.99, lam=0.95)(_body(*PARAMS[:7])).__ktb_mapped__
    assert spec.op == "retrace" and spec.extra == dict(gamma=0.99, lam=0.95)
    spec = kt.mapped("retrace", gamma="g", lam="l", self_check=False)(_body(*PARAMS)).__ktb_mapped__
    assert spec.extra == dict(gamma="g", lam="l", self_check=False)
    assert kt.mapped("retrace", gamma=1, lam=0)(_body(*PARAMS[:7])).__ktb_mapped__.extra == dict(gamma=1, lam=0)


REFUSED = dict(alpha=2.0, beta=0.0, reduce="sum", arg="values", bias=True, output="logits", n=5, rho_bar=1.0,
               c_bar=1.0, pg_rho_bar=1.0, **{k: "x" for k in MLP_FORMS if k not in ("gamma", "alpha")})


@pytest.mark.parametrize("option", sorted(REFUSED))
def test_mapped_refuses_every_other_option(option):
    with pytest.raises(ValueError, match=f"^{option}= is not an option of the 'retrace' op, which takes gamma=, lam= "
                                         f"and self_check=: its callable is \\(log_rhos, rewards, q, values, dones, "
                                         f"baseline, bootstrap_value\\)"):
        kt.mapped("retrace", gamma=0.99, lam=0.95, **{option: REFUSED[option]})


@pytest.mark.parametrize("kw,match", [
    (dict(lam=0.95), "gamma= is required with the 'retrace' op"),
    (dict(gamma=0.99), "lam= is required with the 'retrace' op"),
    (dict(gamma=math.nan, lam=0.95), "gamma must be a finite number"),
    (dict(gamma=0.99, lam=math.inf), "lam must be a finite number"),
    (dict(gamma=True, lam=0.95), "gamma must be a finite number"),
    (dict(gamma=0.99, lam=None), "lam must be a finite number"),
    (dict(gamma=0.99, lam=0.95, self_check=0), "self_check must be True or False"),
])
def test_mapped_refuses_missing_or_bad_parameters(kw, match):
    with pytest.raises(ValueError, match=match):
        kt.mapped("retrace", **kw)


def test_mapped_refuses_a_name_that_is_not_an_argument_and_a_short_callable():
    with pytest.raises(ValueError, match="'gamma' is not an argument"):
        kt.mapped("retrace", gamma="gamma", lam="l")(_body(*PARAMS))
    with pytest.raises(ValueError, match="'lam' is not an argument"):
        kt.mapped("retrace", gamma=0.99, lam="lam")(_body(*PARAMS))
    with pytest.raises(ValueError, match="takes \\(log_rhos, rewards, q, values, dones, baseline, bootstrap_value, "
                                         "...\\) positionally"):
        kt.mapped("retrace", gamma=0.99, lam=0.95)(_body(*PARAMS[:6]))


def test_wrapper_scalars_follow_torch():
    from kubetorch_b200.device.returns import retrace_scalars

    for opts in OPTIONS + [(1 / 3, 0.7), (1, 0)]:
        assert retrace_scalars(*opts) == tuple((torch.ones(1) * x).item() for x in opts), opts
    with pytest.raises(ValueError, match="^gamma=1e\\+39 must be finite in float32"):
        retrace_scalars(1e39, 1e39)
    with pytest.raises(ValueError, match="^lam=-1e\\+39 must be finite in float32"):
        retrace_scalars(0.99, -1e39)
    with pytest.raises(ValueError, match="^gamma must be a finite number"):
        retrace_scalars(math.nan, math.nan)
    with pytest.raises(ValueError, match="^lam must be a finite number"):
        retrace_scalars(0.99, "0.95")


# ---- the C ABI --------------------------------------------------------------------------------------------------------
def test_ctypes_prototype_matches_the_header():
    text = open(HEADER).read()
    m = re.search(r"\bint ktb_retrace_f32\(([^)]*)\);", text)
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    assert [p.split()[-1].lstrip("*") for p in params] == \
        ["dev", "log_rhos", "rewards", "q", "values", "dones", "baseline", "bootstrap", "N", "T", "gamma", "lam", "ret",
         "td", "stream"]
    restype, argtypes = L._SIGNATURES["ktb_retrace_f32"]
    assert restype is ctypes.c_int and len(argtypes) == len(params)
    for p, t in zip(params, argtypes):
        want = ctypes.c_void_p if "*" in p else {"int": ctypes.c_int, "size_t": ctypes.c_size_t, "float": ctypes.c_float,
                                                  "uintptr_t": L.c_uintptr}[p.split()[0]]
        assert t is want, (p, t)


def _kernel_sass(name):
    sass = subprocess.run(["cuobjdump", "-sass", L.lib_path()], capture_output=True, text=True).stdout
    funcs = [f for f in sass.split("Function : ")[1:] if name in f.split("\n", 1)[0]]
    assert len(funcs) == 1
    return funcs[0]


def test_kernel_sass_has_fma_only_inside_expf_and_no_local_memory():
    """The recurrence rounds after every multiply; the only FFMAs are those of CUDA's expf, four per MUFU.EX2.  The
    tiles live in shared memory: no spill or local array."""
    f = _kernel_sass("retrace_kernel")
    ex2 = len(re.findall(r"\bMUFU\.EX2\b", f))
    assert ex2 > 0
    assert len(re.findall(r"\bFFMA(\.\w+)*\b", f)) == 4 * ex2
    assert not re.search(r"\b(STL|LDL)\b", f)
    assert "LDGSTS" in f


def test_header_restatement_is_fp32_throughout():
    out = header_retrace(*rollouts(3, 4, seed=10), GAMMA, LAM)
    assert all(isinstance(x, np.ndarray) and x.dtype == np.float32 for x in out)
