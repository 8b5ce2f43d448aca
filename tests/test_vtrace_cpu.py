"""V-trace without a GPU: the header's fp32 restatement equals the body of tests/policy_vtrace_cases.py bit for bit;
λ = 0 gives one clipped TD error per step and on-policy V-trace gives GAE's λ = 1 returns; a NaN crosses an episode
boundary as the body's products make it; the body gives the same bits on any number of ranks; kt.mapped("vtrace") takes
its options and refuses every other; the ctypes prototype matches the header; and every FFMA of the kernel's SASS
belongs to an expf, with no local-memory traffic."""
import ctypes
import math
import os
import re
import subprocess
from unittest import mock

import pytest
import torch

import kubetorch_b200 as kt
from kubetorch_b200.device import lib as L
from kubetorch_b200.mapped import MLP_FORMS
from oracle import ref_dispatch
from policy_gae_cases import gae
from policy_vtrace_cases import GAMMA, header_vtrace, mapped_vtrace, mapped_vtrace_args, vtrace
from test_gae_cpu import same

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "ktb200.h")
# (gamma, lam, rho_bar, c_bar, pg_rho_bar): TorchBeast's defaults, λ < 1, unclipped, three different thresholds
OPTIONS = [(0.99, 1.0, 1.0, 1.0, 1.0), (0.99, 0.95, 1.0, 1.0, 1.0), (0.997, 1.0, None, None, None),
           (0.9, 0.9, 2.0, 0.8, 1.5), (0.0, 0.5, 0.5, None, 3.0)]
SPECIAL = [0.0, -0.0, 1.0, -1.5, 1e30, -1e30, 1e-40, math.inf, -math.inf, math.nan]


def rollouts(n, t, seed=0, special=True, done_values=(0.0, 1.0, 0.5, math.nan)):
    """Seeded env-major (log_rhos, rewards, values, dones, bootstrap_value): log-ratios around 0 on both sides of every
    threshold, normal values with special values sprinkled in (log-ratios ±inf and NaN among them), and dones drawn
    from done_values (mostly 0)."""
    g = torch.Generator().manual_seed(seed)
    lr = torch.randn(n, t, generator=g)
    r, v = torch.randn(n, t, generator=g) * 2, torch.randn(n, t, generator=g) * 5
    bv = torch.randn(n, generator=g) * 5
    if special:
        s = torch.tensor(SPECIAL)
        for x in (lr, r, v, bv):
            hit = torch.rand(x.shape, generator=g) < 0.03
            x[hit] = s[torch.randint(0, len(SPECIAL), (int(hit.sum()),), generator=g)]
    pick = torch.randint(0, len(done_values), (n, t), generator=g)
    d = torch.tensor(done_values)[pick] * (torch.rand(n, t, generator=g) < 0.3)
    d[torch.rand(n, t, generator=g) < 0.7] = 0.0
    if any(x != x for x in done_values):
        d[0, 0] = math.nan
    return lr, r, v, d, bv


# ---- the header restatement -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("opts", OPTIONS, ids=[str(o) for o in OPTIONS])
@pytest.mark.parametrize("t", [1, 2, 7, 33, 128])
def test_header_restatement_equals_the_body(t, opts):
    args = rollouts(64, t, seed=t)
    for a, b in zip(header_vtrace(*args, *opts), vtrace(*args, *opts)):
        same(a, b, (t, opts))


def test_every_special_value_meets_every_done():
    """Each special value as log-ratio, reward, value and bootstrap against each done flag, on one-step rows and behind
    a second step."""
    s = torch.tensor(SPECIAL)
    grid = torch.cartesian_prod(s, s, s, s, torch.tensor([0.0, 1.0, 0.5, math.nan]))
    lr, r, v, bv, d = (grid[:, i].contiguous() for i in range(5))
    for opts in OPTIONS:
        one = (lr[:, None], r[:, None], v[:, None], d[:, None], bv)
        for a, b in zip(header_vtrace(*one, *opts), vtrace(*one, *opts)):
            same(a, b, opts)
        two = (torch.stack([lr, lr.flip(0)], 1), torch.stack([r.flip(0), r], 1), torch.stack([v, v.flip(0)], 1),
               torch.stack([d.flip(0), d], 1), bv)
        for a, b in zip(header_vtrace(*two, *opts), vtrace(*two, *opts)):
            same(a, b, opts)


# ---- properties -------------------------------------------------------------------------------------------------------
def test_lambda_zero_gives_one_clipped_td_error_per_step():
    """λ = 0: vs = v + clip(ρ)·δ wherever it is finite."""
    lr, r, v, d, bv = rollouts(64, 33, seed=3, special=False, done_values=(0.0, 1.0, 0.5))
    vs, _ = vtrace(lr, r, v, d, bv, GAMMA, lam=0.0, rho_bar=1.2)
    nv = torch.cat([v[:, 1:], bv[:, None]], 1)
    want = torch.clamp(lr.exp(), max=1.2) * (r + GAMMA * (1.0 - d) * nv - v) + v
    finite = vs.isfinite()
    assert finite.all()
    assert torch.equal(vs, want)


def test_on_policy_vs_equals_the_gae_returns_at_lambda_one():
    """log_rhos = 0, ρ̄ = c̄ = 1, λ = 1, done ∈ {0, 1}: ρ = c = 1 and every product by them is exact, so vs is the
    λ = 1 return of GAE bit for bit (both compute r + disc·v' − v, then add (disc·1)·acc and v)."""
    lr, r, v, d, bv = rollouts(64, 128, seed=4, special=False, done_values=(0.0, 1.0))
    lr.zero_()
    vs, _ = vtrace(lr, r, v, d, bv, GAMMA)
    _, ret = gae(r, v, d, bv, GAMMA, 1.0)
    same(vs, ret)


def test_an_infinite_value_leaks_nan_across_a_done():
    """A done multiplies by 1 − d = 0, it does not select: V = inf after the boundary makes every target before it NaN,
    in the body and the header alike.  With finite values the boundary cuts the row."""
    lr, r, v, d, bv = rollouts(4, 12, seed=5, special=False, done_values=(0.0,))
    d[:, 5] = 1.0
    v[0, 6] = math.inf
    vs, pg = vtrace(lr, r, v, d, bv, GAMMA, 0.95)
    for a, b in zip(header_vtrace(lr, r, v, d, bv, GAMMA, 0.95), (vs, pg)):
        same(a, b)
    assert vs[0, :6].isnan().all() and vs[0, 7:].isfinite().all()
    cut = vtrace(lr[1:, :6], r[1:, :6], v[1:, :6], d[1:, :6], torch.zeros(3), GAMMA, 0.95)
    same(vs[1:, :6], cut[0])
    same(pg[1:, :6], cut[1])


# ---- the body on any number of ranks ----------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_body_through_the_oracle_is_independent_of_the_rank_count(n):
    args = rollouts(37, 9, seed=6)
    with mock.patch.dict(os.environ, {"RANK": "0", "WORLD_SIZE": "1"}):
        want = mapped_vtrace(*args)
    got = ref_dispatch.spmd_call(mapped_vtrace, *args, num_proc=n, serialization="pickle")
    assert len(got) == n
    for k in range(2):
        same(torch.cat([g[k] for g in got]), want[k], (n, k))
    named = ref_dispatch.spmd_call(mapped_vtrace_args, *args, GAMMA, 1.0, num_proc=n, serialization="pickle")
    for k in range(2):
        same(torch.cat([g[k] for g in named]), want[k], (n, k))


# ---- kt.mapped("vtrace") ----------------------------------------------------------------------------------------------
def _body(*params):
    ns = {}
    exec(f"def body({', '.join(params)}):\n    pass", ns)
    return ns["body"]


PARAMS = ("log_rhos", "rewards", "values", "dones", "bootstrap_value", "g", "l")
DEFAULTS = dict(lam=1.0, rho_bar=1.0, c_bar=1.0, pg_rho_bar=1.0)


def test_mapped_takes_constants_names_and_defaults():
    spec = kt.mapped("vtrace", gamma=0.99)(_body(*PARAMS[:5])).__ktb_mapped__
    assert spec.op == "vtrace" and spec.extra == dict(gamma=0.99, **DEFAULTS)
    spec = kt.mapped("vtrace", gamma="g", lam="l")(_body(*PARAMS)).__ktb_mapped__
    assert spec.extra == dict(DEFAULTS, gamma="g", lam="l")
    spec = kt.mapped("vtrace", gamma=1, lam=0.9, rho_bar=None, c_bar=0.5, pg_rho_bar=math.inf,
                     self_check=False)(_body(*PARAMS[:5])).__ktb_mapped__
    assert spec.extra == dict(gamma=1, lam=0.9, rho_bar=None, c_bar=0.5, pg_rho_bar=math.inf, self_check=False)


REFUSED = dict(alpha=2.0, beta=0.0, reduce="sum", arg="values", bias=True, output="logits",
               **{k: "x" for k in MLP_FORMS if k not in ("gamma", "alpha")})


@pytest.mark.parametrize("option", sorted(REFUSED))
def test_mapped_refuses_every_other_option(option):
    with pytest.raises(ValueError, match=f"^{option}= is not an option of the 'vtrace' op"):
        kt.mapped("vtrace", gamma=0.99, **{option: REFUSED[option]})


@pytest.mark.parametrize("kw,match", [
    (dict(lam=0.95), "gamma= is required"),
    (dict(gamma=math.nan), "gamma must be a finite number"),
    (dict(gamma=0.99, lam=math.inf), "lam must be a finite number"),
    (dict(gamma=True), "gamma must be a finite number"),
    (dict(gamma=0.99, rho_bar=0.0), "rho_bar must be a number > 0 or None"),
    (dict(gamma=0.99, c_bar=-1.0), "c_bar must be a number > 0 or None"),
    (dict(gamma=0.99, pg_rho_bar=math.nan), "pg_rho_bar must be a number > 0 or None"),
    (dict(gamma=0.99, rho_bar="rb"), "rho_bar must be a number > 0 or None"),
    (dict(gamma=0.99, c_bar=True), "c_bar must be a number > 0 or None"),
    (dict(gamma=0.99, self_check=0), "self_check must be True or False"),
])
def test_mapped_refuses_missing_or_bad_parameters(kw, match):
    with pytest.raises(ValueError, match=match):
        kt.mapped("vtrace", **kw)


def test_mapped_refuses_a_name_that_is_not_an_argument_and_a_short_callable():
    with pytest.raises(ValueError, match="'gamma' is not an argument"):
        kt.mapped("vtrace", gamma="gamma")(_body(*PARAMS))
    with pytest.raises(ValueError, match="takes \\(log_rhos, rewards, values, dones, bootstrap_value, ...\\)"):
        kt.mapped("vtrace", gamma=0.99)(_body(*PARAMS[:4]))


@pytest.mark.parametrize("option", ["rho_bar", "c_bar", "pg_rho_bar"])
def test_gae_refuses_the_thresholds(option):
    with pytest.raises(ValueError, match=f"^{option}= is not an option of the 'gae' op, which takes gamma=, lam= and "
                                         f"self_check="):
        kt.mapped("gae", gamma=0.99, lam=0.95, **{option: 1.0})


def test_wrapper_scalars_follow_torch():
    from kubetorch_b200.device.returns import vtrace_scalars

    for opts in OPTIONS:
        got = vtrace_scalars(*opts)
        want = [(torch.ones(1) * x).item() if x is not None else math.inf for x in opts]
        assert list(got) == want, opts
    with pytest.raises(ValueError, match="gamma=1e\\+39 must be finite in float32"):
        vtrace_scalars(1e39, 1.0, 1.0, 1.0, 1.0)
    with pytest.raises(ValueError, match="lam must be a finite number"):
        vtrace_scalars(0.99, math.nan, 1.0, 1.0, 1.0)
    with pytest.raises(ValueError, match="c_bar=1e-50 must be > 0 in float32"):
        vtrace_scalars(0.99, 1.0, 1.0, 1e-50, 1.0)
    with pytest.raises(ValueError, match="pg_rho_bar must be a number > 0 or None"):
        vtrace_scalars(0.99, 1.0, 1.0, 1.0, -2.0)
    assert vtrace_scalars(0.99, 1.0, 1e39, None, 1.0)[2:4] == (math.inf, math.inf)


# ---- the C ABI --------------------------------------------------------------------------------------------------------
def test_ctypes_prototype_matches_the_header():
    text = open(HEADER).read()
    m = re.search(r"\bint ktb_vtrace_f32\(([^)]*)\);", text)
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    assert [p.split()[-1].lstrip("*") for p in params] == \
        ["dev", "log_rhos", "rewards", "values", "dones", "bootstrap", "N", "T", "gamma", "lam", "rho_bar", "c_bar",
         "pg_rho_bar", "vs", "pg_adv", "stream"]
    restype, argtypes = L._SIGNATURES["ktb_vtrace_f32"]
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
    """The recurrence rounds after every multiply; the only FFMAs are those of CUDA's expf, four per MUFU.EX2 (two
    FFMA, FFMA.RM and FFMA.SAT around it).  The tiles live in shared memory: no spill or local array."""
    f = _kernel_sass("vtrace_kernel")
    ex2 = len(re.findall(r"\bMUFU\.EX2\b", f))
    assert ex2 > 0
    assert len(re.findall(r"\bFFMA(\.\w+)*\b", f)) == 4 * ex2
    assert not re.search(r"\b(STL|LDL)\b", f)
    assert "LDGSTS" in f


def test_gae_kernel_sass_still_has_no_fma():
    f = _kernel_sass("gae_kernel")
    assert not re.search(r"\b(FFMA|STL|LDL)\b", f)
    assert "LDGSTS" in f
