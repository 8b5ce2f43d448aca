"""n-step bootstrapped returns without a GPU: the header's fp32 restatement equals the body of tests/policy_nstep_cases.py
bit for bit; n = 1 is the one-step target; n >= T with no done is GAE's λ = 1 return within an fp64-derived bar; a NaN
crosses an episode boundary as the body's products make it, and the padded end turns −0 into +0; the body gives the
same bits on any number of ranks; kt.mapped("nstep") takes its options and refuses every other; the ctypes prototype
matches the header; and the kernel's SASS has no FFMA and no local-memory traffic."""
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
from policy_gae_cases import gae
from policy_nstep_cases import GAMMA, N_STEP, header_nstep, mapped_nstep, mapped_nstep_args, nstep
from test_gae_cpu import same

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "ktb200.h")
TS = [1, 2, 7, 33, 128]
NS = [1, 2, 3, 5, 31, 32]
GAMMAS = [0.99, 0.9, 0.0, 1.0]
SPECIAL = [0.0, -0.0, 1.0, -1.5, 1e30, -1e30, 3e38, 1e-40, -1e-45, math.inf, -math.inf, math.nan]


def rollouts(n, t, seed=0, special=True, done_values=(0.0, 1.0, 0.5, math.nan)):
    """Seeded env-major (rewards, values, dones, baseline, last_values): normal values with special values sprinkled
    into every input, and dones drawn from done_values (mostly 0)."""
    g = torch.Generator().manual_seed(seed)
    r, v, b = torch.randn(n, t, generator=g) * 2, torch.randn(n, t, generator=g) * 5, torch.randn(n, t, generator=g)
    lv = torch.randn(n, generator=g) * 5
    if special:
        s = torch.tensor(SPECIAL)
        for x in (r, v, b, lv):
            hit = torch.rand(x.shape, generator=g) < 0.03
            x[hit] = s[torch.randint(0, len(SPECIAL), (int(hit.sum()),), generator=g)]
    pick = torch.randint(0, len(done_values), (n, t), generator=g)
    d = torch.tensor(done_values)[pick] * (torch.rand(n, t, generator=g) < 0.3)
    d[torch.rand(n, t, generator=g) < 0.7] = 0.0
    if any(x != x for x in done_values):
        d[0, 0] = math.nan
    return r, v, d, b, lv


# ---- the header restatement -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("gamma", GAMMAS)
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("t", TS)
def test_header_restatement_equals_the_body(t, n, gamma):
    args = rollouts(64, t, seed=100 * t + n)
    for a, b in zip(header_nstep(*args, n, gamma), nstep(*args, n, gamma)):
        same(a, b, (t, n, gamma))


@pytest.mark.parametrize("n", [1, 2, 3])
def test_every_special_value_meets_every_done(n):
    """Each special value as reward, value, baseline and V(s_T) against each done flag, on three-step rows: the windows
    of n = 1, 2 and 3 then reach the bootstrap value, the padding and both."""
    s = torch.tensor(SPECIAL)
    grid = torch.cartesian_prod(s, s, s, s, torch.tensor([0.0, 1.0, 0.5, math.nan]))
    r, v, b, lv, d = (grid[:, i].contiguous() for i in range(5))
    three = (torch.stack([r, r.flip(0), r], 1), torch.stack([v.flip(0), v, v], 1), torch.stack([d, d.flip(0), d], 1),
             torch.stack([b, b, b.flip(0)], 1), lv)
    for a, w in zip(header_nstep(*three, n, GAMMA), nstep(*three, n, GAMMA)):
        same(a, w, n)


# ---- properties -------------------------------------------------------------------------------------------------------
def test_one_step_is_the_one_step_target():
    """n = 1: r + (γ(1 − d))·v_next, as the DQN target's expression, bit for bit; td = that − baseline."""
    r, v, d, b, lv = rollouts(64, 33, seed=3)
    ret, td = nstep(r, v, d, b, lv, 1, GAMMA)
    v_next = torch.cat([v[:, 1:], lv[:, None]], 1)
    want = r + (GAMMA * (1.0 - d)) * v_next
    same(ret, want)
    same(td, want - b)


@pytest.mark.parametrize("n,t", [(5, 5), (32, 7), (32, 32), (31, 2)])
def test_n_at_least_t_without_dones_is_the_gae_lambda_one_return(n, t):
    """n >= T and no done: every return is the discounted sum to the rollout's end bootstrapped from V(s_T), GAE's λ = 1
    return.  The two round in another order, so they agree within a bar derived from fp64: the fp64 return, and 4·(T +
    2)·2⁻²⁴ times the sum of the magnitudes of every term either computation adds."""
    r, v, d, b, lv = rollouts(256, t, seed=4, special=False, done_values=(0.0,))
    ret, _ = nstep(r, v, d, b, lv, n, GAMMA)
    _, gae_ret = gae(r, v, d, lv, GAMMA, 1.0)
    g = float(torch.tensor(GAMMA, dtype=torch.float32))
    r64, v64, lv64 = r.double(), v.double(), lv.double()
    want = torch.empty_like(r64)
    mag = torch.empty_like(r64)
    acc, size = lv64.clone(), lv64.abs()
    for k in reversed(range(t)):
        acc = r64[:, k] + g * acc
        size = r64[:, k].abs() + g * size + 2 * v64[:, k].abs()
        want[:, k], mag[:, k] = acc, size
    bar = 4 * (t + 2) * 2.0 ** -24 * mag
    for got in (ret, gae_ret):
        assert ((got.double() - want).abs() <= bar).all()
    assert not torch.equal(ret, gae_ret)   # the bits differ: another order of operations


def test_an_infinite_value_leaks_nan_across_a_done():
    """A done multiplies by 1 − d = 0, it does not select: V = inf right after the boundary makes the return whose
    window ends there NaN, in the body and the header alike.  With finite values the boundary cuts the row."""
    r, v, d, b, lv = rollouts(4, 12, seed=5, special=False, done_values=(0.0,))
    d[:, 5] = 1.0
    v[0, 6] = math.inf
    ret, td = nstep(r, v, d, b, lv, 3, GAMMA)
    for a, w in zip(header_nstep(r, v, d, b, lv, 3, GAMMA), (ret, td)):
        same(a, w)
    assert ret[0, 3].isnan() and ret[0, :3].isfinite().all() and ret[0, 4:].isfinite().all()
    v2 = v.clone()
    v2[1:, 6:] = torch.randn(3, 6)
    same(nstep(r, v2, d, b, lv, 3, GAMMA)[0][1:, :4], ret[1:, :4])


def test_the_padded_end_turns_negative_zero_into_positive_zero():
    """Past T the windows run 0 + 1·acc: with every reward, value and V(s_T) −0, n = 1 keeps −0 at the last step
    (−0 + γ·−0), and n >= 2 passes it through one padded step and returns +0, in the body and the header alike."""
    z = torch.full((3, 4), -0.0)
    lv, d = torch.full((3,), -0.0), torch.zeros(3, 4)
    for n in (1, 2, 5):
        ret, td = nstep(z, z, d, z, lv, n, GAMMA)
        for a, w in zip(header_nstep(z, z, d, z, lv, n, GAMMA), (ret, td)):
            same(a, w, n)
        sign = torch.signbit(ret[:, -1])
        assert sign.all() if n == 1 else not sign.any(), n


# ---- the body on any number of ranks ----------------------------------------------------------------------------------
@pytest.mark.parametrize("ranks", [1, 2, 3, 4])
def test_body_through_the_oracle_is_independent_of_the_rank_count(ranks):
    args = rollouts(37, 13, seed=6)
    with mock.patch.dict(os.environ, {"RANK": "0", "WORLD_SIZE": "1"}):
        want = mapped_nstep(*args)
    got = ref_dispatch.spmd_call(mapped_nstep, *args, num_proc=ranks, serialization="pickle")
    assert len(got) == ranks
    for k in range(2):
        same(torch.cat([g[k] for g in got]), want[k], (ranks, k))
    named = ref_dispatch.spmd_call(mapped_nstep_args, *args, GAMMA, num_proc=ranks, serialization="pickle")
    for k in range(2):
        same(torch.cat([g[k] for g in named]), want[k], (ranks, k))


# ---- kt.mapped("nstep") -----------------------------------------------------------------------------------------------
def _body(*params):
    ns = {}
    exec(f"def body({', '.join(params)}):\n    pass", ns)
    return ns["body"]


PARAMS = ("rewards", "values", "dones", "baseline", "last_values", "g")


def test_mapped_takes_constants_and_names():
    spec = kt.mapped("nstep", n=5, gamma=0.99)(_body(*PARAMS[:5])).__ktb_mapped__
    assert spec.op == "nstep" and spec.extra == dict(n=5, gamma=0.99)
    spec = kt.mapped("nstep", n=32, gamma="g", self_check=False)(_body(*PARAMS)).__ktb_mapped__
    assert spec.extra == dict(n=32, gamma="g", self_check=False)
    assert kt.mapped("nstep", n=1, gamma=1)(_body(*PARAMS[:5])).__ktb_mapped__.extra == dict(n=1, gamma=1)


REFUSED = dict(alpha=2.0, beta=0.0, reduce="sum", arg="values", bias=True, output="logits", lam=0.95, rho_bar=1.0,
               c_bar=1.0, pg_rho_bar=1.0, **{k: "x" for k in MLP_FORMS if k not in ("gamma", "alpha")})


@pytest.mark.parametrize("option", sorted(REFUSED))
def test_mapped_refuses_every_other_option(option):
    with pytest.raises(ValueError, match=f"^{option}= is not an option of the 'nstep' op, which takes n=, gamma= and "
                                         f"self_check="):
        kt.mapped("nstep", n=5, gamma=0.99, **{option: REFUSED[option]})


@pytest.mark.parametrize("kw,match", [
    (dict(gamma=0.99), "n= is required"),
    (dict(n=5), "gamma= is required"),
    (dict(n=5.0, gamma=0.99), "n must be an int constant in \\[1, 32\\]"),
    (dict(n=True, gamma=0.99), "n must be an int constant in \\[1, 32\\]"),
    (dict(n=0, gamma=0.99), "n must be an int constant in \\[1, 32\\]"),
    (dict(n=33, gamma=0.99), "n must be an int constant in \\[1, 32\\]"),
    (dict(n="n", gamma=0.99), "n must be an int constant in \\[1, 32\\] \\(not the name of a call argument\\)"),
    (dict(n=5, gamma=math.nan), "gamma must be a finite number"),
    (dict(n=5, gamma=True), "gamma must be a finite number"),
    (dict(n=5, gamma=0.99, self_check=0), "self_check must be True or False"),
])
def test_mapped_refuses_missing_or_bad_parameters(kw, match):
    with pytest.raises(ValueError, match=match):
        kt.mapped("nstep", **kw)


def test_mapped_refuses_a_name_that_is_not_an_argument_and_a_short_callable():
    with pytest.raises(ValueError, match="'gamma' is not an argument"):
        kt.mapped("nstep", n=5, gamma="gamma")(_body(*PARAMS))
    with pytest.raises(ValueError, match="takes \\(rewards, values, dones, baseline, last_values, ...\\)"):
        kt.mapped("nstep", n=5, gamma=0.99)(_body(*PARAMS[:4]))


@pytest.mark.parametrize("op,kw", [("gae", dict(gamma=0.99, lam=0.95)), ("vtrace", dict(gamma=0.99))])
def test_gae_and_vtrace_refuse_n(op, kw):
    with pytest.raises(ValueError, match=f"^n= is not an option of the '{op}' op"):
        kt.mapped(op, n=5, **kw)


def test_wrapper_scalars_follow_torch():
    from kubetorch_b200.device.returns import nstep_scalars

    for gamma in GAMMAS + [0.997, 1 / 3]:
        assert nstep_scalars(N_STEP, gamma) == (N_STEP, (torch.ones(1) * gamma).item())
    assert nstep_scalars(32, 1)[0] == 32
    for n in (0, 33, 5.0, True, "5", None):
        with pytest.raises(ValueError, match="^n must be an int in \\[1, 32\\]"):
            nstep_scalars(n, GAMMA)
    with pytest.raises(ValueError, match="gamma=1e\\+39 must be finite in float32"):
        nstep_scalars(5, 1e39)
    with pytest.raises(ValueError, match="gamma must be a finite number"):
        nstep_scalars(5, math.inf)


# ---- the C ABI --------------------------------------------------------------------------------------------------------
def test_ctypes_prototype_matches_the_header():
    text = open(HEADER).read()
    m = re.search(r"\bint ktb_nstep_f32\(([^)]*)\);", text)
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    assert [p.split()[-1].lstrip("*") for p in params] == \
        ["dev", "rewards", "values", "dones", "baseline", "last_values", "N", "T", "n", "gamma", "ret", "td", "stream"]
    restype, argtypes = L._SIGNATURES["ktb_nstep_f32"]
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


def test_kernel_sass_has_no_fma_and_no_local_memory():
    """Every multiply and add is rounded on its own (__fmul_rn / __fadd_rn): no FFMA.  The ring lives in shared memory:
    no spill or local array."""
    f = _kernel_sass("nstep_kernel")
    assert not re.search(r"\b(FFMA|STL|LDL)\b", f)
    assert "LDGSTS" in f and re.search(r"\bLDS\.64\b", f)


def test_header_restatement_is_fp32_throughout():
    out = header_nstep(*rollouts(3, 4, seed=7), 2, GAMMA)
    assert all(isinstance(x, np.ndarray) and x.dtype == np.float32 for x in out)
