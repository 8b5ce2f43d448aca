"""Generalized advantage estimation without a GPU: the header's fp32 restatement equals the body of
tests/policy_gae_cases.py bit for bit; λ = 0 and λ = 1 give the one-step TD errors and the discounted returns less V;
a NaN crosses an episode boundary as the body's products make it; the body gives the same bits on any number of
ranks; kt.mapped("gae") takes gamma=, lam= and self_check= only; the ctypes prototype matches the header; and the
kernel's SASS has no FFMA and no local-memory traffic."""
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
from policy_gae_cases import GAMMA, LAM, gae, header_gae, mapped_gae, mapped_gae_args

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "ktb200.h")
PAIRS = [(0.99, 0.95), (0.0, 0.95), (1.0, 1.0), (0.99, 0.0), (0.997, 0.93)]
SPECIAL = [0.0, -0.0, 1.0, -1.5, 1e30, -1e30, 1e-40, math.inf, -math.inf, math.nan]


def same(got, want, what=""):
    """Bit equality of fp32 tensors or arrays, any NaN equal to any NaN."""
    got, want = (torch.as_tensor(np.asarray(x, dtype=np.float32)) for x in (got, want))
    assert got.shape == want.shape, what
    nan = want.isnan()
    assert torch.equal(got.isnan(), nan), what
    assert torch.equal(got[~nan].view(torch.int32), want[~nan].view(torch.int32)), what


def rollouts(n, t, seed=0, special=True, done_values=(0.0, 1.0, 0.5, math.nan)):
    """Seeded env-major (rewards, values, dones, last_values): normal values with special values sprinkled in, and
    dones drawn from done_values (mostly 0)."""
    g = torch.Generator().manual_seed(seed)
    r, v = torch.randn(n, t, generator=g) * 2, torch.randn(n, t, generator=g) * 5
    lv = torch.randn(n, generator=g) * 5
    if special:
        s = torch.tensor(SPECIAL)
        for x in (r, v, lv):
            hit = torch.rand(x.shape, generator=g) < 0.03
            x[hit] = s[torch.randint(0, len(SPECIAL), (int(hit.sum()),), generator=g)]
    pick = torch.randint(0, len(done_values), (n, t), generator=g)
    d = torch.tensor(done_values)[pick] * (torch.rand(n, t, generator=g) < 0.3)
    d[torch.rand(n, t, generator=g) < 0.7] = 0.0
    if math.nan in done_values or any(x != x for x in done_values):
        d[0, 0] = math.nan   # NaN * (rand < 0.3) is NaN anyway; make sure one is there
    return r, v, d, lv


# ---- the header restatement -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("gamma,lam", PAIRS)
@pytest.mark.parametrize("t", [1, 2, 7, 33, 128])
def test_header_restatement_equals_the_body(t, gamma, lam):
    r, v, d, lv = rollouts(64, t, seed=t)
    adv, ret = gae(r, v, d, lv, gamma, lam)
    hadv, hret = header_gae(r, v, d, lv, gamma, lam)
    same(hadv, adv, (t, gamma, lam))
    same(hret, ret, (t, gamma, lam))


def test_every_special_value_meets_every_done():
    """Each of the special values as reward, value and bootstrap against each done flag, on one-step rows and behind a
    second step."""
    s = torch.tensor(SPECIAL)
    grid = torch.cartesian_prod(s, s, s, torch.tensor([0.0, 1.0, 0.5, math.nan]))
    r, v, lv, d = (grid[:, i].contiguous() for i in range(4))
    for gamma, lam in PAIRS:
        one = (r[:, None], v[:, None], d[:, None], lv)
        same(header_gae(*one, gamma, lam)[0], gae(*one, gamma, lam)[0])
        two = (torch.stack([r.flip(0), r], 1), torch.stack([v, v.flip(0)], 1), torch.stack([d.flip(0), d], 1), lv)
        for a, b in zip(header_gae(*two, gamma, lam), gae(*two, gamma, lam)):
            same(a, b, (gamma, lam))


def test_lambda_zero_gives_the_one_step_td_errors():
    """λ = 0: adv = δ wherever it is finite.  A non-finite advantage still reaches the steps before it, as 0 · inf."""
    r, v, d, lv = rollouts(64, 33, seed=3, special=False, done_values=(0.0, 1.0, 0.5))
    r[5, 20] = math.inf
    adv, _ = gae(r, v, d, lv, GAMMA, 0.0)
    nv = torch.cat([v[:, 1:], lv[:, None]], 1)
    delta = r + GAMMA * nv * (1.0 - d) - v
    finite = adv.isfinite()
    assert adv[5, :20].isnan().all() and adv[5, 20] == math.inf and int((~finite).sum()) == 21
    assert torch.equal(adv[finite], delta[finite])   # == treats -0 and +0 as equal: only the sign of zero may differ


def test_lambda_one_gives_the_discounted_return_less_v():
    """λ = 1: the advantages telescope to G_t − V_t with G_t = r_t + γ(1 − d_t)G_{t+1}, G_T = V(s_T), within a bound of
    the fp32 roundings derived in fp64 from the magnitudes each step adds."""
    r, v, d, lv = rollouts(64, 128, seed=4, special=False, done_values=(0.0, 1.0))
    adv, ret = gae(r, v, d, lv, GAMMA, 1.0)
    r64, v64, d64, lv64 = (x.double() for x in (r, v, d, lv))
    G, S = lv64.clone(), torch.zeros_like(lv64)
    want, bar = torch.empty_like(r64), torch.empty_like(r64)
    nv = lv64
    for t in reversed(range(r.shape[1])):
        nt = 1 - d64[:, t]
        G = r64[:, t] + GAMMA * nt * G
        S = r64[:, t].abs() + GAMMA * nt * nv.abs() + v64[:, t].abs() + GAMMA * nt * S
        want[:, t] = G - v64[:, t]
        bar[:, t] = 8 * (r.shape[1] - t + 1) * 2.0 ** -24 * S
        nv = v64[:, t]
    assert ((adv.double() - want).abs() <= bar).all()
    assert ((ret.double() - (want + v64)).abs() <= bar + v64.abs() * 2.0 ** -23).all()


def test_an_infinite_advantage_leaks_nan_across_a_done():
    """A done multiplies by 1 − d = 0, it does not select: V = inf after the boundary makes every advantage before it
    NaN, in the body and in the header alike.  With finite values the boundary cuts the row."""
    r, v, d, lv = rollouts(4, 12, seed=5, special=False, done_values=(0.0,))
    d[:, 5] = 1.0
    v[0, 6] = math.inf
    adv, ret = gae(r, v, d, lv, GAMMA, LAM)
    same(header_gae(r, v, d, lv, GAMMA, LAM)[0], adv)
    assert adv[0, :6].isnan().all() and adv[0, 6] == -math.inf and adv[0, 7:].isfinite().all()
    cut, _ = gae(r[1:, :6], v[1:, :6], d[1:, :6], torch.zeros(3), GAMMA, LAM)
    same(adv[1:, :6], cut)


# ---- the body on any number of ranks ----------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_body_through_the_oracle_is_independent_of_the_rank_count(n):
    args = rollouts(37, 9, seed=6)
    with mock.patch.dict(os.environ, {"RANK": "0", "WORLD_SIZE": "1"}):
        want = mapped_gae(*args)
    got = ref_dispatch.spmd_call(mapped_gae, *args, num_proc=n, serialization="pickle")
    assert len(got) == n
    for k in range(2):
        same(torch.cat([g[k] for g in got]), want[k], (n, k))
    named = ref_dispatch.spmd_call(mapped_gae_args, *args, GAMMA, LAM, num_proc=n, serialization="pickle")
    for k in range(2):
        same(torch.cat([g[k] for g in named]), want[k], (n, k))


# ---- kt.mapped("gae") -------------------------------------------------------------------------------------------------
def _body(*params):
    ns = {}
    exec(f"def body({', '.join(params)}):\n    pass", ns)
    return ns["body"]


PARAMS = ("rewards", "values", "dones", "last_values", "g", "l")


def test_mapped_takes_constants_and_names():
    spec = kt.mapped("gae", gamma=0.99, lam=0.95)(_body(*PARAMS[:4])).__ktb_mapped__
    assert spec.op == "gae" and spec.extra == dict(gamma=0.99, lam=0.95)
    spec = kt.mapped("gae", gamma="g", lam="l")(_body(*PARAMS)).__ktb_mapped__
    assert spec.extra == dict(gamma="g", lam="l")
    spec = kt.mapped("gae", gamma=1, lam="l", self_check=False)(_body(*PARAMS)).__ktb_mapped__
    assert spec.extra == dict(gamma=1, lam="l", self_check=False)


REFUSED = dict(alpha=2.0, beta=0.0, reduce="sum", arg="values", bias=True, output="logits",
               **{k: "x" for k in MLP_FORMS if k not in ("gamma", "alpha")})


@pytest.mark.parametrize("option", sorted(REFUSED))
def test_mapped_refuses_every_other_option(option):
    with pytest.raises(ValueError, match=f"^{option}= is not an option of the 'gae' op"):
        kt.mapped("gae", gamma=0.99, lam=0.95, **{option: REFUSED[option]})


@pytest.mark.parametrize("kw,match", [
    (dict(lam=0.95), "gamma= is required"),
    (dict(gamma=0.99), "lam= is required"),
    (dict(gamma=math.nan, lam=0.95), "gamma must be a finite number"),
    (dict(gamma=0.99, lam=math.inf), "lam must be a finite number"),
    (dict(gamma=True, lam=0.95), "gamma must be a finite number"),
    (dict(gamma=0.99, lam=[0.95]), "lam must be a finite number"),
    (dict(gamma=0.99, lam=0.95, self_check=0), "self_check must be True or False"),
])
def test_mapped_refuses_missing_or_non_finite_parameters(kw, match):
    with pytest.raises(ValueError, match=match):
        kt.mapped("gae", **kw)


def test_mapped_refuses_a_name_that_is_not_an_argument_and_a_short_callable():
    with pytest.raises(ValueError, match="'gamma' is not an argument"):
        kt.mapped("gae", gamma="gamma", lam=0.95)(_body(*PARAMS))
    with pytest.raises(ValueError, match="takes \\(rewards, values, dones, last_values, ...\\)"):
        kt.mapped("gae", gamma=0.99, lam=0.95)(_body("rewards", "values", "dones"))


def test_existing_ops_keep_their_defaults():
    spec = kt.mapped("affine", alpha=2.0)(_body("x")).__ktb_mapped__
    assert (spec.alpha, spec.beta, spec.reduce) == (2.0, 0.0, None)
    with pytest.raises(ValueError, match="are options of the 'mlp' op"):
        kt.mapped("scale", alpha=2.0, gamma=0.99)


def test_wrapper_scalars_follow_torch():
    from kubetorch_b200.device.returns import gae_scalars

    for gamma, lam in PAIRS:
        g, gl = gae_scalars(gamma, lam)
        assert g == (torch.ones(1) * gamma).item() and gl == (torch.ones(1) * (gamma * lam)).item()
    with pytest.raises(ValueError, match="finite in float32"):
        gae_scalars(1e39, 0.5)
    with pytest.raises(ValueError, match="lam must be a finite number"):
        gae_scalars(0.99, math.nan)


# ---- the C ABI --------------------------------------------------------------------------------------------------------
def test_ctypes_prototype_matches_the_header():
    text = open(HEADER).read()
    m = re.search(r"\bint ktb_gae_f32\(([^)]*)\);", text)
    params = [p.strip() for p in m.group(1).split(",")]
    assert [p.split()[-1].lstrip("*") for p in params] == \
        ["dev", "rewards", "values", "dones", "last_values", "N", "T", "gamma", "gamma_lam", "adv", "ret", "stream"]
    restype, argtypes = L._SIGNATURES["ktb_gae_f32"]
    assert restype is ctypes.c_int and len(argtypes) == len(params)
    for p, t in zip(params, argtypes):
        want = ctypes.c_void_p if "*" in p else {"int": ctypes.c_int, "size_t": ctypes.c_size_t, "float": ctypes.c_float,
                                                  "uintptr_t": L.c_uintptr}[p.split()[0]]
        assert t is want, (p, t)


def test_kernel_sass_has_no_fma_and_no_local_memory():
    """The recurrence must round after every multiply (an FFMA would change the bits), and the tiles live in shared
    memory: no spill or local array."""
    sass = subprocess.run(["cuobjdump", "-sass", L.lib_path()], capture_output=True, text=True).stdout
    funcs = [f for f in sass.split("Function : ")[1:] if "gae_kernel" in f.split("\n", 1)[0]]
    assert len(funcs) == 1
    f = funcs[0]
    assert not re.search(r"\b(FFMA|STL|LDL)\b", f)
    assert "LDGSTS" in f and "FMUL" in f and "FADD" in f
