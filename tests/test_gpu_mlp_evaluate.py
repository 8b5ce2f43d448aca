"""-m gpu: evaluating given actions under the bf16 MLP policy heads (ktb_mlp_bf16_policy_evaluate*,
ktb_mlp_bf16_policy_gaussian_evaluate*, output="evaluate" / "gaussian_evaluate" of mlp_forward, mlp_scatter_gather and
kt.mapped) — the sampling entries' own actions give their log-probabilities bit for bit at every head width; arbitrary,
illegal and out-of-range actions and the entropy against fp64 of the kernel's own logits; groups tied to the masked
single categorical; the Gaussian head against fp64; every form, chunking and row split; guard bands; status codes; the
public API."""
import ctypes
import functools
import math

import pytest
import torch

from conftest import mapped_copy
from kubetorch_b200.device import lib as L
from kubetorch_b200.device import mlp
from mlp_rig import (SHIPPED_CHUNK, Guarded, Head, K, PushRig, config, deployed, entry_args,  # noqa: F401
                     expect_status, from_row, named_args, plain, pushed, randn, stream, tuning)

pytestmark = pytest.mark.gpu

import policy_evaluate_cases as cases  # noqa: E402
from oracle import ref_dispatch  # noqa: E402

WIDTHS = [1, 2, 3, 7, 63, 64, 65, 127, 128, 129, 255, 256]
MICRORTS = (6, 4, 4, 4, 4, 7, 49)
_OUT = {"log_probs": lambda d: 4, "entropy": lambda d: 4}
_OUT_V = dict(_OUT, values=lambda d: 4)


def _cat_head(masked, valued):
    name = "ktb_mlp_bf16_policy_evaluate" + ("_masked" if masked else "") + ("_value" if valued else "")

    def args(a):
        return (a.get("nvec"), a.get("n_groups", 0), *((a["mask"],) if masked else ()), a["taken"], a["log_probs"],
                a["entropy"], *((a["values"],) if valued else ()))
    return Head(name, name, name + "_pushed", True, 0, _OUT_V if valued else _OUT, args)


EV = {(m, v): _cat_head(m, v) for m in (False, True) for v in (False, True)}
GEV = {v: Head(n, n, n + "_pushed", True, 0, _OUT_V if v else _OUT,
               lambda a, v=v: (a["log_std"], a["taken"], a["log_probs"], a["entropy"], *((a["values"],) if v else ())))
       for v, n in ((False, "ktb_mlp_bf16_policy_gaussian_evaluate"),
                    (True, "ktb_mlp_bf16_policy_gaussian_evaluate_value"))}


# ---- helpers -----------------------------------------------------------------------------------------------------------
def random_legal(M, d_out, seed, p=0.6):
    g = torch.Generator(device="cuda").manual_seed(seed)
    legal = torch.rand(M, d_out, generator=g, device="cuda") < p
    legal[3] = False   # a row with no legal column
    return legal


def value_head(seed, biased=True):
    return randn((1, 1024), seed, 0.02), randn((1,), seed + 1, 0.1) if biased else None


def bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def same(got, want, what):
    for g, h in zip(got, want):
        if g.is_floating_point():
            g, h = bits(g), bits(h)
        assert torch.equal(g, h), what


def same_or_nan(got, want, what):
    """Equal bits, or NaN in both (a NaN's payload is not part of the contract)."""
    for g, h in zip(got, want):
        nan = g.isnan()
        assert torch.equal(nan, h.isnan()), what
        assert torch.equal(bits(g)[~nan], bits(h)[~nan]), what


def evaluate(obs, w, b, taken, legal=None, nvec=None, value=None, **kw):
    return mlp.mlp_forward(obs, *w, biases=b, output="evaluate", taken=taken, mask=legal, nvec=nvec, value=value, **kw)


def logits_of(obs, w, b, legal=None):
    """The kernel's own masked bf16 logits: every fp64 reference starts from them."""
    y = mlp.mlp_forward(obs, *w, biases=b, output="logits").float()
    return y if legal is None else y.masked_fill(~legal, float("-inf"))


def exact_terms(y, a):
    """fp64 (lp, H, Σ|w·(y − m)| / S, n) of actions a under the fp32 logits y of one group (rows with a legal column)."""
    y = y.double()
    m = y.amax(-1, keepdim=True)
    e = torch.exp(y - m)
    s = e.sum(-1)
    lp = y.gather(-1, a[:, None].clamp(0, y.shape[1] - 1))[:, 0] - m[:, 0] - s.log()
    p = e / s[:, None]
    ent = torch.special.entr(p).sum(-1)
    t_abs = torch.where(e > 0, e * (y - m).abs(), torch.zeros_like(e)).sum(-1) / s
    return lp, ent, t_abs, torch.isfinite(y).sum(-1).double()


# ---- 1. round trip: the sampling entries' own actions ------------------------------------------------------------------
@pytest.mark.parametrize("valued", [False, True], ids=["policy", "value"])
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("biased", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("d_out", WIDTHS)
def test_sampled_actions_give_the_samplers_log_probs_bit_for_bit(K, d_out, biased, masked, valued):
    """_sample, _masked, _value and _masked_value: evaluating the drawn actions returns the sampler's log_probs bit for
    bit (NaN in the same rows) and its values bit for bit; nvec = (d_out,) gives the bits of n_groups = 0."""
    if valued and d_out == 256:
        pytest.skip("a value head needs d_out <= 255")
    M, seed = 3000, 11 + d_out
    w, b = config(100 + d_out, d_out, bias=biased)
    obs = randn((M, 256), 101)
    legal = random_legal(M, d_out, 102) if masked else None
    value = value_head(103, biased) if valued else None
    drawn = mlp.mlp_forward(obs, *w, biases=b, output="sample", seed=seed, mask=legal, value=value)
    got = evaluate(obs, w, b, drawn[0], legal, value=value)
    same_or_nan([got[0]], [drawn[1]], "log_probs")
    assert not bool(got[0].isnan().all())
    if valued:
        same([got[2]], [drawn[2]], "values")
    one = evaluate(obs, w, b, drawn[0][:, None].contiguous(), legal, nvec=(d_out,), value=value)
    same_or_nan(one, got, "nvec=(d_out,)")


@pytest.mark.parametrize("valued", [False, True], ids=["policy", "value"])
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("nvec", [MICRORTS, (3, 5, 2), (1,) * 9, (100, 100, 55)], ids=["microrts", "3-5-2", "ones",
                                                                                    "wide"])
def test_multidiscrete_sampled_actions_give_the_samplers_log_probs(K, nvec, masked, valued):
    """The _multidiscrete sampling forms' actions give their log_probs (and values) bit for bit."""
    d_out, M, seed = sum(nvec), 3000, 5
    w, b = config(200 + d_out, d_out)
    obs = randn((M, 256), 201)
    legal = random_legal(M, d_out, 202) if masked else None
    value = value_head(203) if valued else None
    drawn = mlp.mlp_forward(obs, *w, biases=b, output="sample", seed=seed, mask=legal, nvec=nvec, value=value)
    got = evaluate(obs, w, b, drawn[0], legal, nvec=nvec, value=value)
    same_or_nan([got[0]], [drawn[1]], "log_probs")
    if valued:
        same([got[2]], [drawn[2]], "values")


# ---- 2, 3. arbitrary actions and the entropy against fp64 ------------------------------------------------------------------
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("d_out", [1, 3, 18, 64, 129, 256])
def test_arbitrary_actions_and_entropy_against_fp64(K, d_out, masked):
    """Uniform, illegal and out-of-range (−1, d_out) actions against fp64 of the kernel's own logits.  Bars (n the
    group's legal columns): each of the n ≤ 256 terms of S is within 2 ulp (expf) and their fp32 sum within n·2^-24
    relative, so logf(S) is within (n + 4)·2^-24 + 1 ulp of log S; lp = y_a − m − logf(S) adds 2 roundings of |lp|:
    |lp − ref| <= (n + 8)·2^-23 + 2^-23·|ref|.  T = Σ w·(y − m) has each term within 4 ulp and the sum within
    (n + 4)·2^-24 of Σ|w·(y − m)|, so |H − ref| <= (n + 8)·2^-23·(1 + Σ|w·(y − m)|/S) + 2^-23·|ref|.  Illegal actions
    give exactly −inf; out-of-range actions and rows with no legal column NaN in both outputs."""
    M = 4096
    w, b = config(300 + d_out, d_out)
    obs = randn((M, 256), 301)
    legal = random_legal(M, d_out, 302) if masked else None
    g = torch.Generator(device="cuda").manual_seed(303)
    a = torch.randint(0, d_out, (M,), generator=g, device="cuda")
    a[5::97], a[7::97] = -1, d_out
    got_lp, got_h = evaluate(obs, w, b, a, legal)
    y = logits_of(obs, w, b, legal)
    oob = (a < 0) | (a >= d_out)
    none = ~torch.isfinite(y).any(-1) if masked else torch.zeros(M, dtype=torch.bool, device="cuda")
    assert bool(got_lp[oob | none].isnan().all()) and bool(got_h[oob | none].isnan().all())
    ok = ~(oob | none)
    illegal = ok & ~legal.gather(1, a.clamp(0, d_out - 1)[:, None])[:, 0] if masked else torch.zeros_like(ok)
    assert bool((got_lp[illegal] == -math.inf).all()) and bool(torch.isfinite(got_h[illegal]).all())
    fin = ok & ~illegal
    lp, ent, t_abs, n = exact_terms(y[ok], a[ok])
    sel = fin[ok]
    tol_lp = (n + 8) * 2.0 ** -23 + 2.0 ** -23 * lp.abs()
    err = (got_lp[ok].double() - lp).abs()
    assert bool((err[sel] <= tol_lp[sel]).all()), float((err - tol_lp)[sel].max())
    tol_h = (n + 8) * 2.0 ** -23 * (1 + t_abs) + 2.0 ** -23 * ent.abs()
    err_h = (got_h[ok].double() - ent).abs()
    assert bool((err_h <= tol_h).all()), float((err_h - tol_h).max())


@pytest.mark.parametrize("d_out", [1, 7, 64, 200])
def test_exact_entropy_cases(K, d_out):
    """One legal column: lp == 0 and H == 0 exactly.  Equal logits over n legal columns (a zero head with a constant
    bias): H == logf(n) and lp == −logf(n)."""
    M = 512
    w, b = config(400 + d_out, d_out)
    w = (w[0], w[1], torch.zeros_like(w[2]))
    b = (b[0], b[1], torch.full((d_out,), 0.75, dtype=torch.bfloat16, device="cuda"))
    obs = randn((M, 256), 401)
    g = torch.Generator(device="cuda").manual_seed(402)
    n = torch.randint(1, d_out + 1, (M,), generator=g, device="cuda")
    n[:64] = 1
    perm = torch.rand(M, d_out, generator=g, device="cuda").argsort(-1)
    legal = perm < n[:, None]
    a = perm.argmin(-1)   # column of rank 0: always legal
    lp, h = evaluate(obs, w, b, a, legal)
    logn = torch.log(n.float())
    assert torch.equal(h, logn) and torch.equal(lp, -logn)
    assert bool((h[:64] == 0).all()) and bool((lp[:64] == 0).all())


# ---- 4. groups ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masked", [False, True], ids=["unmasked", "masked"])
@pytest.mark.parametrize("nvec", [MICRORTS, (3, 5, 2), (64, 65, 127)], ids=["microrts", "3-5-2", "wide"])
def test_each_group_is_the_single_categorical_under_its_mask(K, nvec, masked):
    """Group g's terms are, bit for bit, the single categorical's under legal ∧ (column in group g), and the row's
    outputs their fp32 sums in group order."""
    d_out, M = sum(nvec), 2048
    w, b = config(500 + d_out, d_out)
    obs = randn((M, 256), 501)
    legal = random_legal(M, d_out, 502) if masked else torch.ones(M, d_out, dtype=torch.bool, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(503)
    a = torch.stack([torch.randint(-1, n + 1, (M,), generator=g, device="cuda") for n in nvec], -1)
    got = evaluate(obs, w, b, a, legal if masked else None, nvec=nvec)
    lo, want = 0, None
    for k, n in enumerate(nvec):
        cols = torch.zeros(d_out, dtype=torch.bool, device="cuda")
        cols[lo:lo + n] = True
        ak = a[:, k]
        col = torch.where((ak >= 0) & (ak < n), ak + lo, torch.full_like(ak, -1))
        term = evaluate(obs, w, b, col, legal & cols)
        # the single categorical has d_out columns: an action in range there but outside the group is still out of range
        bad = (ak < 0) | (ak >= n)
        term = [torch.where(bad, torch.full_like(t, math.nan), t) for t in term]
        want = term if want is None else [x + y for x, y in zip(want, term)]
        lo += n
    same_or_nan(got, want, nvec)


# ---- 5. the Gaussian head ---------------------------------------------------------------------------------------------
def _gauss_bar(z, ls, a, sigma, d):
    """fp64 bound on the fp32 log-density: z is within 4 ulp (fsub, expf, fdiv), so 0.5·z² within 9 ulp, and the sum of
    the d terms 0.5·z² + ls within (d + 12)·2^-24·Σ(0.5·z² + |ls|), plus 2 ulp of the result."""
    return 2.0 ** -24 * ((d + 12) * (0.5 * z * z + ls.abs()).sum(-1) + 2 * d)


@pytest.mark.parametrize("d_out", [1, 6, 17, 64, 255, 256])
def test_gaussian_against_fp64(K, d_out):
    """lp against fp64 Normal(μ, σ).log_prob(a).sum(-1) of the kernel's own bf16 means, within _gauss_bar; entropy
    identical in every row and within (d + 4)·2^-24·Σ|ls + 1.42| of fp64."""
    M = 3000
    w, b = config(600 + d_out, d_out)
    obs = randn((M, 256), 601)
    g = torch.Generator(device="cuda").manual_seed(602)
    ls = torch.randn(d_out, generator=g, device="cuda") * 0.7
    a = torch.randn(M, d_out, generator=g, device="cuda") * 2
    lp, h = mlp.mlp_forward(obs, *w, biases=b, output="gaussian_evaluate", log_std=ls, taken=a)
    mu = mlp.mlp_forward(obs, *w, biases=b, output="logits").double()
    sigma = ls.double().exp()
    z = (a.double() - mu) / sigma
    want = (-0.5 * z * z - ls.double() - 0.5 * math.log(2 * math.pi)).sum(-1)
    err = (lp.double() - want).abs()
    tol = _gauss_bar(z, ls.double(), a, sigma, d_out) + 2.0 ** -23 * want.abs()
    assert bool((err <= tol).all()), float((err - tol).max())
    assert bool((h == h[0]).all())
    want_h = float((ls.double() + 0.5 + 0.5 * math.log(2 * math.pi)).sum())
    assert abs(float(h[0]) - want_h) <= (d_out + 4) * 2.0 ** -24 * float((ls.double().abs() + 1.42).sum())


@pytest.mark.parametrize("d_out", [1, 6, 17, 128, 255])
def test_gaussian_round_trip_and_values(K, d_out):
    """_gaussian's own actions give its log-probabilities within a bar conditioned on |a|/σ: the action's two roundings
    move the recomputed z by at most 2^-23·(|a| + σ|z|)/σ, and lp by |z| times that, plus twice _gauss_bar; the values
    equal _gaussian_value's bit for bit."""
    M, seed = 3000, 21
    w, b = config(650 + d_out, d_out)
    obs = randn((M, 256), 651)
    ls = torch.randn(d_out, generator=torch.Generator(device="cuda").manual_seed(652), device="cuda") * 0.7
    value = value_head(653)
    a, lp_s, v_s = mlp.mlp_forward(obs, *w, biases=b, output="gaussian", seed=seed, log_std=ls, value=value)
    lp, h, v = mlp.mlp_forward(obs, *w, biases=b, output="gaussian_evaluate", log_std=ls, taken=a, value=value)
    same([v], [v_s], "values")
    mu = mlp.mlp_forward(obs, *w, biases=b, output="logits").double()
    sigma = ls.double().exp()
    z = (a.double() - mu) / sigma
    tol = (z.abs() * 2.0 ** -23 * (a.double().abs() + sigma * z.abs()) / sigma).sum(-1) + \
        2 * _gauss_bar(z, ls.double(), a, sigma, d_out) + 2.0 ** -22 * lp_s.double().abs()
    err = (lp.double() - lp_s.double()).abs()
    assert bool((err <= tol).all()), float((err - tol).max())
    assert bool((h == h[0]).all())


# ---- 6. forms, chunkings and row splits ---------------------------------------------------------------------------------
def _fresh(M, valued):
    return {k: torch.full((M,), -1, dtype=torch.int32, device="cuda").view(torch.float32)
            for k in ("log_probs", "entropy") + (("values",) if valued else ())}


def _case(kind, M, d_out, seed):
    """(head, legal, taken, nvec, kwargs of mlp_forward, value) of one evaluating case over M fresh rows."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "gaussian":
        taken = torch.randn(M, d_out, generator=g, device="cuda")
        ls = torch.randn(d_out, generator=torch.Generator(device="cuda").manual_seed(1), device="cuda") * 0.5
        return GEV[True], None, taken, None, dict(output="gaussian_evaluate", log_std=ls), ls
    nvec = MICRORTS if kind == "microrts" else None
    legal = random_legal(M, d_out, seed + 1) if kind != "plain" else None
    hi = torch.tensor(nvec or (d_out,), device="cuda")
    taken = (torch.rand(M, len(hi), generator=g, device="cuda") * (hi + 1)).long() - int(kind == "masked")
    taken = taken if nvec else taken[:, 0].contiguous()
    return EV[(legal is not None, True)], legal, taken, nvec, dict(output="evaluate", mask=legal, nvec=nvec), None


@pytest.mark.parametrize("kind,d_out", [("plain", 18), ("masked", 129), ("microrts", 78), ("gaussian", 17)])
def test_every_form_chunking_and_row_split_gives_identical_bits(K, kind, d_out):
    """Repeat calls, chunk sizes 256 / 512 / shipped, plain and staged (pull kernel and copy engine), pushed through the
    rig on 3 ranks (three calls with fresh inputs), the package's pushed and pulled scatter on [0, 0, 0], and
    [0, s) + [s, M): the bits of one plain call; taken and the mask are unchanged."""
    w, b = config(700 + d_out, d_out)
    value = value_head(701)
    M = SHIPPED_CHUNK + 1000
    obs = randn((M, 256), 702)
    head, legal, taken, nvec, kw, ls = _case(kind, M, d_out, 703)
    keep = taken.clone()
    run = lambda o, t, m, **more: mlp.mlp_forward(o, *w, biases=b, taken=t, value=value, **dict(kw, mask=m), **more)  # noqa: E731
    want = run(obs, taken, legal)
    same(run(obs, taken, legal), want, "repeat")
    for chunk in (256, 512, SHIPPED_CHUNK):
        for ce in (None, 0, 1):
            with tuning(chunk, ce):
                same(run(obs, taken, legal, staged=ce is not None), want, (chunk, ce))
    for split in (1, 1000, 16896, 16900):
        parts = [run(obs[s], taken[s], None if legal is None else legal[s]) for s in (slice(0, split), slice(split, M))]
        same([torch.cat([x, y]) for x, y in zip(*parts)], want, split)
    assert torch.equal(taken, keep)
    Mp = 3 * 1408
    taken_row = taken[0].numel() * taken.element_size()
    masked = [("mask", d_out)] if legal is not None else []
    rig = PushRig(K, Mp, 256, 1024, 512, "ce", head, sides=masked + [("taken", taken_row)])
    w3v, b3v = mlp._stacked_head(w[2], b[2], *value)
    wv = (w[0], w[1], w3v)
    bv = (b[0], b[1], b3v)
    for it in range(3):
        obs_p = randn((Mp, 256), 710 + it)
        _, legal_p, taken_p, _, _, _ = _case(kind, Mp, d_out, 720 + it)
        want_p = run(obs_p, taken_p, legal_p)
        out = _fresh(Mp, True)
        groups = {} if nvec is None else dict(nvec=L.arr(ctypes.c_int32, nvec), n_groups=len(nvec))
        rig.call(obs_p, wv, bv, {k: t.data_ptr() for k, t in out.items()}, log_std=ls,
                 sides=dict(taken=taken_p, **({} if legal_p is None else dict(mask=legal_p))), d_out=d_out, **groups)
        torch.cuda.synchronize()
        same([out["log_probs"], out["entropy"], out["values"]], want_p, ("rig", it))
        devs = [0, 0, 0]
        bounds = [K.shard_bounds(Mp, 3, r) for r in range(3)]
        got = _fresh(Mp, True)
        mlp._mlp_scatter_gather_pushed(obs_p, devs, bounds, {0: (*wv, *bv)}, kw["output"], None, got["entropy"],
                                       got["log_probs"], None, None if ls is None else {0: ls}, legal_p,
                                       got["values"], nvec, None, None, taken_p)
        torch.cuda.synchronize()
        same([got["log_probs"], got["entropy"], got["values"]], want_p, ("package push", it))
        pull = mlp.mlp_scatter_gather(obs_p, *w, devices=devs, transfer="pull", biases=b, taken=taken_p, value=value,
                                      log_std=ls, mask=legal_p, output=kw["output"], nvec=nvec)
        torch.cuda.synchronize()
        same([torch.cat([g[k] for g in pull]) for k in range(3)], want_p, ("pull", it))
    assert rig.statuses() == [0] * rig.n
    mlp._push_sessions[(0, 0, 0)].check()


# ---- 7. guard bands ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form,M,chunk,d_out", [("plain", 1000, SHIPPED_CHUNK, 7), ("plain", 1000, 256, 129),
                                                ("staged", 1408, 256, 18), ("pushed", 3 * 1408, 256, 7)])
@pytest.mark.parametrize("kind", ["masked", "microrts", "gaussian"])
def test_writes_stay_inside_the_outputs(K, kind, form, M, chunk, d_out):
    """log_probs, entropy, values, the scratch and the stage between guard bands, offset 4 bytes into their 256-byte
    granule; taken in a guarded buffer is unchanged; the results equal mlp_forward's bit for bit."""
    d_out = 78 if kind == "microrts" else d_out
    w, b = config(900 + d_out, d_out)
    value = value_head(901)
    obs = randn((M, 256), 902)
    head, legal, taken, nvec, kw, ls = _case(kind, M, d_out, 903)
    want = mlp.mlp_forward(obs, *w, biases=b, taken=taken, value=value, **kw)
    gt = Guarded(taken.numel() * taken.element_size(), 8)
    gt.view(taken.dtype).copy_(taken.flatten())
    w3v, b3v = mlp._stacked_head(w[2], b[2], *value)
    wv, bv = (w[0], w[1], w3v), (b[0], b[1], b3v)
    bufs = {name: Guarded(M * 4, 4) for name in ("log_probs", "entropy", "values")}
    out = {name: buf.ptr() for name, buf in bufs.items()}
    groups = {} if nvec is None else dict(nvec=L.arr(ctypes.c_int32, nvec), n_groups=len(nvec))
    more = dict(d_out=d_out, log_std=ls, **groups)
    with tuning(chunk):
        if form == "pushed":
            masked = [("mask", d_out)] if legal is not None else []
            rig = PushRig(K, M, 256, 1024, 512, "ce", head,
                          sides=masked + [("taken", taken[0].numel() * taken.element_size())])
            sides = dict(taken=gt.view(taken.dtype), **({} if legal is None else dict(mask=legal)))
            for _ in range(3):
                rig.call(obs, wv, bv, out, sides=sides, **more)
            torch.cuda.synchronize()
            assert rig.statuses() == [0] * rig.n
            bufs.update({f"stage[{r}]": rig.stage[r] for r in range(1, rig.n)})
            bufs.update({f"scratch[{r}]": rig.scratch[r] for r in range(1, rig.n)})
        else:
            bufs["scratch"] = Guarded(L.load().ktb_mlp_scratch_bytes(M, 1024))
            if form == "staged":
                bufs["stage"] = Guarded(L.load().ktb_mlp_stage_bytes(M, 256))
            L.call(*entry_args(head, named_args(obs, wv, bv, out, mask=0 if legal is None else legal.data_ptr(),
                                                taken=gt.ptr(), scratch=bufs["scratch"].ptr(),
                                                stage=bufs["stage"].ptr() if form == "staged" else None, **more)))
    bufs["taken"] = gt
    for name, buf in bufs.items():
        buf.check(f"{kind} {form} M={M} chunk={chunk}: {name}")
    assert torch.equal(gt.view(taken.dtype), taken.flatten())
    same([bufs[k].view(torch.float32) for k in ("log_probs", "entropy", "values")], want, form)


# ---- 8. status codes ---------------------------------------------------------------------------------------------------
_Z = {}


def _z(name, n, dtype=torch.float32, fill=0):
    if name not in _Z:
        _Z[name] = torch.full((n,), fill, dtype=dtype, device="cuda")
    return _Z[name].data_ptr()


@functools.lru_cache(maxsize=None)
def _nvec9():
    return L.arr(ctypes.c_int32, [9, 9])


def _io(gaussian):
    return dict(taken=_z("taken_f" if gaussian else "taken", 2048 * 512, torch.float32 if gaussian else torch.int64),
                entropy=_z("entropy", 4096), values=_z("values", 4096), mask=_z("mask", 2048 * 512, torch.uint8, 1))


ROWS_BYTES = 256 * 256 * 2
MASK_END = ROWS_BYTES + 256 * 18
STATUS_CASES = {
    "null_taken": (plain, dict(taken=0), L.ERR_ARG),
    "null_log_probs": (plain, dict(log_probs=0), L.ERR_ARG),
    "null_entropy": (plain, dict(entropy=0), L.ERR_ARG),
    "unaligned_taken": (plain, dict(taken_off=2), L.ERR_ARG),
    "unaligned_log_probs": (plain, dict(log_probs_off=2), L.ERR_ARG),
    "unaligned_entropy": (plain, dict(entropy_off=1), L.ERR_ARG),
    "staged_null_taken": (plain, dict(taken=0, stage="zero"), L.ERR_ARG),
    "d_out_257": (plain, dict(d_out=257), L.ERR_UNSUPPORTED),
    "inherited_checks_first": (plain, dict(taken=0, entropy=0, d_out=257), L.ERR_UNSUPPORTED),
    "d_hidden_first": (plain, dict(taken=0, d_hidden=1000), L.ERR_ARG),
    "empty_call_takes_null_outputs": (plain, dict(M=0, taken=0, log_probs=0, entropy=0, values=0), None),
    "pushed_taken_over_the_rows": (pushed, dict(taken=ROWS_BYTES - 8), L.ERR_ARG),
    "pushed_taken_past_stage_stride": (pushed, dict(taken=(1 << 20) - 256 * 4), L.ERR_ARG),
    "pushed_taken_offset_past_stage_stride": (pushed, dict(taken=1 << 21), L.ERR_ARG),
    "pushed_taken_unaligned": (pushed, dict(taken=MASK_END + 258), L.ERR_ARG),
    "pushed_null_entropy": (pushed, dict(entropy=0), L.ERR_ARG),
    "pushed_d_out_257": (pushed, dict(d_out=257), L.ERR_UNSUPPORTED),
    "pushed_empty_shard_acks": (pushed, dict(M=0, taken=0, log_probs=0, entropy=0, values=0, nvec=None), None),
}
CATEGORICAL_ONLY = {
    "nvec_after_inherited": (plain, dict(nvec="9-9", n_groups=2, d_out=257), L.ERR_UNSUPPORTED),
    "nvec_sum": (plain, dict(nvec="9-9", n_groups=2, d_out=17), L.ERR_ARG),
    "nvec_null_with_groups": (plain, dict(nvec=None, n_groups=2), L.ERR_ARG),
    "nvec_before_taken": (plain, dict(nvec="9-9", n_groups=0, taken=0), L.ERR_ARG),
    "nvec_ok": (plain, dict(nvec="9-9", n_groups=2), None),
}
MASKED_ONLY = {
    "null_mask_first": (plain, dict(mask=0, taken=0), L.ERR_ARG),
    "pushed_taken_over_the_mask": (pushed, dict(mask=ROWS_BYTES, taken=ROWS_BYTES + 256), L.ERR_ARG),
    "pushed_taken_ends_in_the_mask": (pushed, dict(mask=ROWS_BYTES + 2040, taken=ROWS_BYTES), L.ERR_ARG),
    "pushed_mask_checks_first": (pushed, dict(mask=0, taken=0), L.ERR_ARG),
}
VALUE_ONLY = {
    "null_values": (plain, dict(values=0), L.ERR_ARG),
    "d_out_256_with_a_value_head": (plain, dict(d_out=256, taken=0), L.ERR_UNSUPPORTED),
}
GAUSSIAN_ONLY = {
    "null_log_std_first": (plain, dict(log_std=0, taken=0), L.ERR_ARG),
}
ALL_CASES = {**STATUS_CASES, **CATEGORICAL_ONLY, **MASKED_ONLY, **VALUE_ONLY, **GAUSSIAN_ONLY}
HEADS = {**{f"cat{'_masked' * m}{'_value' * v}": h for (m, v), h in EV.items()},
         **{f"gauss{'_value' * v}": h for v, h in GEV.items()}}


@pytest.mark.parametrize("head", list(HEADS))
@pytest.mark.parametrize("name", list(ALL_CASES))
def test_bad_arguments_get_the_documented_status(K, head, name):
    h = HEADS[head]
    gaussian = head.startswith("gauss")
    if (name in CATEGORICAL_ONLY and gaussian) or (name in MASKED_ONLY and "masked" not in head) or \
            (name in VALUE_ONLY and "value" not in head) or (name in GAUSSIAN_ONLY and not gaussian):
        pytest.skip("another entry's case")
    form, overrides, status = ALL_CASES[name]
    args = dict(_io(gaussian), nvec=None, n_groups=0)
    if form is pushed:
        args.update(mask=MASK_END - 256 * 18, taken=MASK_END + 256)
    args.update(overrides)
    if args.get("nvec") == "9-9":
        args["nvec"] = _nvec9()
    if args.get("stage") == "zero":
        args["stage"] = _z("stage", 1 << 24, torch.uint8)
    for key in [k for k in args if k.endswith("_off") and k[:-4] in ("taken", "entropy")]:
        args[key[:-4]] = _io(gaussian)[key[:-4]] + args.pop(key)
    call = form(h, **args)
    if status is None:
        L.call(*call)
        torch.cuda.synchronize()
    else:
        expect_status(call, status)


# ---- 9. the public API -------------------------------------------------------------------------------------------------
def _public_case():
    g = torch.Generator().manual_seed(93)
    nvec, M = (3, 5, 2, 8), 2 * 1408 + 100
    d_out = sum(nvec)
    p = [(torch.randn(1024, 256, generator=g) * 0.05).bfloat16(), (torch.randn(1024, generator=g) * 0.1).bfloat16(),
         (torch.randn(1024, 1024, generator=g) * 0.03).bfloat16(), (torch.randn(1024, generator=g) * 0.1).bfloat16(),
         (torch.randn(d_out, 1024, generator=g) * 0.05).bfloat16(), (torch.randn(d_out, generator=g) * 0.1).bfloat16()]
    wv, bv = (torch.randn(1, 1024, generator=g) * 0.05).bfloat16(), (torch.randn(1, generator=g) * 0.1).bfloat16()
    obs = torch.randn(M, 256, generator=g).bfloat16()
    legal = torch.rand(M, d_out, generator=g) < 0.6
    acts = torch.stack([torch.randint(0, n, (M,), generator=g) for n in nvec], -1)
    lo = 0
    for k, n in enumerate(nvec):   # the body's reference: every taken action legal
        legal[torch.arange(M), lo + acts[:, k]] = True
        lo += n
    policy = mapped_copy(cases.mlp_policy_evaluate_masked_nvec_value, "mlp", bias=True, output="evaluate",
                         taken="acts", mask="legal", value=("wv", "bv"), nvec=nvec)
    return obs, p, wv, bv, legal, acts, nvec, policy


def _args(obs, p, wv, bv, legal, acts, nvec, cuda):
    c = (lambda t: t.cuda()) if cuda else (lambda t: t)   # noqa: E731
    return (c(obs), *[c(t) for t in p], c(wv), c(bv), c(legal), c(acts), nvec)


def _mine(obs, p, wv, bv, legal, acts, nvec):
    pc = [t.cuda() for t in p]
    return mlp.mlp_forward(obs.cuda(), pc[0], pc[2], pc[4], biases=(pc[1], pc[3], pc[5]), output="evaluate",
                           taken=acts.cuda(), mask=legal.cuda(), nvec=nvec, value=(wv.cuda(), bv.cuda()))


@pytest.mark.parametrize("devices", [[0], [0, 0, 0]], ids=["1_rank", "3_ranks"])
def test_mapped_evaluate_head_through_public_api(K, devices):
    """@kt.mapped("mlp", bias=True, output="evaluate", taken="acts", mask="legal", value=("wv", "bv"), nvec=...) on
    Compute(gpus=1): each rank returns the bits of mlp_forward over its rows, and is within 2e-2 (bf16 logits of a
    different GEMM order) of the oracle's run of the body."""
    case = _public_case()
    obs, n = case[0], len(devices)
    want = ref_dispatch.spmd_call(cases.mlp_policy_evaluate_masked_nvec_value, *_args(*case[:7], False), num_proc=n,
                                  serialization="pickle")
    mine = _mine(*case[:7])
    with deployed(case[7], f"t-evaluate-{n}", devices) as remote:
        got = remote(*_args(*case[:7], True), serialization="pickle")
        torch.cuda.synchronize()
    assert len(got) == len(want) == n
    for r, (g, h) in enumerate(zip(got, want)):
        lo, hi = K.shard_bounds(obs.shape[0], n, r)
        assert isinstance(g, tuple) and len(g) == 3, r
        same([t.cpu() for t in g], [t[lo:hi].cpu() for t in mine], r)
        for k in range(3):
            assert torch.allclose(g[k].cpu(), h[k], rtol=2e-2, atol=2e-2), (r, k)


def test_mapped_evaluate_head_on_a_workers_subset(K):
    """Two workers of one rank each on cuda:0; workers=[1] returns rank 1's outputs only, the bits of mlp_forward."""
    import kubetorch_b200 as kt

    case = _public_case()
    mine = _mine(*case[:7])
    remote = kt.fn(case[7], name="t-evaluate-workers").to(
        kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute("b200", workers=2, num_proc=1,
                                                                                 devices=[0, 0]))
    try:
        got = remote(*_args(*case[:7], True), serialization="pickle", workers=[1])
        torch.cuda.synchronize()
    finally:
        remote.teardown()
    lo, hi = K.shard_bounds(case[0].shape[0], 2, 1)
    assert len(got) == 1
    same([t.cpu() for t in got[0]], [t[lo:hi].cpu() for t in mine], "workers=[1]")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("transfer", ["pull", "push"])
def test_mapped_evaluate_head_on_two_gpus(K, transfer):
    """Two ranks on two GPUs, staged pull and pushed form: the bits of one plain call."""
    case = _public_case()
    with deployed(case[7], f"t-evaluate-2gpu-{transfer}", [0, 1], transfer=transfer) as remote:
        got = remote(*_args(*case[:7], True), serialization="pickle")
        torch.cuda.synchronize(0)
        torch.cuda.synchronize(1)
    want = _mine(*case[:7])
    same([torch.cat([g[k].cpu() for g in got]) for k in range(3)], [t.cpu() for t in want], "two gpus")
