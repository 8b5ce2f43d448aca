"""-m gpu: the MLP trunk (the two hidden layers every MLP entry runs, layer_pair<true> in ktb_mlp.cu) and every head
on NaN, infinite, overflowing and subnormal inputs, against torch (tests/mlp_ieee_ref.py: the definition of
tests/policy_cases.py in torch on CPU).  The IEEE class of every output (NaN, +inf, -inf, finite) must equal the
reference's exactly; finite values are compared at the end-to-end bar, or bit for bit where the inputs are built of
exact products.  A poisoned row must not touch any other row, which must keep the bits of the clean call."""
import pytest
import torch

import policy_cases
from conftest import mapped_copy
from kubetorch_b200.device import mlp
from mlp_ieee_ref import (BF16_MAX, D_OUT, POISON_SITES, assert_matches, overflow_case, poisoned, random_net,
                          same_bits, subnormal_case, trunk)
from mlp_rig import GREEDY, SHIPPED_CHUNK, K, config, deployed, randn, run_guarded, tuning  # noqa: F401
from oracle import ref_dispatch

pytestmark = pytest.mark.gpu

E2E = dict(rtol=2 ** -7, atol=1e-2)     # the end-to-end bar of the MLP suites
NAN, INF = float("nan"), float("inf")


def cuda(ts):
    return tuple(None if t is None else t.cuda() for t in ts)


def logits_of(obs, net):
    w1, b1, w2, b2, w3, b3 = net
    return mlp.mlp_forward(obs, w1, w2, w3, biases=(b1, b2, b3))


# ---- 1. the trunk: NaN rows, row isolation --------------------------------------------------------------------------
M_EDGES = 17000        # the shipped 16 896-row chunk, then 104 rows: a ragged last tile (and chunk, at 256 rows)


def edge_rows(M):
    """Rows at the edges of 64-row halves, 128-row tiles, the last ragged tile and the shipped chunk."""
    return [0, 63, 64, 127, 128, M - 1, SHIPPED_CHUNK - 1, SHIPPED_CHUNK]


@pytest.mark.parametrize("chunk", [None, 256], ids=["shipped_chunk", "chunk256"])
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
def test_nan_observation_poisons_only_its_row(K, bias, chunk):
    """One NaN in an observation row makes that row's logits all NaN (torch.relu keeps it, and NaN · 0 is NaN), and
    every other row keeps the bits of the clean call: each epilogue thread owns rows r and r + 8, so this is also row
    isolation in the epilogue."""
    net = cuda(random_net(11, bias=bias))
    obs = randn((M_EDGES, 256), 12)
    bad = obs.clone()
    rows = edge_rows(M_EDGES)
    for r in rows:
        bad[r, (37 * r) % 256] = NAN
    with tuning(chunk):
        clean, got = logits_of(obs, net), logits_of(bad, net)
    torch.cuda.synchronize()
    hit = torch.zeros(M_EDGES, dtype=torch.bool, device="cuda")
    hit[rows] = True
    assert bool(got[hit].isnan().all()), f"NaN rows came back with {int((~got[hit].isnan()).sum())} non-NaN logits"
    assert not bool(clean.isnan().any())
    assert torch.equal(got[~hit], clean[~hit])
    near = sorted({min(max(r + d, 0), M_EDGES - 1) for r in rows for d in (-1, 0, 1)})
    assert_matches(got[near], trunk(bad[near], *net), f"rows {near}", **E2E)


@pytest.mark.parametrize("inf", [INF, -INF], ids=["+inf", "-inf"])
@pytest.mark.parametrize("weights", ["mixed", "positive", "negative", "zero"])
def test_infinite_observation_follows_torch(K, weights, inf):
    """±inf in column 77 of some rows against W1 of mixed sign, one sign, or a zero column 77 (inf · 0 = NaN): each
    row's class and value as torch gives them (NaN rows, or finite rows where the ReLU zeroes -inf), the other rows
    bit for bit as the clean call."""
    M, col = 1000, 77
    w1, b1, w2, b2, w3, b3 = random_net(21)
    w1 = {"mixed": w1, "positive": w1.abs(), "negative": -w1.abs(), "zero": w1.index_fill(1, torch.tensor([col]), 0)
          }[weights]
    net = cuda((w1, b1, w2, b2, w3, b3))
    obs = randn((M, 256), 22)
    bad = obs.clone()
    rows = [0, 7, 8, 500, 999]
    bad[rows, col] = inf
    clean, got = logits_of(obs, net), logits_of(bad, net)
    assert_matches(got, trunk(bad, *net), f"{weights} {inf}", **E2E)
    keep = torch.ones(M, dtype=torch.bool, device="cuda")
    keep[rows] = False
    assert torch.equal(got[keep], clean[keep])


@pytest.mark.parametrize("value", [NAN, INF, -INF], ids=["nan", "+inf", "-inf"])
@pytest.mark.parametrize("site", list(POISON_SITES))
def test_non_finite_weight_or_bias_follows_torch(K, site, value):
    """NaN or ±inf in W1 (a column of the first and of the last K block, a row in each 256-wide N tile), in W2, or in
    b1 or b2 (an entry in each N tile): every row's logits as torch gives them.  An infinite W1 entry makes a unit
    +inf on the rows where its observation has one sign and 0 on the others, so rows differ."""
    net = cuda(poisoned(random_net(31), site, value))
    obs = randn((1000, 256), 32)
    got = logits_of(obs, net)
    want = trunk(obs, *net)
    assert_matches(got, want, f"{site} {value}", **E2E)


# ---- 2. overflow and subnormals, built of exact products ---------------------------------------------------------
@pytest.mark.parametrize("layer", ["hidden", "head"])
def test_overflow_rounds_and_accumulates_as_ieee(K, layer):
    """A product exactly on the bf16 overflow tie rounds to ±inf as torch's .bfloat16() does, one fp32 ulp below it
    stays at ±BF16_MAX, and two products above FLT_MAX / 2 overflow the fp32 accumulator to ±inf, in layer 1 (where
    the ReLU and all-nonzero W2 and W3 carry the +inf to every logit with its sign) and in the head (no ReLU: -inf
    too).  Every output bit for bit."""
    obs, *net = cuda(overflow_case(layer))
    got = logits_of(obs, net)
    want = trunk(obs, *net)
    assert_matches(got, want, layer)
    g, kind = got.cpu().float(), torch.arange(obs.shape[0]) % 4
    if layer == "hidden":
        assert bool(g[kind % 2 == 0].isinf().all())
        assert bool((g[kind == 1].abs() == 255 * 2.0 ** 112).all())   # BF16_MAX · 2^-8 · 256 · 2^-8
    else:
        assert bool(g[kind == 0, :2].isinf().all()) and bool(g[kind == 2, 2:4].isinf().all())
        assert bool((g[kind == 1, :2].abs() == BF16_MAX).all())


@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
def test_subnormals_are_not_flushed(K, bias):
    """bf16 subnormal observations and weights times 2^100 give their exact normal products, and normal inputs (with a
    bias, too) whose exact result is subnormal keep it through layer 2 and the head, positive and negative: as torch,
    nothing is flushed to zero.  Every output bit for bit."""
    obs, *net = cuda(subnormal_case(bias))
    got = logits_of(obs, net)
    want = trunk(obs, *net)
    assert bool((want[:, 2].float() != 0).all()) and bool((want[:, D_OUT - 1].float() < 0).all())
    assert_matches(got, want, f"subnormal bias={bias}")


# ---- 3. every form ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", [SHIPPED_CHUNK, 256])
def test_every_form_gives_the_same_bits(K, chunk):
    """NaN, +inf and -inf observation rows and a +inf in W1 (NaN rows where observation 3 is positive): the greedy
    entry's logits and actions are the same in the plain form, the staged form pulled by kernel and by copy engine, and
    the pushed form (3 ranks on cuda:0), with NaN counted as equal."""
    M, d_out = 3 * 1408, 18
    w, b = config(41, d_out)
    w = (w[0].clone(), w[1], w[2])
    w[0][900, 3] = INF
    obs = randn((M, 256), 42)
    for i, r in enumerate((0, 129, 1407, 1408, 2900, M - 1)):
        obs[r, (11 * r) % 256] = (NAN, INF, -INF)[i % 3]
    want_l, want_a = mlp.mlp_forward(obs, *w, biases=b, output="both")
    assert 0 < int(want_l.isnan().all(1).sum()) < M
    for form, ce in (("plain", None), ("staged", 0), ("staged", 1), ("pushed", None)):
        with tuning(stage_ce=ce):
            bufs = run_guarded(form, GREEDY, K, chunk, obs, w, b)
        torch.cuda.synchronize()
        what = f"{form} ce={ce} chunk={chunk}"
        same_bits(bufs["logits"].view(torch.bfloat16).view(M, d_out), want_l, what)
        same_bits(bufs["actions"].view(torch.int64), want_a, what)


# ---- 4. the heads -------------------------------------------------------------------------------------------------
M_HEAD, D_HEAD, NVEC = 640, 18, (3, 5, 10)
HEAD_ROWS = [0, 8, 63, 64, 300, 639]


def _nan_linear(w, b):
    """A layer whose every output is NaN on every row: zero weights, NaN biases."""
    return torch.zeros_like(w), torch.full_like(b, NAN)


def _head_call(kind, obs, net, nan_head):
    """Every output of head `kind` over obs; with nan_head the head's linear layers (W3 and any value or log-std layer)
    are replaced by _nan_linear, the all-NaN logits whose result each head's suite pins."""
    w1, b1, w2, b2, w3, b3 = net
    g = torch.Generator(device="cuda").manual_seed(51)
    M = obs.shape[0]
    wv, bv = randn((1, 1024), 52), randn((1,), 53)
    w_ls, b_ls = randn((D_HEAD, 1024), 54, 0.02), randn((D_HEAD,), 55, 0.1)
    if nan_head:
        (w3, b3), (wv, bv), (w_ls, b_ls) = _nan_linear(w3, b3), _nan_linear(wv, bv), _nan_linear(w_ls, b_ls)
    log_std = torch.linspace(-1.0, 0.5, D_HEAD, device="cuda")
    legal = torch.rand(M, D_HEAD, generator=g, device="cuda") < 0.6
    legal[:, 0] = True
    kw = {
        "greedy": dict(output="both"),
        "sample": dict(output="sample", seed=5),
        "gaussian": dict(output="gaussian", seed=5, log_std=log_std),
        "masked_greedy": dict(output="both", mask=legal),
        "masked_sample": dict(output="sample", seed=5, mask=legal),
        "sample_value": dict(output="sample", seed=5, value=(wv, bv)),
        "gaussian_value": dict(output="gaussian", seed=5, log_std=log_std, value=(wv, bv)),
        "multidiscrete": dict(output="both", nvec=NVEC),
        "multidiscrete_sample": dict(output="sample", seed=5, nvec=NVEC),
        "gaussian_state": dict(output="gaussian", seed=5, log_std=(w_ls, b_ls), squash=True),
        "epsilon_greedy": dict(output="epsilon_greedy", seed=5, epsilon=0.3),
        "evaluate": dict(output="evaluate", taken=torch.randint(0, D_HEAD, (M,), generator=g, device="cuda")),
        "gaussian_evaluate": dict(output="gaussian_evaluate", log_std=log_std,
                                  taken=torch.randn(M, D_HEAD, generator=g, device="cuda")),
        "deterministic": dict(output="deterministic", seed=5, noise=0.2, noise_clip=0.5),
    }[kind]
    out = mlp.mlp_forward(obs, w1, w2, w3, biases=(b1, b2, b3), **kw)
    return out if isinstance(out, tuple) else (out,)


HEAD_KINDS = ["greedy", "sample", "gaussian", "masked_greedy", "masked_sample", "sample_value", "gaussian_value",
              "multidiscrete", "multidiscrete_sample", "gaussian_state", "epsilon_greedy", "evaluate",
              "gaussian_evaluate", "deterministic"]


@pytest.mark.parametrize("kind", HEAD_KINDS)
def test_nan_rows_reach_each_head_as_all_nan_logits(K, kind):
    """NaN observation rows: the clean rows keep the bits of the clean call, and the poisoned rows get what the head
    gives for all-NaN logits (the head called with W3 = 0 and NaN b3; its suite pins that result)."""
    net = cuda(random_net(61, d_out=D_HEAD))
    obs = randn((M_HEAD, 256), 62)
    bad = obs.clone()
    bad[HEAD_ROWS, 100] = NAN
    hit = torch.zeros(M_HEAD, dtype=torch.bool, device="cuda")
    hit[HEAD_ROWS] = True
    clean, got, nan_ref = (_head_call(kind, o, net, n) for o, n in ((obs, False), (bad, False), (obs, True)))
    for i, (c, g, n) in enumerate(zip(clean, got, nan_ref)):
        same_bits(g[~hit], c[~hit], f"{kind} output {i}: clean rows")
        same_bits(g[hit], n[hit], f"{kind} output {i}: NaN rows")
    assert any(bool(g[hit].isnan().any()) for g in got if g.is_floating_point())


def _critic(d_in, d_act, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale: (torch.randn(*s, generator=g) * scale).bfloat16().cuda()   # noqa: E731
    return (r(1024, d_in + d_act, scale=0.05), r(1024, scale=0.1), r(1024, 1024, scale=0.05), r(1024, scale=0.1),
            r(1, 1024, scale=0.05), r(1, scale=0.1))


@pytest.mark.parametrize("twin", [False, True], ids=["critic", "twin"])
def test_critic_nan_rows(K, twin):
    """NaN observation rows and NaN action rows: q (q1, q2 and q_min for the twin) NaN on exactly those rows, the
    others the bits of the clean call."""
    M, d_in, d_act = M_HEAD, 64, 6
    c, c2 = _critic(d_in, d_act, 71), _critic(d_in, d_act, 72)
    obs = randn((M, d_in), 73)
    act = torch.randn(M, d_act, generator=torch.Generator(device="cuda").manual_seed(74), device="cuda")
    bad_obs, bad_act = obs.clone(), act.clone()
    bad_obs[HEAD_ROWS[:3], 5] = NAN
    bad_act[HEAD_ROWS[3:], d_act - 1] = NAN
    hit = torch.zeros(M, dtype=torch.bool, device="cuda")
    hit[HEAD_ROWS] = True

    def q(o, a):
        out = mlp.mlp_forward(o, c[0], c[2], c[4], biases=(c[1], c[3], c[5]), output="critic", action=a,
                              twin=c2 if twin else None)
        return out if isinstance(out, tuple) else (out,)

    for i, (cl, g) in enumerate(zip(q(obs, act), q(bad_obs, bad_act))):
        assert not bool(cl.isnan().any())
        assert bool(g[hit].isnan().all()), (twin, i, g[hit])
        same_bits(g[~hit], cl[~hit], f"q{i}: clean rows")


TD = {"td3": ("deterministic", dict(noise=0.2, noise_clip=0.5, seed=11), True, None),
      "sac": ("gaussian", dict(squash=True, seed=12), True, 0.2)}


def _td_nets(d_in, d_act, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale: (torch.randn(*s, generator=g) * scale).bfloat16().cuda()   # noqa: E731
    net = lambda w: (r(*w[0], scale=0.05), r(w[0][0], scale=0.1), r(*w[1], scale=0.05), r(w[1][0], scale=0.1),  # noqa
                     r(*w[2], scale=0.05), r(w[2][0], scale=0.1))
    critic = lambda: net(((256, d_in + d_act), (256, 256), (1, 256)))   # noqa: E731
    actor = net(((256, d_in), (256, 256), (d_act, 256)))
    return critic(), critic(), actor, (r(d_act, 256, scale=0.05), r(d_act, scale=0.1))


def _td(name, obs, c1, c2, actor, ls, reward, done):
    policy, opts, twin, alpha = TD[name]
    kw = dict(output="td_target", actor=actor, policy=policy, reward=reward, done=done, gamma=0.99,
              twin=c2 if twin else None, **opts)
    if policy == "gaussian":
        kw.update(log_std=ls, alpha=alpha)
    return mlp.mlp_forward(obs, c1[0], c1[2], c1[4], biases=(c1[1], c1[3], c1[5]), **kw)


@pytest.mark.parametrize("name", list(TD))
def test_td_target_nan(K, name):
    """NaN next-observation rows give NaN y on those rows, done = 1 included (0 · NaN), the others the bits of the
    clean call; a NaN in W1 or W2 of either target critic or of the actor gives NaN y on every row."""
    M, d_in, d_act = M_HEAD, 64, 6
    c1, c2, actor, ls = _td_nets(d_in, d_act, 81)
    obs = randn((M, d_in), 82)
    g = torch.Generator(device="cuda").manual_seed(83)
    reward = torch.randn(M, generator=g, device="cuda")
    done = (torch.rand(M, generator=g, device="cuda") < 0.5).float()
    done[HEAD_ROWS[::2]] = 1.0
    bad = obs.clone()
    bad[HEAD_ROWS, 9] = NAN
    hit = torch.zeros(M, dtype=torch.bool, device="cuda")
    hit[HEAD_ROWS] = True
    clean, got = _td(name, obs, c1, c2, actor, ls, reward, done), _td(name, bad, c1, c2, actor, ls, reward, done)
    assert not bool(clean.isnan().any())
    assert bool(got[hit].isnan().all()), got[hit]
    same_bits(got[~hit], clean[~hit], f"{name}: clean rows")
    for which, w in (("critic", 0), ("critic", 2), ("twin", 0), ("twin", 2), ("actor", 0), ("actor", 2)):
        nets = {"critic": c1, "twin": c2, "actor": actor}
        t = nets[which][w].clone()
        t[100, 3] = NAN
        nets[which] = nets[which][:w] + (t,) + nets[which][w + 1:]
        y = _td(name, obs, nets["critic"], nets["twin"], nets["actor"], ls, reward, done)
        assert bool(y.isnan().all()), (name, which, w, int((~y.isnan()).sum()))


# ---- 5. the public API --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_ranks", [1, 3])
def test_mapped_policy_with_non_finite_rows_matches_the_oracle(K, n_ranks):
    """kt.mapped("mlp", bias=True) on ranks of cuda:0 with NaN, +inf and -inf observation rows: every rank's logits
    have the oracle's class everywhere and its values within the end-to-end bar."""
    obs = torch.randn(1000, 256, generator=torch.Generator().manual_seed(91)).bfloat16()
    for i, r in enumerate((0, 1, 332, 333, 334, 666, 667, 998, 999)):
        obs[r, (5 * r) % 256] = (NAN, INF, -INF)[i % 3]
    p = random_net(92, d_out=18)
    want = ref_dispatch.spmd_call(policy_cases.mlp_policy_biased, obs, *p, num_proc=n_ranks, serialization="pickle")
    policy = mapped_copy(policy_cases.mlp_policy_biased, "mlp", bias=True, output="logits")
    with deployed(policy, f"t-ieee-{n_ranks}", [0] * n_ranks) as remote:
        got = remote(obs.cuda(), *[t.cuda() for t in p], serialization="pickle")
        torch.cuda.synchronize()
    assert len(got) == len(want) == n_ranks
    assert any(bool(w.isnan().any()) for w in want)
    for r, (g, w) in enumerate(zip(got, want)):
        assert g.dtype == torch.bfloat16
        assert_matches(g, w, f"rank {r} of {n_ranks}", **E2E)
