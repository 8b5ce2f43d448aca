"""Registry of *mapped callables*: user functions whose body is one of the closed set of ops that
libktb200 executes as sm_90a kernels (identity / scale / affine, their sum-reduced forms, the
bf16 MLP policy, generalized advantage estimation, V-trace, n-step bootstrapped returns, Retrace(λ) and prioritized
replay sampling).

Arbitrary Python cannot become a CUDA kernel, so the device route is opt-in by declaration:

    @kt.mapped("scale", alpha=2.0)
    def double(x):
        r, w = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
        return x.chunk(w)[r] * 2

The Python body stays the semantic definition (it is what the reference would run on each rank,
kt/serving/http_server.py:1845-1891, and what the CPU backends still run); the decorator states
which kernel computes the same thing.  Parity between the two is what tests/ checks.
Parameter values may be constants or the *name* of a call argument (``alpha="alpha"``).
"""
from __future__ import annotations

import inspect
import math
from dataclasses import dataclass, field
from typing import Any, Callable, Dict, Optional

from .sampling import _check_seed

MAPPED_ATTR = "__ktb_mapped__"
ELEMENTWISE_OPS = ("identity", "scale", "affine")
ALL_OPS = ELEMENTWISE_OPS + ("mlp", "gae", "vtrace", "nstep", "retrace", "per")
# The options of op="gae": gamma and lam, each required (a finite number or the name of a call argument holding one),
# and self_check
GAE_OPTIONS = ("gamma", "lam")
# The options of op="vtrace" and their defaults (None: required) beside self_check: gamma and lam a finite number or the
# name of a call argument holding one (VTRACE_ARGUMENTS); rho_bar, c_bar and pg_rho_bar constants, a number > 0 or None
# (no clip).  mapped() stores every default it fills in into MappedSpec.extra.
VTRACE_OPTIONS = dict(gamma=None, lam=1.0, rho_bar=1.0, c_bar=1.0, pg_rho_bar=1.0)
VTRACE_ARGUMENTS = ("gamma", "lam")
# The options of op="nstep" beside self_check, both required (None): n an int constant in [1, 32], gamma a finite number
# or the name of a call argument holding one (NSTEP_ARGUMENTS)
NSTEP_OPTIONS = dict(n=None, gamma=None)
NSTEP_ARGUMENTS = ("gamma",)
# The options of op="retrace": gamma and lam, each required (a finite number or the name of a call argument holding
# one), and self_check
RETRACE_OPTIONS = ("gamma", "lam")
# The options of op="per" beside self_check, all required: batch an int constant in [1, 8192], beta a finite number >= 0
# and seed an int in [0, 2**64), each of the last two or the name of a call argument holding one (PER_ARGUMENTS)
PER_OPTIONS = ("batch", "beta", "seed")
PER_ARGUMENTS = ("beta", "seed")
MLP_OUTPUTS = ("logits", "actions", "both", "sample", "gaussian", "epsilon_greedy", "evaluate",
               "gaussian_evaluate", "deterministic", "critic", "td_target", "dqn_target")   # also device.mlp.OUTPUTS
EVALUATE_OUTPUTS = ("evaluate", "gaussian_evaluate")
# The options of output="td_target" and of output="dqn_target" that no other output takes: the supervisor passes them
# to mlp_scatter_gather with their output only
TD_OPTIONS = ("actor", "policy", "reward", "done", "gamma", "alpha")
DQN_OPTIONS = ("online", "reward", "done", "gamma")

# The options each MLP output takes beside bias= and output=, True for those it requires, keyed by (output, policy):
# a TD target's depend on its policy=, and every other output has none.  mapped() and device.mlp._check_policy refuse
# every other option and report every missing one (check_mlp_options).
MLP_TAKES = {
    ("logits", None): dict(mask=False),
    ("actions", None): dict(mask=False, nvec=False),
    ("both", None): dict(mask=False, nvec=False),
    ("sample", None): dict(seed=True, mask=False, value=False, nvec=False),
    ("gaussian", None): dict(seed=True, log_std=True, value=False, log_std_bounds=False, squash=False),
    ("epsilon_greedy", None): dict(seed=True, epsilon=True, mask=False),
    ("evaluate", None): dict(taken=True, mask=False, value=False, nvec=False),
    ("gaussian_evaluate", None): dict(taken=True, log_std=True, value=False),
    ("deterministic", None): dict(noise=False, noise_clip=False, seed=False, squash=False),
    ("critic", None): dict(action=True, twin=False),
    ("td_target", "deterministic"): dict(actor=True, policy=True, reward=True, done=True, gamma=True, twin=False,
                                         noise=False, noise_clip=False, seed=False, squash=False),
    ("td_target", "gaussian"): dict(actor=True, policy=True, reward=True, done=True, gamma=True, twin=False, seed=True,
                                    alpha=True, log_std=True, log_std_bounds=False, squash=False),
    ("dqn_target", None): dict(reward=True, done=True, gamma=True, online=False, mask=False),
}

# Each MLP option's form at decoration: "name", the name of a call argument; "names", a tuple of such names
# (_NAMES); "name or constant", either; "constant", a value fixed at decoration.  The supervisor binds the names to
# the call's arguments on every call.
MLP_FORMS = dict(seed="name or constant", log_std="names", mask="name", value="names", nvec="constant",
                 log_std_bounds="constant", squash="constant", epsilon="name or constant", taken="name",
                 noise="name or constant", noise_clip="constant", action="name", twin="names", actor="names",
                 policy="constant", reward="name", done="name", gamma="constant", alpha="name or constant",
                 online="names")

# What each "names" option names, for the message that refuses a wrong count (log_std may also be one name)
_NAMES =dict(log_std="one call argument or two (w_ls, b_ls)", value="two call arguments (wv, bv)",
              twin="the second critic's {n} call arguments {what}", actor="the actor's {n} call arguments {what}",
              online="the online network's {n} call arguments {what}")


def check_mlp_options(output: str, policy, given, argument: bool = False) -> dict:
    """MLP_TAKES's row of `output` (with a TD target's `policy`), or ValueError naming the first option of `given` that
    the row does not take, else the first option it requires that `given` lacks.  mapped() says "mask= is not an
    option of output=...", and with `argument` the device layer "mask is not an argument of output=..."."""
    eq, what = ("", "an argument") if argument else ("=", "an option")
    row = MLP_TAKES.get((output, policy if isinstance(policy, str) else None)) or MLP_TAKES.get((output, None))
    if row is None:
        policies = tuple(p for o, p in MLP_TAKES if o == output)
        if policy is None:
            raise ValueError(f'policy{eq} is required with output="{output}": one of {policies}')
        raise ValueError(f'policy{eq} must be one of {policies} with output="{output}", got {policy!r}')
    where = f'output="{output}"' + (f', policy="{policy}"' if "policy" in row else "")
    for name in given:
        if name not in row:
            raise ValueError(f'{name}{eq} is not {what} of {where}, which takes {", ".join(o + eq for o in row)}')
    for name, required in row.items():
        if required and name not in given:
            raise ValueError(f"{name}{eq} is required with {where}")
    return row


def check_noise(name: str, v) -> float:
    """noise or noise_clip of a deterministic actor: a number (not a bool) >= 0, not NaN."""
    if isinstance(v, bool) or not isinstance(v, (int, float)):
        raise ValueError(f"{name} must be a number, got {v!r}")
    if v != v or v < 0:
        raise ValueError(f"{name} must be >= 0 and not NaN, got {v!r}")
    return v


def check_squash(v) -> bool:
    if not isinstance(v, bool):
        raise ValueError(f"squash must be True or False, got {v!r}")
    return v


def check_log_std_bounds(v) -> tuple:
    """log_std_bounds as a pair of floats: two numbers (not bools), not NaN, low <= high."""
    if not isinstance(v, (tuple, list)) or len(v) != 2 or \
            not all(isinstance(b, (int, float)) and not isinstance(b, bool) for b in v):
        raise ValueError(f"log_std_bounds must be (low, high), two numbers, got {v!r}")
    lo, hi = float(v[0]), float(v[1])
    if lo != lo or hi != hi:
        raise ValueError(f"log_std_bounds must not be NaN, got {v!r}")
    if lo > hi:
        raise ValueError(f"log_std_bounds must have low <= high, got {v!r}")
    return lo, hi


def check_epsilon(v):
    """A constant ε: a number (not a bool), not NaN."""
    if isinstance(v, bool) or not isinstance(v, (int, float)):
        raise ValueError(f"epsilon must be a number, got {v!r}")
    if v != v:
        raise ValueError("epsilon must not be NaN (a NaN never explores: pass 0.0 for that)")
    return v


def check_finite(name: str, v):
    """gamma or alpha of a TD target: a finite number (not a bool)."""
    if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v):
        raise ValueError(f"{name} must be a finite number, got {v!r}")
    return v


# The check of each MLP option's constant value, which returns the value as MappedSpec.extra keeps it
CONSTANT_CHECKS = dict(seed=_check_seed, noise=lambda v: check_noise("noise", v),
                        noise_clip=lambda v: check_noise("noise_clip", v), squash=check_squash,
                        log_std_bounds=check_log_std_bounds, epsilon=check_epsilon,
                        gamma=lambda v: check_finite("gamma", v), alpha=lambda v: check_finite("alpha", v),
                        nvec=lambda v: check_nvec(v))


def check_mlp_rules(row: dict, output: str, policy, log_std, given, argument: bool = False) -> None:
    """The rules of the MLP options that are not rows of MLP_TAKES, with the option names `given` and `row` as
    check_mlp_options returned it: seed is given exactly when noise is and noise_clip only with noise (where noise is an
    option); log_std_bounds and squash only with a log_std=(w_ls, b_ls) pair (where log_std is an option); a pair is
    refused by output="gaussian_evaluate" and required by policy="gaussian"."""
    eq = "" if argument else "="
    pair = isinstance(log_std, (tuple, list))
    if "noise" in row:
        if ("noise" in given) != ("seed" in given):
            raise ValueError(f'output="{output}" takes {"a seed" if argument else "seed="} exactly when it takes '
                             f'noise{eq}: the noise-free actor draws nothing')
        if "noise_clip" in given and "noise" not in given:
            raise ValueError(f"noise_clip{eq} is an option of noise{eq} only: it clips the noise")
    if "log_std" in row and not pair and ("log_std_bounds" in given or "squash" in given):
        raise ValueError(f"log_std_bounds{eq} and squash{eq} are options of a state-dependent log_std=(w_ls, b_ls) only")
    if pair and output == "gaussian_evaluate":
        raise ValueError('output="gaussian_evaluate" takes a state-independent log_std, not a log_std=(w_ls, b_ls) '
                         'pair (evaluating a state-dependent or squashed head is not supported)')
    if policy == "gaussian" and not pair:
        raise ValueError(f'log_std=(w_ls, b_ls) is required with policy="gaussian": the actor\'s state-dependent '
                         f'log-std head')


@dataclass
class MappedSpec:
    op: str
    alpha: Any = 1.0
    beta: Any = 0.0
    reduce: Optional[str] = None       # None | "sum"
    arg: str = None                    # name of the tensor argument (default: first parameter)
    extra: Dict[str, Any] = field(default_factory=dict)

    def bind(self, fn: Callable, args, kwargs):
        """Resolve (tensor, alpha, beta, bound_arguments) for one call."""
        sig = self.extra.get("__sig__")
        if sig is None:  # inspect.signature costs ~15 us: once per callable, not per call
            sig = self.extra["__sig__"] = inspect.signature(fn)
            self.extra["__names__"] = list(sig.parameters)
            self.extra["__plain__"] = all(
                p.kind is p.POSITIONAL_OR_KEYWORD and p.default is p.empty for p in sig.parameters.values())
        names = self.extra["__names__"]
        if not kwargs and len(args) == len(names) and self.extra["__plain__"]:
            arguments = dict(zip(names, args))  # the common call shape: skip Signature.bind (~10 us)
        else:
            bound = sig.bind(*args, **kwargs)   # raises the same TypeError the callable itself would
            bound.apply_defaults()
            arguments = bound.arguments
        tensor_name = self.arg or names[0]
        if tensor_name not in arguments:
            raise TypeError(f"mapped callable {fn.__name__}() is missing its tensor argument '{tensor_name}'")

        def resolve(v):
            if isinstance(v, str):
                if v not in arguments:
                    raise TypeError(f"mapped callable {fn.__name__}(): parameter '{v}' not found in the call")
                return arguments[v]
            return v

        return arguments[tensor_name], resolve(self.alpha), resolve(self.beta), arguments


_UNSET = object()   # mapped()'s alpha when not given: 1.0, and no entropy coefficient of a TD target


def mapped(op: str, alpha: Any = _UNSET, beta: Any = _UNSET, reduce: Optional[str] = None, arg: str = None, **extra):
    """Declare that the decorated function is computed by device op `op` (see module docstring).

    The "mlp" op takes more options.  ``bias=True``: the callable is ``(obs, w1, b1, w2, b2, w3, b3, ...)``, an
    nn.Linear policy with biases (default False: ``(obs, w1, w2, w3, ...)``).  ``output``: ``"logits"`` (default),
    ``"actions"`` (int64 greedy actions, argmax of the bf16 logits), ``"both"`` (``(logits, actions)`` per rank) or
    ``"sample"`` (``(actions, log_probs)`` per rank: int64 actions drawn from softmax(logits) by Gumbel-max with the
    noise of kubetorch_b200.sampling.gumbel_noise over the rows' global indices, and the fp32 log-probability of
    each) or ``"gaussian"`` (``(actions, log_probs)`` per rank: fp32 actions ``logits + exp(log_std)·z`` with ``z``
    the noise of kubetorch_b200.sampling.normal_noise over the rows' global indices, and the fp32 log-density of each
    row's action; the callable is ``(obs, w1, b1, w2, b2, w3, b3, log_std, seed)``).  ``seed``, required with
    ``output="sample"`` or ``"gaussian"`` and refused otherwise: an int in [0, 2**64) or the name of a call argument
    that holds one.  ``log_std``, required with ``output="gaussian"`` and refused otherwise: the name of the call
    argument that holds the fp32 [d_out] log standard deviation.  ``mask``, an option of every output but
    ``"gaussian"``: the name of the call argument that holds a per-row legal-action mask, a bool [M, d_out] tensor on
    the device of obs (True: legal); the head then computes ``logits.masked_fill(~mask, -inf)`` and every output is
    taken from those masked logits (the body applies ``legal.chunk(WORLD_SIZE)[RANK]`` to its rows).  ``value``, an
    option of ``output="sample"`` and ``"gaussian"`` with ``bias=True``: the names ``(wv, bv)`` of the two call
    arguments that hold a critic ``nn.Linear(d_hidden, 1)`` on the same trunk, its bf16 weight [1, d_hidden] and bias
    [1]; each rank then returns ``(actions, log_probs, values)`` with fp32 ``values = F.linear(h, wv, bv)`` of its
    rows, the bf16 result widened exactly.  ``nvec``, an option of ``output="actions"``, ``"both"`` and ``"sample"``
    (with ``mask=`` and ``value=`` as those allow): a tuple of ints ``(n_0, ..., n_{G-1})`` summing to d_out, a
    constant of the deployment, for a ``MultiDiscrete(nvec)`` action space.  The logits split into G groups of
    columns, one categorical each: actions become int64 ``[rows, G]`` of group-relative indices (greedy, or sampled
    per group with the same noise), and log_probs the fp32 sum of the groups' log-probabilities in group order.
    ``log_std`` may instead name two call arguments ``(w_ls, b_ls)`` (with ``bias=True``): a state-dependent log-std
    head ``nn.Linear(d_hidden, d_out)`` on the same trunk, clamped to ``log_std_bounds`` (two numbers, default
    ``(-20.0, 2.0)``), with ``squash=True`` for tanh-squashed actions and the log-probability's tanh correction (SAC's
    actor); ``value=`` may go beside it.  ``log_std_bounds`` and ``squash`` are options of that form only.
    ``output="epsilon_greedy"`` (a Q-network's actor: DQN, Ape-X, R2D2) returns ``(actions, q, q_max)`` per rank and
    takes ``seed=`` and ``epsilon=``, a number or the name of a call argument that holds a float or a per-row fp32
    tensor [M] on the device of obs (the body takes ``eps.chunk(WORLD_SIZE)[RANK]`` of a tensor): with ``u, w =
    kubetorch_b200.sampling.explore_noise(seed, row0, rows, d_out)`` a row explores iff ``u < ε`` and takes the legal
    column with the largest ``w``, and otherwise the argmax of its logits; ``q`` is the fp32 logit of the action taken
    and ``q_max`` that of the argmax (``mask=`` applies, ``value=`` and ``nvec=`` do not).
    ``output="evaluate"`` and ``"gaussian_evaluate"`` score actions the caller already holds (SB3's
    ``evaluate_actions``): ``taken=`` names the call argument that holds them, int64 ``[M]`` (``[M, G]`` with
    ``nvec=``) group-relative indices, or fp32 ``[M, d_out]`` with ``"gaussian_evaluate"``, on the device of obs (the
    body takes ``taken.chunk(WORLD_SIZE)[RANK]``).  Each rank returns ``(log_probs, entropy)``, or ``(log_probs,
    entropy, values)`` with ``value=``: the fp32 log-probability of each row's action and the entropy of its policy,
    summed over groups, under ``logits.masked_fill(~mask, -inf)`` (``"evaluate"``; ``mask=`` and ``nvec=`` apply) or
    ``Normal(logits, exp(log_std))`` (``"gaussian_evaluate"``, with ``log_std=`` naming one argument).  They draw no
    noise, so ``seed=``, ``epsilon=``, ``squash=``, ``log_std_bounds=`` and a ``log_std`` pair are refused.
    ``output="deterministic"`` is the actor of DDPG and TD3: each rank returns fp32 actions ``[rows, d_out]``,
    ``tanh(logits)`` with ``squash=True`` (the default) and the fp32 logits with ``squash=False``, plus, with ``noise=``
    σ (a number >= 0 or the name of a call argument that holds one), ``(σ·z).clamp(-c, c)`` with ``z`` the noise of
    ``"gaussian"`` and ``c`` = ``noise_clip=`` (a number >= 0, default +inf), then clamped to [-1, 1] when squashed.
    ``seed=`` is required exactly when ``noise=`` is given.  Exploration is ``noise=0.1``; TD3's target policy
    smoothing is ``noise=0.2, noise_clip=0.5``.  ``mask=``, ``value=``, ``nvec=``, ``log_std=``, ``log_std_bounds=``,
    ``epsilon=`` and ``taken=`` are refused.
    ``output="critic"`` is a Q(s, a) critic (SAC's and TD3's, forward only): ``action=`` names the call argument that
    holds the fp32 actions ``[M, d_act]`` (1 <= d_act <= 64) on the device of obs (the body takes
    ``act.chunk(WORLD_SIZE)[RANK]``), the callable is ``(obs, w1, b1, w2, b2, w3, b3, act, ...)`` (``(obs, w1, w2, w3,
    act, ...)`` without ``bias=True``) with ``w1 [d_hidden, d_in + d_act]`` and ``w3 [1, d_hidden]``, and each rank
    returns the fp32 ``q [rows]`` of ``torch.cat([obs, act.to(torch.bfloat16)], -1)``.  ``twin=`` names the second
    critic's six arguments ``(w1, b1, w2, b2, w3, b3)`` (three, ``(w1, w2, w3)``, without ``bias=True``): each rank then
    returns ``(q1, q2, q_min)`` with ``q_min = torch.minimum(q1, q2)``.  ``seed=``, ``mask=``, ``value=``, ``nvec=``,
    ``log_std=``, ``log_std_bounds=``, ``squash=``, ``epsilon=``, ``taken=``, ``noise=`` and ``noise_clip=`` are
    refused, and ``action=`` and ``twin=`` with every other output.
    ``output="td_target"`` is the Bellman target of TD3, DDPG and SAC (forward only): the callable is ``(next_obs,
    w1, b1, w2, b2, w3, b3, ...)``, the (target) critic as with ``"critic"``, and each rank returns the fp32 ``y`` of
    its rows, ``reward + gamma * (1 - done) * t``.  ``actor=`` names the (target) actor's six arguments (three without
    ``bias=True``); ``policy="deterministic"`` takes its next actions as ``output="deterministic"`` does, with
    ``noise=``, ``noise_clip=``, ``seed=`` and ``squash=`` (TD3: ``noise=0.2, noise_clip=0.5``; DDPG: no noise), and
    ``t`` is the critic's ``q``, or with ``twin=`` the minimum of the two; ``policy="gaussian"`` samples them as
    ``output="gaussian"`` with ``log_std=(w_ls, b_ls)``, ``log_std_bounds=``, ``squash=`` and ``seed=`` (SAC), and
    ``t`` less ``alpha * log_prob``.  ``reward=`` and ``done=`` name fp32 ``[M]`` or ``[M, 1]`` arguments on the device
    of obs (the body takes their ``chunk(WORLD_SIZE)[RANK]``), ``gamma=`` is a finite number and ``alpha=`` (with
    ``"gaussian"`` only, required there) a finite number or the name of a call argument that holds a number or a
    one-element tensor; a CUDA tensor is read with ``float()``, one host synchronisation per call.  ``mask=``,
    ``value=``, ``nvec=``, ``epsilon=``, ``taken=`` and ``action=`` are refused, and these options with every other
    output.
    ``output="dqn_target"`` is the Bellman target of DQN and Double DQN (forward only): the callable is ``(next_obs, w1,
    b1, w2, b2, w3, b3, ...)``, the target Q-network, and each rank returns the fp32 ``y`` of its rows, ``reward + gamma
    * (1 - done) * q``.  ``online=`` names the online Q-network's six arguments (three without ``bias=True``) for Double
    DQN, which picks the greedy next action with the online network; without it the target network picks it (DQN).
    ``mask=`` names the bool ``[M, d_out]`` legal actions of the next states, which mask the ranking only: ``q`` is the
    target network's unmasked Q-value at the chosen action, so a terminal row with no legal action gets ``y = reward``
    at ``done = 1``.  ``reward=``, ``done=`` and ``gamma=`` as with ``"td_target"``.  Every other option is refused,
    and ``online=`` with every other output.

    The "gae" op is generalized advantage estimation, PPO's learner target: the callable is ``(rewards, values, dones,
    last_values, ...)`` with fp32 ``[N, T]`` rewards, values and dones in env-major layout (row i is environment i's
    trajectory, column t its step t) and fp32 ``[N]`` last_values, V(s_T), all CUDA tensors on the root GPU.  Each rank
    returns ``(advantages, returns)`` of its rows, ``x.chunk(WORLD_SIZE)[RANK]``: the backward loop ``delta = r[:, t] +
    gamma * next_v * (1 - d[:, t]) - v[:, t]``, ``acc = delta + gamma * lam * (1 - d[:, t]) * acc``, ``adv[:, t] =
    acc``, returns ``adv + values``, bit for bit as torch computes it in that order.  ``dones[:, t]`` is the done flag of
    transition t: the episode ended after the action at step t.  CleanRL's ``dones[t]`` (and SB3's
    ``episode_starts[t]``) say that observation t starts an episode, so their transition-t flag is ``dones[t + 1]``, or
    ``next_done`` at the last step: from time-major CleanRL buffers, ``torch.cat([dones[1:], next_done[None]]).T
    .contiguous()``.  For truncated episodes add ``gamma * V(final_obs)`` to the reward, as SB3 does.  ``gamma=`` and
    ``lam=`` are required, each a finite number or the name of a call argument that holds one (checked per call);
    ``self_check=False`` skips the deployment's check of a constant γ and λ against the body.  Every other option is
    refused.

    The "vtrace" op is V-trace, IMPALA's off-policy learner target: the callable is ``(log_rhos, rewards, values, dones,
    bootstrap_value, ...)`` with fp32 ``[N, T]`` log_rhos, rewards, values and dones in the env-major layout of "gae"
    and fp32 ``[N]`` bootstrap_value, V(s_T), all CUDA tensors on the root GPU.  Each rank returns ``(vs,
    pg_advantages)`` of its rows, ``x.chunk(WORLD_SIZE)[RANK]``: TorchBeast's ``from_importance_weights`` with
    ``discounts = gamma * (1 - dones)``, ``rhos = exp(log_rhos)`` clipped at ``rho_bar`` in the TD errors, ``lam *
    clamp(rhos, max=c_bar)`` as the traces and ``clamp(rhos, max=pg_rho_bar)`` in the advantages, bit for bit as torch
    computes it on the GPU (tests/policy_vtrace_cases.py).  ``dones[:, t]`` is the done flag of transition t, which is
    TorchBeast's ``batch["done"][1:]``.  From TorchBeast's time-major ``[T, B]`` tensors pass ``x.T.contiguous()`` and
    ``bootstrap_value = baseline[-1]``; from the evaluate head, ``log_rhos = (target_lp - behaviour_lp).view(N, T)``
    with ``behaviour_lp`` the log-probabilities of ``output="sample"`` (or ``"gaussian"``) at rollout and ``target_lp``
    those of ``output="evaluate"`` (or ``"gaussian_evaluate"``) under the learner's weights.  ``gamma=`` is required and
    ``lam=`` (seed_rl's ``lambda_``) defaults to 1.0, each a finite number or the name of a call argument that holds one
    (checked per call); ``rho_bar=``, ``c_bar=`` and ``pg_rho_bar=`` are constants, a number > 0 or None for no clip,
    each 1.0 by default (TorchBeast clamps the traces at 1.0 whatever ``c_bar``: declare ``c_bar=1.0`` for its bits).
    ``self_check=False`` skips the deployment's check of constant options against the body.  Every other option is
    refused.

    The "nstep" op is the n-step bootstrapped return of Ape-X, R2D2, Rainbow and A3C: the callable is ``(rewards,
    values, dones, baseline, last_values, ...)`` with fp32 ``[N, T]`` rewards, values, dones and baseline in the
    env-major layout of "gae" and fp32 ``[N]`` last_values, V(s_T), all CUDA tensors on the root GPU.  Each rank
    returns ``(returns, td)`` of its rows, ``x.chunk(WORLD_SIZE)[RANK]``: ``G_t = r_t + γ r_{t+1} + … + γ^{n−1}
    r_{t+n−1} + γ^n values[:, t + n]`` with ``γ(1 − dones)`` as each step's discount, so the sum is cut at episode
    ends, and past the rollout's end padded with reward 0, discount 1 and ``last_values``; ``td = G − baseline``.  It
    is rlax's ``n_step_bootstrapped_returns`` at ``lambda_t = 1`` made env-major, bit for bit as torch computes the
    padded loop (tests/policy_nstep_cases.py).  ``values[:, t]`` is the bootstrap value of state s_t and ``baseline[:,
    t]`` what the TD error is taken against: for Ape-X's priorities ``values = q_max`` and ``baseline = q`` of
    ``output="epsilon_greedy"`` over the rollout's observations, ``.view(N, T)``; for A3C's n-step advantages ``values``
    from the value head and ``baseline = values``.  ``dones[:, t]`` is the done flag of transition t, so CleanRL-style
    episode-start flags become ``torch.cat([dones[1:], next_done[None]]).T.contiguous()`` as for "gae".  ``n=`` is a
    required int constant in [1, 32] and ``gamma=`` a required finite number or the name of a call argument that holds
    one (checked per call).  ``self_check=False`` skips the deployment's check of a constant γ against the body.  Every
    other option is refused.

    The "retrace" op is Retrace(λ) (Munos et al. 2016), the off-policy Q-value target of ACER, Reactor, MPO and Q(λ)
    agents: the callable is ``(log_rhos, rewards, q, values, dones, baseline, bootstrap_value, ...)`` with fp32 ``[N,
    T]`` log_rhos, rewards, q, values, dones and baseline in the env-major layout of "gae" and fp32 ``[N]``
    bootstrap_value, all CUDA tensors on the root GPU.  Each rank returns ``(returns, td)`` of its rows,
    ``x.chunk(WORLD_SIZE)[RANK]``: from ``g = r[:, T-1] + discounts[:, T-1] * bootstrap_value`` backwards, ``g = r[:, t]
    + discounts[:, t] * (values[:, t+1] - c[:, t+1] * q[:, t+1] + c[:, t+1] * g)`` with ``discounts = gamma * (1 -
    dones)`` and traces ``c = clamp(exp(log_rhos), max=1) * lam``, and ``td = returns - baseline``: rlax's
    ``retrace_continuous`` made env-major, bit for bit as torch computes it on the GPU (tests/policy_retrace_cases.py).
    ``log_rhos[:, t]`` is ``log π(a_t|s_t) − log μ(a_t|s_t)`` of the taken action: for stochastic policies ``(target_lp
    - behaviour_lp).view(N, T)`` with ``behaviour_lp`` from ``output="sample"`` (or ``"gaussian"``) at rollout and
    ``target_lp`` from ``output="evaluate"`` (or ``"gaussian_evaluate"``) under the target weights; for Watkins' Q(λ)
    over ε-greedy data, 0 where the taken action is the target network's greedy one and ``-inf`` elsewhere (the trace
    is cut there), and for Harutyunyan's Q(λ) 0 everywhere.  ``q`` is ``Q_target(s_t, a_t)`` and ``values`` is
    ``E_π Q_target(s_t, ·)``: for a greedy target policy, ``q_max`` of ``output="epsilon_greedy"`` at ``epsilon=0.0``
    on the target network over the rollout's N·(T + 1) observations, ``.view(N, T + 1)``, gives ``values = q_max[:,
    :T]`` and ``bootstrap_value = q_max[:, T]``; under Watkins' log-ratios ``q = values`` is exact, because ``q`` only
    enters multiplied by the trace, which is 0 wherever the taken action is not the greedy one.  ``baseline`` is what
    the TD error is taken against, ``Q_online(s_t, a_t)`` (rlax's ``q_tm1``: ``q`` of the behaviour's
    ``output="epsilon_greedy"`` on the online network), and may be ``q`` itself.  Columns 0 of log_rhos, q and values
    are never read.  ``dones[:, t]`` is the done flag of transition t; from time-major ``[T, N]`` buffers pass
    ``x.T.contiguous()``, and CleanRL-style episode-start flags become ``torch.cat([dones[1:],
    next_done[None]]).T.contiguous()`` as for "gae".  ``gamma=`` and ``lam=`` are required, each a finite number or the
    name of a call argument that holds one (checked per call); ``self_check=False`` skips the deployment's check of a
    constant γ and λ against the body.  Every other option is refused.

    The "per" op is prioritized experience replay's proportional sampler (Schaul et al. 2016; Ape-X, R2D2, Rainbow):
    the callable is ``(priorities, ...)`` with fp32 ``[C]`` priorities, the stored ``p_i^α`` of a replay buffer
    (usually its filled prefix ``prio[:size]``), a CUDA tensor on the root GPU.  Each rank returns ``(indices,
    weights)`` for its strata ``torch.arange(batch).chunk(WORLD_SIZE)[RANK]``: the body builds the sum tree of the
    priorities, each node one fp32 add of its two children over the leaves padded with +0 to a power of two, and
    stratum j descends it from the mass ``(j + u) * (total / batch)``, ``u = kubetorch_b200.sampling.replay_noise(seed,
    j, 1)``, stepping right where ``mass >= left`` and the right child is > 0; int64 ``indices`` and fp32 importance
    weights ``(p_i / total * C) ** -beta / (min p / total * C) ** -beta``, bit for bit as torch computes them on the GPU
    (tests/policy_per_cases.py).  Every index lies in [0, C), no zero-priority item is drawn while the total is
    positive and finite, and the noise depends on (seed, j) only, so every rank count draws the same batch.
    ``batch=`` is a required int constant in [1, 8192]; ``beta=`` a required number >= 0 or the name of a call
    argument that holds one (PER's annealed β), and ``seed=`` a required int in [0, 2**64) or the name of a call
    argument that holds one (a new seed for every batch).  ``self_check=False`` skips the deployment's check of the
    body.  Every other option is refused.  The priority update that follows the learner step is
    ``kubetorch_b200.device.replay.per_update(priorities, indices, td, alpha, eps)``, a device call rather than a
    mapped op: it writes the caller's tensor in place."""
    if op not in ALL_OPS:
        raise ValueError(f"unknown mapped op '{op}'; expected one of {ALL_OPS}")
    if op == "gae":
        _check_gae_options(alpha, beta, reduce, arg, extra)
    if op == "vtrace":
        _check_vtrace_options(alpha, beta, reduce, arg, extra)
    if op == "nstep":
        _check_nstep_options(alpha, beta, reduce, arg, extra)
    if op == "retrace":
        _check_retrace_options(alpha, beta, reduce, arg, extra)
    if op == "per":
        _check_per_options(alpha, beta, reduce, arg, extra)
        beta = _UNSET   # extra keeps it
    beta = 0.0 if beta is _UNSET else beta
    if op == "mlp" and extra.get("output") == "td_target" and alpha is not _UNSET:   # SAC's α, an option of the head
        extra["alpha"] = alpha
    alpha = 1.0 if alpha is _UNSET or op == "mlp" and "alpha" in extra else alpha
    if reduce not in (None, "sum"):
        raise ValueError("reduce must be None or 'sum'")
    if op in ELEMENTWISE_OPS:
        if any(k in extra for k in ("bias", "output", *MLP_FORMS)):
            raise ValueError(f"{', '.join(k + '=' for k in ('bias', 'output', *MLP_FORMS))} are options of the 'mlp' "
                             f"op, not of '{op}'")
    elif op == "mlp":
        bias = extra.get("bias", False)
        if not isinstance(bias, bool):
            raise ValueError(f"bias must be True or False, got {bias!r}")
        output = extra.get("output", "logits")
        if output not in MLP_OUTPUTS:
            raise ValueError(f"output must be one of {MLP_OUTPUTS}, got {output!r}")
        given = [k for k in extra if k in MLP_FORMS]
        row = check_mlp_options(output, extra.get("policy"), given)
        check_mlp_rules(row, output, extra.get("policy"), extra.get("log_std"), given)
        for name in given:
            form, v = MLP_FORMS[name], extra[name]
            if form == "name" and not isinstance(v, str):
                raise ValueError(f"{name} must be the name of a call argument, got {v!r}")
            if form == "names" and not (name == "log_std" and isinstance(v, str)):
                n = (6 if bias else 3) if name in ("twin", "actor", "online") else 2
                if not isinstance(v, (tuple, list)) or len(v) != n or not all(isinstance(x, str) for x in v):
                    what = "(w1, b1, w2, b2, w3, b3)" if n == 6 else "(w1, w2, w3) (bias=False)"
                    raise ValueError(f"{name} must name {_NAMES[name].format(n=n, what=what)}, got {v!r}")
            if name in CONSTANT_CHECKS and not names_arguments(name, v):
                extra[name] = CONSTANT_CHECKS[name](v)
        if not bias and "value" in extra:
            raise ValueError("value= needs bias=True: the critic's bias is given exactly when b3 is")
        if not bias and isinstance(extra.get("log_std"), (tuple, list)):
            raise ValueError("log_std=(w_ls, b_ls) needs bias=True: the log-std head's bias is given exactly when b3 is")

    def deco(fn):
        params = inspect.signature(fn).parameters
        if op == "gae" and len(params) < 4:
            raise ValueError(f"a 'gae' callable takes (rewards, values, dones, last_values, ...) positionally, "
                             f"{getattr(fn, '__name__', fn)!r} has {len(params)} parameters")
        if op == "vtrace" and len(params) < 5:
            raise ValueError(f"a 'vtrace' callable takes (log_rhos, rewards, values, dones, bootstrap_value, ...) "
                             f"positionally, {getattr(fn, '__name__', fn)!r} has {len(params)} parameters")
        if op == "nstep" and len(params) < 5:
            raise ValueError(f"a 'nstep' callable takes (rewards, values, dones, baseline, last_values, ...) "
                             f"positionally, {getattr(fn, '__name__', fn)!r} has {len(params)} parameters")
        if op == "retrace" and len(params) < 7:
            raise ValueError(f"a 'retrace' callable takes (log_rhos, rewards, q, values, dones, baseline, "
                             f"bootstrap_value, ...) positionally, {getattr(fn, '__name__', fn)!r} has {len(params)} "
                             f"parameters")
        if op == "per" and len(params) < 1:
            raise ValueError(f"a 'per' callable takes (priorities, ...) positionally, {getattr(fn, '__name__', fn)!r} "
                             f"has no parameters")
        for option, names in extra.items():
            if not (isinstance(names, str) if op in ("gae", "vtrace", "nstep", "retrace", "per")
                    else names_arguments(option, names)):
                continue
            for name in (names,) if isinstance(names, str) else names:
                if name not in params:
                    raise ValueError(f"{option}={names!r}: {name!r} is not an argument of "
                                     f"{getattr(fn, '__name__', fn)!r}")
        setattr(fn, MAPPED_ATTR, MappedSpec(op=op, alpha=alpha, beta=beta, reduce=reduce, arg=arg, extra=extra))
        return fn

    return deco


def _check_gae_options(alpha, beta, reduce, arg, extra) -> None:
    """The options of op="gae", or ValueError naming the first it does not take or the first it lacks; a constant gamma
    or lam must be a finite number (extra keeps it)."""
    refused = dict(alpha=alpha is not _UNSET, beta=beta is not _UNSET, reduce=reduce is not None, arg=arg is not None)
    refused.update((k, True) for k in extra if k not in GAE_OPTIONS + ("self_check",))
    for name, given in refused.items():
        if given:
            raise ValueError(f"{name}= is not an option of the 'gae' op, which takes gamma=, lam= and self_check=: its "
                             f"callable is (rewards, values, dones, last_values) and it returns (advantages, returns)")
    for name in GAE_OPTIONS:
        if name not in extra:
            raise ValueError(f"{name}= is required with the 'gae' op: a finite number or the name of a call argument "
                             f"that holds one")
        if not isinstance(extra[name], str):
            check_finite(name, extra[name])
    if not isinstance(extra.get("self_check", False), bool):
        raise ValueError(f"self_check must be True or False, got {extra['self_check']!r}")


def _check_vtrace_options(alpha, beta, reduce, arg, extra) -> None:
    """The options of op="vtrace", or ValueError naming the first it does not take or the first it lacks; a constant
    gamma or lam must be a finite number and each threshold a number > 0 or None.  Fills in the defaults of the options
    not given (extra keeps them)."""
    refused = dict(alpha=alpha is not _UNSET, beta=beta is not _UNSET, reduce=reduce is not None, arg=arg is not None)
    refused.update((k, True) for k in extra if k not in (*VTRACE_OPTIONS, "self_check"))
    for name, given in refused.items():
        if given:
            raise ValueError(f"{name}= is not an option of the 'vtrace' op, which takes gamma=, lam=, rho_bar=, c_bar=, "
                             f"pg_rho_bar= and self_check=: its callable is (log_rhos, rewards, values, dones, "
                             f"bootstrap_value) and it returns (vs, pg_advantages)")
    for name, default in VTRACE_OPTIONS.items():
        if name not in extra:
            if default is None:
                raise ValueError(f"{name}= is required with the 'vtrace' op: a finite number or the name of a call "
                                 f"argument that holds one")
            extra[name] = default
        elif name in VTRACE_ARGUMENTS:
            if not isinstance(extra[name], str):
                check_finite(name, extra[name])
        else:
            check_threshold(name, extra[name])
    if not isinstance(extra.get("self_check", False), bool):
        raise ValueError(f"self_check must be True or False, got {extra['self_check']!r}")


def _check_nstep_options(alpha, beta, reduce, arg, extra) -> None:
    """The options of op="nstep", or ValueError naming the first it does not take or the first it lacks; n must be an
    int constant in [1, 32] and a constant gamma a finite number (extra keeps them)."""
    refused = dict(alpha=alpha is not _UNSET, beta=beta is not _UNSET, reduce=reduce is not None, arg=arg is not None)
    refused.update((k, True) for k in extra if k not in (*NSTEP_OPTIONS, "self_check"))
    for name, given in refused.items():
        if given:
            raise ValueError(f"{name}= is not an option of the 'nstep' op, which takes n=, gamma= and self_check=: its "
                             f"callable is (rewards, values, dones, baseline, last_values) and it returns (returns, td)")
    if "n" not in extra:
        raise ValueError("n= is required with the 'nstep' op: an int constant in [1, 32]")
    n = extra["n"]
    if isinstance(n, bool) or not isinstance(n, int) or not 1 <= n <= 32:
        raise ValueError(f"n must be an int constant in [1, 32] (not the name of a call argument), got {n!r}")
    if "gamma" not in extra:
        raise ValueError("gamma= is required with the 'nstep' op: a finite number or the name of a call argument that "
                         "holds one")
    if not isinstance(extra["gamma"], str):
        check_finite("gamma", extra["gamma"])
    if not isinstance(extra.get("self_check", False), bool):
        raise ValueError(f"self_check must be True or False, got {extra['self_check']!r}")


def _check_retrace_options(alpha, beta, reduce, arg, extra) -> None:
    """The options of op="retrace", or ValueError naming the first it does not take or the first it lacks; a constant
    gamma or lam must be a finite number (extra keeps it)."""
    refused = dict(alpha=alpha is not _UNSET, beta=beta is not _UNSET, reduce=reduce is not None, arg=arg is not None)
    refused.update((k, True) for k in extra if k not in RETRACE_OPTIONS + ("self_check",))
    for name, given in refused.items():
        if given:
            raise ValueError(f"{name}= is not an option of the 'retrace' op, which takes gamma=, lam= and self_check=: "
                             f"its callable is (log_rhos, rewards, q, values, dones, baseline, bootstrap_value) and it "
                             f"returns (returns, td)")
    for name in RETRACE_OPTIONS:
        if name not in extra:
            raise ValueError(f"{name}= is required with the 'retrace' op: a finite number or the name of a call "
                             f"argument that holds one")
        if not isinstance(extra[name], str):
            check_finite(name, extra[name])
    if not isinstance(extra.get("self_check", False), bool):
        raise ValueError(f"self_check must be True or False, got {extra['self_check']!r}")


def _check_per_options(alpha, beta, reduce, arg, extra) -> None:
    """The options of op="per", or ValueError naming the first it does not take or the first it lacks: batch an int
    constant in [1, 8192], a constant beta a finite number >= 0 and a constant seed an int in [0, 2**64).  Moves beta
    into extra, which keeps every option."""
    refused = dict(alpha=alpha is not _UNSET, reduce=reduce is not None, arg=arg is not None)
    refused.update((k, True) for k in extra if k not in PER_OPTIONS + ("self_check",))
    for name, given in refused.items():
        if given:
            raise ValueError(f"{name}= is not an option of the 'per' op, which takes batch=, beta=, seed= and "
                             f"self_check=: its callable is (priorities, ...) and it returns (indices, weights)")
    if beta is not _UNSET:
        extra["beta"] = beta
    for name in PER_OPTIONS:
        if name not in extra:
            raise ValueError(f"{name}= is required with the 'per' op: " + (
                "an int constant in [1, 8192]" if name == "batch" else "a constant or the name of a call argument"))
    n = extra["batch"]
    if isinstance(n, bool) or not isinstance(n, int) or not 1 <= n <= 8192:
        raise ValueError(f"batch must be an int constant in [1, 8192] (not the name of a call argument), got {n!r}")
    if not isinstance(extra["beta"], str):
        check_beta(extra["beta"])
    if not isinstance(extra["seed"], str):
        _check_seed(extra["seed"])
    if not isinstance(extra.get("self_check", False), bool):
        raise ValueError(f"self_check must be True or False, got {extra['self_check']!r}")


def check_beta(v):
    """PER's β: a finite number (not a bool) >= 0."""
    check_finite("beta", v)
    if not v >= 0:
        raise ValueError(f"beta must be >= 0, got {v!r}")
    return v


def check_threshold(name: str, v):
    """rho_bar, c_bar or pg_rho_bar of V-trace: a number (not a bool) > 0, or None for no clip."""
    if v is not None and (isinstance(v, bool) or not isinstance(v, (int, float)) or not v > 0):
        raise ValueError(f"{name} must be a number > 0 or None (no clip), got {v!r}")
    return v


def names_arguments(option: str, v) -> bool:
    """Whether the value v of an MLP option names call arguments (one name, or the tuple of a "names" option) rather
    than being a constant."""
    form = MLP_FORMS.get(option, "constant")
    return form == "names" or form != "constant" and isinstance(v, str)


def check_nvec(nvec, d_out: Optional[int] = None) -> tuple:
    """nvec as a tuple, or ValueError naming what is wrong with it: not a tuple or list of ints (bools refused); empty;
    an entry below 1; (with d_out) a sum other than d_out."""
    if not isinstance(nvec, (tuple, list)) or not all(isinstance(n, int) and not isinstance(n, bool) for n in nvec):
        raise ValueError(f"nvec must be a tuple of ints, got {nvec!r}")
    if len(nvec) == 0:
        raise ValueError("nvec is empty: a multi-discrete action space has at least one group")
    if any(n < 1 for n in nvec):
        raise ValueError(f"every entry of nvec must be >= 1 (a group of at least one action), got {tuple(nvec)}")
    if d_out is not None and sum(nvec) != d_out:
        raise ValueError(f"nvec sums to {sum(nvec)}, not d_out={d_out}: its groups tile the head's columns")
    return tuple(nvec)


def mapped_spec(fn) -> Optional[MappedSpec]:
    return getattr(fn, MAPPED_ATTR, None)
