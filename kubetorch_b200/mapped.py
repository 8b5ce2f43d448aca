"""Registry of *mapped callables*: user functions whose body is one of the closed set of ops that
libktb200 executes as sm_90a kernels (identity / scale / affine, their sum-reduced forms, and the
bf16 MLP policy).

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
from dataclasses import dataclass, field
from typing import Any, Callable, Dict, Optional

MAPPED_ATTR = "__ktb_mapped__"
ELEMENTWISE_OPS = ("identity", "scale", "affine")
ALL_OPS = ELEMENTWISE_OPS + ("mlp",)
MLP_OUTPUTS = ("logits", "actions", "both", "sample", "gaussian", "epsilon_greedy", "evaluate",
               "gaussian_evaluate", "deterministic", "critic", "td_target")   # also device.mlp.OUTPUTS
EVALUATE_OUTPUTS = ("evaluate", "gaussian_evaluate")
TD_OPTIONS = ("actor", "policy", "reward", "done", "gamma", "alpha")   # the options of output="td_target" alone


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


def mapped(op: str, alpha: Any = _UNSET, beta: Any = 0.0, reduce: Optional[str] = None, arg: str = None, **extra):
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
    output."""
    if op not in ALL_OPS:
        raise ValueError(f"unknown mapped op '{op}'; expected one of {ALL_OPS}")
    if op == "mlp" and extra.get("output") == "td_target" and alpha is not _UNSET:   # SAC's α, an option of the head
        extra["alpha"] = alpha
    alpha = 1.0 if alpha is _UNSET or op == "mlp" and "alpha" in extra else alpha
    if reduce not in (None, "sum"):
        raise ValueError("reduce must be None or 'sum'")
    if op != "mlp" and any(k in extra for k in ("action", "twin")):
        raise ValueError(f"action= and twin= are options of the 'mlp' op, not of '{op}'")
    if op != "mlp" and any(k in extra for k in TD_OPTIONS):
        raise ValueError(f"actor=, policy=, reward=, done=, gamma= and alpha= are options of the 'mlp' op, not of "
                         f"'{op}'")
    if any(k in extra for k in ("bias", "output", "seed", "log_std", "mask", "value", "nvec", "log_std_bounds",
                                "squash", "epsilon", "taken", "noise", "noise_clip", "action", "twin")):
        if op != "mlp":
            raise ValueError(f"bias=, output=, seed=, log_std=, log_std_bounds=, squash=, mask=, value=, nvec=, "
                             f"epsilon=, taken=, noise= and noise_clip= are options of the 'mlp' op, not of '{op}'")
        if not isinstance(extra.get("bias", False), bool):
            raise ValueError(f"bias must be True or False, got {extra['bias']!r}")
        if extra.get("output", "logits") not in MLP_OUTPUTS:
            raise ValueError(f"output must be one of {MLP_OUTPUTS}, got {extra['output']!r}")
        if extra.get("output") == "td_target":
            _check_td_target(extra)
        elif any(k in extra for k in TD_OPTIONS):
            raise ValueError(f'actor=, policy=, reward=, done=, gamma= and alpha= are options of output="td_target", '
                             f'not of output={extra.get("output", "logits")!r}')
        else:
            if extra.get("output") == "critic":
                _check_critic(extra)
            elif "action" in extra or "twin" in extra:
                raise ValueError(f'action= and twin= are options of output="critic", not of '
                                 f'output={extra.get("output", "logits")!r}')
            sample = extra.get("output") in ("sample", "gaussian")
            eps = extra.get("output") == "epsilon_greedy"
            det = extra.get("output") == "deterministic"
            if det:
                _check_deterministic(extra)
            elif "noise" in extra or "noise_clip" in extra:
                raise ValueError(f'noise= and noise_clip= are options of output="deterministic", not of '
                                 f'output={extra.get("output", "logits")!r}')
            evaluate = extra.get("output") in EVALUATE_OUTPUTS
            if evaluate != ("taken" in extra):
                raise ValueError('taken= is required with output="evaluate" and "gaussian_evaluate" and is an option of '
                                 'those outputs only')
            if evaluate and not isinstance(extra["taken"], str):
                raise ValueError(f"taken must be the name of a call argument, got {extra['taken']!r}")
            if evaluate and "seed" in extra:
                raise ValueError(f'seed= is not an option of output={extra["output"]!r}: evaluating given actions draws '
                                 f'no noise')
            if not det and (sample or eps) != ("seed" in extra):
                raise ValueError('seed= is required with output="sample" or "gaussian" (or "epsilon_greedy") and is an '
                                 'option of those only')
            if (sample or eps or det) and "seed" in extra and not isinstance(extra["seed"], str):
                from .sampling import _check_seed

                _check_seed(extra["seed"])
            gaussian = extra.get("output") in ("gaussian", "gaussian_evaluate")
            if gaussian != ("log_std" in extra):
                raise ValueError('log_std= is required with output="gaussian" (and "gaussian_evaluate") and is an option of '
                                 'those outputs only')
            state = gaussian and isinstance(extra["log_std"], (tuple, list))
            if state and evaluate:
                raise ValueError('output="gaussian_evaluate" takes a state-independent log_std (the name of one call '
                                 'argument), not a log_std=(w_ls, b_ls) pair')
            if state:
                ls = extra["log_std"]
                if len(ls) != 2 or not all(isinstance(n, str) for n in ls):
                    raise ValueError(f"log_std must name one call argument or two (w_ls, b_ls), got {ls!r}")
                if not extra.get("bias", False):
                    raise ValueError("log_std=(w_ls, b_ls) needs bias=True: the log-std head's bias is given exactly when "
                                     "b3 is")
            elif gaussian and not isinstance(extra["log_std"], str):
                raise ValueError(f"log_std must be the name of a call argument, got {extra['log_std']!r}")
            if not state and ("log_std_bounds" in extra or "squash" in extra and not det):
                raise ValueError("log_std_bounds= and squash= are options of a state-dependent log_std=(w_ls, b_ls) only")
            if "log_std_bounds" in extra:
                lb = extra["log_std_bounds"]
                if not isinstance(lb, (tuple, list)) or len(lb) != 2 or \
                        not all(isinstance(b, (int, float)) and not isinstance(b, bool) for b in lb):
                    raise ValueError(f"log_std_bounds must be (low, high), two numbers, got {lb!r}")
                if lb[0] != lb[0] or lb[1] != lb[1]:
                    raise ValueError(f"log_std_bounds must not be NaN, got {lb!r}")
                if lb[0] > lb[1]:
                    raise ValueError(f"log_std_bounds must have low <= high, got {lb!r}")
                extra["log_std_bounds"] = (float(lb[0]), float(lb[1]))
            if "squash" in extra and not isinstance(extra["squash"], bool):
                raise ValueError(f"squash must be True or False, got {extra['squash']!r}")
            if "mask" in extra:
                if gaussian:
                    raise ValueError(f'mask= is an option of the categorical outputs, not of output={extra["output"]!r}')
                if not isinstance(extra["mask"], str):
                    raise ValueError(f"mask must be the name of a call argument, got {extra['mask']!r}")
            if "value" in extra:
                if not (sample or evaluate):
                    raise ValueError('value= is an option of output="sample", "gaussian", "evaluate" and '
                                     '"gaussian_evaluate" only')
                if not extra.get("bias", False):
                    raise ValueError("value= needs bias=True: the critic's bias is given exactly when b3 is")
                v = extra["value"]
                if not isinstance(v, (tuple, list)) or len(v) != 2 or not all(isinstance(n, str) for n in v):
                    raise ValueError(f"value must name two call arguments (wv, bv), got {v!r}")
            if "nvec" in extra:
                extra["nvec"] = check_nvec(extra["nvec"], extra.get("output", "logits"))
            if eps != ("epsilon" in extra):
                raise ValueError('epsilon= is required with output="epsilon_greedy" and is an option of that output only')
            if eps and not isinstance(extra["epsilon"], str):
                e = extra["epsilon"]
                if isinstance(e, bool) or not isinstance(e, (int, float)):
                    raise ValueError(f"epsilon must be a number or the name of a call argument, got {e!r}")
                if e != e:
                    raise ValueError("epsilon must not be NaN (a NaN never explores: pass 0.0 for that)")

    def deco(fn):
        params = inspect.signature(fn).parameters
        for option in ("log_std", "mask", "value", "epsilon", "taken", "noise", "action", "twin", "actor", "reward",
                       "done", "alpha"):
            names = extra.get(option)
            if option in ("epsilon", "noise", "alpha") and not isinstance(names, str):   # a constant names no argument
                continue
            for name in (names,) if isinstance(names, str) or names is None else names:
                if name is not None and name not in params:
                    raise ValueError(f"{option}={names!r}: {name!r} is not an argument of "
                                     f"{getattr(fn, '__name__', fn)!r}")
        setattr(fn, MAPPED_ATTR, MappedSpec(op=op, alpha=alpha, beta=beta, reduce=reduce, arg=arg, extra=extra))
        return fn

    return deco


def _check_deterministic(extra) -> None:
    """mapped()'s checks of output="deterministic", in this order: the options it refuses, seed= given exactly when
    noise= is, noise (a number that is not NaN and >= 0, or the name of a call argument), noise_clip (with noise= only;
    a number that is not NaN and >= 0)."""
    for name in ("mask", "value", "nvec", "log_std", "log_std_bounds", "epsilon", "taken"):
        if name in extra:
            raise ValueError(f'{name}= is not an option of output="deterministic": the deterministic actor takes '
                             f'noise=, noise_clip=, seed= and squash= only')
    if ("noise" in extra) != ("seed" in extra):
        raise ValueError('output="deterministic" takes seed= exactly when it takes noise=: the noise-free actor draws '
                         'nothing')
    if "noise_clip" in extra and "noise" not in extra:
        raise ValueError("noise_clip= is an option of noise= only: it clips the noise")
    for name in ("noise", "noise_clip"):
        v = extra.get(name)
        if v is None or name == "noise" and isinstance(v, str):
            continue
        if isinstance(v, bool) or not isinstance(v, (int, float)):
            what = "a number or the name of a call argument" if name == "noise" else "a number"
            raise ValueError(f"{name} must be {what}, got {v!r}")
        if v != v or v < 0:
            raise ValueError(f"{name} must be >= 0 and not NaN, got {v!r}")


def _check_critic(extra) -> None:
    """mapped()'s checks of output="critic", in this order: the options it refuses, action= (required, the name of a
    call argument), twin= (the names of six call arguments with bias=True, three without)."""
    for name in ("seed", "mask", "value", "nvec", "log_std", "log_std_bounds", "squash", "epsilon", "taken", "noise",
                 "noise_clip"):
        if name in extra:
            raise ValueError(f'{name}= is not an option of output="critic": a critic evaluates Q(s, a) of the given '
                             f'action and takes action= and twin= only')
    if not isinstance(extra.get("action"), str):
        raise ValueError(f'action= is required with output="critic" and must name the call argument that holds the '
                         f'actions, got {extra.get("action")!r}')
    if "twin" in extra:
        n = 6 if extra.get("bias", False) else 3
        t = extra["twin"]
        if not isinstance(t, (tuple, list)) or len(t) != n or not all(isinstance(x, str) for x in t):
            what = "(w1, b1, w2, b2, w3, b3)" if n == 6 else "(w1, w2, w3) (bias=False)"
            raise ValueError(f"twin must name the second critic's {n} call arguments {what}, got {t!r}")


def _check_td_target(extra) -> None:
    """mapped()'s checks of output="td_target", in this order: the options it refuses, policy=, the policy's options
    (noise=, noise_clip= and seed= as output="deterministic" takes them, refusing log_std=, log_std_bounds= and alpha=;
    or seed=, alpha=, log_std=(w_ls, b_ls) with bias=True, log_std_bounds= and squash=, refusing noise= and
    noise_clip=), actor= (six names with bias=True, three without), twin= as output="critic" takes it, reward= and
    done= (names), gamma= (a finite number)."""
    for name in ("mask", "value", "nvec", "epsilon", "taken", "action"):
        if name in extra:
            raise ValueError(f'{name}= is not an option of output="td_target": a TD target takes actor=, policy= and '
                             f'its options, twin=, reward=, done=, gamma= and alpha= only')
    policy = extra.get("policy")
    if policy not in ("deterministic", "gaussian"):
        raise ValueError(f'policy= must be "deterministic" or "gaussian" with output="td_target", got {policy!r}')
    if policy == "deterministic":
        for name in ("log_std", "log_std_bounds", "alpha"):
            if name in extra:
                raise ValueError(f'{name}= is not an option of policy="deterministic": TD3 and DDPG targets take '
                                 f'noise=, noise_clip=, seed= and squash=, and no entropy term')
        _check_deterministic(extra)
        if "seed" in extra and not isinstance(extra["seed"], str):
            from .sampling import _check_seed

            _check_seed(extra["seed"])
    else:
        for name in ("noise", "noise_clip"):
            if name in extra:
                raise ValueError(f'{name}= is not an option of policy="gaussian": SAC\'s next actions are sampled with '
                                 f'the log-std head')
        if "seed" not in extra:
            raise ValueError('seed= is required with policy="gaussian"')
        if not isinstance(extra["seed"], str):
            from .sampling import _check_seed

            _check_seed(extra["seed"])
        a = extra.get("alpha")
        if a is None:
            raise ValueError('alpha= is required with policy="gaussian": a number or the name of a call argument')
        if not isinstance(a, str) and (isinstance(a, bool) or not isinstance(a, (int, float)) or a != a
                                       or a in (float("inf"), float("-inf"))):
            raise ValueError(f"alpha must be a finite number or the name of a call argument, got {a!r}")
        ls = extra.get("log_std")
        if not isinstance(ls, (tuple, list)) or len(ls) != 2 or not all(isinstance(n, str) for n in ls):
            raise ValueError(f'log_std= must name the two call arguments (w_ls, b_ls) of the actor\'s log-std head '
                             f'with policy="gaussian", got {ls!r}')
        if not extra.get("bias", False):
            raise ValueError("log_std=(w_ls, b_ls) needs bias=True: the log-std head's bias is given exactly when b3 is")
        if "log_std_bounds" in extra:
            lb = extra["log_std_bounds"]
            if not isinstance(lb, (tuple, list)) or len(lb) != 2 or \
                    not all(isinstance(b, (int, float)) and not isinstance(b, bool) for b in lb) or \
                    lb[0] != lb[0] or lb[1] != lb[1] or lb[0] > lb[1]:
                raise ValueError(f"log_std_bounds must be (low, high), two numbers, not NaN, low <= high, got {lb!r}")
            extra["log_std_bounds"] = (float(lb[0]), float(lb[1]))
    if "squash" in extra and not isinstance(extra["squash"], bool):
        raise ValueError(f"squash must be True or False, got {extra['squash']!r}")
    n = 6 if extra.get("bias", False) else 3
    for option in ("actor", "twin"):
        if option not in extra and option == "twin":
            continue
        t = extra.get(option)
        if not isinstance(t, (tuple, list)) or len(t) != n or not all(isinstance(x, str) for x in t):
            what = "(w1, b1, w2, b2, w3, b3)" if n == 6 else "(w1, w2, w3) (bias=False)"
            whose = "the actor's" if option == "actor" else "the second critic's"
            raise ValueError(f"{option} must name {whose} {n} call arguments {what}, got {t!r}")
    for option in ("reward", "done"):
        if not isinstance(extra.get(option), str):
            raise ValueError(f'{option}= is required with output="td_target" and must name a call argument, got '
                             f'{extra.get(option)!r}')
    g = extra.get("gamma")
    if isinstance(g, bool) or not isinstance(g, (int, float)) or g != g or g in (float("inf"), float("-inf")):
        raise ValueError(f'gamma= is required with output="td_target" and must be a finite number, got {g!r}')


def check_nvec(nvec, output: str, d_out: Optional[int] = None) -> tuple:
    """nvec as a tuple, or ValueError naming what is wrong with it: given with an output other than "actions", "both",
    "sample" and "evaluate"; not a tuple or list of ints (bools refused); empty; an entry below 1; (with d_out) a sum
    other than d_out."""
    if output not in ("actions", "both", "sample", "evaluate"):
        raise ValueError(f'nvec is an option of output="actions", "both", "sample" and "evaluate", not of '
                         f'output={output!r}')
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
