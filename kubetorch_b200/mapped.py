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
MLP_OUTPUTS = ("logits", "actions", "both", "sample", "gaussian")   # also device.mlp.OUTPUTS


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


def mapped(op: str, alpha: Any = 1.0, beta: Any = 0.0, reduce: Optional[str] = None, arg: str = None, **extra):
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
    argument that holds the fp32 [d_out] log standard deviation."""
    if op not in ALL_OPS:
        raise ValueError(f"unknown mapped op '{op}'; expected one of {ALL_OPS}")
    if reduce not in (None, "sum"):
        raise ValueError("reduce must be None or 'sum'")
    if "bias" in extra or "output" in extra or "seed" in extra or "log_std" in extra:
        if op != "mlp":
            raise ValueError(f"bias=, output=, seed= and log_std= are options of the 'mlp' op, not of '{op}'")
        if not isinstance(extra.get("bias", False), bool):
            raise ValueError(f"bias must be True or False, got {extra['bias']!r}")
        if extra.get("output", "logits") not in MLP_OUTPUTS:
            raise ValueError(f"output must be one of {MLP_OUTPUTS}, got {extra['output']!r}")
        sample = extra.get("output") in ("sample", "gaussian")
        if sample != ("seed" in extra):
            raise ValueError('seed= is required with output="sample" or "gaussian" and is an option of those only')
        if sample and not isinstance(extra["seed"], str):
            from .sampling import _check_seed

            _check_seed(extra["seed"])
        gaussian = extra.get("output") == "gaussian"
        if gaussian != ("log_std" in extra):
            raise ValueError('log_std= is required with output="gaussian" and is an option of that output only')
        if gaussian and not isinstance(extra["log_std"], str):
            raise ValueError(f"log_std must be the name of a call argument, got {extra['log_std']!r}")

    def deco(fn):
        name = extra.get("log_std")
        if name is not None and name not in inspect.signature(fn).parameters:
            raise ValueError(f"log_std={name!r} is not an argument of {getattr(fn, '__name__', fn)!r}")
        setattr(fn, MAPPED_ATTR, MappedSpec(op=op, alpha=alpha, beta=beta, reduce=reduce, arg=arg, extra=extra))
        return fn

    return deco


def mapped_spec(fn) -> Optional[MappedSpec]:
    return getattr(fn, MAPPED_ATTR, None)
