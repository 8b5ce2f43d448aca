"""The options of every MLP output without a GPU: kt.mapped() and _check_policy refuse each option an output does not
take and report each required option left out, naming the option and the output; and the supervisor resolves a
mapped "mlp" callable's named options to the arguments of one mlp_scatter_gather call."""
from types import SimpleNamespace
from unittest import mock

import pytest
import torch

import kubetorch_b200 as kt
from kubetorch_b200.device import mlp
from kubetorch_b200.mapped import mapped_spec
from kubetorch_b200.serving.b200_supervisor import B200Supervisor

# output (a TD target with its policy) -> the options it takes beside bias= and output=; * marks a required one
TAKES = {
    "logits": "mask",
    "actions": "mask nvec",
    "both": "mask nvec",
    "sample": "seed* mask value nvec",
    "gaussian": "seed* log_std* value log_std_bounds squash",
    "epsilon_greedy": "seed* epsilon* mask",
    "evaluate": "taken* mask value nvec",
    "gaussian_evaluate": "taken* log_std* value",
    "deterministic": "noise noise_clip seed squash",
    "critic": "action* twin",
    ("td_target", "deterministic"): "actor* policy* reward* done* gamma* twin noise noise_clip seed squash",
    ("td_target", "gaussian"): "actor* policy* reward* done* gamma* twin seed* alpha* log_std* log_std_bounds squash",
}
OPTIONS = ("seed", "log_std", "mask", "value", "nvec", "log_std_bounds", "squash", "epsilon", "taken", "noise",
           "noise_clip", "action", "twin", "actor", "policy", "reward", "done", "gamma", "alpha")
TD = ("actor", "policy", "reward", "done", "gamma", "alpha")

# a well-formed decoration of every option, each name an argument of _body
DECO = dict(seed=1, log_std="ls", mask="m", value=("wv", "bv"), nvec=(2, 2), log_std_bounds=(-5.0, 2.0), squash=True,
            epsilon=0.1, taken="t", noise=0.1, noise_clip=0.5, action="a", twin=("t1", "tb1", "t2", "tb2", "t3", "tb3"),
            actor=("a1", "ab1", "a2", "ab2", "a3", "ab3"), reward="r", done="d", gamma=0.99, alpha=0.2)
PARAMS = ("obs", "w1", "b1", "w2", "b2", "w3", "b3", "ls", "wls", "bls", "m", "wv", "bv", "t", "a", "t1", "tb1", "t2",
          "tb2", "t3", "tb3", "a1", "ab1", "a2", "ab2", "a3", "ab3", "r", "d", "seed", "eps", "sigma", "temp")


def _body(*params):
    ns = {}
    exec(f"def body({', '.join(params)}):\n    pass", ns)
    return ns["body"]


def _key(key):
    return key if isinstance(key, tuple) else (key, None)


def _takes(key):
    return {o.rstrip("*") for o in TAKES[key].split()}


def _required(key):
    return [o.rstrip("*") for o in TAKES[key].split() if o.endswith("*")]


def _where(key):
    output, policy = _key(key)
    return f'output="{output}"'


def _minimal(key):
    """The required options of `key` as mapped() takes them (bias=True: a log-std pair needs it)."""
    output, policy = _key(key)
    opts = {o: DECO[o] for o in _required(key) if o != "policy"}
    if policy is not None:
        opts["policy"] = policy
    if key == ("td_target", "gaussian"):
        opts["log_std"] = ("wls", "bls")
    return dict(bias=True, output=output, **opts)


def _decorate(**opts):
    return kt.mapped("mlp", **opts)(_body(*PARAMS))


def _device(output, opts):
    """_check_policy with CPU stand-ins: the option checks come before any tensor is looked at."""
    opts = dict(opts)
    td = tuple(opts.pop(k, None) for k in TD)
    w1, w3 = torch.zeros(64, 32, dtype=torch.bfloat16), torch.zeros(4, 64, dtype=torch.bfloat16)
    mlp._check_policy(w1, w3, (None,) * 3, output, td=td, **opts)


def _device_minimal(key):
    output, policy = _key(key)
    return {o: (policy if o == "policy" else 1) for o in _required(key)}


REFUSED = [(key, o) for key in TAKES for o in OPTIONS if o not in _takes(key)]


@pytest.mark.parametrize("key,option", REFUSED, ids=[f"{_key(k)[0]}-{_key(k)[1]}-{o}" for k, o in REFUSED])
def test_mapped_refuses_an_option_the_output_does_not_take(key, option):
    if option == "alpha" and _key(key)[0] != "td_target":
        pytest.skip("mapped()'s alpha= is the element-wise ops' scale with every output but td_target")
    opts = _minimal(key)
    opts[option] = "deterministic" if option == "policy" else DECO[option]
    with pytest.raises(ValueError) as e:
        _decorate(**opts)
    assert f"{option}=" in str(e.value) and _where(key) in str(e.value), str(e.value)


@pytest.mark.parametrize("key,option", REFUSED, ids=[f"{_key(k)[0]}-{_key(k)[1]}-{o}" for k, o in REFUSED])
def test_check_policy_refuses_an_argument_the_output_does_not_take(key, option):
    opts = _device_minimal(key)
    opts[option] = "deterministic" if option == "policy" else 1
    with pytest.raises(ValueError) as e:
        _device(_key(key)[0], opts)
    assert option in str(e.value) and _where(key) in str(e.value), str(e.value)


def test_check_policy_refuses_a_seed_with_the_greedy_outputs():
    for output in ("logits", "actions", "both"):
        with pytest.raises(ValueError, match=f'seed is not an argument of output="{output}"'):
            _device(output, dict(seed=5))


MISSING = [(key, o) for key in TAKES for o in _required(key)]


@pytest.mark.parametrize("key,option", MISSING, ids=[f"{_key(k)[0]}-{_key(k)[1]}-{o}" for k, o in MISSING])
def test_mapped_reports_a_missing_required_option(key, option):
    opts = _minimal(key)
    del opts[option]
    with pytest.raises(ValueError) as e:
        _decorate(**opts)
    assert f"{option}= is required with {_where(key)}" in str(e.value), str(e.value)


@pytest.mark.parametrize("key,option", MISSING, ids=[f"{_key(k)[0]}-{_key(k)[1]}-{o}" for k, o in MISSING])
def test_check_policy_reports_a_missing_required_argument(key, option):
    opts = _device_minimal(key)
    del opts[option]
    with pytest.raises(ValueError) as e:
        _device(_key(key)[0], opts)
    assert f"{option} is required with {_where(key)}" in str(e.value), str(e.value)


@pytest.mark.parametrize("key", list(TAKES), ids=[f"{_key(k)[0]}-{_key(k)[1]}" for k in TAKES])
def test_mapped_accepts_the_minimal_spec_of_every_output(key):
    _decorate(**_minimal(key))


# ---- the supervisor's resolution of named options -----------------------------------------------------------------
CALL_OPTIONS = ("seed", "log_std", "mask", "value", "nvec", "log_std_bounds", "squash", "epsilon", "taken", "noise",
                "noise_clip", "action", "twin")


class _Stub:
    """A stand-in for a call argument, compared by identity."""

    def __init__(self, name):
        self.name = name

    def __repr__(self):
        return f"<{self.name}>"


def _call(spec_kw, params):
    """(args, kwargs) that B200Supervisor._call_mlp passes to mlp_scatter_gather for a callable of `params` decorated
    with kt.mapped("mlp", **spec_kw), called with one stub per parameter."""
    fn = kt.mapped("mlp", **spec_kw)(_body(*params))
    spec = mapped_spec(fn)
    values = {p: _Stub(p) for p in params}
    _, _, _, bound = spec.bind(fn, tuple(values[p] for p in params), {})
    me = SimpleNamespace(devices=[0, 1], transfer="auto", ops=SimpleNamespace(PushTimeout=TimeoutError),
                         _all_ranks=lambda ranks: True)
    with mock.patch.object(mlp, "mlp_scatter_gather", return_value=["r0", "r1"]) as sg:
        assert B200Supervisor._call_mlp(me, spec, bound) == ["r0", "r1"]
    (args, kwargs), = [(c.args, c.kwargs) for c in sg.call_args_list]
    return values, args, kwargs


def _want(v, output, bias=True, **named):
    """The keyword arguments of mlp_scatter_gather: every option None unless given."""
    kw = dict(devices=[0, 1], transfer="auto", output=output,
              biases=(v["b1"], v["b2"], v["b3"]) if bias else (None, None, None), **dict.fromkeys(CALL_OPTIONS))
    kw.update(named)
    return kw


BIASED = ("obs", "w1", "b1", "w2", "b2", "w3", "b3")
PLAIN = ("obs", "w1", "w2", "w3")


def _check_call(spec_kw, params, want):
    v, args, kwargs = _call(spec_kw, params)
    assert args == (v["obs"], v["w1"], v["w2"], v["w3"])
    assert kwargs == want(v), (kwargs, want(v))


CALLS = {
    "logits": (dict(), PLAIN, lambda v: _want(v, "logits", bias=False)),
    "logits-bias-mask": (dict(bias=True, mask="m"), BIASED + ("m",), lambda v: _want(v, "logits", mask=v["m"])),
    "actions-nvec": (dict(output="actions", nvec=[2, 2]), PLAIN,
                     lambda v: _want(v, "actions", bias=False, nvec=(2, 2))),
    "both": (dict(bias=True, output="both"), BIASED, lambda v: _want(v, "both")),
    "sample-named-seed": (dict(bias=True, output="sample", seed="seed", value=("wv", "bv"), mask="m"),
                          BIASED + ("m", "wv", "bv", "seed"),
                          lambda v: _want(v, "sample", seed=v["seed"], value=(v["wv"], v["bv"]), mask=v["m"])),
    "gaussian": (dict(output="gaussian", seed=7, log_std="ls"), PLAIN + ("ls",),
                 lambda v: _want(v, "gaussian", bias=False, seed=7, log_std=v["ls"])),
    "gaussian-state": (dict(bias=True, output="gaussian", seed="seed", log_std=("wls", "bls"), log_std_bounds=(-5, 1),
                            squash=True), BIASED + ("wls", "bls", "seed"),
                       lambda v: _want(v, "gaussian", seed=v["seed"], log_std=(v["wls"], v["bls"]),
                                       log_std_bounds=(-5.0, 1.0), squash=True)),
    "epsilon-named": (dict(bias=True, output="epsilon_greedy", seed=3, epsilon="eps"), BIASED + ("eps",),
                      lambda v: _want(v, "epsilon_greedy", seed=3, epsilon=v["eps"])),
    "epsilon-constant": (dict(output="epsilon_greedy", seed="seed", epsilon=0.25), PLAIN + ("seed",),
                         lambda v: _want(v, "epsilon_greedy", bias=False, seed=v["seed"], epsilon=0.25)),
    "evaluate": (dict(bias=True, output="evaluate", taken="t", nvec=(2, 2)), BIASED + ("t",),
                 lambda v: _want(v, "evaluate", taken=v["t"], nvec=(2, 2))),
    "gaussian_evaluate": (dict(bias=True, output="gaussian_evaluate", taken="t", log_std="ls", value=("wv", "bv")),
                          BIASED + ("t", "ls", "wv", "bv"),
                          lambda v: _want(v, "gaussian_evaluate", taken=v["t"], log_std=v["ls"],
                                          value=(v["wv"], v["bv"]))),
    "deterministic": (dict(output="deterministic", squash=False), PLAIN,
                      lambda v: _want(v, "deterministic", bias=False, squash=False)),
    "deterministic-named-noise": (dict(bias=True, output="deterministic", noise="sigma", noise_clip=0.5, seed="seed"),
                                  BIASED + ("sigma", "seed"),
                                  lambda v: _want(v, "deterministic", noise=v["sigma"], noise_clip=0.5,
                                                  seed=v["seed"])),
    "deterministic-constant-noise": (dict(output="deterministic", noise=0.1, seed=9), PLAIN,
                                     lambda v: _want(v, "deterministic", bias=False, noise=0.1, seed=9)),
    "critic": (dict(output="critic", action="a"), PLAIN + ("a",),
               lambda v: _want(v, "critic", bias=False, action=v["a"])),
    "critic-twin3": (dict(output="critic", action="a", twin=("t1", "t2", "t3")), PLAIN + ("a", "t1", "t2", "t3"),
                     lambda v: _want(v, "critic", bias=False, action=v["a"],
                                     twin=(v["t1"], None, v["t2"], None, v["t3"], None))),
    "critic-twin6": (dict(bias=True, output="critic", action="a", twin=("t1", "tb1", "t2", "tb2", "t3", "tb3")),
                     BIASED + ("a", "t1", "tb1", "t2", "tb2", "t3", "tb3"),
                     lambda v: _want(v, "critic", action=v["a"],
                                     twin=tuple(v[n] for n in ("t1", "tb1", "t2", "tb2", "t3", "tb3")))),
    "td3-actor3": (dict(output="td_target", policy="deterministic", actor=("a1", "a2", "a3"), reward="r", done="d",
                        gamma=0.99, twin=("t1", "t2", "t3"), noise=0.2, noise_clip=0.5, seed="seed"),
                   PLAIN + ("a1", "a2", "a3", "t1", "t2", "t3", "r", "d", "seed"),
                   lambda v: _want(v, "td_target", bias=False, twin=(v["t1"], None, v["t2"], None, v["t3"], None),
                                   noise=0.2, noise_clip=0.5, seed=v["seed"],
                                   actor=(v["a1"], None, v["a2"], None, v["a3"], None), policy="deterministic",
                                   reward=v["r"], done=v["d"], gamma=0.99, alpha=None)),
    "td3-named-noise": (dict(bias=True, output="td_target", policy="deterministic",
                             actor=("a1", "ab1", "a2", "ab2", "a3", "ab3"), reward="r", done="d", gamma=0.9,
                             noise="sigma", seed=4),
                        BIASED + ("a1", "ab1", "a2", "ab2", "a3", "ab3", "r", "d", "sigma"),
                        lambda v: _want(v, "td_target", noise=v["sigma"], seed=4,
                                        actor=tuple(v[n] for n in ("a1", "ab1", "a2", "ab2", "a3", "ab3")),
                                        policy="deterministic", reward=v["r"], done=v["d"], gamma=0.9, alpha=None)),
    "sac-constant-alpha": (dict(bias=True, output="td_target", policy="gaussian",
                                actor=("a1", "ab1", "a2", "ab2", "a3", "ab3"), log_std=("wls", "bls"), reward="r",
                                done="d", gamma=0.99, seed=11, alpha=0.2, squash=True),
                           BIASED + ("a1", "ab1", "a2", "ab2", "a3", "ab3", "wls", "bls", "r", "d"),
                           lambda v: _want(v, "td_target", seed=11, log_std=(v["wls"], v["bls"]), squash=True,
                                           actor=tuple(v[n] for n in ("a1", "ab1", "a2", "ab2", "a3", "ab3")),
                                           policy="gaussian", reward=v["r"], done=v["d"], gamma=0.99, alpha=0.2)),
}


@pytest.mark.parametrize("name", list(CALLS))
def test_call_mlp_resolves_named_options(name):
    _check_call(*CALLS[name])


def test_call_mlp_reads_a_named_alpha_with_float():
    params = BIASED + ("a1", "ab1", "a2", "ab2", "a3", "ab3", "wls", "bls", "r", "d", "temp")
    fn = kt.mapped("mlp", bias=True, output="td_target", policy="gaussian", actor=("a1", "ab1", "a2", "ab2", "a3", "ab3"),
                   log_std=("wls", "bls"), reward="r", done="d", gamma=0.99, seed=1,
                   alpha="temp")(_body(*params))
    spec = mapped_spec(fn)
    args = [_Stub(p) for p in params]
    args[-1] = torch.tensor([0.125])
    _, _, _, bound = spec.bind(fn, tuple(args), {})
    me = SimpleNamespace(devices=[0], transfer="pull", ops=SimpleNamespace(PushTimeout=TimeoutError),
                         _all_ranks=lambda ranks: True)
    with mock.patch.object(mlp, "mlp_scatter_gather", return_value=["r0"]) as sg:
        B200Supervisor._call_mlp(me, spec, bound)
    alpha = sg.call_args.kwargs["alpha"]
    assert type(alpha) is float and alpha == 0.125
