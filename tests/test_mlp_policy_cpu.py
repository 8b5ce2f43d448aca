"""not-gpu: the nn.Linear policy form of the mapped "mlp" op without a GPU — its decoration options, the semantic
definition of its cases on 1 and 3 ranks, the Python argument checks and the serialisation of (logits, actions)
results."""
import base64
import pickle

import pytest
import torch
import torch.nn.functional as F

import policy_cases
from oracle import ref_dispatch


# ---- decoration -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kwargs", [
    {"bias": "yes"}, {"bias": 1}, {"output": "probs"}, {"output": None}, {"bias": True, "output": "argmax"},
])
def test_bad_mlp_options_raise_at_decoration(kwargs):
    import kubetorch_b200 as kt

    with pytest.raises(ValueError):
        kt.mapped("mlp", **kwargs)


@pytest.mark.parametrize("op", ["identity", "scale", "affine"])
def test_policy_options_belong_to_the_mlp_op(op):
    import kubetorch_b200 as kt

    with pytest.raises(ValueError):
        kt.mapped(op, bias=True)
    with pytest.raises(ValueError):
        kt.mapped(op, output="actions")


@pytest.mark.parametrize("output", ["logits", "actions", "both"])
def test_policy_options_are_recorded_on_the_spec(output):
    import kubetorch_b200 as kt
    from kubetorch_b200.mapped import mapped_spec

    fn = kt.mapped("mlp", bias=True, output=output)(lambda obs, w1, b1, w2, b2, w3, b3: None)
    spec = mapped_spec(fn)
    assert spec.op == "mlp" and spec.extra["bias"] is True and spec.extra["output"] == output
    plain = mapped_spec(kt.mapped("mlp")(lambda obs, w1, w2, w3: None))
    assert "bias" not in plain.extra and "output" not in plain.extra   # the defaults leave the spec as it was


# ---- the semantic definition ----------------------------------------------------------------------------------------
def _policy(seed, d_in=64, d_hidden=256, d_out=6):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).bfloat16()   # noqa: E731
    return (r(d_hidden, d_in, scale=0.1), r(d_hidden, scale=0.5), r(d_hidden, d_hidden, scale=0.05),
            r(d_hidden, scale=0.5), r(d_out, d_hidden, scale=0.05), r(d_out, scale=0.5))


def _direct(obs, w1, b1, w2, b2, w3, b3):
    h = torch.relu(F.linear(obs, w1, b1))
    h = torch.relu(F.linear(h, w2, b2))
    return F.linear(h, w3, b3)


@pytest.mark.parametrize("rows,n_ranks", [(10, 1), (10, 3), (2, 3), (0, 3)])
def test_policy_cases_shard_and_evaluate_like_torch(rows, n_ranks):
    """Rank r of the oracle's SPMD call evaluates the policy on obs.chunk(n_ranks)[r], empty shards included."""
    p = _policy(rows * 7 + n_ranks)
    obs = torch.randn(rows, 64, generator=torch.Generator().manual_seed(rows)).bfloat16()
    chunks = list(obs.chunk(n_ranks)) if rows else []
    shards = chunks + [obs[:0]] * (n_ranks - len(chunks))
    want = [_direct(s, *p) for s in shards]
    logits = ref_dispatch.spmd_call(policy_cases.mlp_policy_biased, obs, *p, num_proc=n_ranks)
    actions = ref_dispatch.spmd_call(policy_cases.mlp_policy_actions, obs, *p, num_proc=n_ranks)
    both = ref_dispatch.spmd_call(policy_cases.mlp_policy_both, obs, *p, num_proc=n_ranks)
    assert len(logits) == len(actions) == len(both) == n_ranks
    for r in range(n_ranks):
        assert logits[r].dtype == torch.bfloat16 and torch.equal(logits[r], want[r])
        assert actions[r].dtype == torch.int64 and actions[r].shape == (want[r].shape[0],)
        assert torch.equal(actions[r], want[r].argmax(-1))
        assert isinstance(both[r], tuple) and torch.equal(both[r][0], want[r]) and torch.equal(both[r][1], actions[r])


def test_argmax_semantics_the_kernels_follow():
    """The tie and NaN rules of torch.argmax that the device actions reproduce."""
    t = torch.tensor([[1.0, 3.0, 3.0, 2.0], [float("nan"), 5.0, float("nan"), 1.0], [-0.0, 0.0, -1.0, -2.0],
                      [float("inf"), 0.0, float("inf"), 1.0], [-5.0, -1.0, -3.0, -1.0]]).bfloat16()
    assert t.argmax(-1).tolist() == [1, 0, 0, 0, 1]


# ---- Python argument checks -----------------------------------------------------------------------------------------
def _w(d_in=256, d_hidden=1024, d_out=18):
    return (torch.zeros(d_hidden, d_in, dtype=torch.bfloat16), torch.zeros(d_out, d_hidden, dtype=torch.bfloat16))


def test_python_checks_accept_every_head_and_output():
    """Every output mode at the head widths the kernels take (1 to 256) passes the checks."""
    from kubetorch_b200.device import mlp

    for d_out in (1, 18, 64, 256):
        w1, w3 = _w(d_out=d_out)
        for output in ("logits", "actions", "both"):
            assert mlp._check_policy(w1, w3, (None, None, None), output) is None


@pytest.mark.parametrize("case", [
    "d_out_0", "d_out_257", "output", "b1_length", "b3_length", "b2_dtype", "b1_2d", "b3_not_contiguous", "b1_on_cpu",
    "biases_not_three",
])
def test_python_checks_raise_value_error(case):
    """Shapes, dtypes and head widths the kernels do not take are a ValueError before anything reaches the device
    (the serving layer turns it into the reference's 400 envelope)."""
    from kubetorch_b200.device import mlp

    w1, w3 = _w()
    meta = lambda n, dtype=torch.bfloat16: torch.empty(n, dtype=dtype, device="meta")   # noqa: E731
    biases, output = [None, None, None], "logits"
    if case == "d_out_0":
        w1, w3 = _w(d_out=0)
    elif case == "d_out_257":
        w1, w3 = _w(d_out=257)
    elif case == "output":
        output = "probs"
    elif case == "b1_length":
        biases[0] = meta(1023)
    elif case == "b3_length":
        biases[2] = meta(64)
    elif case == "b2_dtype":
        biases[1] = meta(1024, torch.float32)
    elif case == "b1_2d":
        biases[0] = torch.empty(1, 1024, dtype=torch.bfloat16, device="meta")
    elif case == "b3_not_contiguous":
        biases[2] = meta(36)[::2]
    elif case == "b1_on_cpu":
        biases[0] = torch.zeros(1024, dtype=torch.bfloat16)
    elif case == "biases_not_three":
        biases = [None, None]
    with pytest.raises(ValueError):
        mlp._check_policy(w1, w3, tuple(biases), output)


# ---- serialisation of a (logits, actions) result --------------------------------------------------------------------
def test_pickled_tuple_result_carries_only_its_shard():
    """Each rank's (logits, actions) are views of the root buffers: pickled, they must carry their own rows only."""
    from kubetorch_b200.serving.b200_supervisor import B200Supervisor

    logits_root, actions_root = torch.zeros(3000, 18, dtype=torch.bfloat16), torch.arange(3000)
    shard = (logits_root[1000:1010], actions_root[1000:1010])
    wire = B200Supervisor._serialize_result(shard, "pickle", True)
    back = pickle.loads(base64.b64decode(wire["data"]))
    assert isinstance(back, tuple) and len(back) == 2
    assert torch.equal(back[0], shard[0]) and torch.equal(back[1], shard[1])
    assert back[0].untyped_storage().nbytes() == 10 * 18 * 2
    assert back[1].untyped_storage().nbytes() == 10 * 8
    assert len(wire["data"]) < 4 * (10 * 18 * 2 + 10 * 8) + 4096
