"""not-gpu: B200Supervisor at the reference server's supervisor seam, against what the UNMODIFIED reference server returned.

tests/golden/b3_seam.json holds the responses of the reference's own FastAPI app (kubetorch.serving.http_server under
TestClient) with distribution_type "b200" routed to B200Supervisor through the 3-line supervisor_factory hook of
INTEGRATION.md.  Here the server's part is played the way the reference server plays it (http_server.py:971-1002 and
its exception handler, restated in oracle/ref_dispatch.py): the supervisor is built from the JSON distributed config
alone, the callable comes from the KT_* environment, RAW request bodies built by the reference client's codec go into
B200Supervisor.call, results leave through the reference client's decoder, and exceptions through the server's error
envelope.  Status codes, results and error envelopes must equal the recorded ones.  The device layer is a torch-CPU
stub (no GPU needed); tests/test_gpu_api.py::test_b3_* run the same contract against the real kernels."""
import json
import os

import torch

from conftest import REPO
from oracle import ref_dispatch

with open(os.path.join(REPO, "tests", "golden", "b3_seam.json")) as _f:
    GOLDEN = json.load(_f)["configs"]


def _stub_device():
    from kubetorch_b200.device import ops as real

    class Stub:
        shard_bounds = staticmethod(real.shard_bounds)
        row_elems = staticmethod(real.row_elems)
        calls = []

        @staticmethod
        def device_count():
            return 8

        @staticmethod
        def ensure_init(devs):
            pass

        @staticmethod
        def synchronize(dev):
            pass

        @staticmethod
        def join_devices(root, devs):
            pass

        @staticmethod
        def is_pinned(t):
            return True

        @staticmethod
        def pinned_empty(shape, dtype, devices=None):
            return torch.empty(shape, dtype=dtype)

        @staticmethod
        def _apply(x, op, alpha, beta):
            if op == "identity":
                return x.clone()
            return x * alpha if op == "scale" else x * alpha + beta

        @classmethod
        def map_host(cls, x, op, alpha=1.0, beta=0.0, out_host=None, devices=(0,), ranks=None, chunk_bytes=None):
            cls.calls.append(["map_host", len(devices)] + ([list(ranks)] if ranks is not None else []))
            out_host.copy_(cls._apply(x, op, alpha, beta))
            return out_host

    return Stub


def _tensor(spec):
    g = torch.Generator().manual_seed(spec.get("seed", 0))
    dt = getattr(torch, spec["dtype"])
    if dt.is_floating_point:
        return torch.randn(spec["shape"], generator=g).to(dt)
    return torch.randint(-1000, 1000, spec["shape"], generator=g, dtype=dt)


def _resolve(v):
    if isinstance(v, dict) and "tensor" in v:
        return _tensor(v["tensor"])
    if isinstance(v, list):
        return [_resolve(a) for a in v]
    return v


def _replay(name, monkeypatch):
    """The recorded calls of one server deployment, through B200Supervisor, in the recorded response format."""
    from kubetorch_b200.serving.b200_supervisor import B200Supervisor
    from kubetorch_b200.serving.supervisors import Request

    cfg = GOLDEN[name]["config"]
    monkeypatch.setenv("POD_NAME", "b3-pod")
    monkeypatch.setenv("KT_FILE_PATH", os.path.join(REPO, "tests"))
    monkeypatch.setenv("KT_MODULE_NAME", "b3_user_module")
    monkeypatch.setenv("KT_CLS_OR_FN_NAME", cfg["callable"])
    monkeypatch.setenv("KT_INIT_ARGS", json.dumps(cfg.get("init_args")))
    monkeypatch.setenv("KT_ALLOWED_SERIALIZATION", cfg.get("allowed", "json,pickle"))
    stub = _stub_device()
    monkeypatch.setattr(B200Supervisor, "_load_device", lambda self: stub)
    dist = dict(cfg["distributed_config"])
    assert dist.pop("distribution_type") == "b200"
    sup = B200Supervisor(**dist)
    sup.setup()
    records = []
    try:
        for call in cfg["calls"]:
            ser = call.get("serialization", "pickle")
            body = ref_dispatch.serialize_body(
                ref_dispatch.build_call_body(*_resolve(call.get("args", [])), **dict(call.get("kwargs") or {})), ser)
            try:
                raw = sup.call(Request({"X-Serialization": ser, "X-Request-ID": "b3"}), cfg["callable"],
                               call.get("method"), body)
                raw = json.loads(json.dumps(raw))        # the HTTP hop: JSON values only
                res = ref_dispatch.deserialize_response(raw, ser)
                rec = {"status_code": 200,
                       "result": [{"dtype": str(t.dtype), "shape": list(t.shape), "data": t.reshape(-1).tolist()}
                                  if isinstance(t, torch.Tensor) else t for t in res] if isinstance(res, list) else res}
            except Exception as e:  # noqa: BLE001
                status, env = ref_dispatch.package_exception(e)
                rec = {"status_code": status, "error": {k: env[k] for k in ("error_type", "message", "pod_name")}}
            records.append(rec)
    finally:
        sup.cleanup()
    return records, stub.calls


def _check(name, monkeypatch):
    records, calls = _replay(name, monkeypatch)
    want = GOLDEN[name]
    assert len(records) == len(want["records"])
    for i, (got, rec) in enumerate(zip(records, want["records"])):
        assert got == rec, f"{name} call {i}"
    assert calls == want["device_calls"], name


def _shards(x, world):
    ch = x.chunk(world)
    return [ch[r] if r < len(ch) else x[:0] for r in range(world)]


def test_reference_server_drives_b200_supervisor_with_raw_pickle_bodies(monkeypatch):
    _check("raw_pickle_bodies", monkeypatch)
    # the recorded results are the reference's SPMD semantics: rank-ordered x.chunk(4) shards, doubled
    recs = GOLDEN["raw_pickle_bodies"]["records"]
    x = _tensor({"dtype": "float32", "shape": [1003], "seed": 0})
    assert [r["data"] for r in recs[0]["result"]] == [(s * 2).tolist() for s in _shards(x, 4)]
    assert recs[3]["error"]["message"] == "Worker index 10 out of range. Valid range: 0-0"
    assert recs[5]["status_code"] == 200 and len(recs[5]["result"]) == 4      # "any" = the coordinator's local ranks


def test_reference_server_multi_node_config_and_workers_subset(monkeypatch):
    """quorum_workers=2 x num_proc=2: `workers=[1]` returns node 1's ranks only, which keep their GLOBAL rank / world
    size (recorded shapes [(251,), (250,)])."""
    _check("multi_node_workers_subset", monkeypatch)
    full, sub, bad = GOLDEN["multi_node_workers_subset"]["records"]
    assert [r["shape"] for r in full["result"]] == [[251], [251], [251], [250]]
    assert [r["shape"] for r in sub["result"]] == [[251], [250]]
    assert bad["status_code"] == 400


def test_reference_server_allow_list_json_mode_and_class_callable(monkeypatch):
    """The allow-list refusal, a class built from KT_INIT_ARGS with its method from the URL (and a missing one), and
    kwargs-bound parameters of an affine op (and a non-integral alpha on an int tensor)."""
    for name in ("allow_list_json", "class_callable", "affine_kwargs"):
        with monkeypatch.context() as mp:
            _check(name, mp)
    assert GOLDEN["allow_list_json"]["records"][0]["status_code"] == 400
    assert GOLDEN["class_callable"]["records"][1]["status_code"] == 404
    assert GOLDEN["affine_kwargs"]["records"][1]["error"]["error_type"] == "TypeError"
