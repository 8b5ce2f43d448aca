"""-m gpu: the public API (kt.fn / .to / remote __call__) on the GPU device backend against the
recorded reference runtime results and the oracle."""
import os

import pytest
import torch

from conftest import resolve_args

pytestmark = pytest.mark.gpu

import kubetorch_b200 as kt  # noqa: E402
from oracle import cases, ref_dispatch  # noqa: E402


from conftest import mapped_copy as _mapped  # noqa: E402


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    assert torch.cuda.is_available()


def _deploy(fn, n_ranks, name, placement="ranks"):
    """placement="ranks": every call fans out into one launch per rank (ranks time-sliced on cuda:0 on a 1-GPU box:
    same kernels, same shard arithmetic); "auto" adds the small-call lane (one launch on the root below 4 MiB)."""
    comp = kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute(
        "b200", workers=1, num_proc=n_ranks, devices=[0] * n_ranks, placement=placement)
    return kt.fn(fn, name=name).to(comp)


def test_recorded_reference_calls_through_public_api(golden):
    specs = {
        "double": _mapped(cases.double, "scale", alpha=2.0),
        "identity": _mapped(cases.identity, "identity"),
        "scale": _mapped(cases.scale, "scale", alpha="alpha"),
        "affine": _mapped(cases.affine, "affine", alpha="alpha", beta="beta"),
    }
    n = 0
    for name, rec in golden["cases"].items():
        if rec["status_code"] != 200 or rec["callable"] not in specs or (rec.get("kwargs") or {}).get("workers"):
            continue  # `workers=` sub-selections are host logic, covered on the CPU backends
        args = resolve_args(golden, rec["args"])
        # records taken on K real pods x P ranks have world size K*P: same shards, here as K*P local ranks
        world = rec["distributed_config"]["num_proc"] * len(rec.get("pods") or [None])
        remote = _deploy(specs[rec["callable"]], world, f"t-{name}")
        try:
            for resident in ("device", "host"):
                call_args = [a.cuda() if (resident == "device" and isinstance(a, torch.Tensor)) else a for a in args]
                got = remote(*call_args, serialization="pickle")
                assert isinstance(got, list) and len(got) == len(rec["result"])
                for g, w in zip(got, rec["result"]):
                    assert g.dtype == w.dtype and tuple(g.shape) == tuple(w.shape), (name, resident)
                    assert torch.equal(g.cpu().view(torch.uint8), w.view(torch.uint8)), (name, resident)
        finally:
            remote.teardown()
        n += 1
    assert n >= 10


def test_gather_reduce_through_public_api(golden):
    ssum = _mapped(cases.shard_sum, "affine", alpha="alpha", beta="beta", reduce="sum")
    remote = _deploy(ssum, 4, "t-sum")
    try:
        for name in ("sum_i64_130_x4", "sum_i32_515_x4"):
            rec = golden["cases"][name]
            args = resolve_args(golden, rec["args"])
            got = remote(*[a.cuda() if isinstance(a, torch.Tensor) else a for a in args], serialization="pickle")
            assert got == rec["result"], name
        rec = golden["cases"]["sum_f32_1001_x4"]
        x = resolve_args(golden, rec["args"])[0]
        got = remote(x.cuda(), serialization="pickle")
        tol = 8 * torch.finfo(torch.float32).eps * float(x.abs().sum())  # fp32 sum, order differs from torch
        assert all(abs(g - w) <= tol for g, w in zip(got, rec["result"]))
        # 2-byte floats and i32 products that wrap: integer-valued inputs keep every float sum exact in any order, so
        # the ranks' sums must equal the oracle's exactly
        g = torch.Generator().manual_seed(13)
        for dtype, bound, a, b in ((torch.bfloat16, 127, 0.5, 0.25), (torch.float16, 1023, 0.5, 0.25),
                                   (torch.float16, 1023, -1, 1), (torch.int32, 2**31, 65537, -7)):
            x = torch.randint(-bound, bound, (10_003,), generator=g).to(dtype)   # |partial sums| < 2^22 per shard
            want = ref_dispatch.spmd_call(cases.shard_sum, x, a, b, num_proc=4, serialization="pickle")
            got = remote(x.cuda(), a, b, serialization="pickle")
            assert got == want, (dtype, a, b)
            assert all(isinstance(v, float if dtype.is_floating_point else int) for v in got), dtype
    finally:
        remote.teardown()


def test_non_distributed_gpu_call_returns_bare_tensor():
    double = _mapped(cases.double, "scale", alpha=2.0)
    remote = kt.fn(double, name="t-bare").to(kt.Compute(gpus=1))
    try:
        x = torch.randn(4099)
        y = remote(x.cuda(), serialization="pickle")
        assert isinstance(y, torch.Tensor) and torch.equal(y.cpu(), x * 2)
    finally:
        remote.teardown()


def test_rows_are_the_shard_unit():
    """2-D args shard like x.chunk(world) along dim 0 (whole rows), as the reference's user code does."""
    double = _mapped(cases.double, "scale", alpha=2.0)
    remote = _deploy(double, 4, "t-rows")
    try:
        x = torch.randn(10, 37)
        want = ref_dispatch.spmd_call(cases.double, x, num_proc=4, serialization="pickle")
        got = remote(x.cuda(), serialization="pickle")
        assert [tuple(g.shape) for g in got] == [tuple(w.shape) for w in want]
        assert all(torch.equal(g.cpu(), w) for g, w in zip(got, want))
    finally:
        remote.teardown()


def test_errors_keep_the_reference_envelope():
    double = _mapped(cases.double, "scale", alpha=2.0)
    remote = kt.fn(double, name="t-err").to(
        kt.Compute(gpus=1, allowed_serialization=["json"]).distribute("b200", num_proc=2, devices=[0, 0]))
    try:
        with pytest.raises(Exception) as ei:
            remote(torch.ones(4).cuda(), serialization="pickle")
        assert "Serialization format 'pickle' not allowed. Allowed formats: ['json']" in str(ei.value)
        assert ei.value.pod_name and "Traceback" in ei.value.remote_traceback
    finally:
        remote.teardown()
    r2 = _deploy(double, 2, "t-err2")
    try:
        with pytest.raises(TypeError) as ei:
            r2("not a tensor", serialization="pickle")
        assert ei.value.status_code == 422 if hasattr(ei.value, "status_code") else True
    finally:
        r2.teardown()


def test_unmapped_callable_is_rejected_loudly():
    remote = kt.fn(cases.summer, name="t-unmapped").to(kt.Compute(gpus=1).distribute("b200", num_proc=1))
    try:
        with pytest.raises(TypeError, match="not a @kt.mapped callable"):
            remote(1, 2)
    finally:
        remote.teardown()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_peer_path_matches_oracle():
    from kubetorch_b200.device import ops

    ops.ensure_init([0, 1])
    x = torch.randn((1 << 22) + 5)
    want = torch.cat(ref_dispatch.spmd_call(cases.affine, x, 0.5, 1.5, num_proc=2, serialization="pickle"))
    for variant in (1, 2):
        y = ops.scatter_map_gather(x.cuda(0), "affine", 0.5, 1.5, devices=[0, 1], variant=variant)
        torch.cuda.synchronize(0)
        assert torch.equal(y.cpu(), want), variant
    # concurrent callers on their own streams (per-call events keep their joins apart)
    import threading

    errs = []

    def worker(i):
        try:
            xi_ = torch.randn((1 << 20) + i, generator=torch.Generator().manual_seed(i))
            with torch.cuda.device(0), torch.cuda.stream(torch.cuda.Stream(0)):
                for _ in range(5):
                    yi_ = ops.scatter_map_gather(xi_.cuda(0), "scale", float(i + 2), devices=[0, 1])
                    torch.cuda.current_stream(0).synchronize()
                    assert torch.equal(yi_.cpu(), xi_ * float(i + 2))
        except BaseException as e:  # noqa: BLE001
            errs.append(e)

    ths = [threading.Thread(target=worker, args=(i,)) for i in range(4)]
    [t.start() for t in ths]
    [t.join() for t in ths]
    assert not errs, errs
    sess = ops.PushSession([0, 1], ops.shard_bounds(x.numel(), 2, 0)[1] * 4)
    for it in range(4):  # consecutive calls exercise staging parity and the ack back-pressure
        y = torch.zeros_like(x, device="cuda:0")
        sess.call(x.cuda(0), y, "affine", 0.5, 1.5)
        torch.cuda.synchronize(0)
        assert torch.equal(y.cpu(), want), ("push", it)
    sess.check()
    xi = torch.randint(-(2**40), 2**40, (100_003,), dtype=torch.int64)
    total, partials = ops.scatter_map_reduce(xi.cuda(0), "identity", devices=[0, 1])
    assert partials.tolist() == ref_dispatch.spmd_call(cases.shard_sum, xi, num_proc=2, serialization="pickle")
    xh = torch.randn((1 << 21) + 3).pin_memory()   # host-resident, both GPUs from one host thread
    assert torch.equal(ops.map_host_multi(xh, "scale", 2.0, devices=[0, 1]), xh * 2.0)
    from kubetorch_b200.device import mlp

    g = torch.Generator().manual_seed(3)
    obs = torch.randn(1024, 256, generator=g).bfloat16().cuda(0)
    w = [(torch.randn(s, generator=g) * 0.02).bfloat16().cuda(0) for s in ((1024, 256), (1024, 1024), (64, 1024))]
    single = mlp.mlp_forward(obs, *w)
    views = mlp.mlp_scatter_gather(obs, *w, devices=[0, 1], transfer="pull")   # rank 1: staged NVLink pull + peer-store epilogue
    torch.cuda.synchronize(0)
    assert torch.equal(torch.cat(views).cpu(), single.cpu())
    for it in range(3):   # pushed form: the root pushes row chunks, rank 1's GEMMs wait in-stream on the landing flags
        views = mlp.mlp_scatter_gather(obs, *w, devices=[0, 1], transfer="push")
        torch.cuda.synchronize(0)
        torch.cuda.synchronize(1)
        assert torch.equal(torch.cat(views).cpu(), single.cpu()), it
    g2 = torch.Generator().manual_seed(4)
    big = torch.randn(2 * 37888 + 2 * 1280, 256, generator=g2).bfloat16().cuda(0)   # several push chunks per rank, ragged tail
    ref_big = mlp.mlp_forward(big, *w)
    views = mlp.mlp_scatter_gather(big, *w, devices=[0, 1], transfer="push")
    torch.cuda.synchronize(0)
    torch.cuda.synchronize(1)
    # the pushed chunks and the single-GPU chunks split the rows differently, and every tile is computed the same way
    # whatever the chunking: identical bits
    assert torch.equal(torch.cat(views).cpu(), ref_big.cpu())
    dst = torch.empty(1 << 20, dtype=torch.uint8, device="cuda:1")
    src = torch.randint(0, 255, (1 << 20,), dtype=torch.uint8, device="cuda:0")
    ops.broadcast(src, [dst])
    torch.cuda.synchronize(0)
    assert torch.equal(dst.cpu(), src.cpu())


def test_arbitrary_callables_on_gpu_ranks_use_hbm_arenas(golden):
    """.distribute("spmd") on a GPU compute runs ARBITRARY Python on rank processes; CUDA tensor args travel
    through pack → broadcast → zero-copy views, CUDA tensor results through pack → unpack (no pickling of
    tensor data). Same results as the recorded reference runtime."""
    comp = kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute(
        "spmd", workers=1, num_proc=2, devices=[0, 0], arena_bytes=1 << 20)
    remote = kt.fn(cases.affine, name="t-gpu-spmd").to(comp)  # plain Python body, not @mapped here
    try:
        assert remote._supervisor.__class__.__name__ == "GpuSPMDSupervisor"
        rec = golden["cases"]["affine_f32_1001_x2"]
        x, a, b = resolve_args(golden, rec["args"])
        got = remote(x.cuda(), a, b, serialization="pickle")
        assert all(g.is_cuda for g in got)
        for g, w in zip(got, rec["result"]):
            assert torch.equal(g.cpu(), w)
        # arena growth: 8 MiB of args through 1 MiB arenas, twice (second call reuses the grown arenas)
        big = torch.randn(1 << 21)
        for _ in range(2):
            got = remote(big.cuda(), 2.0, 1.0, serialization="pickle")
            assert torch.equal(torch.cat(got).cpu(), big * 2.0 + 1.0)
    finally:
        remote.teardown()
    mixed = kt.fn(cases.mixed_payload, name="t-gpu-mixed").to(
        kt.Compute(gpus=1).distribute("spmd", workers=1, num_proc=2, devices=[0, 0]))
    try:
        x = torch.arange(12, dtype=torch.float32).reshape(3, 4).cuda()
        t = torch.tensor([10, 20], dtype=torch.int64).cuda()
        out = mixed(x, {"t": t, "tag": "hello"}, scale=2, serialization="pickle")
        assert [o["rank"] for o in out] == [0, 1] and out[0]["tag"] == "hello" and out[1]["shape"] == [3, 4]
        assert float(out[0]["sum"]) == 132.0 and out[1]["y"].tolist() == [11, 21] and out[1]["y"].is_cuda
    finally:
        mixed.teardown()


def test_kt_put_get_gpu_store_patterns():
    """kt.put / kt.get of GPU tensors and state dicts (SURVEY §8(f) #1) with the reference's test patterns:
    torch.full fills, several dtypes, state dicts, packed BroadcastWindow (tests/assets/kv_store/gpu_helper.py)."""
    import threading

    n_dev = torch.cuda.device_count()
    dst_dev = f"cuda:{1 if n_dev > 1 else 0}"
    for dtype, fill in ((torch.float32, 3.5), (torch.bfloat16, -2.0), (torch.int64, 7), (torch.uint8, 200)):
        src = torch.full((257, 33), fill, dtype=dtype, device="cuda:0")
        kt.put(key=f"t/{dtype}", src=src)
        dest = torch.zeros_like(src, device=dst_dev)
        kt.get(key=f"t/{dtype}", dest=dest)
        torch.cuda.synchronize()
        assert torch.equal(dest.cpu(), src.cpu())
    sd = {"layer1": {"weight": torch.randn(64, 32, device="cuda:0"), "bias": torch.randn(64, device="cuda:0")},
          "head.weight": torch.randn(10, 64, device="cuda:0").bfloat16(), "step": torch.tensor(5, device="cuda:0")}
    kt.put(key="model/weights", src=sd)
    assert kt.ls("model/weights") == ["model/weights/head.weight", "model/weights/layer1.bias",
                                      "model/weights/layer1.weight", "model/weights/step"]
    dest_sd = {"layer1": {"weight": torch.zeros(64, 32, device=dst_dev), "bias": torch.zeros(64, device=dst_dev)},
               "head.weight": torch.zeros(10, 64, device=dst_dev).bfloat16(), "step": torch.tensor(0, device=dst_dev)}
    kt.get(key="model/weights", dest=dest_sd)
    one = torch.zeros(64, device=dst_dev)
    kt.get(key="model/weights/layer1.bias", dest=one)   # a single leaf of a published state dict
    torch.cuda.synchronize()
    assert torch.equal(dest_sd["layer1"]["weight"].cpu(), sd["layer1"]["weight"].cpu())
    assert torch.equal(dest_sd["head.weight"].cpu(), sd["head.weight"].cpu()) and int(dest_sd["step"]) == 5
    assert torch.equal(one.cpu(), sd["layer1"]["bias"].cpu())
    # packed broadcast: 1 putter + 2 getters, one read of the source, unpack on arrival
    bw = kt.BroadcastWindow(world_size=3, timeout=30.0, group_id="g1", pack=True)
    dests = [{k: torch.zeros_like(v, device=dst_dev if i else "cuda:0") for k, v in
              {"a": sd["layer1"]["weight"], "b": sd["layer1"]["bias"]}.items()} for i in range(2)]
    results = []
    ths = [threading.Thread(target=lambda d=d: results.append(kt.get(key="bc", dest=d, broadcast=bw))) for d in dests]
    [t.start() for t in ths]
    r = kt.put(key="bc", src={"a": sd["layer1"]["weight"], "b": sd["layer1"]["bias"]}, broadcast=bw)
    [t.join() for t in ths]
    torch.cuda.synchronize()
    assert r["world_size"] == 3 and len(results) == 2
    for d in dests:
        assert torch.equal(d["a"].cpu(), sd["layer1"]["weight"].cpu()) and torch.equal(d["b"].cpu(), sd["layer1"]["bias"].cpu())
    with pytest.raises(kt.DataStoreError, match="not found"):
        kt.get(key="nope", dest=torch.zeros(1, device="cuda:0"))
    with pytest.raises(ValueError, match="stored tensor"):
        kt.get(key="model/weights/layer1.bias", dest=torch.zeros(65, device="cuda:0"))
    with pytest.raises(ValueError, match="must be on a CUDA device"):
        kt.put(key="cpu", src={"w": torch.zeros(2), "g": torch.zeros(2, device="cuda:0")})
    kt.rm("model/weights")
    assert kt.ls("model/weights") == []
    with pytest.raises(kt.DataStoreError, match="timed out"):
        kt.get(key="late", dest=torch.zeros(1, device="cuda:0"), broadcast=kt.BroadcastWindow(world_size=2, timeout=0.3))


def test_results_are_fresh_tensors_not_aliases_of_a_cache():
    double = _mapped(cases.double, "scale", alpha=2.0)
    remote = _deploy(double, 2, "t-fresh")
    try:
        a = torch.arange(10, dtype=torch.float32)
        r1 = remote(a, serialization="pickle")               # host path
        r2 = remote(a + 100, serialization="pickle")
        assert torch.equal(torch.cat(r1), a * 2) and torch.equal(torch.cat(r2), (a + 100) * 2)
        d1 = remote(a.cuda(), serialization="pickle")          # device path
        d2 = remote((a + 100).cuda(), serialization="pickle")
        torch.cuda.synchronize()
        assert torch.equal(torch.cat(d1).cpu(), a * 2) and torch.equal(torch.cat(d2).cpu(), (a + 100) * 2)
    finally:
        remote.teardown()


def test_edge_inputs_empty_noncontiguous_unsupported_dtype():
    double = _mapped(cases.double, "scale", alpha=2.0)
    remote = _deploy(double, 3, "t-edge")
    try:
        empty = remote(torch.empty(0).cuda(), serialization="pickle")
        assert len(empty) == 3 and all(e.numel() == 0 for e in empty)
        one = remote(torch.tensor([5.0]).cuda(), serialization="pickle")       # fewer rows than ranks
        assert [o.numel() for o in one] == [1, 0, 0] and float(one[0]) == 10.0
        x = torch.randn(7, 5)
        xt = x.t()                                                             # non-contiguous view, 5 rows of 7
        want = ref_dispatch.spmd_call(cases.double, xt, num_proc=3, serialization="pickle")
        got = remote(xt.cuda(), serialization="pickle")
        assert [tuple(g.shape) for g in got] == [tuple(w.shape) for w in want]
        assert all(torch.equal(g.cpu(), w) for g, w in zip(got, want))
        got_h = remote(xt, serialization="pickle")                             # same through the host path
        assert all(torch.equal(g, w) for g, w in zip(got_h, want))
        with pytest.raises(TypeError, match="support"):
            remote(torch.ones(4, dtype=torch.float64).cuda(), serialization="pickle")
    finally:
        remote.teardown()


def test_kt_put_get_between_rank_processes():
    """kt.put in one rank process, kt.get in another (CUDA IPC arenas + descriptor files under KTB_STORE_DIR)."""
    comp = lambda: kt.Compute(gpus=1).distribute("spmd", workers=1, num_proc=2, devices=[0, 0])  # noqa: E731
    cls_put = kt.fn(cases.store_put_by_rank, name="t-store")
    cls_put.to(comp())
    try:
        assert cls_put(1000) == [0, 1]
        # same deployment (same rank processes, same store dir): a second callable would restart the ranks, so reuse
        # the worker pool through a tiny dispatcher: deploy the getter on the SAME supervisor's store dir
        store_dir = cls_put._supervisor.env_vars["KTB_STORE_DIR"]
        getter = kt.fn(cases.store_get_from_rank, name="t-store-get").to(
            kt.Compute(gpus=1, env_vars={"KTB_STORE_DIR": store_dir}).distribute("spmd", workers=1, num_proc=2,
                                                                                 devices=[0, 0]))
        try:
            out = getter(1, 1000)        # both getter ranks (new processes) read what putter rank 1 published
            assert [o[0] for o in out] == [1000.0, 1000.0]
            assert out[0][1] == ["by-rank/0", "by-rank/1"]
            out0 = getter(0, 1000)
            assert [o[0] for o in out0] == [0.0, 0.0]
        finally:
            getter.teardown()
    finally:
        cls_put.teardown()


def test_root_placement_option_gives_identical_results():
    double = _mapped(cases.double, "scale", alpha=2.0)
    n_dev = torch.cuda.device_count()
    devices = list(range(min(n_dev, 2))) * (2 if n_dev < 2 else 1)
    remote = kt.fn(double, name="t-placement").to(
        kt.Compute(gpus=1).distribute("b200", workers=1, num_proc=len(devices), devices=devices, placement="root"))
    try:
        x = torch.randn(10_007)
        got = remote(x.cuda(0), serialization="pickle")
        want = ref_dispatch.spmd_call(cases.double, x, num_proc=len(devices), serialization="pickle")
        assert all(torch.equal(g.cpu(), w) for g, w in zip(got, want))
    finally:
        remote.teardown()


# ---- seam B3: the reference's supervisor contract, on the real kernels -------------------------------------------
def _b3_supervisor(monkeypatch, name, cfg, world, allowed="json,pickle", init_args=None):
    """Build the supervisor the way the reference's server does (http_server.py:971-1002): from the JSON
    distributed config alone, with the callable named by the KT_* environment."""
    import json

    from conftest import REPO
    from kubetorch_b200.serving.b200_supervisor import B200Supervisor

    monkeypatch.setenv("KT_FILE_PATH", os.path.join(REPO, "tests"))
    monkeypatch.setenv("KT_MODULE_NAME", "b3_user_module")
    monkeypatch.setenv("KT_CLS_OR_FN_NAME", name)
    monkeypatch.setenv("KT_INIT_ARGS", json.dumps(init_args))
    monkeypatch.setenv("KT_ALLOWED_SERIALIZATION", allowed)
    monkeypatch.setenv("POD_NAME", "b3-pod")
    wire_cfg = json.loads(json.dumps({**cfg, "distribution_type": "b200", "devices": [0] * world}))   # JSON values only
    wire_cfg.pop("distribution_type")
    sup = B200Supervisor(**wire_cfg)
    sup.setup()
    return sup


def test_b3_raw_reference_request_bodies_bit_equal_to_recorded_results(golden, monkeypatch):
    """Every recorded tensor call of the reference runtime, replayed at the supervisor seam: the RAW request body the
    reference's client produces (`{"data": b64(pickle)}` + hoisted workers) goes into B200Supervisor.call, the return
    value goes through the reference client's response decoder, and the result must be bit-equal to what the
    reference's own pods returned."""
    from kubetorch_b200.serving.supervisors import Request

    names = {"double", "identity", "scale", "affine", "shard_sum"}
    n = 0
    for case, rec in golden["cases"].items():
        if rec["callable"] not in names or rec["serialization"] != "pickle":
            continue
        cfg = rec["distributed_config"]
        pods = len(rec.get("pods") or [None])
        world = cfg["num_proc"] * pods
        sup = _b3_supervisor(monkeypatch, rec["callable"], {"num_proc": cfg["num_proc"], "quorum_workers": pods}, world)
        try:
            args = resolve_args(golden, rec["args"])
            body = ref_dispatch.serialize_body(ref_dispatch.build_call_body(*args, **dict(rec.get("kwargs") or {})), "pickle")
            assert set(body) <= {"data", "workers", "restart_procs"} and isinstance(body["data"], str)
            raw = sup.call(Request({"X-Serialization": "pickle", "X-Request-ID": case}), rec["callable"], None, body)
            assert isinstance(raw, list) and all(isinstance(r, dict) and set(r) == {"data"} for r in raw), case
            got = ref_dispatch.deserialize_response(raw, "pickle")
            want = rec["result"]
            assert len(got) == len(want), case
            for g, w in zip(got, want):
                if isinstance(w, torch.Tensor):
                    assert g.dtype == w.dtype and tuple(g.shape) == tuple(w.shape), case
                    assert torch.equal(g.cpu().reshape(-1).view(torch.uint8), w.reshape(-1).view(torch.uint8)), case
                elif isinstance(w, float):
                    x = args[0]
                    assert abs(g - w) <= 8 * torch.finfo(torch.float32).eps * float(x.float().abs().sum()), case
                else:
                    assert g == w, case
        finally:
            sup.cleanup()
        n += 1
    assert n >= 14


def test_b3_workers_restart_and_errors_on_the_device_route(monkeypatch):
    from kubetorch_b200.serving.supervisors import Request

    req = Request({"X-Serialization": "pickle"})
    x = torch.arange(1003, dtype=torch.float32)
    sup = _b3_supervisor(monkeypatch, "double", {"num_proc": 2, "quorum_workers": 2}, 4)
    try:
        def call(**magic):
            body = ref_dispatch.serialize_body(ref_dispatch.build_call_body(x, **magic), "pickle")
            return ref_dispatch.deserialize_response(sup.call(req, "double", None, body), "pickle")

        full = call()
        assert [tuple(t.shape) for t in full] == [(251,), (251,), (251,), (250,)]
        sub = call(workers=[1])                          # node 1 = global ranks 2, 3 (recorded: mp_double_f32_1003_workers_1)
        assert [tuple(t.shape) for t in sub] == [(251,), (250,)]
        assert torch.equal(sub[0], x[502:753] * 2) and torch.equal(sub[1], x[753:] * 2)
        assert len(call(workers=["1"])) == 2 and len(call(workers="any")) == 2 and len(call(workers=[0, 1])) == 4
        with pytest.raises(ValueError, match=r"Worker index 10 out of range. Valid range: 0-1"):
            call(workers=[10])
        with pytest.raises(ValueError, match=r"Invalid worker specification: 1.5. Must be an IP address"):
            call(workers=[1.5])
        before = sup._callable
        assert len(call(restart_procs=True)) == 4 and sup._callable is not None
        # device-resident args take the same selectors
        body = {"args": [x.cuda()], "kwargs": {}, "workers": [1]}
        live = sup.call(req, "double", None, body)          # live objects (LocalClient form): tensors come back live
        assert [tuple(t.shape) for t in live] == [(251,), (250,)] and live[0].is_cuda
        torch.cuda.synchronize()
        assert torch.equal(live[1].cpu(), x[753:] * 2)
        del before
    finally:
        sup.cleanup()
    # a kt.cls behind the seam: restart_procs re-creates the instance (fresh state)
    sup = _b3_supervisor(monkeypatch, "Scaler", {"num_proc": 3}, 3, init_args={"tag": "a"})
    try:
        inst = sup._callable
        assert inst.tag == "a"
        body = ref_dispatch.serialize_body(ref_dispatch.build_call_body(torch.arange(130), restart_procs=True), "pickle")
        got = ref_dispatch.deserialize_response(sup.call(req, "Scaler", "triple", body), "pickle")
        assert torch.equal(torch.cat(got), torch.arange(130) * 3) and sup._callable is not inst
        from kubetorch_b200.serving.codec import HTTPException
        with pytest.raises(HTTPException, match="Method 'nope' not found in class 'Scaler'"):
            sup.call(req, "Scaler", "nope", {"args": [], "kwargs": {}})
    finally:
        sup.cleanup()
    # json mode: tensors are not JSON-serialisable (the reference's SerializationError), scalars are
    sup = _b3_supervisor(monkeypatch, "shard_sum", {"num_proc": 4}, 4)
    try:
        xi = torch.arange(130)
        body = ref_dispatch.serialize_body(ref_dispatch.build_call_body(xi, 1, 0), "pickle")
        got = ref_dispatch.deserialize_response(sup.call(req, "shard_sum", None, body), "pickle")
        assert got == [int(c.sum()) for c in xi.chunk(4)]
        with pytest.raises(TypeError, match="is not an integer"):
            sup.call(req, "shard_sum", None, {"args": [xi, 0.5, 0], "kwargs": {}})
    finally:
        sup.cleanup()


def test_mapped_self_check_refuses_a_wrong_declaration(monkeypatch):
    from kubetorch_b200.serving.b200_supervisor import B200Supervisor

    monkeypatch.setenv("KT_FILE_PATH", os.path.join(os.path.dirname(__file__)))
    monkeypatch.setenv("KT_MODULE_NAME", "b3_user_module")
    monkeypatch.setenv("KT_CLS_OR_FN_NAME", "not_really_double")
    monkeypatch.setenv("KT_INIT_ARGS", "null")
    sup = B200Supervisor(num_proc=2, devices=[0, 0])
    with pytest.raises(ValueError, match="self-check failed"):
        sup.setup()
    sup.cleanup()
    import b3_user_module

    remote = kt.fn(b3_user_module.not_really_double, name="t-wrong")
    with pytest.raises(ValueError, match="self-check failed"):
        remote.to(kt.Compute(gpus=1).distribute("b200", num_proc=2, devices=[0, 0]))


# ---- (f4) kt.cls state and concurrency on GPU rank processes ------------------------------------------------------
def test_cls_on_gpu_ranks_keeps_owned_args_state_and_overlaps_calls():
    """A kt.cls on GPU rank processes: (a) a CUDA tensor ARGUMENT kept across calls still holds its own bytes after
    later calls reused the arg arena (the reference deserialises fresh tensors per call); (b) per-rank state persists
    and a re-deploy resets it (tests/test_distributed.py:115-128); (c) async methods overlap on one loop and sync
    methods run on the rank's thread pool (kt/serving/design.md:67-85)."""
    import asyncio
    import threading
    import time

    comp = kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute(
        "spmd", workers=1, num_proc=2, devices=[0, 0], arena_bytes=1 << 20)
    holder = kt.cls(cases.WeightHolder, name="t-holder").to(comp, init_args={"scale": 2})
    try:
        assert holder._supervisor.__class__.__name__ == "GpuSPMDSupervisor"
        a = torch.arange(4096, dtype=torch.float32).cuda()
        assert holder.keep(a, serialization="pickle") == [1, 1]
        other = torch.full((4096,), -7.0).cuda()
        assert holder.overwrite(other, serialization="pickle") == [float(other.sum())] * 2     # reuses the arena
        assert holder.keep(a * 3, serialization="pickle") == [2, 2]
        got = holder.kept_sum(serialization="pickle")
        assert got == [[float((a * 3).double().sum()) * 2, 2]] * 2, got
        holder.keep(a, serialization="pickle")
        holder.overwrite(other, serialization="pickle")
        holder.overwrite(other * 2, serialization="pickle")
        got = holder.kept_sum(serialization="pickle")
        assert got == [[float(a.double().sum()) * 2, 3]] * 2, got         # the kept arg was NOT overwritten
        # async methods overlap: 4 concurrent 0.25 s sleeps finish in well under 1 s
        async def burst():
            return await asyncio.gather(*[holder.slow_echo(i, 0.25, async_=True) for i in range(4)])

        t0 = time.perf_counter()
        res = asyncio.run(burst())
        dt_async = time.perf_counter() - t0
        assert res == [[i, i] for i in range(4)] and dt_async < 0.9, dt_async
        # sync methods from caller threads run concurrently on the ranks' thread pools
        out = [None] * 4

        def work(i):
            out[i] = holder.slow_sync(i, 0.25)

        ths = [threading.Thread(target=work, args=(i,)) for i in range(4)]
        t0 = time.perf_counter()
        [t.start() for t in ths]
        [t.join() for t in ths]
        assert out == [[i, i] for i in range(4)] and time.perf_counter() - t0 < 0.9
        # restart_procs re-creates the rank processes: state is gone
        assert holder.kept_sum(restart_procs=True, serialization="pickle") == [[None, 0]] * 2
    finally:
        holder.teardown()
    again = kt.cls(cases.WeightHolder, name="t-holder").to(comp, init_args={"scale": 5})   # a new deploy resets state
    try:
        assert again.kept_sum() == [[None, 0]] * 2
    finally:
        again.teardown()


def test_small_call_lane_is_indistinguishable_from_the_general_path(golden):
    """placement="auto": calls under 4 MiB take the small-call lane (one launch on the root, no body/endpoint/header
    work).  Same rank-ordered shards, dtypes and bits as the fan-out path and as the recorded reference results;
    everything the lane does not cover (host tensors, kwargs, non-contiguous, empty, int tensors with a fractional
    alpha) falls through to the general path with the general path's behaviour."""
    double = _mapped(cases.double, "scale", alpha=2.0)
    for world in (1, 3, 4):
        lane = _deploy(double, world, f"t-lane-{world}", placement="auto")
        spread = _deploy(double, world, f"t-spread-{world}", placement="ranks")
        try:
            assert lane._fast is not None and (spread._fast is None) == (world > 1)   # 1 rank: nothing to spread
            for name in ("f32_1003", "f32_3", "bf16_777", "i64_130", "i32_515"):
                x = golden["all_inputs"][name]
                want = ref_dispatch.spmd_call(cases.double, x, num_proc=world, serialization="pickle")
                a = lane(x.cuda(), serialization="pickle")
                b = spread(x.cuda(), serialization="pickle")
                assert len(a) == len(b) == len(want) == world
                for g, h, w in zip(a, b, want):
                    assert g.dtype == w.dtype and tuple(g.shape) == tuple(w.shape) == tuple(h.shape), (name, world)
                    assert torch.equal(g.cpu(), w) and torch.equal(h.cpu(), w), (name, world)
            x2 = torch.randn(10, 37)
            want = ref_dispatch.spmd_call(cases.double, x2, num_proc=world, serialization="pickle")
            got = lane(x2.cuda(), serialization="pickle")
            assert [tuple(g.shape) for g in got] == [tuple(w.shape) for w in want]
            assert all(torch.equal(g.cpu(), w) for g, w in zip(got, want))
            # fall-through cases behave as before
            host = lane(x2, serialization="pickle")
            assert all(torch.equal(g, w) for g, w in zip(host, want)) and not host[0].is_cuda
            nc = lane(x2.cuda().t().contiguous().t(), serialization="pickle")     # non-contiguous
            assert all(torch.equal(g.cpu(), w) for g, w in zip(nc, want))
            assert [g.numel() for g in lane(torch.empty(0).cuda(), serialization="pickle")] == [0] * world
            with pytest.raises(TypeError):
                lane(x2.cuda())          # default serialization is json: tensors are not JSON (same as the general path)
            lane.serialization = "pickle"
            assert torch.equal(torch.cat(lane(x2.cuda())).cpu(), x2 * 2)
        finally:
            lane.teardown()
            spread.teardown()
    half = _mapped(cases.scale, "scale", alpha=0.5)     # constant fractional alpha: int tensors must not take the lane

    def half_fn(x):
        return cases._shard(x) * 0.5

    half = kt.mapped("scale", alpha=0.5)(half_fn)
    r = _deploy(half, 2, "t-lane-half", placement="auto")
    try:
        with pytest.raises(TypeError, match="not an integer"):
            r(torch.arange(10).cuda(), serialization="pickle")
        assert torch.equal(torch.cat(r(torch.arange(10.0).cuda(), serialization="pickle")).cpu(), torch.arange(10.0) * 0.5)
    finally:
        r.teardown()


def test_broadcast_window_across_rank_processes_and_the_timeout_fault_case():
    """(f1) BroadcastWindow with participants in DIFFERENT rank processes (file rendezvous under KTB_STORE_DIR + CUDA-IPC
    arenas), and the reference's fault-injection pattern: a receive that can never complete fails with a timeout,
    leaves nothing behind, and the very next window on the same group id works (gpu_helper.py:607-670)."""
    n_dev = torch.cuda.device_count()
    world = 3
    devices = [r % n_dev for r in range(world)]
    comp = kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute(
        "spmd", workers=1, num_proc=world, devices=devices)
    win = kt.cls(cases.StoreWindows, name="t-bw-ranks").to(comp)
    try:
        out = win.fault(0.3, "bw-shared", serialization="pickle")
        assert all(o["expected_failure"] and "timed out with 0 putter(s)" in o["error"] for o in out), out
        for it in range(2):                       # same store, same group id as the failed window, twice
            n = 100_003 + it
            out = win.broadcast(n, world, 30.0, "bw-shared", serialization="pickle")
            want = float((torch.arange(n, dtype=torch.float32) * 0.5).sum())
            assert [o["role"] for o in out] == ["put", "get", "get"]
            assert all(o["world"] == world and o["b"] == [3] * 7 and o["sum"] == want for o in out), out
    finally:
        win.teardown()


def test_device_stall_maps_to_pod_terminated_error():
    """A rank whose piece never arrives (its peer stalled or died): the in-kernel wait gives up, the consume kernel stores
    NOTHING, the sticky status word reaches the host behind the next call and the caller gets the reference's
    PodTerminatedError (kt/serving/utils.py:111-190), not stale bytes."""
    import ctypes

    from kubetorch_b200.device import lib as L
    from kubetorch_b200.device import ops

    double = _mapped(cases.double, "scale", alpha=2.0)
    remote = kt.fn(double, name="t-stall").to(
        kt.Compute(gpus=1, allowed_serialization=["json", "pickle"]).distribute(
            "b200", workers=1, num_proc=2, devices=[0, 0], placement="ranks", transfer="push"))
    try:
        x = torch.arange(1 << 16, dtype=torch.float32).cuda()
        assert torch.equal(torch.cat(remote(x, serialization="pickle")).cpu(), x.cpu() * 2)
        sup = remote._supervisor
        sess = sup._push
        sess.set_spin_timeout(0.05)
        # sabotage: rank 1 is asked to consume call seq+1, which the root never scatters
        sentinel = torch.full((1 << 15,), -1.0, device="cuda:0")
        L.call("ktb_push_consume", 0, L.OP_SCALE, L.F32, sess.stage[1].data_ptr(), sess.stride, sentinel.data_ptr(),
               sentinel.numel(), 2.0, 0.0, sess.ctrl[1].data_ptr(), sess.ctrl[0].data_ptr(), 1, sess.n_chunks,
               ctypes.c_ulonglong(sess.seq + 1000), ops.current_stream_handle(0))
        torch.cuda.synchronize(0)
        assert bool((sentinel == -1.0).all())                     # a timed-out consumer writes nothing
        with pytest.raises(kt.PodTerminatedError) as ei:
            sup.check_device_health()
        assert ei.value.reason == "DeviceTimeout" and ei.value.status_code == 503
    finally:
        remote.teardown()


def test_map_coalesces_small_calls_and_equals_a_loop_of_calls(golden):
    """remote.map(xs) == [remote(x) for x in xs] — one segmented launch for the covered case, a plain loop otherwise."""
    double = _mapped(cases.double, "scale", alpha=2.0)
    for world in (1, 3):
        r = _deploy(double, world, f"t-map-{world}", placement="auto")
        try:
            assert r._batch is not None
            gen = torch.Generator().manual_seed(7)
            xs = [torch.randn(n, generator=gen).cuda() for n in (1, 3, 255, 256, 257, 1003, 4099)] * 40
            got = r.map(xs, serialization="pickle")
            want = [r(x, serialization="pickle") for x in xs]
            assert len(got) == len(want) == len(xs)
            for g, w, x in zip(got, want, xs):
                assert len(g) == len(w) == world
                assert all(a.dtype == b.dtype and tuple(a.shape) == tuple(b.shape) and torch.equal(a, b) for a, b in zip(g, w))
                assert torch.equal(torch.cat(g).cpu(), x.cpu() * 2)
            mixed = [torch.randn(5), torch.randn(7).cuda()]              # a host tensor in the list: plain loop, same results
            out = r.map(mixed, serialization="pickle")
            assert torch.equal(torch.cat(out[0]), mixed[0] * 2) and torch.equal(torch.cat(out[1]).cpu(), mixed[1].cpu() * 2)
            assert r.map([], serialization="pickle") == []
        finally:
            r.teardown()
