"""User callables of the parity cases, written exactly as a kubetorch user writes SPMD functions:
they read RANK / WORLD_SIZE from the environment the reference's worker sets
(kt/serving/process_worker.py:75-102,128-129) and shard their own input.

TEST INFRASTRUCTURE.  These functions are the *semantic definition* of the registered device
ops: the reference runtime (oracle/make_golden.py) and the oracle restatement
(oracle/ref_dispatch.py) execute them on CPU; the CUDA path must reproduce their results.
"""
import os


def _rank_world():
    return int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])


def _shard(x):
    """`x.chunk(WORLD_SIZE)[RANK]` with the empty shard torch.chunk omits for ranks past the data."""
    r, w = _rank_world()
    chunks = x.chunk(w)  # along dim 0
    return chunks[r] if r < len(chunks) else x[:0]


# ---- reference test assets restated (tests/assets/*/.py) -------------------------------------------
def summer(a, b):
    return a + b


def torch_summer(a, b):
    import torch

    return int(torch.sum(torch.tensor([a, b])))


async def async_summer(a, b, sleep_time=0.01, return_times=False):
    import asyncio

    await asyncio.sleep(sleep_time)
    return a + b


def hello_world():
    return "Hello from Kubetorch!"


class Number:
    def __init__(self, size=5):
        self.size = size
        self.calls = 0

    def add(self, x, y):
        self.calls += 1
        return x + y

    def count(self):
        return self.calls


def env_report():
    keys = ["WORLD_SIZE", "RANK", "LOCAL_RANK", "NODE_RANK", "POD_IPS", "MASTER_ADDR", "MASTER_PORT"]
    return {k: os.environ.get(k) for k in keys}


def env_get(name):
    return os.environ.get(name)


def raise_value_error(msg):
    raise ValueError(msg)


# ---- mapped-callable semantics (BASELINE configs C2 / C5 and variants) ------------------------------
def identity(x):
    return _shard(x)


def double(x):
    return _shard(x) * 2


def scale(x, alpha):
    return _shard(x) * alpha


def affine(x, alpha, beta):
    return _shard(x) * alpha + beta


def shard_sum(x, alpha=1, beta=0):
    """Gather-reduce variant: each rank returns the sum of its mapped shard.

    Floating-point shards are summed in fp32 after the op has rounded each element to the tensor dtype, so a
    bf16 or fp16 sum does not round or overflow in the 2-byte dtype; integer shards are summed in int64."""
    import torch

    y = _shard(x) * alpha + beta if (alpha != 1 or beta != 0) else _shard(x)
    if y.dtype in (torch.float32, torch.bfloat16, torch.float16):
        return float(y.float().sum())
    return int(y.sum())


def spmd_identity(x):
    """Reference broadcast semantics: every rank sees (and returns) the full argument."""
    return x


def mlp_policy(obs, w1, w2, w3):
    """bf16 MLP policy of BASELINE config C4 on this rank's shard of observations (rows)."""
    import torch

    r, w = _rank_world()
    rows = obs.chunk(w, dim=0)
    o = rows[r] if r < len(rows) else obs[:0]
    h = torch.relu(o @ w1.t())
    h = torch.relu(h @ w2.t())
    return h @ w3.t()


def torch_ddp(epochs):
    """DDP smoke callable with the shape of the reference asset (tests/assets/torch_ddp/torch_ddp.py):
    gloo process group from the env contract, a tiny DDP-wrapped Linear, `epochs` SGD steps."""
    import torch
    from torch.nn.parallel import DistributedDataParallel as DDP

    if not torch.distributed.is_initialized():
        torch.distributed.init_process_group(backend="gloo")
    model = DDP(torch.nn.Linear(10, 1))
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    for _ in range(epochs):
        opt.zero_grad()
        model(torch.randn(10)).sum().backward()
        opt.step()
    return "Success"


def all_reduce_rank():
    """Sum of ranks through a gloo all_reduce (tests/test_distributed.py:259-260 expects 6.0 at world 4)."""
    import torch

    if not torch.distributed.is_initialized():
        torch.distributed.init_process_group(backend="gloo")
    t = torch.tensor([float(os.environ["RANK"])])
    torch.distributed.all_reduce(t)
    return float(t.item())


def mixed_payload(x, meta, scale=1):
    """Arbitrary Python over a pytree of tensors and plain objects (no registered kernel):
    returns this rank's view of the inputs."""
    r, w = _rank_world()
    return {"rank": r, "sum": x.sum() * scale, "y": meta["t"] + r, "tag": meta["tag"], "shape": list(x.shape)}


def store_put_by_rank(n):
    """Every rank publishes a tensor filled with its rank (tests/assets/kv_store/gpu_helper.py:303-351 pattern)."""
    import torch

    import kubetorch_b200 as kt

    r, _ = _rank_world()
    t = torch.full((n,), float(r), device=f"cuda:{torch.cuda.current_device()}")
    kt.put(key=f"by-rank/{r}", src=t)
    _KEEP.append(t)
    return r


def store_get_from_rank(src_rank, n):
    """Every rank fetches the tensor another rank published; returns (sum, listing)."""
    import torch

    import kubetorch_b200 as kt

    dest = torch.zeros(n, device=f"cuda:{torch.cuda.current_device()}")
    kt.get(key=f"by-rank/{src_rank}", dest=dest)
    torch.cuda.synchronize()
    return [float(dest.sum()), kt.ls("by-rank")]


def store_broadcast(n, world_size, timeout=30.0, group_id="bw-ranks"):
    """One BroadcastWindow across the rank processes (tests/assets/kv_store/gpu_helper.py broadcast patterns): rank 0
    puts a state dict, every other rank gets it into its own GPU tensors; returns this rank's view."""
    import torch

    import kubetorch_b200 as kt

    r, _ = _rank_world()
    dev = f"cuda:{torch.cuda.current_device()}"
    bw = kt.BroadcastWindow(world_size=world_size, timeout=timeout, group_id=group_id)
    if r == 0:
        sd = {"w": torch.arange(n, dtype=torch.float32, device=dev) * 0.5, "b": torch.full((7,), 3, dtype=torch.int64, device=dev)}
        _KEEP.append(sd)
        info = kt.put(key="bw/sd", src=sd, broadcast=bw)
        return {"role": "put", "world": info["world_size"], "sum": float(sd["w"].sum()), "b": sd["b"].tolist()}
    dest = {"w": torch.zeros(n, dtype=torch.float32, device=dev), "b": torch.zeros(7, dtype=torch.int64, device=dev)}
    info = kt.get(key="bw/sd", dest=dest, broadcast=bw)
    torch.cuda.synchronize()
    return {"role": "get", "world": info["world_size"], "sum": float(dest["w"].sum()), "b": dest["b"].tolist()}


def store_broadcast_without_putter(timeout=0.3, group_id="bw-ranks"):
    """The fault case (gpu_helper.py:607-670): a window that can never close fails with a timeout on every
    participant ... and the store stays usable (the caller runs store_broadcast on the same group right after)."""
    import torch

    import kubetorch_b200 as kt

    dest = torch.zeros(4, device=f"cuda:{torch.cuda.current_device()}")
    try:
        kt.get(key="bw/never", dest=dest, broadcast=kt.BroadcastWindow(world_size=99, timeout=timeout, group_id=group_id))
    except kt.DataStoreError as e:
        return {"expected_failure": True, "error": str(e)}
    return {"expected_failure": False}


class StoreWindows:
    """Both window patterns on ONE deployment (one store): the fault case first, then real broadcasts."""

    def fault(self, timeout=0.3, group_id="bw-ranks"):
        return store_broadcast_without_putter(timeout, group_id)

    def broadcast(self, n, world_size, timeout=30.0, group_id="bw-ranks"):
        return store_broadcast(n, world_size, timeout, group_id)


_KEEP = []


# ---- pydantic payloads (kt tests/test_deployment_fixtures.py:116-205, tests/utils.py:83-86,254-290) -------------
try:
    from pydantic import BaseModel

    class PairModel(BaseModel):
        name: str
        value: int

    class OSInfoRequest(BaseModel):
        method: str

    class OSInfoResponse(BaseModel):
        name: str
        value: str
except ImportError:  # pragma: no cover - pydantic is in the image
    BaseModel = PairModel = OSInfoRequest = OSInfoResponse = None


def model_summer(a, b):
    """`summer` as the reference's test utilities write it: Pydantic models in → a model of the same type out."""
    model_type = type(a) if hasattr(a, "model_dump") else None
    a = a.value if hasattr(a, "model_dump") else a
    b = b.value if hasattr(b, "model_dump") else b
    if model_type is not None:
        return model_type(name="sum_result", value=a + b)
    return a + b


class OSInfo:
    """Stateful class with model-typed arguments and results (the reference's ResourceHungryGremlin.os_info shape)."""

    def __init__(self, size=3):
        self.size = size

    def cpu_count(self):
        import os

        return os.cpu_count()

    def size_minus_cpus(self):
        import os

        return self.size - os.cpu_count()

    def os_info(self, requests):
        import os

        out = []
        for req in requests:
            if req.method == "uname":
                out.append(OSInfoResponse(name="uname", value=str(os.uname())))
            elif req.method == "cpu_count":
                out.append(OSInfoResponse(name="cpu_count", value=str(os.cpu_count())))
            elif req.method == "getpid":
                out.append(OSInfoResponse(name="getpid", value=str(os.getpid())))
        return out


# ---- stateful GPU ranks (kt.cls on rank processes; reference: tests/test_http_server.py:484-599, test_distributed.py:92-193)
class WeightHolder:
    """Keeps a tensor ARGUMENT across calls (the `self.weights = state_dict` pattern) and counts its calls."""

    def __init__(self, scale=1):
        self.scale = scale
        self.kept = None
        self.calls = 0

    def keep(self, t):
        self.calls += 1
        self.kept = t
        return self.calls

    def kept_sum(self):
        """[sum of the kept tensor * scale, number of keep() calls]; the kept tensor must still hold ITS bytes."""
        self_sum = None if self.kept is None else float(self.kept.double().sum()) * self.scale
        return [self_sum, self.calls]

    def overwrite(self, t):
        """Another tensor-carrying call between keep() and kept_sum(): must not disturb the kept tensor."""
        return float(t.double().sum())

    async def slow_echo(self, x, sleep_time=0.2):
        import asyncio

        await asyncio.sleep(sleep_time)
        return x

    def slow_sync(self, x, sleep_time=0.2):
        import time

        time.sleep(sleep_time)
        return x
