"""kubetorch_b200 — a Hopper-native dispatch backend for kubetorch's data-parallel remote-call
path.  `import kubetorch_b200 as kt` is a drop-in for the subset of `import kubetorch as kt` on
that path: kt.Compute / kt.fn / kt.cls / .to() / .distribute() / remote __call__
(exports mirror kt/__init__.py:1-36), with `kt.Compute(gpus=N)` bound to N local H100s.
"""
from . import distributed  # noqa: F401
from .data_store import BroadcastWindow, get, ls, put, rm  # noqa: F401
from .config import DebugConfig, LoggingConfig, MetricsConfig, config  # noqa: F401
from .exceptions import (  # noqa: F401
    EXCEPTION_REGISTRY,
    ControllerRequestError,
    DataStoreError,
    ImagePullError,
    KnativeServiceConflictError,
    KubernetesCredentialsError,
    NotebookError,
    PodContainerError,
    PodTerminatedError,
    ResourceNotAvailableError,
    RsyncError,
    SecretNotFound,
    SerializationError,
    ServiceHealthError,
    ServiceTimeoutError,
    StartupError,
    VersionMismatchError,
    WorkerMembershipChanged,
)
from .mapped import mapped, mapped_spec  # noqa: F401
from .sampling import explore_noise, gumbel_noise, normal_noise, replay_noise  # noqa: F401
from .resources.callables import Cls, Fn, Module, cls, fn  # noqa: F401
from .resources.compute import Compute  # noqa: F401
from .resources.decorators import async_, autoscale, compute, distribute  # noqa: F401
from .resources.inert import Image, Secret, Volume, images, secret  # noqa: F401  (call-site stand-ins, see inert.py)



def pinned_empty(shape, dtype=None, gpus=None, devices=None, module=None):
    """Uninitialised PINNED host tensor for host-resident calls.  With `module=<deployed kt.fn>` (the GPUs that
    deployment's ranks run on), `gpus=N` or explicit `devices`, the pages of `x.chunk(N)[r]` are placed on the NUMA node
    of rank r's GPU, so a sharded call moves every shard over its own socket's memory controllers and its own GPU's
    PCIe link (ktb_host_alloc_sharded)."""
    import torch

    from .device import ops

    if module is not None and getattr(getattr(module, "_supervisor", None), "devices", None):
        devices = module._supervisor.devices
    devs = list(devices) if devices is not None else (list(range(int(gpus))) if gpus else None)
    return ops.pinned_empty(shape, dtype or torch.float32, devices=devs)


for _exc in EXCEPTION_REGISTRY.values():
    _exc.__module__ = "kubetorch_b200"

__version__ = "0.1.0"
