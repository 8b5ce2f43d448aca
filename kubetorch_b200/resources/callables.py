"""kt.fn / kt.cls / Module.to() / remote __call__ — the user-facing half of the path, with the
reference's signatures (kt/resources/callables/module.py:486-572, fn/fn.py:46-195,
cls/cls.py:54-215, utils.py:53-102,255-261) and a local bind instead of a Kubernetes deploy:
`.to(compute)` chooses a supervisor (in-process, rank processes, or the GPU device backend) and
starts it; no kubeconfig gate (module.py:529-532), no rsync, no controller.
"""
from __future__ import annotations

import inspect
import os
import re
from pathlib import Path
from typing import Any, Callable, Dict, List, Type, Union

from ..config import DebugConfig, config as kt_config
from ..mapped import mapped_spec
from ..serving.codec import SERIALIZATION_FORMATS
from ..serving.local_client import LocalClient
from ..serving.supervisor_factory import SPMD_TYPES, supervisor_factory


# ---- pointers & call body -----------------------------------------------------------------------------
def extract_pointers(raw_cls_or_fn: Union[Type, Callable]):
    """(root_path, module_name, qualname): enough for another Python process to import the callable."""
    if not (isinstance(raw_cls_or_fn, type) or callable(raw_cls_or_fn)):
        raise TypeError(f"Expected Type or Callable but received {type(raw_cls_or_fn)}")
    py_module = inspect.getmodule(raw_cls_or_fn)
    module_file = getattr(py_module, "__file__", None)
    name = getattr(raw_cls_or_fn, "__qualname__", raw_cls_or_fn.__name__)
    if not module_file or module_file.endswith("ipynb"):
        return os.getcwd(), "notebook", raw_cls_or_fn.__name__
    module_path = str(Path(module_file).resolve())
    root_path, module_name = os.path.dirname(module_path), inspect.getmodulename(module_path)
    package = getattr(py_module, "__package__", None)
    if package:
        top = __import__(package.split(".")[0])
        bases = [os.path.abspath(p) for p in getattr(top, "__path__", [])
                 if os.path.commonpath((os.path.abspath(p), module_path)) == os.path.abspath(p)]
        if len(bases) != 1:
            raise Exception("Wasn't able to find the package directory!")
        root_path = os.path.dirname(bases[0])
        spec = getattr(py_module, "__spec__", None)
        module_name = spec.name if spec is not None else py_module.__name__
    return root_path, module_name, name


def build_call_body(*args, debug: Union[bool, DebugConfig] = None, pdb=None, **kwargs):
    body = {"args": list(args), "kwargs": kwargs}
    if debug or pdb:
        if isinstance(debug, DebugConfig):
            dbg = debug
        elif debug is None or isinstance(debug, bool):
            port = 5678 if (pdb is None or isinstance(pdb, bool)) else pdb
            dbg = DebugConfig(port=port, mode=os.getenv("KT_DEBUG_MODE", "pdb").lower())
        else:
            raise ValueError(
                f"debug parameter must be a bool or DebugConfig instance, got {type(debug).__name__}. "
                "Use debug=True or debug=kt.DebugConfig(port=..., mode=...) instead."
            )
        body["debugger"] = dbg.to_dict()
    return body


def _clean_name(name: str) -> str:
    cleaned = re.sub(r"[^a-z0-9-]+", "-", name.lower().replace("_", "-")).strip("-")
    return cleaned[:63] or "kt-service"


# ---- Module ---------------------------------------------------------------------------------------------
class Module:
    MODULE_TYPE = None

    def __init__(self, name: str, pointers: tuple = None, sync_dir=None, remote_dir=None, remote_import_path: str = None):
        if sync_dir and remote_dir:
            raise ValueError(
                "sync_dir and remote_dir can not both be set. Use sync_dir to sync a local directory, or remote_dir "
                "to specify where files already exist on the container."
            )
        if remote_import_path and not remote_dir:
            raise ValueError("remote_import_path can only be set when remote_dir is also set. ")
        self._compute = None
        self._http_client = None
        self._supervisor = None
        self._fast = None
        self._batch = None
        self._fast_sers = frozenset()
        self._serialization = "json"
        self._async = False
        self._get_if_exists = True
        self._reload_prefixes = None
        self._root_path, self._import_path, self._callable_name = pointers
        self._callable_obj = None
        self.name = _clean_name(name) if name else None
        self.service_name = self.name
        self.sync_dir, self.remote_dir, self.remote_import_path = sync_dir, remote_dir, remote_import_path
        self.logging_config = None

    # -- properties mirrored from the reference -------------------------------------------------------------
    @property
    def callable_name(self):
        return self._callable_name

    @property
    def compute(self):
        return self._compute

    @compute.setter
    def compute(self, value):
        self._compute = value

    @property
    def serialization(self):
        return self._serialization

    @serialization.setter
    def serialization(self, value: str):
        if value not in SERIALIZATION_FORMATS:
            raise ValueError("Serialization must be 'json', 'pickle', or 'none'")
        self._serialization = value

    @property
    def async_(self):
        return self._async

    @async_.setter
    def async_(self, value: bool):
        if not isinstance(value, bool):
            raise ValueError("`async_` must be a boolean")
        self._async = value

    @property
    def stream_logs(self):
        lc = self.logging_config
        if lc is not None and lc.stream_logs is not None:
            return lc.stream_logs
        return bool(kt_config.stream_logs)

    @property
    def request_headers(self):
        return {}

    @property
    def reload_prefixes(self):
        return self._reload_prefixes or []

    @reload_prefixes.setter
    def reload_prefixes(self, value):
        if isinstance(value, list):
            self._reload_prefixes = value
        elif isinstance(value, str):
            self._reload_prefixes = [value]
        else:
            raise ValueError("`reload_prefixes` must be a string or a list.")

    @property
    def get_if_exists(self):
        return self._get_if_exists

    @get_if_exists.setter
    def get_if_exists(self, value):
        self._get_if_exists = value

    @property
    def base_endpoint(self):
        return f"local://{self.service_name}"

    def endpoint(self, method_name: str = None):
        if not hasattr(self, "init_args"):
            return f"{self.base_endpoint}/{self.callable_name}"
        return f"{self.base_endpoint}/{self.callable_name}/{method_name}"

    @classmethod
    def from_name(cls, name: str, namespace: str = None, reload_prefixes=None):
        mod = _DEPLOYED.get(_clean_name(name))
        if mod is None:
            raise ValueError(f"Service '{name}' not found in namespace '{namespace}' with reload_prefixes={reload_prefixes}")
        return mod

    # -- deploy = local bind ----------------------------------------------------------------------------------
    def _supervisor_config(self, compute, init_args) -> Dict[str, Any]:
        dist = dict(compute.distributed_config)
        dtype = dist.get("distribution_type") if dist else None
        target = self._callable_obj
        spec = mapped_spec(target) if target is not None and not inspect.isclass(target) else None
        backend = str(getattr(kt_config, "backend", "auto") or "auto")
        common = dict(pointers=(self._root_path, self._import_path, self._callable_name), init_args=init_args,
                      name=self.callable_name, allowed_serialization=compute.allowed_serialization_str)
        workers = int(dist.get("workers") or dist.get("quorum_workers") or compute.replicas or 1) if dist else 1
        num_proc = dist.get("num_proc") if dist else None

        use_b200 = dtype == "b200" or (spec is not None and compute.gpus and backend != "cpu"
                                       and dtype in (None, "spmd", "pytorch"))
        if use_b200:
            per_worker = None if num_proc in ("auto", None) and not compute.gpus else \
                (None if num_proc == "auto" else int(num_proc or compute.gpus or 1))
            extra = {k: dist[k] for k in ("devices", "transfer", "placement", "self_check") if dist and k in dist}
            return dict(distribution_type="b200", callable_obj=target, num_proc=per_worker, workers=workers,
                        distributed=bool(dist), **extra, **common)
        if dtype in SPMD_TYPES:
            extra = {k: v for k, v in dist.items()
                     if k not in ("distribution_type", "workers", "quorum_workers", "num_proc", "port",
                                  "quorum_timeout", "monitor_members")}
            gpu = bool(compute.gpus) and backend != "cpu"
            devices = extra.pop("devices", None)
            extra.pop("transfer", None)
            return dict(distribution_type=dtype, workers=workers, num_proc=num_proc, port=dist.get("port"),
                        env_vars={k: str(v) for k, v in compute.env_vars.items()}, gpu_arenas=gpu,
                        devices=devices, **extra, **common)
        if dtype not in (None, "local"):
            return dict(distribution_type=dtype, **common)  # factory raises the reference's error text
        return dict(distribution_type="local", callable_obj=target, **common)

    def to(self, compute, init_args: Dict = None, stream_logs: Union[bool, None] = None, get_if_exists: bool = False,
           reload_prefixes: Union[str, List[str]] = [], dryrun: bool = False):
        """Bind the function or class to `compute` (start its ranks). Returns self."""
        if get_if_exists:
            existing = _DEPLOYED.get(self.service_name)
            if existing is not None and existing._supervisor is not None:
                return existing
        if self._supervisor is not None:  # redeploy resets state (tests/test_distributed.py:115-128)
            self.teardown()
        self.compute = compute
        compute.service_name = self.service_name
        self.logging_config = compute.logging_config
        if hasattr(self, "init_args"):
            self.init_args = init_args
        if dryrun:
            return self
        cfg = self._supervisor_config(compute, init_args)
        dtype = cfg.pop("distribution_type")
        sup = supervisor_factory(dtype, **cfg)
        sup.setup()
        self._supervisor = sup
        self._http_client = LocalClient(sup, self.service_name)
        self._fast = None
        if hasattr(sup, "fast_path") and self.MODULE_TYPE == "fn":
            allowed = compute.allowed_serialization_str.split(",")
            self._fast_sers = frozenset(s for s in ("pickle", "none") if s in allowed)
            self._fast = sup.fast_path(bool(self._fast_sers))
            self._batch = sup.batch_path(bool(self._fast_sers)) if hasattr(sup, "batch_path") else None
        _DEPLOYED[self.service_name] = self
        return self

    async def to_async(self, compute, init_args: Dict = None, stream_logs=None, get_if_exists: bool = False,
                       reload_prefixes=[], dryrun: bool = False):
        import asyncio

        loop = asyncio.get_running_loop()
        return await loop.run_in_executor(
            None, lambda: self.to(compute, init_args, stream_logs, get_if_exists, reload_prefixes, dryrun))

    def deploy(self):
        if self.compute is None:
            raise ValueError("Compute must be set before deploying the module.")
        return self.to(self.compute, init_args=getattr(self, "init_args", None))

    def teardown(self):
        """Stop this module's ranks and release its device resources."""
        if self._supervisor is not None:
            self._supervisor.cleanup()
            self._supervisor = None
        self._http_client = None
        self._fast = self._batch = None
        _DEPLOYED.pop(self.service_name, None)

    def _client(self, *args, **kwargs):
        if self._http_client is None:
            raise ValueError(
                f"Service '{self.service_name}' is not deployed: call .to(kt.Compute(...)) before invoking it"
            )
        return self._http_client

    def _pop_call_options(self, kwargs):
        stream_logs = kwargs.pop("stream_logs", None)
        stream_metrics = kwargs.pop("stream_metrics", None)
        debug = kwargs.pop("debug", None)
        pdb = kwargs.pop("pdb", None)
        serialization = kwargs.pop("serialization", self.serialization)
        if debug is None and pdb is not None:
            debug = pdb
        stream_logs = stream_logs if stream_logs is not None else self.stream_logs
        return stream_logs, stream_metrics, debug, pdb, serialization


_DEPLOYED: Dict[str, Module] = {}


# ---- Fn -----------------------------------------------------------------------------------------------------
class Fn(Module):
    MODULE_TYPE = "fn"

    def __call__(self, *args, **kwargs):
        fast = self._fast
        if fast is not None and len(args) == 1 and not self._async:
            # small-call lane: one tensor argument, at most the `serialization` option, a format that may carry tensors
            if (not kwargs and self._serialization in self._fast_sers) or \
                    (len(kwargs) == 1 and kwargs.get("serialization") in self._fast_sers):
                out = fast(args[0])
                if out is not None:
                    return out
        async_ = kwargs.pop("async_", self.async_)
        return self._call_async(*args, **kwargs) if async_ else self._call_sync(*args, **kwargs)

    def _call_sync(self, *args, **kwargs):
        client = self._client()
        stream_logs, stream_metrics, debug, pdb, serialization = self._pop_call_options(kwargs)
        body = build_call_body(*args, **kwargs, debug=debug, pdb=pdb)
        return client.call_method(self.endpoint(), stream_logs, self.logging_config, stream_metrics=stream_metrics,
                                  headers=self.request_headers, body=body, serialization=serialization)

    async def _call_async(self, *args, **kwargs):
        client = self._client()
        stream_logs, stream_metrics, debug, pdb, serialization = self._pop_call_options(kwargs)
        body = build_call_body(*args, **kwargs, debug=debug, pdb=pdb)
        return await client.call_method_async(self.endpoint(), stream_logs, self.logging_config,
                                              stream_metrics=stream_metrics, headers=self.request_headers, body=body,
                                              serialization=serialization)

    def map(self, inputs, **kwargs):
        """`[remote(x, **kwargs) for x in inputs]` — the results are exactly those — but a run of small device-resident
        tensors for a @kt.mapped element-wise function is coalesced into ONE segmented kernel launch (not in the
        reference's API: its remote-map is one HTTP call per item)."""
        inputs = list(inputs)
        batch = self._batch
        ser = kwargs.get("serialization", self._serialization)
        if batch is not None and not self._async and ser in self._fast_sers and set(kwargs) <= {"serialization"}:
            out = batch(inputs)
            if out is not None:
                return out
        return [self(x, **kwargs) for x in inputs]


def fn(function_obj=None, name: str = None, get_if_exists=True, reload_prefixes=None, sync_dir=None, remote_dir=None,
       remote_import_path: str = None) -> Fn:
    """Builds an instance of :class:`Fn` (same signature as the reference's kt.fn)."""
    if function_obj:
        pointers = extract_pointers(function_obj)
        name = name or pointers[2] or function_obj.__name__
        new_fn = Fn(name=name, pointers=pointers, sync_dir=sync_dir, remote_dir=remote_dir,
                    remote_import_path=remote_import_path)
        new_fn._callable_obj = function_obj
        new_fn.get_if_exists = get_if_exists
        new_fn.reload_prefixes = reload_prefixes or []
        return new_fn
    if name is None:
        raise ValueError("Name must be provided to reload an existing function")
    if get_if_exists is False:
        raise ValueError(
            "Either provide a function object or a name with get_if_exists=True to reload an existing function"
        )
    return Fn.from_name(name, reload_prefixes=reload_prefixes)


# ---- Cls ----------------------------------------------------------------------------------------------------
class Cls(Module):
    MODULE_TYPE = "cls"

    def __init__(self, name: str, pointers: tuple = None, init_args: dict = None, sync_dir=None, remote_dir=None,
                 remote_import_path: str = None):
        self._init_args = init_args
        super().__init__(name=name, pointers=pointers, sync_dir=sync_dir, remote_dir=remote_dir,
                         remote_import_path=remote_import_path)

    @property
    def init_args(self):
        return self._init_args

    @init_args.setter
    def init_args(self, value):
        self._init_args = value

    def __getattr__(self, attr_name) -> Any:
        if attr_name.startswith("_") or attr_name in _CLS_RESERVED:
            raise AttributeError(attr_name)

        def remote_method_wrapper(*args, **kwargs):
            async_ = kwargs.pop("async_", self.async_)
            if async_:
                return self._call_async(attr_name, *args, **kwargs)
            return self._call_sync(attr_name, *args, **kwargs)

        return remote_method_wrapper

    def _call_sync(self, method_name, *args, **kwargs):
        client = self._client(method_name=method_name)
        stream_logs, stream_metrics, debug, pdb, serialization = self._pop_call_options(kwargs)
        body = build_call_body(*args, **kwargs, debug=debug, pdb=pdb)
        return client.call_method(self.endpoint(method_name), stream_logs, self.logging_config,
                                  stream_metrics=stream_metrics, headers=self.request_headers, body=body,
                                  serialization=serialization)

    async def _call_async(self, method_name, *args, **kwargs):
        client = self._client(method_name=method_name)
        stream_logs, stream_metrics, debug, pdb, serialization = self._pop_call_options(kwargs)
        body = build_call_body(*args, **kwargs, debug=debug, pdb=pdb)
        return await client.call_method_async(self.endpoint(method_name), stream_logs, self.logging_config,
                                              stream_metrics=stream_metrics, headers=self.request_headers, body=body,
                                              serialization=serialization)


_CLS_RESERVED = set(dir(Module)) | {"init_args", "sync_dir", "remote_dir", "remote_import_path", "name",
                                    "service_name", "logging_config"}


def cls(class_obj=None, name: str = None, get_if_exists=True, reload_prefixes=None, sync_dir=None, remote_dir=None,
        remote_import_path: str = None) -> Cls:
    """Builds an instance of :class:`Cls` (same signature as the reference's kt.cls)."""
    if class_obj:
        pointers = extract_pointers(class_obj)
        name = name or pointers[2] or class_obj.__name__
        new_cls = Cls(name=name, pointers=pointers, sync_dir=sync_dir, remote_dir=remote_dir,
                      remote_import_path=remote_import_path)
        new_cls._callable_obj = class_obj
        new_cls.get_if_exists = get_if_exists
        new_cls.reload_prefixes = reload_prefixes or []
        return new_cls
    if name is None:
        raise ValueError("Name must be provided to reload an existing class")
    if get_if_exists is False:
        raise ValueError("Either provide a class object or a name with get_if_exists=True to reload an existing class")
    return Cls.from_name(name, reload_prefixes=reload_prefixes)
