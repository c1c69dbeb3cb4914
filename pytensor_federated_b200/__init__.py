"""GPU-native federated log-probability / gradient engine.

The top level offers the names a user of the reference imports from ``pytensor_federated``
(``pytensor_federated/__init__.py:1-22``) plus, lazily, the engine-side entry points
(``FederatedEngine``, ``NodeFederation``, ``launch_federation``, ``DynamicBatcher``).  Nodes need neither
PyTensor nor torch to import this package: the graph Ops come from the backend shim
(:mod:`._graph_backend`) and everything GPU-related is imported on first use.
"""
import importlib

__version__ = "0.1.0"

# -- transport, wrappers, type aliases: always available ------------------------------------------------
from .signatures import ComputeFunc, LogpFunc, LogpGradFunc  # noqa: E402
from .service import ArraysToArraysService, ArraysToArraysServiceClient  # noqa: E402
from .common import LogpGradServiceClient, LogpServiceClient, wrap_logp_func, wrap_logp_grad_func  # noqa: E402

__all__ = [
    "ComputeFunc", "LogpFunc", "LogpGradFunc",
    "ArraysToArraysService", "ArraysToArraysServiceClient",
    "LogpServiceClient", "LogpGradServiceClient", "wrap_logp_func", "wrap_logp_grad_func",
]

# -- graph Ops: present whenever a graph backend can be imported (built-in IR or PyTensor) ----------------
_GRAPH_NAMES = {
    "AsyncOp": "op_async",
    "ArraysToArraysOp": "wrapper_ops",
    "AsyncArraysToArraysOp": "wrapper_ops",
    "LogpOp": "wrapper_ops",
    "AsyncLogpOp": "wrapper_ops",
    "LogpGradOp": "wrapper_ops",
    "AsyncLogpGradOp": "wrapper_ops",
}
try:
    for _name, _module in _GRAPH_NAMES.items():
        globals()[_name] = getattr(importlib.import_module(f".{_module}", __name__), _name)
    __all__ += list(_GRAPH_NAMES)
except ModuleNotFoundError:  # a node without any graph backend still serves compute functions
    pass

# -- engine-side names: resolved on first access (they pull in torch) -------------------------------------
_LAZY = {
    "FederatedEngine": "parallel",
    "FederationError": "parallel",
    "FederationTimeout": "parallel",
    "NodeFederation": "federation",
    "launch_federation": "federation",
    "DynamicBatcher": "batching",
    "FederatedLogpGradOp": "wrapper_ops",
}


def __getattr__(name):
    module = _LAZY.get(name)
    if module is None:
        raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
    value = getattr(importlib.import_module(f".{module}", __name__), name)
    globals()[name] = value
    return value


def __dir__():
    return sorted(set(globals()) | set(_LAZY))
