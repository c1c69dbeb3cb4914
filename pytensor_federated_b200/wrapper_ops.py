"""Ops that put federated functions into a differentiable graph.

Capabilities of ``pytensor_federated/wrapper_ops.py``: ``ArraysToArraysOp``
(``:14-33``), ``LogpOp`` (``:44-69``), ``LogpGradOp`` with its ``grad`` (``:84-132``) and their
``Async*`` twins (``:36-41``, ``:72-81``, ``:135-146``).  ``make_node`` arities, output types and
the ``grad`` contract are the reference's, so a PyMC model that used its ``LogpGradOp`` compiles
unchanged; the implementation is new and adds :class:`FederatedLogpGradOp`, whose sibling applies
inside one fused node are answered by a single multi-GPU engine launch.
"""
from __future__ import annotations

from typing import Any, Callable, List, Optional, Sequence, Union

import numpy as np

from ._graph_backend import Apply, DisconnectedType, FromFunctionOp, Op, Variable, at
from .op_async import AsyncFromFunctionOp, AsyncOp, FusableAsyncOp
from .signatures import ComputeFunc, LogpFunc, LogpGradFunc

OutputStorageType = List[List[Optional[Any]]]
TensorLike = Union[Variable, int, float, np.ndarray]


def _as_tensors(inputs) -> List[Variable]:
    return [at.as_tensor(i) for i in inputs]


class ArraysToArraysOp(FromFunctionOp):
    """``FromFunctionOp`` under the package's name; inputs may be plain numbers/arrays."""

    def __init__(self, compute_func: ComputeFunc, itypes: Sequence, otypes: Sequence,
                 infer_shape: Optional[Callable] = None):
        super().__init__(compute_func, itypes, otypes, infer_shape)

    def make_node(self, *inputs: TensorLike) -> Apply:
        return super().make_node(*_as_tensors(inputs))


class AsyncArraysToArraysOp(AsyncFromFunctionOp):
    """Async equivalent of :class:`ArraysToArraysOp` (``compute_func`` is a coroutine function)."""

    def make_node(self, *inputs: TensorLike) -> Apply:
        return super().make_node(*_as_tensors(inputs))


class LogpOp(Op):
    """Wraps a callable returning a scalar log-potential (no gradient)."""

    def __init__(self, logp_func: LogpFunc) -> None:
        self._logp_func = logp_func
        super().__init__()

    def make_node(self, *inputs: TensorLike) -> Apply:
        return Apply(self, _as_tensors(inputs), [at.scalar()])

    def perform(self, node: Apply, inputs: Sequence[np.ndarray], output_storage: OutputStorageType) -> None:
        output_storage[0][0] = self._logp_func(*inputs)


class AsyncLogpOp(AsyncOp, LogpOp):
    """:class:`LogpOp` whose ``logp_func`` is a coroutine function (e.g. ``LogpServiceClient.evaluate_async``);
    several of them in one graph are awaited concurrently after the ``fuse_asyncs`` rewrite."""

    async def perform_async(self, node: Apply, inputs: Sequence[Any], output_storage: OutputStorageType) -> None:
        output_storage[0][0] = await self._logp_func(*inputs)


class LogpGradOp(Op):
    """Wraps a callable returning a log-potential AND its gradient w.r.t. every input.

    Outputs: ``[logp, d logp / d input_0, ...]`` — one gradient per input, typed like the input.
    ``grad()`` hands those gradient outputs to the autodiff, so differentiating the log-potential
    costs no extra remote call: the second application below is merged with the forward one.
    """

    def __init__(self, logp_grad_func: LogpGradFunc) -> None:
        self._logp_grad_func = logp_grad_func
        super().__init__()

    def make_node(self, *inputs: TensorLike) -> Apply:
        tensors = _as_tensors(inputs)
        return Apply(self, tensors, [at.scalar(), *[t.type() for t in tensors]])

    @staticmethod
    def _store(result, output_storage: OutputStorageType) -> None:
        logp, gradient = result
        output_storage[0][0] = logp
        for g, value in enumerate(gradient):
            output_storage[1 + g][0] = value

    def perform(self, node: Apply, inputs: Sequence[np.ndarray], output_storage: OutputStorageType) -> None:
        self._store(self._logp_grad_func(*inputs), output_storage)

    def grad(self, inputs: Sequence[Variable], output_grads: List[Variable]) -> List[Variable]:
        g_logp, *g_grads = output_grads
        # Second derivatives are not available from the federated function: nobody may
        # differentiate through the gradient outputs.
        for i, g in enumerate(g_grads):
            if not isinstance(g.type, DisconnectedType):
                raise ValueError(f"Can't propagate gradients wrt parameter {i + 1}")
        _, *gradients = self(*inputs)
        return [g_logp * g for g in gradients]


class AsyncLogpGradOp(AsyncOp, LogpGradOp):
    """:class:`LogpGradOp` whose ``logp_grad_func`` is a coroutine function (e.g.
    ``LogpGradServiceClient.evaluate_async``); fusable into a :class:`ParallelAsyncOp`."""

    async def perform_async(self, node: Apply, inputs: Sequence[Any], output_storage: OutputStorageType) -> None:
        self._store(await self._logp_grad_func(*inputs), output_storage)


class FederatedLogpGradOp(FusableAsyncOp, LogpGradOp):
    """``LogpGradOp`` bound to ONE shard ("node") of a GPU federation.

    ``federation`` is a :class:`pytensor_federated_b200.federation.NodeFederation`; ``node`` the
    shard index.  Evaluated alone it asks the engine for that node's ``(logp, grads)``.  When the
    ``fuse_asyncs`` rewrite has put several such applies (same federation) into one
    :class:`ParallelAsyncOp`, they are all answered by a single fused broadcast->compute->reduce
    launch across the GPUs — the GPU-native replacement of N concurrent gRPC round trips
    (``pytensor_federated/op_async.py:114-130``).
    """

    def __init__(self, federation, node: int) -> None:
        self.federation = federation
        self.node = int(node)
        LogpGradOp.__init__(self, lambda *inputs: federation.evaluate_node(self.node, *inputs))

    def fusion_key(self):
        return ("federation", id(self.federation))

    async def perform_async(self, node: Apply, inputs: Sequence[Any], output_storage: OutputStorageType) -> None:
        self._store(self.federation.evaluate_node(self.node, *inputs), output_storage)

    async def perform_fused(self, members) -> None:
        self.perform_fused_sync(members)

    def perform_fused_sync(self, members) -> None:
        requests = {apply.op.node: list(ins) for apply, ins, _ in members}
        results = self.federation.evaluate_nodes(requests)
        for apply, _, outs in members:
            self._store(results[apply.op.node], outs)


__all__ = [
    "ArraysToArraysOp",
    "AsyncArraysToArraysOp",
    "LogpOp",
    "AsyncLogpOp",
    "LogpGradOp",
    "AsyncLogpGradOp",
    "FederatedLogpGradOp",
]
