"""Asynchronous Ops and the graph rewrite that runs independent ones concurrently.

Capabilities of ``pytensor_federated/op_async.py``:

* ``AsyncOp`` — an Op whose computation is a coroutine (``perform_async``); the synchronous
  ``perform`` drives it on a re-entrant event loop (``:16-34``).
* ``AsyncFromFunctionOp`` — wraps ``async def fn(*arrays)`` (``:37-65``).
* ``ParallelAsyncOp`` — one node that awaits the coroutines of several child applies at once
  (``:68-132``).
* ``find_parallelizable_applies`` / ``parallelize_async_applies`` /
  ``parallelize_all_async_applies`` and the ``fuse_asyncs`` rewriter registered for
  ``fast_run`` at position 90 (``:135-234``).

Differences on purpose:

* Exceptions raised by a child are **re-raised** after all children finished (the reference
  gathers with ``return_exceptions=True`` and never looks at the results, ``:127-130``, so a
  failed remote call silently leaves stale values in the output storage).
* Children that share a *fusable engine* (a GPU federation) are evaluated by one fused launch
  instead of N awaits — see :class:`FusableAsyncOp`.
"""
from __future__ import annotations

import asyncio
from typing import Any, Callable, List, Optional, Sequence

from ._graph_backend import (
    Apply,
    FromFunctionOp,
    FunctionGraph,
    GraphRewriter,
    Op,
    ReplaceValidate,
    Variable,
    optdb,
)
from .utils import get_useful_event_loop

OutputStorageType = List[List[Optional[Any]]]


class AsyncOp(Op):
    """Base class: implement :meth:`perform_async`; ``perform`` blocks on it."""

    def perform(self, node: Apply, inputs: Sequence[Any], output_storage: OutputStorageType) -> None:
        loop = get_useful_event_loop()
        loop.run_until_complete(self.perform_async(node, inputs, output_storage))

    async def perform_async(self, node: Apply, inputs: Sequence[Any], output_storage: OutputStorageType) -> None:
        raise NotImplementedError()


class AsyncFromFunctionOp(AsyncOp, FromFunctionOp):
    """Async twin of ``FromFunctionOp``: ``fn`` is a coroutine function of arrays.

    ``AsyncOp.perform`` wins over ``FromFunctionOp.perform`` by MRO.
    """

    def __init__(self, fn: Callable, itypes: Sequence, otypes: Sequence, infer_shape: Optional[Callable] = None):
        self._async_fn = fn
        super().__init__(fn, itypes, otypes, infer_shape)

    async def perform_async(self, node: Apply, inputs: Sequence[Any], output_storage: OutputStorageType) -> None:
        outs = await self._async_fn(*inputs)
        if not isinstance(outs, (list, tuple)):
            outs = (outs,)
        if len(outs) != len(output_storage):
            raise ValueError(f"Function returned {len(outs)} outputs, the Op declares {len(output_storage)}.")
        for cell, value in zip(output_storage, outs):
            cell[0] = value


class ParallelAsyncError(RuntimeError):
    """Several children of one :class:`ParallelAsyncOp` failed; ``errors`` holds all of them
    (a single failure is re-raised as it is, so its type stays catchable)."""

    def __init__(self, errors: Sequence[BaseException]) -> None:
        self.errors = list(errors)
        summary = "; ".join(f"{type(e).__name__}: {e}" for e in self.errors)
        super().__init__(f"{len(self.errors)} parallel async children failed: {summary}")


class ParallelAsyncOp(AsyncOp):
    """Runs the ``perform_async`` of several ``AsyncOp`` apply nodes concurrently.

    Inputs/outputs are the concatenation of the children's inputs/outputs, in order.
    """

    def __init__(self, applies: Sequence[Apply]) -> None:
        applies = tuple(applies)
        for a, apply in enumerate(applies):
            if not isinstance(apply.op, AsyncOp):
                raise ValueError(
                    f"Cannot run {type(apply.op).__name__} concurrently: apply node {a} is not an `AsyncOp` application."
                )
        self.applies = applies
        super().__init__()

    def make_node(self, *inputs: Variable) -> Apply:
        nin_exp = sum(a.nin for a in self.applies)
        if len(inputs) != nin_exp:
            raise ValueError(
                f"`ParallelAsyncOp` received {len(inputs)} inputs, expected {nin_exp} for {len(self.applies)} children."
            )
        outputs = [out.type() for app in self.applies for out in app.outputs]
        return Apply(self, list(inputs), outputs)

    def _slices(self, inputs, output_storage):
        ifrom = ofrom = 0
        for apply in self.applies:
            yield apply, inputs[ifrom : ifrom + apply.nin], output_storage[ofrom : ofrom + apply.nout]
            ifrom += apply.nin
            ofrom += apply.nout

    async def perform_async(self, node: Apply, inputs: Sequence[Any], output_storage: OutputStorageType) -> None:
        parts = list(self._slices(list(inputs), output_storage))
        pending = []
        # children that can be answered by one fused multi-GPU launch are grouped first
        groups = {}
        for apply, ins, outs in parts:
            key = apply.op.fusion_key() if isinstance(apply.op, FusableAsyncOp) else None
            if key is None:
                pending.append(apply.op.perform_async(apply, ins, outs))
            else:
                groups.setdefault(key, []).append((apply, ins, outs))
        for members in groups.values():
            pending.append(members[0][0].op.perform_fused(members))
        results = await asyncio.gather(*pending, return_exceptions=True)
        errors = [r for r in results if isinstance(r, BaseException)]
        if len(errors) == 1:
            raise errors[0]
        if errors:
            raise ParallelAsyncError(errors) from errors[0]

    def perform(self, node: Apply, inputs: Sequence[Any], output_storage: OutputStorageType) -> None:
        if self._perform_fused_sync(list(inputs), output_storage):
            return
        loop = get_useful_event_loop()
        loop.run_until_complete(self.perform_async(node, inputs, output_storage))

    def _perform_fused_sync(self, inputs, output_storage) -> bool:
        """Fast path: every child belongs to a fusable group whose engine call is synchronous anyway
        (``FusableAsyncOp.perform_fused_sync``) — one call per group, no event loop.  Returns False (nothing
        done) when any child needs the loop.  Errors are reported exactly like on the asynchronous path."""
        layout = self.__dict__.get("_sync_layout")
        if layout is None:
            # the grouping is a property of the children (their ops and fusion keys), computed once:
            # [[(apply, first input, end input, first output, end output), ...] per group], or () = needs the loop
            groups, ifrom, ofrom = {}, 0, 0
            for apply in self.applies:
                op = apply.op
                key = op.fusion_key() if isinstance(op, FusableAsyncOp) and op.has_sync_fused() else None
                if key is None:
                    groups = None
                    break
                groups.setdefault(key, []).append((apply, ifrom, ifrom + apply.nin, ofrom, ofrom + apply.nout))
                ifrom += apply.nin
                ofrom += apply.nout
            layout = self._sync_layout = tuple(groups.values()) if groups else ()
        if not layout:
            return False
        errors = []
        for group in layout:
            members = [(apply, inputs[i0:i1], output_storage[o0:o1]) for apply, i0, i1, o0, o1 in group]
            try:
                members[0][0].op.perform_fused_sync(members)
            except Exception as ex:  # noqa: BLE001 - aggregated below, as asyncio.gather(return_exceptions=True) does
                errors.append(ex)
        if len(errors) == 1:
            raise errors[0]
        if errors:
            raise ParallelAsyncError(errors) from errors[0]
        return True


class FusableAsyncOp(AsyncOp):
    """An ``AsyncOp`` whose siblings can be evaluated together by one engine call.

    ``fusion_key()`` returns a hashable key (e.g. the id of a :class:`FederatedEngine`) or ``None``;
    ``perform_fused(members)`` receives ``[(apply, inputs, output_storage), ...]`` of all siblings
    with the same key inside one :class:`ParallelAsyncOp`.
    """

    def fusion_key(self):
        return None

    async def perform_fused(self, members) -> None:
        await asyncio.gather(*[a.op.perform_async(a, i, o) for a, i, o in members])

    def has_sync_fused(self) -> bool:
        """True if :meth:`perform_fused_sync` is implemented: the fused call blocks anyway (an engine launch), so a
        :class:`ParallelAsyncOp` made only of such children skips the event loop."""
        return type(self).perform_fused_sync is not FusableAsyncOp.perform_fused_sync

    def perform_fused_sync(self, members) -> None:
        raise NotImplementedError


def _async_depths(fg: FunctionGraph, op_cls: type) -> dict:
    """Maps every ``op_cls`` apply of ``fg`` to the length of the longest chain of ``op_cls``
    applies above it (0 = no such ancestor).  One pass over the topological order."""
    above: dict = {}   # apply -> max number of op_cls applies on a path that ends just before it
    depths: dict = {}
    for node in fg.toposort():
        level = 0
        for var in node.inputs:
            parent = var.owner
            if parent is not None and parent in above:
                level = max(level, above[parent] + (1 if parent in depths else 0))
        above[node] = level
        if isinstance(node.op, op_cls):
            depths[node] = level
    return depths


def find_parallelizable_applies(fg: FunctionGraph, op_cls: type) -> List[Apply]:
    """Returns a maximal set (>= 2, else ``[]``) of mutually independent ``op_cls`` applies.

    Nodes are ranked by how many ``op_cls`` nodes lie on the longest path above them; two nodes
    of equal rank can never depend on one another, so every rank is an antichain.  The shallowest
    rank with at least two members is returned, in topological order.  Calling this repeatedly
    while fusing (see :func:`parallelize_all_async_applies`) therefore works through a dependency
    chain level by level, like the reference's greedy scan
    (``pytensor_federated/op_async.py:135-167``), but it also pairs up independent
    nodes that a dependent node separates in the topological order.
    """
    by_rank: dict = {}
    for node, rank in _async_depths(fg, op_cls).items():
        by_rank.setdefault(rank, []).append(node)
    for rank in sorted(by_rank):
        if len(by_rank[rank]) >= 2:
            return by_rank[rank]
    return []


def parallelize_async_applies(fg: FunctionGraph, applies: Sequence[Apply]) -> None:
    """Substitutes one :class:`ParallelAsyncOp` node for the independent ``applies`` (in place).

    The fused node takes the children's inputs back to back and yields their outputs back to
    back; every old output variable is rerouted to its twin.  With the ``ReplaceValidate``
    feature attached the validated replacement is used.
    """
    members = tuple(applies)
    fused = ParallelAsyncOp(members).make_node(*[v for m in members for v in m.inputs])
    pairs = [(old, new) for old, new in zip((v for m in members for v in m.outputs), fused.outputs)]
    if hasattr(fg, "replace_all_validate"):
        fg.replace_all_validate(pairs)
    else:
        fg.replace_all(pairs)


def parallelize_all_async_applies(fg: FunctionGraph) -> None:
    """Fuses until no two independent ``AsyncOp`` applies remain.

    ``ParallelAsyncOp`` is itself an ``AsyncOp``; a fused node is never fused again with the
    nodes it already contains because those are gone from the graph, so this terminates.
    """
    applies = find_parallelizable_applies(fg, AsyncOp)
    while applies:
        parallelize_async_applies(fg, applies)
        applies = find_parallelizable_applies(fg, AsyncOp)


class AsyncFusionOptimizer(GraphRewriter):
    """Graph rewriter that parallelises ``AsyncOp.perform_async`` calls."""

    def add_requirements(self, fgraph: FunctionGraph) -> None:
        fgraph.attach_feature(ReplaceValidate())

    def apply(self, fgraph: FunctionGraph) -> None:
        parallelize_all_async_applies(fgraph)


if "fuse_asyncs" not in optdb:
    optdb.register("fuse_asyncs", AsyncFusionOptimizer(), "fast_run", position=90)

__all__ = [
    "AsyncOp",
    "AsyncFromFunctionOp",
    "ParallelAsyncOp",
    "ParallelAsyncError",
    "FusableAsyncOp",
    "find_parallelizable_applies",
    "parallelize_async_applies",
    "parallelize_all_async_applies",
    "AsyncFusionOptimizer",
]
