"""Dynamic batching of concurrent requests on a serving node.

The reference serves every request of every client one after the other
(``pytensor_federated/service.py:104-112``): four MCMC chains that share a node cost four
evaluations.  On a GPU node the tensor-core GLM kernel evaluates up to 16 chains in ONE launch for
roughly the price of one (the design matrix is streamed once, chains ride along the MMA N dimension —
``csrc/glm_tc.cu``).  :class:`DynamicBatcher` is the piece that lets a gRPC node exploit this: requests
that arrive within a short window are stacked, evaluated by one batched call, and un-stacked into their
responses — the inference-server pattern, applied to log-probability evaluations.

    batcher = DynamicBatcher(stacked_compute_func(engine.evaluate, max_batch=8), max_batch=8)
    service = ArraysToArraysService(batcher)          # the service awaits coroutine compute functions
"""
from __future__ import annotations

import asyncio
import time
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

__all__ = ["DynamicBatcher", "stacked_compute_func"]

Request = Tuple[np.ndarray, ...]
BatchedFunc = Callable[[List[Request]], List[Sequence[np.ndarray]]]


class DynamicBatcher:
    """Coroutine ``ComputeFunc`` that groups concurrent calls into batches.

    Parameters
    ----------
    batched_func
        ``f([inputs_0, inputs_1, ...]) -> [outputs_0, outputs_1, ...]`` — evaluates up to ``max_batch``
        requests at once (synchronously; it is called from the event loop like any ``ComputeFunc``, or in
        the default executor with ``offload=True``).
    max_batch
        Upper bound of a batch (the kernel's chain capacity).
    max_delay
        Seconds the first request of a batch may wait for company.  ``0`` still batches whatever is
        already queued when the worker wakes up (requests that arrived during the previous evaluation).
    """

    is_coroutine_compute_func = True

    def __init__(self, batched_func: BatchedFunc, max_batch: int, max_delay: float = 0.0005, offload: bool = False) -> None:
        if max_batch < 1:
            raise ValueError("max_batch must be >= 1")
        self._func = batched_func
        self.max_batch = int(max_batch)
        self.max_delay = float(max_delay)
        self._offload = offload
        self._queue: Optional[asyncio.Queue] = None
        self._worker: Optional[asyncio.Task] = None
        self._loop = None
        self.n_batches = 0
        self.n_requests = 0

    def _ensure_worker(self) -> None:
        loop = asyncio.get_running_loop()
        if self._worker is None or self._worker.done() or self._loop is not loop:
            self._loop = loop
            self._queue = asyncio.Queue()
            self._worker = loop.create_task(self._run())

    async def __call__(self, *inputs: np.ndarray) -> Sequence[np.ndarray]:
        self._ensure_worker()
        future = self._loop.create_future()
        self._queue.put_nowait((inputs, future))
        return await future

    async def _run(self) -> None:
        queue = self._queue
        while True:
            batch = [await queue.get()]
            deadline = time.monotonic() + self.max_delay
            while len(batch) < self.max_batch:
                if not queue.empty():
                    batch.append(queue.get_nowait())
                    continue
                remaining = deadline - time.monotonic()
                if remaining <= 0:
                    break
                try:
                    batch.append(await asyncio.wait_for(queue.get(), remaining))
                except asyncio.TimeoutError:
                    break
            requests = [req for req, _ in batch]
            try:
                if self._offload:
                    results = await self._loop.run_in_executor(None, self._func, requests)
                else:
                    results = self._func(requests)
                if len(results) != len(requests):
                    raise RuntimeError(f"batched function returned {len(results)} results for {len(requests)} requests")
            except Exception as ex:  # noqa: BLE001 - every waiting request sees the failure
                for _, future in batch:
                    if not future.done():
                        future.set_exception(ex)
                continue
            self.n_batches += 1
            self.n_requests += len(requests)
            for (_, future), result in zip(batch, results):
                if not future.done():
                    future.set_result(result)

    async def close(self) -> None:
        if self._worker is not None:
            self._worker.cancel()
            try:
                await self._worker
            except (asyncio.CancelledError, Exception):  # noqa: BLE001
                pass
            self._worker = None


def stacked_compute_func(evaluate: Callable[..., Sequence[np.ndarray]], max_batch: int, pad: bool = True) -> BatchedFunc:
    """Adapts a multi-chain evaluator to :class:`DynamicBatcher`.

    ``evaluate(*stacked_inputs)`` takes every input with a leading chain axis of length ``max_batch`` (e.g.
    ``FederatedEngine(GlmShards(..., n_chains=K)).evaluate``) and returns outputs with the same leading
    axis.  Requests are stacked along that axis; a short batch is padded by repeating its last request
    (``pad=True``: fixed-shape kernels) and the padding rows are dropped from the answers."""

    def batched(requests: List[Request]) -> List[Sequence[np.ndarray]]:
        n = len(requests)
        if n > max_batch:
            raise ValueError(f"batch of {n} exceeds the evaluator's capacity {max_batch}")
        rows = list(requests) + ([requests[-1]] * (max_batch - n) if pad else [])
        stacked = [np.stack([np.asarray(r[i]) for r in rows], axis=0) for i in range(len(requests[0]))]
        outputs = evaluate(*stacked)
        return [[np.asarray(o)[k] for o in outputs] for k in range(n)]

    return batched
