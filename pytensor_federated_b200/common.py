"""Bayesian-flavoured adapters around the ArraysToArrays transport.

Reference: ``pytensor_federated/common.py:12-161``.  Server side:
``wrap_logp_func`` / ``wrap_logp_grad_func`` turn a log-probability function into a
``ComputeFunc`` and validate what it returns (same exception types and messages as
the reference, ``:17-21`` and ``:31-46``).  Client side: ``LogpServiceClient`` /
``LogpGradServiceClient`` give the transport client a ``LogpFunc`` /
``LogpGradFunc`` signature.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from .service import ArraysToArraysServiceClient
from .signatures import ComputeFunc, LogpFunc, LogpGradFunc

HostPort = Tuple[str, int]


def _check_logp(logp, verb: str) -> None:
    if not isinstance(logp, np.ndarray):
        raise TypeError(f"The logp value must be a scalar ndarray. Got {type(logp)} instead.")
    if not logp.shape == ():
        raise Exception(f"Returned logp {verb} be scalar, but got shape {logp.shape}")


def wrap_logp_func(logp_func: LogpFunc) -> ComputeFunc:
    """Wraps a non-differentiable logp function as a ``ComputeFunc``."""

    def compute_func(*inputs):
        logp = logp_func(*inputs)
        _check_logp(logp, "must")
        return (logp,)

    return compute_func


def wrap_logp_grad_func(logp_grad_func: LogpGradFunc) -> ComputeFunc:
    """Wraps a logp function that also returns gradients as a ``ComputeFunc``.

    The returned function yields the flat sequence ``(logp, *gradients)``.
    """

    def compute_func(*inputs):
        result = logp_grad_func(*inputs)
        if not len(result) == 2:
            raise TypeError(
                "The return value of the logp function must be a tuple"
                " of a scalar ndarray and a list of ndarrays for the gradients."
                f" Got {type(result)} instead."
            )
        logp, gradients = result
        _check_logp(logp, "should")
        if not len(gradients) == len(inputs):
            raise Exception(
                "Number of gradients does not match number of inputs."
                f"\ninputs: {inputs}\ngradients: {gradients}"
            )
        return (logp, *gradients)

    return compute_func


class _ClientAdapter:
    """Shared constructor: owns one :class:`ArraysToArraysServiceClient`."""

    def __init__(
        self,
        host: Optional[str] = None,
        port: Optional[int] = None,
        *,
        hosts_and_ports: Optional[Sequence[HostPort]] = None,
    ) -> None:
        self._client = ArraysToArraysServiceClient(host, port, hosts_and_ports=hosts_and_ports)
        super().__init__()


class LogpServiceClient(_ClientAdapter):
    """Gives the :class:`ArraysToArraysServiceClient` a ``LogpFunc`` signature."""

    def __call__(self, *inputs: np.ndarray) -> np.ndarray:
        """Alias for ``.evaluate(*inputs)``."""
        return self.evaluate(*inputs)

    def evaluate(self, *inputs: np.ndarray, use_stream: bool = True, **kwargs) -> np.ndarray:
        """Evaluates the federated log-potential; returns the scalar ``logp``
        (``retries`` / ``timeout`` are passed on to :meth:`ArraysToArraysServiceClient.evaluate_async`)."""
        (logp,) = self._client.evaluate(*inputs, use_stream=use_stream, **kwargs)
        return logp

    async def evaluate_async(self, *inputs: np.ndarray, use_stream: bool = True, **kwargs) -> np.ndarray:
        (logp,) = await self._client.evaluate_async(*inputs, use_stream=use_stream, **kwargs)
        return logp


class LogpGradServiceClient(_ClientAdapter):
    """Gives the :class:`ArraysToArraysServiceClient` a ``LogpGradFunc`` signature."""

    def __call__(self, *inputs: np.ndarray) -> Tuple[np.ndarray, List[np.ndarray]]:
        """Alias for ``.evaluate(*inputs)``."""
        return self.evaluate(*inputs)

    def evaluate(
        self, *inputs: np.ndarray, use_stream: bool = True, **kwargs
    ) -> Tuple[np.ndarray, List[np.ndarray]]:
        """Evaluates the federated log-potential and its gradients.

        Returns ``(logp, gradients)`` with one gradient per input
        (``retries`` / ``timeout`` are passed on to :meth:`ArraysToArraysServiceClient.evaluate_async`).
        """
        logp, *gradients = self._client.evaluate(*inputs, use_stream=use_stream, **kwargs)
        return logp, gradients

    async def evaluate_async(
        self, *inputs: np.ndarray, use_stream: bool = True, **kwargs
    ) -> Tuple[np.ndarray, List[np.ndarray]]:
        logp, *gradients = await self._client.evaluate_async(*inputs, use_stream=use_stream, **kwargs)
        return logp, gradients


__all__ = [
    "wrap_logp_func",
    "wrap_logp_grad_func",
    "LogpServiceClient",
    "LogpGradServiceClient",
]
