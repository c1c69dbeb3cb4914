"""``torch.autograd`` twins of the graph Ops.

The reference integrates with PyTensor only.  Users whose sampler or optimiser lives in PyTorch
(Pyro, custom HMC, ``torch.optim``) get the same contract here: a federated ``LogpGradFunc``
becomes a differentiable scalar whose backward pass re-uses the gradients returned by the same
remote evaluation — one federated call per forward+backward, like ``LogpGradOp.grad``
(``pytensor_federated/wrapper_ops.py:119-132``).
"""
from __future__ import annotations

from typing import Callable, Sequence

import numpy as np
import torch

from .signatures import LogpFunc, LogpGradFunc


class _FederatedLogpGrad(torch.autograd.Function):
    @staticmethod
    def forward(ctx, fn, *inputs):
        arrays = [np.asarray(t.detach().cpu().numpy(), dtype=np.float64) for t in inputs]
        logp, grads = fn(*arrays)
        if len(grads) != len(inputs):
            raise ValueError("Number of gradients does not match number of inputs.")
        ctx.grads = [torch.as_tensor(np.asarray(g, dtype=np.float64)).reshape(t.shape).to(t.device, t.dtype)
                     for g, t in zip(grads, inputs)]
        out = torch.as_tensor(np.asarray(logp, dtype=np.float64))
        return out.to(inputs[0].device, inputs[0].dtype) if inputs else out

    @staticmethod
    def backward(ctx, g_logp):
        return (None, *[g_logp * g for g in ctx.grads])


def federated_logp(logp_grad_func: LogpGradFunc, *inputs: torch.Tensor) -> torch.Tensor:
    """Scalar tensor ``logp(*inputs)`` with gradients supplied by the federated function."""
    return _FederatedLogpGrad.apply(logp_grad_func, *inputs)


class FederatedLogp(torch.nn.Module):
    """Module form: ``FederatedLogp(client_or_engine.logp_grad)(theta0, theta1, ...)``."""

    def __init__(self, logp_grad_func: LogpGradFunc) -> None:
        super().__init__()
        self._fn = logp_grad_func

    def forward(self, *inputs: torch.Tensor) -> torch.Tensor:
        return federated_logp(self._fn, *inputs)


def arrays_to_arrays(compute_func: Callable[..., Sequence[np.ndarray]], *inputs: torch.Tensor):
    """Non-differentiable black box: tensors in, tensors out (``ArraysToArraysOp`` twin)."""
    outs = compute_func(*[t.detach().cpu().numpy() for t in inputs])
    return [torch.as_tensor(np.array(o)) for o in outs]


def logp_only(logp_func: LogpFunc, *inputs: torch.Tensor) -> torch.Tensor:
    """``LogpOp`` twin: a constant w.r.t. autograd."""
    return torch.as_tensor(np.array(logp_func(*[t.detach().cpu().numpy() for t in inputs])))


__all__ = ["federated_logp", "FederatedLogp", "arrays_to_arrays", "logp_only"]
