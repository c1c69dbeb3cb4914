"""Contract between a model family and the federation engine.

A *shard model* is the GPU-native counterpart of the black-box ``compute_func`` that a
reference node serves (``pytensor_federated/service.py:78-86``): it owns the
node's private data (resident in HBM) and knows

* how the client's input arrays are packed into the theta mailbox (32-bit words),
* how those words are turned back into input arrays (``inputs_from_words(words)``, what the peers of the
  collective backend evaluate; every model but ``LinregShards`` has it),
* how the reduced ``[LL, dLL/dtheta ...]`` vector of doubles is unpacked into the flat
  ``(logp, *gradients)`` tuple of the ``wrap_logp_grad_func`` convention
  (``pytensor_federated/common.py:26-49``),
* how to attach itself to a native engine (which kernel, which launch shape), and
* an eager PyTorch implementation of the same maths (numerics oracle for the kernels and the
  compute step of the NCCL/gloo baseline path).
"""
from __future__ import annotations

from typing import List, Sequence

import numpy as np


class ShardModel:
    """Base class; subclasses set ``n_theta_words`` and ``n_vals``."""

    #: number of 32-bit words in the theta mailbox
    n_theta_words: int = 0
    #: number of float64 values in a node partial / the reduced result
    n_vals: int = 0
    #: number of input arrays of the ArraysToArrays signature
    n_inputs: int = 0

    def call_context(self, inputs: Sequence[np.ndarray]):
        """Whatever :meth:`unpack_result` must know about THIS call's inputs (their shapes).  The
        engine carries it from ``pack_theta`` to ``unpack_result`` so that concurrent callers never
        see each other's shapes; it is never stored on the model by the engine path."""
        return None

    def pack_theta(self, inputs: Sequence[np.ndarray], out: np.ndarray):
        """Writes the inputs into ``out`` (``uint32[n_theta_words]`` view of pinned memory) and
        returns :meth:`call_context` of the inputs."""
        raise NotImplementedError

    def unpack_result(self, vals: np.ndarray, ctx=None) -> List[np.ndarray]:
        """``float64[n_vals]`` → ``[logp, grad_0, grad_1, ...]`` (fresh arrays).  ``ctx`` is the
        value ``pack_theta`` returned for the same call (``None``: the most recent single-threaded
        ``pack_theta`` / ``reference_partial`` call, kept for interactive use)."""
        raise NotImplementedError

    def attach(self, lib, handle) -> None:
        """Registers data pointers and kernel choice with the native engine."""
        raise NotImplementedError

    def reference_partial(self, inputs: Sequence[np.ndarray]) -> np.ndarray:
        """This node's partial ``float64[n_vals]`` computed with stock PyTorch ops."""
        raise NotImplementedError

    # -- conveniences --------------------------------------------------------------------
    def reference(self, inputs: Sequence[np.ndarray]) -> List[np.ndarray]:
        return self.unpack_result(self.reference_partial(inputs), self.call_context(inputs))

    def bytes_per_eval(self) -> int:
        """Algorithmic HBM bytes one evaluation must move on this node (roofline input)."""
        return 0

    def flops_per_eval(self) -> int:
        return 0
