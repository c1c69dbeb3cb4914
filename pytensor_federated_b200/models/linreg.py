"""Gaussian linear regression shards — the reference's demo model, GPU-resident.

Maths: ``demo_node.py:31-43`` (``LinearModelBlackbox``); data synthesis for the
demo: ``demo_node.py:59-61``.  One :class:`LinregShards` object holds the shards
that live on ONE GPU; ``theta`` is ``[(intercept_s, slope_s) for s in all shards of the
federation]`` so that a hierarchical model with per-group intercepts
(``demo_model.py:28-36``) is evaluated in one fused launch, and the result
keeps per-shard ``[LL, dLL/da, dLL/db]`` so the client graph can weight/sum them itself.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import numpy as np

from .base import ShardModel

LOG_SQRT_2PI = 0.91893853320467274178


def make_demo_data(seed: int = 123, n: int = 10, sigma: float = 0.4):
    """The reference demo's "secret" dataset (``demo_node.py:59-61``)."""
    x = np.linspace(0, 10, n)
    y = np.random.RandomState(seed).normal(1.5 + 0.5 * x, scale=sigma)
    return x, y, sigma


class LinregShards(ShardModel):
    """Shards ``local_ids`` (global shard indices) of an ``n_shards_total`` federation."""

    #: largest federation the kernel takes: theta (16 bytes per shard) and a 256-byte reduction buffer share the
    #: 227 KB of shared memory one CTA can have on the H100, less 256 bytes for the kernel's static variables
    MAX_SHARDS_TOTAL = (227 * 1024 - 256 - 256) // 16

    def __init__(
        self,
        xs: Sequence,
        ys: Sequence,
        sigmas: Sequence[float],
        *,
        local_ids: Optional[Sequence[int]] = None,
        n_shards_total: Optional[int] = None,
        device=None,
        dtype=None,
    ) -> None:
        import torch

        self.device = torch.device(device) if device is not None else torch.device("cpu")
        self.dtype = dtype or torch.float64
        self.local_ids = list(local_ids) if local_ids is not None else list(range(len(xs)))
        self.n_shards_total = int(n_shards_total if n_shards_total is not None else len(xs))
        if len(xs) != len(ys) or len(xs) != len(sigmas) or len(xs) != len(self.local_ids):
            raise ValueError("xs, ys, sigmas and local_ids must have the same length")
        if self.n_shards_total > self.MAX_SHARDS_TOTAL:
            raise ValueError(f"{self.n_shards_total} shards in total: the kernel keeps theta in shared memory, which "
                             f"holds at most {self.MAX_SHARDS_TOTAL}")
        if not all(0 <= s < self.n_shards_total for s in self.local_ids) or len(set(self.local_ids)) != len(self.local_ids):
            raise ValueError(f"local_ids must be distinct shard indices in [0, {self.n_shards_total})")
        for s, (x, y, sigma) in enumerate(zip(xs, ys, sigmas)):
            # the kernel reads n = len(x) rows of both arrays
            if np.ndim(x) != 1 or np.ndim(y) != 1 or np.shape(x) != np.shape(y):
                raise ValueError(f"x and y of shard {s} must be 1-D with the same length, got shapes "
                                 f"{tuple(np.shape(x))} and {tuple(np.shape(y))}")
            if not (np.isfinite(float(sigma)) and float(sigma) > 0.0):
                raise ValueError(f"sigma of shard {s} must be finite and > 0, got {sigma}")
        self.xs = [torch.as_tensor(np.asarray(x), dtype=self.dtype).to(self.device).contiguous() for x in xs]
        self.ys = [torch.as_tensor(np.asarray(y), dtype=self.dtype).to(self.device).contiguous() for y in ys]
        self.sigmas = [float(s) for s in sigmas]
        self.n_inputs = 2  # (intercepts[S], slopes[S]) — scalars broadcast to every shard
        self.n_theta_words = 4 * self.n_shards_total  # 2 doubles per shard
        self.n_vals = 3 * self.n_shards_total

    # -- packing ---------------------------------------------------------------------------
    def call_context(self, inputs):
        intercept, slope = inputs
        return (np.shape(intercept), np.shape(slope))

    def pack_theta(self, inputs, out: np.ndarray):
        intercept, slope = inputs
        ctx = self._input_shapes = self.call_context(inputs)
        th = out.view(np.float64).reshape(self.n_shards_total, 2)
        th[:, 0] = np.asarray(intercept, dtype=np.float64)  # broadcasts scalars
        th[:, 1] = np.asarray(slope, dtype=np.float64)
        return ctx

    def unpack_result(self, vals: np.ndarray, ctx=None) -> List[np.ndarray]:
        """``[logp_total, d/d intercept, d/d slope]``; per-shard values via :meth:`per_shard`."""
        v = np.asarray(vals, dtype=np.float64).reshape(self.n_shards_total, 3)
        shape_a, shape_b = ctx if ctx is not None else self._input_shapes
        da = v[:, 1].copy() if shape_a != () else np.asarray(v[:, 1].sum())
        db = v[:, 2].copy() if shape_b != () else np.asarray(v[:, 2].sum())
        return [np.asarray(v[:, 0].sum()), da, db]

    #: shapes of the last packed (intercept, slope): scalars are shared by all shards and get
    #: their gradients summed; vectors are per-shard and get per-shard gradients
    _input_shapes = ((), ())

    @staticmethod
    def per_shard(vals: np.ndarray) -> np.ndarray:
        return np.asarray(vals, dtype=np.float64).reshape(-1, 3)

    # -- native ----------------------------------------------------------------------------
    def attach(self, lib, handle) -> None:
        from ..ops import native

        n = len(self.xs)
        xp = native.void_p_array([t.data_ptr() for t in self.xs])
        yp = native.void_p_array([t.data_ptr() for t in self.ys])
        ns = (C.c_longlong * n)(*[t.numel() for t in self.xs])
        sg = (C.c_double * n)(*self.sigmas)
        off = (C.c_int * n)(*[2 * s for s in self.local_ids])
        import torch

        native.check(
            lib.b200_engine_set_linreg(handle, n, xp, yp, ns, sg, off, int(self.dtype == torch.float64)),
            "set_linreg",
        )

    # -- eager oracle ----------------------------------------------------------------------
    def reference_partial(self, inputs) -> np.ndarray:
        import torch

        intercept, slope = inputs
        a = np.broadcast_to(np.asarray(intercept, dtype=np.float64), (self.n_shards_total,))
        b = np.broadcast_to(np.asarray(slope, dtype=np.float64), (self.n_shards_total,))
        out = np.zeros((self.n_shards_total, 3))
        for x, y, sigma, sid in zip(self.xs, self.ys, self.sigmas, self.local_ids):
            x64, y64 = x.double(), y.double()
            r = y64 - (a[sid] + b[sid] * x64)
            inv_var = 1.0 / sigma**2
            ll = -0.5 * torch.sum(r * r) * inv_var - x64.numel() * (np.log(sigma) + LOG_SQRT_2PI)
            out[sid] = [float(ll), float(torch.sum(r) * inv_var), float(torch.sum(r * x64) * inv_var)]
        return out.reshape(-1)

    def bytes_per_eval(self) -> int:
        return sum(2 * t.numel() * t.element_size() for t in self.xs)
