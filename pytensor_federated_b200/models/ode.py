"""ODE parameter-estimation shards (RK4 with forward sensitivities).

Workload from ``BASELINE.json`` ("federated ODE parameter estimation
([timepoints, theta] -> trajectory -> LL), 4 shards on 4 GPUs"); the reference describes the
use-case only in prose (``README.md:39-52``).  Every series has its own known
initial state; Gaussian observation noise on every state.

The default system is Lotka–Volterra, ``theta = (alpha, beta, gamma, delta)``, with hand-written
sensitivities (``csrc/ode.cu``).  ANY other system is an :class:`OdeSystem`: the right-hand side as a
few lines of CUDA C, compiled into the fused broadcast -> solve -> reduce kernel
(``csrc/ode_generic.cu``, forward-mode dual numbers — no Jacobians to write), plus the same function in
PyTorch for the oracle / CPU path.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import math
import numbers
from pathlib import Path
from typing import Callable, List, Optional, Sequence

import numpy as np

from .base import ShardModel

_PKG = Path(__file__).resolve().parent.parent
_CSRC = _PKG / "csrc"


def lv_rhs(u, v, th):
    a, b, g, d = th
    return a * u - b * u * v, d * u * v - g * v


class OdeSystem:
    """A user-defined ODE ``y' = f(y, theta, t)`` for the fused kernel.

    ``rhs_cuda``
        CUDA C statements assigning ``dy[0..n_states)`` from ``y[...]``, ``th[...]`` and the float ``t``.
        ``y`` and ``th`` are dual numbers (value and d/dtheta); do not name their type.  ``+ - * /`` and unary
        minus take two duals or a dual and a float, in either order.  ``exp log sqrt sin cos tanh square`` and
        ``pow(x, p)`` take a dual ``x`` (then ``p`` is a float) or a float, such as ``t`` or a literal, and then
        return a float: ``sin(1.5f * t)`` is a float forcing term, ``cos(th[2] * t)`` a dual.  ``pow`` of a
        dual exponent is not available.
    ``rhs_torch``
        The same right-hand side for tensors: ``rhs_torch(y, th, t) -> sequence of n_states tensors`` with
        ``y`` a sequence of state tensors and ``th`` a 1-D tensor — used by the eager oracle, whose
        gradient comes from autograd.

    Example — SIR epidemic (2 parameters, 3 states)::

        sir = OdeSystem(
            "const auto inf = th[0] * y[0] * y[1]; dy[0] = -inf; dy[1] = inf - th[1] * y[1]; dy[2] = th[1] * y[1];",
            lambda y, th, t: (-th[0] * y[0] * y[1], th[0] * y[0] * y[1] - th[1] * y[1], th[1] * y[1]),
            n_states=3, n_params=2)
    """

    def __init__(self, rhs_cuda: str, rhs_torch: Optional[Callable], *, n_states: int, n_params: int,
                 name: str = "custom-ode") -> None:
        if not (1 <= n_states <= 8 and 1 <= n_params <= 16):
            raise ValueError("the fused ODE kernel keeps states x parameters in registers: n_states <= 8, n_params <= 16")
        self.rhs_cuda = " ".join(rhs_cuda.split())
        self.rhs_torch = rhs_torch
        self.n_states = int(n_states)
        self.n_params = int(n_params)
        self.name = name
        self._lib = None

    def __repr__(self) -> str:
        return f"OdeSystem(name={self.name!r}, n_states={self.n_states}, n_params={self.n_params})"

    def digest(self) -> str:
        h = hashlib.sha256(f"{self.n_states}|{self.n_params}|{self.rhs_cuda}".encode())
        for f in ("ode_generic.cu", "fed_comm.cuh", "models.h"):
            h.update((_CSRC / f).read_bytes())
        return h.hexdigest()[:16]

    def compile(self) -> C.CDLL:
        """Builds (or loads from the cache) the shared object of this system for sm_90a."""
        if self._lib is not None:
            return self._lib
        from .. import build as native_build

        so = native_build.build_snippet_library(
            "ode_generic.cu", "B200FED_ODE_RHS", self.rhs_cuda,
            [f"-DB200FED_ODE_NS={self.n_states}", f"-DB200FED_ODE_NP={self.n_params}",
             "-DB200FED_ODE_ENTRY=b200_launch_ode_custom"],
            f"libb200fed_ode_{self.digest()}", "ODE right-hand side")
        self._lib = C.CDLL(str(so))
        return self._lib

    def launcher_address(self) -> int:
        return C.cast(self.compile().b200_launch_ode_custom, C.c_void_p).value


#: the built-in system as an OdeSystem (what ``csrc/ode_generic.cu`` builds without macros): cross-check of ode.cu
LOTKA_VOLTERRA = OdeSystem(
    "dy[0] = th[0] * y[0] - th[1] * y[0] * y[1]; dy[1] = th[3] * y[0] * y[1] - th[2] * y[1];",
    lambda y, th, t: (th[0] * y[0] - th[1] * y[0] * y[1], th[3] * y[0] * y[1] - th[2] * y[1]),
    n_states=2, n_params=4, name="lotka-volterra",
)


class OdeShards(ShardModel):
    """ODE parameter estimation: every shard holds many observed time series; one evaluation integrates
    them (RK4 with forward sensitivities) and returns the Gaussian log-likelihood and its gradient w.r.t.
    ``theta``.  ``system=None`` is Lotka–Volterra (``csrc/ode.cu``, ``theta = (alpha, beta, gamma,
    delta)``); any :class:`OdeSystem` runs through ``csrc/ode_generic.cu``.  The reference only describes this
    workload in prose (``README.md:39-52``)."""

    def __init__(self, ts: Sequence, y0s: Sequence, y_obs: Sequence, sigmas: Sequence[float], substeps: int = 8,
                 system: Optional[OdeSystem] = None, node_ids: Optional[Sequence[int]] = None,
                 n_nodes: Optional[int] = None):
        """``node_ids`` / ``n_nodes``: shard ``s`` is node ``node_ids[s]`` of an ``n_nodes`` federation; theta then
        holds one parameter vector PER NODE (a single vector is broadcast) and the result one
        ``[LL, dLL/dtheta]`` block per node — what ``NodeFederation`` needs to give every node its own Op."""
        import torch

        if (node_ids is None) != (n_nodes is None):
            raise ValueError("node_ids and n_nodes come together")
        self.node_ids = list(node_ids) if node_ids is not None else None
        self.n_nodes = int(n_nodes) if n_nodes is not None else 1
        self.system = system
        self.n_states = system.n_states if system is not None else 2
        self.n_params = system.n_params if system is not None else 4
        self.ts = [t.to(torch.float32).contiguous() for t in ts]            # [n_t]
        self.y0s = [y.to(torch.float32).contiguous() for y in y0s]          # [n_states, n_series]
        self.y_obs = [y.to(torch.float32).contiguous() for y in y_obs]      # [n_t, n_states, n_series]
        for y0, yo, t in zip(self.y0s, self.y_obs, self.ts):
            if y0.shape[0] != self.n_states or yo.shape[1] != self.n_states or yo.shape[0] != t.numel() or yo.shape[2] != y0.shape[1]:
                raise ValueError("expected y0 [n_states, n_series] and y_obs [n_t, n_states, n_series]")
            if not bool(torch.isfinite(t).all()):
                raise ValueError("every time point must be finite")
        self.sigmas = [float(np.float32(s)) for s in sigmas]    # what the kernels see, and so the oracle too
        if len(self.sigmas) != len(self.ts) or not all(math.isfinite(s) and s > 0 for s in self.sigmas):
            raise ValueError(f"sigmas needs one finite sigma > 0 per shard, got {sigmas!r}")
        # substeps = 0 would give h = inf and no RK4 step at all: the likelihood of y0 at every time point
        if isinstance(substeps, bool) or not isinstance(substeps, numbers.Integral) or substeps < 1:
            raise ValueError(f"substeps must be an integer >= 1, got {substeps!r}")
        self.substeps = int(substeps)
        self.device = self.ts[0].device
        if self.node_ids is not None and (len(self.node_ids) != len(self.ts) or not all(0 <= i < self.n_nodes for i in self.node_ids)):
            raise ValueError("node_ids needs one node index in [0, n_nodes) per shard")
        if self.n_nodes * self.n_params > 1024:
            raise ValueError("theta of all nodes must fit 1024 floats")
        self.n_inputs = 1
        self.n_theta_words = self.n_nodes * self.n_params
        self.n_vals = self.n_nodes * (1 + self.n_params)

    def call_context(self, inputs):
        (theta,) = inputs
        return np.ndim(theta) == 2        # one parameter vector per node?

    def pack_theta(self, inputs, out: np.ndarray):
        (theta,) = inputs
        th = np.asarray(theta, dtype=np.float32)
        rows = out.view(np.float32)[: self.n_nodes * self.n_params].reshape(self.n_nodes, self.n_params)
        rows[:] = th.reshape(-1, self.n_params)    # [n_nodes, NP], or one vector broadcast to every node
        return th.ndim == 2

    def per_node(self, vals: np.ndarray) -> np.ndarray:
        """The reduced vector as ``[n_nodes, 1 + n_params]`` (``[LL, dLL/dtheta]`` per node)."""
        return np.asarray(vals, dtype=np.float64).reshape(self.n_nodes, 1 + self.n_params)

    def unpack_result(self, vals: np.ndarray, ctx=None) -> List[np.ndarray]:
        v = self.per_node(vals)
        if ctx:   # per-node parameters in, per-node gradients out
            return [np.asarray(v[:, 0].sum()), v[:, 1:].copy()]
        return [np.asarray(v[:, 0].sum()), v[:, 1:].sum(axis=0)]

    def inputs_from_words(self, words: np.ndarray):
        rows = words.view(np.float32)[: self.n_nodes * self.n_params].reshape(self.n_nodes, self.n_params).copy()
        return (rows,)

    def attach(self, lib, handle) -> None:
        from ..ops import native

        n = len(self.ts)
        native.check(
            lib.b200_engine_set_ode(
                handle, n,
                native.void_p_array([t.data_ptr() for t in self.ts]),
                native.void_p_array([t.data_ptr() for t in self.y0s]),
                native.void_p_array([t.data_ptr() for t in self.y_obs]),
                (C.c_int * n)(*[y.shape[1] for y in self.y0s]),
                (C.c_int * n)(*[t.numel() for t in self.ts]),
                (C.c_float * n)(*self.sigmas),
                (C.c_int * n)(*([self.substeps] * n)),
                (C.c_int * n)(*[self._node(s) * self.n_params for s in range(n)]),
                (C.c_int * n)(*[self._node(s) * (1 + self.n_params) for s in range(n)]),
            ),
            "set_ode",
        )
        if self.system is not None:
            lib.b200_engine_set_ode_launcher(handle, C.c_void_p(self.system.launcher_address()))

    def _node(self, s: int) -> int:
        return self.node_ids[s] if self.node_ids is not None else 0

    # -- eager oracle: same RK4 discretisation, autograd for the gradient, float64 -----------
    def reference_partial(self, inputs) -> np.ndarray:
        """``[n_nodes, 1 + n_params]`` flattened: every local shard evaluated at its node's parameters."""
        (theta,) = inputs
        rows = np.broadcast_to(np.asarray(theta, dtype=np.float64).reshape(-1, self.n_params), (self.n_nodes, self.n_params))
        out = np.zeros((self.n_nodes, 1 + self.n_params))
        for s in range(len(self.ts)):
            out[self._node(s)] += self._shard_partial(s, rows[self._node(s)])
        return out.reshape(-1)

    def _shard_partial(self, s: int, theta) -> np.ndarray:
        import torch

        th = torch.tensor(np.asarray(theta, dtype=np.float64).reshape(self.n_params), device=self.device, requires_grad=True)
        if self.system is None:
            f = lambda y, t: lv_rhs(y[0], y[1], th)
        else:
            if self.system.rhs_torch is None:
                raise ValueError("this OdeSystem has no rhs_torch oracle")
            f = lambda y, t: self.system.rhs_torch(y, th, t)
        total = torch.zeros((), dtype=torch.float64, device=self.device)
        for t, y0, yo, sigma in [(self.ts[s], self.y0s[s], self.y_obs[s], self.sigmas[s])]:
            y = [y0[c].double() for c in range(self.n_states)]
            t_prev = 0.0
            for j in range(t.numel()):
                h = (float(t[j]) - t_prev) / self.substeps
                for q in range(self.substeps):
                    tq = t_prev + q * h
                    k1 = f(y, tq)
                    k2 = f([yi + 0.5 * h * ki for yi, ki in zip(y, k1)], tq + 0.5 * h)
                    k3 = f([yi + 0.5 * h * ki for yi, ki in zip(y, k2)], tq + 0.5 * h)
                    k4 = f([yi + h * ki for yi, ki in zip(y, k3)], tq + h)
                    y = [yi + h / 6 * (a + 2 * b + 2 * c + d) for yi, a, b, c, d in zip(y, k1, k2, k3, k4)]
                t_prev = float(t[j])
                for c in range(self.n_states):
                    r = yo[j, c].double() - y[c]
                    total = total + (-0.5 * r * r / sigma**2).sum() - r.numel() * (np.log(sigma) + 0.918938533204672742)
        (grad,) = torch.autograd.grad(total, th)
        return np.concatenate([[float(total.detach())], grad.cpu().numpy()])


def synth_lv_shard(n_series: int, n_t: int, *, seed: int, device, theta=(1.0, 0.4, 0.8, 0.2), sigma=0.1,
                   t_end: float = 6.0, substeps: int = 8):
    """Simulates noisy Lotka–Volterra observations with the same RK4 scheme."""
    import torch

    gen = torch.Generator(device="cpu")
    gen.manual_seed(seed)
    t = torch.linspace(t_end / n_t, t_end, n_t)
    y0 = torch.stack([1.0 + torch.rand(n_series, generator=gen), 0.5 + torch.rand(n_series, generator=gen)])
    u, v = y0[0].double(), y0[1].double()
    th = torch.tensor(theta, dtype=torch.float64)
    obs = torch.empty(n_t, 2, n_series)
    t_prev = 0.0
    for j in range(n_t):
        h = (float(t[j]) - t_prev) / substeps
        for _ in range(substeps):
            k1 = lv_rhs(u, v, th)
            k2 = lv_rhs(u + 0.5 * h * k1[0], v + 0.5 * h * k1[1], th)
            k3 = lv_rhs(u + 0.5 * h * k2[0], v + 0.5 * h * k2[1], th)
            k4 = lv_rhs(u + h * k3[0], v + h * k3[1], th)
            u = u + h / 6 * (k1[0] + 2 * k2[0] + 2 * k3[0] + k4[0])
            v = v + h / 6 * (k1[1] + 2 * k2[1] + 2 * k3[1] + k4[1])
        t_prev = float(t[j])
        obs[j, 0] = (u + sigma * torch.randn(n_series, generator=gen, dtype=torch.float64)).float()
        obs[j, 1] = (v + sigma * torch.randn(n_series, generator=gen, dtype=torch.float64)).float()
    return t.to(device), y0.to(device), obs.to(device), sigma


def synth_ode_shard(system: OdeSystem, theta, y0, n_t: int, *, seed: int, device, sigma: float = 0.05,
                    t_end: float = 4.0, substeps: int = 8):
    """Noisy observations of ``system`` simulated with the kernel's own RK4 scheme (float64, CPU).

    ``y0``: ``[n_states, n_series]`` initial states.  Returns ``(t, y0, y_obs, sigma)`` on ``device``."""
    import torch

    gen = torch.Generator(device="cpu")
    gen.manual_seed(seed)
    y0 = torch.as_tensor(np.asarray(y0, dtype=np.float64))
    th = torch.tensor(np.asarray(theta, dtype=np.float64))
    t = torch.linspace(t_end / n_t, t_end, n_t)
    y = [y0[c].clone() for c in range(system.n_states)]
    obs = torch.empty(n_t, system.n_states, y0.shape[1])
    f = lambda yy, tt: system.rhs_torch(yy, th, tt)
    t_prev = 0.0
    for j in range(n_t):
        h = (float(t[j]) - t_prev) / substeps
        for q in range(substeps):
            tq = t_prev + q * h
            k1 = f(y, tq)
            k2 = f([yi + 0.5 * h * ki for yi, ki in zip(y, k1)], tq + 0.5 * h)
            k3 = f([yi + 0.5 * h * ki for yi, ki in zip(y, k2)], tq + 0.5 * h)
            k4 = f([yi + h * ki for yi, ki in zip(y, k3)], tq + h)
            y = [yi + h / 6 * (a + 2 * b + 2 * c + d) for yi, a, b, c, d in zip(y, k1, k2, k3, k4)]
        t_prev = float(t[j])
        for c in range(system.n_states):
            obs[j, c] = (y[c] + sigma * torch.randn(y0.shape[1], generator=gen, dtype=torch.float64)).float()
    return t.to(device), y0.float().to(device), obs.to(device), sigma
