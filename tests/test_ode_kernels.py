"""The ODE kernels (``csrc/ode.cu`` and the dual-number ``csrc/ode_generic.cu``) against an independent fp64 oracle.

The oracle is NumPy only (no ``models/ode.py``, no torch).  It computes the kernels' discrete scheme: integrate from
``t = 0`` at ``y0``; interval ``j`` has ``h = (t_j - t_{j-1}) / substeps`` with ``t_{-1} = 0``; substep ``q`` starts at
``tau = t_{j-1} + q h``; RK4 evaluates its stages at ``tau, tau + h/2, tau + h/2, tau + h``; and
``LL = sum -r^2 / (2 sigma^2) - log sigma - log(2 pi) / 2`` over every time point, state and series.  The gradient is
a complex step, ``Im f(theta + i eps e_k) / eps`` in complex128 with ``eps = 1e-30``: exact to rounding and free of any
derivative rule.  Each system has a NumPy right-hand side next to its CUDA snippet and its torch function.

Tolerances come from the same oracle run in complex64 with ``eps = 2^-40``, an fp32 twin of the kernels' computation
(fp32 states and sums per series, fp64 across series): per component ``max(8 |twin - oracle|, 2^-18 S)``, where ``S``
is the sum of |per-term ll| for the LL and ``sum (|r| + |y|) |dy/dtheta_k| / sigma^2`` for gradient component k.  The
``|y|`` term is the scale of the fp32 rounding of the state itself, which reaches the gradient through ``r``: with
``r`` much smaller than ``y`` and few series per node, the twin's own rounding is a single draw that can be 8 times
smaller than the kernel's by chance (ode.cu with 1 to 3 series per node went past ``sum |r dy/dtheta_k|`` alone).

CPU: the oracle against the closed-form solution of a forced linear system, ``OdeShards.reference_partial`` against
the oracle in every case, plausible kernel bugs applied to the oracle each move some case by more than 4x its
tolerance, the function-coverage system stays inside every function's domain, ``OdeShards`` validates its input,
and snippets with commas or float arguments of the elementary functions compile.
GPU: every node block of every case against the oracle, and a second evaluation gives the same bits.
"""
from __future__ import annotations

import math
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass
from functools import lru_cache
from typing import Callable, List, Optional, Tuple

import numpy as np
import pytest
import torch

from pytensor_federated_b200.models import LOTKA_VOLTERRA, CustomFamily, OdeShards, OdeSystem

EPS = {np.complex128: 1e-30, np.complex64: 2.0**-40}
TWIN_FACTOR = 8.0        # the kernel may be this much further from the oracle than the fp32 twin
FLOOR = 2.0**-18         # ... or this fraction of the sum of magnitudes, whichever is larger
MOVE_FACTOR = 4.0        # a bug must move some component by more than this many tolerances
LOG_SQRT_2PI = 0.918938533204672742


# ------------------------------------------------------------------------------------ elementary functions
class Ops:
    """The functions a NumPy right-hand side may call, on real or complex-step arrays.  ``bug`` replaces one
    derivative rule by a wrong one, as ``f(Re z) + i Im z wrong'(Re z)``; ``domain`` keeps the smallest argument
    of ``log``, ``sqrt`` and ``pow`` and the smallest |denominator| of ``div``."""

    def __init__(self, bug: Optional[str] = None):
        self.bug = bug
        self.domain = {}

    def _seen(self, name, x):
        self.domain[name] = min(self.domain.get(name, np.inf), float(np.min(x)))

    def _fn(self, name, f, wrong, z):
        if self.bug == name + "'":
            re = np.real(z)
            return f(re) + 1j * np.imag(z) * wrong(re)
        return f(z)

    def exp(self, z):
        return np.exp(z)

    def log(self, z):
        self._seen("log", np.real(z))
        return self._fn("log", np.log, lambda x: -1.0 / x, z)

    def sqrt(self, z):
        self._seen("sqrt", np.real(z))
        return self._fn("sqrt", np.sqrt, lambda x: 1.0 / np.sqrt(x), z)

    def sin(self, z):
        return self._fn("sin", np.sin, lambda x: -np.cos(x), z)

    def cos(self, z):
        return self._fn("cos", np.cos, np.sin, z)

    def tanh(self, z):
        return self._fn("tanh", np.tanh, lambda x: 1.0 + np.tanh(x) ** 2, z)

    def pow(self, z, p):
        self._seen("pow", np.real(z))
        return self._fn("pow", lambda x: np.power(x, p), lambda x: p * np.power(x, p), z)

    def square(self, z):
        return z * z

    def div(self, a, b):
        """``a / b`` for a dual ``b`` (the dual / float case needs no rule)."""
        self._seen("div", np.abs(np.real(b)))
        if self.bug == "quotient'" and np.iscomplexobj(a):
            return a.real / b.real + 1j * (a.imag / b.real + a.real * b.imag / b.real**2)
        if self.bug == "float/dual'" and not np.iscomplexobj(a):
            return a / b.real + 1j * (a * b.imag / b.real**2)
        return a / b


# ------------------------------------------------------------------------------------------------ systems
@dataclass(frozen=True)
class System:
    name: str
    ns: int
    np_: int
    rhs: Callable                  # NumPy: (y, th, t, ops) -> n_states arrays
    cuda: Optional[str] = None     # None: the hand-written csrc/ode.cu (Lotka-Volterra only)
    torch_rhs: Optional[Callable] = None


def _lv(y, th, t, m):
    return [th[0] * y[0] - th[1] * y[0] * y[1], th[3] * y[0] * y[1] - th[2] * y[1]]


def _forced(y, th, t, m):
    return [-th[0] * y[0] + th[1] * m.sin(1.5 * t) + m.cos(th[2] * t)]


def _forced_torch(y, th, t):
    return (-th[0] * y[0] + th[1] * math.sin(1.5 * t) + torch.cos(th[2] * t),)


FUNCS_CUDA = (
    "dy[0] = th[0] * sin(y[1]) - th[1] * tanh(y[0]);"
    "dy[1] = -y[0] / sqrt(1.f + square(y[1])) + th[2] * log(1.f + square(y[2])) - y[1] / 4.f;"
    "dy[2] = th[3] * (2.f - exp(-square(y[0]))) / pow(1.5f + cos(y[1]), 1.5f) - y[2] / 3.f - 1.f / (1.f + square(y[2]));"
)


def _funcs(y, th, t, m):
    return [
        th[0] * m.sin(y[1]) - th[1] * m.tanh(y[0]),
        m.div(-y[0], m.sqrt(1.0 + m.square(y[1]))) + th[2] * m.log(1.0 + m.square(y[2])) - y[1] / 4.0,
        m.div(th[3] * (2.0 - m.exp(-m.square(y[0]))), m.pow(1.5 + m.cos(y[1]), 1.5)) - y[2] / 3.0
        - m.div(1.0, 1.0 + m.square(y[2])),
    ]


def _funcs_torch(y, th, t):
    return (
        th[0] * torch.sin(y[1]) - th[1] * torch.tanh(y[0]),
        -y[0] / torch.sqrt(1.0 + y[1] ** 2) + th[2] * torch.log(1.0 + y[2] ** 2) - y[1] / 4.0,
        th[3] * (2.0 - torch.exp(-y[0] ** 2)) / torch.pow(1.5 + torch.cos(y[1]), 1.5) - y[2] / 3.0 - 1.0 / (1.0 + y[2] ** 2),
    )


CHAIN_CUDA = " ".join(["dy[0] = th[0] - th[1] * y[0];"]
                      + [f"dy[{i}] = th[{2 * i}] * y[{i - 1}] - th[{2 * i + 1}] * y[{i}];" for i in range(1, 8)])


def _chain(y, th, t, m):
    return [th[0] - th[1] * y[0]] + [th[2 * i] * y[i - 1] - th[2 * i + 1] * y[i] for i in range(1, 8)]


def _pow1(y, th, t, m):
    return [m.pow(y[0], 0.5) * th[0]]


SYSTEMS = {
    "lv": System("lv", 2, 4, _lv, LOTKA_VOLTERRA.rhs_cuda, LOTKA_VOLTERRA.rhs_torch),
    # y' = -a y + b sin(1.5 t) + cos(w t): a float forcing term and a dual one
    "forced": System("forced", 1, 3, _forced, "dy[0] = -th[0] * y[0] + th[1] * sin(1.5f * t) + cos(th[2] * t);",
                     _forced_torch),
    # every elementary function, pow with p = 1.5, dual/dual, float/dual, dual/float, float - dual, unary minus
    "funcs": System("funcs", 3, 4, _funcs, FUNCS_CUDA, _funcs_torch),
    # the limits OdeSystem accepts: 8 states, 16 parameters (a linear chain), and 1 state, 1 parameter
    "chain": System("chain", 8, 16, _chain, CHAIN_CUDA,
                    lambda y, th, t: _chain(y, th, t, None)),
    "pow1": System("pow1", 1, 1, _pow1, "dy[0] = pow(y[0], 0.5f) * th[0];",
                   lambda y, th, t: (torch.pow(y[0], 0.5) * th[0],)),
}


@lru_cache(maxsize=None)
def ode_system(name: str) -> OdeSystem:
    s = SYSTEMS[name]
    if name == "lv":
        return LOTKA_VOLTERRA
    return OdeSystem(s.cuda, s.torch_rhs, n_states=s.ns, n_params=s.np_, name=f"test-{name}")


# ------------------------------------------------------------------------------------------------- oracle
def integrate(system: System, t, y0, th, substeps: int, ops: Ops, rd, bug: Optional[str] = None):
    """RK4 as the kernels step it; yields ``(j, y)`` after interval ``j``.  ``t`` [n_t] and the arithmetic on time
    are in ``rd``; ``y0`` [n_states, ...] and ``th`` [n_params, ...] broadcast against each other."""
    f = lambda yy, tt: system.rhs(yy, th, tt, ops)
    y = [np.asarray(v) for v in y0]
    t_prev = t[0] if bug == "t0_origin" else rd(0.0)
    for j in range(t.size):
        h = (t[j] - t_prev) / rd(substeps)
        half = rd(0.5) * h
        for q in range(substeps - 1 if bug == "drop_substep" else substeps):
            tau = t_prev if bug == "tau_frozen" else t_prev + rd(q) * h
            t23 = tau if bug == "stage23_at_tau" else tau + half
            t4 = tau + half if bug == "stage4_at_half" else tau + h
            k1 = f(y, tau)
            k2 = f([a + half * b for a, b in zip(y, k1)], t23)
            k3 = f([a + half * b for a, b in zip(y, k2)], t23)
            k4 = f([a + h * b for a, b in zip(y, k3)], t4)
            h6 = h * rd(1.0 / 6.0)
            y = [a + h6 * (b1 + 2.0 * b2 + 2.0 * b3 + b4) for a, b1, b2, b3, b4 in zip(y, k1, k2, k3, k4)]
        t_prev = t[j]
        yield j, y


@dataclass
class Shard:
    t: np.ndarray        # float32 [n_t]
    y0: np.ndarray       # float32 [n_states, n_series]
    y_obs: np.ndarray    # float32 [n_t, n_states, n_series]
    sigma: float
    node: int = 0


@dataclass
class Case:
    name: str
    system: str
    shards: List[Shard]
    theta: np.ndarray              # float32 [n_nodes, n_params]
    substeps: int
    kernels: Tuple[str, ...] = ("dual",)   # "hand": csrc/ode.cu, "dual": csrc/ode_generic.cu
    per_node: bool = False
    grid: Optional[int] = None
    expect_grid: Optional[int] = None


BUGS = ["stage23_at_tau", "stage4_at_half", "tau_frozen", "drop_substep", "t0_origin", "obs_transposed", "y0_shift",
        "drop_last_series", "neighbour_theta", "cos'", "sin'", "tanh'", "sqrt'", "log'", "pow'", "quotient'",
        "float/dual'"]


def oracle(case: Case, cdt=np.complex128, bug: Optional[str] = None, ops: Optional[Ops] = None):
    """``(vals, scale)``, both ``[n_nodes, 1 + n_params]``: the kernels' node blocks ``[LL, dLL/dtheta]`` and the sums
    of magnitudes that set the tolerance floor (complex128 only).  ``bug`` applies one of :data:`BUGS`."""
    system = SYSTEMS[case.system]
    ns, npar = system.ns, system.np_
    rd = np.float64 if cdt is np.complex128 else np.float32
    eps = EPS[cdt]
    n_nodes = case.theta.shape[0]
    ops = ops or Ops(bug)
    vals = np.zeros((n_nodes, 1 + npar))
    scale = np.zeros((n_nodes, 1 + npar))
    groups = {}   # shards on the same time grid are integrated together, each series with its node's theta
    for sh in case.shards:
        y0, yo = sh.y0, sh.y_obs
        n_t, n = yo.shape[0], yo.shape[2]
        if bug == "obs_transposed":
            yo = yo.reshape(ns, n_t, n).transpose(1, 0, 2)
        if bug == "y0_shift":
            y0 = np.roll(y0, -1, axis=1)
        if bug == "drop_last_series":
            y0, yo = y0[:, :-1], yo[:, :, :-1]
        node_theta = (sh.node + 1) % n_nodes if bug == "neighbour_theta" else sh.node
        m = y0.shape[1]
        g = groups.setdefault(sh.t.tobytes(), {"t": sh.t, "y0": [], "yo": [], "th": [], "sig": [], "node": []})
        g["y0"].append(y0)
        g["yo"].append(yo)
        g["th"].append(np.repeat(case.theta[node_theta][:, None], m, axis=1))
        g["sig"].append(np.full(m, sh.sigma, dtype=np.float32))
        g["node"].append(np.full(m, sh.node))
    for g in groups.values():
        y0 = np.concatenate(g["y0"], axis=1)
        yo = np.concatenate(g["yo"], axis=2)
        th_real = np.concatenate(g["th"], axis=1)            # [n_params, n]
        sig = np.concatenate(g["sig"]).astype(rd)
        node = np.concatenate(g["node"])
        n = y0.shape[1]
        # direction k of the complex step perturbs parameter k: th [n_params, n_params (direction), n]
        th = np.repeat(th_real[:, None, :], npar, axis=1).astype(cdt)
        th[np.arange(npar), np.arange(npar)] += 1j * eps
        ys = [np.repeat(y0[c][None, :], npar, axis=0).astype(cdt) for c in range(ns)]
        inv_var = rd(1.0) / (sig * sig)
        log_norm = -np.log(sig) - rd(LOG_SQRT_2PI)
        acc = np.zeros((npar, n), dtype=cdt)                   # per series, in the working precision
        s_acc = np.zeros((1 + npar, n))
        for j, y in integrate(system, g["t"].astype(rd), ys, th, case.substeps, ops, rd, bug):
            for c in range(ns):
                r = yo[j, c].astype(rd) - y[c]
                term = -0.5 * r * r * inv_var + log_norm
                acc += term
                if cdt is np.complex128:
                    s_acc[0] += np.abs(term.real[0])
                    s_acc[1:] += (np.abs(r.real) + np.abs(y[c].real)) * np.abs(y[c].imag / eps) * inv_var
        per_series = np.concatenate([acc.real[:1].astype(np.float64), (acc.imag / rd(eps)).astype(np.float64)])
        for k in range(1 + npar):
            np.add.at(vals[:, k], node, per_series[k])
            np.add.at(scale[:, k], node, s_acc[k])
    return vals, scale


@lru_cache(maxsize=None)
def expected(name: str):
    """``(oracle, tolerance, scale)`` of a case."""
    case = CASES[name]
    want, scale = oracle(case)
    twin, _ = oracle(case, np.complex64)
    return want, np.maximum(TWIN_FACTOR * np.abs(twin - want), FLOOR * scale), scale


# -------------------------------------------------------------------------------------------------- cases
def _grid(n_t: int, t_end: float, rng, uniform: bool) -> np.ndarray:
    if uniform:
        return np.linspace(t_end / n_t, t_end, n_t).astype(np.float32)
    t = np.sort(rng.uniform(0.0, t_end, size=n_t))
    if n_t >= 6:
        t[0] = 0.0           # a zero-length first interval
        t[4] = t[3]          # a repeated time point
    return t.astype(np.float32)


Y0_RANGE = {"lv": [(1.0, 2.0), (0.5, 1.5)], "forced": [(-1.0, 1.0)], "funcs": [(-0.6, 0.6)] * 3,
            "chain": [(0.0, 1.0)] * 8, "pow1": [(0.5, 2.0)]}
THETA = {"lv": [1.0, 0.4, 0.8, 0.2], "forced": [0.7, 1.2, 2.0], "funcs": [0.9, 0.6, 0.5, 0.8],
         "chain": [1.0, 0.8] + [0.9, 0.7] * 7, "pow1": [0.6]}


def make_case(name, system, sizes, *, n_t=12, t_end=4.0, uniform=False, sigmas=(0.05,), substeps=8, nodes=None,
              n_nodes=None, seed=0, **kw) -> Case:
    """Shards of ``sizes`` series on one time grid, observed around the kernel scheme's own trajectory at a node's
    true parameters; the case evaluates each node at parameters a few percent off."""
    s = SYSTEMS[system]
    rng = np.random.default_rng(seed)
    per_node = nodes is not None
    nodes = list(nodes) if per_node else [0] * len(sizes)
    n_nodes = n_nodes if per_node else 1
    true = np.asarray(THETA[system]) * (1.0 + 0.05 * rng.standard_normal((n_nodes, s.np_)))
    probe = (true * (1.0 + 0.03 * rng.standard_normal(true.shape))).astype(np.float32)
    t = _grid(n_t, t_end, rng, uniform)
    shards = []
    for i, (n, node) in enumerate(zip(sizes, nodes)):
        y0 = np.stack([rng.uniform(lo, hi, size=n) for lo, hi in Y0_RANGE[system]]).astype(np.float32)
        th = np.repeat(true[node][:, None], n, axis=1)
        traj = np.stack([np.stack(y) for _, y in integrate(s, t.astype(np.float64), y0.astype(np.float64), th,
                                                            substeps, Ops(), np.float64)])
        sigma = float(sigmas[i % len(sigmas)])
        y_obs = (traj + sigma * rng.standard_normal(traj.shape)).astype(np.float32)
        shards.append(Shard(t, y0, y_obs, sigma, node))
    return Case(name, system, shards, probe, substeps, per_node=per_node, **kw)


LV = ("hand", "dual")


def _cases() -> List[Case]:
    return [
        # Lotka-Volterra on both kernels: substeps 1, 3, 8, 32; grids with t_0 = 0 and a repeated point; sigma 0.01, 2
        make_case("lv-substeps1-nt64", "lv", [150], n_t=64, t_end=6.0, substeps=1, sigmas=(0.01,), seed=1, kernels=LV),
        make_case("lv-substeps3-nt1", "lv", [70, 90], n_t=1, t_end=1.5, substeps=3, sigmas=(2.0, 0.01), seed=2, kernels=LV),
        make_case("lv-substeps8", "lv", [200, 60], n_t=20, t_end=6.0, substeps=8, sigmas=(0.01, 2.0), seed=3, kernels=LV),
        make_case("lv-substeps32", "lv", [100], n_t=8, t_end=5.0, substeps=32, sigmas=(0.1,), seed=4, kernels=LV),
        # launch shapes: series across CTA boundaries, the default grid, one CTA, and grid strides that wrap
        make_case("shapes-default-grid", "lv", [1, 127, 128, 129, 1000], n_t=6, uniform=True, substeps=4, seed=5,
                  sigmas=(0.05, 0.2), kernels=LV, expect_grid=11),
        make_case("shapes-grid1", "lv", [1, 127, 128, 129, 1000], n_t=6, uniform=True, substeps=4, seed=5,
                  sigmas=(0.05, 0.2), kernels=LV, grid=1, expect_grid=1),
        make_case("shapes-grid2", "lv", [900], n_t=5, substeps=4, seed=6, kernels=LV, grid=2, expect_grid=2),
        make_case("shapes-grid3", "lv", [1000], n_t=5, substeps=4, seed=7, kernels=LV, grid=3, expect_grid=3),
        # per-node blocks: 256 nodes x 4 parameters = 1024 theta words; nodes owning 0, 1 and 3 non-adjacent shards
        make_case("nodes-256", "lv", [12 + i % 9 for i in range(256)], n_t=3, t_end=2.0, substeps=2, seed=8,
                  nodes=list(np.random.default_rng(8).permutation(256)), n_nodes=256, kernels=LV),
        make_case("nodes-0-1-3", "lv", [40, 129, 7, 300, 64], n_t=10, substeps=4, seed=9, sigmas=(0.05, 0.3),
                  nodes=[2, 0, 2, 3, 2], n_nodes=4, kernels=LV),
        # user systems
        make_case("forced", "forced", [300, 45], n_t=24, t_end=5.0, substeps=4, sigmas=(0.05, 0.5), seed=10),
        make_case("funcs", "funcs", [200, 130], n_t=12, t_end=4.0, substeps=6, sigmas=(0.05, 0.2), seed=11,
                  nodes=[1, 0], n_nodes=2),
        make_case("chain-8x16", "chain", [257], n_t=8, t_end=3.0, substeps=6, seed=12),
        make_case("chain-8x16-64nodes", "chain", [8] * 64, n_t=4, t_end=2.0, substeps=2, seed=13,
                  nodes=list(range(64)), n_nodes=64),
        make_case("pow-1x1", "pow1", [129], n_t=10, t_end=3.0, substeps=5, seed=14),
    ]


CASES = {c.name: c for c in _cases()}


def shard_model(case: Case, kernel: str, device) -> OdeShards:
    sh = case.shards
    kw = {"node_ids": [s.node for s in sh], "n_nodes": case.theta.shape[0]} if case.per_node else {}
    return OdeShards([torch.from_numpy(s.t).to(device) for s in sh], [torch.from_numpy(s.y0).to(device) for s in sh],
                     [torch.from_numpy(s.y_obs).to(device) for s in sh], [s.sigma for s in sh], substeps=case.substeps,
                     system=None if kernel == "hand" else ode_system(case.system), **kw)


# ----------------------------------------------------------------------------------------- CPU: the oracle
def test_oracle_matches_the_closed_form_of_a_forced_linear_system():
    """y' = -a y + b sin(1.5 t) + cos(w t) at 64 substeps: trajectory and its parameter derivatives within 1e-9 of
    the closed form, on a grid with t_0 = 0 and a repeated time point."""
    case = make_case("closed-form", "forced", [40], n_t=16, t_end=5.0, substeps=64, seed=20)
    sh = case.shards[0]
    n, eps = sh.y0.shape[1], 1e-30
    th = np.repeat(case.theta[0].astype(np.complex128)[:, None, None], 3, axis=1).repeat(n, axis=2)
    th[np.arange(3), np.arange(3)] += 1j * eps
    y0 = sh.y0[0].astype(np.float64)
    got = np.stack([y[0] for _, y in integrate(SYSTEMS["forced"], sh.t.astype(np.float64), [y0[None, :] + 0j],
                                                th, 64, Ops(), np.float64)])          # [n_t, direction, n]

    a, b, w = th[0], th[1], th[2]
    t = sh.t.astype(np.float64)[:, None, None]
    ea = np.exp(-a * t)
    want = (y0 * ea + b * (a * np.sin(1.5 * t) - 1.5 * np.cos(1.5 * t) + 1.5 * ea) / (a * a + 2.25)
            + (a * np.cos(w * t) + w * np.sin(w * t) - a * ea) / (a * a + w * w))
    assert np.max(np.abs(got.real - want.real)) < 1e-9
    assert np.max(np.abs(got.imag - want.imag)) / eps < 1e-9
    assert t[0, 0, 0] == 0.0 and t[4, 0, 0] == t[3, 0, 0]


@pytest.mark.parametrize("name", list(CASES))
def test_reference_partial_matches_the_oracle(name):
    """``OdeShards.reference_partial`` (torch autograd, what ``bench.py`` checks against) equals the oracle."""
    case = CASES[name]
    want, _, scale = expected(name)
    for kernel in case.kernels:
        model = shard_model(case, kernel, "cpu")
        got = model.per_node(model.reference_partial([case.theta.astype(np.float64)]))
        assert np.all(np.abs(got - want) <= 1e-10 * scale), f"{name} {kernel}: {np.max(np.abs(got - want) / scale)}"


def _moves(case_name: str, bug: str) -> float:
    want, tol, _ = expected(case_name)
    moved, _ = oracle(CASES[case_name], bug=bug)
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.nanmax(np.where(tol > 0, np.abs(moved - want) / tol, np.where(moved != want, np.inf, 0.0))))


# cases that can show each bug, cheapest first (a derivative rule only matters where its function is used)
MUTATION_CASES = {"cos'": ["funcs", "forced"], "sin'": ["funcs"], "tanh'": ["funcs"], "sqrt'": ["funcs"],
                  "log'": ["funcs"], "pow'": ["funcs", "pow-1x1"], "quotient'": ["funcs"], "float/dual'": ["funcs"],
                  "neighbour_theta": ["nodes-0-1-3", "funcs"]}


@pytest.mark.parametrize("bug", BUGS)
def test_each_kernel_bug_moves_some_case_beyond_its_tolerance(bug):
    names = MUTATION_CASES.get(bug, ["lv-substeps8", "lv-substeps3-nt1", "forced", "funcs"])
    ratios = {}
    for name in names:
        ratios[name] = _moves(name, bug)
        if ratios[name] > MOVE_FACTOR:
            return
    pytest.fail(f"{bug} moves no case by more than {MOVE_FACTOR} tolerances: {ratios}")


def test_function_coverage_system_stays_inside_every_domain():
    ops = Ops()
    oracle(CASES["funcs"], ops=ops)
    assert set(ops.domain) == {"log", "sqrt", "pow", "div"}
    assert ops.domain["log"] >= 1.0 and ops.domain["sqrt"] >= 1.0 and ops.domain["pow"] > 0.3
    assert ops.domain["div"] > 0.3
    # the observed series stay in a bounded range, far from tanh / exp saturation
    assert all(np.max(np.abs(s.y_obs)) < 10 for s in CASES["funcs"].shards)


def test_tolerances_are_tight():
    """The tolerance is a small fraction of what each component measures (so a GPU pass is a real check)."""
    for name in CASES:
        want, tol, scale = expected(name)
        live = scale > 0
        assert np.all(tol[live] < 1e-3 * scale[live]), name
        assert np.all(tol[~live] == 0) and np.all(want[~live] == 0), name


# ------------------------------------------------------------------------------- CPU: validation, compilation
def _lv_args(n_t=4):
    t = torch.linspace(0.5, 2.0, n_t)
    return [t], [torch.ones(2, 3)], [torch.ones(n_t, 2, 3)]


@pytest.mark.parametrize("substeps", [0, -1, 2.5, True, "8"])
def test_ode_shards_reject_bad_substeps(substeps):
    with pytest.raises(ValueError, match="substeps"):
        OdeShards(*_lv_args(), [0.1], substeps=substeps)


@pytest.mark.parametrize("sigma", [0.0, -0.1, float("nan"), float("inf")])
def test_ode_shards_reject_bad_sigma(sigma):
    with pytest.raises(ValueError, match="sigma"):
        OdeShards(*_lv_args(), [sigma])


@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
def test_ode_shards_reject_times_that_are_not_finite(bad):
    ts, y0s, obs = _lv_args()
    ts[0][2] = bad
    with pytest.raises(ValueError, match="time"):
        OdeShards(ts, y0s, obs, [0.1])
    assert OdeShards(*_lv_args(), [0.1], substeps=np.int64(3)).substeps == 3


@pytest.fixture(scope="module")
def compiled():
    """Builds the snippets of the two tests below in parallel: ``{name: library or the exception}``."""
    snippets = {
        "pow": ode_system("pow1"),
        "powf": CustomFamily("const float d = y - eta; ll = -0.5f * powf(d, 2.f); r = d;", name="comma"),
        "forced": ode_system("forced"),
        "floats": OdeSystem("dy[0] = th[0] * (exp(0.5f) + log(2.f + t) + sqrt(t) + cos(t) + tanh(t) + pow(2.f, t)) - y[0];",
                            None, n_states=1, n_params=1, name="float-args"),
    }

    def build(s):
        try:
            return s.compile()
        except RuntimeError as ex:
            return ex

    with ThreadPoolExecutor(len(snippets)) as pool:
        return dict(zip(snippets, pool.map(build, snippets.values())))


def test_snippets_with_commas_compile(compiled):
    """nvcc splits -D values at commas; the snippet travels in a header instead."""
    assert not isinstance(compiled["pow"], Exception), compiled["pow"]
    assert not isinstance(compiled["powf"], Exception), compiled["powf"]
    assert compiled["pow"].b200_launch_ode_custom is not None and compiled["powf"].b200_launch_glm_custom is not None


def test_elementary_functions_take_float_arguments(compiled):
    """``sin(1.5f * t)`` is a float forcing term; ``exp``, ``log``, ``sqrt``, ``cos``, ``tanh`` and ``pow`` of floats
    compile too."""
    for name in ("forced", "floats"):
        assert not isinstance(compiled[name], Exception), compiled[name]
        assert compiled[name].b200_launch_ode_custom is not None


# --------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from pytensor_federated_b200.ops import native

    native.load()  # a GPU box without the native library is a failure, not a skip
    return torch.device("cuda:0")


@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", list(CASES))
def test_kernel_matches_the_oracle(dev, name):
    from pytensor_federated_b200.parallel import FederatedEngine

    case = CASES[name]
    want, tol, _ = expected(name)
    for kernel in case.kernels:
        model = shard_model(case, kernel, dev)
        with FederatedEngine(model, grid=case.grid) as eng:
            if case.expect_grid is not None:
                assert eng.grid == case.expect_grid
            raw = eng.evaluate_raw([case.theta])
            again = eng.evaluate_raw([case.theta])
        assert np.array_equal(raw, again), f"{name} {kernel}: a second evaluation changed bits"
        got = model.per_node(raw)
        err = np.abs(got - want)
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(tol > 0, err / tol, np.where(err > 0, np.inf, 0.0))
        print(f"{name} [{kernel}]: max |kernel - oracle| / tolerance = {ratio.max():.3g} (LL {ratio[:, 0].max():.3g})")
        worst = np.unravel_index(np.argmax(ratio), ratio.shape)
        assert np.all(err <= tol), (f"{name} {kernel}: node {worst[0]} component {worst[1]}: kernel {got[worst]!r}, "
                                    f"oracle {want[worst]!r}, tolerance {tol[worst]!r}")
