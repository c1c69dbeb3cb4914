"""Curvature of federated GLMs: Hessian-vector products, the full Hessian, and the Laplace approximation.

The Hessian of a GLM log-likelihood is a sum over private rows, ``sum_i w_i h_i x_i x_i'``, so like the gradient it
is computed on each node and reduced by the fused epoch: ``GlmShards(..., hvp=True)`` evaluates K products ``H v``
per launch (:func:`glm_hvp_fn`), :func:`glm_hessian` assembles H from ``ceil(D / K)`` launches, and :func:`laplace`
turns the mode and H into a Gaussian approximation of the posterior and its evidence.
"""
from __future__ import annotations

import logging
import math
from typing import Callable, Tuple

import numpy as np

from .mcmc import find_map

_log = logging.getLogger(__name__)

HvpFn = Callable[[np.ndarray, np.ndarray], Tuple[np.ndarray, np.ndarray, np.ndarray]]


def glm_hvp_fn(engine) -> HvpFn:
    """Adapts ``FederatedEngine(GlmShards(..., hvp=True, n_chains=K))`` to ``(theta[n, D], v[n, D]) -> (logp[n],
    grad[n, D], hv[n, D])`` with the flat ``theta = [intercept[G], beta[P]]`` of
    :func:`~pytensor_federated_b200.sampling.glm_batch_fn` and a direction ``v`` in the same layout.  ``hv`` is the
    Hessian of the log-likelihood at ``theta`` times ``v``.  Any n is evaluated in ``ceil(n / K)`` launches; a short
    last tile is padded by repeating its last row."""
    m = engine.model
    if not getattr(m, "hvp", False):
        raise ValueError("glm_hvp_fn needs an engine whose model was built with GlmShards(..., hvp=True)")
    cap, D = int(m.n_chains), m.n_params // 2

    def tile(theta: np.ndarray, v: np.ndarray):
        rows = np.concatenate([theta, v], axis=1)
        logp, *outs = engine.evaluate(*m.inputs_from_theta(rows if cap > 1 else rows[0]))
        flat = np.concatenate([np.asarray(o).reshape(cap, -1) for o in outs], axis=1)   # [cap, 2 D]
        return np.asarray(logp).reshape(-1), flat[:, :D], flat[:, D:]

    def fn(theta: np.ndarray, v: np.ndarray):
        theta, v = np.asarray(theta, dtype=np.float64), np.asarray(v, dtype=np.float64)
        if theta.ndim != 2 or theta.shape[1] != D or v.shape != theta.shape:
            raise ValueError(f"theta and v must both be [n, {D}], got {theta.shape} and {v.shape}")
        logps, grads, hvs = [], [], []
        for first in range(0, theta.shape[0], cap):
            tb, vb = theta[first : first + cap], v[first : first + cap]
            k = tb.shape[0]
            if k < cap:
                tb = np.concatenate([tb, np.repeat(tb[-1:], cap - k, axis=0)], axis=0)
                vb = np.concatenate([vb, np.repeat(vb[-1:], cap - k, axis=0)], axis=0)
            lp, gr, hv = tile(tb, vb)
            logps.append(lp[:k])
            grads.append(gr[:k])
            hvs.append(hv[:k])
        return np.concatenate(logps), np.concatenate(grads, axis=0), np.concatenate(hvs, axis=0)

    return fn


def glm_hessian(engine, theta: np.ndarray) -> Tuple[float, np.ndarray, np.ndarray]:
    """``(logp, grad[D], H[D, D])`` of the log-likelihood at the flat ``theta[D]`` (:func:`glm_hvp_fn`'s layout).

    H is built column by column from ``ceil(D / K)`` launches whose K pairs all carry ``theta`` and one unit
    direction each, then symmetrised as ``(H + H') / 2``; the largest asymmetry removed, ``max |H - H'| / 2``, is
    logged at INFO level (it is rounding: the kernel sums each column in its own order)."""
    theta = np.asarray(theta, dtype=np.float64).reshape(-1)
    D = theta.shape[0]
    logp, grad, cols = glm_hvp_fn(engine)(np.broadcast_to(theta, (D, D)), np.eye(D))
    H = cols.T   # launch column j is H e_j
    asym = 0.5 * float(np.max(np.abs(H - H.T))) if D else 0.0
    _log.info("glm_hessian: D = %d, largest asymmetry removed %.3e (largest |H| %.3e)", D, asym,
              float(np.max(np.abs(H))) if D else 0.0)
    return float(logp[0]), grad[0].copy(), 0.5 * (H + H.T)


def laplace(logp_dlogp: Callable, hessian: Callable, x0: np.ndarray, **find_map_kwargs) -> dict:
    """Laplace approximation of the density ``exp(logp)`` around its mode.

    ``logp_dlogp(theta) -> (logp, grad)`` as for :func:`find_map`, and ``hessian(theta) -> H[D, D]`` the Hessian of
    the same logp (for a federated GLM, ``lambda th: glm_hessian(engine, th)[2]``).  The mode comes from
    :func:`find_map` (``find_map_kwargs`` go to it); then ``cov = (-H)^-1`` through a Cholesky factorisation of
    ``-H``.  Returns a dict with ``mean``, ``cov``, ``sd``, ``logp`` (at the mode), ``log_evidence = logp + D / 2
    log(2 pi) - log det(-H) / 2`` (the log normalising constant of ``exp(logp)`` under the approximation),
    ``n_evals`` (of ``logp_dlogp``), ``n_hessian_evals`` and ``converged`` (of the optimiser).  Raises ValueError,
    naming the smallest eigenvalue, when ``-H`` is not positive definite at the mode.

    Priors are the caller's to add to both callables.  For ``theta ~ N(0, tau^2 I)``::

        def logp_dlogp(th):
            lp, g = loglik_grad(th)
            return lp - th @ th / (2 tau^2) - D / 2 log(2 pi tau^2), g - th / tau^2

        def hessian(th):
            return glm_hessian(engine, th)[2] - np.eye(D) / tau^2

    With the prior's normalising constant included, ``log_evidence`` approximates the log marginal likelihood.
    """
    from scipy.linalg import cho_solve, solve_triangular

    mean, info = find_map(logp_dlogp, x0, **find_map_kwargs)
    n_evals, D = int(info["n_evals"]), mean.shape[0]

    def factor(x):
        H = np.asarray(hessian(x), dtype=np.float64)
        if H.shape != (D, D):
            raise ValueError(f"hessian returned shape {H.shape}, expected {(D, D)}")
        A = -0.5 * (H + H.T)
        try:
            return np.linalg.cholesky(A)
        except np.linalg.LinAlgError:
            lam = float(np.linalg.eigvalsh(A)[0])
            raise ValueError(f"-H is not positive definite at the mode: its smallest eigenvalue is {lam:.6g}") from None

    # L-BFGS-B stops once the gradient is small, not at the mode itself: one Newton step with the Hessian there
    # moves to the mode of the local quadratic (exact for a Gaussian density), and is kept where logp does not drop
    L = factor(mean)
    n_hessian = 1
    lp0, g = logp_dlogp(mean)
    step = cho_solve((L, True), np.asarray(g, dtype=np.float64))
    lp1, _ = logp_dlogp(mean + step)
    n_evals += 2
    logp = float(lp0)
    if np.isfinite(lp1) and lp1 >= lp0:
        mean, logp = mean + step, float(lp1)
        L = factor(mean)
        n_hessian += 1
    Linv = solve_triangular(L, np.eye(D), lower=True)
    cov = Linv.T @ Linv
    logdet = 2.0 * float(np.sum(np.log(np.diag(L))))
    return {"mean": mean, "cov": cov, "sd": np.sqrt(np.diag(cov)), "logp": logp,
            "log_evidence": logp + 0.5 * D * math.log(2.0 * math.pi) - 0.5 * logdet,
            "n_evals": n_evals, "n_hessian_evals": n_hessian,
            "converged": bool(info["converged"])}


__all__ = ["glm_hvp_fn", "glm_hessian", "laplace"]
