"""Convergence diagnostics for multi-chain draws: split-R-hat, effective sample size, a summary table.

The reference's demo prints PyMC/ArviZ's summary after ``pm.sample`` (``demo_model.py:44``);
these are the same estimators (Vehtari et al. 2021: rank-free split-R-hat, Geyer initial-positive-sequence
ESS with FFT autocovariances) for the in-repo samplers, including the lock-step batched HMC whose draws
already come as ``[draws, chains, dim]``.
"""
from __future__ import annotations

from typing import Dict, Mapping

import numpy as np

__all__ = ["split_rhat", "effective_sample_size", "summarize"]


def _as_chains(x: np.ndarray) -> np.ndarray:
    """``[draws]`` or ``[draws, chains]`` -> ``[chains, draws]`` float64."""
    a = np.asarray(x, dtype=np.float64)
    if a.ndim == 1:
        a = a[:, None]
    if a.ndim != 2:
        raise ValueError("expected draws of one scalar quantity: [draws] or [draws, chains]")
    return a.T


def _split(chains: np.ndarray) -> np.ndarray:
    n = chains.shape[1] // 2
    if n < 2:
        raise ValueError("need at least 4 draws per chain")
    return np.concatenate([chains[:, :n], chains[:, -n:]], axis=0)


def split_rhat(x: np.ndarray) -> float:
    """Potential scale reduction on split chains; ~1.0 at convergence (> 1.01 is suspicious)."""
    c = _split(_as_chains(x))
    n = c.shape[1]
    within = c.var(axis=1, ddof=1).mean()
    between = n * c.mean(axis=1).var(ddof=1)
    if within == 0.0:
        return 1.0 if between == 0.0 else float("inf")
    return float(np.sqrt(((n - 1) / n * within + between / n) / within))


def _autocovariance(c: np.ndarray) -> np.ndarray:
    n = c.shape[1]
    size = 1 << (2 * n - 1).bit_length()
    f = np.fft.rfft(c - c.mean(axis=1, keepdims=True), size, axis=1)
    return np.fft.irfft(f * np.conj(f), size, axis=1)[:, :n] / n


def effective_sample_size(x: np.ndarray) -> float:
    """Bulk ESS of the mean over all chains (split chains, Geyer's initial monotone positive sequence)."""
    c = _split(_as_chains(x))
    m, n = c.shape
    acov = _autocovariance(c)
    within = acov[:, 0].mean() * n / (n - 1)
    var_plus = acov[:, 0].mean() + c.mean(axis=1).var(ddof=1) if m > 1 else acov[:, 0].mean()
    if var_plus == 0.0:
        return float(m * n)
    rho = 1.0 - (within - acov.mean(axis=0)) / var_plus
    rho[0] = 1.0
    # sum of adjacent pairs must stay positive and non-increasing
    tau = -1.0
    prev_pair = np.inf
    for t in range(0, n - 1, 2):
        pair = rho[t] + rho[t + 1]
        if pair < 0.0:
            break
        pair = min(pair, prev_pair)
        tau += 2.0 * pair
        prev_pair = pair
    tau = max(tau, 1.0 / np.log10(m * n))
    return float(m * n / tau)


def summarize(draws: Mapping[str, np.ndarray]) -> Dict[str, Dict[str, float]]:
    """``{name: draws[draws, chains] or [draws]}`` -> mean / sd / 3 % / 97 % quantiles / ESS / R-hat per name.
    Vector-valued entries (``[draws, chains, k]``) are reported per component as ``name[i]``."""
    table: Dict[str, Dict[str, float]] = {}
    for name, values in draws.items():
        a = np.asarray(values, dtype=np.float64)
        if a.ndim == 3:
            parts = {f"{name}[{i}]": a[:, :, i] for i in range(a.shape[2])}
        else:
            parts = {name: a}
        for key, v in parts.items():
            flat = v.reshape(-1)
            lo, hi = np.quantile(flat, [0.03, 0.97])
            table[key] = {
                "mean": float(flat.mean()), "sd": float(flat.std(ddof=1)), "q3": float(lo), "q97": float(hi),
                "ess": effective_sample_size(v), "rhat": split_rhat(v),
            }
    return table
