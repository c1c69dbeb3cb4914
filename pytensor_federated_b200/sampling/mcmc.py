"""MAP, HMC and NUTS over a flat parameter vector."""
from __future__ import annotations

import dataclasses
import math
from math import inf, isfinite
from typing import Callable, Dict, Optional, Tuple

import numpy as np

LogpDlogp = Callable[[np.ndarray], Tuple[float, np.ndarray]]


@dataclasses.dataclass
class SamplerResult:
    """Draws and diagnostics of one chain (``hmc_sample`` / ``nuts_sample``)."""

    samples: np.ndarray            # [draws, dim]
    logp: np.ndarray               # [draws]
    accept_rate: float
    step_size: float
    n_logp_evals: int
    tree_depth: Optional[np.ndarray] = None
    divergences: int = 0
    inv_mass: Optional[np.ndarray] = None       # adapted diagonal inverse mass matrix
    rng_state: Optional[dict] = None            # numpy Generator state after the last draw

    # -- checkpoint / resume (the reference keeps no sampler state; PyMC does it for its users) --
    def save(self, path: str) -> None:
        """Writes everything needed to continue the chain to ``path`` (``.npz``)."""
        import json

        np.savez(
            path, samples=self.samples, logp=self.logp, accept_rate=self.accept_rate, step_size=self.step_size,
            n_logp_evals=self.n_logp_evals, divergences=self.divergences,
            tree_depth=self.tree_depth if self.tree_depth is not None else np.zeros(0, dtype=np.int64),
            inv_mass=self.inv_mass if self.inv_mass is not None else np.zeros(0),
            rng_state=np.frombuffer(json.dumps(self.rng_state, default=int).encode(), dtype=np.uint8),
        )

    @classmethod
    def load(cls, path: str) -> "SamplerResult":
        import json

        z = np.load(path if str(path).endswith(".npz") else str(path) + ".npz")
        rng_state = json.loads(bytes(z["rng_state"]).decode()) if z["rng_state"].size else None
        return cls(
            samples=z["samples"], logp=z["logp"], accept_rate=float(z["accept_rate"]), step_size=float(z["step_size"]),
            n_logp_evals=int(z["n_logp_evals"]), tree_depth=z["tree_depth"] if z["tree_depth"].size else None,
            divergences=int(z["divergences"]), inv_mass=z["inv_mass"] if z["inv_mass"].size else None, rng_state=rng_state,
        )

    def summary(self, names=None) -> Dict[str, Dict[str, float]]:
        names = names or [f"theta[{i}]" for i in range(self.samples.shape[1])]
        out = {}
        for i, n in enumerate(names):
            col = self.samples[:, i]
            out[n] = {"mean": float(col.mean()), "sd": float(col.std(ddof=1)) if len(col) > 1 else 0.0,
                      "median": float(np.median(col)), "ess": float(effective_sample_size(col))}
        return out


def effective_sample_size(x: np.ndarray) -> float:
    """ESS of one chain (or ``[draws, chains]``); see :mod:`.diagnostics`."""
    from .diagnostics import effective_sample_size as _ess

    x = np.asarray(x, dtype=np.float64)
    if x.shape[0] < 4 or np.var(x) == 0:
        return float(x.size)
    return _ess(x)


def find_map(logp_dlogp: LogpDlogp, x0: np.ndarray, *, maxiter: int = 500, tol: float = 1e-10):
    """Maximum a posteriori by L-BFGS-B on ``-logp`` (the reference calls ``pm.find_MAP()``)."""
    import scipy.optimize

    n_evals = 0

    def objective(x):
        nonlocal n_evals
        n_evals += 1
        lp, g = logp_dlogp(np.asarray(x, dtype=np.float64))
        return -float(lp), -np.asarray(g, dtype=np.float64)

    res = scipy.optimize.minimize(objective, np.asarray(x0, dtype=np.float64), jac=True, method="L-BFGS-B",
                                  options={"maxiter": maxiter, "ftol": tol, "gtol": 1e-8})
    return res.x, {"logp": -float(res.fun), "n_evals": n_evals, "converged": bool(res.success), "message": str(res.message)}


class _DualAveraging:
    """Nesterov dual averaging of log(step size) (Hoffman & Gelman 2014, §3.2)."""

    def __init__(self, eps0: float, target: float = 0.8, gamma: float = 0.05, t0: float = 10.0, kappa: float = 0.75):
        self.mu = math.log(10.0 * eps0)
        self.target, self.gamma, self.t0, self.kappa = target, gamma, t0, kappa
        self.h_bar = 0.0
        self.log_eps_bar = 0.0
        self.t = 0

    def update(self, accept: float) -> float:
        self.t += 1
        w = 1.0 / (self.t + self.t0)
        self.h_bar = (1 - w) * self.h_bar + w * (self.target - accept)
        log_eps = self.mu - math.sqrt(self.t) / self.gamma * self.h_bar
        eta = self.t ** (-self.kappa)
        self.log_eps_bar = eta * log_eps + (1 - eta) * self.log_eps_bar
        return math.exp(log_eps)

    def final(self) -> float:
        return math.exp(self.log_eps_bar)


def _find_reasonable_step(logp_dlogp, x, lp, g, rng, inv_mass) -> Tuple[float, int]:
    eps, n = 1.0, 0
    p = rng.normal(size=x.shape) / np.sqrt(inv_mass)

    def trial(e):
        ph = p + 0.5 * e * g
        xn = x + e * inv_mass * ph
        lpn, gn = logp_dlogp(xn)
        pn = ph + 0.5 * e * gn
        return lpn - 0.5 * np.sum(inv_mass * pn * pn) - (lp - 0.5 * np.sum(inv_mass * p * p))

    d = trial(eps)
    n += 1
    direction = 1.0 if (np.isfinite(d) and d > math.log(0.5)) else -1.0
    for _ in range(50):
        eps *= 2.0**direction
        d = trial(eps)
        n += 1
        ok = np.isfinite(d) and d > math.log(0.5)
        if (direction > 0 and not ok) or (direction < 0 and ok):
            break
    return eps, n


def hmc_sample(logp_dlogp: LogpDlogp, x0: np.ndarray, *, draws: int = 500, tune: int = 500, n_leapfrog: int = 16,
               step_size: Optional[float] = None, target_accept: float = 0.8, seed: int = 0,
               adapt_mass: bool = True, resume: Optional[SamplerResult] = None) -> SamplerResult:
    """Static-trajectory HMC with dual-averaging step size and diagonal mass adaptation.
    ``resume=<SamplerResult>`` continues a finished / checkpointed chain without re-tuning (see ``nuts_sample``)."""
    rng = np.random.default_rng(seed)
    if resume is not None:
        x0, tune, step_size = resume.samples[-1], 0, resume.step_size
        if resume.rng_state is not None:
            rng.bit_generator.state = resume.rng_state
    x = np.asarray(x0, dtype=np.float64).copy()
    lp, g = logp_dlogp(x)
    n_evals = 1
    inv_mass = np.ones_like(x)
    if resume is not None and resume.inv_mass is not None:
        inv_mass = np.asarray(resume.inv_mass, dtype=np.float64).copy()
    if step_size is None:
        step_size, k = _find_reasonable_step(logp_dlogp, x, lp, g, rng, inv_mass)
        n_evals += k
    da = _DualAveraging(step_size, target_accept)
    eps = step_size
    samples = np.empty((draws, x.size))
    lps = np.empty(draws)
    acc_sum, warm = 0.0, []
    for it in range(tune + draws):
        p = rng.normal(size=x.shape) / np.sqrt(inv_mass)
        h0 = lp - 0.5 * np.sum(inv_mass * p * p)
        xn, pn, lpn, gn = x, p, lp, g
        ok = True
        jitter = eps * rng.uniform(0.8, 1.2)
        for _ in range(n_leapfrog):
            pn = pn + 0.5 * jitter * gn
            xn = xn + jitter * inv_mass * pn
            lpn, gn = logp_dlogp(xn)
            n_evals += 1
            if not np.isfinite(lpn):
                ok = False
                break
            pn = pn + 0.5 * jitter * gn
        h1 = lpn - 0.5 * np.sum(inv_mass * pn * pn) if ok else -np.inf
        a = min(1.0, math.exp(min(0.0, h1 - h0))) if np.isfinite(h1) else 0.0
        if rng.uniform() < a:
            x, lp, g = xn, lpn, gn
        if it < tune:
            eps = da.update(a)
            warm.append(x.copy())
            if adapt_mass and it == int(0.6 * tune) and len(warm) > 20:
                var = np.var(np.asarray(warm[len(warm) // 3:]), axis=0)
                inv_mass = np.where(var > 1e-12, var, 1.0)
                da = _DualAveraging(eps, target_accept)
            if it == tune - 1:
                eps = da.final()
        else:
            samples[it - tune] = x
            lps[it - tune] = lp
            acc_sum += a
    return SamplerResult(samples, lps, acc_sum / max(1, draws), eps, n_evals, inv_mass=inv_mass,
                         rng_state=rng.bit_generator.state)


def _logaddexp(a: float, b: float) -> float:
    """``log(exp(a) + exp(b))`` for Python floats (``np.logaddexp`` costs ten times as much on scalars)."""
    if a == -inf:
        return b
    if b == -inf:
        return a
    m = a if a > b else b
    return m + math.log1p(math.exp(-abs(a - b)))


def nuts_sample(logp_dlogp: LogpDlogp, x0: Optional[np.ndarray] = None, *, draws: int = 200, tune: int = 500,
                max_depth: int = 8, target_accept: float = 0.8, seed: int = 0, adapt_mass: bool = True,
                resume: Optional[SamplerResult] = None) -> SamplerResult:
    """No-U-Turn sampler (multinomial variant, iterative tree doubling, diagonal mass matrix).

    ``resume=<SamplerResult>`` continues a finished/checkpointed chain: starts at its last draw with
    its adapted step size, mass matrix and random-number state, and skips warm-up.
    """
    rng = np.random.default_rng(seed)
    if resume is not None:
        x0 = resume.samples[-1]
        tune = 0
        if resume.rng_state is not None:
            rng.bit_generator.state = resume.rng_state
    x = np.asarray(x0, dtype=np.float64).copy()
    lp, g = logp_dlogp(x)
    counter = {"n": 1, "div": 0}
    inv_mass = np.ones_like(x)
    if resume is not None:
        eps = resume.step_size
        if resume.inv_mass is not None:
            inv_mass = np.asarray(resume.inv_mass, dtype=np.float64)
    else:
        eps, k = _find_reasonable_step(logp_dlogp, x, lp, g, rng, inv_mass)
        counter["n"] += k
    da = _DualAveraging(eps, target_accept)

    def leapfrog(xq, pq, gq, e):
        ph = pq + 0.5 * e * gq
        xn = xq + e * inv_mass * ph
        lpn, gn = logp_dlogp(xn)
        counter["n"] += 1
        return xn, ph + 0.5 * e * gn, lpn, gn

    def uturn(xm, xp, pm, pp):
        d = xp - xm
        return np.dot(d, inv_mass * pm) < 0 or np.dot(d, inv_mass * pp) < 0

    def build_tree(xq, pq, gq, direction, depth, e, h0):
        """Returns the subtree: edges, proposal, log-weight, stop flag, accept stats."""
        if depth == 0:
            xn, pn, lpn, gn = leapfrog(xq, pq, gq, direction * e)
            # (scalar bookkeeping stays in the math module: this runs once per gradient evaluation)
            h = float(lpn - 0.5 * np.sum(inv_mass * pn * pn)) if isfinite(lpn) else -inf
            finite = isfinite(h)
            diverged = not finite or (h0 - h) > 1000.0
            if diverged:
                counter["div"] += 1
            acc = min(1.0, math.exp(min(0.0, h - h0))) if finite else 0.0
            return (xn, pn, gn, xn, pn, gn, xn, lpn, gn, h - h0 if finite else -inf, diverged, acc, 1)
        (xm, pm, gm, xp, pp, gp, xprop, lpprop, gprop, logw, stop, acc, n) = build_tree(xq, pq, gq, direction, depth - 1, e, h0)
        if not stop:
            if direction < 0:
                (xm, pm, gm, _, _, _, x2, lp2, g2, logw2, stop2, acc2, n2) = build_tree(xm, pm, gm, direction, depth - 1, e, h0)
            else:
                (_, _, _, xp, pp, gp, x2, lp2, g2, logw2, stop2, acc2, n2) = build_tree(xp, pp, gp, direction, depth - 1, e, h0)
            tot = _logaddexp(logw, logw2)
            if isfinite(logw2) and math.log(rng.uniform() + 1e-300) < logw2 - tot:
                xprop, lpprop, gprop = x2, lp2, g2
            logw = tot
            acc += acc2
            n += n2
            stop = stop2 or uturn(xm, xp, pm, pp)
        return (xm, pm, gm, xp, pp, gp, xprop, lpprop, gprop, logw, stop, acc, n)

    samples = np.empty((draws, x.size))
    lps = np.empty(draws)
    depths = np.empty(draws, dtype=np.int64)
    acc_total = 0.0
    warm = []
    for it in range(tune + draws):
        p = rng.normal(size=x.shape) / np.sqrt(inv_mass)
        h0 = lp - 0.5 * np.sum(inv_mass * p * p)
        xm = xp = x
        pm = pp = p
        gm = gp = g
        logw = 0.0
        depth = 0
        acc_sum, n_sum = 0.0, 0
        x_new, lp_new, g_new = x, lp, g
        while depth < max_depth:
            direction = 1 if rng.uniform() < 0.5 else -1
            if direction < 0:
                (xm, pm, gm, _, _, _, x2, lp2, g2, logw2, stop2, a2, n2) = build_tree(xm, pm, gm, -1, depth, eps, h0)
            else:
                (_, _, _, xp, pp, gp, x2, lp2, g2, logw2, stop2, a2, n2) = build_tree(xp, pp, gp, 1, depth, eps, h0)
            acc_sum += a2
            n_sum += n2
            if stop2:
                break
            if isfinite(logw2) and math.log(rng.uniform() + 1e-300) < logw2 - logw:
                x_new, lp_new, g_new = x2, lp2, g2
            logw = _logaddexp(logw, logw2)
            depth += 1
            if uturn(xm, xp, pm, pp):
                break
        x, lp, g = x_new, lp_new, g_new
        a = acc_sum / max(1, n_sum)
        if it < tune:
            eps = da.update(a)
            warm.append(x.copy())
            if adapt_mass and it == int(0.6 * tune) and len(warm) > 20:
                var = np.var(np.asarray(warm[len(warm) // 3:]), axis=0)
                inv_mass = np.where(var > 1e-12, var, 1.0)
                da = _DualAveraging(eps, target_accept)
            if it == tune - 1:
                eps = da.final()
                counter["div"] = 0  # report post-warm-up divergences only
        else:
            samples[it - tune] = x
            lps[it - tune] = lp
            depths[it - tune] = depth
            acc_total += a
    return SamplerResult(samples, lps, acc_total / max(1, draws), eps, counter["n"], depths, counter["div"],
                         inv_mass=inv_mass.copy(), rng_state=rng.bit_generator.state)


def metropolis_sample(
    logp: Callable[[np.ndarray], float],
    x0: Optional[np.ndarray] = None,
    *,
    draws: int = 1000,
    tune: int = 1000,
    seed: int = 0,
    scale: float = 1.0,
    tune_interval: int = 100,
    resume: Optional[SamplerResult] = None,
) -> SamplerResult:
    """Random-walk Metropolis for gradient-free potentials (``LogpOp`` / ``LogpServiceClient``).

    The reference samples its gradient-free black box with ``pm.Metropolis()``
    (``pytensor_federated/test_wrapper_ops.py:68-118``); this is the in-repo counterpart:
    all coordinates are proposed jointly from ``N(0, (scale * s)^2)`` with a per-coordinate ``s``; during
    ``tune`` the global scale is adapted every ``tune_interval`` steps from the acceptance rate of the
    interval (the schedule PyMC uses: shrink below 20 % / 5 % / 0.1 %, grow above 50 % / 75 % / 95 %) and
    ``s`` follows the running standard deviation of the chain.  One ``logp`` call per step.
    ``resume`` continues a finished run with its proposal and random state (no further tuning).
    """
    if resume is not None:
        x = np.array(resume.samples[-1], dtype=np.float64)
        rng = np.random.default_rng()
        if resume.rng_state is not None:
            rng.bit_generator.state = resume.rng_state
        step = float(resume.step_size)
        spread = np.ones_like(x) if resume.inv_mass is None else np.sqrt(np.asarray(resume.inv_mass, dtype=np.float64))
        tune = 0
    else:
        if x0 is None:
            raise ValueError("x0 is required unless resuming")
        x = np.atleast_1d(np.asarray(x0, dtype=np.float64)).copy()
        rng = np.random.default_rng(seed)
        step = float(scale)
        spread = np.ones_like(x)
    cur = float(logp(x))
    if not np.isfinite(cur):
        raise ValueError("Metropolis needs a finite log-probability at the starting point")
    n_evals = 1
    samples = np.empty((draws, x.size))
    logps = np.empty(draws)
    accepted_interval = 0
    accepted_draws = 0
    # Welford running moments of the tuning phase -> per-coordinate proposal spread
    n_seen, mean, m2 = 0, np.zeros_like(x), np.zeros_like(x)
    for it in range(tune + draws):
        proposal = x + step * spread * rng.normal(size=x.size)
        new = float(logp(proposal))
        n_evals += 1
        accept = np.isfinite(new) and np.log(rng.uniform()) < new - cur
        if accept:
            x, cur = proposal, new
        if it < tune:
            accepted_interval += int(accept)
            n_seen += 1
            delta = x - mean
            mean += delta / n_seen
            m2 += delta * (x - mean)
            if (it + 1) % tune_interval == 0:
                rate = accepted_interval / tune_interval
                for bound, factor in ((0.001, 0.1), (0.05, 0.5), (0.2, 0.9)):
                    if rate < bound:
                        step *= factor
                        break
                else:
                    for bound, factor in ((0.95, 10.0), (0.75, 2.0), (0.5, 1.1)):
                        if rate > bound:
                            step *= factor
                            break
                accepted_interval = 0
                if n_seen >= 2 * tune_interval and x.size > 1:
                    sd = np.sqrt(m2 / (n_seen - 1))
                    if np.all(sd > 0):
                        spread = sd / np.exp(np.mean(np.log(sd)))   # shape only; `step` keeps the overall size
        else:
            samples[it - tune] = x
            logps[it - tune] = cur
            accepted_draws += int(accept)
    return SamplerResult(
        samples=samples, logp=logps, accept_rate=accepted_draws / max(draws, 1), step_size=step, n_logp_evals=n_evals,
        inv_mass=spread**2, rng_state=rng.bit_generator.state,
    )
