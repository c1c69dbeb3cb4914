"""Chains in separate processes — the reference's replica parallelism.

With PyMC the reference runs one chain per process (``pm.sample(cores=4)``); every process gets its own
connection (``thread_pid_id`` keyed connection cache) and ``hosts_and_ports`` places it on the replica
with the fewest open streams (``pytensor_federated/service.py:239-275``,
``test_wrapper_ops.py:305-317``).  :func:`sample_parallel` is that driver for the in-repo samplers: the
model is *built inside each worker* by a picklable factory, so clients connect (and balance) there.
"""
from __future__ import annotations

import multiprocessing
from typing import Callable, List, Optional

import numpy as np

from .mcmc import LogpDlogp, SamplerResult, hmc_sample, metropolis_sample, nuts_sample

__all__ = ["sample_parallel"]

_SAMPLERS = {"nuts": nuts_sample, "hmc": hmc_sample, "metropolis": metropolis_sample}


def _run_chain(job) -> SamplerResult:
    factory, x0, sampler, seed, kwargs = job
    logp_dlogp = factory()
    return _SAMPLERS[sampler](logp_dlogp, np.asarray(x0, dtype=np.float64), seed=seed, **kwargs)


def sample_parallel(
    make_logp_dlogp: Callable[[], LogpDlogp],
    x0: np.ndarray,
    *,
    chains: int = 4,
    cores: Optional[int] = None,
    sampler: str = "nuts",
    seed: int = 0,
    mp_start_method: str = "spawn",
    **kwargs,
) -> List[SamplerResult]:
    """Runs ``chains`` chains on ``cores`` worker processes; chain ``c`` uses seed ``seed + c``.

    ``sampler="metropolis"`` is the gradient-free driver: the factory then returns ``logp(theta) -> float``.
    ``make_logp_dlogp`` is called once per chain *in the worker* and must be picklable (a module-level
    function or a ``functools.partial`` of one).  ``spawn`` is the default start method: a forked child
    inherits neither CUDA contexts nor gRPC channels safely.  Remaining keyword arguments go to the
    sampler (``draws``, ``tune``, ...).  ``cores=1`` runs in-process (handy for debugging).
    """
    if sampler not in _SAMPLERS:
        raise ValueError(f"unknown sampler {sampler!r}; choose from {sorted(_SAMPLERS)}")
    if chains < 1:
        raise ValueError("need at least one chain")
    jobs = [(make_logp_dlogp, x0, sampler, seed + c, kwargs) for c in range(chains)]
    cores = min(chains, cores or chains)
    if cores == 1:
        return [_run_chain(job) for job in jobs]
    ctx = multiprocessing.get_context(mp_start_method)
    with ctx.Pool(cores) as pool:
        return pool.map(_run_chain, jobs, chunksize=1)
