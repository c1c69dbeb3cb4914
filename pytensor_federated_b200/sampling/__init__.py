"""Gradient-based inference drivers for federated log-potentials.

The reference delegates sampling to PyMC (``demo_model.py:38-44``:
``pm.find_MAP()`` + ``pm.sample()``/NUTS).  PyMC is not available in the offline image, so this
package ships the drivers that exercise the hot path — MAP by L-BFGS, HMC and NUTS with
dual-averaging step-size adaptation, and random-walk Metropolis for gradient-free potentials (``LogpOp``) — on top of any ``logp_dlogp(theta) -> (float, ndarray)``
callable, plus a minimal model builder over the graph IR.  With PyMC installed the Ops plug into
``pm.Potential`` exactly as the reference's do.
"""
from .batched import BatchedResult, glm_batch_fn, hmc_sample_batched
from .diagnostics import effective_sample_size, split_rhat, summarize
from .laplace import glm_hessian, glm_hvp_fn, laplace
from .mcmc import SamplerResult, find_map, hmc_sample, metropolis_sample, nuts_sample
from .model import Model
from .parallel import sample_parallel

__all__ = ["Model", "SamplerResult", "find_map", "hmc_sample", "nuts_sample", "metropolis_sample", "BatchedResult", "hmc_sample_batched", "glm_batch_fn",
           "glm_hvp_fn", "glm_hessian", "laplace", "split_rhat", "effective_sample_size", "summarize", "sample_parallel"]
