"""Type and signature definitions (no runtime behaviour).

Reference: ``pytensor_federated/signatures.py:8-33``.
"""
from typing import Callable, Sequence, Tuple

import numpy as np

ComputeFunc = Callable[..., Sequence[np.ndarray]]
"""``f(*ndarrays) -> sequence of ndarrays`` — the most generic federated function."""

LogpFunc = Callable[..., np.ndarray]
"""``f(*ndarrays) -> scalar ndarray`` — a log-probability without gradients."""

LogpGradFunc = Callable[..., Tuple[np.ndarray, Sequence[np.ndarray]]]
"""``f(*ndarrays) -> (scalar ndarray, [d logp / d input_i ...])``."""

__all__ = ["ComputeFunc", "LogpFunc", "LogpGradFunc"]
