"""User-defined likelihoods on the fused path.

The reference's premise is that a node serves an *arbitrary* function
(``README.md:26-35``).  Arbitrary Python still goes through
``ArraysToArraysService`` / ``register_local_node``; but any GLM-shaped model
``eta = intercept[group] + X beta`` with a custom per-observation log-likelihood can run inside the
fused broadcast -> compute -> reduce kernel: the likelihood is a snippet of CUDA C that assigns

    ll  — log-likelihood of one observation,   r  — d ll / d eta

from ``y`` and ``eta`` (floats).  It is compiled for sm_90a into its own shared object (nvcc, cached
by content hash under ``csrc/build/custom``) and plugged into the general-shape kernel
(``csrc/glm_generic.cu``).  Example — Student-t regression with 4 degrees of freedom::

    family = CustomFamily(
        "const float d = y - eta; ll = -2.5f * log1pf(d * d * 0.25f); r = 5.f * d / (4.f + d * d);",
        torch_fn=lambda y, eta: (-2.5 * torch.log1p((y - eta) ** 2 / 4), 5 * (y - eta) / (4 + (y - eta) ** 2)),
    )
    model = GlmShards(Xs, ys, family=family)
"""
from __future__ import annotations

import ctypes as C
import hashlib
from pathlib import Path
from typing import Callable, Optional

_PKG = Path(__file__).resolve().parent.parent
_CSRC = _PKG / "csrc"


class CustomFamily:
    """A likelihood given as CUDA C (``ll`` and ``r`` from ``y`` and ``eta``) plus an optional
    PyTorch oracle ``torch_fn(y, eta) -> (ll, r)`` used by the eager reference implementation."""

    code_id = 99

    def __init__(self, cuda_code: str, torch_fn: Optional[Callable] = None, name: str = "custom") -> None:
        self.cuda_code = " ".join(cuda_code.split())
        self.torch_fn = torch_fn
        self.name = name
        self._lib = None

    def digest(self) -> str:
        h = hashlib.sha256(self.cuda_code.encode())
        for f in ("glm_generic.cu", "fed_comm.cuh", "models.h"):
            h.update((_CSRC / f).read_bytes())
        return h.hexdigest()[:16]

    def compile(self) -> C.CDLL:
        """Builds (or loads from the cache) the shared object with this likelihood."""
        if self._lib is not None:
            return self._lib
        from .. import build as native_build

        so = native_build.build_snippet_library(
            "glm_generic.cu", "B200FED_CUSTOM_LINK", self.cuda_code, ["-DB200FED_GENERIC_ENTRY=b200_launch_glm_custom"],
            f"libb200fed_custom_{self.digest()}", "custom likelihood")
        self._lib = C.CDLL(str(so))
        return self._lib

    def launcher_address(self) -> int:
        lib = self.compile()
        return C.cast(lib.b200_launch_glm_custom, C.c_void_p).value


__all__ = ["CustomFamily"]
