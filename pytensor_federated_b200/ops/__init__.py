"""Native operators: ctypes access to the sm_90a kernels and the host runtime."""
from . import native

__all__ = ["native"]
