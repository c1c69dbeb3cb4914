"""Generic helpers with only external dependencies.

Reference: ``pytensor_federated/utils.py:13-61``.
"""
from .aio import argmin_none_or_func, get_useful_event_loop

__all__ = ["argmin_none_or_func", "get_useful_event_loop"]
