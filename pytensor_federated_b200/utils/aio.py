"""Event-loop and selection helpers.

Reference behaviour: ``pytensor_federated/utils.py:13-34`` (argmin
that ignores ``None``) and ``:37-61`` (a loop one can always ``run_until_complete``
on, re-entrantly patched with ``nest_asyncio`` when already running).
"""
from __future__ import annotations

import asyncio
import logging
import math
import warnings
from typing import Callable, Iterable, Optional, TypeVar

T = TypeVar("T")
_log = logging.getLogger(__name__)


def argmin_none_or_func(
    items: Iterable[Optional[T]],
    func: Callable[[T], float],
) -> Optional[int]:
    """Index of the smallest ``func(item)`` among the non-``None`` items.

    Returns ``None`` if there are no items or all of them are ``None``.  Ties go to
    the first occurrence (callers shuffle beforehand to randomise tie-breaks).
    """
    best_index: Optional[int] = None
    best_value = math.inf
    for index, item in enumerate(items):
        if item is None:
            continue
        value = func(item)
        if best_index is None or value < best_value:
            best_index = index
            best_value = value
    return best_index


def get_useful_event_loop() -> asyncio.AbstractEventLoop:
    """Like ``asyncio.get_event_loop()`` but usable from inside a running loop.

    * Called from a coroutine: the running loop is patched (once) with
      ``nest_asyncio`` so that ``run_until_complete`` may be nested.
    * Called from plain code: the thread's current loop, or a fresh one that is
      installed as the current loop (Python ≥ 3.12 no longer creates it implicitly).
    """
    loop = asyncio._get_running_loop()
    if loop is not None:
        if not hasattr(loop, "_nest_patched"):
            import nest_asyncio

            _log.debug("Event loop is already running. Patching with nest_asyncio.")
            nest_asyncio.apply(loop)
        return loop
    with warnings.catch_warnings():
        # 3.12 warns (and 3.14 raises) when there is no current loop yet.
        warnings.simplefilter("ignore", DeprecationWarning)
        try:
            loop = asyncio.get_event_loop_policy().get_event_loop()
        except RuntimeError:
            loop = None
    if loop is None or loop.is_closed():
        loop = asyncio.new_event_loop()
        asyncio.set_event_loop(loop)
    return loop
