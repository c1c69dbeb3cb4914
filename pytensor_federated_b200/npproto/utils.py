"""Converters between ``numpy.ndarray``/``torch.Tensor`` and :class:`Ndarray`.

Reference: ``pytensor_federated/npproto/utils.py:9-24``.

Differences on purpose (SURVEY.md §2.1):

* The reference ships ``bytes(arr.data)`` (logical C order) together with the
  *original* strides, which silently corrupts F-ordered / transposed arrays and
  raises on sliced ones.  Here arrays are canonicalised to C order on encode and
  the strides that are sent describe the bytes that are sent.  Messages produced
  by a reference peer (C-contiguous arrays) decode identically.
* ``dtype=object`` only "works" in the reference inside one process (raw
  ``PyObject*`` are copied).  Here object arrays are pickled into ``data`` so they
  survive a process boundary; the dtype string stays ``"object"``.  **Decoding**
  them means unpickling bytes that came from a peer, so it is refused unless the
  receiving process opts in with ``B200FED_ALLOW_PICKLE=1`` (or
  ``allow_pickle(True)``) — only do that between parties that trust each other.
"""
from __future__ import annotations

import pickle

import numpy

from . import Ndarray

_OBJECT_MAGIC = b"\x93B200OBJ"
_allow_pickle = None  # None: ask the environment


def allow_pickle(flag) -> None:
    """Lets this process decode object-dtype arrays (``True``), forbids it (``False``) or defers to the
    ``B200FED_ALLOW_PICKLE`` environment variable (``None``, the default)."""
    global _allow_pickle
    _allow_pickle = flag


def _pickle_allowed() -> bool:
    if _allow_pickle is not None:
        return bool(_allow_pickle)
    import os

    return os.environ.get("B200FED_ALLOW_PICKLE", "") not in ("", "0")


def ndarray_from_numpy(arr: numpy.ndarray) -> Ndarray:
    arr = numpy.asarray(arr)
    if arr.dtype.hasobject:
        payload = _OBJECT_MAGIC + pickle.dumps(arr.tolist(), protocol=pickle.HIGHEST_PROTOCOL)
        strides = list(numpy.empty(arr.shape, dtype=object).strides)
        return Ndarray(data=payload, dtype=str(arr.dtype), shape=list(arr.shape), strides=strides)
    if not arr.flags.c_contiguous:
        # numpy.ascontiguousarray would promote 0-d to 1-d; copy(order="C") keeps ndim.
        arr = arr.copy(order="C")
    return Ndarray(
        shape=list(arr.shape),
        dtype=str(arr.dtype),
        data=arr.tobytes() if arr.ndim == 0 else bytes(arr.data),
        strides=list(arr.strides),
    )


def ndarray_to_numpy(nda: Ndarray) -> numpy.ndarray:
    dtype = numpy.dtype(nda.dtype)
    shape = tuple(nda.shape)
    if dtype.hasobject:
        data = bytes(nda.data)
        if not data.startswith(_OBJECT_MAGIC):
            raise TypeError(
                "Received an object-dtype array that was not encoded by this package. "
                "Object arrays from the reference implementation carry process-local "
                "pointers and cannot be decoded."
            )
        if not _pickle_allowed():
            raise TypeError(
                "Refusing to unpickle an object-dtype array received from a peer. Set B200FED_ALLOW_PICKLE=1 "
                "(or call npproto.utils.allow_pickle(True)) if every party on this federation is trusted."
            )
        items = pickle.loads(data[len(_OBJECT_MAGIC) :])
        result = numpy.empty(shape, dtype=object)
        if shape == ():
            result[()] = items
        else:
            # assign element-wise over the first axis so ragged rows stay Python objects
            _fill_object(result, items)
        return result
    strides = tuple(nda.strides) if len(nda.strides) == len(shape) else None
    return numpy.ndarray(buffer=nda.data, shape=shape, dtype=dtype, strides=strides)


def _fill_object(target: numpy.ndarray, items) -> None:
    if target.ndim == 1:
        for i, item in enumerate(items):
            target[i] = item
        return
    for i, item in enumerate(items):
        _fill_object(target[i], item)


def ndarray_from_tensor(tensor) -> Ndarray:
    """Encodes a ``torch.Tensor`` (any device) — convenience for GPU nodes."""
    import torch

    t = tensor.detach()
    if t.dtype == torch.bfloat16:
        t = t.to(torch.float32)
    return ndarray_from_numpy(t.cpu().numpy())


def ndarray_to_tensor(nda: Ndarray, device=None):
    """Decodes into a ``torch.Tensor`` (copies; the wire buffer is read-only)."""
    import torch

    arr = numpy.array(ndarray_to_numpy(nda))
    t = torch.from_numpy(arr)
    return t.to(device) if device is not None else t
