"""``npproto.ndarray`` message (wire-compatible with the reference).

Schema: ``protobufs/npproto/ndarray.proto:7-12`` —
``bytes data=1; string dtype=2; repeated int64 shape=3; repeated int64 strides=4``.
The reference's class is betterproto-generated
(``pytensor_federated/npproto/__init__.py:12-22``); this one is
hand-written on top of :mod:`pytensor_federated_b200._pb` and keeps the two
methods the reference's users touch: ``bytes(msg)`` and ``Msg().parse(data)``.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

from .. import _pb


class Ndarray:
    """Represents a NumPy array of arbitrary shape or dtype."""

    __slots__ = ("data", "dtype", "shape", "strides")

    def __init__(
        self,
        data: bytes = b"",
        dtype: str = "",
        shape: Optional[Sequence[int]] = None,
        strides: Optional[Sequence[int]] = None,
    ) -> None:
        self.data = data
        self.dtype = dtype
        self.shape: List[int] = list(shape) if shape is not None else []
        self.strides: List[int] = list(strides) if strides is not None else []

    # -- wire format -------------------------------------------------------
    def __bytes__(self) -> bytes:
        parts = []
        if len(self.data):
            parts.append(_pb.enc_len_field(1, bytes(self.data)))
        if self.dtype:
            parts.append(_pb.enc_len_field(2, self.dtype.encode("utf-8")))
        parts.append(_pb.enc_packed_int64(3, self.shape))
        parts.append(_pb.enc_packed_int64(4, self.strides))
        return b"".join(parts)

    SerializeToString = __bytes__

    def parse(self, data) -> "Ndarray":
        self.data = b""
        self.dtype = ""
        self.shape = []
        self.strides = []
        for field, wt, value in _pb.iter_fields(data):
            if field == 1 and wt == _pb.WIRE_LEN:
                self.data = bytes(value)
            elif field == 2 and wt == _pb.WIRE_LEN:
                self.dtype = bytes(value).decode("utf-8")
            elif field == 3:
                _pb.dec_packed_int64(value, wt, self.shape)
            elif field == 4:
                _pb.dec_packed_int64(value, wt, self.strides)
            # unknown fields are skipped (proto3 forward compatibility)
        return self

    @classmethod
    def FromString(cls, data) -> "Ndarray":
        return cls().parse(data)

    # -- conveniences ------------------------------------------------------
    def __eq__(self, other) -> bool:
        if not isinstance(other, Ndarray):
            return NotImplemented
        return (
            bytes(self.data) == bytes(other.data)
            and self.dtype == other.dtype
            and list(self.shape) == list(other.shape)
            and list(self.strides) == list(other.strides)
        )

    def __repr__(self) -> str:
        return (
            f"Ndarray(dtype={self.dtype!r}, shape={self.shape}, strides={self.strides}, "
            f"data=<{len(self.data)} bytes>)"
        )


# The proto message is spelled lower-case in the IDL.
ndarray = Ndarray

__all__ = ["Ndarray", "ndarray"]
