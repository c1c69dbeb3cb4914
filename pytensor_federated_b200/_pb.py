"""Minimal proto3 wire-format primitives (no protoc, no generated code).

The reference generates its message classes with ``protoc`` + the betterproto
plugin (``protobufs/generate.py:15-27``).  Neither tool exists in
this image, and the schema is five tiny messages, so the wire format is written
out by hand here: varints, length-delimited fields and fixed32 floats.  The byte
layout is the proto3 standard one, so these messages interoperate with a stock
reference server/client (tags listed in SURVEY.md §2.1).
"""
from __future__ import annotations

import struct
from typing import Iterator, List, Tuple

WIRE_VARINT = 0
WIRE_FIXED64 = 1
WIRE_LEN = 2
WIRE_FIXED32 = 5

_U64 = (1 << 64) - 1


def encode_varint(value: int) -> bytes:
    """Unsigned LEB128; negative ints are sent as 64-bit two's complement."""
    value &= _U64
    out = bytearray()
    while value > 0x7F:
        out.append((value & 0x7F) | 0x80)
        value >>= 7
    out.append(value)
    return bytes(out)


def decode_varint(buf, pos: int) -> Tuple[int, int]:
    result = 0
    shift = 0
    while True:
        if pos >= len(buf):
            raise ValueError("Truncated varint.")
        b = buf[pos]
        pos += 1
        result |= (b & 0x7F) << shift
        if not b & 0x80:
            break
        shift += 7
        if shift > 63:
            raise ValueError("Varint is longer than 10 bytes.")
    return result & _U64, pos


def to_signed64(value: int) -> int:
    return value - (1 << 64) if value & (1 << 63) else value


def to_signed32(value: int) -> int:
    value &= 0xFFFFFFFF
    return value - (1 << 32) if value & (1 << 31) else value


def tag(field: int, wire_type: int) -> bytes:
    return encode_varint((field << 3) | wire_type)


def enc_len_field(field: int, payload: bytes) -> bytes:
    return tag(field, WIRE_LEN) + encode_varint(len(payload)) + payload


def enc_packed_int64(field: int, values) -> bytes:
    if len(values) == 0:
        return b""
    payload = b"".join(encode_varint(int(v)) for v in values)
    return enc_len_field(field, payload)


def enc_varint_field(field: int, value: int) -> bytes:
    if value == 0:
        return b""
    return tag(field, WIRE_VARINT) + encode_varint(value)


def enc_float_field(field: int, value: float) -> bytes:
    if value == 0.0:
        return b""
    return tag(field, WIRE_FIXED32) + struct.pack("<f", value)


def iter_fields(buf) -> Iterator[Tuple[int, int, object]]:
    """Yields ``(field_number, wire_type, value)``; LEN values are memoryviews."""
    view = memoryview(buf)
    pos = 0
    end = len(view)
    while pos < end:
        key, pos = decode_varint(view, pos)
        field, wt = key >> 3, key & 7
        if wt == WIRE_VARINT:
            value, pos = decode_varint(view, pos)
        elif wt == WIRE_LEN:
            n, pos = decode_varint(view, pos)
            if pos + n > end:
                raise ValueError("Truncated length-delimited field.")
            value = view[pos : pos + n]
            pos += n
        elif wt == WIRE_FIXED32:
            if pos + 4 > end:
                raise ValueError("Truncated fixed32 field.")
            value = bytes(view[pos : pos + 4])
            pos += 4
        elif wt == WIRE_FIXED64:
            if pos + 8 > end:
                raise ValueError("Truncated fixed64 field.")
            value = bytes(view[pos : pos + 8])
            pos += 8
        else:
            raise ValueError(f"Unsupported wire type {wt}.")
        yield field, wt, value


def dec_packed_int64(value, wt: int, into: List[int]) -> None:
    """Accepts both packed (LEN) and unpacked (VARINT) repeated int64."""
    if wt == WIRE_VARINT:
        into.append(to_signed64(value))
        return
    pos = 0
    n = len(value)
    while pos < n:
        v, pos = decode_varint(value, pos)
        into.append(to_signed64(v))
