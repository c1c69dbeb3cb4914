"""Runtime-built protobuf descriptors of the wire schema.

The reference generates Python classes from ``protobufs/*.proto`` with ``protoc``
(``protobufs/generate.py:15-27``).  ``protoc`` is not part of the
offline image, so the same schema is assembled as a ``FileDescriptorProto`` here.
It serves two purposes: (1) an independent oracle for the hand-written codec in
:mod:`pytensor_federated_b200._pb` (see ``tests/test_npproto.py``) and (2)
stock ``google.protobuf`` message classes for users who want them, e.g. to talk
to a node from ``grpcio`` code generated elsewhere.
"""
from __future__ import annotations

from typing import Dict


def build_file_descriptors():
    from google.protobuf import descriptor_pb2 as d

    F = d.FieldDescriptorProto

    nd = d.FileDescriptorProto(name="npproto/ndarray.proto", package="npproto", syntax="proto3")
    m = nd.message_type.add(name="ndarray")
    m.field.add(name="data", number=1, type=F.TYPE_BYTES, label=F.LABEL_OPTIONAL)
    m.field.add(name="dtype", number=2, type=F.TYPE_STRING, label=F.LABEL_OPTIONAL)
    m.field.add(name="shape", number=3, type=F.TYPE_INT64, label=F.LABEL_REPEATED)
    m.field.add(name="strides", number=4, type=F.TYPE_INT64, label=F.LABEL_REPEATED)

    sv = d.FileDescriptorProto(name="service.proto", syntax="proto3")
    sv.dependency.append("npproto/ndarray.proto")
    for name in ("InputArrays", "OutputArrays"):
        m = sv.message_type.add(name=name)
        m.field.add(
            name="items",
            number=1,
            type=F.TYPE_MESSAGE,
            type_name=".npproto.ndarray",
            label=F.LABEL_REPEATED,
        )
        m.field.add(name="uuid", number=2, type=F.TYPE_STRING, label=F.LABEL_OPTIONAL)
    sv.message_type.add(name="GetLoadParams")
    m = sv.message_type.add(name="GetLoadResult")
    m.field.add(name="n_clients", number=1, type=F.TYPE_INT32, label=F.LABEL_OPTIONAL)
    m.field.add(name="percent_cpu", number=2, type=F.TYPE_FLOAT, label=F.LABEL_OPTIONAL)
    m.field.add(name="percent_ram", number=3, type=F.TYPE_FLOAT, label=F.LABEL_OPTIONAL)
    svc = sv.service.add(name="ArraysToArraysService")
    svc.method.add(name="Evaluate", input_type=".InputArrays", output_type=".OutputArrays")
    svc.method.add(
        name="EvaluateStream",
        input_type=".InputArrays",
        output_type=".OutputArrays",
        client_streaming=True,
        server_streaming=True,
    )
    svc.method.add(name="GetLoad", input_type=".GetLoadParams", output_type=".GetLoadResult")
    return nd, sv


def build_message_classes() -> Dict[str, type]:
    """``{"npproto.ndarray": cls, "InputArrays": cls, ...}`` from a private pool."""
    from google.protobuf import descriptor_pool, message_factory

    pool = descriptor_pool.DescriptorPool()
    for fd in build_file_descriptors():
        pool.Add(fd)
    names = ["npproto.ndarray", "InputArrays", "OutputArrays", "GetLoadParams", "GetLoadResult"]
    return {n: message_factory.GetMessageClass(pool.FindMessageTypeByName(n)) for n in names}
