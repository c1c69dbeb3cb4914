"""Service messages, async client stub and server base of ``ArraysToArraysService``.

Schema: ``protobufs/service.proto:6-41``.  The reference's module
of the same role is betterproto/grpclib-generated
(``pytensor_federated/rpc.py:31-187``).  This one is hand-written
against ``grpc.aio`` (the gRPC stack that ships in the offline image) and is used
for the *compatibility* data path only (off-box clients, arbitrary Python
compute functions).  On-box GPU nodes are reached through the fused NVLink path
in :mod:`pytensor_federated_b200.parallel` and never touch this module.

Routes are un-packaged, exactly like the reference: ``/ArraysToArraysService/<Rpc>``.
"""
from __future__ import annotations

import struct
from typing import AsyncIterator, Dict, List, Optional, Sequence

from . import _pb
from .npproto import Ndarray

SERVICE_NAME = "ArraysToArraysService"
ROUTE_EVALUATE = f"/{SERVICE_NAME}/Evaluate"
ROUTE_EVALUATE_STREAM = f"/{SERVICE_NAME}/EvaluateStream"
ROUTE_GET_LOAD = f"/{SERVICE_NAME}/GetLoad"

# gRPC defaults to 4 MiB messages; design matrices are not sent over this path,
# but parameter/gradient vectors of large models can exceed that.
MAX_MESSAGE_BYTES = 1 << 30
CHANNEL_OPTIONS = (
    ("grpc.max_send_message_length", MAX_MESSAGE_BYTES),
    ("grpc.max_receive_message_length", MAX_MESSAGE_BYTES),
)


def encode_arrays_message(arrays, uuid: str = "") -> bytes:
    """One Input/OutputArrays message from NumPy arrays — native codec when built, else Python."""
    import numpy as np

    from .npproto import native_codec
    from .npproto.utils import ndarray_from_numpy

    arrs = [np.asarray(a) for a in arrays]
    if native_codec.available() and not any(a.dtype.hasobject for a in arrs):
        return native_codec.encode_arrays(arrs, uuid)
    parts = [_pb.enc_len_field(1, bytes(ndarray_from_numpy(a))) for a in arrs]
    if uuid:
        parts.append(_pb.enc_len_field(2, uuid.encode("utf-8")))
    return b"".join(parts)


class _ArraysMessage:
    """Shared implementation of ``InputArrays`` and ``OutputArrays``.

    Public surface as in the reference (``items``, ``uuid``, ``bytes(msg)``, ``parse``).  Internally a
    message can also carry its wire bytes and/or the decoded NumPy arrays, so that the hot path
    (``from_arrays`` -> wire -> ``parse`` -> ``arrays``) goes through the native codec
    (``csrc/codec.cu``) without ever materialising per-item Python message objects.
    """

    __slots__ = ("_items", "uuid", "_payload", "_arrays")

    def __init__(self, items: Optional[Sequence[Ndarray]] = None, uuid: str = "") -> None:
        self._items: Optional[List[Ndarray]] = list(items) if items is not None else []
        self.uuid = uuid
        self._payload: Optional[bytes] = None
        self._arrays = None

    @classmethod
    def from_arrays(cls, arrays, uuid: str = ""):
        """Builds the message straight from NumPy arrays (encodes once, natively when possible)."""
        msg = cls.__new__(cls)
        msg._items = None
        msg.uuid = uuid
        msg._payload = encode_arrays_message(arrays, uuid)
        msg._arrays = None
        return msg

    @property
    def items(self) -> List[Ndarray]:
        if self._items is None:
            self._items = []
            for field, wt, value in _pb.iter_fields(self._payload):
                if field == 1 and wt == _pb.WIRE_LEN:
                    self._items.append(Ndarray().parse(value))
            self._payload = None  # the item list may be mutated from now on
        return self._items

    @items.setter
    def items(self, value) -> None:
        self._items = list(value)
        self._payload = None
        self._arrays = None

    @property
    def arrays(self):
        """The items as NumPy arrays (zero-copy, read-only views over the wire bytes)."""
        if self._arrays is None:
            from .npproto.utils import ndarray_to_numpy

            self._arrays = [ndarray_to_numpy(i) for i in self.items]
        return self._arrays

    def __bytes__(self) -> bytes:
        if self._payload is not None:
            return self._payload
        parts = [_pb.enc_len_field(1, bytes(item)) for item in self._items]
        if self.uuid:
            parts.append(_pb.enc_len_field(2, self.uuid.encode("utf-8")))
        return b"".join(parts)

    SerializeToString = __bytes__

    def parse(self, data):
        from .npproto import native_codec

        self._payload = bytes(data)
        self._items = None
        self._arrays = None
        self.uuid = ""
        if native_codec.available():
            try:
                self._arrays, self.uuid = native_codec.decode_arrays(self._payload)
                return self
            except TypeError:  # object arrays: Python path below
                self._arrays = None
        for field, wt, value in _pb.iter_fields(self._payload):
            if field == 2 and wt == _pb.WIRE_LEN:
                self.uuid = bytes(value).decode("utf-8")
            elif field == 1 and wt == _pb.WIRE_LEN:
                pass  # items are parsed lazily
            # other fields: skipped (validated by iter_fields)
        return self

    @classmethod
    def FromString(cls, data):
        return cls().parse(data)

    def __eq__(self, other) -> bool:
        if type(other) is not type(self):
            return NotImplemented
        return self.uuid == other.uuid and self.items == other.items

    def __repr__(self) -> str:
        return f"{type(self).__name__}(items={self.items!r}, uuid={self.uuid!r})"


class InputArrays(_ArraysMessage):
    """Input type message of the ArraysToArraysService."""

    __slots__ = ()


class OutputArrays(_ArraysMessage):
    """Output type message of the ArraysToArraysService."""

    __slots__ = ()


class GetLoadParams:
    """Input message for a GetLoad query (empty)."""

    __slots__ = ()

    def __bytes__(self) -> bytes:
        return b""

    SerializeToString = __bytes__

    def parse(self, data):
        return self

    @classmethod
    def FromString(cls, data):
        return cls()

    def __eq__(self, other) -> bool:
        return isinstance(other, GetLoadParams)

    def __repr__(self) -> str:
        return "GetLoadParams()"


class GetLoadResult:
    """Result message of a GetLoad query."""

    __slots__ = ("n_clients", "percent_cpu", "percent_ram", "gpu")

    def __init__(self, n_clients: int = 0, percent_cpu: float = 0.0, percent_ram: float = 0.0):
        self.n_clients = n_clients
        self.percent_cpu = percent_cpu
        self.percent_ram = percent_ram
        self.gpu = None  # optional (SM %, HBM %) — local only, never on the wire

    def __bytes__(self) -> bytes:
        return (
            _pb.enc_varint_field(1, int(self.n_clients))
            + _pb.enc_float_field(2, float(self.percent_cpu))
            + _pb.enc_float_field(3, float(self.percent_ram))
        )

    SerializeToString = __bytes__

    def parse(self, data):
        self.n_clients = 0
        self.percent_cpu = 0.0
        self.percent_ram = 0.0
        for field, wt, value in _pb.iter_fields(data):
            if field == 1 and wt == _pb.WIRE_VARINT:
                self.n_clients = _pb.to_signed32(value)
            elif field == 2 and wt == _pb.WIRE_FIXED32:
                (self.percent_cpu,) = struct.unpack("<f", value)
            elif field == 3 and wt == _pb.WIRE_FIXED32:
                (self.percent_ram,) = struct.unpack("<f", value)
        return self

    @classmethod
    def FromString(cls, data):
        return cls().parse(data)

    def __eq__(self, other) -> bool:
        if not isinstance(other, GetLoadResult):
            return NotImplemented
        return (self.n_clients, self.percent_cpu, self.percent_ram) == (
            other.n_clients,
            other.percent_cpu,
            other.percent_ram,
        )

    def __repr__(self) -> str:
        return (
            f"GetLoadResult(n_clients={self.n_clients}, percent_cpu={self.percent_cpu}, "
            f"percent_ram={self.percent_ram})"
        )


def _serialize(message) -> bytes:
    return bytes(message)


class ArraysToArraysServiceStub:
    """Async client stub over a ``grpc.aio`` channel.

    Counterpart of ``pytensor_federated/rpc.py:74-126``.
    """

    def __init__(self, channel) -> None:
        self.channel = channel
        self._evaluate = channel.unary_unary(
            ROUTE_EVALUATE,
            request_serializer=_serialize,
            response_deserializer=OutputArrays.FromString,
        )
        self._evaluate_stream = channel.stream_stream(
            ROUTE_EVALUATE_STREAM,
            request_serializer=_serialize,
            response_deserializer=OutputArrays.FromString,
        )
        self._get_load = channel.unary_unary(
            ROUTE_GET_LOAD,
            request_serializer=_serialize,
            response_deserializer=GetLoadResult.FromString,
        )

    async def evaluate(self, input_arrays: InputArrays, *, timeout: Optional[float] = None):
        return await self._evaluate(input_arrays, timeout=timeout)

    def open_evaluate_stream(self, *, timeout: Optional[float] = None):
        """Opens the long-lived bidirectional stream and returns the call object
        (``await call.write(msg)`` / ``await call.read()``)."""
        return self._evaluate_stream(timeout=timeout)

    async def evaluate_stream(
        self, input_arrays_iterator, *, timeout: Optional[float] = None
    ) -> AsyncIterator[OutputArrays]:
        call = self._evaluate_stream(input_arrays_iterator, timeout=timeout)
        async for response in call:
            yield response

    async def get_load(
        self, get_load_params: Optional[GetLoadParams] = None, *, timeout: Optional[float] = None
    ) -> GetLoadResult:
        return await self._get_load(get_load_params or GetLoadParams(), timeout=timeout)


class ArraysToArraysServiceBase:
    """Server base: subclasses implement the three coroutines; ``__mapping__`` and
    :meth:`generic_handler` expose them to a ``grpc.aio`` server.

    Counterpart of ``pytensor_federated/rpc.py:129-187``.
    """

    async def evaluate(self, input_arrays: InputArrays) -> OutputArrays:
        raise NotImplementedError()

    async def evaluate_stream(
        self, input_arrays_iterator: AsyncIterator[InputArrays]
    ) -> AsyncIterator[OutputArrays]:
        raise NotImplementedError()
        yield OutputArrays()  # pragma: no cover

    async def get_load(self, get_load_params: GetLoadParams) -> GetLoadResult:
        raise NotImplementedError()

    # -- grpc.aio plumbing ---------------------------------------------------
    async def _rpc_evaluate(self, request, context):
        return await self.evaluate(request)

    async def _rpc_evaluate_stream(self, request_iterator, context):
        # explicit read()/write() on the call instead of returning an async generator: grpc.aio
        # wraps generator handlers in extra tasks, which costs ~15 % of the loopback round trip
        import grpc

        async def requests():
            while True:
                message = await context.read()
                if message is grpc.aio.EOF:
                    return
                yield message

        async for response in self.evaluate_stream(requests()):
            await context.write(response)

    async def _rpc_get_load(self, request, context):
        return await self.get_load(request)

    def __mapping__(self) -> Dict[str, object]:
        import grpc

        return {
            ROUTE_EVALUATE: grpc.unary_unary_rpc_method_handler(
                self._rpc_evaluate,
                request_deserializer=InputArrays.FromString,
                response_serializer=_serialize,
            ),
            ROUTE_EVALUATE_STREAM: grpc.stream_stream_rpc_method_handler(
                self._rpc_evaluate_stream,
                request_deserializer=InputArrays.FromString,
                response_serializer=_serialize,
            ),
            ROUTE_GET_LOAD: grpc.unary_unary_rpc_method_handler(
                self._rpc_get_load,
                request_deserializer=GetLoadParams.FromString,
                response_serializer=_serialize,
            ),
        }

    def generic_handler(self):
        import grpc

        methods = {route.rsplit("/", 1)[1]: h for route, h in self.__mapping__().items()}
        return grpc.method_handlers_generic_handler(SERVICE_NAME, methods)


class Server:
    """Tiny façade over ``grpc.aio.server`` with the grpclib-style lifecycle the
    reference's launchers use (``Server([service]); await start(host, port);
    await wait_closed()`` — ``demo_node.py:76-79``)."""

    def __init__(self, services: Sequence[ArraysToArraysServiceBase], *, tls=None) -> None:
        """``tls``: a :class:`~pytensor_federated_b200.config.TlsConfig` with ``cert`` + ``key`` (+ ``ca`` when
        ``mutual``); ``None`` = the ``B200FED_TLS_*`` environment, else plaintext like the reference;
        ``False`` = plaintext no matter what the environment says.  An incomplete configuration raises
        :class:`~pytensor_federated_b200.config.TlsConfigError` at ``start`` — it never degrades to plaintext."""
        self._services = list(services)
        self._server = None
        self._tls = tls
        self.port: Optional[int] = None

    async def start(self, host: str = "127.0.0.1", port: int = 0) -> int:
        import grpc.aio

        self._server = grpc.aio.server(options=CHANNEL_OPTIONS)
        self._server.add_generic_rpc_handlers(tuple(s.generic_handler() for s in self._services))
        from .config import tls_from_env

        tls = None if self._tls is False else (self._tls if self._tls is not None else tls_from_env())
        if tls is not None:
            import grpc

            tls.check_server()
            credentials = grpc.ssl_server_credentials(
                [(tls.key, tls.cert)], root_certificates=tls.ca if tls.mutual else None,
                require_client_auth=bool(tls.mutual),
            )
            self.port = self._server.add_secure_port(f"{host}:{port}", credentials)
        else:
            self.port = self._server.add_insecure_port(f"{host}:{port}")
        if self.port == 0:
            raise OSError(f"Could not bind {host}:{port}")
        await self._server.start()
        return self.port

    async def wait_closed(self) -> None:
        await self._server.wait_for_termination()

    def install_signal_handlers(self, grace: float = 5.0, signals=None) -> None:
        """SIGTERM / SIGINT drain the node instead of killing it mid-request: no new calls are accepted,
        requests in flight get ``grace`` seconds to finish, then the (long-lived) streams are cancelled —
        clients see ``StreamTerminatedError`` on their next call and fail over.  Call from the running loop."""
        import asyncio
        import signal

        loop = asyncio.get_running_loop()
        for sig in signals or (signal.SIGTERM, signal.SIGINT):
            loop.add_signal_handler(sig, lambda: loop.create_task(self.close(grace)))

    async def close(self, grace: Optional[float] = None) -> None:
        if self._server is not None:
            await self._server.stop(grace)


__all__ = [
    "InputArrays",
    "OutputArrays",
    "GetLoadParams",
    "GetLoadResult",
    "ArraysToArraysServiceStub",
    "ArraysToArraysServiceBase",
    "Server",
]
