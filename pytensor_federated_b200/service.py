"""``ArraysToArraysService`` / ``ArraysToArraysServiceClient`` — transport layer.

Capabilities mirrored from ``pytensor_federated/service.py``:

* server wrapper around a ``ComputeFunc`` with ``Evaluate`` / ``EvaluateStream`` /
  ``GetLoad`` (``:75-115``), load metric = 1-min loadavg per core and RAM % (``:88-96``)
* long-lived bidirectional evaluation stream (``:118-158``)
* load probes that map unreachable servers to ``None`` (``:161-211``)
* client-side balancing on the fewest connected clients (``:239-263``)
* per-(object, process, thread) connection cache so clients survive pickling,
  ``fork`` and ``spawn`` (``:266-275``)
* retry/failover on a terminated stream, ``TimeoutError`` when nobody answers
  (``:376-423``)

What is different, deliberately:

* **Two data planes.**  A ``(host, port)`` that was registered in this process with
  :func:`register_local_node` (a GPU node of the local NVSwitch domain, see
  :mod:`pytensor_federated_b200.parallel`) is evaluated by a direct call — no
  serialisation, no sockets.  Everything else goes through ``grpc.aio`` with the
  reference's exact wire schema, so reference servers and clients interoperate.
* ``n_clients`` is decremented in a ``finally`` (the reference leaks a count when a
  stream is torn down by an exception).
* The server can run slow compute functions off the event loop (``offload=True``)
  so ``GetLoad`` keeps answering while a model evaluates.
"""
from __future__ import annotations

import asyncio
import logging
import os
import random
import threading
import time
import uuid
from typing import AsyncIterator, Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import psutil

from .npproto.utils import ndarray_from_numpy, ndarray_to_numpy  # noqa: F401  (importable from here, as in the reference)
from .rpc import (
    CHANNEL_OPTIONS,
    ROUTE_EVALUATE_STREAM,
    ArraysToArraysServiceBase,
    ArraysToArraysServiceStub,
    GetLoadParams,
    GetLoadResult,
    InputArrays,
    OutputArrays,
)
from .signatures import ComputeFunc
from .utils import argmin_none_or_func, get_useful_event_loop

_log = logging.getLogger(__name__)

HostPort = Tuple[str, int]

CONNECT_SLEEP_RANGE: Tuple[float, float] = (0.2, 2.0)
"""Random delay before load probing that de-synchronises parallel MCMC chains
(``pytensor_federated/service.py:250``).  Override with the
``B200FED_CONNECT_SLEEP="lo,hi"`` environment variable (e.g. ``"0,0"`` in tests)."""


class StreamTerminatedError(Exception):
    """The evaluation stream (or the node behind it) went away mid-call.

    Plays the role of ``grpclib.exceptions.StreamTerminatedError`` in the
    reference's retry loop (``service.py:412``).
    """


def _connect_sleep_range() -> Tuple[float, float]:
    env = os.environ.get("B200FED_CONNECT_SLEEP")
    if env:
        lo, hi = (float(x) for x in env.split(","))
        return lo, hi
    return CONNECT_SLEEP_RANGE


def _run_compute_func(func_input: InputArrays, func: ComputeFunc) -> OutputArrays:
    """Decode → compute → encode; the request ``uuid`` is echoed.

    Reference: ``service.py:45-72``.
    """
    outputs = func(*func_input.arrays)
    return OutputArrays.from_arrays([np.asarray(o) for o in outputs], uuid=func_input.uuid)


def gpu_load(gpu_index: int) -> Optional[Tuple[float, float]]:
    """``(SM utilisation %, HBM used %)`` of a GPU via NVML, or ``None`` when NVML is unavailable.

    Kept out of the wire message (the proto has exactly three fields, SURVEY.md §5); exposed as
    ``GetLoadResult.percent_gpu`` / ``.percent_hbm`` attributes on the serving side and in the
    in-process registry so that custom balancing policies can use them.
    """
    try:
        import pynvml

        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(int(gpu_index))
        util = pynvml.nvmlDeviceGetUtilizationRates(h)
        mem = pynvml.nvmlDeviceGetMemoryInfo(h)
        return float(util.gpu), 100.0 * float(mem.used) / float(mem.total)
    except Exception:  # noqa: BLE001 - no driver / no NVML on CPU boxes
        return None


class ArraysToArraysService(ArraysToArraysServiceBase):
    """Serves a ``ComputeFunc`` over the ``ArraysToArraysService`` gRPC schema."""

    def __init__(self, compute_func: ComputeFunc, *, offload: bool = False, gpu_index: Optional[int] = None,
                 metrics=None) -> None:
        self._compute_func = compute_func
        self._n_clients = 0
        self._offload = offload
        self._gpu_index = gpu_index
        self._metrics = metrics  # optional metrics.ServiceMetrics (Prometheus counters / latency histogram)
        # psutil's load average needs one priming call to start monitoring.
        self.determine_load()
        # Load the message codec now: the first request should not pay for a library load.
        from .npproto import native_codec

        native_codec.available()
        super().__init__()

    def determine_load(self) -> GetLoadResult:
        """Current load: open evaluation streams, CPU % (1-min loadavg), RAM %."""
        load_1, _, _ = psutil.getloadavg()
        result = GetLoadResult(
            n_clients=self._n_clients,
            percent_cpu=load_1 / psutil.cpu_count() * 100,
            percent_ram=psutil.virtual_memory().percent,
        )
        if self._gpu_index is not None:
            result.gpu = gpu_load(self._gpu_index)  # local attribute, not serialised
        return result

    async def _run(self, input_arrays: InputArrays) -> OutputArrays:
        if self._metrics is None:
            return await self._run_unmetered(input_arrays)
        t0 = time.perf_counter()
        ok = False
        try:
            result = await self._run_unmetered(input_arrays)
            ok = True
            return result
        finally:
            self._metrics.observe(t0, ok)

    async def _run_unmetered(self, input_arrays: InputArrays) -> OutputArrays:
        if getattr(self._compute_func, "is_coroutine_compute_func", False) or asyncio.iscoroutinefunction(self._compute_func):
            # coroutine compute functions (e.g. batching.DynamicBatcher) overlap waiting requests
            outputs = await self._compute_func(*input_arrays.arrays)
            return OutputArrays.from_arrays([np.asarray(o) for o in outputs], uuid=input_arrays.uuid)
        if self._offload:
            loop = asyncio.get_running_loop()
            return await loop.run_in_executor(
                None, _run_compute_func, input_arrays, self._compute_func
            )
        return _run_compute_func(input_arrays, self._compute_func)

    def _clients_changed(self) -> None:
        if self._metrics is not None:
            self._metrics.set_clients(self._n_clients)

    async def evaluate(self, input_arrays: InputArrays) -> OutputArrays:
        return await self._run(input_arrays)

    async def evaluate_stream(
        self, input_arrays_iterator: AsyncIterator[InputArrays]
    ) -> AsyncIterator[OutputArrays]:
        _log.info("Evaluation stream opened")
        self._n_clients += 1
        self._clients_changed()
        try:
            async for input_arrays in input_arrays_iterator:
                yield await self._run(input_arrays)
        finally:
            self._n_clients -= 1
            self._clients_changed()
            _log.info("Evaluation stream closed")

    async def get_load(self, get_load_params: GetLoadParams) -> GetLoadResult:
        return self.determine_load()


# ---------------------------------------------------------------------------
# In-process nodes (the NVLink data plane plugs in here)
# ---------------------------------------------------------------------------


class LocalNode:
    """A node that lives in this process: a callable plus a client counter."""

    def __init__(self, compute_func: ComputeFunc, name: str = "") -> None:
        self.compute_func = compute_func
        self.name = name
        self.n_clients = 0
        self.alive = True

    def determine_load(self) -> GetLoadResult:
        load_1, _, _ = psutil.getloadavg()
        return GetLoadResult(
            n_clients=self.n_clients,
            percent_cpu=load_1 / psutil.cpu_count() * 100,
            percent_ram=psutil.virtual_memory().percent,
        )


_local_nodes: Dict[Tuple[str, int], LocalNode] = {}


def register_local_node(host: str, port: int, compute_func: ComputeFunc, name: str = "") -> LocalNode:
    """Makes ``(host, port)`` resolve to an in-process compute function.

    Clients that connect to this address skip gRPC and the npproto codec
    entirely.  GPU federations register their nodes here, which is how
    ``ArraysToArraysServiceClient("gpu", 3)`` reaches GPU 3 over NVLink.
    """
    node = LocalNode(compute_func, name=name or f"{host}:{port}")
    _local_nodes[(str(host), int(port))] = node
    return node


def unregister_local_node(host: str, port: int) -> None:
    """Removes an in-process node; clients connected to it get ``StreamTerminatedError`` on their next call."""
    node = _local_nodes.pop((str(host), int(port)), None)
    if node is not None:
        node.alive = False


def _lookup_local(host, port) -> Optional[LocalNode]:
    try:
        return _local_nodes.get((str(host), int(port)))
    except (TypeError, ValueError):
        return None


# ---------------------------------------------------------------------------
# Streams and load probes
# ---------------------------------------------------------------------------


_default_tls = None
_default_tls_set = False


def set_default_tls(tls) -> None:
    """Process-wide TLS material for outgoing connections (a :class:`~pytensor_federated_b200.config.TlsConfig`
    with at least ``ca``); ``None`` = plaintext.  Without a call the ``B200FED_TLS_*`` environment decides, so
    worker processes of a sampler inherit the setting.  Clients stay picklable: no credentials live on them."""
    global _default_tls, _default_tls_set
    _default_tls, _default_tls_set = tls, True


def _channel_tls():
    if _default_tls_set:
        return _default_tls
    from .config import tls_from_env

    return tls_from_env()


class _Channel:
    """``grpc.aio`` channel plus the bookkeeping the reference exposes on its
    channel objects (``_host`` / ``_port``; tests and log lines read them)."""

    def __init__(self, host: str, port: int) -> None:
        import grpc.aio

        self._host = host
        self._port = port
        tls = _channel_tls()
        if tls is not None:
            import grpc

            tls.check_client()  # incomplete material raises: a client never falls back to plaintext

            credentials = grpc.ssl_channel_credentials(root_certificates=tls.ca, private_key=tls.key,
                                                       certificate_chain=tls.cert)
            options = CHANNEL_OPTIONS
            if tls.server_name:
                options = options + (("grpc.ssl_target_name_override", tls.server_name),)
            self._channel = grpc.aio.secure_channel(f"{host}:{port}", credentials, options=options)
        else:
            self._channel = grpc.aio.insecure_channel(f"{host}:{port}", options=CHANNEL_OPTIONS)
        self._closed = False

    @property
    def raw(self):
        return self._channel

    @property
    def closed(self) -> bool:
        return self._closed

    def close(self) -> None:
        """Synchronous, idempotent close (safe inside and outside a running loop)."""
        if self._closed:
            return
        self._closed = True
        coro = self._channel.close(None)
        try:
            loop = asyncio.get_running_loop()
        except RuntimeError:
            loop = None
        try:
            if loop is not None:
                loop.create_task(coro)
            else:
                get_useful_event_loop().run_until_complete(coro)
        except Exception:  # pragma: no cover - best effort during teardown
            coro.close()


class RemoteComputeError(Exception):
    """The node answered the call with an application error (its compute function raised, or it
    rejected the request): re-running the same call would fail the same way, so it is reported once,
    with the server's status and message, instead of being retried like a lost connection."""

    def __init__(self, code, details: str) -> None:
        self.code = code
        self.details = details
        super().__init__(f"Remote evaluation failed ({getattr(code, 'name', code)}): {details}")


def _translate_rpc_error(ex) -> Exception:
    """``grpc.aio.AioRpcError`` -> connection loss (retry elsewhere) or application error (report)."""
    import grpc

    code = ex.code() if hasattr(ex, "code") else None
    sc = grpc.StatusCode
    # Codes a *handler* produces (a raised exception arrives as UNKNOWN; the others are explicit aborts).
    # Transport-level trouble — UNAVAILABLE, CANCELLED, DEADLINE_EXCEEDED, but also the INTERNAL
    # "error from Core" of a write to a peer that just died — means the connection is gone: retry elsewhere.
    application = (sc.UNKNOWN, sc.INVALID_ARGUMENT, sc.NOT_FOUND, sc.ALREADY_EXISTS, sc.PERMISSION_DENIED,
                   sc.FAILED_PRECONDITION, sc.OUT_OF_RANGE, sc.UNIMPLEMENTED, sc.UNAUTHENTICATED)
    if code not in application:
        return StreamTerminatedError(str(ex))
    details = ex.details() if hasattr(ex, "details") else str(ex)
    return RemoteComputeError(code, details or str(ex))


class EvaluationStream:
    """Bidirectional ``EvaluateStream`` call with grpclib-like method names."""

    def __init__(self, call) -> None:
        self._call = call

    async def send_message(self, message: InputArrays) -> None:
        import grpc

        try:
            await self._call.write(message)
        except asyncio.InvalidStateError as ex:
            raise StreamTerminatedError(str(ex)) from ex
        except grpc.aio.AioRpcError as ex:
            raise _translate_rpc_error(ex) from ex

    async def recv_message(self) -> Optional[OutputArrays]:
        import grpc

        try:
            response = await self._call.read()
        except grpc.aio.AioRpcError as ex:
            raise _translate_rpc_error(ex) from ex
        if response is grpc.aio.EOF:
            raise StreamTerminatedError("The evaluation stream was closed by the server.")
        return response

    async def end(self) -> None:
        try:
            await self._call.done_writing()
        except Exception:
            pass
        self._call.cancel()


async def start_bidirectional_stream(
    *,
    client: ArraysToArraysServiceStub,
    route: str = ROUTE_EVALUATE_STREAM,
    request_type=InputArrays,
    response_type=OutputArrays,
    timeout: Optional[float] = None,
    connect_timeout: Optional[float] = 5.0,
) -> EvaluationStream:
    """Opens the evaluation stream and keeps it open across calls.

    One long-lived stream avoids per-call stream setup, which is what makes the
    streamed mode "much faster" than unary calls in the reference
    (``service.py:118-147``).
    """
    import grpc

    call = client.channel.stream_stream(
        route,
        request_serializer=bytes,
        response_deserializer=response_type.FromString,
    )(timeout=timeout)
    try:
        await asyncio.wait_for(call.wait_for_connection(), connect_timeout)
    except (grpc.aio.AioRpcError, asyncio.TimeoutError) as ex:
        call.cancel()
        raise StreamTerminatedError(f"Could not open evaluation stream: {ex}") from ex
    return EvaluationStream(call)


async def _streamed_evaluate(input: InputArrays, stream: EvaluationStream) -> OutputArrays:
    await stream.send_message(input)
    response = await stream.recv_message()
    if response is None:
        raise Exception("Received unexpected `None` response.")
    return response


async def get_load_async(host: str, port: int, timeout: float = 5) -> Optional[GetLoadResult]:
    """Load of one server, or ``None`` if it does not answer in time.

    Reference: ``service.py:161-186``.
    """
    local = _lookup_local(host, port)
    if local is not None:
        return local.determine_load() if local.alive else None

    import grpc

    channel = _Channel(host, port)
    client = ArraysToArraysServiceStub(channel.raw)
    try:
        load = await client.get_load(GetLoadParams(), timeout=timeout)
    except (grpc.aio.AioRpcError, ConnectionRefusedError, asyncio.TimeoutError, OSError):
        load = None
    finally:
        await channel.raw.close(None)
        channel._closed = True
    return load


async def get_loads_async(
    hosts_and_ports: Sequence[HostPort], *, timeout: float = 5
) -> List[Optional[GetLoadResult]]:
    """Loads of all servers, concurrently; failures become ``None``.

    Reference: ``service.py:189-211``.
    """
    coros = [get_load_async(host, int(port), timeout) for host, port in hosts_and_ports]
    loads = await asyncio.gather(*coros, return_exceptions=True)
    return [(l if isinstance(l, GetLoadResult) else None) for l in loads]


class ClientPrivates:
    """Un-picklable connection state private to one (client, process, thread)."""

    def __init__(self, channel, client, stream, *, local: Optional[LocalNode] = None) -> None:
        self.channel = channel
        self.client = client
        self.stream = stream
        self.local = local
        self.loop = asyncio._get_running_loop()
        # One request/response pair at a time per stream: several coroutines of a fused graph
        # node may share one client object (the reference relies on FIFO luck here, SURVEY §3.3).
        self.lock = asyncio.Lock() if self.loop is not None else None

    @staticmethod
    async def connect(host: str, port: int) -> "ClientPrivates":
        local = _lookup_local(host, port)
        if local is not None:
            if not local.alive:
                raise StreamTerminatedError(f"Local node {host}:{port} is gone.")
            local.n_clients += 1
            return ClientPrivates(_LocalChannel(host, port, local), None, None, local=local)
        channel = _Channel(host, int(port))
        client = ArraysToArraysServiceStub(channel.raw)
        try:
            stream = await start_bidirectional_stream(client=client)
        except StreamTerminatedError:
            channel.close()
            raise
        return ClientPrivates(channel, client, stream)

    @staticmethod
    async def connect_balanced(hosts_and_ports: Sequence[HostPort]) -> "ClientPrivates":
        """Connects to the server with the fewest clients.

        Shuffle (random probe order and random tie-break) → random pause (chains
        started together do not all see the same snapshot) → probe → argmin.
        Reference: ``service.py:239-263``.
        """
        rng = random.Random(random.randint(0, 100_000) ^ os.getpid() ^ threading.get_ident())
        candidates = [(str(h), int(p)) for h, p in hosts_and_ports]
        # replicas that recently stalled on a call sit out (unless nothing else is left)
        now = time.monotonic()
        healthy = [c for c in candidates if _quarantine.get(c, 0.0) <= now]
        candidates = healthy or candidates
        rng.shuffle(candidates)

        lo, hi = _connect_sleep_range()
        if hi > 0:
            await asyncio.sleep(rng.uniform(lo, hi))

        loads = await get_loads_async(candidates)
        isel = argmin_none_or_func(loads, lambda l: l.n_clients)
        if isel is None:
            raise TimeoutError(
                f"None of {len(candidates)} servers responded to load information requests."
            )
        host, port = candidates[isel]
        return await ClientPrivates.connect(host, port)

    def close(self) -> None:
        if self.local is not None:
            self.local.n_clients = max(0, self.local.n_clients - 1)
            self.local = None
        if self.channel is not None:
            self.channel.close()


class _LocalChannel:
    """Stands in for a network channel when the node is in-process."""

    def __init__(self, host: str, port: int, node: LocalNode) -> None:
        self._host = host
        self._port = port
        self._node = node
        self._closed = False

    @property
    def closed(self) -> bool:
        return self._closed

    def close(self) -> None:
        self._closed = True


QUARANTINE_SECONDS = 30.0
_quarantine: Dict[Tuple[str, int], float] = {}
"""Replicas that exceeded a caller's ``timeout``: (host, port) -> monotonic time until which the balancer
skips them.  Process-local, like the connection cache."""

_privates: Dict[str, ClientPrivates] = {}
"""Non-reusable connections, keyed by :func:`thread_pid_id`."""


def thread_pid_id(obj: object) -> str:
    """A process- and thread-specific identifier of an object."""
    return f"{id(obj)}-{os.getpid()}-{threading.get_ident()}"


async def _connect_evaluate_async(
    input: InputArrays,
    cid: str,
    hosts_and_ports: Sequence[HostPort],
    use_stream: bool,
) -> OutputArrays:
    """Connects (or re-uses the cached connection) and evaluates over gRPC.

    Reference: ``service.py:278-323``.
    """
    priv = await _get_connection(cid, hosts_and_ports)
    if use_stream:
        async with priv.lock:
            output = await _streamed_evaluate(input, priv.stream)
    else:
        import grpc

        try:
            output = await priv.client.evaluate(input)
        except grpc.aio.AioRpcError as ex:
            raise _translate_rpc_error(ex) from ex
    if output.uuid != input.uuid:
        raise Exception("Response does not correspond to the request.")
    return output


_connect_locks: Dict[Tuple[str, int], asyncio.Lock] = {}


async def _get_connection(cid: str, hosts_and_ports: Sequence[HostPort]) -> ClientPrivates:
    # concurrent first calls of one client (fused graph node) must not race to connect
    key = (cid, id(asyncio.get_running_loop()))
    lock = _connect_locks.get(key)
    if lock is None:
        lock = _connect_locks[key] = asyncio.Lock()
    async with lock:
        return await _get_connection_locked(cid, hosts_and_ports)


async def _get_connection_locked(cid: str, hosts_and_ports: Sequence[HostPort]) -> ClientPrivates:
    priv = _privates.get(cid)
    if priv is not None and priv.local is None and priv.loop is not asyncio._get_running_loop():
        # grpc.aio objects are bound to the loop they were created on.
        _privates.pop(cid).close()
        priv = None
    if priv is None:
        _log.debug("Connecting client %s", cid)
        if len(hosts_and_ports) == 1:
            host, port = hosts_and_ports[0]
            priv = await ClientPrivates.connect(host, port)
        else:
            priv = await ClientPrivates.connect_balanced(hosts_and_ports)
        _privates[cid] = priv
        _log.info("Client %s connected to %s:%s", cid, priv.channel._host, priv.channel._port)
    return priv


class ArraysToArraysServiceClient:
    """A picklable ``ComputeFunc`` that evaluates on a (possibly remote) node.

    Parameters
    ----------
    host, port
        Address of one node.
    hosts_and_ports
        Several replica nodes; takes precedence over ``host``/``port`` and enables
        client-side load balancing and failover.

    Only the addresses are stored on the object; connections live in
    :data:`_privates` and are created lazily per process and thread, which is what
    makes the client safe to pickle into ``multiprocessing`` workers
    (reference: ``service.py:326-423``).
    """

    def __init__(
        self,
        host: Optional[str] = None,
        port: Optional[int] = None,
        *,
        hosts_and_ports: Optional[Sequence[HostPort]] = None,
    ) -> None:
        self._host = host
        self._port = port
        self._hosts_and_ports = hosts_and_ports
        super().__init__()

    def __del__(self):
        try:
            _id = thread_pid_id(self)
            for key in [k for k in _connect_locks if k[0] == _id]:
                _connect_locks.pop(key, None)
            priv = _privates.pop(_id, None)
            if priv is None:
                return
            _log.info("Closing evaluation stream")
            if priv.stream is not None:
                loop = get_useful_event_loop()
                if not loop.is_closed() and not loop.is_running():
                    loop.run_until_complete(priv.stream.end())
            priv.close()
        except Exception:  # pragma: no cover - interpreter shutdown
            pass

    def __call__(self, *inputs: np.ndarray) -> List[np.ndarray]:
        """Alias for ``.evaluate(*inputs)``."""
        return self.evaluate(*inputs)

    def evaluate(self, *inputs: np.ndarray, **kwargs) -> List[np.ndarray]:
        retries = kwargs.get("retries", 2)
        if retries < 0:
            raise ValueError("Number of retries must be >= 0.")
        # Fast path: a cached in-process node needs no event loop at all.
        priv = _privates.get(thread_pid_id(self))
        if priv is not None and priv.local is not None and priv.local.alive:
            try:
                return _evaluate_local(priv.local, inputs)
            except StreamTerminatedError:
                pass  # the node died under this call: the general path below reconnects (to another replica)
        loop = get_useful_event_loop()
        return loop.run_until_complete(self.evaluate_async(*inputs, **kwargs))

    async def evaluate_async(
        self, *inputs: np.ndarray, use_stream: bool = True, retries: int = 2, timeout: Optional[float] = None
    ) -> List[np.ndarray]:
        """Evaluates the federated compute function on ``inputs``.

        Parameters
        ----------
        *inputs
            NumPy ``ndarray`` inputs.
        use_stream
            ``True`` (default) sends the call through the long-lived bidirectional
            stream; ``False`` makes a unary RPC per call (slower).
        retries
            How many times to re-connect (possibly to another replica) when the
            connection is lost mid-call.
        timeout
            Seconds one attempt may take (default: unbounded, like the reference).  A node that accepts
            the call but never answers is treated like a lost connection: the stream is dropped, the node
            is skipped by the balancer for ``QUARANTINE_SECONDS``, the next attempt re-balances over the
            remaining replicas, and ``TimeoutError`` is raised when every attempt timed out.
        """
        if retries < 0:
            raise ValueError("Number of retries must be >= 0.")

        cid = thread_pid_id(self)
        hap = self._hosts_and_ports or [(self._host, self._port)]

        input: Optional[InputArrays] = None
        output: Optional[OutputArrays] = None
        last_error: Optional[Exception] = None
        for _ in range(retries + 1):
            try:
                priv = await _get_connection(cid, hap)
                if priv.local is not None:
                    if not priv.local.alive:
                        raise StreamTerminatedError("Local node was unregistered.")
                    return _evaluate_local(priv.local, inputs)
                if input is None:
                    input = InputArrays.from_arrays([np.asarray(i) for i in inputs], uuid=str(uuid.uuid4()))
                call = _connect_evaluate_async(input, cid, hap, use_stream)
                output = await (call if timeout is None else _bounded(call, timeout))
                break
            except RemoteComputeError:
                # the stream died with the failed call; the next evaluation reconnects, this one reports
                cp = _privates.pop(cid, None)
                if cp is not None:
                    cp.close()
                raise
            except (StreamTerminatedError, _AttemptTimedOut) as ex:
                last_error = ex
                cp = _privates.pop(cid, None)
                if cp is not None:
                    what = "No answer within the timeout from" if isinstance(ex, _AttemptTimedOut) else "Lost connection to"
                    _log.warning("%s %s:%s.", what, cp.channel._host, cp.channel._port)
                    if isinstance(ex, _AttemptTimedOut):
                        try:
                            _quarantine[(str(cp.channel._host), int(cp.channel._port))] = time.monotonic() + QUARANTINE_SECONDS
                        except (TypeError, ValueError):  # in-process nodes have symbolic addresses
                            pass
                    if cp.stream is not None:
                        cp.stream._call.cancel()  # a half-finished request must not be answered into the next one
                    cp.close()

        if output is None:
            if isinstance(last_error, _AttemptTimedOut):
                raise TimeoutError(f"No answer within {timeout} s in {retries + 1} attempt(s).")
            raise StreamTerminatedError(
                f"Evaluation failed after {retries + 1} attempt(s): {last_error}"
            )
        return list(output.arrays)


class _AttemptTimedOut(Exception):
    """One evaluation attempt exceeded the caller's ``timeout`` (distinct from the ``TimeoutError`` that
    ``connect_balanced`` raises when no server answers the load probes)."""


async def _bounded(coro, timeout: float):
    task = asyncio.ensure_future(coro)
    done, _ = await asyncio.wait({task}, timeout=timeout)
    if not done:
        task.cancel()
        try:
            await task
        except BaseException:  # noqa: BLE001 - the cancelled attempt's outcome is irrelevant
            pass
        raise _AttemptTimedOut()
    return task.result()


def _evaluate_local(node: LocalNode, inputs) -> List[np.ndarray]:
    try:
        outputs = node.compute_func(*[np.asarray(i) for i in inputs])
        if asyncio.iscoroutine(outputs):  # coroutine compute functions (e.g. a DynamicBatcher) work in-process too
            outputs = get_useful_event_loop().run_until_complete(outputs)
    except Exception as ex:
        # An in-process node whose engine is gone (GPU lost, peer timed out, engine shut down) is the local
        # counterpart of a dropped connection: the node is marked dead and the client's retry loop fails over to
        # another replica (reference semantics: service.py:407-416).  Exceptions opt in with `marks_node_lost`.
        if getattr(ex, "marks_node_lost", False):
            node.alive = False
            raise StreamTerminatedError(f"In-process node {node.name} is gone: {ex}") from ex
        raise
    return [np.asarray(o) for o in outputs]


async def serve(
    compute_func: ComputeFunc,
    bind: str = "127.0.0.1",
    port: int = 0,
    *,
    offload: bool = False,
    ready: Optional[Callable[[int], None]] = None,
) -> None:
    """Serves ``compute_func`` until cancelled (helper for node launchers)."""
    from .metrics import metrics_from_env
    from .rpc import Server

    service = ArraysToArraysService(compute_func, offload=offload, metrics=metrics_from_env())
    server = Server([service])
    bound = await server.start(bind, port)
    try:
        server.install_signal_handlers()
    except (NotImplementedError, RuntimeError, ValueError):  # no signal support here (non-main thread, Windows)
        pass
    _log.info("Serving on %s:%i", bind, bound)
    if ready is not None:
        ready(bound)
    try:
        await server.wait_closed()
    finally:
        await server.close(None)


__all__ = [
    "ArraysToArraysService",
    "ArraysToArraysServiceClient",
    "ClientPrivates",
    "EvaluationStream",
    "LocalNode",
    "RemoteComputeError",
    "StreamTerminatedError",
    "get_load_async",
    "get_loads_async",
    "register_local_node",
    "set_default_tls",
    "unregister_local_node",
    "serve",
    "start_bidirectional_stream",
    "thread_pid_id",
]
