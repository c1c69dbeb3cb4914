"""Runtime configuration: one dataclass, environment overrides.

The reference has no configuration system (constructor kwargs and hard-coded constants only,
SURVEY.md §5 "Config / flag system"); its kwargs are kept verbatim on the public classes and the
knobs that were constants there are gathered here.

Environment variables (all optional):

``B200FED_COMM``            ``auto`` | ``symm`` | ``ipc`` — how peers' comm blocks are mapped
``B200FED_NO_MULTICAST``    set to disable NVSwitch multicast stores (P2P stores instead)
``B200FED_GLM_KERNEL``      ``auto`` | ``tc`` | ``simt`` | ``fp8``
``B200FED_TIMEOUT``         seconds ONE evaluation may take before ``FederationTimeout`` (dead peer, lost theta)
``B200FED_IDLE_TIMEOUT``    seconds a peer keeps waiting between evaluations (0 = for ever; it re-arms its kernels)
``B200FED_SERVE_AHEAD``     kernels a peer keeps pre-enqueued
``B200FED_CONNECT_SLEEP``   ``"lo,hi"`` seconds of the balanced-connect de-synchronisation pause
``B200FED_PROBE_TIMEOUT``   seconds to wait for a ``GetLoad`` answer
``B200FED_GRAPH_BACKEND``   ``auto`` | ``builtin`` — graph IR of the Op layer
``B200FED_NVTX``            set to wrap every evaluation in an NVTX range (host-side tracing)
``B200FED_METRICS_PORT``    Prometheus ``/metrics`` port of a node started with ``service.serve`` (``metrics.py``)
``B200FED_TLS_CA`` / ``B200FED_TLS_CERT`` / ``B200FED_TLS_KEY`` / ``B200FED_TLS_SERVER_NAME`` / ``B200FED_TLS_MUTUAL``
                            PEM files that switch the gRPC path to TLS (see :class:`TlsConfig`)
``B200FED_ALLOW_PICKLE``    set to decode object-dtype arrays (unpickles peer data: trusted federations only)
``B200FED_NO_LL``           set to force the fence + flag protocol for small results (default: flag-in-data words)
``B200FED_LL_MAX_VALS`` / ``B200FED_LL_MAX_THETA``   size thresholds of the flag-in-data protocol (2048 values / 4096 words)
"""
from __future__ import annotations

import dataclasses
import os
from typing import Optional, Tuple


def _env_float(name: str, default: float) -> float:
    try:
        return float(os.environ[name])
    except (KeyError, ValueError):
        return default


def _env_int(name: str, default: int) -> int:
    try:
        return int(os.environ[name])
    except (KeyError, ValueError):
        return default


def _env_pair(name: str, default: Tuple[float, float]) -> Tuple[float, float]:
    try:
        lo, hi = (float(x) for x in os.environ[name].split(","))
        return lo, hi
    except (KeyError, ValueError):
        return default


@dataclasses.dataclass
class FederationConfig:
    """Engine / client knobs with environment overrides (``B200FED_COMM``, ``B200FED_TIMEOUT``, ...)."""

    comm: str = "auto"
    multicast: bool = True
    glm_kernel: str = "auto"
    timeout: float = 20.0
    idle_timeout: float = 0.0     # peers: give up after this long without an evaluation (0 = never)
    serve_ahead: int = 8
    speculative_us: float = 0.0   # root: keep kernels enqueued ahead of the next theta, each waits this long (0 = off)
    connect_sleep: Tuple[float, float] = (0.2, 2.0)
    probe_timeout: float = 5.0
    retries: int = 2
    graph_backend: str = "auto"

    @classmethod
    def from_env(cls) -> "FederationConfig":
        return cls(
            comm=os.environ.get("B200FED_COMM", "auto"),
            multicast=not os.environ.get("B200FED_NO_MULTICAST"),
            glm_kernel=os.environ.get("B200FED_GLM_KERNEL", "auto"),
            timeout=_env_float("B200FED_TIMEOUT", 20.0),
            idle_timeout=_env_float("B200FED_IDLE_TIMEOUT", 0.0),
            serve_ahead=_env_int("B200FED_SERVE_AHEAD", 8),
            speculative_us=_env_float("B200FED_SPECULATIVE_US", 0.0),
            connect_sleep=_env_pair("B200FED_CONNECT_SLEEP", (0.2, 2.0)),
            probe_timeout=_env_float("B200FED_PROBE_TIMEOUT", 5.0),
            graph_backend=os.environ.get("B200FED_GRAPH_BACKEND", "auto"),
        )


class TlsConfigError(ValueError):
    """TLS was requested (explicitly or through ``B200FED_TLS_*``) but the material is incomplete for the
    role; the process refuses to fall back to plaintext."""


@dataclasses.dataclass(frozen=True)
class TlsConfig:
    """TLS material of the gRPC path (PEM bytes).  The reference only speaks plaintext
    (``grpclib.client.Channel(host, port)``, ``pytensor_federated/service.py:230``); nodes
    that hold private data usually sit behind TLS, optionally with client certificates.

    Server: ``cert`` + ``key`` (its identity); ``ca`` + ``mutual=True`` additionally demands client certs.
    Client: ``ca`` (who signed the server), optionally ``cert`` + ``key`` (its identity for mutual TLS) and
    ``server_name`` when the certificate was issued for a name other than the dialled host."""

    ca: Optional[bytes] = None
    cert: Optional[bytes] = None
    key: Optional[bytes] = None
    server_name: Optional[str] = None
    mutual: bool = False

    def check_server(self) -> "TlsConfig":
        """A server needs its identity (``cert`` + ``key``) and, for mutual TLS, the ``ca`` that signed the
        clients.  Anything less raises instead of silently serving private data in cleartext."""
        missing = [name for name in ("cert", "key") if not getattr(self, name)]
        if self.mutual and not self.ca:
            missing.append("ca (mutual TLS)")
        if missing:
            raise TlsConfigError(f"incomplete TLS configuration for a server: missing {', '.join(missing)}")
        return self

    def check_client(self) -> "TlsConfig":
        """A client needs the ``ca`` it trusts; ``cert`` and ``key`` (mutual TLS) only come as a pair."""
        missing = [] if self.ca else ["ca"]
        if bool(self.cert) != bool(self.key):
            missing.append("key" if self.cert else "cert")
        if missing:
            raise TlsConfigError(f"incomplete TLS configuration for a client: missing {', '.join(missing)}")
        return self

    @classmethod
    def from_files(cls, ca: Optional[str] = None, cert: Optional[str] = None, key: Optional[str] = None,
                   server_name: Optional[str] = None, mutual: bool = False) -> "TlsConfig":
        def read(path):
            if not path:
                return None
            with open(path, "rb") as fh:
                return fh.read()

        return cls(ca=read(ca), cert=read(cert), key=read(key), server_name=server_name, mutual=mutual)


def tls_from_env() -> Optional[TlsConfig]:
    """``TlsConfig`` from the ``B200FED_TLS_*`` variables (paths to PEM files), or ``None`` = plaintext (none
    of them set).  A partially filled environment yields a config whose ``check_server`` / ``check_client``
    raises :class:`TlsConfigError` — it never degrades to plaintext."""
    ca, cert, key = (os.environ.get(f"B200FED_TLS_{k}") for k in ("CA", "CERT", "KEY"))
    if not (ca or cert or key or os.environ.get("B200FED_TLS_MUTUAL")):
        return None
    return TlsConfig.from_files(ca, cert, key, os.environ.get("B200FED_TLS_SERVER_NAME"),
                                bool(os.environ.get("B200FED_TLS_MUTUAL")))


def get_config() -> FederationConfig:
    """The configuration in effect: defaults overridden by ``B200FED_*`` environment variables."""
    return FederationConfig.from_env()
