"""Optional Prometheus metrics of a serving node.

The reference's only metric endpoint is the ``GetLoad`` RPC (``pytensor_federated/
service.py:88-96``).  A production node additionally wants scrapeable counters and latency histograms;
``ServiceMetrics`` wraps ``prometheus_client`` (when installed) behind a no-op fallback, so the service
code never has to test for it:

    metrics = ServiceMetrics(port=9100)            # starts the /metrics HTTP endpoint
    service = ArraysToArraysService(fn, metrics=metrics)

or set ``B200FED_METRICS_PORT=9100`` before starting ``demo_node.py`` / ``service.serve``.
"""
from __future__ import annotations

import os
import time
from typing import Optional

__all__ = ["ServiceMetrics", "metrics_from_env"]

_BUCKETS = (1e-5, 3e-5, 1e-4, 3e-4, 1e-3, 3e-3, 1e-2, 3e-2, 0.1, 0.3, 1.0, 3.0, 10.0)


class ServiceMetrics:
    """Counters / histogram / gauge of one ``ArraysToArraysService`` (own registry, so several services and
    repeated construction in tests never collide on metric names)."""

    def __init__(self, port: Optional[int] = None, addr: str = "0.0.0.0", namespace: str = "b200fed") -> None:
        self.enabled = False
        self.port = None
        self._server = None
        try:
            import prometheus_client as prom
        except ModuleNotFoundError:  # metrics are optional
            return
        self._prom = prom
        self.registry = prom.CollectorRegistry()
        self.evaluations = prom.Counter("evaluations", "Evaluate / EvaluateStream requests answered",
                                        namespace=namespace, registry=self.registry)
        self.errors = prom.Counter("errors", "Requests whose compute function raised", namespace=namespace,
                                   registry=self.registry)
        self.seconds = prom.Histogram("compute_seconds", "Decode + compute + encode time per request",
                                      namespace=namespace, buckets=_BUCKETS, registry=self.registry)
        self.clients = prom.Gauge("clients", "Open evaluation streams (the balancer's n_clients)",
                                  namespace=namespace, registry=self.registry)
        self.enabled = True
        if port is not None:
            started = prom.start_http_server(int(port), addr=addr, registry=self.registry)
            # prometheus_client >= 0.17 returns (server, thread); older versions return None
            self._server = started[0] if isinstance(started, tuple) else None
            self.port = self._server.server_port if self._server is not None else int(port)

    # -- hooks used by the service -----------------------------------------------------------------
    def observe(self, t_start: float, ok: bool) -> None:
        if not self.enabled:
            return
        self.evaluations.inc()
        if not ok:
            self.errors.inc()
        self.seconds.observe(time.perf_counter() - t_start)

    def set_clients(self, n: int) -> None:
        if self.enabled:
            self.clients.set(n)

    def render(self) -> str:
        """The exposition text (what the HTTP endpoint serves); empty when prometheus_client is missing."""
        return self._prom.generate_latest(self.registry).decode() if self.enabled else ""

    def close(self) -> None:
        if self._server is not None:
            self._server.shutdown()
            self._server.server_close()
            self._server = None


def metrics_from_env() -> Optional[ServiceMetrics]:
    """``ServiceMetrics`` on ``B200FED_METRICS_PORT`` when that variable is set, else ``None``."""
    port = os.environ.get("B200FED_METRICS_PORT")
    if not port:
        return None
    return ServiceMetrics(port=int(port))
