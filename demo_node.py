"""Worker-node launcher: serves the demo linear model behind the ArraysToArrays gRPC schema.

CLI-compatible with the reference's ``demo_node.py`` (``--bind --ports --delay``, one OS process
per port, ``demo_node.py:98-134``); any pytensor-federated client can connect.
The node's private dataset lives on the GPU when one is visible (``--device cuda``) and each
evaluation is one fused sm_90a kernel launch; ``--device cpu`` uses the eager oracle.

For the on-box data plane (no sockets at all) see ``demo_model.py --fused``.
"""
import argparse
import asyncio
import logging
import multiprocessing
import time
from typing import Sequence, Tuple

import numpy as np

_log = logging.getLogger("demo_node")


class LinearModelBlackbox:
    """``(intercept, slope) -> (logp, [d_intercept, d_slope])`` on a private dataset."""

    def __init__(self, data_x, data_y, sigma: float, delay: float = 0.0, device: str = "auto") -> None:
        import torch

        from pytensor_federated_b200.models import LinregShards
        from pytensor_federated_b200.parallel import FederatedEngine

        if device == "auto":
            device = "cuda" if torch.cuda.is_available() else "cpu"
        self._delay = delay
        model = LinregShards([data_x], [data_y], [sigma], device=torch.device(device))
        self._engine = FederatedEngine(model, backend="fused" if device.startswith("cuda") else "collective")

    def __call__(self, *parameters) -> Tuple[np.ndarray, Sequence[np.ndarray]]:
        t0 = time.perf_counter()
        logp, grads = self._engine.logp_grad(*parameters)
        time.sleep(max(0.0, self._delay - (time.perf_counter() - t0)))
        return logp, grads


async def run_node_async(*, bind: str, port: int, delay: float, device: str, metrics_port: int = 0) -> None:
    from pytensor_federated_b200 import ArraysToArraysService, wrap_logp_grad_func
    from pytensor_federated_b200.metrics import ServiceMetrics
    from pytensor_federated_b200.models import make_demo_data
    from pytensor_federated_b200.rpc import Server

    _log.info("Generating a secret dataset")
    x, y, sigma = make_demo_data()
    import scipy.stats

    print(scipy.stats.linregress(x, y))
    model_fn = LinearModelBlackbox(x, y, sigma, delay=delay, device=device)
    _log.info("Binding the service to %s on port %i", bind, port)
    metrics = ServiceMetrics(port=metrics_port) if metrics_port else None   # Prometheus /metrics endpoint
    server = Server([ArraysToArraysService(wrap_logp_grad_func(model_fn), metrics=metrics)])
    await server.start(bind, port)
    server.install_signal_handlers()      # SIGTERM / SIGINT: finish the request in flight, then close
    await server.wait_closed()


def run_node(args: Tuple[str, int, float, str, int]) -> None:
    bind, port, delay, device, metrics_port = args
    logging.basicConfig(level=logging.INFO)
    try:
        asyncio.new_event_loop().run_until_complete(
            run_node_async(bind=bind, port=port, delay=delay, device=device, metrics_port=metrics_port))
    except KeyboardInterrupt:
        pass


def run_node_pool(bind: str, ports: Sequence[int], delay: float, device: str, metrics_port: int = 0) -> None:
    _log.info("Launching workers on %i subprocesses", len(ports))
    ctx = multiprocessing.get_context("spawn")  # CUDA contexts do not survive fork()
    with ctx.Pool(len(ports)) as pool:
        try:
            pool.map(run_node, [(bind, p, delay, device, metrics_port + i if metrics_port else 0)
                                for i, p in enumerate(ports)])
        except KeyboardInterrupt:
            _log.info("Stopping workers...")
            pool.terminate()
    _log.info("All workers exited.")


if __name__ == "__main__":
    logging.basicConfig(level=logging.INFO)
    parser = argparse.ArgumentParser(description="Runs a toy model as a worker node.")
    parser.add_argument("--bind", default="0.0.0.0", help="IP address to run the ArraysToArrays gRPC service on.")
    parser.add_argument("--ports", default=",".join(map(str, range(50000, 50003))), type=str,
                        help="Port numbers for the ArraysToArrays gRPC service.")
    parser.add_argument("--delay", default=0, type=float, help="Seconds to sleep in each evaluation.")
    parser.add_argument("--device", default="auto", choices=["auto", "cuda", "cpu"])
    parser.add_argument("--metrics-port", default=0, type=int,
                        help="Prometheus endpoint of the first worker (worker i serves on this port + i); 0 = off.")
    args, _ = parser.parse_known_args()
    run_node_pool(args.bind, [int(p) for p in str(args.ports).split(",")], args.delay, args.device, args.metrics_port)
