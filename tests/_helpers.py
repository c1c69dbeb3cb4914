"""Shared helpers for multi-process service tests (CPU only)."""
import asyncio
import multiprocessing
import socket
import time
from typing import Optional, Sequence, Tuple

import numpy as np


def product_func(*inputs) -> Tuple[np.ndarray]:
    return (np.prod(inputs),)


def free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def slow_product_func(a, b):
    """Like the product, but a == 99 takes two seconds (a node that accepts a call and then stalls)."""
    if a == 99:
        time.sleep(2.0)
    return [a * b]


def gaussian_logp_grad_func(theta):
    """ComputeFunc of a N(1, 0.5^2 I) log-density: ``(logp, dlogp/dtheta)``."""
    z = (np.asarray(theta, dtype=np.float64) - 1.0) / 0.5
    return [np.asarray(-0.5 * np.sum(z * z)), -z / 0.5]


def remote_gaussian_logp_dlogp(hosts_and_ports):
    """Picklable model factory for sample_parallel: connects (load-balanced) inside the worker."""
    from pytensor_federated_b200 import LogpGradServiceClient

    client = LogpGradServiceClient(hosts_and_ports=hosts_and_ports)

    def logp_dlogp(theta):
        logp, (grad,) = client.evaluate(theta)
        return float(logp), np.asarray(grad, dtype=np.float64)

    return logp_dlogp


def straight_line_blackbox(intercept, slope):
    """Gradient-free black box: log-likelihood of y = 2 x + 0.5 (+ noise, sd 0.1) at 15 points.

    The fixture of the reference's gradient-free end-to-end test
    (``pytensor_federated/test_wrapper_ops.py:55-65``): same data-generating recipe, so the
    golden value of that test, ``logp(0.4, 1.2) = -1511.41423640139``, must come out here too."""
    import scipy.stats

    x = np.linspace(-3.0, 3.0, num=15)
    y = np.random.RandomState(42).normal(loc=2.0 * x + 0.5, scale=0.1)
    return np.asarray(scipy.stats.norm(loc=intercept + slope * x, scale=0.1).logpdf(y).sum())


def slope_posterior_logp(port: int, use_async: bool):
    """Picklable model factory for ``sample_parallel(sampler="metropolis")``: builds, INSIDE the worker, the
    model of the reference test — fixed intercept 0.5, ``slope ~ N(0, 2)``, the remote black box as a
    ``Potential`` through ``LogpOp`` / ``AsyncLogpOp`` — and returns its gradient-free ``logp(theta)``."""
    from pytensor_federated_b200 import AsyncLogpOp, LogpOp, LogpServiceClient
    from pytensor_federated_b200._graph_backend import at
    from pytensor_federated_b200.sampling import Model

    client = LogpServiceClient("127.0.0.1", port)
    op = AsyncLogpOp(client.evaluate_async) if use_async else LogpOp(client)
    m = Model()
    slope = m.Normal("slope", 0.0, 2.0)
    m.Potential("L", op(at.constant(0.5), slope))
    m._client = client   # keeps the connection alive as long as the model
    return m.logp


def _serve(port: int, n_clients: int, func_name: str, ready) -> None:
    from pytensor_federated_b200 import service
    from pytensor_federated_b200.rpc import Server

    from pytensor_federated_b200 import wrap_logp_func

    func = {"product": product_func, "gaussian": gaussian_logp_grad_func, "slow_product": slow_product_func,
            "blackbox_logp": wrap_logp_func(straight_line_blackbox)}[func_name]

    async def main():
        svc = service.ArraysToArraysService(func)
        svc._n_clients = n_clients  # fake load, like the reference's tests do
        server = Server([svc])
        await server.start("127.0.0.1", port)
        ready.set()
        await server.wait_closed()

    asyncio.new_event_loop().run_until_complete(main())


class ServerProcess:
    """A node in a child process; ``terminate()`` is the fault-injection knob."""

    def __init__(self, port: Optional[int] = None, n_clients: int = 0, func: str = "product"):
        self.port = port or free_port()
        ctx = multiprocessing.get_context("spawn")
        self._ready = ctx.Event()
        self._proc = ctx.Process(
            target=_serve, args=(self.port, n_clients, func, self._ready), daemon=True
        )

    def start(self, timeout: float = 60.0) -> "ServerProcess":
        self._proc.start()
        if not self._ready.wait(timeout):
            self.terminate()
            raise RuntimeError("server did not come up")
        return self

    def terminate(self) -> None:
        if self._proc.is_alive():
            self._proc.terminate()
        self._proc.join(10)

    def __enter__(self):
        return self.start()

    def __exit__(self, *exc):
        self.terminate()


def start_fleet(loads: Sequence[int]):
    servers = [ServerProcess(n_clients=n) for n in loads]
    for s in servers:
        s._proc.start()
    deadline = time.time() + 90
    for s in servers:
        if not s._ready.wait(max(0.1, deadline - time.time())):
            for t in servers:
                t.terminate()
            raise RuntimeError("fleet did not come up")
    return servers


def run_product_queries(client, n: int = 50) -> bool:
    rng = np.random.default_rng()
    try:
        for _ in range(n):
            a, b = rng.integers(0, 50, size=2)
            (prod,) = client.evaluate(a, b)
            assert prod == a * b
    except Exception:
        import traceback

        traceback.print_exc()
        return False
    return True


class ProductTester:
    def __init__(self, client) -> None:
        self.client = client

    def run(self, n: int) -> bool:
        return run_product_queries(self.client, n)


def fork_pool_scenario(port: int) -> None:
    """Runs in a FRESH interpreter (see test_client_multiprocessing): a picklable client is handed to
    fork()-ed pool workers before gRPC was ever initialised in the parent."""
    import multiprocessing

    from pytensor_federated_b200 import service

    ctx = multiprocessing.get_context("fork")
    client = service.ArraysToArraysServiceClient("127.0.0.1", port)
    tester = ProductTester(client)
    with ctx.Pool(processes=3) as pool:
        assert all(pool.map(run_product_queries, [client] * 4))
    with ctx.Pool(processes=3) as pool:
        assert all(pool.map(tester.run, [25] * 4))
    print("FORK-OK", flush=True)
