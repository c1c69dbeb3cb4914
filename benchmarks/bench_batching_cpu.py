"""Dynamic batching over gRPC with a SYNTHETIC kernel cost model (CPU only, no GPU involved).

A node whose evaluator costs ``--launch-ms`` per launch *regardless of how many chains ride in it* — the
cost model of the multi-chain tensor-core kernel, where the design matrix is streamed once per launch —
is driven by C concurrent clients, with and without :class:`DynamicBatcher`.  This isolates what the
batcher and the gRPC path add; the real kernel numbers come from ``examples/batched_serving.py`` on an H100.

    python benchmarks/bench_batching_cpu.py [--chains 8] [--launch-ms 2.0] [--out results.jsonl]
"""
import argparse
import asyncio
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run(chains: int, evals: int, launch_ms: float, batching: bool) -> dict:
    from pytensor_federated_b200 import ArraysToArraysService, ArraysToArraysServiceClient
    from pytensor_federated_b200.batching import DynamicBatcher, stacked_compute_func
    from pytensor_federated_b200.rpc import Server
    from pytensor_federated_b200.utils import get_useful_event_loop

    launches = [0]

    def evaluate(theta):                       # [K, D] -> logp[K], grad[K, D]; fixed cost per launch
        launches[0] += 1
        t_end = time.perf_counter() + launch_ms * 1e-3
        while time.perf_counter() < t_end:
            pass
        return [-0.5 * np.sum(theta * theta, axis=1), -theta]

    if batching:
        compute = DynamicBatcher(stacked_compute_func(evaluate, max_batch=chains), max_batch=chains, max_delay=0.0003)
    else:
        def compute(theta):
            logp, grad = evaluate(theta[None, :])
            return [logp[0], grad[0]]

    loop = get_useful_event_loop()
    server = Server([ArraysToArraysService(compute)])
    port = loop.run_until_complete(server.start("127.0.0.1", 0))
    clients = [ArraysToArraysServiceClient("127.0.0.1", port) for _ in range(chains)]
    thetas = np.random.default_rng(0).normal(size=(chains, 256))

    async def chain(i, n):
        for _ in range(n):
            await clients[i].evaluate_async(thetas[i])

    async def timed():
        await asyncio.gather(*[chain(i, 5) for i in range(chains)])       # connect + warm up
        launches[0] = 0
        t0 = time.perf_counter()
        await asyncio.gather(*[chain(i, evals) for i in range(chains)])
        return time.perf_counter() - t0

    dt = loop.run_until_complete(timed())
    del clients
    if batching:
        loop.run_until_complete(compute.close())
    loop.run_until_complete(server.close(None))
    total = chains * evals
    return {"chains": chains, "batching": batching, "launch_ms": launch_ms, "chain_evals_per_s": total / dt,
            "launches": launches[0], "requests": total, "data": "synthetic cost model, CPU, loopback gRPC"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--evals", type=int, default=200)
    ap.add_argument("--launch-ms", type=float, default=2.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    os.environ.setdefault("B200FED_CONNECT_SLEEP", "0,0")
    rows = []
    for c in args.chains:
        for batching in (False, True):
            row = run(c, args.evals, args.launch_ms, batching)
            rows.append(row)
            print(json.dumps(row))
    if args.out:
        with open(args.out, "a") as fh:
            for row in rows:
                fh.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
