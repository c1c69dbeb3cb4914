"""Chains in separate PROCESSES -> gRPC -> one GPU node, with and without dynamic batching.

The reference's deployment: every chain of a sampler is a process with its own connection to the node
(``pytensor_federated/service.py:266-275``, ``test_wrapper_ops.py:305-317``), and the node
answers the requests one after the other.  Here the node puts the requests that are waiting into ONE
multi-chain launch of the tensor-core GLM kernel (``DynamicBatcher`` + ``GlmShards(n_chains=K)``).

    python benchmarks/bench_batching_gpu.py --chains 8 16 --evals 300 --out results.jsonl

One JSON line per (chains, mode): aggregate chain-evaluations per second measured in the client processes
(start barrier -> last client done), launches used, mean batch size.
"""
import argparse
import asyncio
import json
import multiprocessing
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def chain_process(port: int, index: int, features: int, evals: int, warmup: int, barrier, out_queue) -> None:
    """One MCMC chain: its own process, its own gRPC stream, evaluations strictly one after the other."""
    os.environ.setdefault("B200FED_CONNECT_SLEEP", "0,0")
    from pytensor_federated_b200 import ArraysToArraysServiceClient

    rng = np.random.default_rng(100 + index)
    client = ArraysToArraysServiceClient("127.0.0.1", port)
    ic = np.zeros(1, dtype=np.float32)
    betas = (rng.normal(size=(evals + warmup, features)) * 0.02).astype(np.float32)
    for i in range(warmup):
        client.evaluate(ic, betas[i])
    barrier.wait()
    t0 = time.perf_counter()
    last = None
    for i in range(evals):
        last = client.evaluate(ic, betas[warmup + i])
    dt = time.perf_counter() - t0
    out_queue.put((index, t0, t0 + dt, float(np.asarray(last[0]).reshape(-1)[0])))
    del client


def serve_in_thread(compute):
    """The node's gRPC server on its own event loop in a background thread; returns (port, stop())."""
    from pytensor_federated_b200 import ArraysToArraysService
    from pytensor_federated_b200.rpc import Server

    ready = threading.Event()
    state = {}

    async def node():
        server = Server([ArraysToArraysService(compute)], tls=False)
        state["port"] = await server.start("127.0.0.1", 0)
        state["stop"] = asyncio.Event()
        ready.set()
        await state["stop"].wait()
        if hasattr(compute, "close"):   # the batcher's worker task lives on this loop
            await compute.close()
        await server.close(1.0)

    def run():
        loop = asyncio.new_event_loop()
        asyncio.set_event_loop(loop)
        state["loop"] = loop
        loop.run_until_complete(node())

    thread = threading.Thread(target=run, daemon=True)
    thread.start()
    ready.wait(60)

    def stop():
        state["loop"].call_soon_threadsafe(state["stop"].set)
        thread.join(30)

    return state["port"], stop


def main() -> None:
    import torch

    from pytensor_federated_b200.batching import DynamicBatcher, stacked_compute_func
    from pytensor_federated_b200.models import GlmShards, synth_logistic_shard
    from pytensor_federated_b200.parallel import FederatedEngine

    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=256)
    ap.add_argument("--chains", type=int, nargs="+", default=[8, 16])
    ap.add_argument("--evals", type=int, default=300, help="timed evaluations per chain")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--max-delay", type=float, default=0.0002)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    cuda = torch.cuda.is_available()
    dev = torch.device("cuda", 0) if cuda else torch.device("cpu")
    rows = args.rows if cuda else min(args.rows, 20_000)
    X, y, _ = synth_logistic_shard(rows, args.features, seed=1, device=dev)
    ctx = multiprocessing.get_context("spawn")
    lines = []
    for chains in args.chains:
        for batching in (False, True):
            K = chains if batching else 1
            engine = FederatedEngine(GlmShards([X], [y], n_chains=K, kernel="auto" if cuda else "simt"), timeout=60.0)
            if batching:
                compute = DynamicBatcher(stacked_compute_func(engine.evaluate, max_batch=K), max_batch=K,
                                         max_delay=args.max_delay)
            else:
                compute = engine.evaluate
            port, stop = serve_in_thread(compute)
            barrier = ctx.Barrier(chains)
            q = ctx.Queue()
            procs = [ctx.Process(target=chain_process, args=(port, i, args.features, args.evals, args.warmup, barrier, q))
                     for i in range(chains)]
            for p in procs:
                p.start()
            results = [q.get(timeout=900) for _ in procs]
            for p in procs:
                p.join(60)
            launches = engine.kernel_launches if cuda else None
            span = max(r[2] for r in results) - min(r[1] for r in results)
            total = chains * args.evals
            line = {
                "config": f"{chains} chain processes -> gRPC -> 1 GPU node, logistic GLM {rows} x {args.features} bf16",
                "chains": chains, "batching": batching, "chains_per_launch_capacity": K, "evals_per_chain": args.evals,
                "chain_evals_per_s": total / span, "seconds": span,
                "mean_batch": (compute.n_requests / max(compute.n_batches, 1)) if batching else 1.0,
                "launches_total_incl_warmup": launches, "requests_total_incl_warmup": chains * (args.evals + args.warmup),
                "device": dev.type,
            }
            print(json.dumps(line), flush=True)
            lines.append(line)
            stop()
            engine.shutdown()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)) or ".", exist_ok=True)
        with open(args.out, "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
