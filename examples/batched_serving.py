"""One GPU node serving several MCMC chains (= clients) with dynamic batching.

    python examples/batched_serving.py --chains 4 --evals 200 [--no-batching]

Starts a gRPC node whose compute function is a K-chain `FederatedEngine(GlmShards(..., n_chains=K))`
behind a `DynamicBatcher`, then drives it with `--chains` concurrent clients the way independent chains of
a sampler would.  Requests that arrive together ride in ONE fused launch (chains sit on the MMA N axis of
the tensor-core kernel), so the node's throughput grows with the number of chains instead of being divided
by it.  `--no-batching` serves the same clients one request per launch for comparison.  Runs on CPU too
(eager baseline kernel), where it only demonstrates the plumbing.
"""
import argparse
import asyncio
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch

    from pytensor_federated_b200 import ArraysToArraysService, ArraysToArraysServiceClient
    from pytensor_federated_b200.batching import DynamicBatcher, stacked_compute_func
    from pytensor_federated_b200.models import GlmShards, synth_logistic_shard
    from pytensor_federated_b200.parallel import FederatedEngine
    from pytensor_federated_b200.rpc import Server
    from pytensor_federated_b200.utils import get_useful_event_loop

    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--features", type=int, default=256)
    ap.add_argument("--chains", type=int, default=4)
    ap.add_argument("--evals", type=int, default=100, help="evaluations per chain")
    ap.add_argument("--no-batching", action="store_true")
    args = ap.parse_args()
    os.environ.setdefault("B200FED_CONNECT_SLEEP", "0,0")

    cuda = torch.cuda.is_available()
    dev = torch.device("cuda", 0) if cuda else torch.device("cpu")
    rows = args.rows if cuda else min(args.rows, 20_000)
    X, y, _ = synth_logistic_shard(rows, args.features, seed=1, device=dev)
    K = 1 if args.no_batching else args.chains
    engine = FederatedEngine(GlmShards([X], [y], n_chains=K, kernel="auto" if cuda else "simt"))

    if args.no_batching:
        compute = engine.evaluate                              # (intercept[1], beta[P]) per request
    else:
        compute = DynamicBatcher(stacked_compute_func(engine.evaluate, max_batch=K), max_batch=K, max_delay=0.0003)

    loop = get_useful_event_loop()
    server = Server([ArraysToArraysService(compute)])
    port = loop.run_until_complete(server.start("127.0.0.1", 0))
    clients = [ArraysToArraysServiceClient("127.0.0.1", port) for _ in range(args.chains)]
    rng = np.random.default_rng(0)
    betas = (rng.normal(size=(args.chains, args.features)) * 0.02).astype(np.float32)

    async def chain(i):
        out = None
        for _ in range(args.evals):
            out = await clients[i].evaluate_async(np.zeros(1, dtype=np.float32), betas[i])
        return out

    async def run():
        await asyncio.gather(*[chain(i) for i in range(args.chains)])      # warm-up (connects the streams)
        t0 = time.perf_counter()
        outs = await asyncio.gather(*[chain(i) for i in range(args.chains)])
        return outs, time.perf_counter() - t0

    launches0 = engine.kernel_launches
    outs, dt = loop.run_until_complete(run())
    total = args.chains * args.evals
    launches = (engine.kernel_launches - launches0) / 2 if cuda else float("nan")   # warm-up + timed run
    print(f"{args.chains} chains x {args.evals} evals on {dev.type}: {total / dt:.0f} chain-evals/s over gRPC, "
          f"{'no batching' if args.no_batching else f'dynamic batching (K={K})'}; "
          f"~{launches:.0f} launches for {total} requests; logp[0] = {float(outs[0][0]):.3f}")
    del clients
    if not args.no_batching:
        loop.run_until_complete(compute.close())
    loop.run_until_complete(server.close(None))
    engine.shutdown()


if __name__ == "__main__":
    main()
