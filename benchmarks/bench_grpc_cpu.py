"""BASELINE.json config 1: the demo linear regression behind 2 gRPC workers on CPU over loopback.

Runs the SAME numpy model behind (a) the unmodified reference's ArraysToArraysService (baseline/_ref
+ dependency shims) and (b) this package's service, and times the reference-style client calls:
sequential ``evaluate`` and the ``asyncio.gather`` fan-out of a fused graph node.  CPU only.

    python benchmarks/bench_grpc_cpu.py [--out results.jsonl]
"""
import argparse
import asyncio
import json
import os
import subprocess
import sys
import textwrap
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

SERVER = textwrap.dedent(
    """
    import asyncio, sys
    import numpy as np
    impl, port = sys.argv[1], int(sys.argv[2])
    x = np.linspace(0, 10, 10); sigma = 0.4
    y = np.random.RandomState(123).normal(1.5 + 0.5 * x, scale=sigma)
    def model(a, b):
        r = y - (a + b * x)
        return (np.asarray(-0.5 * np.sum(r * r) / sigma**2 - 10 * np.log(sigma * np.sqrt(2 * np.pi))),
                [np.asarray(np.sum(r) / sigma**2), np.asarray(np.sum(r * x) / sigma**2)])
    if impl == "reference":
        import grpclib.server
        from pytensor_federated import ArraysToArraysService, wrap_logp_grad_func
        Server = grpclib.server.Server
    else:
        from pytensor_federated_b200 import ArraysToArraysService, wrap_logp_grad_func
        from pytensor_federated_b200.rpc import Server
    async def main():
        server = Server([ArraysToArraysService(wrap_logp_grad_func(model))])
        await server.start("127.0.0.1", port)
        print("READY", flush=True)
        await server.wait_closed()
    asyncio.new_event_loop().run_until_complete(main())
    """
)


def run(impl: str, n_workers: int, n_evals: int):
    from _helpers import free_port

    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(ROOT, "baseline", "shims"), os.path.join(ROOT, "baseline", "_ref"), ROOT])
    ports = [free_port() for _ in range(n_workers)]
    procs = [subprocess.Popen([sys.executable, "-c", SERVER, impl, str(p)], env=env, stdout=subprocess.PIPE, text=True) for p in ports]
    try:
        for p in procs:
            assert p.stdout.readline().strip() == "READY"
        if impl == "reference":
            sys.path[:0] = [os.path.join(ROOT, "baseline", "shims"), os.path.join(ROOT, "baseline", "_ref")]
            from pytensor_federated import LogpGradServiceClient
        else:
            from pytensor_federated_b200 import LogpGradServiceClient
        clients = [LogpGradServiceClient("127.0.0.1", p) for p in ports]
        a, b = np.array(0.4), np.array(1.2)
        for c in clients:
            c.evaluate(a, b)
        t0 = time.perf_counter()
        for _ in range(n_evals):
            for c in clients:
                c.evaluate(a, b)
        seq = time.perf_counter() - t0

        async def fan_out():
            return await asyncio.gather(*[c.evaluate_async(a, b) for c in clients])

        loop = asyncio.new_event_loop()
        asyncio.set_event_loop(loop)
        clients2 = [LogpGradServiceClient("127.0.0.1", p) for p in ports]
        loop.run_until_complete(fan_out.__call__()) if False else None
        clients = clients2
        loop.run_until_complete(fan_out())
        t0 = time.perf_counter()
        for _ in range(n_evals):
            loop.run_until_complete(fan_out())
        par = time.perf_counter() - t0
        del clients, clients2
        return {"impl": impl, "workers": n_workers, "evals": n_evals,
                "sequential_model_evals_per_s": n_evals / seq, "sequential_us_per_node_call": 1e6 * seq / (n_evals * n_workers),
                "gather_model_evals_per_s": n_evals / par, "gather_us_per_model_eval": 1e6 * par / n_evals}
    finally:
        for p in procs:
            p.terminate()
        for p in procs:
            p.wait(10)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--evals", type=int, default=2000)
    ap.add_argument("--impl", default="both")
    args = ap.parse_args()
    impls = ["product", "reference"] if args.impl == "both" else [args.impl]
    for impl in impls:
        # separate interpreter per implementation: both packages patch the event loop / grpc state
        if args.impl == "both":
            res = subprocess.run([sys.executable, __file__, "--impl", impl, "--evals", str(args.evals)] +
                                 (["--out", args.out] if args.out else []), cwd=ROOT)
            continue
        line = run(impl, 2, args.evals)
        line["config"] = "demo linear regression, 2 gRPC workers on CPU over loopback"
        print(json.dumps(line), flush=True)
        if args.out:
            with open(args.out, "a") as fh:
                fh.write(json.dumps(line) + "\n")
