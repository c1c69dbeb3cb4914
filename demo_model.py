"""Client-side demo: a hierarchical linear model over N federated nodes, MAP + NUTS.

Same model as the reference's ``demo_model.py`` (``demo_model.py:24-44``):
``intercept_mu ~ N(0,1)``, ``intercept[i] ~ N(intercept_mu, 0.1)``, ``slope ~ N(0,1)`` and one
remote log-likelihood per node with offset intercepts, each entering as a potential.

Three ways to reach the nodes:

* ``--host/--ports`` (default): gRPC to ``demo_node.py`` workers — the reference's topology; with
  ``--parallel true`` the async Ops are fused into one concurrent fan-out.
* ``--fused N``: the nodes are N data shards resident on this machine's GPUs (CPU when none), spread over
  ``--gpus M`` of them (default: all visible, at most N; one process per GPU is started for you); the fused
  graph node answers all N remote calls with ONE kernel launch per GPU.
* PyMC available: pass ``--pymc`` to sample with ``pm.sample`` instead of the in-repo NUTS.
"""
import argparse
import logging
import time
from typing import Sequence

import numpy as np

_log = logging.getLogger("demo_model")


def build_model(remote_ops, n: int):
    from pytensor_federated_b200.sampling import Model

    m = Model()
    intercept_mu = m.Normal("intercept_mu", 0.0, 1.0)
    intercept = m.Normal("intercept", intercept_mu, 0.1, size=n)
    slope = m.Normal("slope", 0.0, 1.0)
    for i, off in enumerate(np.linspace(-n / 2, n / 2, n)):
        logp, *_ = remote_ops[i](intercept[i] + off, slope)
        m.Potential(f"potential_{i}", logp)
    return m


def run_model(remote_ops, n: int, tune: int, draws: int, chains: int = 1):
    from pytensor_federated_b200.sampling import find_map, nuts_sample, summarize

    m = build_model(remote_ops, n)
    m.compile()
    _log.info("Running MAP estimation")
    t0 = time.perf_counter()
    theta_map, info = find_map(m.logp_dlogp, np.zeros(m.dim))
    print({k: np.round(v, 4) for k, v in m.point(theta_map).items()}, info)
    res = nuts_sample(m.logp_dlogp, theta_map, draws=draws, tune=tune, seed=1234)
    dt = time.perf_counter() - t0
    for name, row in res.summary(m.names()).items():
        print(f"{name:>16s}  mean {row['mean']:8.4f}  sd {row['sd']:7.4f}  ess {row['ess']:7.1f}")
    print(f"{res.n_logp_evals} logp+grad evaluations in {dt:.2f} s "
          f"({res.n_logp_evals / dt:.0f} model evals/s, {n * res.n_logp_evals / dt:.0f} node evals/s); "
          f"accept {res.accept_rate:.2f}, divergences {res.divergences}")
    if chains > 1:  # further chains (the reference's pm.sample runs 4) and the cross-chain diagnostics
        _, cols = m.sample(draws=draws, tune=tune, chains=chains, start=theta_map, seed=1234)
        for name, row in summarize(cols).items():
            print(f"{name:>16s}  mean {row['mean']:8.4f}  sd {row['sd']:7.4f}  ess {row['ess']:7.1f}  rhat {row['rhat']:.3f}")
    return res


def run_model_pymc(remote_ops, n: int, tune: int, draws: int):
    """The same model through PyMC (needs PyMC + PyTensor; the Ops are then genuine PyTensor Ops).

    Mirrors ``demo_model.py:28-44``; not executable in the offline image.
    """
    import arviz
    import pymc as pm

    with pm.Model():
        intercept_mu = pm.Normal("intercept_mu")
        intercept = pm.Normal("intercept", intercept_mu, sigma=0.1, size=n)
        slope = pm.Normal("slope")
        for i, off in enumerate(np.linspace(-n / 2, n / 2, n)):
            logp, *_ = remote_ops[i](intercept[i] + off, slope)
            pm.Potential(f"potential_{i}", var=logp)
        _log.info("Running MAP estimation")
        print(pm.find_MAP())
        idata = pm.sample(tune=tune, draws=draws)
        print(arviz.summary(idata))
    return idata


def remote_ops_grpc(host: str, ports: Sequence[int], n: int, use_async: bool):
    from pytensor_federated_b200 import AsyncLogpGradOp, LogpGradOp, LogpGradServiceClient

    client = LogpGradServiceClient(hosts_and_ports=[(host, p) for p in ports])
    op = AsyncLogpGradOp(client.evaluate_async) if use_async else LogpGradOp(client.evaluate)
    return [op] * n, client


class _DemoShards:
    """Picklable model factory for ``launch_federation``: rank r of `world` holds the demo shards r, r + world, ..."""

    def __init__(self, n: int) -> None:
        self.n = n

    def __call__(self, rank: int, world: int, device):
        from pytensor_federated_b200.models import LinregShards, make_demo_data

        x, y, sigma = make_demo_data()   # identical "remote" datasets, like the reference demo
        mine = [s for s in range(self.n) if s % world == rank]
        return LinregShards([x] * len(mine), [y] * len(mine), [sigma] * len(mine), local_ids=mine, n_shards_total=self.n,
                            device=device)


def remote_ops_fused(n: int, gpus: int = 0):
    """N shards on min(N, visible GPUs) GPUs (``gpus`` overrides): one process per GPU, shard s on GPU s % M."""
    import contextlib

    import torch

    from pytensor_federated_b200.federation import NodeFederation, launch_federation

    visible = torch.cuda.device_count() if torch.cuda.is_available() else 0
    world = max(1, min(n, gpus or visible or 1))
    stack = contextlib.ExitStack()
    engine = stack.enter_context(launch_federation(_DemoShards(n), world, device_type="cuda" if visible else "cpu",
                                                   backend="auto" if visible else "collective"))
    _log.info("%d shards on %d %s", n, world, "GPU(s), fused NVLink data plane" if visible else "CPU process(es)")
    fed = NodeFederation(engine)
    fed.shutdown = lambda: (fed.unregister_services(), stack.close())   # the launcher joins the peer processes
    return fed.node_ops(), fed


if __name__ == "__main__":
    logging.basicConfig(level=logging.INFO)
    parser = argparse.ArgumentParser(description="Runs the hierarchical demo model against federated nodes.")
    parser.add_argument("--host", default="127.0.0.1")
    parser.add_argument("--ports", default=",".join(map(str, range(50000, 50003))), type=str)
    parser.add_argument("--parallel", default="true", choices=["true", "false"])
    parser.add_argument("--fused", default=0, type=int, help="use N on-box shards instead of gRPC workers")
    parser.add_argument("--gpus", default=0, type=int, help="--fused: GPUs (processes) to spread the shards over; 0 = all visible")
    parser.add_argument("--nodes", default=3, type=int, help="remote calls per model evaluation")
    parser.add_argument("--tune", default=500, type=int)
    parser.add_argument("--draws", default=200, type=int)
    parser.add_argument("--chains", default=1, type=int, help="> 1: run further chains and print ESS / R-hat")
    parser.add_argument("--pymc", action="store_true", help="sample with PyMC instead of the in-repo NUTS")
    args, _ = parser.parse_known_args()
    runner = run_model_pymc if args.pymc else (lambda *a: run_model(*a, chains=args.chains))
    if args.fused:
        ops, handle = remote_ops_fused(args.fused, args.gpus)
        runner(ops, args.fused, args.tune, args.draws)
        handle.shutdown()
    else:
        ops, handle = remote_ops_grpc(args.host, [int(p) for p in args.ports.split(",")], args.nodes,
                                      args.parallel.lower() == "true")
        runner(ops, args.nodes, args.tune, args.draws)
