"""Federated parameter estimation for YOUR ODE — the use case the reference's README sketches
(`README.md:39-52`: the data and the solver stay on the node, only theta and [LL, dLL/dtheta] travel).

    python examples/custom_ode.py [--series 2000] [--nodes 3]

The right-hand side is written once in CUDA C (for the fused kernel; forward-mode dual numbers give the
sensitivities, no Jacobians) and once in PyTorch (oracle / CPU path).  Every node holds its own time series; the
nodes are given their own Ops, exactly like the reference's demo_model.py gives every gRPC worker its own Op, and the
MAP estimate is found from the summed log-potentials — one fused launch per model evaluation.  On a machine
without a GPU the same script runs through the eager oracle.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch

    from pytensor_federated_b200._graph_backend import at
    from pytensor_federated_b200.federation import NodeFederation
    from pytensor_federated_b200.models import OdeShards, OdeSystem, synth_ode_shard
    from pytensor_federated_b200.parallel import FederatedEngine
    from pytensor_federated_b200.sampling import Model

    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=2000, help="observed time series per node")
    ap.add_argument("--nodes", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda:0" if torch.cuda.is_available() else "cpu")

    # SIR epidemic: S' = -b S I, I' = b S I - g I, R' = g I ; theta = (b, g)
    sir = OdeSystem(
        "const auto inf = th[0] * y[0] * y[1]; dy[0] = -inf; dy[1] = inf - th[1] * y[1]; dy[2] = th[1] * y[1];",
        lambda y, th, t: (-th[0] * y[0] * y[1], th[0] * y[0] * y[1] - th[1] * y[1], th[1] * y[1]),
        n_states=3, n_params=2, name="sir",
    )
    truth = np.array([1.8, 0.5])
    rng = np.random.default_rng(0)
    shards = []
    for node in range(args.nodes):
        i0 = rng.uniform(0.02, 0.2, size=args.series)
        y0 = np.stack([1.0 - i0, i0, np.zeros(args.series)])
        shards.append(synth_ode_shard(sir, truth, y0, 10, seed=node, device=dev, sigma=0.02, t_end=6.0))
    model = OdeShards([s[0] for s in shards], [s[1] for s in shards], [s[2] for s in shards], [s[3] for s in shards],
                      system=sir, node_ids=list(range(args.nodes)), n_nodes=args.nodes)
    fed = NodeFederation(FederatedEngine(model))

    m = Model()
    log_theta = m.Normal("log_theta", 0.0, 1.0, size=2)       # positive rates, sampled on the log scale
    theta = at.exp(log_theta)
    for op in fed.node_ops():                                  # one Op per node; fused into ONE launch per evaluation
        m.Potential(f"node{op.node}", op(theta)[0])
    point, info = m.find_map(start=np.log(np.array([1.0, 1.0])))
    print(f"{args.nodes} nodes x {args.series} series on {dev.type}: MAP theta = {np.exp(point['log_theta']).round(4)} "
          f"(truth {truth}), {info['n_evals']} model evaluations = {fed.n_launches} fused launches")
    fed.shutdown()


if __name__ == "__main__":
    main()
