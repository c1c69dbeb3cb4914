"""The reference's demo — a hierarchical linear regression whose likelihood terms live on federated nodes —
written the two ways this package offers, on N nodes (GPUs, or CPU processes for a dry run):

    python examples/hierarchical_linreg.py --nodes 8 --draws 300

1. one `FederatedLogpGradOp` per node, as in the reference (`demo_model.py:28-36`): the
   `fuse_asyncs` rewrite answers all of them with ONE fused launch per model evaluation;
2. ONE Op for the whole federation (`NodeFederation.all_nodes_op`): vector of node intercepts in, summed
   log-likelihood and per-node gradients out — the graph no longer grows with the number of nodes.

On GPUs the root also keeps the next evaluation's kernel enqueued before the sampler has produced theta
(`speculative_us`, `docs/PROTOCOL.md`).
"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


class Shards:
    """Picklable model factory: node r of `world` holds the shards r, r + world, ... (private data of that node)."""

    def __init__(self, n: int) -> None:
        self.n = n

    def __call__(self, rank: int, world: int, device):
        from pytensor_federated_b200.models import LinregShards

        mine = [s for s in range(self.n) if s % world == rank]
        xs, ys = [], []
        for s in mine:
            rng = np.random.default_rng(1000 + s)
            x = np.linspace(0, 10, 25)
            xs.append(x)
            ys.append(1.0 + 0.3 * s + 0.5 * x + rng.normal(scale=0.4, size=x.size))   # node s: intercept 1 + 0.3 s
        return LinregShards(xs, ys, [0.4] * len(mine), local_ids=mine, n_shards_total=self.n, device=device)


def build(fed, n, one_op):
    from pytensor_federated_b200.graph import core as at
    from pytensor_federated_b200.sampling import Model

    m = Model()
    mu = m.Normal("intercept_mu", 0.0, 5.0)
    icpt = m.Normal("intercept", mu, 2.0, size=n)
    slope = m.Normal("slope", 0.0, 2.0)
    if one_op:
        logp, *_ = fed.all_nodes_op()(icpt, slope)
        m.Potential("likelihood", logp)
    else:
        for i, op in enumerate(fed.node_ops()):
            logp, *_ = op(icpt[i], slope)
            m.Potential(f"likelihood_{i}", logp)
    m.compile()
    return m


def main():
    import torch

    from pytensor_federated_b200.federation import NodeFederation, launch_federation
    from pytensor_federated_b200.sampling import nuts_sample

    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=4)
    ap.add_argument("--gpus", type=int, default=0, help="processes / GPUs to spread the nodes over (0 = all visible, or 1 on CPU)")
    ap.add_argument("--draws", type=int, default=200)
    args = ap.parse_args()

    visible = torch.cuda.device_count() if torch.cuda.is_available() else 0
    world = max(1, min(args.nodes, args.gpus or visible or 1))
    with launch_federation(Shards(args.nodes), world, device_type="cuda" if visible else "cpu",
                           backend="auto" if visible else "collective", speculative_us=1000.0) as engine:
        fed = NodeFederation(engine)
        print(f"{args.nodes} nodes on {world} {'GPU(s)' if visible else 'CPU process(es)'}, backend={engine.backend}, "
              f"speculative launches: {engine.speculative}")
        for one_op in (False, True):
            m = build(fed, args.nodes, one_op)
            fed.n_launches = 0
            t0 = time.perf_counter()
            res = nuts_sample(m.logp_dlogp, np.zeros(m.dim), draws=args.draws, tune=args.draws, seed=3)
            dt = time.perf_counter() - t0
            post = m.point(res.samples.mean(0))
            print(f"{'one Op for the federation' if one_op else 'one Op per node':>26}: "
                  f"{len(m._compiled.maker.fgraph.toposort()):3d} graph nodes, {res.n_logp_evals} model evaluations = "
                  f"{fed.n_launches} fused launches in {dt:.2f} s ({res.n_logp_evals / dt:.0f}/s); "
                  f"slope = {float(post['slope']):.2f}, intercepts = {np.round(post['intercept'], 1).tolist()}")


if __name__ == "__main__":
    main()
