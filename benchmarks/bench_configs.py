"""Secondary benchmarks for the other BASELINE.json configurations (single process, GPU 0..N-1 via
the in-process launcher is not used here: these are per-GPU numbers at N = 1 unless torchrun is used).

    python benchmarks/bench_configs.py --out configs.jsonl

Each line: config name, backend (fused | collective = stock PyTorch eager + (no-op) collectives),
evals/s measured end to end through ``FederatedEngine.evaluate`` (pinned H2D theta, D2H result),
and the mean latency per evaluation.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def timed(engine, thetas, warmup=20):
    for th in thetas[:warmup]:
        engine.evaluate(*th)
    t0 = time.perf_counter()
    for th in thetas[warmup:]:
        engine.evaluate(*th)
    dt = time.perf_counter() - t0
    n = len(thetas) - warmup
    return n / dt, 1e6 * dt / n


def main():
    import torch

    from pytensor_federated_b200.federation import NodeFederation
    from pytensor_federated_b200.models import (
        Fp8GlmShards, LinregShards, OdeShards, make_demo_data, synth_logistic_shard_fp8, synth_lv_shard,
    )
    from pytensor_federated_b200.parallel import FederatedEngine
    from pytensor_federated_b200.sampling import Model, nuts_sample

    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--fp8-rows", type=int, default=10_000_000)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    lines = []

    def emit(**kw):
        lines.append(kw)
        print(json.dumps(kw), flush=True)

    # 1) the reference's demo model: 8 shards of 10 rows, evaluation latency
    x, y, sigma = make_demo_data()
    for backend in ("fused", "collective"):
        model = LinregShards([x] * 8, [y] * 8, [sigma] * 8, device=dev)
        with FederatedEngine(model, backend=backend) as eng:
            thetas = [(rng.normal(size=8), np.asarray(rng.normal())) for _ in range(2020)]
            rate, lat = timed(eng, thetas)
            emit(config="linreg demo model, 8 shards x 10 rows, 1 GPU", backend=backend, evals_per_s=rate, latency_us=lat)

    # 2) NUTS driving the fused federated Ops (hierarchical demo model, 8 nodes)
    model = LinregShards([x] * 8, [y] * 8, [sigma] * 8, device=dev)
    fed = NodeFederation(FederatedEngine(model))
    ops = fed.node_ops()
    m = Model()
    mu = m.Normal("intercept_mu", 0.0, 1.0)
    icpt = m.Normal("intercept", mu, 0.1, size=8)
    slope = m.Normal("slope", 0.0, 1.0)
    for i, off in enumerate(np.linspace(-4, 4, 8)):
        logp, *_ = ops[i](icpt[i] + off, slope)
        m.Potential(f"p{i}", logp)
    m.compile()
    t0 = time.perf_counter()
    res = nuts_sample(m.logp_dlogp, np.zeros(m.dim), draws=200, tune=300, seed=1)
    dt = time.perf_counter() - t0
    emit(config="hierarchical linreg, 8 federated nodes, NUTS tune=300 draws=200 (graph + sampler in Python)",
         backend="fused", model_evals_per_s=res.n_logp_evals / dt, node_evals_per_s=8 * res.n_logp_evals / dt,
         engine_launches=fed.n_launches, n_logp_evals=res.n_logp_evals, divergences=res.divergences)
    fed.shutdown()

    # 3) ODE parameter estimation: 4 shards x 20k series x 32 time points
    shards = [synth_lv_shard(20_000, 32, seed=s, device=dev) for s in range(4)]
    ode = OdeShards([s[0] for s in shards], [s[1] for s in shards], [s[2] for s in shards], [s[3] for s in shards])
    th = [(np.array([1.0, 0.4, 0.8, 0.2]) + 0.01 * rng.normal(size=4),) for _ in range(120)]
    with FederatedEngine(ode) as eng:
        rate, lat = timed(eng, th, warmup=20)
        emit(config="Lotka-Volterra ODE, 4 shards x 20k series x 32 obs, RK4 x8 + sensitivities, 1 GPU", backend="fused",
             evals_per_s=rate, latency_us=lat)

    # 4) hierarchical GLM, block-scaled fp8, 8 groups (one per shard) on ONE GPU
    Xs, scs, ys = [], [], []
    for s in range(8):
        Xq, sc, yy = synth_logistic_shard_fp8(args.fp8_rows, 256, seed=1000 + s, device=dev)
        Xs.append(Xq); scs.append(sc); ys.append(yy)
    model = Fp8GlmShards(Xs, scs, ys, groups=list(range(8)), n_groups=8)
    with FederatedEngine(model, timeout=60) as eng:
        thetas = [(rng.normal(size=8).astype(np.float32) * 0.1, rng.normal(size=256).astype(np.float32) * 0.02) for _ in range(45)]
        rate, lat = timed(eng, thetas, warmup=5)
        emit(config=f"hierarchical logistic GLM, 8 groups x {args.fp8_rows} x 256, fp8 block-scaled, 1 GPU", backend="fused",
             evals_per_s=rate, latency_us=lat, hbm_bytes_per_eval=model.bytes_per_eval(),
             hbm_tb_per_s=model.bytes_per_eval() * rate / 1e12)
    # 5) sampling throughput: lock-step HMC, K chains per fused launch (tensor-core kernel) vs K = 1
    from pytensor_federated_b200.models import GlmShards, synth_logistic_shard
    from pytensor_federated_b200.sampling import glm_batch_fn, hmc_sample_batched

    Xs, ys = [], []
    for s in range(8):
        X, yy, _ = synth_logistic_shard(1_000_000, 256, seed=2000 + s, device=dev)
        Xs.append(X); ys.append(yy)
    for K in (1, 16):
        with FederatedEngine(GlmShards(Xs, ys, n_chains=K, kernel="tc"), timeout=60) as eng:
            t0 = time.perf_counter()
            res = hmc_sample_batched(glm_batch_fn(eng, 1), np.zeros((K, 257)), draws=20, tune=20, n_leapfrog=8,
                                     step_size=2e-4, seed=1)
            dt = time.perf_counter() - t0
            emit(config="lock-step HMC on logistic GLM 8 x 1M x 256 (bf16), 1 GPU", chains=K, backend="fused",
                 fused_launches=res.n_batched_evals, leapfrog_steps_per_s=K * res.n_batched_evals / dt,
                 launches_per_s=res.n_batched_evals / dt, accept_rate=float(res.accept_rate.mean()))
    if args.out:
        with open(args.out, "a") as fh:
            for l in lines:
                fh.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
