"""Rate of the right-censored survival families against the families with the same MMA shapes and bytes (one GPU).

The workload is the design matrix of ``bench.py``: 8 shards x 10M rows x 256 features, bf16, tensor-core kernel.
Pairs at K = 1, 4 and 16 chains:
- weibull against poisson (the Poisson model of the events, ``y = delta``: what Weibull regression is at sigma = 1);
- lognormal against gaussian_scale (the Gaussian model of ``log t``: what the log-normal one is without censoring).
About 30% of the rows are censored.  Per row, the survival epilogue adds one accurate ``logf`` (log t, shared by the
chains); per row and chain the Weibull one adds an accurate ``expf``, and the log-normal one, on censored rows, an
``erfcxf``, an ``expf`` and a log.  The chains get sigma from 0.5 to 2.

Every model shares X.  Each is checked against the fp64 oracle first.  Then timed windows of all models alternate,
so drift of the shared machine hits them alike.  Prints one JSON line with the device-timed evaluations/s (median
and all windows) and HBM bytes/s of each model, the ratios, and the card's name and power limit read in the same run.

    python benchmarks/bench_glm_survival.py [--shards 8] [--rows 10000000] [--features 256] [--steps 50] [--rounds 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_glm_row_data import card_info  # noqa: E402

KS = (1, 4, 16)
PAIRS = (("weibull", "poisson"), ("lognormal", "gaussian_scale"))


def survival_data(X, family: str, *, seed: int, censor_fraction: float = 0.3, chunk_rows: int = 1 << 20):
    """float32 ``(time, event)`` for an existing bf16 design matrix: ``log T = X beta* + 0.5 + eps`` (eps minimum-Gumbel
    for Weibull, N(0, 1) for log-normal) and a ``censor_fraction`` share of the rows censored at a uniform fraction of
    their event time."""
    import torch

    gen = torch.Generator(device=X.device)
    gen.manual_seed(seed)
    beta = torch.randn(X.shape[1], generator=gen, device=X.device) * 0.03
    t = torch.empty(X.shape[0], dtype=torch.float32, device=X.device)
    ev = torch.empty(X.shape[0], dtype=torch.float32, device=X.device)
    for r0 in range(0, X.shape[0], chunk_rows):
        r1 = min(X.shape[0], r0 + chunk_rows)
        eta = X[r0:r1].float() @ beta + 0.5
        if family == "weibull":
            eps = torch.log(-torch.log(torch.rand(r1 - r0, generator=gen, device=X.device).clamp_min(1e-30)))
        else:
            eps = torch.randn(r1 - r0, generator=gen, device=X.device)
        cens = torch.rand(r1 - r0, generator=gen, device=X.device) < censor_fraction
        shrink = torch.where(cens, torch.rand(r1 - r0, generator=gen, device=X.device) * 0.7 + 0.3, torch.ones_like(eta))
        t[r0:r1] = torch.exp(eta + eps) * shrink
        ev[r0:r1] = (~cens).float()
    return t, ev


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--shards", type=int, default=8)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=256)
    ap.add_argument("--steps", type=int, default=50, help="evaluations per timed window")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5, help="timed windows per model, alternating")
    args = ap.parse_args()

    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_glm_survival.py measures the GPU kernels and needs a CUDA device")
    from pytensor_federated_b200.models import GlmShards, synth_logistic_shard
    from pytensor_federated_b200.parallel import FederatedEngine

    dev = torch.device("cuda:0")
    P = args.features
    Xs = [synth_logistic_shard(args.rows, P, seed=1000 + s, device=dev)[0] for s in range(args.shards)]
    data = {fam: [survival_data(X, fam, seed=2000 + 100 * i + s) for s, X in enumerate(Xs)]
            for i, fam in enumerate(("weibull", "lognormal"))}
    rng = np.random.default_rng(7)
    lss = np.log([1.0, 0.5, 2.0, 1.5])
    models, thetas = {}, {}
    for surv, other in PAIRS:
        ts = [d[0] for d in data[surv]]
        es = [d[1] for d in data[surv]]
        ys = es if other == "poisson" else [torch.log(t) for t in ts]
        for K in KS:
            lead = (K,) if K > 1 else ()
            ic = rng.normal(size=lead + (1,)).astype(np.float32) * 0.1 + 0.5
            beta = rng.normal(size=lead + (P,)).astype(np.float32) * 0.02
            ls = np.resize(lss, K).astype(np.float32) if K > 1 else np.float32(lss[0])
            models[f"{surv}_K{K}"] = GlmShards(Xs, ts, kernel="tc", family=surv, events=es, n_chains=K)
            thetas[f"{surv}_K{K}"] = (ic, beta, ls)
            models[f"{other}_K{K}"] = GlmShards(Xs, ys, kernel="tc", family=other, n_chains=K)
            thetas[f"{other}_K{K}"] = (-ic, -beta) if other == "poisson" else (ic, beta, ls)
    torch.cuda.synchronize()

    engines = {k: FederatedEngine(m) for k, m in models.items()}
    result = {"config": f"{args.shards} x {args.rows} x {P} bf16, tc kernel, 1 GPU, 30% censored", "steps": args.steps,
              "rounds": args.rounds}
    try:
        # ---- correctness first: each model against its fp64 oracle (the kernel's raw output layout)
        for k, m in models.items():
            th = list(thetas[k])
            width = 1 + m.n_params
            got = np.asarray(engines[k].evaluate_raw(th), dtype=np.float64).reshape(-1, width)
            want = m.reference_partial(th, dtype=torch.float64).reshape(-1, width)
            err_ll = float(np.max(np.abs(got[:, 0] - want[:, 0]) / np.abs(want[:, 0])))
            err_g = float(np.abs(got[:, 1:] - want[:, 1:]).max() / np.abs(want[:, 1:]).max())
            result[f"{k}_max_rel_err"] = max(err_ll, err_g)
            if not max(err_ll, err_g) <= 2e-4:
                print(json.dumps({"error": f"{k}: verification failed", "max_rel_err": max(err_ll, err_g)}), flush=True)
                raise SystemExit(1)
            assert m.selected_kernel == "tc"

        def window(k, n):
            """Device time of n back-to-back evaluations (theta from device memory, as bench.py times them)."""
            eng = engines[k]
            stream = eng.torch_stream()
            eng.set_device_theta(list(thetas[k]), enable=True)
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record(stream)
            last = 0
            for _ in range(n):
                last = eng.launch()
            end.record(stream)
            eng.wait(last)
            end.synchronize()
            eng.set_device_theta(list(thetas[k]), enable=False)
            return start.elapsed_time(end) / 1e3

        for k in engines:
            window(k, args.warmup)
        rates = {k: [] for k in models}
        for _ in range(args.rounds):
            for k in engines:
                rates[k].append(args.steps / window(k, args.steps))
    finally:
        for eng in engines.values():
            eng.shutdown()
    result.update(card_info(0))
    for k, m in models.items():
        med = float(np.median(rates[k]))
        result[f"{k}_evals_per_s"] = round(med, 3)
        result[f"{k}_evals_per_s_all"] = [round(r, 3) for r in rates[k]]
        result[f"{k}_hbm_tb_per_s"] = round(m.bytes_per_eval() * med / 1e12, 3)
    for surv, other in PAIRS:
        for K in KS:
            result[f"{surv}_K{K}_vs_{other}_K{K}"] = round(result[f"{surv}_K{K}_evals_per_s"] /
                                                           result[f"{other}_K{K}_evals_per_s"], 4)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
