"""Rate of Hessian-vector-product launches against logistic launches of the same columns (one GPU).

The workload is the design matrix of ``bench.py``: 8 shards x 10M rows x 256 features, bf16, tensor-core kernel.
An HVP launch of K pairs runs 2K columns (the parameters and a direction per pair), so it is compared with
- logistic at 2K chains: the same GEMM shapes, without the direction columns' epilogue (h and s = w h u);
- logistic at K = 1.
The configurations are HVP at 1, 4 and 8 pairs.  Then one timed assembly of the full 257 x 257 Hessian
(``sampling.glm_hessian``: ceil(257 / 8) = 33 launches at 8 pairs), host packing and unpacking included.

Each model is checked against the fp64 oracle first.  Then timed windows of all models alternate, so drift of the
shared machine hits them alike.  Prints one JSON line with the device-timed evaluations/s of each model, the ratios,
the Hessian's wall time, and the card's name, power limit and maximum SM clock read in the same run.

    python benchmarks/bench_glm_hvp.py [--shards 8] [--rows 10000000] [--features 256] [--steps 50] [--rounds 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_glm_row_data import card_info  # noqa: E402

PAIRS = (1, 4, 8)


def max_sm_clock(index: int):
    """The card's maximum SM clock in MHz (a read-only query), or None."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


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
        raise SystemExit("bench_glm_hvp.py measures the GPU kernels and needs a CUDA device")
    from pytensor_federated_b200.models import GlmShards, synth_logistic_shard
    from pytensor_federated_b200.parallel import FederatedEngine
    from pytensor_federated_b200.sampling import glm_hessian

    dev = torch.device("cuda:0")
    P = args.features
    Xs, ys = [], []
    for s in range(args.shards):
        X, y, _ = synth_logistic_shard(args.rows, P, seed=1000 + s, device=dev)
        Xs.append(X)
        ys.append(y)
    rng = np.random.default_rng(7)
    models, thetas = {}, {}
    for K in (1,) + tuple(2 * k for k in PAIRS):
        models[f"logistic_K{K}"] = GlmShards(Xs, ys, kernel="tc", n_chains=K)
        lead = (K,) if K > 1 else ()
        thetas[f"logistic_K{K}"] = (rng.normal(size=lead + (1,)).astype(np.float32) * 0.1,
                                    rng.normal(size=lead + (P,)).astype(np.float32) * 0.02)
    for K in PAIRS:
        models[f"hvp_K{K}"] = GlmShards(Xs, ys, kernel="tc", n_chains=K, hvp=True)
        lead = (K,) if K > 1 else ()
        thetas[f"hvp_K{K}"] = (rng.normal(size=lead + (1,)).astype(np.float32) * 0.1,
                               rng.normal(size=lead + (P,)).astype(np.float32) * 0.02,
                               rng.normal(size=lead + (1,)).astype(np.float32),
                               rng.normal(size=lead + (P,)).astype(np.float32))
    torch.cuda.synchronize()

    engines = {k: FederatedEngine(m) for k, m in models.items()}
    result = {"config": f"{args.shards} x {args.rows} x {P} bf16, tc kernel, 1 GPU", "steps": args.steps,
              "rounds": args.rounds}
    try:
        # ---- correctness first: each model against its fp64 oracle, per kernel column [LL, gi, g[P]]
        for k, m in models.items():
            th = list(thetas[k])
            got = np.asarray(engines[k].evaluate_raw(th), dtype=np.float64).reshape(-1, 2 + P)
            want = m.reference_partial(th, dtype=torch.float64).reshape(-1, 2 + P)
            step = 2 if m.hvp else 1   # the direction columns' LL is 0
            err_ll = float(np.max(np.abs(got[::step, 0] - want[::step, 0]) / np.abs(want[::step, 0])))
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

        # ---- the full Hessian of the 1 + P parameters at 8 pairs per launch (warm-up call first)
        eng8 = engines[f"hvp_K{PAIRS[-1]}"]
        theta = np.concatenate([[0.1], rng.normal(size=P) * 0.02])
        glm_hessian(eng8, theta)
        t0 = time.perf_counter()
        _, _, H = glm_hessian(eng8, theta)
        result["hessian_seconds"] = round(time.perf_counter() - t0, 4)
        result["hessian_launches"] = -(-(1 + P) // PAIRS[-1])
        result["hessian_finite"] = bool(np.all(np.isfinite(H)))
    finally:
        for eng in engines.values():
            eng.shutdown()
    result.update(card_info(0))
    result["max_sm_clock_mhz"] = max_sm_clock(0)
    for k, m in models.items():
        med = float(np.median(rates[k]))
        result[f"{k}_evals_per_s"] = round(med, 3)
        result[f"{k}_evals_per_s_all"] = [round(r, 3) for r in rates[k]]
        result[f"{k}_hbm_tb_per_s"] = round(m.bytes_per_eval() * med / 1e12, 3)
    for K in PAIRS:
        key = f"hvp_K{K}"
        result[f"{key}_vs_logistic_K{2 * K}"] = round(result[f"{key}_evals_per_s"] / result[f"logistic_K{2 * K}_evals_per_s"], 4)
        result[f"{key}_vs_logistic_K1"] = round(result[f"{key}_evals_per_s"] / result["logistic_K1_evals_per_s"], 4)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
