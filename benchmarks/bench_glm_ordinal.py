"""Rate of ordinal (cumulative-logit) regression against the logistic GLM of the same MMA shapes (one GPU).

The workload is the design matrix of ``bench.py``: 8 shards x 10M rows x 256 features, bf16, tensor-core kernel.
A C-category ordinal model at K chains runs K (C - 1) virtual chains (one per cutpoint) through the kernel, so it is
compared with
- logistic at K (C - 1) chains: the same GEMM shapes, without the cumulative-logit epilogue;
- logistic at K = 1.
The configurations are ordinal C in {3, 5, 9, 17} at K = 1, plus C = 3 at K = 8. The last one has the most chains
per quad of lanes, and so the most epilogue work per row (per chain: four shuffles and the transcendental functions
of softplus, sigmoid and log(1 - e^-gap), which every lane of the quad evaluates).

Every model shares X and gets its own labels. Each is checked against the fp64 oracle first. Then timed windows
of all models alternate, so drift of the shared machine hits them alike. Prints one JSON line with the device-timed
evaluations/s and HBM bytes/s of each model, the ratios, and the card's name and power limit read in the same run.

    python benchmarks/bench_glm_ordinal.py [--shards 8] [--rows 10000000] [--features 256] [--steps 50] [--rounds 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_glm_row_data import card_info  # noqa: E402


CONFIGS = ((3, 1), (5, 1), (9, 1), (17, 1), (3, 8))   # (C, K)


def ordinal_labels(X, cuts, *, seed: int, chunk_rows: int = 1 << 20):
    """float32 labels ``y = #{j : U > sigmoid(c_j - X beta*)}`` (cumulative logit) for an existing bf16 design matrix."""
    import torch

    gen = torch.Generator(device=X.device)
    gen.manual_seed(seed)
    beta = torch.randn(X.shape[1], generator=gen, device=X.device) * 0.05
    c = torch.as_tensor(cuts, dtype=torch.float32, device=X.device)
    y = torch.empty(X.shape[0], dtype=torch.float32, device=X.device)
    for r0 in range(0, X.shape[0], chunk_rows):
        r1 = min(X.shape[0], r0 + chunk_rows)
        cdf = torch.sigmoid(c[None, :] - (X[r0:r1].float() @ beta)[:, None])
        u = torch.rand(r1 - r0, 1, generator=gen, device=X.device)
        y[r0:r1] = (u > cdf).sum(1).float()
    return y


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
        raise SystemExit("bench_glm_ordinal.py measures the GPU kernels and needs a CUDA device")
    from pytensor_federated_b200.models import GlmShards, synth_logistic_shard
    from pytensor_federated_b200.parallel import FederatedEngine

    dev = torch.device("cuda:0")
    P = args.features
    Xs, ys = [], []
    for s in range(args.shards):
        X, y, _ = synth_logistic_shard(args.rows, P, seed=1000 + s, device=dev)
        Xs.append(X)
        ys.append(y)
    rng = np.random.default_rng(7)
    models, thetas = {}, {}
    for K in (1, 2, 4, 8, 16):
        models[f"logistic_K{K}"] = GlmShards(Xs, ys, kernel="tc", n_chains=K)
        lead = (K,) if K > 1 else ()
        thetas[f"logistic_K{K}"] = (rng.normal(size=lead + (1,)).astype(np.float32) * 0.1,
                                    rng.normal(size=lead + (P,)).astype(np.float32) * 0.02)
    for Cn, K in CONFIGS:
        cuts = np.linspace(-2.0, 2.0, Cn - 1)
        labels = [ordinal_labels(X, cuts, seed=2000 + 17 * Cn + s) for s, X in enumerate(Xs)]
        key = f"ordinal_C{Cn}_K{K}"
        models[key] = GlmShards(Xs, labels, kernel="tc", family="ordinal", n_classes=Cn, n_chains=K)
        lead = (K,) if K > 1 else ()
        cp = np.sort(cuts + rng.normal(size=lead + (Cn - 1,)) * 0.02, axis=-1)
        thetas[key] = (np.zeros(lead + (1,), np.float32), rng.normal(size=lead + (P,)).astype(np.float32) * 0.02,
                       cp.astype(np.float32))
    torch.cuda.synchronize()

    engines = {k: FederatedEngine(m) for k, m in models.items()}
    result = {"config": f"{args.shards} x {args.rows} x {P} bf16, tc kernel, 1 GPU", "steps": args.steps,
              "rounds": args.rounds}
    try:
        # ---- correctness first: each model against its fp64 oracle (the kernel's raw output layout)
        for k, m in models.items():
            th = list(thetas[k])
            got = np.asarray(engines[k].evaluate_raw(th), dtype=np.float64)
            want = m.reference_partial(th, dtype=torch.float64)
            blocks = got.reshape(-1, 1 + 1 + P), want.reshape(-1, 1 + 1 + P)   # [LL, gi, g[P]] per (virtual) chain
            # (the ordinal oracle keeps the kernel's layout: each cutpoint column's block, LL credited as the kernel does)
            err_ll = float(np.max(np.abs(blocks[0][:, 0] - blocks[1][:, 0]) / np.abs(blocks[1][:, 0])))
            err_g = float(np.abs(blocks[0][:, 1:] - blocks[1][:, 1:]).max() / np.abs(blocks[1][:, 1:]).max())
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
    for Cn, K in CONFIGS:
        key, cols = f"ordinal_C{Cn}_K{K}", (Cn - 1) * K
        result[f"{key}_vs_logistic_K{cols}"] = round(result[f"{key}_evals_per_s"] / result[f"logistic_K{cols}_evals_per_s"], 4)
        result[f"{key}_vs_logistic_K1"] = round(result[f"{key}_evals_per_s"] / result["logistic_K1_evals_per_s"], 4)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
