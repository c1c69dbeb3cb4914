"""Rate of the gamma and inverse-Gaussian families against gaussian_scale at the same chains (one GPU).

The workload is the design matrix of ``bench.py``: 8 shards x 10M rows x 256 features, bf16, tensor-core kernel.
``gamma`` and ``inverse_gaussian`` at K = 1, 4 and 16 chains are each compared with ``gaussian_scale`` at the same K:
the same theta and output layout (one log-dispersion word per chain), the same columns and the same bytes, so the ratio
is the cost of the epilogue.  Per row, the positive-response epilogue adds one accurate ``logf`` (log y, shared by the
chains; the inverse Gaussian also one reciprocal); per row and chain, one accurate ``expf``.  The responses are drawn
from each family (``draw_positive``) at mean ``exp(X beta* + 0.5)`` and shape 2; the chains get shapes from 1 to 20.

Every model reads X as bf16 (``B200FED_NO_PACKED_X=1``): the launches of up to 4 columns would read it packed, but
each model keeps its own packed copy and at this shape device memory holds one, so the pairs would not be alike.
Each model is checked against the fp64 oracle first.  Then timed windows of all models alternate, so drift of the
shared machine hits them alike.  Prints one JSON line with the device-timed evaluations/s of each model, the ratios,
and the card's name, power limit and SM clock (NVML, read right after the timed windows) from the same run.

    python benchmarks/bench_glm_positive.py [--shards 8] [--rows 10000000] [--features 256] [--steps 50] [--rounds 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_glm_row_data import card_info  # noqa: E402
from bench_glm_zero_inflated import sm_clock  # noqa: E402

KS = (1, 4, 16)
FAMILIES = ("gamma", "inverse_gaussian", "gaussian_scale")


def positive_data(X, family: str, *, seed: int, shape: float = 2.0, chunk_rows: int = 1 << 20):
    """float32 responses > 0 for an existing bf16 design matrix, mean ``exp(X beta* + 0.5)``."""
    import torch

    from pytensor_federated_b200.models.glm import draw_positive

    gen = torch.Generator(device=X.device)
    gen.manual_seed(seed)
    beta = torch.randn(X.shape[1], generator=gen, device=X.device) * 0.03
    y = torch.empty(X.shape[0], dtype=torch.float32, device=X.device)
    for r0 in range(0, X.shape[0], chunk_rows):
        r1 = min(X.shape[0], r0 + chunk_rows)
        mu = torch.exp(X[r0:r1].float() @ beta + 0.5).double()
        y[r0:r1] = draw_positive(mu, family=family, shape=shape, generator=gen)
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
    os.environ["B200FED_NO_PACKED_X"] = "1"

    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_glm_positive.py measures the GPU kernels and needs a CUDA device")
    from pytensor_federated_b200.models import GlmShards, synth_logistic_shard
    from pytensor_federated_b200.parallel import FederatedEngine

    dev = torch.device("cuda:0")
    P = args.features
    Xs = [synth_logistic_shard(args.rows, P, seed=1000 + s, device=dev)[0] for s in range(args.shards)]
    ys = {fam: [positive_data(X, fam, seed=2000 + 100 * i + s) for s, X in enumerate(Xs)]
          for i, fam in enumerate(FAMILIES[:2])}
    ys["gaussian_scale"] = [torch.log(y) for y in ys["gamma"]]
    rng = np.random.default_rng(7)
    lds = np.log([2.0, 1.0, 5.0, 20.0])
    models, thetas = {}, {}
    for K in KS:
        lead = (K,) if K > 1 else ()
        ic = (rng.normal(size=lead + (1,)) * 0.1 + 0.5).astype(np.float32)
        beta = (rng.normal(size=lead + (P,)) * 0.02).astype(np.float32)
        ld = np.resize(lds, K).astype(np.float32) if K > 1 else np.float32(lds[0])
        for fam in FAMILIES:
            models[f"{fam}_K{K}"] = GlmShards(Xs, ys[fam], kernel="tc", family=fam, n_chains=K)
            thetas[f"{fam}_K{K}"] = (ic, beta, ld)
    torch.cuda.synchronize()

    engines = {k: FederatedEngine(m) for k, m in models.items()}
    result = {"config": f"{args.shards} x {args.rows} x {P} bf16, tc kernel, 1 GPU", "steps": args.steps,
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
        result.update(sm_clock(0))
    finally:
        for eng in engines.values():
            eng.shutdown()
    result.update(card_info(0))
    for k, m in models.items():
        med = float(np.median(rates[k]))
        result[f"{k}_evals_per_s"] = round(med, 3)
        result[f"{k}_evals_per_s_all"] = [round(r, 3) for r in rates[k]]
        result[f"{k}_hbm_tb_per_s"] = round(m.bytes_per_eval() * med / 1e12, 3)
    for fam in FAMILIES[:2]:
        for K in KS:
            result[f"{fam}_K{K}_vs_gaussian_scale_K{K}"] = round(result[f"{fam}_K{K}_evals_per_s"] /
                                                                 result[f"gaussian_scale_K{K}_evals_per_s"], 4)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
