"""Rate of beta regression against gaussian_scale and negative_binomial at the same chains (one GPU).

The workload is the design matrix of ``bench.py``: 8 shards x 10M rows x 256 features, bf16, tensor-core kernel.
``beta`` at K = 1, 4 and 16 chains is compared with ``gaussian_scale`` and ``negative_binomial`` at the same K: the
same theta and output layout (one log-dispersion word per chain), the same columns and the same bytes, so the ratios
are the cost of the epilogue.  Per row, the beta epilogue adds ``logf(y)`` and ``log1pf(-y)`` (shared by the chains);
per row and chain, one ``expf`` and one ``log1pf`` (mu, 1 - mu and their logs), two series for the relative
differences and, for each of A = mu phi and B = (1 - mu) phi, a Stirling evaluation with a predicated shift (two
``__logf``, two divisions, one ``logf``).  The negative binomial does one such Stirling evaluation per row and chain.
The proportions are drawn from Beta(mu phi, (1 - mu) phi) at mu = sigmoid(X beta* + 0.5) and phi = 30; the counts
from NB2 at mean exp(X beta* + 0.5) and alpha = 2; the Gaussian responses are the logits of the proportions.  The
chains get precisions (dispersions) from 1 to 300.

Every model reads X as bf16 (``B200FED_NO_PACKED_X=1``): the launches of up to 4 columns would read it packed, but
each model keeps its own packed copy and at this shape device memory holds one, so the models would not be alike.
Each model is checked against the fp64 oracle first.  Then timed windows of all models alternate, so drift of the
shared machine hits them alike.  Prints one JSON line with the device-timed evaluations/s of each model (median and
every window), the ratios, and the card's name, power limit and SM clock (NVML, read right after the timed windows)
from the same run.

    python benchmarks/bench_glm_beta.py [--shards 8] [--rows 10000000] [--features 256] [--steps 50] [--rounds 5]
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
FAMILIES = ("beta", "gaussian_scale", "negative_binomial")


def responses(X, *, seed: int, chunk_rows: int = 1 << 20):
    """``(proportions, counts)`` for an existing bf16 design matrix, both at linear predictor ``X beta* + 0.5``."""
    import torch

    gen = torch.Generator(device=X.device)
    gen.manual_seed(seed)
    beta = torch.randn(X.shape[1], generator=gen, device=X.device) * 0.03
    props = torch.empty(X.shape[0], dtype=torch.float32, device=X.device)
    counts = torch.empty_like(props)
    for r0 in range(0, X.shape[0], chunk_rows):
        r1 = min(X.shape[0], r0 + chunk_rows)
        eta = (X[r0:r1].float() @ beta + 0.5).double()
        mu = torch.sigmoid(eta)
        ga = torch._standard_gamma(mu * 30.0, generator=gen)
        gb = torch._standard_gamma((1.0 - mu) * 30.0, generator=gen)
        props[r0:r1] = (ga / (ga + gb)).clamp(torch.finfo(torch.float32).tiny, 1.0 - 2.0 ** -24).float()
        lam = torch._standard_gamma(torch.full_like(eta, 2.0), generator=gen) * (torch.exp(eta) / 2.0)
        counts[r0:r1] = torch.poisson(lam, generator=gen).clamp(max=2.0 ** 24).float()
    return props, counts


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
        raise SystemExit("bench_glm_beta.py measures the GPU kernels and needs a CUDA device")
    from pytensor_federated_b200.models import GlmShards, synth_logistic_shard
    from pytensor_federated_b200.parallel import FederatedEngine

    dev = torch.device("cuda:0")
    P = args.features
    Xs = [synth_logistic_shard(args.rows, P, seed=1000 + s, device=dev)[0] for s in range(args.shards)]
    drawn = [responses(X, seed=2000 + s) for s, X in enumerate(Xs)]
    ys = {"beta": [d[0] for d in drawn], "negative_binomial": [d[1] for d in drawn],
          "gaussian_scale": [torch.logit(d[0]) for d in drawn]}
    del drawn
    rng = np.random.default_rng(7)
    lds = {"beta": np.log([30.0, 1.0, 300.0, 10.0]), "negative_binomial": np.log([2.0, 1.0, 5.0, 20.0]),
           "gaussian_scale": np.log([0.4, 0.2, 1.0, 2.0])}
    models, thetas = {}, {}
    for K in KS:
        lead = (K,) if K > 1 else ()
        ic = (rng.normal(size=lead + (1,)) * 0.1 + 0.5).astype(np.float32)
        beta = (rng.normal(size=lead + (P,)) * 0.02).astype(np.float32)
        for fam in FAMILIES:
            ld = np.resize(lds[fam], K).astype(np.float32) if K > 1 else np.float32(lds[fam][0])
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
        result[f"{k}_evals_per_s_range"] = [round(min(rates[k]), 3), round(max(rates[k]), 3)]
        result[f"{k}_evals_per_s_all"] = [round(r, 3) for r in rates[k]]
        result[f"{k}_hbm_tb_per_s"] = round(m.bytes_per_eval() * med / 1e12, 3)
    for other in FAMILIES[1:]:
        for K in KS:
            result[f"beta_K{K}_vs_{other}_K{K}"] = round(result[f"beta_K{K}_evals_per_s"] /
                                                        result[f"{other}_K{K}_evals_per_s"], 4)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
