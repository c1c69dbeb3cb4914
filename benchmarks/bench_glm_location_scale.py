"""Rate of Gaussian location-scale / Student-t launches against the Gaussian family at the same columns (one GPU).

The workload is the design matrix of ``bench.py``: 8 shards x 10M rows x 256 features, bf16, tensor-core kernel, with
Student-t responses whose scale depends on x (``synth_location_scale_shard``, nu = 4, 1 % of the rows gross outliers).
A location-scale launch of K chains runs 2K columns (the mean and the log scale of each chain), so it is compared with
``gaussian`` at 2K chains: the same GEMM shapes and the same bytes, without the location-scale epilogue.  The
configurations are ``gaussian_location_scale`` and ``student_t`` at K = 1, 4 and 8, each against ``gaussian`` at 2K
chains.

Every model reads X as bf16 (``B200FED_NO_PACKED_X=1``): the launches of up to 4 columns would read it packed, but
each model keeps its own packed copy and at this shape device memory holds one, so the pairs would not be alike.
Each model is checked against the fp64 oracle first.  Then timed windows of all models alternate, so drift of the
shared machine hits them alike.  Prints one JSON line with the device-timed evaluations/s of each model, the ratios,
and the card's name, power limit and SM clock (NVML, read right after the timed windows) from the same run.

    python benchmarks/bench_glm_location_scale.py [--shards 8] [--rows 10000000] [--features 256] [--steps 50] [--rounds 5]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_glm_row_data import card_info  # noqa: E402

CHAINS = (1, 4, 8)
PAIRS = (("gaussian_location_scale", "gaussian"), ("student_t", "gaussian"))


def sm_clock(index: int):
    """The SM clock in MHz NVML reports now, and the card's maximum (read-only queries), or None."""
    try:
        import pynvml as nv

        nv.nvmlInit()
        h = nv.nvmlDeviceGetHandleByIndex(index)
        return {"sm_clock_mhz": nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM),
                "max_sm_clock_mhz": nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)}
    except Exception as ex:   # reported, never guessed
        return {"sm_clock_mhz": None, "max_sm_clock_mhz": None, "nvml_error": f"{type(ex).__name__}: {ex}"}


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
        raise SystemExit("bench_glm_location_scale.py measures the GPU kernels and needs a CUDA device")
    from pytensor_federated_b200.models import GlmShards, synth_location_scale_shard
    from pytensor_federated_b200.parallel import FederatedEngine

    dev = torch.device("cuda:0")
    P = args.features
    Xs, ys = [], []
    for s in range(args.shards):
        X, y, _, _ = synth_location_scale_shard(args.rows, P, family="student_t", nu=4.0, seed=1000 + s, device=dev)
        gen = torch.Generator(device=dev)
        gen.manual_seed(2000 + s)
        out = torch.rand(args.rows, generator=gen, device=dev) < 0.01
        y = torch.where(out, y + 50.0, y)
        Xs.append(X)
        ys.append(y)
    rng = np.random.default_rng(7)
    models, thetas = {}, {}
    for family, base in PAIRS:
        t = family == "student_t"
        for K in CHAINS:
            lead = (K,) if K > 1 else ()
            ic, beta = rng.normal(size=lead + (1,)) * 0.1 + 0.5, rng.normal(size=lead + (P,)) * 0.02
            sic, sbeta = rng.normal(size=lead + (1,)) * 0.1, rng.normal(size=lead + (P,)) * 0.02
            ld = np.full(lead, np.log(4.0))
            models[f"{family}_K{K}"] = GlmShards(Xs, ys, kernel="tc", family=family, n_chains=K)
            thetas[f"{family}_K{K}"] = [v.astype(np.float32) for v in (ic, beta, sic, sbeta) + ((ld,) if t else ())]
            # the Gaussian family at 2K chains: chain 2k = (intercept, beta), 2k + 1 = (sigma_intercept, sigma_beta)
            stack = lambda a, b: np.stack([np.reshape(a, (K, -1)), np.reshape(b, (K, -1))], axis=1).reshape(2 * K, -1)
            if f"{base}_K{2 * K}" not in models:
                models[f"{base}_K{2 * K}"] = GlmShards(Xs, ys, kernel="tc", family=base, n_chains=2 * K)
                thetas[f"{base}_K{2 * K}"] = [v.astype(np.float32) for v in (stack(ic, sic), stack(beta, sbeta))]
    torch.cuda.synchronize()

    engines = {k: FederatedEngine(m) for k, m in models.items()}
    result = {"config": f"{args.shards} x {args.rows} x {P} bf16, tc kernel, 1 GPU", "steps": args.steps,
              "rounds": args.rounds}
    try:
        # ---- correctness first: each model against its fp64 oracle, per kernel column [LL, gi, g[P](, q)]
        for k, m in models.items():
            th = list(thetas[k])
            width = 1 + m._layout.words
            got = np.asarray(engines[k].evaluate_raw(th), dtype=np.float64).reshape(-1, width)
            want = m.reference_partial(th, dtype=torch.float64).reshape(-1, width)
            step = 2 if m.kernel_chains == 2 * m.n_chains else 1   # the log-scale columns' LL is 0
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
        result[f"{k}_packed_x"] = bool(getattr(m, "packed_x", False))
    for family, base in PAIRS:
        for K in CHAINS:
            key = f"{family}_K{K}"
            result[f"{key}_vs_{base}_K{2 * K}"] = round(result[f"{key}_evals_per_s"] / result[f"{base}_K{2 * K}_evals_per_s"], 4)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
