"""Cost of per-row offsets and weights on the headline GLM (one GPU).

Times the bf16 logistic GLM of ``bench.py`` (8 shards x 10M rows x 256 features, tensor-core kernel) twice in one
process, on the same design matrix and responses: plain, and with exposure offsets (``log t``) plus binomial
trial-count weights.  Both models are checked against the fp64 oracle first; then timed windows of the two
alternate, so drift of the shared machine hits both alike.  Prints one JSON line with the device-timed
evaluations/s and HBM bytes/s of each, their ratio, and the card's name and power limit read in the same run.

    python benchmarks/bench_glm_row_data.py [--shards 8] [--rows 10000000] [--features 256] [--steps 100] [--rounds 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card_info(index: int) -> dict:
    """Name and power limit of the device (read-only queries)."""
    import torch

    info = {"device": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        import pynvml as nv

        nv.nvmlInit()
        h = nv.nvmlDeviceGetHandleByIndex(index)
        info["power_limit_w"] = nv.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
    except Exception:
        try:
            out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                 capture_output=True, text=True, timeout=30)
            info["power_limit_w"] = float(out.stdout.strip().splitlines()[0])
        except Exception:
            pass
    return info


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--shards", type=int, default=8)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=256)
    ap.add_argument("--steps", type=int, default=100, help="evaluations per timed window")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5, help="timed windows per model, alternating")
    args = ap.parse_args()

    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_glm_row_data.py measures the GPU kernels and needs a CUDA device")
    from pytensor_federated_b200.models import GlmShards, synth_logistic_shard
    from pytensor_federated_b200.parallel import FederatedEngine

    dev = torch.device("cuda:0")
    P = args.features
    Xs, ys, offs, wts = [], [], [], []
    gen = torch.Generator(device=dev)
    gen.manual_seed(4242)
    for s in range(args.shards):
        X, y, _ = synth_logistic_shard(args.rows, P, seed=1000 + s, device=dev)
        Xs.append(X)
        ys.append(y)
        t = torch.rand(args.rows, generator=gen, device=dev) * 1.5 + 0.5                        # exposure in [0.5, 2)
        offs.append(torch.log(t))
        wts.append(torch.randint(1, 11, (args.rows,), generator=gen, device=dev).float())      # trials per row
    torch.cuda.synchronize()
    models = {
        "plain": GlmShards(Xs, ys, kernel="tc"),
        "offsets_weights": GlmShards(Xs, ys, kernel="tc", offsets=offs, weights=wts),
    }
    rng = np.random.default_rng(7)
    theta = (rng.normal(size=1).astype(np.float32) * 0.1, rng.normal(size=P).astype(np.float32) * 0.02)

    engines = {k: FederatedEngine(m) for k, m in models.items()}
    result = {"config": f"{args.shards} x {args.rows} x {P} bf16 logistic, tc kernel, 1 GPU", "steps": args.steps,
              "rounds": args.rounds}
    try:
        # ---- correctness first: each model against its fp64 oracle
        for k, m in models.items():
            got = np.asarray(engines[k].evaluate_raw(list(theta)), dtype=np.float64)
            want = m.reference_partial(list(theta), dtype=torch.float64)
            err_ll = abs(got[0] - want[0]) / abs(want[0])
            err_g = np.abs(got[1:] - want[1:]).max() / np.abs(want[1:]).max()
            result[f"{k}_max_rel_err"] = float(max(err_ll, err_g))
            if not max(err_ll, err_g) <= 2e-4:
                print(json.dumps({"error": f"{k}: verification failed", "max_rel_err": float(max(err_ll, err_g))}), flush=True)
                raise SystemExit(1)
            assert m.selected_kernel == "tc"

        def window(eng, n):
            """Device time of n back-to-back evaluations (theta from device memory, as bench.py times them)."""
            stream = eng.torch_stream()
            eng.set_device_theta(list(theta), enable=True)
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record(stream)
            last = 0
            for _ in range(n):
                last = eng.launch()
            end.record(stream)
            eng.wait(last)
            end.synchronize()
            eng.set_device_theta(list(theta), enable=False)
            return start.elapsed_time(end) / 1e3

        for eng in engines.values():
            window(eng, args.warmup)
        rates = {k: [] for k in models}
        for _ in range(args.rounds):
            for k, eng in engines.items():
                rates[k].append(args.steps / window(eng, args.steps))
    finally:
        for eng in engines.values():
            eng.shutdown()
    result.update(card_info(0))
    for k, m in models.items():
        med = float(np.median(rates[k]))
        result[f"{k}_evals_per_s"] = round(med, 3)
        result[f"{k}_evals_per_s_all"] = [round(r, 3) for r in rates[k]]
        result[f"{k}_bytes_per_eval"] = m.bytes_per_eval()
        result[f"{k}_hbm_gb_per_s"] = round(m.bytes_per_eval() * med / 1e9, 1)
    result["rate_ratio"] = round(result["offsets_weights_evals_per_s"] / result["plain_evals_per_s"], 4)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
