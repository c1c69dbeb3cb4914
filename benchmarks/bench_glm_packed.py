"""Packed (12-bit) against bf16 X in the tensor-core GLM kernel, and the kernel's ceiling with X in L2 (one GPU).

The headline GLM (``bench.py``: 8 shards x 10M rows x 256 features, bf16 logistic, K = 1) streams X from HBM at
close to the card's bandwidth.  Reading fewer bytes per row (a compressed X decoded on chip) can only pay off if
the rest of the kernel's per-tile chain (wait -> MMA #1 -> epilogue -> barrier -> MMA #2 -> release) is clearly
faster than the HBM stream.  This script measures that chain on its own: a model of the same row count whose
segments all point at one 32K x 256 bf16 matrix (16 MB, resident in the 50 MB L2), so X costs almost no HBM
traffic, timed in windows that alternate with the flagship shape in one process: read as bf16 (``bf16``, as with
``B200FED_NO_PACKED_X=1``) and in its packed form (``packed``), the two checked to compute the same bits.  The same
L2-resident model is also read packed (``l2-packed``): all its segments share one packed copy of the matrix (about
12 MB), so it measures the packed kernel's on-chip ceiling (decode, hand-off and consumer chain) without the HBM
stream; it is checked bitwise against ``l2``.  ``l2-packed`` well above ``packed`` means the HBM stream binds the
packed kernel; close to it, the on-chip chain does.

Prints one JSON line: device-timed evaluations/s of the four models, the rows/s of each, the bytes each reads per
evaluation over its time, the packed / bf16, l2 / bf16 and packed / l2-packed ratios, and the card's name, power limit
and NVML-sampled SM clock.

    python benchmarks/bench_glm_packed.py [--shards 8] [--rows 10000000] [--features 256] [--chains 1] [--steps 30]
                                          [--rounds 5] [--no-l2]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--shards", type=int, default=8)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--features", type=int, default=256)
    ap.add_argument("--l2-rows", type=int, default=32768, help="rows of the one matrix the L2-resident segments share")
    ap.add_argument("--steps", type=int, default=30, help="evaluations per timed window")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5, help="timed windows per model, alternating")
    ap.add_argument("--chains", type=int, default=1, help="parameter vectors per evaluation (K)")
    ap.add_argument("--no-l2", action="store_true", help="time only the bf16 and packed models")
    args = ap.parse_args()

    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_glm_packed.py measures the GPU kernels and needs a CUDA device")
    from bench import ClockSampler
    from benchmarks.bench_glm_row_data import card_info
    from pytensor_federated_b200.models import GlmShards, synth_logistic_shard
    from pytensor_federated_b200.models.glm import pack_x12
    from pytensor_federated_b200.parallel import FederatedEngine

    dev = torch.device("cuda:0")
    P = args.features
    Xs, ys = [], []
    for s in range(args.shards):
        X, y, _ = synth_logistic_shard(args.rows, P, seed=1000 + s, device=dev)
        Xs.append(X)
        ys.append(y)
    K = args.chains
    models = {
        "bf16": GlmShards(Xs, ys, kernel="tc", n_chains=K),
        "packed": GlmShards(Xs, ys, kernel="tc", n_chains=K),
    }
    n_l2 = args.shards * args.rows // args.l2_rows   # as many rows as the flagship, give or take one segment
    if not args.no_l2:
        X2, y2, _ = synth_logistic_shard(args.l2_rows, P, seed=77, device=dev)
        models["l2"] = GlmShards([X2] * n_l2, [y2] * n_l2, kernel="tc", n_chains=K)
        # one packed copy for every segment, as the bf16 segments share one matrix: packing each segment on its own
        # would make n_l2 copies (29 GB at the flagship shape), which would not stay in L2
        models["l2-packed"] = GlmShards([X2] * n_l2, [y2] * n_l2, kernel="tc", n_chains=K)
        models["l2-packed"]._packs = [pack_x12(X2)] * n_l2
    packed_models = ("packed", "l2-packed")
    torch.cuda.synchronize()
    rows = {k: m.n_rows for k, m in models.items()}
    rng = np.random.default_rng(7)
    if K == 1:
        theta = (rng.normal(size=1).astype(np.float32) * 0.1, rng.normal(size=P).astype(np.float32) * 0.02)
    else:
        theta = (rng.normal(size=K).astype(np.float32) * 0.1, rng.normal(size=(K, P)).astype(np.float32) * 0.02)

    engines = {}
    saved = os.environ.get("B200FED_NO_PACKED_X")
    try:
        for k, m in models.items():   # the switch is read when an engine attaches the model
            os.environ["B200FED_NO_PACKED_X"] = "0" if k in packed_models else "1"
            engines[k] = FederatedEngine(m)
    finally:
        if saved is None:
            os.environ.pop("B200FED_NO_PACKED_X", None)
        else:
            os.environ["B200FED_NO_PACKED_X"] = saved
    result = {"config": f"{args.shards} x {args.rows} x {P} bf16 logistic (bf16, packed)"
                        + ("" if args.no_l2 else f" against {n_l2} x {args.l2_rows} x {P} segments of one matrix "
                                                 "(l2, l2-packed)")
                        + f", tc kernel, K = {K}, 1 GPU",
              "steps": args.steps, "rounds": args.rounds}
    try:
        # every model must compute what the oracle computes before its time means anything; a packed model, the bits
        # of its bf16 twin
        assert all(m.packed_x == (k in packed_models) for k, m in models.items())
        raw = {k: np.asarray(engines[k].evaluate_raw(list(theta)), dtype=np.float64) for k in models}
        for pk, twin in (("packed", "bf16"), ("l2-packed", "l2")):
            if pk not in models:
                continue
            key = "packed_bitwise_equal" if pk == "packed" else "l2_packed_bitwise_equal"
            result[key] = raw[twin].tobytes() == raw[pk].tobytes()
            if not result[key]:
                print(json.dumps({"error": f"{pk} and {twin} results differ"}), flush=True)
                raise SystemExit(1)
        for k, m in models.items():
            if k in packed_models:
                continue
            assert m.selected_kernel == "tc"
            got = np.asarray(engines[k].evaluate_raw(list(theta)), dtype=np.float64)
            want = m.reference_partial(list(theta), dtype=torch.float64)
            err = max(abs(got[0] - want[0]) / abs(want[0]), np.abs(got[1:] - want[1:]).max() / np.abs(want[1:]).max())
            result[f"{k}_max_rel_err"] = float(err)
            if not err <= 2e-4:
                print(json.dumps({"error": f"{k}: verification failed", "max_rel_err": float(err)}), flush=True)
                raise SystemExit(1)

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
        sampler = ClockSampler(0).start()
        for _ in range(args.rounds):
            for k, eng in engines.items():
                rates[k].append(args.steps / window(eng, args.steps))
        result["clocks"] = sampler.stop()
    finally:
        for eng in engines.values():
            eng.shutdown()
    result.update(card_info(0))
    for k, m in models.items():
        med = float(np.median(rates[k]))
        result[f"{k}_evals_per_s"] = round(med, 3)
        result[f"{k}_evals_per_s_all"] = [round(r, 3) for r in rates[k]]
        result[f"{k}_rows"] = rows[k]
        result[f"{k}_grows_per_s"] = round(rows[k] * med / 1e9, 3)
        result[f"{k}_bytes_per_eval"] = m.bytes_per_eval()
        result[f"{k}_gb_per_s"] = round(m.bytes_per_eval() * med / 1e9, 1)
    result["packed_over_bf16"] = round(result["packed_evals_per_s"] / result["bf16_evals_per_s"], 4)
    # rows per second, so that the l2 model's slightly different row count does not bias the ratio
    if "l2" in models:
        result["l2_over_bf16_rows_per_s"] = round(result["l2_grows_per_s"] / result["bf16_grows_per_s"], 4)
        result["packed_over_l2_packed_rows_per_s"] = round(result["packed_grows_per_s"] / result["l2-packed_grows_per_s"], 4)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
