"""Several `bench.py` configurations (and the phase breakdown) in ONE process group.

A fresh `torchrun` costs ~30 s of imports per rank before anything is measured; on an 8-GPU box that is charged
eight-fold.  This runner initialises NCCL once and then calls `bench.run_b200` for each requested configuration
(every run still prints its own JSON line and verifies against the fp64 oracle first).

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29600 \
        benchmarks/run_configs.py --gpus 8 --out results.jsonl glm trace fp8 linreg nccl
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

import bench  # noqa: E402

RUNS = {
    # name: (extra bench.py arguments)
    "glm": ["--steps", "30", "--warmup", "5"],
    "fp8": ["--config", "fp8", "--steps", "30", "--warmup", "5"],
    "ode": ["--config", "ode", "--steps", "30", "--warmup", "5", "--shards", "4"],   # BASELINE.json: 4 shards on 4 GPUs
    "linreg": ["--config", "linreg", "--steps", "200", "--warmup", "20"],
    "nccl": ["--impl", "nccl", "--steps", "20", "--warmup", "3"],
    "glm16": ["--chains", "16", "--steps", "10", "--warmup", "3"],
}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, required=True)
    ap.add_argument("--out", default=None)
    ap.add_argument("--shards", type=int, default=8)
    ap.add_argument("runs", nargs="+", help=f"any of {sorted(RUNS)} or 'trace'")
    a = ap.parse_args()

    import torch
    import torch.distributed as dist

    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    for name in a.runs:
        try:
            if name == "trace":
                import trace_breakdown

                argv = ["--shards", str(a.shards)] + (["--out", a.out.replace(".jsonl", "_trace.jsonl")] if a.out else [])
                trace_breakdown.main(argv)
            else:
                argv = ["--gpus", str(a.gpus), "--shards", str(a.shards)] + RUNS[name] + (["--out", a.out] if a.out else [])
                saved = sys.argv
                sys.argv = ["bench.py"] + argv
                try:
                    bench.run_b200(bench.parse_args())
                finally:
                    sys.argv = saved
        except SystemExit as ex:   # a failed verification must not take the remaining runs down
            print(f"run {name}: exit {ex.code}", flush=True)
        if world > 1:
            dist.barrier()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
