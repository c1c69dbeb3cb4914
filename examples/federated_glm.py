"""Federated logistic regression across N nodes (GPUs, or CPU processes for a dry run).

    python examples/federated_glm.py                                   # one node
    torchrun --nproc-per-node 4 --master-addr 127.0.0.1 examples/federated_glm.py --chains 8

Every rank builds its *private* shard; rank 0 is the client and runs lock-step HMC with `--chains`
chains per fused evaluation; the other ranks serve.  On GPUs the evaluation is the fused sm_90a
kernel (θ multicast over NVSwitch → wgmma GEMMs → NVLink reduce); on CPU it is the gloo/eager
baseline with the same API.
"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch
    import torch.distributed as dist

    from pytensor_federated_b200.models import GlmShards, synth_logistic_shard
    from pytensor_federated_b200.parallel import FederatedEngine
    from pytensor_federated_b200.sampling import glm_batch_fn, hmc_sample_batched

    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=200_000)
    ap.add_argument("--features", type=int, default=128)
    ap.add_argument("--chains", type=int, default=4)
    ap.add_argument("--draws", type=int, default=100)
    args = ap.parse_args()

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    cuda = torch.cuda.is_available()
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0"))) if cuda else torch.device("cpu")
    if cuda:
        torch.cuda.set_device(dev)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl" if cuda else "gloo", **({"device_id": dev} if cuda else {}))

    X, y, beta_true = synth_logistic_shard(args.rows, args.features, seed=100 + rank, device=dev)
    model = GlmShards([X], [y], n_chains=args.chains, kernel="auto" if cuda else "simt")
    engine = FederatedEngine(model, timeout=120.0)
    if rank == 0:
        K, D = args.chains, 1 + args.features
        t0 = time.perf_counter()
        res = hmc_sample_batched(glm_batch_fn(engine, 1), np.zeros((K, D)), draws=args.draws, tune=args.draws,
                                 n_leapfrog=8, step_size=0.5 / np.sqrt(args.rows * world), seed=0)
        dt = time.perf_counter() - t0
        post = res.samples.reshape(-1, D).mean(0)
        print(f"{world} node(s) on {dev.type}, backend={engine.backend}, comm={engine.comm_mode}")
        print(f"{res.n_batched_evals} fused evaluations x {K} chains in {dt:.2f} s "
              f"({K * res.n_batched_evals / dt:.0f} chain-evals/s); accept {res.accept_rate.mean():.2f}")
        print("posterior mean of the first coefficients:", np.round(post[1:6], 3))
        engine.shutdown()
    else:
        engine.serve()
        engine.shutdown()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
