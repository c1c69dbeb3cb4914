"""Fused broadcast -> compute -> reduce across GPUs (needs >= 2 GPUs).

Every scenario runs at world = 2, 4 and 8; a world larger than the number of visible GPUs is skipped."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu, pytest.mark.timeout(900)]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


WORLDS = [2, 4, 8]


def _shard_data(rank, n=5000):
    rng = np.random.default_rng(100 + rank)
    x = rng.normal(size=n)
    y = 1.0 + 0.5 * x + rng.normal(scale=0.7, size=n)
    return x, y


def _worker(rank, world, port, comm, scenario, q):
    import torch.distributed as dist

    from pytensor_federated_b200.models import GlmShards, LinregShards, synth_logistic_shard
    from pytensor_federated_b200.parallel import FederatedEngine, FederationTimeout

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        if scenario == "linreg":
            x, y = _shard_data(rank)
            model = LinregShards([x], [y], [0.7], local_ids=[rank], n_shards_total=world, device=dev)
            eng = FederatedEngine(model, comm=comm, timeout=20.0)
            if rank == 0:
                outs = []
                for a, b in [(0.3, -0.2), (1.0, 0.5), (0.0, 0.0)]:
                    outs.append([np.asarray(v).tolist() for v in eng.evaluate(np.array(a), np.array(b))])
                per = LinregShards.per_shard(eng.evaluate_raw([np.array(1.0), np.array(0.5)])).tolist()
                q.put(("root", eng.comm_mode, outs, per))
                eng.shutdown()
            else:
                served = eng.serve()
                q.put(("peer", served))
                eng.shutdown()
        elif scenario.startswith("glm"):
            from pytensor_federated_b200.models import Fp8GlmShards

            spec = scenario.endswith("-spec")      # root keeps kernels enqueued ahead of theta (set_speculative)
            if spec:
                scenario = scenario[: -len("-spec")]
            kernel = scenario.split("-")[1]
            chains = int(scenario.split("-")[2]) if scenario.count("-") >= 2 else 1
            X, y, _ = synth_logistic_shard(30_000 + 17 * rank, 256, seed=50 + rank, device=dev)
            if kernel == "fp8":
                model = Fp8GlmShards.from_dense([X], [y], groups=[rank % 2], n_groups=2, n_chains=chains)
            else:
                model = GlmShards([X], [y], groups=[rank % 2], n_groups=2, kernel=kernel, n_chains=chains)
            eng = FederatedEngine(model, comm=comm, timeout=20.0)
            rng = np.random.default_rng(1)
            if chains == 1:
                ic = np.array([0.2, -0.1])
                beta = (rng.normal(size=256) * 0.03).astype(np.float32)
            else:
                ic = rng.normal(size=(chains, 2)) * 0.1
                beta = (rng.normal(size=(chains, 256)) * 0.03).astype(np.float32)
            local = model.reference_partial([ic, beta], dtype=torch.float64)
            gathered = [None] * world
            dist.all_gather_object(gathered, local)
            if rank == 0:
                got = eng.evaluate(ic, beta)
                if spec:
                    assert eng.set_speculative(300.0)
                again = eng.evaluate(ic, beta)   # dynamic work distribution, same bits
                same = all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(got, again))
                if spec:
                    import time

                    for pause in (0.0, 0.0, 0.01, 0.0):      # 10 ms: the waiting kernels give up, the next call relaunches
                        time.sleep(pause)
                        more = eng.evaluate(ic, beta)
                        same = same and all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(got, more))
                want = model.unpack_result(np.sum(gathered, axis=0), model.call_context([ic, beta]))
                q.put(("root", eng.comm_mode, [np.asarray(g).tolist() for g in got], [np.asarray(w).tolist() for w in want], same))
                eng.shutdown()
            else:
                eng.serve()
                eng.shutdown()
                q.put(("peer", 1))
        elif scenario == "dead-peer":
            x, y = _shard_data(rank, 100)
            model = LinregShards([x], [y], [0.7], local_ids=[rank], n_shards_total=world, device=dev)
            eng = FederatedEngine(model, comm=comm, timeout=1.0)
            if rank == 0:
                try:
                    eng.evaluate(np.array(0.1), np.array(0.2))
                    q.put(("root", "no error"))
                except FederationTimeout as ex:
                    q.put(("root", "timeout", str(ex)))
                dist.barrier()
                eng.shutdown()
            elif rank == world - 1:
                dist.barrier()  # fault injection: this node never serves
                eng.shutdown()
                q.put(("peer", 0))
            else:
                try:
                    eng.serve(max_epochs=1)  # the healthy nodes answer; the root still misses one partial
                except Exception:
                    pass
                dist.barrier()
                eng.shutdown()
                q.put(("peer", 1))
    finally:
        dist.destroy_process_group()


def _run(world, comm, scenario):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, comm, scenario, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    return results


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("comm", ["ipc", "symm", "auto"])
def test_linreg_across_gpus_matches_numpy(comm, world):
    import scipy.stats

    results = _run(world, comm, "linreg")
    root = [r for r in results if r[0] == "root"][0]
    peers = [r for r in results if r[0] == "peer"]
    assert len(peers) == world - 1 and all(p[1] == 4 for p in peers)  # 4 evaluations served by every node
    for (a, b), got in zip([(0.3, -0.2), (1.0, 0.5), (0.0, 0.0)], root[2]):
        want_lp, want_da, want_db = 0.0, 0.0, 0.0
        for rank in range(world):
            x, y = _shard_data(rank)
            want_lp += scipy.stats.norm.logpdf(y, a + b * x, 0.7).sum()
            r = y - (a + b * x)
            want_da += r.sum() / 0.49
            want_db += (r * x).sum() / 0.49
        np.testing.assert_allclose(got, [want_lp, want_da, want_db], rtol=1e-11)
    per = np.asarray(root[3])
    assert per.shape == (world, 3) and np.all(per[:, 0] < 0)
    print("comm mode:", root[1])


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("kernel", ["simt", "tc", "tc-4", "tc-16", "fp8", "tc-1-spec", "fp8-1-spec"])
def test_glm_across_gpus_matches_reference(kernel, world):
    results = _run(world, "auto", f"glm-{kernel}")
    root = [r for r in results if r[0] == "root"][0]
    got, want, same = root[2], root[3], root[4]
    assert same, "two evaluations of the same theta must agree bit for bit"
    if kernel.startswith("fp8"):
        np.testing.assert_allclose(got[0], want[0], rtol=2e-5)
        np.testing.assert_allclose(got[2], want[2], rtol=2e-4, atol=2e-4 * np.abs(want[2]).max())
        return
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)
    np.testing.assert_allclose(got[1], want[1], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(got[2], want[2], rtol=1e-4, atol=0.5)


@pytest.mark.parametrize("world", WORLDS)
def test_dead_peer_raises_timeout_instead_of_hanging(world):
    results = _run(world, "ipc", "dead-peer")
    root = [r for r in results if r[0] == "root"][0]
    assert root[1] == "timeout" and "did not deliver" in root[2]


def _build_linreg(rank, world, dev):
    from pytensor_federated_b200.models import LinregShards

    x, y = _shard_data(rank, 64)
    return LinregShards([x], [y], [0.7], local_ids=[rank], n_shards_total=world, device=dev)


def test_launch_federation_context_manager_on_gpus():
    """The user-facing launcher: peers are spawned, the caller is the client, nodes are addressable
    through NodeFederation and the reference's client API."""
    import scipy.stats

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from pytensor_federated_b200 import LogpGradServiceClient
    from pytensor_federated_b200.federation import NodeFederation, launch_federation

    with launch_federation(_build_linreg, 2, timeout=30.0) as eng:
        assert eng.backend == "fused" and eng.world == 2
        fed = NodeFederation(eng)
        addresses = fed.register_services("gpu", 0)
        client = LogpGradServiceClient(*addresses[1])
        logp, grads = client.evaluate(np.array(0.3), np.array(-0.2))
        x, y = _shard_data(1, 64)
        np.testing.assert_allclose(logp, scipy.stats.norm.logpdf(y, 0.3 - 0.2 * x, 0.7).sum(), rtol=1e-11)
        del client
        fed.unregister_services()
