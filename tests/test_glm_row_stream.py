"""Row data (responses, offsets, weights) streamed into the tensor-core kernel's TMA stages with the X tile.

CPU: ``GlmShards`` gives the kernel 16-byte aligned row arrays, copying a misaligned view once.
GPU: segment lengths that cover every residue mod 4 and mod 128, a single-row segment, odd tile counts (the empty
padding tile of a chunk) and a segment of a million rows, several in one model, against the fp64 oracle; a shape at the
shared-memory boundary; and a misaligned pointer handed to the runtime directly is refused before the engine's
model changes.  CPU: no shape gets fewer TMA stages than before the row slots existed.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from pytensor_federated_b200.models import GlmShards
from pytensor_federated_b200.parallel import FederatedEngine

ROWS = [1, 3, 127, 129, 130, 131, 1_000_003]


def test_glm_shards_realigns_misaligned_row_arrays():
    n, P = 64, 16
    X = torch.randn(n, P).to(torch.bfloat16)
    y_full = torch.rand(n + 1)
    o_full = torch.randn(n + 3)
    w_full = torch.rand(n + 2)
    y, o, w = y_full[1:], o_full[3:], w_full[2:]
    assert all(t.data_ptr() % 16 != 0 for t in (y, o, w))
    model = GlmShards([X], [y], offsets=[o], weights=[w], kernel="simt")
    for got, want in ((model.ys[0], y), (model.offsets[0], o), (model.weights[0], w)):
        assert got.data_ptr() % 16 == 0
        assert got.is_contiguous() and got.dtype == torch.float32
        assert torch.equal(got, want)
    # an aligned float32 array is used as it is, not copied
    y_ok = torch.rand(n)
    assert GlmShards([X], [y_ok], kernel="simt").ys[0].data_ptr() == y_ok.data_ptr()


def _stages_before_row_slots(P, K, G, family):
    """Stage count of the layout before row data travelled with the tile (intercept table [KC][G] in shared memory,
    no row slots): the shapes that launched then (>= 2 stages) must still launch."""
    kc = 1 if K <= 1 else 4 if K <= 4 else 8 if K <= 8 else 16
    n1, n2 = (24 if kc <= 8 else 48), ((2 * kc + 7) // 8) * 8
    panels = ((P + 127) // 128 * 128) // 64
    table = G + (9 if family in (4, 5) else 0)
    fixed = panels * n1 * 128 + 2 * 128 * n2 * 2 + ((kc * table * 4 + 15) & ~15) + 16 * 24 + 192 + 1024
    return min(4, (227 * 1024 - fixed) // (panels * 128 * 128))


def test_row_slots_cost_no_stage():
    from pytensor_federated_b200.ops import native

    lib = native.load()
    for P in (128, 256, 384):
        for K in (1, 4, 8, 16):
            for family in (0, 3, 4, 6):
                for G in (1, 2, 8, 64, 142, 143, 206, 207, 238, 239, 287, 300):
                    for row_data in (0, 1, 2, 3):
                        got = lib.b200_glm_tc_stages(P, K, G, family, row_data)
                        assert got >= _stages_before_row_slots(P, K, G, family), (P, K, G, family, row_data)
    # the benchmark shapes
    assert lib.b200_glm_tc_stages(256, 1, 1, 0, 0) == 3
    assert lib.b200_glm_tc_stages(256, 16, 1, 0, 3) == 2
    assert lib.b200_glm_tc_stages(384, 8, 238, 0, 3) == 2


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from pytensor_federated_b200.ops import native

    native.load()  # a GPU box without the native library is a failure, not a skip
    return torch.device("cuda:0")


def _case(rows, P, dev, *, row_data, seed):
    """Logistic segments of the given lengths; with row data, binomial trial weights (some 0) and offsets."""
    g = torch.Generator(device=dev).manual_seed(seed)
    beta = torch.randn(P, device=dev, generator=g) * 0.05
    Xs, ys, offs, wts = [], [], [], []
    for n in rows:
        X = torch.randn(n, P, device=dev, generator=g)
        eta = X @ beta + 0.2
        p = torch.sigmoid(eta)
        if row_data:
            trials = torch.randint(1, 4, (n,), device=dev, generator=g).float()
            k = torch.binomial(trials, p, generator=g)
            y, w = k / trials, trials
            w[::17] = 0.0   # masked rows
            o = torch.randn(n, device=dev, generator=g) * 0.3
            offs.append(o)
            wts.append(w)
        else:
            y = torch.bernoulli(p, generator=g)
        Xs.append(X.to(torch.bfloat16))
        ys.append(y.float())
    return Xs, ys, (offs if row_data else None), (wts if row_data else None)


def _rel(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30))


@pytest.mark.parametrize("K", [1, 16])
@pytest.mark.parametrize("row_data", [False, True])
@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_tc_kernel_streams_rows_of_every_segment_length(dev, K, row_data):
    P, G = 64, 3
    Xs, ys, offs, wts = _case(ROWS, P, dev, row_data=row_data, seed=K + 2 * row_data)
    groups = [i % G for i in range(len(ROWS))]
    model = GlmShards(Xs, ys, groups=groups, n_groups=G, n_chains=K, kernel="tc", offsets=offs, weights=wts)
    rng = np.random.default_rng(K)
    shape = (K,) if K > 1 else ()
    ic = (rng.normal(size=shape + (G,)) * 0.2).astype(np.float32)
    beta = (rng.normal(size=shape + (P,)) * 0.03).astype(np.float32)
    with FederatedEngine(model) as eng:
        got = [np.asarray(v).copy() for v in eng.evaluate(ic, beta)]
    assert model.selected_kernel == "tc"
    want = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    assert all(np.all(np.isfinite(v)) for v in got)
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)
    assert _rel(got[1], want[1]) < 1e-4
    assert _rel(got[2], want[2]) < 1e-4


@pytest.mark.parametrize("row_data", [False, True])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_at_the_shared_memory_boundary(dev, row_data):
    """P = 384, K = 8, G = 238: two 96 KB stages, 8 chains and a large intercept table; the row slots must not
    cost the ring a stage."""
    P, G, K = 384, 238, 8
    rows = [128 * 9 + 5, 3000, 700]
    Xs, ys, offs, wts = _case(rows, P, dev, row_data=row_data, seed=21 + row_data)
    model = GlmShards(Xs, ys, groups=[0, 119, G - 1], n_groups=G, n_chains=K, kernel="tc", offsets=offs, weights=wts)
    rng = np.random.default_rng(5)
    ic = (rng.normal(size=(K, G)) * 0.2).astype(np.float32)
    beta = (rng.normal(size=(K, P)) * 0.01).astype(np.float32)
    with FederatedEngine(model) as eng:
        got = [np.asarray(v).copy() for v in eng.evaluate(ic, beta)]
    assert model.selected_kernel == "tc"
    want = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)
    assert _rel(got[1], want[1]) < 1e-4
    assert _rel(got[2], want[2]) < 1e-4


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_runtime_rejects_misaligned_row_arrays(dev):
    """y, offsets and weights are read through TMA, so the runtime refuses an address that is not 16-byte aligned
    (error -19), before the engine's model changes: the engine then still evaluates the model it had."""
    from pytensor_federated_b200.ops import native

    n, P = 256, 16
    Xs, ys, _, _ = _case([n], P, dev, row_data=False, seed=11)
    model = GlmShards(Xs, ys, kernel="tc")   # n_vals = 1 + 1 + 16
    buf = torch.zeros(n + 4, device=dev)
    good, bad = buf.data_ptr(), buf.data_ptr() + 4
    with FederatedEngine(model) as eng:
        lib, h = eng._lib, eng._handle
        Xp = native.void_p_array([Xs[0].data_ptr()])
        rows, grp = (C.c_longlong * 1)(n), (C.c_int * 1)(0)

        def set_glm(y, o, w):
            return int(lib.b200_engine_set_glm(h, 1, Xp, native.void_p_array([y]), None, rows, grp, P, P, 1, 1, 0, 1, None,
                                               1, native.void_p_array([o]), native.void_p_array([w]), 1))

        for args in ((bad, 0, 0), (good, bad, 0), (good, 0, bad), (good, bad, bad)):
            assert set_glm(*args) == -19
            assert "16-byte aligned" in native.last_error()
        ic, beta = np.float32(0.1), np.full(P, 0.01, np.float32)
        got = eng.evaluate(ic, beta)
    want = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)
    np.testing.assert_allclose(got[2], want[2], rtol=1e-3, atol=1e-2)
