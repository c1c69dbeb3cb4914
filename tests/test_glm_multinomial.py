"""Multinomial (softmax) regression: ``GlmShards(..., family="multinomial", n_classes=C)``.

CPU tests check the fp64 oracle and the collective backend against independent formulas (autograd of
``log_softmax``, scipy, finite differences) and the model's packing; GPU tests check the tensor-core kernel against
that oracle."""
import ctypes as C

import numpy as np
import pytest
import torch

from pytensor_federated_b200.models import Fp8GlmShards, GlmShards, synth_multinomial_shard
from pytensor_federated_b200.parallel import FederatedEngine
from pytensor_federated_b200.parallel.engine import default_inputs_from_words


# ----------------------------------------------------------------------------------------------- fixtures
def _case(rows, P, n_classes, *, seed=0, device="cpu", n_masked=5, weighted=True):
    """Ragged bf16 segments with labels drawn from a softmax model.  With ``weighted``, every segment but the last
    has weights; the first ``n_masked`` rows of segment 0 have weight 0 and carry a NaN, a negative, a too large
    and a fractional label."""
    rng = np.random.default_rng(seed)
    Xs, ys, ws = [], [], []
    for si, n in enumerate(rows):
        X = torch.tensor(rng.normal(size=(n, P)), dtype=torch.float32).to(torch.bfloat16)
        eta = X.double().numpy() @ (rng.normal(size=(P, n_classes)) * 0.1) + rng.normal(size=n_classes) * 0.3
        p = np.exp(eta - eta.max(1, keepdims=True))
        p /= p.sum(1, keepdims=True)
        y = np.array([rng.choice(n_classes, p=pi) for pi in p], dtype=np.float64)
        w = rng.uniform(0.2, 2.0, size=n)
        if si == 0 and n_masked:
            w[:n_masked] = 0.0
            y[:4] = [np.nan, -1.0, n_classes, 0.5][: min(4, n_masked)]
        Xs.append(X.to(device))
        ys.append(torch.tensor(y, dtype=torch.float32, device=device))
        ws.append(torch.tensor(w, dtype=torch.float32, device=device) if weighted and si < len(rows) - 1 else None)
    return Xs, ys, ws


def _theta(G, P, n_classes, K=1, seed=3, scale=0.03):
    rng = np.random.default_rng(seed)
    lead = (K,) if K > 1 else ()
    return ((rng.normal(size=lead + (G, n_classes)) * 0.2).astype(np.float32),
            (rng.normal(size=lead + (P, n_classes)) * scale).astype(np.float32))


def _explicit_fp64(Xs, ys, ws, groups, ic, beta):
    """``[LL, dLL/dintercept, dLL/dbeta]`` per chain by autograd of the textbook formula with ``log_softmax``."""
    ic, beta = np.asarray(ic, dtype=np.float64), np.asarray(beta, dtype=np.float64)
    batched = beta.ndim == 3
    if not batched:
        ic, beta = ic.reshape((1,) + ic.shape), beta[None]
    K, P, Cn = beta.shape
    t_ic = torch.tensor(ic.reshape(K, -1, Cn), requires_grad=True)
    t_b = torch.tensor(beta, requires_grad=True)
    total = torch.zeros(K, dtype=torch.float64)
    for X, y, w, g in zip(Xs, ys, ws, groups):
        X, y = X.double().cpu(), y.double().cpu()
        keep = torch.ones_like(y, dtype=torch.bool) if w is None else w.cpu() != 0
        lab = torch.where(keep, y, torch.zeros_like(y)).long()
        eta = torch.einsum("np,kpc->knc", X, t_b) + t_ic[:, g, None, :]
        ll = torch.gather(torch.log_softmax(eta, dim=-1), 2, lab.view(1, -1, 1).expand(K, -1, 1)).squeeze(2)   # [K, n]
        if w is not None:
            ll = torch.where(keep, w.double().cpu() * ll, torch.zeros_like(ll))
        total = total + ll.sum(1)
    total.sum().backward()
    out = [total.detach().numpy(), t_ic.grad.numpy().reshape(ic.shape), t_b.grad.numpy()]
    return out if batched else [out[0][0], out[1][0], out[2][0]]


def _oracle(model, ic, beta):
    return model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64, chunk_rows=128))


def _collective(model, ic, beta):
    with FederatedEngine(model, backend="collective") as eng:
        return [np.asarray(v, dtype=np.float64) for v in eng.evaluate(ic, beta)]


# ----------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("K", [1, 3])
def test_oracle_matches_autograd_of_log_softmax(K):
    rows, P, Cn, groups = [150, 70, 201], 16, 4, [0, 1, 0]
    Xs, ys, ws = _case(rows, P, Cn, seed=1)
    model = GlmShards(Xs, ys, groups=groups, n_groups=2, family="multinomial", n_classes=Cn, n_chains=K, weights=ws)
    ic, beta = _theta(2, P, Cn, K)
    got = _oracle(model, ic, beta)
    want = _explicit_fp64(Xs, ys, ws, groups, ic, beta)
    assert np.all(np.isfinite(got[0]))
    assert got[1].shape == ic.shape and got[2].shape == beta.shape
    np.testing.assert_allclose(got[0], want[0], rtol=1e-12)
    np.testing.assert_allclose(got[1], want[1], rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(got[2], want[2], rtol=1e-10, atol=1e-10)


def test_oracle_matches_scipy_logsumexp_and_finite_differences():
    import scipy.special

    rows, P, Cn = [90, 60], 8, 3
    Xs, ys, ws = _case(rows, P, Cn, seed=2, n_masked=0)
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family="multinomial", n_classes=Cn, weights=ws)
    Xn = [X.double().numpy() for X in Xs]
    yn = [y.numpy().astype(int) for y in ys]
    wn = [w.double().numpy() if w is not None else np.ones(len(y)) for w, y in zip(ws, ys)]

    def truth(ic, beta):
        total = 0.0
        for g, (X, y, w) in enumerate(zip(Xn, yn, wn)):
            eta = X @ beta + ic[g]
            total += np.sum(w * (eta[np.arange(len(y)), y] - scipy.special.logsumexp(eta, axis=1)))
        return total

    ic, beta = [v.astype(np.float64) for v in _theta(2, P, Cn)]
    got = _oracle(model, ic, beta)
    np.testing.assert_allclose(got[0], truth(ic, beta), rtol=1e-12)
    eps = 1e-6
    for arr, grad in ((ic, got[1]), (beta, got[2])):
        fd = np.zeros_like(arr)
        for idx in np.ndindex(arr.shape):
            orig = arr[idx]
            arr[idx] = orig + eps
            hi = truth(ic, beta)
            arr[idx] = orig - eps
            lo = truth(ic, beta)
            arr[idx] = orig
            fd[idx] = (hi - lo) / (2 * eps)
        np.testing.assert_allclose(grad, fd, rtol=1e-6, atol=1e-6)


def test_two_classes_with_a_zero_column_are_the_logistic_model():
    rows, P = [130, 77], 16
    Xs, ys, ws = _case(rows, P, 2, seed=3)
    multi = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family="multinomial", n_classes=2, weights=ws)
    ys_logit = [torch.nan_to_num(y).clamp(0, 1) for y in ys]   # masked rows: any finite response
    logit = GlmShards(Xs, ys_logit, groups=[0, 1], n_groups=2, weights=ws)
    ic_b, b = _theta(2, P, 1)
    ic, beta = np.zeros((2, 2)), np.zeros((P, 2))
    ic[:, 1], beta[:, 1] = ic_b[:, 0], b[:, 0]
    m = _oracle(multi, ic, beta)
    lg = logit.unpack_result(logit.reference_partial([ic_b[:, 0], b[:, 0]], dtype=torch.float64))
    np.testing.assert_allclose(m[0], lg[0], rtol=1e-12)
    np.testing.assert_allclose(m[1][:, 1], lg[1], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(m[2][:, 1], lg[2], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(m[1][:, 0], -m[1][:, 1], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(m[2][:, 0], -m[2][:, 1], rtol=1e-12, atol=1e-12)


def test_shift_invariance_and_gradients_sum_to_zero_over_classes():
    rows, P, Cn = [100, 50], 8, 5
    Xs, ys, ws = _case(rows, P, Cn, seed=4)
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family="multinomial", n_classes=Cn, weights=ws)
    ic, beta = _theta(2, P, Cn)
    rng = np.random.default_rng(5)
    a = _oracle(model, ic, beta)
    b = _oracle(model, ic + rng.normal(size=(2, 1)), beta + rng.normal(size=(P, 1)) * 0.1)
    np.testing.assert_allclose(a[0], b[0], rtol=1e-10)
    for g in (a[1], a[2], b[1], b[2]):
        scale = np.abs(g).max()
        np.testing.assert_allclose(g.sum(axis=1), 0.0, atol=1e-10 * scale)


@pytest.mark.parametrize("K", [1, 4])
def test_collective_backend_equals_the_oracle(K):
    rows, P, Cn = [300, 45, 129], 24, 3
    Xs, ys, ws = _case(rows, P, Cn, seed=6)
    model = GlmShards(Xs, ys, groups=[0, 1, 1], n_groups=2, family="multinomial", n_classes=Cn, n_chains=K,
                      weights=ws)
    ic, beta = _theta(2, P, Cn, K)
    got, want = _collective(model, ic, beta), _oracle(model, ic, beta)
    for u, v in zip(got, want):
        assert u.shape == v.shape and np.all(np.isfinite(u))
        np.testing.assert_allclose(u, v, rtol=1e-5, atol=1e-4)


def test_multinomial_validation():
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ys = [torch.zeros(10), torch.full((6,), 2.0)]
    ok = dict(family="multinomial", n_classes=3)
    GlmShards(Xs, ys, **ok)
    for n_classes in (None, 1, 17):
        with pytest.raises(ValueError, match="n_classes"):
            GlmShards(Xs, ys, family="multinomial", n_classes=n_classes)
    with pytest.raises(ValueError, match="n_chains x n_classes"):
        GlmShards(Xs, ys, family="multinomial", n_classes=4, n_chains=5)
    GlmShards(Xs, ys, family="multinomial", n_classes=4, n_chains=4)
    for kernel in ("simt", "generic", "fp8"):
        with pytest.raises(ValueError, match="tensor-core kernel only"):
            GlmShards(Xs, ys, kernel=kernel, **ok)
    with pytest.raises(ValueError, match="tensor-core kernel only"):
        Fp8GlmShards.from_dense([torch.randn(10, 32), torch.randn(6, 32)], ys, family="multinomial")
    with pytest.raises(ValueError, match="offsets"):
        GlmShards(Xs, ys, offsets=[torch.zeros(10), None], **ok)
    with pytest.raises(ValueError, match="multinomial"):
        GlmShards(Xs, ys, n_classes=3)
    for bad in (3.0, -1.0, 0.5, float("nan")):
        y0 = torch.zeros(10)
        y0[4] = bad
        with pytest.raises(ValueError, match="labels of segment 0"):
            GlmShards(Xs, [y0, ys[1]], **ok)
        w0 = torch.ones(10)
        w0[4] = 0.0
        GlmShards(Xs, [y0, ys[1]], weights=[w0, None], **ok)   # a masked row may carry anything
    # shapes outside the tensor-core kernel's: an error, never another kernel
    for X in (torch.randn(10, 12).to(torch.bfloat16), torch.randn(10, 392).to(torch.bfloat16), torch.randn(10, 16)):
        with pytest.raises(ValueError, match="tensor-core kernel only"):
            GlmShards([X], [torch.zeros(10)], **ok).use_tensor_cores()
    assert GlmShards(Xs, ys, kernel="tc", **ok).use_tensor_cores() == 1


def test_sizes_and_flops():
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ys = [torch.zeros(10), torch.zeros(6)]
    m = GlmShards(Xs, ys, n_groups=2, groups=[0, 1], family="multinomial", n_classes=3, n_chains=2,
                  node_ids=[0, 1], n_nodes=2)
    assert m.n_params == 3 * (2 + 16) and m.n_theta_words == 2 * 3 * 18
    assert m.n_vals == 2 * 2 * 3 * (1 + 2 + 16)
    assert m.flops_per_eval() == 4 * 16 * 16 * 2 * 3
    assert m.bytes_per_eval() == GlmShards(Xs, ys).bytes_per_eval()
    assert m.per_node(np.zeros(m.n_vals)).shape == (2, 2, 1 + 2 * 3 + 16 * 3)


@pytest.mark.parametrize("K,G", [(1, 1), (1, 2), (4, 2)])
def test_pack_unpack_and_words_round_trip(K, G):
    P, Cn = 8, 3
    Xs, ys, _ = _case([20] * G, P, Cn, seed=7, n_masked=0, weighted=False)
    model = GlmShards(Xs, ys, groups=list(range(G)), n_groups=G, family="multinomial", n_classes=Cn, n_chains=K)
    ic, beta = _theta(G, P, Cn, K, scale=1.0)
    if K == 1 and G == 1:
        ic = ic.reshape(Cn)   # [C] is accepted for one group
    words = np.zeros(model.n_theta_words, dtype=np.uint32)
    ctx = model.pack_theta([ic, beta], words)
    assert ctx == model.call_context([ic, beta]) == (K > 1, ic.shape)
    # the kernel's layout: row k C + c = (intercept[:, c], beta[:, c]) of chain k
    th = words.view(np.float32).reshape(K * Cn, G + P)
    ic_k, b_k = ic.reshape(K, G, Cn), beta.reshape(K, P, Cn)
    for k in range(K):
        for c in range(Cn):
            assert np.array_equal(th[k * Cn + c, :G], ic_k[k, :, c]) and np.array_equal(th[k * Cn + c, G:], b_k[k, :, c])
    ic2, b2 = default_inputs_from_words(model, words)
    assert np.array_equal(ic2.reshape(ic.shape), ic) and np.array_equal(b2, beta)
    words2 = np.zeros_like(words)
    model.pack_theta([ic2, b2], words2)
    assert np.array_equal(words, words2)
    # unpack: block k C + c of the raw vector holds [LL, gi[G], g[P]] of chain k, class c
    raw = np.arange(model.n_vals, dtype=np.float64).reshape(K, Cn, 1 + G + P)
    logp, d_ic, d_b = model.unpack_result(raw.reshape(-1), ctx)
    assert d_ic.shape == ic.shape and d_b.shape == beta.shape
    np.testing.assert_array_equal(np.reshape(logp, -1), raw[:, :, 0].sum(1))
    np.testing.assert_array_equal(d_ic.reshape(K, G, Cn), raw[:, :, 1 : 1 + G].transpose(0, 2, 1))
    np.testing.assert_array_equal(d_b.reshape(K, P, Cn), raw[:, :, 1 + G :].transpose(0, 2, 1))


def test_glm_batch_fn_splits_theta_for_the_multinomial_model():
    from pytensor_federated_b200.sampling import glm_batch_fn

    P, Cn, G = 8, 3, 2
    Xs, ys, ws = _case([60, 40], P, Cn, seed=8)
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=G, family="multinomial", n_classes=Cn, n_chains=2, weights=ws)
    rng = np.random.default_rng(9)
    theta = rng.normal(size=(3, Cn * (G + P))) * 0.1
    with FederatedEngine(model, backend="collective") as eng:
        logp, grad = glm_batch_fn(eng, G)(theta)
    assert logp.shape == (3,) and grad.shape == theta.shape
    single = GlmShards(Xs, ys, groups=[0, 1], n_groups=G, family="multinomial", n_classes=Cn, weights=ws)
    for i in range(3):
        want = _oracle(single, theta[i, : G * Cn].reshape(G, Cn), theta[i, G * Cn :].reshape(P, Cn))
        np.testing.assert_allclose(logp[i], want[0], rtol=1e-5)
        np.testing.assert_allclose(grad[i], np.concatenate([want[1].ravel(), want[2].ravel()]), rtol=1e-4, atol=1e-4)


def test_synth_multinomial_shard():
    X, y, beta = synth_multinomial_shard(3000, 16, 4, seed=1, device="cpu", chunk_rows=1024)
    assert X.dtype == torch.bfloat16 and X.shape == (3000, 16) and beta.shape == (16, 4)
    assert y.dtype == torch.float32 and set(np.unique(y.numpy())) <= {0.0, 1.0, 2.0, 3.0}
    X2, y2, _ = synth_multinomial_shard(3000, 16, 4, seed=1, device="cpu", chunk_rows=1024)
    assert torch.equal(X, X2) and torch.equal(y, y2)


# ----------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from pytensor_federated_b200.ops import native

    native.load()  # a GPU box without the native library is a failure, not a skip
    return torch.device("cuda:0")


def _run(model, ic, beta, repeats=1):
    with FederatedEngine(model) as eng:
        out = [[np.asarray(v).copy() for v in eng.evaluate(ic, beta)] for _ in range(repeats)]
    return out[0] if repeats == 1 else out


def _check(got, want, rtol_ll, rtol_g, atol_ic, atol_b):
    assert all(np.all(np.isfinite(g)) for g in got)
    for u, v in zip(got, want):
        assert np.shape(u) == np.shape(v)
    np.testing.assert_allclose(got[0], want[0], rtol=rtol_ll)
    np.testing.assert_allclose(got[1], want[1], rtol=rtol_g, atol=atol_ic)
    np.testing.assert_allclose(got[2], want[2], rtol=rtol_g, atol=atol_b)


@pytest.mark.parametrize("weighted", [True, False])
@pytest.mark.parametrize("Cn,K", [(2, 1), (2, 2), (3, 1), (4, 1), (2, 8), (3, 5), (4, 4), (5, 1), (16, 1)])
@pytest.mark.parametrize("P", [256, 200, 8])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_multinomial_matches_oracle(dev, Cn, K, P, weighted):
    """K C <= 4, <= 8 and <= 16 select the kernel's three SOFTMAX buckets; ``weighted`` its ROWS variant."""
    rows = [128 * 37, 77, 4099, 1]
    Xs, ys, ws = _case(rows, P, Cn, seed=Cn + K + P, device=dev, weighted=weighted, n_masked=5 if weighted else 0)
    model = GlmShards(Xs, ys, groups=[0, 1, 0, 1], n_groups=2, family="multinomial", n_classes=Cn, n_chains=K,
                      kernel="auto", weights=ws)
    assert model.has_row_data == weighted
    ic, beta = _theta(2, P, Cn, K)
    got = _run(model, ic, beta)
    assert model.selected_kernel == "tc"
    _check(got, _oracle(model, ic, beta), 2e-5, 1e-4, 2e-3, 2e-3 * np.sqrt(sum(rows)) if K == 1 else 0.2)


@pytest.mark.parametrize("Cn,K,weighted", [(2, 1, False), (3, 1, True), (2, 2, False), (4, 2, True)])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_multinomial_with_many_groups_matches_oracle(dev, Cn, K, weighted):
    """A hierarchical model with 300 intercepts per class: the intercept table is KC x G floats, and the lanes'
    columns past K C (up to 7 in the KC = 4 bucket) must not index past it."""
    G, P = 300, 256
    rows = [128 * 9 + 5, 999, 64, 1, 3000]
    groups = [0, 299, 150, 7, 299]
    Xs, ys, ws = _case(rows, P, Cn, seed=40 + Cn + K, device=dev, weighted=weighted, n_masked=5 if weighted else 0)
    model = GlmShards(Xs, ys, groups=groups, n_groups=G, family="multinomial", n_classes=Cn, n_chains=K,
                      kernel="tc", weights=ws)
    ic, beta = _theta(G, P, Cn, K)
    got = _run(model, ic, beta)
    want = _oracle(model, ic, beta)
    _check(got, want, 2e-5, 1e-4, 2e-3, 2e-3 * np.sqrt(sum(rows)) if K == 1 else 0.2)
    unused = np.ones(G, dtype=bool)
    unused[groups] = False
    assert np.all(got[1][..., unused, :] == 0.0)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_two_classes_with_a_zero_column_are_the_logistic_kernel(dev):
    rows, P = [128 * 30 + 9, 5000, 77], 256
    Xs, ys, ws = _case(rows, P, 2, seed=11, device=dev)
    ys_logit = [torch.nan_to_num(y).clamp(0, 1) for y in ys]
    multi = GlmShards(Xs, ys, groups=[0, 1, 0], n_groups=2, family="multinomial", n_classes=2, kernel="tc", weights=ws)
    logit = GlmShards(Xs, ys_logit, groups=[0, 1, 0], n_groups=2, kernel="tc", weights=ws)
    ic_b, b = _theta(2, P, 1)
    ic, beta = np.zeros((2, 2), np.float32), np.zeros((P, 2), np.float32)
    ic[:, 1], beta[:, 1] = ic_b[:, 0], b[:, 0]
    m, lg = _run(multi, ic, beta), _run(logit, ic_b[:, 0], b[:, 0])
    np.testing.assert_allclose(m[0], lg[0], rtol=2e-5)
    np.testing.assert_allclose(m[1][:, 1], lg[1], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(m[2][:, 1], lg[2], rtol=1e-4, atol=0.2)
    np.testing.assert_allclose(m[1][:, 0], -m[1][:, 1], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(m[2][:, 0], -m[2][:, 1], rtol=1e-4, atol=0.2)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_multinomial_evaluations_are_bit_reproducible(dev):
    rows = [40_000, 25_000, 33_333, 128, 19_999]
    Xs, ys, ws = _case(rows, 256, 4, seed=12, device=dev)
    model = GlmShards(Xs, ys, groups=[0, 1, 2, 1, 0], n_groups=3, family="multinomial", n_classes=4, n_chains=2,
                      kernel="tc", weights=ws)
    ic, beta = _theta(3, 256, 4, 2)
    runs = _run(model, ic, beta, repeats=10)
    for run in runs[1:]:
        for u, v in zip(runs[0], run):
            assert np.array_equal(u, v)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_node_federation_multinomial_blocks_equal_single_node_models(dev):
    from pytensor_federated_b200.federation import NodeFederation

    rows = [20_000, 128 * 33, 7777]
    node_ids, groups, Cn = [0, 1, 1], [0, 1, 0], 3
    Xs, ys, ws = _case(rows, 256, Cn, seed=13, device=dev)
    model = GlmShards(Xs, ys, groups=groups, n_groups=2, family="multinomial", n_classes=Cn, kernel="tc",
                      node_ids=node_ids, n_nodes=2, weights=ws)
    ic, beta = _theta(2, 256, Cn)
    with FederatedEngine(model) as eng:
        n0 = eng.kernel_launches
        blocks = model.per_node(eng.evaluate_raw([ic, beta]))
        assert eng.kernel_launches - n0 == 1
        fed = NodeFederation(eng)
        res = fed.evaluate_nodes({0: (ic, beta), 1: (ic, beta)})
        total = fed.all_nodes_func()(ic, beta)
    for node in (0, 1):
        segs = [i for i, n in enumerate(node_ids) if n == node]
        single = GlmShards([Xs[i] for i in segs], [ys[i] for i in segs], groups=[groups[i] for i in segs], n_groups=2,
                           family="multinomial", n_classes=Cn, kernel="tc", weights=[ws[i] for i in segs])
        want = _run(single, ic, beta)
        np.testing.assert_allclose(blocks[node, 0, 0], want[0], rtol=2e-5)
        np.testing.assert_allclose(blocks[node, 0, 1 : 1 + 2 * Cn], want[1].ravel(), rtol=1e-4, atol=2e-3)
        np.testing.assert_allclose(blocks[node, 0, 1 + 2 * Cn :], want[2].ravel(), rtol=1e-4, atol=0.5)
        np.testing.assert_allclose(res[node][0], blocks[node, 0, 0], rtol=1e-12)
        assert res[node][1][0].shape == (2, Cn) and res[node][1][1].shape == (256, Cn)
        np.testing.assert_allclose(res[node][1][1], want[2], rtol=1e-4, atol=0.5)
    np.testing.assert_allclose(total[0], blocks[:, 0, 0].sum(), rtol=1e-12)
    assert total[1][1].shape == (256, Cn)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_lock_step_hmc_on_a_multinomial_engine(dev):
    from pytensor_federated_b200.sampling import glm_batch_fn, hmc_sample_batched

    Cn, K, P = 3, 4, 16
    X, y, _ = synth_multinomial_shard(20_000, P, Cn, seed=3, device=dev)
    model = GlmShards([X], [y], family="multinomial", n_classes=Cn, n_chains=K, kernel="tc")
    with FederatedEngine(model) as eng:
        res = hmc_sample_batched(glm_batch_fn(eng, 1), np.zeros((K, Cn * (1 + P))), draws=5, tune=5, n_leapfrog=4,
                                 step_size=1e-3, seed=1)
        assert eng.n_evals == res.n_batched_evals
    assert res.samples.shape[-1] == Cn * (1 + P) and np.all(np.isfinite(res.samples))


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_runtime_rejects_the_multinomial_family_outside_the_tc_kernel(dev):
    """The C ABI refuses what the Python layer never sends: family 3 on a CUDA-core kernel (which would take an
    unknown family for the Gaussian one), bad class counts, offsets, and n_classes on the other families."""
    from pytensor_federated_b200.ops import native

    Xs, ys, _ = _case([256], 16, 2, seed=14, device=dev, n_masked=0, weighted=False)
    model = GlmShards(Xs, ys, kernel="simt")
    with FederatedEngine(model) as eng:
        lib, h = eng._lib, eng._handle
        Xp, yp = native.void_p_array([Xs[0].data_ptr()]), native.void_p_array([ys[0].data_ptr()])
        rows, grp = (C.c_longlong * 1)(256), (C.c_int * 1)(0)
        offs = native.void_p_array([ys[0].data_ptr()])

        def set_glm(n_chains, family, code, n_classes, offsets=None):
            return int(lib.b200_engine_set_glm(h, 1, Xp, yp, None, rows, grp, 16, 16, 1, n_chains, family, code, None, 1,
                                               offsets, None, n_classes))

        for code in (0, 2, 3, 4):
            assert set_glm(2, 3, code, 2) != 0
            assert "tensor-core kernel only" in native.last_error()
        assert set_glm(2, 3, 1, 1) != 0 and "n_classes" in native.last_error()
        assert set_glm(17, 3, 1, 17) != 0 and "n_classes" in native.last_error()
        assert set_glm(3, 3, 1, 2) != 0 and "n_chains" in native.last_error()
        assert set_glm(2, 3, 1, 2, offs) != 0 and "offsets" in native.last_error()
        assert set_glm(1, 0, 0, 2) != 0 and "n_classes must be 1" in native.last_error()
        # the engine still evaluates its own model
        ic, beta = np.float32(0.1), np.zeros(16, np.float32)
        got = eng.evaluate(ic, beta)
    want = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)


def _build_multinomial_model(rank, world, dev):
    Xs, ys, ws = _case([30_000 + 17 * rank, 999], 256, 4, seed=50 + rank, device=dev)
    return GlmShards(Xs, ys, groups=[rank % 2, 1 - rank % 2], n_groups=2, family="multinomial", n_classes=4,
                     n_chains=2, kernel="tc", weights=ws)


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.timeout(900)
def test_two_rank_multinomial_federation_matches_oracle():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from pytensor_federated_b200.federation import launch_federation

    ic, beta = _theta(2, 256, 4, 2)
    dev = torch.device("cuda:0")
    models = [_build_multinomial_model(r, 2, dev) for r in range(2)]
    want = models[0].unpack_result(sum(m.reference_partial([ic, beta], dtype=torch.float64) for m in models),
                                   models[0].call_context([ic, beta]))
    del models
    with launch_federation(_build_multinomial_model, 2, timeout=30.0) as eng:
        got = eng.evaluate(ic, beta)
    _check(got, want, 2e-5, 1e-4, 2e-3, 0.5)
