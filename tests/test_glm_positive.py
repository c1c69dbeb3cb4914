"""Positive continuous responses with a model for the mean: ``GlmShards(Xs, ys, family="gamma" | "inverse_gaussian")``,
log link, ``log_dispersion`` = the log of the shape (nu, lambda).

CPU tests check the fp64 oracle and the collective backend against independent formulas (scipy's densities, central
differences of them), the Weibull family the gamma one reduces to at nu = 1, validation, the model's packing and the
synthetic data; GPU tests check the tensor-core kernel against that oracle within a rounding bound derived from the
magnitudes of each sum's terms, per row across the families' domain, and bit for bit against itself."""
import ctypes as C

import numpy as np
import pytest
import torch

from pytensor_federated_b200.models import Fp8GlmShards, GlmShards, synth_positive_shard
from pytensor_federated_b200.models.glm import FAMILIES as CODES
from pytensor_federated_b200.models.glm import _DISPERSION_TERMS, _gamma_shape_terms
from pytensor_federated_b200.parallel import FederatedEngine
from pytensor_federated_b200.parallel.engine import default_inputs_from_words

FAMILIES = ("gamma", "inverse_gaussian")
# log shape of the GPU tests: nu / lambda from e^-3 to e^9, and 1e4
LOG_SHAPE = np.array([-3.0, -1.0, 0.0, 1.0, 3.0, 6.0, 9.0, np.log(1e4)])


# ----------------------------------------------------------------------------------------------- fixtures
def _beta_true(P):
    return np.random.default_rng(1000 + P).normal(size=P) * 0.01


def _draw(rng, family, mu, shape):
    """y with mean mu and shape nu (gamma) or lambda (inverse Gaussian), float64."""
    if family == "gamma":
        return rng.gamma(shape, mu / shape)
    return rng.wald(mu, shape)


def _case(rows, P, family, *, seed=0, device="cpu", n_masked=5, weighted=True, offsets=True, shape=2.0,
          icpt=(0.4, -1.0)):
    """Ragged bf16 segments with responses drawn from the family at ``intercept = icpt[segment % 2]``, ``beta =
    _beta_true(P)`` and ``shape``.  With ``weighted``, every segment but the last has weights; the first ``n_masked``
    rows of segment 0 have weight 0 and carry NaN, a negative, a zero and an infinite y.  With ``offsets``, every
    segment but the second has offsets.  Returns ``(Xs, ys, weights, offsets)``."""
    rng = np.random.default_rng(seed)
    Xs, ys, ws, os_ = [], [], [], []
    for si, n in enumerate(rows):
        X = torch.tensor(rng.normal(size=(n, P)), dtype=torch.float32).to(torch.bfloat16)
        o = rng.uniform(-0.5, 0.5, size=n)
        eta = X.double().numpy() @ _beta_true(P) + icpt[si % 2] + (o if offsets else 0.0)
        y = np.maximum(_draw(rng, family, np.exp(eta), shape), 1e-30)
        w = rng.uniform(0.2, 2.0, size=n)
        if si == 0 and n_masked:
            w[:n_masked] = 0.0
            y[:4] = [np.nan, -1.0, 0.0, np.inf][: min(4, n_masked)]
        Xs.append(X.to(device))
        ys.append(torch.tensor(y, dtype=torch.float32, device=device))
        ws.append(torch.tensor(w, dtype=torch.float32, device=device) if weighted and si < len(rows) - 1 else None)
        os_.append(torch.tensor(o, dtype=torch.float32, device=device) if offsets and si != 1 else None)
    return Xs, ys, ws, os_


def _theta(G, P, K=1, log_shape=np.log(2.0), seed=3, scale=0.002):
    """``(intercept, beta, log_shape)`` near the parameters the data were drawn at; batched (``[K, G]``, ``[K, P]``,
    ``[K]``) for K > 1, where ``log_shape`` may give one value per chain."""
    rng = np.random.default_rng(seed)
    b0 = _beta_true(P)
    base = np.resize([0.4, -1.0], G)
    if K == 1:
        return ((base + rng.normal(size=G) * 0.02).astype(np.float32),
                (b0 + rng.normal(size=P) * scale).astype(np.float32), np.float32(log_shape))
    return ((base + rng.normal(size=(K, G)) * 0.02).astype(np.float32),
            (b0 + rng.normal(size=(K, P)) * scale).astype(np.float32),
            np.broadcast_to(np.asarray(log_shape, dtype=np.float32), (K,)).copy())


def _model(Xs, ys, ws, os_, family, **kw):
    return GlmShards(Xs, ys, family=family, weights=ws, offsets=os_, **kw)


def _oracle(model, *inputs, chunk_rows=128):
    return model.unpack_result(model.reference_partial(list(inputs), dtype=torch.float64, chunk_rows=chunk_rows))


def _collective(model, *inputs):
    with FederatedEngine(model, backend="collective") as eng:
        return [np.asarray(v, dtype=np.float64) for v in eng.evaluate(*inputs)]


def _scipy_logpdf(family, y, mu, shape):
    import scipy.stats

    if family == "gamma":
        return scipy.stats.gamma(a=shape, scale=mu / shape).logpdf(y)
    return scipy.stats.invgauss(mu=mu / shape, scale=shape).logpdf(y)


# ----------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("family", FAMILIES)
def test_terms_match_scipy_across_the_domain(family):
    """Per row, on a grid of shape e^-3 .. e^9, mu 1e-4 .. 1e4 and y 1e-6 .. 1e6: ll is scipy's logpdf, dll/deta and
    dll/da are central differences of it, in fp64; the fp32 terms (the collective backend's) stay within a few
    hundred fp32 roundings of the terms' magnitudes."""
    fn = _DISPERSION_TERMS[family]
    a = np.linspace(-3.0, 9.0, 13)
    mu = np.geomspace(1e-4, 1e4, 9)
    y = np.geomspace(1e-6, 1e6, 25)
    A, M, Y = (v.reshape(-1) for v in np.meshgrid(a, mu, y, indexing="ij"))
    eta = np.log(M)
    ll, r, q = (t.numpy() for t in fn(torch.tensor(Y), torch.tensor(eta), torch.tensor(A)))
    want = _scipy_logpdf(family, Y, M, np.exp(A))
    np.testing.assert_allclose(ll, want, rtol=1e-11, atol=1e-11)
    # five-point central differences of scipy's logpdf (truncation O(h^4)), in eta and in a; their rounding is
    # ~1e-16 / h of the magnitudes scipy forms: |ll|, nu (1 + |a|) and, for the inverse Gaussian, lambda / mu
    h = 1e-3
    for got, (d_eta, d_a) in ((r, (1, 0)), (q, (0, 1))):
        f = lambda s: _scipy_logpdf(family, Y, np.exp(eta + s * h * d_eta), np.exp(A + s * h * d_a))
        fd = (8 * (f(1) - f(-1)) - (f(2) - f(-2))) / (12 * h)
        nu = np.exp(A)
        noise = 1e-10 * np.maximum(np.maximum(1.0, np.abs(want)), nu * (1 + np.abs(A))) + 1e-12 * nu / M
        assert np.all(np.abs(got - fd) <= 1e-6 * np.abs(fd) + noise)
    # fp32 (the collective backend's terms) against fp64 at the same fp32 inputs
    l32, r32, q32 = (t.double().numpy() for t in fn(torch.tensor(Y, dtype=torch.float32),
                                                     torch.tensor(eta, dtype=torch.float32),
                                                     torch.tensor(A, dtype=torch.float32)))
    y32, eta32, a32 = (torch.tensor(v, dtype=torch.float32).double() for v in (Y, eta, A))
    l64, r64, q64 = (t.numpy() for t in fn(y32, eta32, a32))   # the fp32 inputs, evaluated in fp64
    # per row: a few roundings of the parts each value is formed from, plus its slope in eta times the error of z
    lt = np.abs(np.log(Y))
    dz = 2.0 ** -21 * (1.0 + lt + np.abs(eta))
    mag = np.abs(l64) + lt + np.abs(q64) + 5.0 + np.abs(A)
    slope = _slope(family, y32, eta32, a32).numpy()
    assert np.all(np.abs(l32 - l64) <= 2.0 ** -18 * mag + np.abs(r64) * dz)
    assert np.all(np.abs(q32 - q64) <= 2.0 ** -18 * mag + np.abs(r64) * dz)
    assert np.all(np.abs(r32 - r64) <= 2.0 ** -18 * np.abs(r64) + slope * dz)


def test_gamma_shape_terms_are_continuous_at_the_series_switch():
    """C(nu) and Q(nu) switch from lgamma / digamma to their Stirling series at nu = 1e3; both sides agree."""
    a = torch.tensor(np.log([999.999999, 1000.0, 1e4, 1e6, 0.05, 1.0, 8.0]), dtype=torch.float64)
    nu, Cn, Q = _gamma_shape_terms(a)
    direct_C = nu * torch.log(nu) - nu - torch.lgamma(nu)
    direct_Q = nu * (torch.log(nu) - torch.digamma(nu))
    np.testing.assert_allclose(Cn.numpy(), direct_C.numpy(), rtol=1e-9)
    np.testing.assert_allclose(Q.numpy()[[0, 1, 4, 5, 6]], direct_Q.numpy()[[0, 1, 4, 5, 6]], rtol=1e-8)
    np.testing.assert_allclose(Q.numpy()[3], 0.5 + 1 / 12e6, rtol=1e-12)


@pytest.mark.parametrize("log_shape", [-3.0, 0.0, 3.0, 9.0])
@pytest.mark.parametrize("family", FAMILIES)
def test_oracle_matches_scipy_and_finite_differences(family, log_shape):
    """Three groups at mu ~ 1e-4, 1 and 1e4, offsets, weights with masked NaN / negative / zero / inf rows, and two
    nodes: each node's LL is the weighted sum of scipy's logpdf, and its gradients are central differences of it."""
    P, G = 8, 3
    rows, groups, node_ids = [60, 45, 50, 33], [0, 1, 2, 1], [0, 1, 1, 0]
    rng = np.random.default_rng(int(log_shape * 10) + 100)
    ic = np.log([1e-4, 1.0, 1e4]) + rng.normal(size=G) * 0.1
    beta = rng.normal(size=P) * 0.1
    Xs, ys, ws, os_ = [], [], [], []
    for si, n in enumerate(rows):
        X = torch.tensor(rng.normal(size=(n, P)), dtype=torch.float32).to(torch.bfloat16)
        o = rng.uniform(-0.3, 0.3, size=n)
        eta = X.double().numpy() @ beta + ic[groups[si]] + o
        # y from 1e-6 to 1e6, at most 20 e-folds from the mean
        y = np.exp(np.clip(eta + rng.uniform(-20, 20, size=n), np.log(1e-6), np.log(1e6)))
        w = rng.uniform(0.2, 2.0, size=n)
        if si == 0:
            w[:4] = 0.0
            y[:4] = [np.nan, -1.0, 0.0, np.inf]
        Xs.append(X)
        ys.append(torch.tensor(y, dtype=torch.float32))
        ws.append(torch.tensor(w, dtype=torch.float32))
        os_.append(torch.tensor(o, dtype=torch.float32))
    model = GlmShards(Xs, ys, groups=groups, n_groups=G, family=family, weights=ws, offsets=os_, node_ids=node_ids,
                      n_nodes=2)
    Xn = [X.double().numpy() for X in Xs]
    yn = [y.double().numpy() for y in ys]
    wn = [w.double().numpy() for w in ws]
    on = [o.double().numpy() for o in os_]

    def truth(ic, beta, ls, node):
        total = 0.0
        for si in range(len(rows)):
            if node_ids[si] != node:
                continue
            keep = wn[si] != 0
            mu = np.exp(Xn[si] @ beta + ic[groups[si]] + on[si])[keep]
            total += np.sum(wn[si][keep] * _scipy_logpdf(family, yn[si][keep], mu, np.exp(ls[()])))
        return total

    ls = np.asarray(log_shape)
    blocks = model.per_node(model.reference_partial([ic, beta, ls], dtype=torch.float64, chunk_rows=128))
    assert blocks.shape == (2, 1, 2 + G + P)
    for node in (0, 1):
        got = blocks[node, 0]
        np.testing.assert_allclose(got[0], truth(ic, beta, ls, node), rtol=1e-10)
        for arr, sl in ((ic, slice(1, 1 + G)), (beta, slice(1 + G, 1 + G + P)), (ls, slice(1 + G + P, None))):
            fd = np.zeros(arr.size)
            for i, idx in enumerate(np.ndindex(arr.shape)):
                orig = arr[idx].copy()
                h = 1e-6
                arr[idx] = orig + h
                hi = truth(ic, beta, ls, node)
                arr[idx] = orig - h
                lo = truth(ic, beta, ls, node)
                arr[idx] = orig
                fd[i] = (hi - lo) / (2 * h)
            np.testing.assert_allclose(got[sl], fd, rtol=1e-5, atol=1e-6 * np.max(np.abs(fd)))


def _gamma_weibull_pair(rows, P, *, seed, device="cpu", weighted=True, **kw):
    """A gamma model and the Weibull model on the same data with every row an event."""
    Xs, ys, ws, os_ = _case(rows, P, "gamma", seed=seed, device=device, weighted=weighted, offsets=weighted,
                            n_masked=5 if weighted else 0, shape=1.0)
    groups = [0, 1, 0][: len(rows)]
    ga = _model(Xs, ys, ws, os_, "gamma", groups=groups, n_groups=2, **kw)
    wb = _model(Xs, ys, ws, os_, "weibull", groups=groups, n_groups=2, **kw)
    return ga, wb


@pytest.mark.parametrize("weighted", [False, True])
def test_gamma_at_unit_shape_is_weibull_at_unit_sigma(weighted):
    """At nu = 1 the gamma family is the exponential distribution with mean mu, as is the Weibull family at s = 0
    with every row an event: the same LL and the same intercept and beta gradients."""
    ga, wb = _gamma_weibull_pair([130, 77, 64], 16, seed=4, weighted=weighted)
    ic, beta, _ = _theta(2, 16)
    a, b = _oracle(ga, ic, beta, np.float32(0.0)), _oracle(wb, ic, beta, np.float32(0.0))
    np.testing.assert_allclose(a[0], b[0], rtol=1e-12)
    np.testing.assert_allclose(a[1], b[1], rtol=1e-10, atol=1e-12 * np.max(np.abs(b[1])))
    np.testing.assert_allclose(a[2], b[2], rtol=1e-10, atol=1e-12 * np.max(np.abs(b[2])))


@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("family", FAMILIES)
def test_collective_backend_equals_the_oracle(family, K):
    rows, P = [300, 45, 129], 24
    Xs, ys, ws, os_ = _case(rows, P, family, seed=6)
    model = _model(Xs, ys, ws, os_, family, groups=[0, 1, 1], n_groups=2, n_chains=K)
    ic, beta, ls = _theta(2, P, K, log_shape=[-0.5, 0.7, 2.0, 5.0][:K] if K > 1 else 0.7)
    got, want = _collective(model, ic, beta, ls), _oracle(model, ic, beta, ls)
    for u, v in zip(got, want):
        assert np.shape(u) == np.shape(v) and np.all(np.isfinite(u))
        np.testing.assert_allclose(u, v, rtol=1e-4, atol=1e-3 * max(1.0, np.max(np.abs(v))))


def test_validation():
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ys = [torch.full((10,), 2.0), torch.full((6,), 0.5)]
    for family in FAMILIES:
        GlmShards(Xs, ys, family=family)
        GlmShards(Xs, ys, family=family, n_chains=16, offsets=[torch.zeros(10), None], weights=[None, torch.ones(6)])
        for kernel in ("simt", "generic", "fp8"):
            with pytest.raises(ValueError, match="tensor-core kernel only"):
                GlmShards(Xs, ys, family=family, kernel=kernel)
        with pytest.raises(ValueError, match="tensor-core kernel only"):
            Fp8GlmShards.from_dense([torch.randn(10, 32), torch.randn(6, 32)], ys, family=family)
        with pytest.raises(ValueError, match="n_classes"):
            GlmShards(Xs, ys, family=family, n_classes=2)
        with pytest.raises(ValueError, match="events="):
            GlmShards(Xs, ys, family=family, events=[None, None])
        with pytest.raises(ValueError, match="hvp=True is for family"):
            GlmShards(Xs, ys, family=family, hvp=True)
        for X in (torch.randn(10, 12).to(torch.bfloat16), torch.randn(10, 392).to(torch.bfloat16), torch.randn(10, 16)):
            with pytest.raises(ValueError, match="tensor-core kernel only"):
                GlmShards([X], [torch.ones(10)], family=family).use_tensor_cores()
        assert GlmShards(Xs, ys, family=family, kernel="tc").use_tensor_cores() == 1
        for bad in (0.0, -0.0, -1.0, float("nan"), float("inf"), float("-inf")):
            y1 = torch.full((6,), 0.5)
            y1[2] = bad
            with pytest.raises(ValueError, match="responses of segment 1 must be finite and > 0"):
                GlmShards(Xs, [ys[0], y1], family=family)
            w1 = torch.ones(6)
            w1[2] = 0.0
            GlmShards(Xs, [ys[0], y1], family=family, weights=[None, w1])   # a masked row may carry anything
        y0 = torch.full((10,), 2.0)
        y0[3] = 1e-38   # positive subnormal-adjacent values are valid responses
        GlmShards(Xs, [y0, ys[1]], family=family)


def test_the_responses_passed_in_are_read_as_they_are():
    Xs = [torch.randn(10, 16).to(torch.bfloat16)]
    y = torch.linspace(0.5, 3.0, 10)
    m = GlmShards(Xs, [y], family="gamma")
    assert m._layout.kernel_ys[0] is m.ys[0] and torch.equal(m.ys[0], y)


@pytest.mark.parametrize("family", FAMILIES)
def test_sizes_and_flops(family):
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ys = [torch.ones(10), torch.ones(6)]
    m = GlmShards(Xs, ys, n_groups=2, groups=[0, 1], family=family, n_chains=3, node_ids=[0, 1], n_nodes=2)
    assert m.n_inputs == 3 and m.input_shapes == [(2,), (16,), ()]
    assert m.n_params == 2 + 16 + 1 and m.n_theta_words == 3 * 19
    assert m.n_vals == 2 * 3 * (2 + 2 + 16)
    assert m.flops_per_eval() == GlmShards(Xs, ys, n_chains=3).flops_per_eval()
    assert m.bytes_per_eval() == GlmShards(Xs, ys).bytes_per_eval()
    assert m.per_node(np.zeros(m.n_vals)).shape == (2, 3, 2 + 2 + 16)


@pytest.mark.parametrize("K,G", [(1, 1), (1, 2), (4, 2)])
@pytest.mark.parametrize("family", FAMILIES)
def test_pack_unpack_and_words_round_trip(family, K, G):
    P = 8
    Xs, ys, _, _ = _case([20] * G, P, family, seed=7, n_masked=0, weighted=False, offsets=False)
    model = GlmShards(Xs, ys, groups=list(range(G)), n_groups=G, family=family, n_chains=K)
    ic, beta, ls = _theta(G, P, K, log_shape=np.arange(K) - 0.5 if K > 1 else -0.5, scale=1.0)
    if K == 1 and G == 1:
        ic = ic.reshape(())   # a scalar intercept for one group
    words = np.zeros(model.n_theta_words, dtype=np.uint32)
    ctx = model.pack_theta([ic, beta, ls], words)
    assert ctx == model.call_context([ic, beta, ls]) == (K > 1, ic.shape, np.shape(ls))
    th = words.view(np.float32).reshape(K, G + P + 1)
    np.testing.assert_array_equal(th[:, :G], np.reshape(ic, (K, G)))
    np.testing.assert_array_equal(th[:, G : G + P], np.reshape(beta, (K, P)))
    np.testing.assert_array_equal(th[:, G + P], np.reshape(ls, K))
    ic2, b2, ls2 = default_inputs_from_words(model, words)
    assert np.array_equal(ic2.reshape(ic.shape), ic) and np.array_equal(b2, beta) and np.array_equal(ls2, ls)
    theta = np.concatenate([np.reshape(ic, (K, G)), np.reshape(beta, (K, P)), np.reshape(ls, (K, 1))], axis=1)
    for u, v in zip(model.inputs_from_theta(theta), (ic, beta, ls)):
        assert np.array_equal(np.reshape(u, np.shape(v)), v)
    raw = np.arange(model.n_vals, dtype=np.float64).reshape(K, 2 + G + P)
    logp, d_ic, d_b, d_ls = model.unpack_result(raw.reshape(-1), ctx)
    assert d_ic.shape == np.shape(ic) and d_b.shape == beta.shape and np.shape(d_ls) == np.shape(ls)
    np.testing.assert_array_equal(np.reshape(logp, -1), raw[:, 0])
    np.testing.assert_array_equal(np.reshape(d_ic, (K, G)), raw[:, 1 : 1 + G])
    np.testing.assert_array_equal(np.reshape(d_b, (K, P)), raw[:, 1 + G : 1 + G + P])
    np.testing.assert_array_equal(np.reshape(d_ls, K), raw[:, -1])
    np.testing.assert_array_equal(model._layout.fold(raw[None], ctx), raw[None])


@pytest.mark.parametrize("family", FAMILIES)
def test_batched_chains_equal_unbatched_calls(family):
    P, G, K = 16, 2, 3
    Xs, ys, ws, os_ = _case([90, 40], P, family, seed=17)
    one = _model(Xs, ys, ws, os_, family, groups=[0, 1], n_groups=G)
    many = _model(Xs, ys, ws, os_, family, groups=[0, 1], n_groups=G, n_chains=K)
    ic, beta, ls = _theta(G, P, K, log_shape=[-1.0, 0.5, 4.0])
    got = _oracle(many, ic, beta, ls)
    for k in range(K):
        want = _oracle(one, ic[k], beta[k], ls[k])
        for u, v in zip(got, want):
            np.testing.assert_allclose(u[k], v, rtol=1e-13, atol=1e-13 * np.max(np.abs(v)))


@pytest.mark.parametrize("family", FAMILIES)
def test_glm_batch_fn_splits_theta_with_log_shape(family):
    from pytensor_federated_b200.sampling import glm_batch_fn

    P, G = 8, 2
    Xs, ys, ws, os_ = _case([60, 40], P, family, seed=8)
    model = _model(Xs, ys, ws, os_, family, groups=[0, 1], n_groups=G, n_chains=2)
    rng = np.random.default_rng(9)
    theta = np.concatenate([np.array([0.4, -1.0]) + rng.normal(size=(3, G)) * 0.05, rng.normal(size=(3, P)) * 0.01,
                            np.log(2.0) + rng.normal(size=(3, 1)) * 0.1], axis=1)
    with FederatedEngine(model, backend="collective") as eng:
        logp, grad = glm_batch_fn(eng, G)(theta)
    assert logp.shape == (3,) and grad.shape == theta.shape
    single = _model(Xs, ys, ws, os_, family, groups=[0, 1], n_groups=G)
    for i in range(3):
        want = _oracle(single, theta[i, :G], theta[i, G : G + P], theta[i, -1])
        np.testing.assert_allclose(logp[i], want[0], rtol=1e-5)
        np.testing.assert_allclose(grad[i], np.concatenate([want[1], want[2], [want[3]]]), rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("family", FAMILIES)
def test_tc_stages_are_the_dispersion_layouts(family):
    """The new codes take the shared-memory layout of the other dispersion families: one more theta word per chain
    and the dispersion table."""
    from pytensor_federated_b200.ops import native

    lib = native.load()
    code = CODES[family]
    for P, K, G, rows in ((8, 1, 1, 0), (256, 4, 2, 3), (256, 16, 300, 1), (384, 8, 1, 0), (384, 16, 1, 3)):
        got = lib.b200_glm_tc_stages(P, K, G, code, rows)
        assert got == lib.b200_glm_tc_stages(P, K, G, CODES["negative_binomial"], rows)
        assert got == lib.b200_glm_tc_stages(P, K, G, CODES["weibull"], rows)
    assert lib.b200_glm_tc_stages(256, 16, 1, code, 3) >= 2


@pytest.mark.parametrize("family", FAMILIES)
def test_synth_positive_shard(family):
    import scipy.stats

    n, shape = 200_000, 3.0
    X, y, beta = synth_positive_shard(n, 16, family=family, shape=shape, seed=1, device="cpu", chunk_rows=65536)
    assert X.dtype == torch.bfloat16 and X.shape == (n, 16) and beta.shape == (16,)
    assert y.dtype == torch.float32 and bool(torch.all(torch.isfinite(y) & (y > 0)))
    X2, y2, _ = synth_positive_shard(n, 16, family=family, shape=shape, seed=1, device="cpu", chunk_rows=65536)
    assert torch.equal(X, X2) and torch.equal(y, y2)
    # at beta* = 0 every y is a draw at mean e^intercept: its moments and distribution
    mu = np.exp(0.5)
    _, y0, _ = synth_positive_shard(n, 8, family=family, shape=shape, seed=2, device="cpu", beta_scale=0.0,
                                    intercept=0.5)
    v = y0.double().numpy()
    var = mu * mu / shape if family == "gamma" else mu ** 3 / shape
    assert abs(v.mean() - mu) < 5 * np.sqrt(var / n)
    # the sample variance's standard error, from the fourth central moment of the family
    m4 = (3 + (6 / shape if family == "gamma" else 15 * mu / shape)) * var * var
    assert abs(v.var() - var) < 5 * np.sqrt((m4 - var * var) / n)
    dist = (scipy.stats.gamma(a=shape, scale=mu / shape) if family == "gamma"
            else scipy.stats.invgauss(mu=mu / shape, scale=shape))
    assert scipy.stats.kstest(v[:50_000], dist.cdf).pvalue > 1e-3
    # every y is > 0 even where float32 would underflow: a tiny shape, tiny means
    _, yt, _ = synth_positive_shard(20_000, 8, family=family, shape=np.exp(-3.0), seed=3, device="cpu",
                                    intercept=-9.0)
    assert bool(torch.all(torch.isfinite(yt) & (yt > 0)))
    # and the model the data came from fits it: dLL/da at the true shape is ~0 relative to its scale
    m = GlmShards([X], [y], family=family)
    got = _oracle(m, np.float32(0.5), beta.numpy(), np.float32(np.log(shape)), chunk_rows=1 << 16)
    assert abs(got[3]) < 5 * np.sqrt(n)
    with pytest.raises(ValueError, match="family must be"):
        synth_positive_shard(10, 8, family="weibull", shape=1.0, seed=0, device="cpu")


# ----------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from pytensor_federated_b200.ops import native

    native.load()  # a GPU box without the native library is a failure, not a skip
    return torch.device("cuda:0")


def _run(model, inputs_list, raw=False, grid=None):
    """The engine's results (``raw``: the kernel's output blocks) for each set of inputs, one engine."""
    with FederatedEngine(model, grid=grid) as eng:
        if raw:
            return [np.asarray(eng.evaluate_raw(list(inputs)), dtype=np.float64).copy() for inputs in inputs_list]
        return [[np.asarray(v).copy() for v in eng.evaluate(*inputs)] for inputs in inputs_list]


def _slope(family, y, eta, a):
    """|d r / d eta| per row: gamma nu e^z, inverse Gaussian lambda e^-eta |2 e^z - 1|."""
    z = torch.log(y) - eta
    if family == "gamma":
        return torch.exp(a) * torch.exp(z)
    return torch.exp(a) * torch.exp(-eta) * (2 * torch.exp(z) - 1).abs()


def _bound(model, ic, beta, ls):
    """A bound on the kernel's error, per output and in the shapes of the results, from the fp64 magnitudes of the
    terms each one sums.  Per row, eta is off by at most ``d_eta = 2^-18 (1 + |eta| + sum_j |x_j beta_j|)`` (the
    three-term bf16 split of beta keeps 24 bits, the fp32 MMA sums over P), and the kernel's ll, r and q by a few fp32
    roundings of the values they are formed from.  The per-thread fp32 sums of a chunk add at most 64 rows, so
    LL and q get ``2^-16`` of the summed magnitudes plus ``|r| d_eta``; the gradients get ``2^-14`` of ``sum w |r|
    |x|`` (the (hi, lo) bf16 split of r keeps ~2^-17 of it, then fp32 MMA sums) plus ``sum w |dr/deta| d_eta |x|``."""
    fam = model.family
    fn = _DISPERSION_TERMS[fam]
    batched = np.ndim(beta) == 2
    K, G, P = model.n_chains, model.n_groups, model.n_features
    dv = model.device
    icd = torch.tensor(np.reshape(ic, (K, G)), dtype=torch.float64, device=dv)
    bd = torch.tensor(np.reshape(beta, (K, P)), dtype=torch.float64, device=dv)
    ad = torch.tensor(np.reshape(ls, (K,)), dtype=torch.float64, device=dv)
    _, Cn, Q = _gamma_shape_terms(ad)
    if fam == "inverse_gaussian":
        Cn, Q = 0.5 * ad.abs() + 1.0, torch.ones_like(ad)
    t_ll = torch.zeros(K, dtype=torch.float64, device=dv)
    t_q = torch.zeros_like(t_ll)
    t_gi = torch.zeros(K, G, dtype=torch.float64, device=dv)
    t_g = torch.zeros(K, P, dtype=torch.float64, device=dv)
    for si, (X, y, g) in enumerate(zip(model.Xs, model.ys, model.groups)):
        w = model.weights[si]
        keep = torch.ones_like(y, dtype=torch.bool) if w is None else w != 0
        ww = (torch.ones_like(y) if w is None else w).double()[keep].unsqueeze(1)
        Xd = X.double()[keep]
        yy = y.double()[keep].unsqueeze(1)
        eta = Xd @ bd.T + icd[:, g]
        if model.offsets[si] is not None:
            eta = eta + model.offsets[si].double()[keep].unsqueeze(1)
        d_eta = 2.0 ** -18 * (1.0 + eta.abs() + Xd.abs() @ bd.abs().T)
        ll, r, q = fn(yy, eta, ad)
        lt = torch.log(yy).abs()
        s_ll = ll.abs() + lt + Cn.abs() + (q - Q).abs()
        t_ll += (ww * (2.0 ** -16 * s_ll + r.abs() * d_eta)).sum(0)
        t_q += (ww * (2.0 ** -16 * ((q - Q).abs() + Q.abs() + 1.0) + r.abs() * d_eta)).sum(0)
        e = ww * (2.0 ** -14 * r.abs() + _slope(fam, yy, eta, ad) * d_eta)
        t_gi[:, g] += e.sum(0)
        t_g += e.T @ Xd.abs()
    out = [t.cpu().numpy() for t in (t_ll, t_gi, t_g, t_q)]
    return out if batched else [out[0][0], out[1][0], out[2][0], out[3][0]]


def _check(got, want, tol):
    assert all(np.all(np.isfinite(g)) for g in got)
    for u, v, t in zip(got, want, tol):
        assert np.shape(u) == np.shape(v)
        err = np.abs(np.asarray(u, dtype=np.float64) - v)
        assert np.all(err <= t), (np.max(err / t), np.max(err))


@pytest.mark.parametrize("row_data", [True, False])
@pytest.mark.parametrize("P,K", [(P, K) for P in (8, 128, 256, 384) for K in (1, 3, 4, 8, 13, 16) if P < 384 or K <= 8])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_matches_oracle(dev, family, P, K, row_data):
    """K <= 1, 4, 8 and 16 select the kernel's four buckets; ``row_data`` (offsets and weights, masked rows with
    NaN / negative / zero / inf responses) its ROWS variant.  The chains cycle through the shapes e^-3 .. 1e4; with
    K = 1 three of them are evaluated, one launch each.  At P = 384 the 16-column bucket gets one pipeline stage
    (as for every dispersion family), so it runs up to K = 8."""
    rows = [128 * 37, 77, 4099, 1]
    Xs, ys, ws, os_ = _case(rows, P, family, seed=K + P, device=dev, weighted=row_data, offsets=row_data,
                            n_masked=5 if row_data else 0)
    model = _model(Xs, ys, ws, os_, family, groups=[0, 1, 0, 1], n_groups=2, n_chains=K, kernel="auto")
    assert model.has_row_data == row_data
    if K == 1:
        inputs = [_theta(2, P, 1, log_shape=v, seed=5 + i) for i, v in enumerate(LOG_SHAPE[[0, 3, 7]])]
    else:
        inputs = [_theta(2, P, K, log_shape=np.resize(LOG_SHAPE, K))]
    got = _run(model, inputs)
    assert model.selected_kernel == "tc"
    for g, inp in zip(got, inputs):
        _check(g, _oracle(model, *inp, chunk_rows=1 << 20), _bound(model, *inp))


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("K,row_data", [(1, False), (4, True), (13, True)])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_with_many_groups_matches_oracle(dev, family, K, row_data):
    G, P = 300, 256
    rows = [128 * 9 + 5, 999, 64, 1, 3000]
    groups = [0, 299, 150, 7, 299]
    Xs, ys, ws, os_ = _case(rows, P, family, seed=40 + K, device=dev, weighted=row_data, offsets=row_data,
                            n_masked=5 if row_data else 0)
    model = _model(Xs, ys, ws, os_, family, groups=groups, n_groups=G, n_chains=K, kernel="tc")
    inp = _theta(G, P, K, log_shape=np.resize(LOG_SHAPE[::-1], K) if K > 1 else LOG_SHAPE[2])
    (got,) = _run(model, [inp])
    _check(got, _oracle(model, *inp, chunk_rows=1 << 20), _bound(model, *inp))
    unused = np.ones(G, dtype=bool)
    unused[groups] = False
    assert np.all(got[1][..., unused] == 0.0)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_tc_kernel_over_a_segment_of_more_than_a_million_rows(dev, family):
    P, K = 256, 4
    n = (1 << 20) + 12_345
    X, y, beta = synth_positive_shard(n, P, family=family, shape=2.0, seed=31, device=dev)
    w = torch.rand(n, generator=torch.Generator(device=dev).manual_seed(5), device=dev) * 2
    w[::1000] = 0.0
    model = GlmShards([X, X[:5000]], [y, y[:5000]], groups=[0, 1], n_groups=2, family=family, n_chains=K,
                      weights=[w, None], kernel="tc")
    rng = np.random.default_rng(2)
    inp = (np.float32(0.5) + rng.normal(size=(K, 2)).astype(np.float32) * 0.05,
           beta.cpu().numpy()[None] + rng.normal(size=(K, P)).astype(np.float32) * 0.002,
           np.array([0.0, 0.7, 3.0, 9.0], dtype=np.float32))
    (got,) = _run(model, [inp])
    _check(got, _oracle(model, *inp, chunk_rows=1 << 18), _bound(model, *inp))


#: log shapes of the domain sweep: one launch of 16 chains, e^-3 .. e^9 and 1e4
SWEEP_LOG_SHAPE = np.concatenate([np.linspace(-3.0, 9.0, 15), [np.log(1e4)]]).astype(np.float32)


def _sweep(family):
    """One row per (eta, z) point, each its own segment and output block: intercept eta (beta = 0, x = e_0, so eta is
    exact in the kernel) and y = e^(eta + z) rounded to float32, for eta = log 1e-4, 0, log 1e4, z from -20 to 20
    with points near 0 on both sides of the series switch at |z| = 1/2, and y in [1e-6, 1e6]."""
    zs = np.concatenate([[0.0], np.outer([1, -1], [1e-6, 1e-4, 1e-3, 2e-3, 5e-3, 1e-2, 0.03, 0.1, 0.3, 0.49, 0.5, 0.51,
                                                    1.0, 2.0, 5.0, 10.0, 20.0]).reshape(-1)])
    pts = [(e, z) for e in (np.log(1e-4), 0.0, np.log(1e4)) for z in zs if 1e-6 <= np.exp(e + z) <= 1e6]
    etas = np.array([p[0] for p in pts], dtype=np.float32)
    ys = np.exp(etas.astype(np.float64) + np.array([p[1] for p in pts])).astype(np.float32)
    return etas, ys


def _sweep_failures(family, etas, ys, a, ll, r, g0, q):
    """The per-row checks of the domain sweep that some row fails, for the kernel's values ``[rows, chains]`` of the
    rows ``(etas, ys)`` at log shapes ``a``.  Each value may be off by 16 fp32 roundings (``u = 2^-20``) of the
    magnitudes it is formed from, plus its slope in z times the error of z = logf(y) - eta: ``dz = 2^-21 (|log y| +
    |eta|)`` (one ulp of logf and the subtraction's rounding; eta is exact here), and where the kernel takes
    ``expf``, its error as a share of e^z: ``2^-20`` for the gamma family from |z| = 1/2 up, ``2^-21`` everywhere
    for the inverse Gaussian.  Below |z| = 1/2 the gamma family uses no ``expf``, so there ``dz`` has no absolute
    floor: ``nu g(z)`` must be relatively accurate, which ``"near zero"`` checks on ``q - fl(Q) = nu g`` to ``2^-18``
    of itself plus the rounding of q and of Q.  ``z - expm1f(z)`` in place of the series loses about ``2 eps / |z|``
    of g and fails it (``test_sweep_bound_tells_the_series_from_z_minus_expm1``)."""
    y64 = torch.tensor(ys, dtype=torch.float64).unsqueeze(1)
    e64 = torch.tensor(etas, dtype=torch.float64).unsqueeze(1)
    a64 = torch.tensor(a, dtype=torch.float64)
    wl, wr, wq = (t.numpy() for t in _DISPERSION_TERMS[family](y64, e64, a64))
    lt = np.abs(np.log(ys.astype(np.float64)))[:, None]
    z = np.log(ys.astype(np.float64))[:, None] - etas[:, None]
    dz = 2.0 ** -21 * (lt + np.abs(etas)[:, None])
    slope = _slope(family, y64, e64, a64).numpy()
    if family == "gamma":
        dz = dz + np.where(np.abs(z) >= 0.5, 2.0 ** -20, 0.0)
        _, Cn, Q = (t.numpy() for t in _gamma_shape_terms(a64))
        parts = np.abs(wq - Q) + np.abs(Cn) + lt
    else:
        dz = dz + 2.0 ** -21
        Q = np.full(len(a), 0.5)
        parts = np.abs(wq - Q) + np.abs(0.5 * a) + 1.0 + 1.5 * lt
    u = 2.0 ** -20
    ok = {
        "ll": np.abs(ll - wl) <= u * (parts + np.abs(wl)) + np.abs(wr) * dz,
        "r": np.abs(r - wr) <= u * np.abs(wr) + slope * dz,
        "g0": np.abs(g0 - wr) <= 2.0 ** -16 * np.abs(wr) + slope * dz,   # through the (hi, lo) split and MMA #2
        "q": np.abs(q - wq) <= u * (np.abs(wq - Q) + np.abs(Q) + np.abs(wq)) + np.abs(wr) * dz,
    }
    if family == "gamma":
        near = np.abs(z[:, 0]) < 0.5
        ng = (wq - Q)[near]
        got = q[near] - Q.astype(np.float32).astype(np.float64)
        ok["near zero"] = (np.abs(got - ng) <= 2.0 ** -18 * np.abs(ng) + 2.0 ** -24 * (np.abs(q[near]) + np.abs(Q)) +
                           np.abs(wr[near]) * dz[near])
    return sorted(k for k, v in ok.items() if not np.all(v))


def _emulate_gamma(etas, ys, a, naive=False):
    """The kernel's ``gamma_loglik`` in fp32 (numpy), ``(ll, r, q)`` of each row and chain; ``naive``: with ``g = z -
    expm1(z)`` for every z in place of the series."""
    f = np.float32
    nu, Cn, Q = (t.numpy().astype(f) for t in _gamma_shape_terms(torch.tensor(a, dtype=torch.float64)))
    lt = np.log(ys.astype(f))[:, None]
    z = lt - etas.astype(f)[:, None]
    if naive:
        em = np.expm1(z)
        g = z - em
    else:
        gs = np.full_like(z, f(1.0 / 40320))
        for c in (1.0 / 5040, 1.0 / 720, 1.0 / 120, 1.0 / 24, 1.0 / 6, 0.5):
            gs = z * gs + f(c)
        gs = -(z * z) * gs
        small = np.abs(z) < f(0.5)
        em = np.where(small, z - gs, np.exp(z) - f(1.0))
        g = np.where(small, gs, z - em)
    ng = nu * g
    return ((ng + Cn) - lt).astype(np.float64), (nu * em).astype(np.float64), (ng + Q).astype(np.float64)


def test_sweep_bound_tells_the_series_from_z_minus_expm1():
    """The per-row bound of the domain sweep holds for an fp32 emulation of the kernel's gamma code and is broken by
    the same code with ``g = z - expm1(z)``, which loses g's relative accuracy near z = 0."""
    etas, ys = _sweep("gamma")
    ll, r, q = _emulate_gamma(etas, ys, SWEEP_LOG_SHAPE)
    assert _sweep_failures("gamma", etas, ys, SWEEP_LOG_SHAPE, ll, r, r, q) == []
    ll, r, q = _emulate_gamma(etas, ys, SWEEP_LOG_SHAPE, naive=True)
    failed = _sweep_failures("gamma", etas, ys, SWEEP_LOG_SHAPE, ll, r, r, q)
    assert "near zero" in failed and "q" in failed


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_per_row_values_across_the_domain(dev, family):
    """The kernel's ll, r = dll/deta and q = dll/da of single rows (one output block each), at 16 shapes e^-3 .. 1e4
    (one launch, K = 16), within the per-row bound of :func:`_sweep_failures`.  This covers the gamma family near
    z = 0, where g(z) = 1 + z - e^z is its series and ``nu g`` must be relatively accurate (at nu = 1e4 too)."""
    P, K = 8, 16
    etas, ys = _sweep(family)
    n = len(ys)
    X = torch.zeros(n, P, dtype=torch.bfloat16, device=dev)
    X[:, 0] = 1.0
    Xs = [X[i : i + 1].clone() for i in range(n)]
    yl = [torch.tensor(ys[i : i + 1], device=dev) for i in range(n)]
    model = GlmShards(Xs, yl, groups=list(range(n)), n_groups=n, family=family, n_chains=K, kernel="tc",
                      node_ids=list(range(n)), n_nodes=n)
    ic = np.broadcast_to(etas, (K, n)).copy()
    inp = (ic, np.zeros((K, P), np.float32), SWEEP_LOG_SHAPE)
    with FederatedEngine(model) as eng:
        blocks = model.per_node(eng.evaluate_raw(list(inp)))   # [n, K, 2 + n + P]
    idx = np.arange(n)
    ll, r, g0, q = blocks[idx, :, 0], blocks[idx, :, 1 + idx], blocks[:, :, 1 + n], blocks[:, :, -1]
    assert np.all(np.isfinite(blocks))
    assert _sweep_failures(family, etas, ys, SWEEP_LOG_SHAPE, ll, r, g0, q) == []


@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("row_data", [False, True])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_gamma_at_unit_shape_is_weibull_at_unit_sigma(dev, row_data, K):
    ga, wb = _gamma_weibull_pair([128 * 30 + 9, 5000, 77], 256, seed=11, device=dev, weighted=row_data, n_chains=K,
                                 kernel="tc")
    ic, beta, ls = _theta(2, 256, K, log_shape=0.0)
    (a,), (b,) = _run(ga, [(ic, beta, ls)]), _run(wb, [(ic, beta, ls)])
    tol = _bound(ga, ic, beta, ls)
    for i in range(3):   # LL, intercept and beta gradients; d log shape and d log sigma differ
        assert np.all(np.abs(np.asarray(a[i]) - b[i]) <= tol[i])


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_evaluations_are_reproducible_over_grids_and_transports(dev, family):
    """The same bits whatever the grid, and in both result transports: 8 chains x (2 + 3 + 256) values > 2048, and
    one chain at P = 16 (20 values)."""
    rows = [40_000, 25_000, 33_333, 128, 19_999]
    for P, K in ((256, 8), (16, 1)):
        Xs, ys, ws, os_ = _case(rows, P, family, seed=12, device=dev)
        model = _model(Xs, ys, ws, os_, family, groups=[0, 1, 2, 1, 0], n_groups=3, n_chains=K, kernel="tc")
        assert (model.n_vals > 2048) == (K == 8)
        inp = _theta(3, P, K, log_shape=np.resize(LOG_SHAPE, K) if K > 1 else LOG_SHAPE[4])
        outs = []
        for grid in (None, 7, 200):
            outs += _run(model, [inp] * 2, raw=True, grid=grid)
        for o in outs[1:]:
            assert o.tobytes() == outs[0].tobytes()


@pytest.mark.parametrize("rows_data", [False, True])
@pytest.mark.parametrize("K", [1, 2, 4])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_packed_launch_is_bitwise_the_unpacked_one(dev, family, K, rows_data, monkeypatch):
    """P = 200 and 256 with at most 4 columns are packed by default."""
    for P in (200, 256):
        Xs, ys, ws, os_ = _case([3 * 128 + 5, 1000, 128], P, family, seed=21 + K, device=dev, weighted=rows_data,
                                offsets=rows_data, n_masked=5 if rows_data else 0)
        inp = _theta(2, P, K, log_shape=np.resize(LOG_SHAPE, K) if K > 1 else 1.0)
        outs = {}
        for packed in (True, False):
            if packed:
                monkeypatch.delenv("B200FED_NO_PACKED_X", raising=False)
            else:
                monkeypatch.setenv("B200FED_NO_PACKED_X", "1")
            model = _model(Xs, ys, ws, os_, family, groups=[0, 1, 0], n_groups=2, n_chains=K, kernel="tc")
            (outs[packed],) = _run(model, [inp], raw=True)
            assert model.packed_x is packed
        assert np.all(np.isfinite(outs[True]))
        assert outs[True].tobytes() == outs[False].tobytes()


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_node_federation_blocks_equal_single_node_models(dev, family):
    from pytensor_federated_b200.federation import NodeFederation

    rows = [20_000, 128 * 33, 7777]
    node_ids, groups = [0, 1, 1], [0, 1, 0]
    Xs, ys, ws, os_ = _case(rows, 256, family, seed=13, device=dev)
    model = _model(Xs, ys, ws, os_, family, groups=groups, n_groups=2, kernel="tc", node_ids=node_ids, n_nodes=2)
    ic, beta, ls = _theta(2, 256, log_shape=np.log(3.0))
    with FederatedEngine(model) as eng:
        n0 = eng.kernel_launches
        blocks = model.per_node(eng.evaluate_raw([ic, beta, ls]))
        assert eng.kernel_launches - n0 == 1
        assert blocks.shape == (2, 1, 2 + 2 + 256)
        fed = NodeFederation(eng)
        res = fed.evaluate_nodes({0: (ic, beta, ls), 1: (ic, beta, ls)})
        total = fed.all_nodes_func()(ic, beta, ls)
    for node in (0, 1):
        segs = [i for i, n in enumerate(node_ids) if n == node]
        single = _model([Xs[i] for i in segs], [ys[i] for i in segs], [ws[i] for i in segs], [os_[i] for i in segs],
                        family, groups=[groups[i] for i in segs], n_groups=2, kernel="tc")
        want = _oracle(single, ic, beta, ls, chunk_rows=1 << 20)
        tol = _bound(single, ic, beta, ls)
        got = [blocks[node, 0, 0], blocks[node, 0, 1:3], blocks[node, 0, 3:-1], blocks[node, 0, -1]]
        _check(got, want, tol)
        np.testing.assert_allclose(res[node][0], blocks[node, 0, 0], rtol=1e-12)
        assert len(res[node][1]) == 3 and res[node][1][0].shape == (2,) and res[node][1][1].shape == (256,)
        np.testing.assert_allclose(res[node][1][2], blocks[node, 0, -1], rtol=1e-12)
    np.testing.assert_allclose(total[0], blocks[:, 0, 0].sum(), rtol=1e-12)
    np.testing.assert_allclose(total[1][2], blocks[:, 0, -1].sum(), rtol=1e-12)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_map_recovers_the_parameters(dev, family):
    """L-BFGS on the kernel's LL and gradient finds beta*, the intercept and the log shape the data were drawn at,
    each within 5 standard errors (from the inverse of the observed information, by finite differences of the
    kernel's gradient at the MAP)."""
    from pytensor_federated_b200.sampling import find_map, glm_batch_fn

    n, P, shape = 200_000, 8, 4.0
    X, y, beta = synth_positive_shard(n, P, family=family, shape=shape, seed=7, device=dev, beta_scale=0.2)
    model = GlmShards([X], [y], family=family, kernel="tc")
    truth = np.concatenate([[0.5], beta.cpu().numpy(), [np.log(shape)]])
    with FederatedEngine(model) as eng:
        fn = glm_batch_fn(eng, 1)

        def logp_dlogp(x):
            lp, g = fn(x[None])
            return lp[0], g[0]

        x0 = np.zeros_like(truth)
        x_map, info = find_map(logp_dlogp, x0, maxiter=300)
        D = len(truth)
        H = np.zeros((D, D))
        for i in range(D):
            e = np.zeros(D)
            e[i] = 1e-3
            H[i] = (logp_dlogp(x_map + e)[1] - logp_dlogp(x_map - e)[1]) / 2e-3
    cov = np.linalg.inv(-0.5 * (H + H.T))
    se = np.sqrt(np.diag(cov))
    assert np.all(np.isfinite(se)) and np.all(se > 0)
    assert np.all(np.abs(x_map - truth) < 5 * se), (x_map - truth) / se


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_runtime_rejects_the_positive_families_outside_the_tc_kernel(dev):
    """The C ABI refuses what the Python layer never sends: families 11 and 12 on a CUDA-core kernel, n_classes != 1,
    an output size without the log-shape gradient, and the Hessian-vector-product flag.  The engine keeps its model."""
    from pytensor_federated_b200.ops import native

    Xs, ys, _, _ = _case([256], 16, "gamma", seed=14, device=dev, n_masked=0, weighted=False, offsets=False)
    model = GlmShards(Xs, ys, family="poisson", kernel="simt")
    with FederatedEngine(model) as eng:
        lib, h = eng._lib, eng._handle
        Xp, yp = native.void_p_array([Xs[0].data_ptr()]), native.void_p_array([ys[0].data_ptr()])
        rows, grp = (C.c_longlong * 1)(256), (C.c_int * 1)(0)

        def set_glm(n_chains, family, code, n_classes=1):
            return int(lib.b200_engine_set_glm(h, 1, Xp, yp, None, rows, grp, 16, 16, 1, n_chains, family, code, None, 1,
                                               None, None, n_classes))

        for family in FAMILIES:
            code = CODES[family]
            for kernel in (0, 2, 3, 4):
                assert set_glm(1, code, kernel) == -39
                assert f"the {family} family runs on the bf16 tensor-core kernel only" in native.last_error()
            assert set_glm(1, code, 1, 2) != 0 and "n_classes must be 1" in native.last_error()
            # this engine's n_vals is 1 + G + P: one value short of these families' block
            assert set_glm(1, code, 1) != 0 and "2 + n_groups + n_features" in native.last_error()
            assert set_glm(2, code | 16, 1) != 0 and "Hessian-vector products exist for" in native.last_error()
        ic, beta = np.float32(0.1), np.zeros(16, np.float32)
        got = eng.evaluate(ic, beta)
    want = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)


def _build_gamma_model(rank, world, dev):
    Xs, ys, ws, os_ = _case([30_000 + 17 * rank, 999, 77], 256, "gamma", seed=50 + rank, device=dev)
    return _model(Xs, ys, ws, os_, "gamma", groups=[rank % 2, 1 - rank % 2, 0], n_groups=2, n_chains=2, kernel="tc")


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.timeout(900)
def test_two_rank_gamma_federation_matches_oracle():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from pytensor_federated_b200.federation import launch_federation

    inp = _theta(2, 256, 2, log_shape=[np.log(0.5), 3.0])
    dev = torch.device("cuda:0")
    models = [_build_gamma_model(r, 2, dev) for r in range(2)]
    want = models[0].unpack_result(sum(m.reference_partial(list(inp), dtype=torch.float64) for m in models),
                                   models[0].call_context(list(inp)))
    tol = [sum(v) for v in zip(*(_bound(m, *inp) for m in models))]
    del models
    with launch_federation(_build_gamma_model, 2, timeout=30.0) as eng:
        got = eng.evaluate(*inp)
    _check(got, want, tol)
