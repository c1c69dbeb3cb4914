"""GLM families with a learned dispersion parameter: ``GlmShards(..., family="gaussian_scale")`` (s = log sigma) and
``family="negative_binomial"`` (a = log alpha, NB2).

CPU tests check the fp64 oracle and the collective backend against independent formulas (scipy, autograd of the
textbook log-likelihood, finite differences), the limits the families reduce to, validation and the model's packing;
GPU tests check the tensor-core kernel against that oracle."""
import ctypes as C

import numpy as np
import pytest
import torch

from pytensor_federated_b200.models import Fp8GlmShards, GlmShards, synth_negative_binomial_shard
from pytensor_federated_b200.parallel import FederatedEngine
from pytensor_federated_b200.parallel.engine import default_inputs_from_words

FAMILIES = ("gaussian_scale", "negative_binomial")
# dispersion values of the GPU tests: log sigma, log alpha
LOG_DISP = {"gaussian_scale": np.log([0.05, 1.0, 20.0]), "negative_binomial": np.log([0.2, 1.0, 5.0, 50.0, 1e4])}


# ----------------------------------------------------------------------------------------------- fixtures
def _case(rows, P, family, *, seed=0, device="cpu", n_masked=5, weighted=True, offsets=True, alpha=5.0, sigma=1.0):
    """Ragged bf16 segments with responses drawn from the family (NB: alpha, Gaussian: sigma).  With ``weighted``,
    every segment but the last has weights; the first ``n_masked`` rows of segment 0 have weight 0 and carry a NaN, a
    negative and a fractional response.  With ``offsets``, every segment but the second has exposure offsets."""
    rng = np.random.default_rng(seed)
    Xs, ys, ws, os_ = [], [], [], []
    for si, n in enumerate(rows):
        X = torch.tensor(rng.normal(size=(n, P)), dtype=torch.float32).to(torch.bfloat16)
        o = np.log(rng.uniform(0.5, 2.0, size=n))
        eta = X.double().numpy() @ (rng.normal(size=P) * 0.03) + 0.4 + (o if offsets else 0.0)
        if family == "negative_binomial":
            mu = np.exp(eta)
            y = rng.negative_binomial(alpha, alpha / (alpha + mu)).astype(np.float64)
        else:
            y = eta + sigma * rng.normal(size=n)
        w = rng.uniform(0.2, 2.0, size=n)
        if si == 0 and n_masked:
            w[:n_masked] = 0.0
            y[:3] = [np.nan, -1.0, 0.5][: min(3, n_masked)]
        Xs.append(X.to(device))
        ys.append(torch.tensor(y, dtype=torch.float32, device=device))
        ws.append(torch.tensor(w, dtype=torch.float32, device=device) if weighted and si < len(rows) - 1 else None)
        os_.append(torch.tensor(o, dtype=torch.float32, device=device) if offsets and si != 1 else None)
    return Xs, ys, ws, os_


def _theta(G, P, K=1, log_disp=0.3, seed=3, scale=0.03):
    """``(intercept, beta, log_dispersion)``; batched (``[K, G]``, ``[K, P]``, ``[K]``) for K > 1, where
    ``log_disp`` may give one value per chain."""
    rng = np.random.default_rng(seed)
    if K == 1:
        return ((rng.normal(size=G) * 0.2).astype(np.float32), (rng.normal(size=P) * scale).astype(np.float32),
                np.float32(log_disp))
    return ((rng.normal(size=(K, G)) * 0.2).astype(np.float32), (rng.normal(size=(K, P)) * scale).astype(np.float32),
            np.broadcast_to(np.asarray(log_disp, dtype=np.float32), (K,)).copy())


def _textbook_fp64(family, Xs, ys, ws, os_, groups, ic, beta, ld):
    """``[LL, d intercept, d beta, d log_dispersion]`` by autograd of the textbook formula (``torch.lgamma``)."""
    batched = np.ndim(beta) == 2
    ic, beta, ld = (np.asarray(v, dtype=np.float64) for v in (ic, beta, ld))
    if not batched:
        ic, beta, ld = ic.reshape(1, -1), beta[None], ld.reshape(1)
    t_ic, t_b, t_ld = (torch.tensor(v, requires_grad=True) for v in (ic, beta, ld))
    total = torch.zeros(beta.shape[0], dtype=torch.float64)
    for X, y, w, o, g in zip(Xs, ys, ws, os_, groups):
        X, y = X.double().cpu(), y.double().cpu()
        keep = torch.ones_like(y, dtype=torch.bool) if w is None else w.cpu() != 0
        y = torch.where(keep, y, torch.zeros_like(y))
        eta = t_b @ X.T + t_ic[:, g, None]                             # [K, n]
        if o is not None:
            eta = eta + o.double().cpu()
        if family == "negative_binomial":
            alpha, mu = torch.exp(t_ld)[:, None], torch.exp(eta)
            ll = (torch.lgamma(y + alpha) - torch.lgamma(alpha) + alpha * torch.log(alpha / (alpha + mu))
                  + y * torch.log(mu / (alpha + mu)))
        else:
            sigma = torch.exp(t_ld)[:, None]
            ll = -0.5 * ((y - eta) / sigma) ** 2 - torch.log(sigma) - 0.5 * np.log(2 * np.pi)
        if w is not None:
            ll = torch.where(keep, w.double().cpu() * ll, torch.zeros_like(ll))
        total = total + ll.sum(1)
    total.sum().backward()
    out = [total.detach().numpy(), t_ic.grad.numpy(), t_b.grad.numpy(), t_ld.grad.numpy()]
    return out if batched else [out[0][0], out[1][0], out[2][0], out[3][0]]


def _oracle(model, *inputs, chunk_rows=128):
    return model.unpack_result(model.reference_partial(list(inputs), dtype=torch.float64, chunk_rows=chunk_rows))


def _collective(model, *inputs):
    with FederatedEngine(model, backend="collective") as eng:
        return [np.asarray(v, dtype=np.float64) for v in eng.evaluate(*inputs)]


# ----------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("K", [1, 3])
@pytest.mark.parametrize("family", FAMILIES)
def test_oracle_matches_autograd_of_the_textbook_loglik(family, K):
    rows, P, groups = [150, 70, 201], 16, [0, 1, 0]
    Xs, ys, ws, os_ = _case(rows, P, family, seed=1)
    model = GlmShards(Xs, ys, groups=groups, n_groups=2, family=family, n_chains=K, weights=ws, offsets=os_)
    ic, beta, ld = _theta(2, P, K, log_disp=[0.3, -1.2, 2.5][:K] if K > 1 else -0.4)
    got = _oracle(model, ic, beta, ld)
    want = _textbook_fp64(family, Xs, ys, ws, os_, groups, ic, beta, ld)
    assert np.all(np.isfinite(got[0]))
    assert got[1].shape == ic.shape and got[2].shape == beta.shape and np.shape(got[3]) == np.shape(ld)
    np.testing.assert_allclose(got[0], want[0], rtol=1e-12)
    for u, v in zip(got[1:], want[1:]):
        np.testing.assert_allclose(u, v, rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("log_disp", [np.log(0.3), np.log(7.9), np.log(40.0), np.log(1e4)])
@pytest.mark.parametrize("family", FAMILIES)
def test_oracle_matches_scipy_and_finite_differences(family, log_disp):
    """Both sides of the oracle's switch to the Stirling-series differences (alpha >= 1e3 in fp64)."""
    import scipy.stats
    from scipy.special import gammaln

    rows, P = [90, 60], 8
    Xs, ys, ws, os_ = _case(rows, P, family, seed=2, n_masked=0)
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family=family, weights=ws, offsets=os_)
    Xn = [X.double().numpy() for X in Xs]
    yn = [y.double().numpy() for y in ys]
    wn = [w.double().numpy() if w is not None else np.ones(len(y)) for w, y in zip(ws, ys)]
    on = [o.double().numpy() if o is not None else np.zeros(len(y)) for o, y in zip(os_, ys)]

    def truth(ic, beta, ld):
        total = 0.0
        for g, (X, y, w, o) in enumerate(zip(Xn, yn, wn, on)):
            eta = X @ beta + ic[g] + o
            if family == "negative_binomial":
                alpha, mu = np.exp(ld[()]), np.exp(eta)
                ll = scipy.stats.nbinom.logpmf(y, alpha, alpha / (alpha + mu)) + gammaln(y + 1)
            else:
                ll = scipy.stats.norm.logpdf(y, eta, np.exp(ld[()]))
            total += np.sum(w * ll)
        return total

    ic, beta, ld = [np.asarray(v, dtype=np.float64) for v in _theta(2, P, log_disp=log_disp)]
    got = _oracle(model, ic, beta, ld)
    np.testing.assert_allclose(got[0], truth(ic, beta, ld), rtol=1e-10)
    eps = 1e-4   # scipy's lgamma differences lose ~1e-11 at alpha = 1e4: a wider step keeps that out of the quotient
    for arr, grad in ((ic, got[1]), (beta, got[2]), (ld, got[3])):
        fd = np.zeros_like(arr)
        for idx in np.ndindex(arr.shape):
            orig = arr[idx]
            arr[idx] = orig + eps
            hi = truth(ic, beta, ld)
            arr[idx] = orig - eps
            lo = truth(ic, beta, ld)
            arr[idx] = orig
            fd[idx] = (hi - lo) / (2 * eps)
        np.testing.assert_allclose(grad, fd, rtol=1e-6, atol=1e-5)


def test_negative_binomial_tends_to_poisson():
    """At log alpha = 20 the NB model differs from the Poisson one by O(sum (y + mu)^2 / alpha)."""
    rows, P = [300, 120], 16
    Xs, ys, ws, os_ = _case(rows, P, "negative_binomial", seed=3)
    nb = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family="negative_binomial", weights=ws, offsets=os_)
    ys_p = [torch.nan_to_num(y).clamp(min=0) for y in ys]   # masked rows: any finite response
    pois = GlmShards(Xs, ys_p, groups=[0, 1], n_groups=2, family="poisson", weights=ws, offsets=os_)
    ic, beta, ld = _theta(2, P, log_disp=20.0)
    a = _oracle(nb, ic, beta, ld)
    b = pois.unpack_result(pois.reference_partial([ic, beta], dtype=torch.float64))
    alpha = np.exp(20.0)
    bound = 0.0
    for X, y, w, o, g in zip(Xs, ys_p, ws, os_, [0, 1]):
        eta = X.double().numpy() @ beta.astype(np.float64) + ic[g] + (o.double().numpy() if o is not None else 0.0)
        ww = w.double().numpy() if w is not None else 1.0
        bound += np.sum(ww * (y.double().numpy() + np.exp(eta)) ** 2) / alpha
    assert 0 < bound < 1e-4
    assert abs(a[0] - b[0]) <= bound
    assert np.max(np.abs(a[1] - b[1])) <= bound
    assert np.max(np.abs(a[2] - b[2])) <= bound * max(float(X.float().abs().max()) for X in Xs)
    assert abs(a[3]) <= bound


@pytest.mark.parametrize("weighted", [False, True])
def test_gaussian_scale_at_unit_sigma_is_the_gaussian_family(weighted):
    rows, P = [130, 77], 16
    Xs, ys, ws, os_ = _case(rows, P, "gaussian_scale", seed=4, weighted=weighted, offsets=weighted)
    gs = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family="gaussian_scale", weights=ws, offsets=os_)
    ga = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family="gaussian", weights=ws, offsets=os_)
    ic, beta, _ = _theta(2, P)
    a = _oracle(gs, ic, beta, np.float32(0.0))
    b = ga.unpack_result(ga.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(a[0], b[0], rtol=1e-12)
    np.testing.assert_allclose(a[1], b[1], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(a[2], b[2], rtol=1e-12, atol=1e-12)
    # dLL/ds = sum w (d^2 - 1)
    want = 0.0
    for X, y, w, o, g in zip(Xs, ys, ws, os_, [0, 1]):
        eta = X.double().numpy() @ beta.astype(np.float64) + ic[g] + (o.double().numpy() if o is not None else 0.0)
        d2 = (y.double().numpy() - eta) ** 2 - 1.0
        if w is not None:
            d2 = np.where(w.numpy() != 0, w.double().numpy() * d2, 0.0)
        want += d2.sum()
    np.testing.assert_allclose(a[3], want, rtol=1e-12)


@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("family", FAMILIES)
def test_collective_backend_equals_the_oracle(family, K):
    rows, P = [300, 45, 129], 24
    Xs, ys, ws, os_ = _case(rows, P, family, seed=6)
    model = GlmShards(Xs, ys, groups=[0, 1, 1], n_groups=2, family=family, n_chains=K, weights=ws, offsets=os_)
    ic, beta, ld = _theta(2, P, K, log_disp=[0.5, -1.0, 2.0, 9.0][:K] if K > 1 else 0.5)
    got, want = _collective(model, ic, beta, ld), _oracle(model, ic, beta, ld)
    for u, v in zip(got, want):
        assert np.shape(u) == np.shape(v) and np.all(np.isfinite(u))
        np.testing.assert_allclose(u, v, rtol=1e-4, atol=1e-3)


def test_dispersion_validation():
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ys = [torch.zeros(10), torch.full((6,), 2.0)]
    for family in FAMILIES:
        GlmShards(Xs, ys, family=family)
        GlmShards(Xs, ys, family=family, offsets=[torch.zeros(10), None], weights=[None, torch.ones(6)])
        for kernel in ("simt", "generic", "fp8"):
            with pytest.raises(ValueError, match="tensor-core kernel only"):
                GlmShards(Xs, ys, family=family, kernel=kernel)
        with pytest.raises(ValueError, match="tensor-core kernel only"):
            Fp8GlmShards.from_dense([torch.randn(10, 32), torch.randn(6, 32)], ys, family=family)
        with pytest.raises(ValueError, match="n_classes"):
            GlmShards(Xs, ys, family=family, n_classes=2)
        # shapes outside the tensor-core kernel's: an error, never another kernel
        for X in (torch.randn(10, 12).to(torch.bfloat16), torch.randn(10, 392).to(torch.bfloat16), torch.randn(10, 16)):
            with pytest.raises(ValueError, match="tensor-core kernel only"):
                GlmShards([X], [torch.zeros(10)], family=family).use_tensor_cores()
        with pytest.raises(ValueError, match="tensor-core kernel only"):
            GlmShards(Xs, ys, family=family, n_chains=17).use_tensor_cores()
        assert GlmShards(Xs, ys, family=family, kernel="tc").use_tensor_cores() == 1
    for bad in (-1.0, 0.5, float("nan"), float("inf"), 2.0 ** 24 + 2):
        y0 = torch.zeros(10)
        y0[4] = bad
        with pytest.raises(ValueError, match="counts of segment 0"):
            GlmShards(Xs, [y0, ys[1]], family="negative_binomial")
        w0 = torch.ones(10)
        w0[4] = 0.0
        GlmShards(Xs, [y0, ys[1]], weights=[w0, None], family="negative_binomial")   # a masked row may carry anything
        GlmShards(Xs, [y0.nan_to_num(), ys[1]], family="gaussian_scale")            # any finite real response
    y0 = torch.zeros(10)
    y0[4] = 2.0 ** 24
    GlmShards(Xs, [y0, ys[1]], family="negative_binomial")


@pytest.mark.parametrize("family", FAMILIES)
def test_sizes_and_flops(family):
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ys = [torch.zeros(10), torch.zeros(6)]
    m = GlmShards(Xs, ys, n_groups=2, groups=[0, 1], family=family, n_chains=3, node_ids=[0, 1], n_nodes=2)
    assert m.n_inputs == 3
    assert m.n_params == 2 + 16 + 1 and m.n_theta_words == 3 * 19
    assert m.n_vals == 2 * 3 * (2 + 2 + 16)
    assert m.flops_per_eval() == GlmShards(Xs, ys, n_chains=3).flops_per_eval() == 4 * 16 * 16 * 3
    assert m.bytes_per_eval() == GlmShards(Xs, ys).bytes_per_eval()
    assert m.per_node(np.zeros(m.n_vals)).shape == (2, 3, 2 + 2 + 16)


@pytest.mark.parametrize("K,G", [(1, 1), (1, 2), (4, 2)])
def test_pack_unpack_and_words_round_trip(K, G):
    P = 8
    Xs, ys, _, _ = _case([20] * G, P, "negative_binomial", seed=7, n_masked=0, weighted=False, offsets=False)
    model = GlmShards(Xs, ys, groups=list(range(G)), n_groups=G, family="negative_binomial", n_chains=K)
    ic, beta, ld = _theta(G, P, K, log_disp=np.arange(K) - 0.5 if K > 1 else -0.5, scale=1.0)
    if K == 1 and G == 1:
        ic = ic.reshape(())   # a scalar intercept for one group
    words = np.zeros(model.n_theta_words, dtype=np.uint32)
    ctx = model.pack_theta([ic, beta, ld], words)
    assert ctx == model.call_context([ic, beta, ld]) == (K > 1, ic.shape, np.shape(ld))
    # the kernel's layout: row k = (intercept[G], beta[P], log_dispersion) of chain k
    th = words.view(np.float32).reshape(K, G + P + 1)
    np.testing.assert_array_equal(th[:, :G], np.reshape(ic, (K, G)))
    np.testing.assert_array_equal(th[:, G : G + P], np.reshape(beta, (K, P)))
    np.testing.assert_array_equal(th[:, G + P], np.reshape(ld, K))
    ic2, b2, ld2 = default_inputs_from_words(model, words)
    assert np.array_equal(ic2.reshape(ic.shape), ic) and np.array_equal(b2, beta) and np.array_equal(ld2, ld)
    words2 = np.zeros_like(words)
    model.pack_theta([ic2, b2, ld2], words2)
    assert np.array_equal(words, words2)
    # unpack: block k of the raw vector holds [LL, gi[G], g[P], q] of chain k
    raw = np.arange(model.n_vals, dtype=np.float64).reshape(K, 2 + G + P)
    logp, d_ic, d_b, d_ld = model.unpack_result(raw.reshape(-1), ctx)
    assert d_ic.shape == np.shape(ic) and d_b.shape == beta.shape and np.shape(d_ld) == np.shape(ld)
    np.testing.assert_array_equal(np.reshape(logp, -1), raw[:, 0])
    np.testing.assert_array_equal(np.reshape(d_ic, (K, G)), raw[:, 1 : 1 + G])
    np.testing.assert_array_equal(np.reshape(d_b, (K, P)), raw[:, 1 + G : 1 + G + P])
    np.testing.assert_array_equal(np.reshape(d_ld, K), raw[:, -1])


@pytest.mark.parametrize("family", FAMILIES)
def test_glm_batch_fn_splits_theta_with_a_dispersion_parameter(family):
    from pytensor_federated_b200.sampling import glm_batch_fn

    P, G = 8, 2
    Xs, ys, ws, os_ = _case([60, 40], P, family, seed=8)
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=G, family=family, n_chains=2, weights=ws, offsets=os_)
    rng = np.random.default_rng(9)
    theta = rng.normal(size=(3, G + P + 1)) * 0.1
    with FederatedEngine(model, backend="collective") as eng:
        logp, grad = glm_batch_fn(eng, G)(theta)
    assert logp.shape == (3,) and grad.shape == theta.shape
    single = GlmShards(Xs, ys, groups=[0, 1], n_groups=G, family=family, weights=ws, offsets=os_)
    for i in range(3):
        want = _oracle(single, theta[i, :G], theta[i, G : G + P], theta[i, -1])
        np.testing.assert_allclose(logp[i], want[0], rtol=1e-5)
        np.testing.assert_allclose(grad[i], np.concatenate([want[1], want[2], [want[3]]]), rtol=1e-4, atol=1e-3)


def test_synth_negative_binomial_shard():
    n, alpha = 200_000, 2.5
    X, y, beta = synth_negative_binomial_shard(n, 16, alpha=alpha, seed=1, device="cpu", chunk_rows=65536,
                                               beta_scale=0.0, intercept=0.7)
    assert X.dtype == torch.bfloat16 and X.shape == (n, 16) and beta.shape == (16,)
    yn = y.double().numpy()
    assert y.dtype == torch.float32 and np.all(yn == np.floor(yn)) and yn.min() >= 0
    mu = np.exp(0.7)
    var = mu + mu * mu / alpha
    assert abs(yn.mean() - mu) < 5 * np.sqrt(var / n)
    # the sample variance's standard error sqrt((m4 - var^2) / n), with the sample's fourth central moment
    se_var = np.sqrt((np.mean((yn - yn.mean()) ** 4) - yn.var() ** 2) / n)
    assert abs(yn.var() - var) < 5 * se_var
    assert abs(yn.var() - mu) > 20 * se_var   # over-dispersed: not the Poisson variance
    X2, y2, _ = synth_negative_binomial_shard(n, 16, alpha=alpha, seed=1, device="cpu", chunk_rows=65536,
                                              beta_scale=0.0, intercept=0.7)
    assert torch.equal(X, X2) and torch.equal(y, y2)


# ----------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from pytensor_federated_b200.ops import native

    native.load()  # a GPU box without the native library is a failure, not a skip
    return torch.device("cuda:0")


def _run(model, inputs_list):
    """The engine's results for each set of inputs, one engine."""
    with FederatedEngine(model) as eng:
        return [[np.asarray(v).copy() for v in eng.evaluate(*inputs)] for inputs in inputs_list]


def _check(got, want, n_rows, K, family, log_disp):
    """The tolerances of the multinomial suite, and d log_dispersion at rtol 1e-4 / atol 2e-3 sqrt(n).

    The absolute tolerances of the intercept and beta gradients are per chain, times the scale of its residuals
    relative to the multinomial suite's |r| <= 1: gaussian_scale has r = d / sigma^2, so the rounding of r (the
    (hi, lo) bf16 split of R keeps ~2^-17 of |r|) and with it the absolute error of a gradient component that
    nearly cancels grow as 1 / sigma^2 (400 at sigma = 0.05).  Negative-binomial residuals are of the size of
    Poisson ones, scale 1."""
    assert all(np.all(np.isfinite(g)) for g in got)
    for u, v in zip(got, want):
        assert np.shape(u) == np.shape(v)
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)
    lds = np.reshape(log_disp, -1).astype(np.float64)
    scale = np.maximum(1.0, np.exp(-2.0 * lds)) if family == "gaussian_scale" else np.ones_like(lds)
    atol_b = 2e-3 * np.sqrt(n_rows) if K == 1 else 0.2
    for k in range(K):
        pick = (lambda a: a[k]) if K > 1 else (lambda a: a)
        np.testing.assert_allclose(pick(got[1]), pick(want[1]), rtol=1e-4, atol=2e-3 * scale[k])
        np.testing.assert_allclose(pick(got[2]), pick(want[2]), rtol=1e-4, atol=atol_b * scale[k])
    np.testing.assert_allclose(got[3], want[3], rtol=1e-4, atol=2e-3 * np.sqrt(n_rows))


@pytest.mark.parametrize("row_data", [True, False])
@pytest.mark.parametrize("K", [1, 2, 4, 5, 8, 16])
@pytest.mark.parametrize("P", [256, 200, 8])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_matches_oracle(dev, family, P, K, row_data):
    """K <= 1, 4, 8 and 16 select the kernel's four DISP buckets; ``row_data`` (offsets and weights, masked rows
    with NaN / negative / fractional responses) its ROWS variant.  The chains cycle through the dispersion values
    (sigma 0.05, 1, 20; alpha 0.2, 1, 5, 50, 1e4); with K = 1 each value is one evaluation."""
    rows = [128 * 37, 77, 4099, 1]
    Xs, ys, ws, os_ = _case(rows, P, family, seed=K + P, device=dev, weighted=row_data, offsets=row_data,
                            n_masked=5 if row_data else 0)
    model = GlmShards(Xs, ys, groups=[0, 1, 0, 1], n_groups=2, family=family, n_chains=K, kernel="auto",
                      weights=ws, offsets=os_)
    assert model.has_row_data == row_data
    lds = LOG_DISP[family]
    if K == 1:
        inputs = [_theta(2, P, 1, log_disp=v, seed=5 + i) for i, v in enumerate(lds)]
    else:
        inputs = [_theta(2, P, K, log_disp=np.resize(lds, K))]
    got = _run(model, inputs)
    assert model.selected_kernel == "tc"
    for g, inp in zip(got, inputs):
        _check(g, _oracle(model, *inp, chunk_rows=1 << 20), sum(rows), K, family, inp[2])


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("K,row_data", [(1, False), (2, True), (5, False), (5, True)])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_with_many_groups_matches_oracle(dev, family, K, row_data):
    """300 intercepts: the intercept table is KC x G floats and the per-chain dispersion table follows it."""
    G, P = 300, 256
    rows = [128 * 9 + 5, 999, 64, 1, 3000]
    groups = [0, 299, 150, 7, 299]
    Xs, ys, ws, os_ = _case(rows, P, family, seed=40 + K, device=dev, weighted=row_data, offsets=row_data,
                            n_masked=5 if row_data else 0)
    model = GlmShards(Xs, ys, groups=groups, n_groups=G, family=family, n_chains=K, kernel="tc", weights=ws,
                      offsets=os_)
    inp = _theta(G, P, K, log_disp=np.resize(LOG_DISP[family][::-1], K) if K > 1 else LOG_DISP[family][0])
    (got,) = _run(model, [inp])
    _check(got, _oracle(model, *inp, chunk_rows=1 << 20), sum(rows), K, family, inp[2])
    unused = np.ones(G, dtype=bool)
    unused[groups] = False
    assert np.all(got[1][..., unused] == 0.0)


@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("row_data", [False, True])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_gaussian_scale_at_unit_sigma_is_bit_identical_to_gaussian(dev, row_data, K):
    rows, P = [128 * 30 + 9, 5000, 77], 256
    Xs, ys, ws, os_ = _case(rows, P, "gaussian_scale", seed=11, device=dev, weighted=row_data, offsets=row_data,
                            n_masked=5 if row_data else 0)
    gs = GlmShards(Xs, ys, groups=[0, 1, 0], n_groups=2, family="gaussian_scale", n_chains=K, kernel="tc",
                   weights=ws, offsets=os_)
    ga = GlmShards(Xs, ys, groups=[0, 1, 0], n_groups=2, family="gaussian", n_chains=K, kernel="tc", weights=ws,
                   offsets=os_)
    ic, beta, ld = _theta(2, P, K, log_disp=0.0)
    (a,), (b,) = _run(gs, [(ic, beta, ld)]), _run(ga, [(ic, beta)])
    for u, v in zip(a[:3], b):
        assert np.array_equal(u, v)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_dispersion_evaluations_are_bit_reproducible(dev, family):
    rows = [40_000, 25_000, 33_333, 128, 19_999]
    Xs, ys, ws, os_ = _case(rows, 256, family, seed=12, device=dev)
    model = GlmShards(Xs, ys, groups=[0, 1, 2, 1, 0], n_groups=3, family=family, n_chains=4, kernel="tc",
                      weights=ws, offsets=os_)
    inp = _theta(3, 256, 4, log_disp=np.resize(LOG_DISP[family], 4))
    runs = _run(model, [inp] * 10)
    for run in runs[1:]:
        for u, v in zip(runs[0], run):
            assert np.array_equal(u, v)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_node_federation_blocks_equal_single_node_models(dev, family):
    from pytensor_federated_b200.federation import NodeFederation

    rows = [20_000, 128 * 33, 7777]
    node_ids, groups = [0, 1, 1], [0, 1, 0]
    Xs, ys, ws, os_ = _case(rows, 256, family, seed=13, device=dev)
    model = GlmShards(Xs, ys, groups=groups, n_groups=2, family=family, kernel="tc", node_ids=node_ids, n_nodes=2,
                      weights=ws, offsets=os_)
    ic, beta, ld = _theta(2, 256, log_disp=0.7)
    with FederatedEngine(model) as eng:
        n0 = eng.kernel_launches
        blocks = model.per_node(eng.evaluate_raw([ic, beta, ld]))
        assert eng.kernel_launches - n0 == 1
        assert blocks.shape == (2, 1, 2 + 2 + 256)
        fed = NodeFederation(eng)
        res = fed.evaluate_nodes({0: (ic, beta, ld), 1: (ic, beta, ld)})
        total = fed.all_nodes_func()(ic, beta, ld)
    for node in (0, 1):
        segs = [i for i, n in enumerate(node_ids) if n == node]
        single = GlmShards([Xs[i] for i in segs], [ys[i] for i in segs], groups=[groups[i] for i in segs], n_groups=2,
                           family=family, kernel="tc", weights=[ws[i] for i in segs], offsets=[os_[i] for i in segs])
        (want,) = _run(single, [(ic, beta, ld)])
        np.testing.assert_allclose(blocks[node, 0, 0], want[0], rtol=2e-5)
        np.testing.assert_allclose(blocks[node, 0, 1:3], want[1], rtol=1e-4, atol=2e-3)
        np.testing.assert_allclose(blocks[node, 0, 3:-1], want[2], rtol=1e-4, atol=0.5)
        np.testing.assert_allclose(blocks[node, 0, -1], want[3], rtol=1e-4, atol=2e-3)
        np.testing.assert_allclose(res[node][0], blocks[node, 0, 0], rtol=1e-12)
        assert len(res[node][1]) == 3 and res[node][1][0].shape == (2,) and res[node][1][1].shape == (256,)
        assert np.shape(res[node][1][2]) == ()
        np.testing.assert_allclose(res[node][1][2], want[3], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(total[0], blocks[:, 0, 0].sum(), rtol=1e-12)
    np.testing.assert_allclose(total[1][2], blocks[:, 0, -1].sum(), rtol=1e-12)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_lock_step_hmc_on_a_negative_binomial_engine(dev):
    from pytensor_federated_b200.sampling import glm_batch_fn, hmc_sample_batched

    K, P = 4, 16
    X, y, _ = synth_negative_binomial_shard(20_000, P, alpha=3.0, seed=3, device=dev)
    model = GlmShards([X], [y], family="negative_binomial", n_chains=K, kernel="tc")
    x0 = np.zeros((K, 1 + P + 1))
    x0[:, -1] = np.log(3.0)
    with FederatedEngine(model) as eng:
        res = hmc_sample_batched(glm_batch_fn(eng, 1), x0, draws=5, tune=5, n_leapfrog=4, step_size=1e-3, seed=1)
        assert eng.n_evals == res.n_batched_evals
    assert res.samples.shape[-1] == 1 + P + 1 and np.all(np.isfinite(res.samples))


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_runtime_rejects_the_dispersion_families_outside_the_tc_kernel(dev):
    """The C ABI refuses what the Python layer never sends: families 4 and 5 on a CUDA-core kernel (which would take
    an unknown family for the Gaussian one), n_classes != 1, and an output size without the dispersion gradient."""
    from pytensor_federated_b200.ops import native

    Xs, ys, _, _ = _case([256], 16, "negative_binomial", seed=14, device=dev, n_masked=0, weighted=False, offsets=False)
    model = GlmShards(Xs, ys, kernel="simt")
    with FederatedEngine(model) as eng:
        lib, h = eng._lib, eng._handle
        Xp, yp = native.void_p_array([Xs[0].data_ptr()]), native.void_p_array([ys[0].data_ptr()])
        rows, grp = (C.c_longlong * 1)(256), (C.c_int * 1)(0)

        def set_glm(n_chains, family, code, n_classes=1):
            return int(lib.b200_engine_set_glm(h, 1, Xp, yp, None, rows, grp, 16, 16, 1, n_chains, family, code, None, 1,
                                               None, None, n_classes))

        for family, name in ((4, "gaussian_scale"), (5, "negative_binomial")):
            for code in (0, 2, 3, 4):
                assert set_glm(1, family, code) != 0
                assert f"the {name} family runs on the bf16 tensor-core kernel only" in native.last_error()
            assert set_glm(1, family, 1, 2) != 0 and "n_classes must be 1" in native.last_error()
            # this engine's n_vals is 1 + G + P: one value short of the dispersion families' block
            assert set_glm(1, family, 1) != 0 and "2 + n_groups + n_features" in native.last_error()
        # the engine still evaluates its own model
        ic, beta = np.float32(0.1), np.zeros(16, np.float32)
        got = eng.evaluate(ic, beta)
    want = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)


def _build_nb_model(rank, world, dev):
    Xs, ys, ws, os_ = _case([30_000 + 17 * rank, 999], 256, "negative_binomial", seed=50 + rank, device=dev)
    return GlmShards(Xs, ys, groups=[rank % 2, 1 - rank % 2], n_groups=2, family="negative_binomial", n_chains=2,
                     kernel="tc", weights=ws, offsets=os_)


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.timeout(900)
def test_two_rank_negative_binomial_federation_matches_oracle():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from pytensor_federated_b200.federation import launch_federation

    inp = _theta(2, 256, 2, log_disp=[0.0, 3.0])
    dev = torch.device("cuda:0")
    models = [_build_nb_model(r, 2, dev) for r in range(2)]
    want = models[0].unpack_result(sum(m.reference_partial(list(inp), dtype=torch.float64) for m in models),
                                   models[0].call_context(list(inp)))
    del models
    with launch_federation(_build_nb_model, 2, timeout=30.0) as eng:
        got = eng.evaluate(*inp)
    _check(got, want, 2 * 31_000, 2, "negative_binomial", inp[2])
