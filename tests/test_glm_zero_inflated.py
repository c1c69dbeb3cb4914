"""Zero-inflated count regression: ``GlmShards(..., family="zero_inflated_poisson")`` and
``family="zero_inflated_negative_binomial"`` (inputs ``intercept, beta, zi_intercept, zi_beta[, log_dispersion]``).

CPU tests check the fp64 oracle against scipy mixtures and finite differences, its limit as the zero logit goes to
-inf, the layout (packing, words, fold, sizes), validation and the collective backend; GPU tests check the tensor-core
kernel against that oracle, bit for bit against the plain Poisson / negative-binomial launch where the zero part
vanishes, and its packed-X, per-node and sampling paths."""
import ctypes as C

import numpy as np
import pytest
import torch

from pytensor_federated_b200.models import Fp8GlmShards, GlmShards, synth_zero_inflated_shard
from pytensor_federated_b200.parallel import FederatedEngine
from pytensor_federated_b200.parallel.engine import default_inputs_from_words

FAMILIES = ("zero_inflated_poisson", "zero_inflated_negative_binomial")
BASE = {"zero_inflated_poisson": "poisson", "zero_inflated_negative_binomial": "negative_binomial"}
NB = "zero_inflated_negative_binomial"
# log alpha of the GPU tests' chains, zero-inflation intercepts of their chains
LOG_ALPHA = np.log([0.3, 1.0, 5.0, 50.0, 1e4])
ZI_ICPT = np.array([-3.0, -0.5, 0.0, 1.0, 4.0])


# ----------------------------------------------------------------------------------------------- fixtures
def _case(rows, P, family, *, seed=0, device="cpu", n_masked=5, weighted=True, offsets=True, alpha=3.0, pi=0.3,
          beta_scale=0.03, log_mu=None):
    """Ragged bf16 segments of zero-inflated counts: a structural zero with probability ``pi``, else Poisson or NB
    (alpha) counts around ``exp(eta)``.  With ``weighted``, every segment but the last has weights; the first
    ``n_masked`` rows of segment 0 have weight 0 and carry a NaN, a negative and a fractional count.  With ``offsets``,
    every segment but the second has exposure offsets (``log_mu``: offsets spread evenly over that range instead)."""
    rng = np.random.default_rng(seed)
    Xs, ys, ws, os_ = [], [], [], []
    for si, n in enumerate(rows):
        X = torch.tensor(rng.normal(size=(n, P)), dtype=torch.float32).to(torch.bfloat16)
        o = np.log(rng.uniform(0.5, 2.0, size=n)) if log_mu is None else rng.permutation(np.linspace(*log_mu, n))
        eta = X.double().numpy() @ (rng.normal(size=P) * beta_scale) + 0.4 + (o if offsets else 0.0)
        mu = np.exp(eta)
        if family == NB:
            y = rng.negative_binomial(alpha, alpha / (alpha + mu)).astype(np.float64)
        else:
            y = rng.poisson(mu).astype(np.float64)
        y[rng.uniform(size=n) < pi] = 0.0
        w = rng.uniform(0.2, 2.0, size=n)
        if si == 0 and n_masked:
            w[:n_masked] = 0.0
            y[:3] = [np.nan, -1.0, 0.5][: min(3, n_masked)]
        Xs.append(X.to(device))
        ys.append(torch.tensor(y, dtype=torch.float32, device=device))
        ws.append(torch.tensor(w, dtype=torch.float32, device=device) if weighted and si < len(rows) - 1 else None)
        os_.append(torch.tensor(o, dtype=torch.float32, device=device) if offsets and si != 1 else None)
    return Xs, ys, ws, os_


def _theta(family, G, P, K=1, *, zi=-0.5, log_alpha=1.0, seed=3, scale=0.03):
    """``(intercept, beta, zi_intercept, zi_beta[, log_dispersion])``, batched for K > 1 (``zi`` and ``log_alpha``
    may give one value per chain: the zero-inflation intercepts are ``zi`` plus noise)."""
    rng = np.random.default_rng(seed)
    lead = (K,) if K > 1 else ()
    zi = np.asarray(zi, dtype=np.float64)
    out = [(rng.normal(size=lead + (G,)) * 0.2).astype(np.float32),
           (rng.normal(size=lead + (P,)) * scale).astype(np.float32),
           ((zi[..., None] if zi.ndim else zi) + rng.normal(size=lead + (G,)) * 0.2).astype(np.float32),
           (rng.normal(size=lead + (P,)) * scale).astype(np.float32)]
    if family == NB:
        out.append(np.broadcast_to(np.asarray(log_alpha, dtype=np.float32), lead).copy() if K > 1
                   else np.float32(log_alpha))
    return tuple(out)


def _oracle(model, *inputs, chunk_rows=128):
    return model.unpack_result(model.reference_partial(list(inputs), dtype=torch.float64, chunk_rows=chunk_rows))


def _collective(model, *inputs):
    with FederatedEngine(model, backend="collective") as eng:
        return [np.asarray(v, dtype=np.float64) for v in eng.evaluate(*inputs)]


def _scipy_truth(family, Xn, yn, wn, on, groups):
    """The log-likelihood as a function of the inputs, from scipy's pmfs (plus the ``lgamma(y + 1)`` the model omits on
    rows with y > 0): ``log(pi + (1 - pi) f(0))`` and ``log(1 - pi) + log f(y)`` by ``logsumexp`` / ``log_expit``."""
    import scipy.stats
    from scipy.special import gammaln, log_expit, logsumexp

    def truth(ic, beta, zic, zbeta, ld=None):
        total = 0.0
        for X, y, w, o, g in zip(Xn, yn, wn, on, groups):
            eta = X @ beta + ic[g] + o
            zeta = X @ zbeta + zic[g]
            mu = np.exp(eta)
            if family == NB:
                alpha = np.exp(ld[()])
                logf = scipy.stats.nbinom.logpmf(y, alpha, alpha / (alpha + mu))
            else:
                logf = scipy.stats.poisson.logpmf(y, mu)
            lpi, l1pi = log_expit(zeta), log_expit(-zeta)
            ll = np.where(y == 0, logsumexp(np.stack([lpi, l1pi + logf]), axis=0), l1pi + logf + gammaln(y + 1))
            total += np.sum(w * ll)
        return total

    return truth


# ----------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("zi", [-30.0, -4.0, 0.0, 3.0, 30.0])
@pytest.mark.parametrize("family,log_alpha", [("zero_inflated_poisson", 0.0)] +
                         [(NB, la) for la in np.log([0.3, 7.9, 1e4])])
def test_oracle_matches_scipy_and_finite_differences(family, log_alpha, zi):
    """Zero logits from -30 to 30, alpha from 0.3 to 1e4 (both sides of the NB oracle's series switch), and rows whose
    mean runs from 1e-6 to 1e3, zeros among them."""
    rows, P = [90, 60], 8
    Xs, ys, ws, os_ = _case(rows, P, family, seed=2, n_masked=0, alpha=np.exp(log_alpha), log_mu=(np.log(1e-6), np.log(1e3)))
    assert all(bool((y == 0).any()) and bool((y > 0).any()) for y in ys)
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family=family, weights=ws, offsets=os_)
    Xn = [X.double().numpy() for X in Xs]
    yn = [y.double().numpy() for y in ys]
    wn = [w.double().numpy() if w is not None else np.ones(len(y)) for w, y in zip(ws, ys)]
    on = [o.double().numpy() if o is not None else np.zeros(len(y)) for o, y in zip(os_, ys)]
    truth = _scipy_truth(family, Xn, yn, wn, on, [0, 1])
    inputs = [np.asarray(v, dtype=np.float64) for v in _theta(family, 2, P, zi=zi, log_alpha=log_alpha, scale=0.2)]
    # the mean of the first segment's rows ranges over 1e-6 .. 1e3 with these inputs as well
    eta0 = Xn[0] @ inputs[1] + inputs[0][0] + on[0]
    assert eta0.min() < np.log(1e-5) and eta0.max() > np.log(3e2)
    got = _oracle(model, *inputs)
    assert len(got) == len(inputs) + 1
    for g, x in zip(got[1:], inputs):
        assert np.shape(g) == np.shape(x)
    np.testing.assert_allclose(got[0], truth(*inputs), rtol=1e-10)
    eps = 1e-4   # scipy's lgamma differences lose ~1e-11 at alpha = 1e4: a wider step keeps that out of the quotient
    for arr, grad in zip(inputs, got[1:]):
        fd = np.zeros_like(arr)
        for idx in np.ndindex(arr.shape):
            orig = arr[idx]
            arr[idx] = orig + eps
            hi = truth(*inputs)
            arr[idx] = orig - eps
            lo = truth(*inputs)
            arr[idx] = orig
            fd[idx] = (hi - lo) / (2 * eps)
        np.testing.assert_allclose(grad, fd, rtol=1e-6, atol=1e-5)


@pytest.mark.parametrize("family", FAMILIES)
def test_oracle_at_a_vanishing_zero_part_is_the_plain_family(family):
    """zeta = -1000: sigmoid(zeta) and exp(zeta) are 0 in fp64, so the oracle is the Poisson / NB oracle and the zero
    part's gradients are exactly 0."""
    rows, P, K = [150, 70, 201], 16, 3
    Xs, ys, ws, os_ = _case(rows, P, family, seed=1)
    zi = GlmShards(Xs, ys, groups=[0, 1, 0], n_groups=2, family=family, n_chains=K, weights=ws, offsets=os_)
    ys_b = [torch.nan_to_num(y).clamp(min=0).round() for y in ys]   # masked rows: any valid count
    base = GlmShards(Xs, ys_b, groups=[0, 1, 0], n_groups=2, family=BASE[family], n_chains=K, weights=ws, offsets=os_)
    inp = _theta(family, 2, P, K, log_alpha=[0.3, -1.2, 2.5])
    inp = (inp[0], inp[1], np.full_like(inp[2], -1000.0), inp[3]) + inp[4:]
    a = _oracle(zi, *inp)
    b = base.unpack_result(base.reference_partial([inp[0], inp[1], *inp[4:]], dtype=torch.float64))
    np.testing.assert_allclose(a[0], b[0], rtol=1e-13)
    np.testing.assert_allclose(a[1], b[1], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(a[2], b[2], rtol=1e-12, atol=1e-12)
    assert np.all(a[3] == 0.0) and np.all(a[4] == 0.0)
    if family == NB:
        np.testing.assert_allclose(a[5], b[3], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("K,G", [(1, 1), (1, 2), (3, 2)])
@pytest.mark.parametrize("family", FAMILIES)
def test_pack_unpack_and_words_round_trip(family, K, G):
    P = 8
    Xs, ys, _, _ = _case([20] * G, P, family, seed=7, n_masked=0, weighted=False, offsets=False)
    model = GlmShards(Xs, ys, groups=list(range(G)), n_groups=G, family=family, n_chains=K)
    inp = list(_theta(family, G, P, K, log_alpha=np.arange(K) - 0.5 if K > 1 else -0.5, scale=1.0))
    if K == 1 and G == 1:
        inp[0], inp[2] = inp[0].reshape(()), inp[2].reshape(())   # scalar intercepts for one group
    nb = family == NB
    words = np.zeros(model.n_theta_words, dtype=np.uint32)
    ctx = model.pack_theta(inp, words)
    assert ctx == model.call_context(inp) == (K > 1, np.shape(inp[0])) + tuple(np.shape(x) for x in inp[2:])
    # the kernel's layout: rows 2k = (intercept, beta[, log_dispersion]), 2k + 1 = (zi_intercept, zi_beta[, same])
    th = words.view(np.float32).reshape(K, 2, G + P + nb)
    np.testing.assert_array_equal(th[:, 0, :G], np.reshape(inp[0], (K, G)))
    np.testing.assert_array_equal(th[:, 0, G : G + P], np.reshape(inp[1], (K, P)))
    np.testing.assert_array_equal(th[:, 1, :G], np.reshape(inp[2], (K, G)))
    np.testing.assert_array_equal(th[:, 1, G : G + P], np.reshape(inp[3], (K, P)))
    if nb:
        np.testing.assert_array_equal(th[:, 0, -1], np.reshape(inp[4], K))
        np.testing.assert_array_equal(th[:, 1, -1], np.reshape(inp[4], K))
    back = default_inputs_from_words(model, words)
    assert len(back) == len(inp)
    for u, v in zip(back, inp):
        assert np.array_equal(np.reshape(u, np.shape(v)), v)
    words2 = np.zeros_like(words)
    model.pack_theta(back, words2)
    assert np.array_equal(words, words2)
    # unpack: block 2k holds [LL, gi[G], g[P](, q)] of the count predictor, block 2k + 1 [0, gi, g(, 0)] of zeta
    raw = np.arange(model.n_vals, dtype=np.float64).reshape(K, 2, 1 + G + P + nb)
    got = model.unpack_result(raw.reshape(-1), ctx)
    assert len(got) == 1 + len(inp)
    for g, x in zip(got[1:], inp):
        assert np.shape(g) == np.shape(x)
    np.testing.assert_array_equal(np.reshape(got[0], -1), raw[:, 0, 0])
    np.testing.assert_array_equal(np.reshape(got[1], (K, G)), raw[:, 0, 1 : 1 + G])
    np.testing.assert_array_equal(np.reshape(got[2], (K, P)), raw[:, 0, 1 + G : 1 + G + P])
    np.testing.assert_array_equal(np.reshape(got[3], (K, G)), raw[:, 1, 1 : 1 + G])
    np.testing.assert_array_equal(np.reshape(got[4], (K, P)), raw[:, 1, 1 + G : 1 + G + P])
    if nb:
        np.testing.assert_array_equal(np.reshape(got[5], K), raw[:, 0, -1])


@pytest.mark.parametrize("family", FAMILIES)
def test_sizes_and_flops(family):
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ys = [torch.zeros(10), torch.zeros(6)]
    nb = int(family == NB)
    m = GlmShards(Xs, ys, n_groups=2, groups=[0, 1], family=family, n_chains=3, node_ids=[0, 1], n_nodes=2)
    assert m.n_inputs == 4 + nb and m.kernel_chains == 6
    assert m.input_shapes == [(2,), (16,), (2,), (16,)] + [()] * nb
    assert m.n_params == 2 * (2 + 16) + nb and m.n_theta_words == 6 * (2 + 16 + nb)
    assert m.n_vals == 2 * 6 * (1 + 2 + 16 + nb)
    assert m.flops_per_eval() == GlmShards(Xs, ys, n_chains=6).flops_per_eval() == 4 * 16 * 16 * 6
    assert m.bytes_per_eval() == GlmShards(Xs, ys).bytes_per_eval()
    assert m.per_node(np.zeros(m.n_vals)).shape == (2, 3, 1 + m.n_params)


def test_validation():
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ys = [torch.zeros(10), torch.full((6,), 2.0)]
    for family in FAMILIES:
        GlmShards(Xs, ys, family=family)
        GlmShards(Xs, ys, family=family, n_chains=8, offsets=[torch.zeros(10), None], weights=[None, torch.ones(6)])
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
        with pytest.raises(ValueError, match=r"n_chains in \[1, 8\]"):
            GlmShards(Xs, ys, family=family, n_chains=9)
        # shapes outside the tensor-core kernel's: an error, never another kernel
        for X in (torch.randn(10, 12).to(torch.bfloat16), torch.randn(10, 392).to(torch.bfloat16), torch.randn(10, 16)):
            with pytest.raises(ValueError, match="tensor-core kernel only"):
                GlmShards([X], [torch.zeros(10)], family=family).use_tensor_cores()
        assert GlmShards(Xs, ys, family=family, kernel="tc").use_tensor_cores() == 1
        for bad in (-1.0, 0.5, float("nan"), float("inf"), 2.0 ** 24 + 2):
            y0 = torch.zeros(10)
            y0[4] = bad
            with pytest.raises(ValueError, match="counts of segment 0"):
                GlmShards(Xs, [y0, ys[1]], family=family)
            w0 = torch.ones(10)
            w0[4] = 0.0
            GlmShards(Xs, [y0, ys[1]], weights=[w0, None], family=family)   # a masked row may carry anything
        y0 = torch.zeros(10)
        y0[4] = 2.0 ** 24
        GlmShards(Xs, [y0, ys[1]], family=family)


@pytest.mark.parametrize("family", FAMILIES)
def test_too_few_stages_refused_at_attach(family):
    from pytensor_federated_b200.ops import native

    lib = native.load()
    m = GlmShards([torch.zeros(8, 384, dtype=torch.bfloat16)], [torch.zeros(8)], n_chains=8, family=family)
    with pytest.raises(ValueError, match="fewer than two pipeline stages"):
        m.attach(lib, None)   # raises before the engine is touched
    code = 9 if family == "zero_inflated_poisson" else 10
    assert lib.b200_glm_tc_stages(384, 16, 1, code, 0) < 2
    assert lib.b200_glm_tc_stages(384, 8, 1, code, 3) >= 2   # 4 pairs with offsets and weights fit
    assert lib.b200_glm_tc_stages(256, 16, 1, code, 3) >= 2


@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("family", FAMILIES)
def test_collective_backend_equals_the_oracle(family, K):
    rows, P = [300, 45, 129], 24
    Xs, ys, ws, os_ = _case(rows, P, family, seed=6)
    model = GlmShards(Xs, ys, groups=[0, 1, 1], n_groups=2, family=family, n_chains=K, weights=ws, offsets=os_)
    inp = _theta(family, 2, P, K, zi=[-2.0, 0.0, 1.0, 3.0][:K] if K > 1 else -1.0,
                 log_alpha=[0.5, -1.0, 2.0, 9.0][:K] if K > 1 else 0.5)
    got, want = _collective(model, *inp), _oracle(model, *inp)
    assert len(got) == len(want) == 1 + len(inp)
    for u, v in zip(got, want):
        assert np.shape(u) == np.shape(v) and np.all(np.isfinite(u))
        np.testing.assert_allclose(u, v, rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("family", FAMILIES)
def test_glm_batch_fn_splits_theta_in_input_order(family):
    from pytensor_federated_b200.sampling import glm_batch_fn

    P, G = 8, 2
    Xs, ys, ws, os_ = _case([60, 40], P, family, seed=8)
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=G, family=family, n_chains=2, weights=ws, offsets=os_)
    rng = np.random.default_rng(9)
    theta = rng.normal(size=(3, model.n_params)) * 0.1
    with FederatedEngine(model, backend="collective") as eng:
        logp, grad = glm_batch_fn(eng, G)(theta)
    assert logp.shape == (3,) and grad.shape == theta.shape
    single = GlmShards(Xs, ys, groups=[0, 1], n_groups=G, family=family, weights=ws, offsets=os_)
    for i in range(3):
        # theta = [intercept[G], beta[P], zi_intercept[G], zi_beta[P](, log_dispersion)]
        parts = np.split(theta[i], np.cumsum([G, P, G, P])[: single.n_inputs - 1])
        want = _oracle(single, *[p if p.size > 1 else p.reshape(()) for p in parts])
        np.testing.assert_allclose(logp[i], want[0], rtol=1e-5)
        np.testing.assert_allclose(grad[i], np.concatenate([np.reshape(w, -1) for w in want[1:]]), rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("alpha", [None, 2.5])
def test_synth_zero_inflated_shard(alpha):
    n, mu, zi = 200_000, np.exp(0.7), -0.4
    X, y, beta, zbeta = synth_zero_inflated_shard(n, 16, alpha=alpha, seed=1, device="cpu", chunk_rows=65536,
                                                  beta_scale=0.0, intercept=0.7, zi_intercept=zi, zi_beta_scale=0.0)
    assert X.dtype == torch.bfloat16 and X.shape == (n, 16) and beta.shape == zbeta.shape == (16,)
    yn = y.double().numpy()
    assert y.dtype == torch.float32 and np.all(yn == np.floor(yn)) and yn.min() >= 0
    pi = 1.0 / (1.0 + np.exp(-zi))
    f0 = np.exp(-mu) if alpha is None else (alpha / (alpha + mu)) ** alpha
    p0 = pi + (1 - pi) * f0
    assert abs(np.mean(yn == 0) - p0) < 5 * np.sqrt(p0 * (1 - p0) / n)
    assert abs(yn.mean() - (1 - pi) * mu) < 5 * yn.std() / np.sqrt(n)
    X2, y2, _, _ = synth_zero_inflated_shard(n, 16, alpha=alpha, seed=1, device="cpu", chunk_rows=65536,
                                             beta_scale=0.0, intercept=0.7, zi_intercept=zi, zi_beta_scale=0.0)
    assert torch.equal(X, X2) and torch.equal(y, y2)


# ----------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from pytensor_federated_b200.ops import native

    native.load()  # a GPU box without the native library is a failure, not a skip
    return torch.device("cuda:0")


def _run(model, inputs_list, raw=False):
    """The engine's results (``raw``: the kernel's output blocks) for each set of inputs, one engine."""
    with FederatedEngine(model) as eng:
        if raw:
            return [np.asarray(eng.evaluate_raw(list(inputs)), dtype=np.float64).copy() for inputs in inputs_list]
        return [[np.asarray(v).copy() for v in eng.evaluate(*inputs)] for inputs in inputs_list]


def _check(got, want, n_rows, K):
    """The tolerances of the dispersion suite: LL at rtol 2e-5; gradients at rtol 1e-4 and an absolute tolerance for
    components that nearly cancel (intercepts 2e-3, beta 2e-3 sqrt(n) for one chain, 0.2 per chain otherwise; both
    predictors' residuals are of the size of Poisson ones, the zero logit's bounded by 1); d log_dispersion at
    2e-3 sqrt(n)."""
    assert len(got) == len(want)
    assert all(np.all(np.isfinite(g)) for g in got)
    for u, v in zip(got, want):
        assert np.shape(u) == np.shape(v)
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)
    atol_b = 2e-3 * np.sqrt(n_rows) if K == 1 else 0.2
    for i in (1, 3):
        np.testing.assert_allclose(got[i], want[i], rtol=1e-4, atol=2e-3)
        np.testing.assert_allclose(got[i + 1], want[i + 1], rtol=1e-4, atol=atol_b)
    if len(got) == 6:
        np.testing.assert_allclose(got[5], want[5], rtol=1e-4, atol=2e-3 * np.sqrt(n_rows))


@pytest.mark.parametrize("row_data", [True, False])
@pytest.mark.parametrize("K", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("P", [256, 200, 8])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_matches_oracle(dev, family, P, K, row_data):
    """K pairs run 2K columns: K <= 2, <= 4 and <= 8 select the kernel's 4, 8 and 16 buckets; ``row_data`` (offsets
    and weights, masked rows with NaN / negative / fractional counts) its ROWS variant.  The chains cycle through the
    zero-inflation intercepts (-3 .. 4) and the dispersion values (alpha 0.3 .. 1e4)."""
    rows = [128 * 37, 77, 4099, 1]
    Xs, ys, ws, os_ = _case(rows, P, family, seed=K + P, device=dev, weighted=row_data, offsets=row_data,
                            n_masked=5 if row_data else 0)
    model = GlmShards(Xs, ys, groups=[0, 1, 0, 1], n_groups=2, family=family, n_chains=K, kernel="auto",
                      weights=ws, offsets=os_)
    assert model.has_row_data == row_data
    if K == 1:
        inputs = [_theta(family, 2, P, 1, zi=z, log_alpha=a, seed=5 + i)
                  for i, (z, a) in enumerate(zip(ZI_ICPT, LOG_ALPHA))]
    else:
        inputs = [_theta(family, 2, P, K, zi=np.resize(ZI_ICPT, K), log_alpha=np.resize(LOG_ALPHA, K))]
    got = _run(model, inputs)
    assert model.selected_kernel == "tc"
    for g, inp in zip(got, inputs):
        _check(g, _oracle(model, *inp, chunk_rows=1 << 20), sum(rows), K)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("K,row_data", [(1, False), (2, True), (5, False), (5, True)])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_with_many_groups_matches_oracle(dev, family, K, row_data):
    """300 intercepts per predictor: the intercept table is KC x G floats, both predictors' rows of it in use."""
    G, P = 300, 256
    rows = [128 * 9 + 5, 999, 64, 1, 3000]
    groups = [0, 299, 150, 7, 299]
    Xs, ys, ws, os_ = _case(rows, P, family, seed=40 + K, device=dev, weighted=row_data, offsets=row_data,
                            n_masked=5 if row_data else 0)
    model = GlmShards(Xs, ys, groups=groups, n_groups=G, family=family, n_chains=K, kernel="tc", weights=ws,
                      offsets=os_)
    inp = _theta(family, G, P, K, zi=np.resize(ZI_ICPT[::-1], K) if K > 1 else 0.5,
                 log_alpha=np.resize(LOG_ALPHA[::-1], K) if K > 1 else LOG_ALPHA[0])
    (got,) = _run(model, [inp])
    _check(got, _oracle(model, *inp, chunk_rows=1 << 20), sum(rows), K)
    unused = np.ones(G, dtype=bool)
    unused[groups] = False
    assert np.all(got[1][..., unused] == 0.0) and np.all(got[3][..., unused] == 0.0)


@pytest.mark.parametrize("row_data", [False, True])
@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_vanishing_zero_part_is_bit_identical_to_the_plain_family(dev, family, K, row_data):
    """zeta = -120 and log f(0) >= -15 on every row (|eta| <= 2.5, alpha >= 1): the count columns of a K-pair launch
    are the even blocks of a 2K-chain Poisson / negative-binomial launch (same bucket, same column positions, same
    theta rows), and the zero columns are exactly 0."""
    rows, P = [128 * 30 + 9, 5000, 77], 256
    Xs, ys, ws, os_ = _case(rows, P, family, seed=11 + K, device=dev, weighted=row_data, offsets=row_data,
                            n_masked=5 if row_data else 0, beta_scale=0.01)
    zi = GlmShards(Xs, ys, groups=[0, 1, 0], n_groups=2, family=family, n_chains=K, kernel="tc", weights=ws,
                   offsets=os_)
    base = GlmShards(Xs, ys, groups=[0, 1, 0], n_groups=2, family=BASE[family], n_chains=2 * K, kernel="tc",
                     weights=ws, offsets=os_)
    inp = list(_theta(family, 2, P, K, log_alpha=np.resize([0.0, 1.0, 2.5], K) if K > 1 else 0.5, scale=0.01))
    inp[2] = np.full_like(inp[2], -120.0)
    inp[3] = np.zeros_like(inp[3])
    # |eta| <= 2.5 on every row: log f(0) >= -e^2.5 > -15 for Poisson and NB (alpha >= 1) alike
    ic, bt = np.reshape(inp[0], (K, 2)), np.reshape(inp[1], (K, P))
    for X, o, g in zip(Xs, os_, [0, 1, 0]):
        eta = X.double().cpu().numpy() @ bt.T.astype(np.float64) + ic[:, g] + (o.double().cpu().numpy()[:, None] if o is not None else 0.0)
        assert np.abs(eta).max() <= 2.5
    # the plain launch with the same theta rows: column 2k = (intercept, beta[, a]), 2k + 1 = (-120, 0[, a])
    lead = lambda x: np.reshape(x, (K, -1))
    b_ic = np.stack([lead(inp[0]), lead(inp[2])], axis=1).reshape(2 * K, 2)
    b_bt = np.stack([lead(inp[1]), lead(inp[3])], axis=1).reshape(2 * K, P)
    b_inp = [b_ic, b_bt] + ([np.repeat(np.reshape(inp[4], K), 2)] if family == NB else [])
    (a,), (b,) = _run(zi, [inp], raw=True), _run(base, [b_inp], raw=True)
    width = 1 + 2 + P + (family == NB)
    a, b = a.reshape(2 * K, width), b.reshape(2 * K, width)
    assert np.all(np.isfinite(a))
    assert a[0::2].tobytes() == b[0::2].tobytes()
    assert np.all(a[1::2] == 0.0)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_evaluations_are_bit_reproducible(dev, family):
    rows = [40_000, 25_000, 33_333, 128, 19_999]
    Xs, ys, ws, os_ = _case(rows, 256, family, seed=12, device=dev)
    model = GlmShards(Xs, ys, groups=[0, 1, 2, 1, 0], n_groups=3, family=family, n_chains=4, kernel="tc",
                      weights=ws, offsets=os_)
    inp = _theta(family, 3, 256, 4, zi=ZI_ICPT[:4], log_alpha=LOG_ALPHA[:4])
    runs = _run(model, [inp] * 10)
    for run in runs[1:]:
        for u, v in zip(runs[0], run):
            assert np.array_equal(u, v)


@pytest.mark.parametrize("rows_data", [False, True])
@pytest.mark.parametrize("K", [1, 2, 4])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_packed_launch_is_bitwise_the_unpacked_one(dev, family, K, rows_data, monkeypatch):
    """K = 1 and 2 are packed by default at P = 256 (2 and 4 columns); K = 4 (8 columns) is forced to pack."""
    P = 256
    Xs, ys, ws, os_ = _case([3 * 128 + 5, 1000, 128], P, family, seed=21 + K, device=dev, weighted=rows_data,
                            offsets=rows_data, n_masked=5 if rows_data else 0)
    inp = _theta(family, 1, P, K, zi=np.resize(ZI_ICPT, K) if K > 1 else 0.0,
                 log_alpha=np.resize(LOG_ALPHA, K) if K > 1 else 1.0)
    outs = {}
    for packed in (True, False):
        if packed:
            monkeypatch.delenv("B200FED_NO_PACKED_X", raising=False)
        else:
            monkeypatch.setenv("B200FED_NO_PACKED_X", "1")
        model = GlmShards(Xs, ys, family=family, n_chains=K, kernel="tc", weights=ws, offsets=os_)
        assert model._packing_pays(0) == (K <= 2)
        model._packing_pays = lambda row_data: True
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
    model = GlmShards(Xs, ys, groups=groups, n_groups=2, family=family, kernel="tc", node_ids=node_ids, n_nodes=2,
                      weights=ws, offsets=os_)
    inp = _theta(family, 2, 256, zi=-0.3, log_alpha=0.7)
    n_params = model.n_params
    with FederatedEngine(model) as eng:
        n0 = eng.kernel_launches
        blocks = model.per_node(eng.evaluate_raw(list(inp)))
        assert eng.kernel_launches - n0 == 1
        assert blocks.shape == (2, 1, 1 + n_params)
        fed = NodeFederation(eng)
        res = fed.evaluate_nodes({0: inp, 1: inp})
        total = fed.all_nodes_func()(*inp)
    for node in (0, 1):
        segs = [i for i, n in enumerate(node_ids) if n == node]
        single = GlmShards([Xs[i] for i in segs], [ys[i] for i in segs], groups=[groups[i] for i in segs], n_groups=2,
                           family=family, kernel="tc", weights=[ws[i] for i in segs], offsets=[os_[i] for i in segs])
        (want,) = _run(single, [inp])
        np.testing.assert_allclose(blocks[node, 0, 0], want[0], rtol=2e-5)
        flat = np.concatenate([np.reshape(w, -1) for w in want[1:]])
        np.testing.assert_allclose(blocks[node, 0, 1:], flat, rtol=1e-4, atol=0.5)
        np.testing.assert_allclose(res[node][0], blocks[node, 0, 0], rtol=1e-12)
        assert len(res[node][1]) == len(inp)
        for g, x in zip(res[node][1], inp):
            assert np.shape(g) == np.shape(x)
        np.testing.assert_allclose(np.concatenate([np.reshape(g, -1) for g in res[node][1]]), blocks[node, 0, 1:],
                                   rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(total[0], blocks[:, 0, 0].sum(), rtol=1e-12)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_lock_step_hmc_on_a_zero_inflated_negative_binomial_engine(dev):
    from pytensor_federated_b200.sampling import glm_batch_fn, hmc_sample_batched

    K, P = 4, 16
    X, y, _, _ = synth_zero_inflated_shard(20_000, P, alpha=3.0, seed=3, device=dev)
    model = GlmShards([X], [y], family=NB, n_chains=K, kernel="tc")
    x0 = np.zeros((K, model.n_params))
    x0[:, 1 + P] = -1.0        # zi_intercept
    x0[:, -1] = np.log(3.0)    # log_dispersion
    with FederatedEngine(model) as eng:
        res = hmc_sample_batched(glm_batch_fn(eng, 1), x0, draws=5, tune=5, n_leapfrog=4, step_size=1e-3, seed=1)
        assert eng.n_evals == res.n_batched_evals
    assert res.samples.shape[-1] == model.n_params and np.all(np.isfinite(res.samples))
    assert np.all(res.accept_rate > 0)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_runtime_rejects_the_zero_inflated_families_outside_their_launch(dev):
    """The C ABI refuses what the Python layer never sends: codes 9 and 10 on a CUDA-core kernel, an odd n_chains,
    n_classes != 1 and an output size that does not match, and the engine keeps evaluating its own model."""
    from pytensor_federated_b200.ops import native

    Xs, ys, _, _ = _case([256], 16, NB, seed=14, device=dev, n_masked=0, weighted=False, offsets=False)
    model = GlmShards(Xs, ys, kernel="simt")
    with FederatedEngine(model) as eng:
        lib, h = eng._lib, eng._handle
        Xp, yp = native.void_p_array([Xs[0].data_ptr()]), native.void_p_array([ys[0].data_ptr()])
        rows, grp = (C.c_longlong * 1)(256), (C.c_int * 1)(0)

        def set_glm(n_chains, family, code, n_classes=1):
            return int(lib.b200_engine_set_glm(h, 1, Xp, yp, None, rows, grp, 16, 16, 1, n_chains, family, code, None, 1,
                                               None, None, n_classes))

        for family, name in ((9, "zero_inflated_poisson"), (10, "zero_inflated_negative_binomial")):
            for code in (0, 2, 3, 4):
                assert set_glm(2, family, code) != 0
                assert f"the {name} family runs on the bf16 tensor-core kernel only" in native.last_error()
            assert set_glm(2, family, 1, 2) != 0 and "n_classes must be 1" in native.last_error()
            for n_chains in (1, 3, 18):
                assert set_glm(n_chains, family, 1) == -44 and "even n_chains in [2, 16]" in native.last_error()
            # this engine's n_vals is 1 + G + P: a 2-column launch needs twice that (plus the dispersion words)
            assert set_glm(2, family, 1) == -33 and "n_vals does not match" in native.last_error()
            assert set_glm(2, family | 16, 1) != 0   # no Hessian-vector products of these families
        ic, beta = np.float32(0.1), np.zeros(16, np.float32)
        got = eng.evaluate(ic, beta)
    want = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)


def _build_zinb_model(rank, world, dev):
    Xs, ys, ws, os_ = _case([30_000 + 17 * rank, 999], 256, NB, seed=50 + rank, device=dev)
    return GlmShards(Xs, ys, groups=[rank % 2, 1 - rank % 2], n_groups=2, family=NB, n_chains=2, kernel="tc",
                     weights=ws, offsets=os_)


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.timeout(900)
def test_two_rank_zero_inflated_negative_binomial_federation_matches_oracle():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from pytensor_federated_b200.federation import launch_federation

    inp = _theta(NB, 2, 256, 2, zi=[-1.0, 0.5], log_alpha=[0.0, 3.0])
    dev = torch.device("cuda:0")
    models = [_build_zinb_model(r, 2, dev) for r in range(2)]
    want = models[0].unpack_result(sum(m.reference_partial(list(inp), dtype=torch.float64) for m in models),
                                   models[0].call_context(list(inp)))
    del models
    with launch_federation(_build_zinb_model, 2, timeout=30.0) as eng:
        got = eng.evaluate(*inp)
    _check(got, want, 2 * 31_000, 2)
