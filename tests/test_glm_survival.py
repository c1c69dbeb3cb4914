"""Right-censored survival regression: ``GlmShards(Xs, times, family="weibull" | "lognormal", events=[...])``,
accelerated failure time with s = log sigma learned.

CPU tests check the fp64 oracle and the collective backend against independent formulas (scipy, autograd of the
textbook log-likelihood, finite differences), the families the two reduce to, validation and the model's packing;
GPU tests check the tensor-core kernel against that oracle."""
import ctypes as C

import numpy as np
import pytest
import torch

from pytensor_federated_b200.models import Fp8GlmShards, GlmShards, synth_survival_shard
from pytensor_federated_b200.parallel import FederatedEngine
from pytensor_federated_b200.parallel.engine import default_inputs_from_words

FAMILIES = ("weibull", "lognormal")
# log sigma of the GPU tests
LOG_SIGMA = np.log([0.05, 0.5, 1.0, 3.0])


# ----------------------------------------------------------------------------------------------- fixtures
def _beta_true(P):
    return np.random.default_rng(1000 + P).normal(size=P) * 0.01


def _eps(rng, family, n):
    """Standard minimum-Gumbel (Weibull) or standard normal (log-normal) draws."""
    return np.log(-np.log(rng.uniform(size=n))) if family == "weibull" else rng.normal(size=n)


def _case(rows, P, family, *, seed=0, device="cpu", n_masked=5, weighted=True, offsets=True, censor=0.3, sigma=0.1):
    """Ragged bf16 segments with times drawn from the family at ``intercept = 0.4``, ``beta = _beta_true(P)`` and
    ``sigma``; a ``censor`` share of the rows is censored at a time drawn uniformly below its event time.  With
    ``weighted``, every segment but the last has weights; the first ``n_masked`` rows of segment 0 have weight 0 and
    carry a NaN, a negative and a zero time and events NaN and 2.  With ``offsets``, every segment but the second has
    offsets.  Returns ``(Xs, times, events, weights, offsets)``; events are None for the third segment."""
    rng = np.random.default_rng(seed)
    Xs, ts, es, ws, os_ = [], [], [], [], []
    for si, n in enumerate(rows):
        X = torch.tensor(rng.normal(size=(n, P)), dtype=torch.float32).to(torch.bfloat16)
        o = rng.uniform(-0.5, 0.5, size=n)
        eta = X.double().numpy() @ _beta_true(P) + 0.4 + (o if offsets else 0.0)
        t = np.exp(eta + sigma * _eps(rng, family, n))
        ev = (rng.uniform(size=n) >= censor).astype(np.float64)
        if si == 2:
            ev[:] = 1.0
        t = np.where(ev == 1, t, t * rng.uniform(0.3, 1.0, size=n))
        w = rng.uniform(0.2, 2.0, size=n)
        if si == 0 and n_masked:
            w[:n_masked] = 0.0
            t[:3] = [np.nan, -1.0, 0.0][: min(3, n_masked)]
            ev[:2] = [np.nan, 2.0][: min(2, n_masked)]
        Xs.append(X.to(device))
        ts.append(torch.tensor(t, dtype=torch.float32, device=device))
        es.append(None if si == 2 else torch.tensor(ev, dtype=torch.float32, device=device))
        ws.append(torch.tensor(w, dtype=torch.float32, device=device) if weighted and si < len(rows) - 1 else None)
        os_.append(torch.tensor(o, dtype=torch.float32, device=device) if offsets and si != 1 else None)
    return Xs, ts, es, ws, os_


def _theta(G, P, K=1, log_sigma=np.log(0.1), seed=3, scale=0.002):
    """``(intercept, beta, log_sigma)`` near the parameters the data were drawn at; batched (``[K, G]``, ``[K, P]``,
    ``[K]``) for K > 1, where ``log_sigma`` may give one value per chain."""
    rng = np.random.default_rng(seed)
    b0 = _beta_true(P)
    if K == 1:
        return ((0.4 + rng.normal(size=G) * 0.02).astype(np.float32), (b0 + rng.normal(size=P) * scale).astype(np.float32),
                np.float32(log_sigma))
    return ((0.4 + rng.normal(size=(K, G)) * 0.02).astype(np.float32),
            (b0 + rng.normal(size=(K, P)) * scale).astype(np.float32),
            np.broadcast_to(np.asarray(log_sigma, dtype=np.float32), (K,)).copy())


def _model(Xs, ts, es, ws, os_, family, **kw):
    return GlmShards(Xs, ts, family=family, events=es, weights=ws, offsets=os_, **kw)


def _event_arrays(ts, es, ws):
    """Per segment: (time, delta, weight) as float64 numpy with masked rows set to t = 1, delta = 1, w = 0."""
    out = []
    for t, e, w in zip(ts, es, ws):
        t = t.double().cpu().numpy()
        d = np.ones_like(t) if e is None else e.double().cpu().numpy()
        w = np.ones_like(t) if w is None else w.double().cpu().numpy()
        out.append((np.where(w != 0, t, 1.0), np.where(w != 0, d, 1.0), w))
    return out


def _textbook_fp64(family, Xs, ts, es, ws, os_, groups, ic, beta, ls):
    """``[LL, d intercept, d beta, d log_sigma]`` by autograd of the textbook densities in scale / shape form."""
    batched = np.ndim(beta) == 2
    ic, beta, ls = (np.asarray(v, dtype=np.float64) for v in (ic, beta, ls))
    if not batched:
        ic, beta, ls = ic.reshape(1, -1), beta[None], ls.reshape(1)
    t_ic, t_b, t_ls = (torch.tensor(v, requires_grad=True) for v in (ic, beta, ls))
    total = torch.zeros(beta.shape[0], dtype=torch.float64)
    for X, (t, d, w), o, g in zip(Xs, _event_arrays(ts, es, ws), os_, groups):
        X, t, d, w = X.double().cpu(), torch.tensor(t), torch.tensor(d), torch.tensor(w)
        eta = t_b @ X.T + t_ic[:, g, None]                             # [K, n]
        if o is not None:
            eta = eta + torch.where(w != 0, o.double().cpu(), torch.zeros_like(w))
        sigma = torch.exp(t_ls)[:, None]
        if family == "weibull":
            k, lam = 1.0 / sigma, torch.exp(eta)                       # shape, scale
            H = (t / lam) ** k                                          # cumulative hazard
            logf = torch.log(k) - torch.log(lam) + (k - 1) * torch.log(t / lam) - H
            ll = torch.where(d == 1, logf, -H)
        else:
            z = (torch.log(t) - eta) / sigma
            logf = -0.5 * z * z - torch.log(sigma) - 0.5 * np.log(2 * np.pi) - torch.log(t)
            ll = torch.where(d == 1, logf, torch.log(0.5 * torch.erfc(z / np.sqrt(2.0))))
        ll = torch.where(w != 0, w * ll, torch.zeros_like(ll))
        total = total + ll.sum(1)
    total.sum().backward()
    out = [total.detach().numpy(), t_ic.grad.numpy(), t_b.grad.numpy(), t_ls.grad.numpy()]
    return out if batched else [out[0][0], out[1][0], out[2][0], out[3][0]]


def _oracle(model, *inputs, chunk_rows=128):
    return model.unpack_result(model.reference_partial(list(inputs), dtype=torch.float64, chunk_rows=chunk_rows))


def _collective(model, *inputs):
    with FederatedEngine(model, backend="collective") as eng:
        return [np.asarray(v, dtype=np.float64) for v in eng.evaluate(*inputs)]


def _tail_case(family, sigma, seed):
    """Two segments whose rows sit at z = (log t - eta) / sigma spread over [-30, 30] (|log t| < 80 for float32),
    half of them censored, at the parameters ``_theta(2, 8, seed=seed)``."""
    rng = np.random.default_rng(seed)
    P = 8
    ic, beta, _ = _theta(2, P, seed=seed)
    zmax = min(30.0, 80.0 / sigma)
    Xs, ts, es = [], [], []
    for g, n in enumerate((61, 40)):
        X = torch.tensor(rng.normal(size=(n, P)), dtype=torch.float32).to(torch.bfloat16)
        eta = X.double().numpy() @ beta.astype(np.float64) + float(ic[g])
        z = np.concatenate([[-zmax, zmax, -zmax, zmax], rng.uniform(-zmax, zmax, size=n - 4)])
        Xs.append(X)
        ts.append(torch.tensor(np.exp(eta + sigma * z), dtype=torch.float32))
        es.append(torch.tensor(np.arange(n) % 2, dtype=torch.float32))
    return Xs, ts, es, (ic, beta)


# ----------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("sigma", [0.05, 0.5, 1.0, 3.0])
@pytest.mark.parametrize("family", FAMILIES)
def test_oracle_matches_scipy_and_finite_differences(family, sigma):
    """Mixed censoring, rows with |z| up to 30: the oracle's LL is scipy's logpdf (events) + logsf (censored rows),
    and its gradients are central differences of that sum."""
    import scipy.stats

    Xs, ts, es, (ic, beta) = _tail_case(family, sigma, seed=int(sigma * 100))
    model = GlmShards(Xs, ts, groups=[0, 1], n_groups=2, family=family, events=es)
    Xn = [X.double().numpy() for X in Xs]
    tn = [t.double().numpy() for t in ts]
    dn = [e.numpy() == 1 for e in es]

    def truth(ic, beta, ls):
        total = 0.0
        for g, (X, t, d) in enumerate(zip(Xn, tn, dn)):
            eta = X @ beta + ic[g]
            sg = np.exp(ls[()])
            dist = (scipy.stats.weibull_min(c=1.0 / sg, scale=np.exp(eta)) if family == "weibull"
                    else scipy.stats.lognorm(s=sg, scale=np.exp(eta)))
            total += np.sum(np.where(d, dist.logpdf(t), dist.logsf(t)))
        return total

    ic, beta = ic.astype(np.float64), beta.astype(np.float64)
    ls = np.asarray(np.log(sigma))
    got = _oracle(model, ic, beta, ls)
    np.testing.assert_allclose(got[0], truth(ic, beta, ls), rtol=1e-10)
    eps = 1e-6 * sigma
    for arr, grad in ((ic, got[1]), (beta, got[2]), (ls, got[3])):
        fd = np.zeros_like(arr)
        for idx in np.ndindex(arr.shape):
            orig = arr[idx].copy()
            arr[idx] = orig + eps
            hi = truth(ic, beta, ls)
            arr[idx] = orig - eps
            lo = truth(ic, beta, ls)
            arr[idx] = orig
            fd[idx] = (hi - lo) / (2 * eps)
        np.testing.assert_allclose(grad, fd, rtol=1e-5, atol=1e-5 * np.max(np.abs(fd)))


@pytest.mark.parametrize("K", [1, 3])
@pytest.mark.parametrize("family", FAMILIES)
def test_oracle_matches_autograd_of_the_textbook_loglik(family, K):
    rows, P, groups = [150, 70, 201], 16, [0, 1, 0]
    Xs, ts, es, ws, os_ = _case(rows, P, family, seed=1)
    model = _model(Xs, ts, es, ws, os_, family, groups=groups, n_groups=2, n_chains=K)
    ic, beta, ls = _theta(2, P, K, log_sigma=[-2.0, 0.3, 1.1][:K] if K > 1 else -1.5)
    got = _oracle(model, ic, beta, ls)
    want = _textbook_fp64(family, Xs, ts, es, ws, os_, groups, ic, beta, ls)
    assert np.all(np.isfinite(got[0]))
    assert got[1].shape == ic.shape and got[2].shape == beta.shape and np.shape(got[3]) == np.shape(ls)
    np.testing.assert_allclose(got[0], want[0], rtol=1e-12)
    for u, v in zip(got[1:], want[1:]):
        np.testing.assert_allclose(u, v, rtol=1e-10, atol=1e-10 * np.max(np.abs(v)))


def _weibull_poisson_pair(rows, P, *, seed, device="cpu", weighted=True, **kw):
    """A Weibull model and the Poisson model it equals at s = 0: y = delta, offset = log t - o."""
    Xs, ts, es, ws, os_ = _case(rows, P, "weibull", seed=seed, device=device, weighted=weighted, offsets=weighted,
                                n_masked=5 if weighted else 0)
    wb = _model(Xs, ts, es, ws, os_, "weibull", groups=[0, 1, 0][: len(rows)], n_groups=2, **kw)
    ys_p, os_p = [], []
    for t, e, o in zip(ts, es, os_):
        ys_p.append(torch.ones_like(t) if e is None else e.clone())
        os_p.append(torch.log(t) - (o if o is not None else 0.0))
    po = GlmShards(Xs, ys_p, groups=[0, 1, 0][: len(rows)], n_groups=2, family="poisson", weights=ws, offsets=os_p, **kw)
    shift = 0.0   # sum w delta log t
    for t, (tt, d, w) in zip(ts, _event_arrays(ts, es, ws)):
        shift += float(np.sum(np.where(w != 0, w * d * np.log(tt), 0.0)))
    return wb, po, shift


@pytest.mark.parametrize("weighted", [False, True])
def test_weibull_at_unit_sigma_is_poisson_on_the_events(weighted):
    """Weibull at s = 0: ll = delta (z - log t) - e^z with z = log t - eta, i.e. Poisson with y = delta,
    offset = log t - o and negated (intercept, beta), less delta log t."""
    wb, po, shift = _weibull_poisson_pair([130, 77, 64], 16, seed=4, weighted=weighted)
    ic, beta, _ = _theta(2, 16)
    a = _oracle(wb, ic, beta, np.float32(0.0))
    b = po.unpack_result(po.reference_partial([-ic, -beta], dtype=torch.float64))
    # the Poisson offsets log t - o are stored as float32, so the two differ by that rounding (~1e-8 per row)
    np.testing.assert_allclose(a[0], b[0] - shift, rtol=1e-8)
    np.testing.assert_allclose(a[1], -b[1], rtol=1e-6, atol=1e-6 * np.max(np.abs(b[1])))
    np.testing.assert_allclose(a[2], -b[2], rtol=1e-6, atol=1e-6 * np.max(np.abs(b[2])))


def _lognormal_gaussian_pair(rows, P, *, seed, device="cpu", weighted=True, **kw):
    """A log-normal model with every row an event and the gaussian_scale model on y = log t."""
    Xs, ts, _, ws, os_ = _case(rows, P, "lognormal", seed=seed, device=device, weighted=weighted, offsets=weighted,
                               n_masked=5 if weighted else 0, censor=0.0)
    ln = _model(Xs, ts, None, ws, os_, "lognormal", groups=[0, 1, 0][: len(rows)], n_groups=2, **kw)
    gs = GlmShards(Xs, [torch.log(t) for t in ts], groups=[0, 1, 0][: len(rows)], n_groups=2, family="gaussian_scale",
                   weights=ws, offsets=os_, **kw)
    shift = 0.0   # sum w log t
    for tt, _, w in _event_arrays(ts, [None] * len(ts), ws):
        shift += float(np.sum(np.where(w != 0, w * np.log(tt), 0.0)))
    return ln, gs, shift


@pytest.mark.parametrize("weighted", [False, True])
def test_lognormal_without_censoring_is_gaussian_scale_on_log_times(weighted):
    ln, gs, shift = _lognormal_gaussian_pair([130, 77, 64], 16, seed=5, weighted=weighted)
    ic, beta, ls = _theta(2, 16, log_sigma=-0.7)
    a, b = _oracle(ln, ic, beta, ls), _oracle(gs, ic, beta, ls)
    # the Gaussian responses log t are stored as float32, so the two differ by that rounding
    np.testing.assert_allclose(a[0], b[0] - shift, rtol=1e-8)
    for u, v in zip(a[1:], b[1:]):
        np.testing.assert_allclose(u, v, rtol=1e-6, atol=1e-6 * np.max(np.abs(v)))


@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("family", FAMILIES)
def test_collective_backend_equals_the_oracle(family, K):
    rows, P = [300, 45, 129], 24
    Xs, ts, es, ws, os_ = _case(rows, P, family, seed=6, sigma=0.5)
    model = _model(Xs, ts, es, ws, os_, family, groups=[0, 1, 1], n_groups=2, n_chains=K)
    ic, beta, ls = _theta(2, P, K, log_sigma=[-0.5, 0.0, 0.7, -1.0][:K] if K > 1 else -0.5)
    got, want = _collective(model, ic, beta, ls), _oracle(model, ic, beta, ls)
    for u, v in zip(got, want):
        assert np.shape(u) == np.shape(v) and np.all(np.isfinite(u))
        np.testing.assert_allclose(u, v, rtol=1e-4, atol=1e-3)


def test_survival_validation():
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ts = [torch.full((10,), 2.0), torch.full((6,), 0.5)]
    es = [torch.ones(10), None]
    for family in FAMILIES:
        GlmShards(Xs, ts, family=family)
        GlmShards(Xs, ts, family=family, events=es, offsets=[torch.zeros(10), None], weights=[None, torch.ones(6)])
        GlmShards(Xs, ts, family=family, events=[np.zeros(10), [1, 0, 1, 0, 1, 0]])   # arrays and lists
        for kernel in ("simt", "generic", "fp8"):
            with pytest.raises(ValueError, match="tensor-core kernel only"):
                GlmShards(Xs, ts, family=family, kernel=kernel)
        with pytest.raises(ValueError, match="tensor-core kernel only"):
            Fp8GlmShards.from_dense([torch.randn(10, 32), torch.randn(6, 32)], ts, family=family)
        with pytest.raises(ValueError, match="n_classes"):
            GlmShards(Xs, ts, family=family, n_classes=2)
        for X in (torch.randn(10, 12).to(torch.bfloat16), torch.randn(10, 392).to(torch.bfloat16), torch.randn(10, 16)):
            with pytest.raises(ValueError, match="tensor-core kernel only"):
                GlmShards([X], [torch.ones(10)], family=family).use_tensor_cores()
        assert GlmShards(Xs, ts, family=family, kernel="tc").use_tensor_cores() == 1
        for bad in (0.0, -1.0, float("nan"), float("inf"), float("-inf")):
            t0 = torch.full((10,), 2.0)
            t0[4] = bad
            with pytest.raises(ValueError, match="times of segment 0 must be finite and > 0"):
                GlmShards(Xs, [t0, ts[1]], family=family)
            w0 = torch.ones(10)
            w0[4] = 0.0
            GlmShards(Xs, [t0, ts[1]], family=family, weights=[w0, None])   # a masked row may carry anything
        for bad in (0.5, 2.0, -1.0, float("nan")):
            e1 = torch.ones(6)
            e1[2] = bad
            with pytest.raises(ValueError, match="events of segment 1 must be 0 or 1"):
                GlmShards(Xs, ts, family=family, events=[None, e1])
            w1 = torch.ones(6)
            w1[2] = 0.0
            GlmShards(Xs, ts, family=family, events=[None, e1], weights=[None, w1])
        with pytest.raises(ValueError, match="events needs one entry"):
            GlmShards(Xs, ts, family=family, events=[None])
        with pytest.raises(ValueError, match="events of segment 0 must be 1-D with 10 rows"):
            GlmShards(Xs, ts, family=family, events=[torch.ones(9), None])
    for family in ("logistic", "poisson", "gaussian", "gaussian_scale", "negative_binomial"):
        with pytest.raises(ValueError, match="events= is for family='weibull' or 'lognormal' only"):
            GlmShards(Xs, [torch.zeros(10), torch.zeros(6)], family=family, events=es)


def test_the_times_passed_in_are_not_modified():
    Xs = [torch.randn(10, 16).to(torch.bfloat16)]
    t = torch.linspace(0.5, 3.0, 10)
    keep = t.clone()
    ev = torch.tensor([1, 0] * 5, dtype=torch.float32)
    m = GlmShards(Xs, [t], family="weibull", events=[ev])
    assert torch.equal(t, keep) and torch.equal(m.ys[0], keep)
    assert torch.equal(m._layout.kernel_ys[0], torch.where(ev == 1, t, -t))
    assert GlmShards(Xs, [t], family="lognormal")._layout.kernel_ys[0] is m.ys[0]   # all events: no copy


@pytest.mark.parametrize("family", FAMILIES)
def test_sizes_and_flops(family):
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ts = [torch.ones(10), torch.ones(6)]
    m = GlmShards(Xs, ts, n_groups=2, groups=[0, 1], family=family, n_chains=3, node_ids=[0, 1], n_nodes=2,
                  events=[torch.zeros(10), None])
    assert m.n_inputs == 3 and m.input_shapes == [(2,), (16,), ()]
    assert m.n_params == 2 + 16 + 1 and m.n_theta_words == 3 * 19
    assert m.n_vals == 2 * 3 * (2 + 2 + 16)
    assert m.flops_per_eval() == GlmShards(Xs, ts, n_chains=3).flops_per_eval() == 4 * 16 * 16 * 3
    assert m.bytes_per_eval() == GlmShards(Xs, ts).bytes_per_eval()   # the event rides in y's sign bit
    assert m.per_node(np.zeros(m.n_vals)).shape == (2, 3, 2 + 2 + 16)


@pytest.mark.parametrize("K,G", [(1, 1), (1, 2), (4, 2)])
def test_pack_unpack_and_words_round_trip(K, G):
    P = 8
    Xs, ts, es, _, _ = _case([20] * G, P, "weibull", seed=7, n_masked=0, weighted=False, offsets=False)
    model = GlmShards(Xs, ts, groups=list(range(G)), n_groups=G, family="weibull", n_chains=K, events=es)
    ic, beta, ls = _theta(G, P, K, log_sigma=np.arange(K) - 0.5 if K > 1 else -0.5, scale=1.0)
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
    words2 = np.zeros_like(words)
    model.pack_theta([ic2, b2, ls2], words2)
    assert np.array_equal(words, words2)
    raw = np.arange(model.n_vals, dtype=np.float64).reshape(K, 2 + G + P)
    logp, d_ic, d_b, d_ls = model.unpack_result(raw.reshape(-1), ctx)
    assert d_ic.shape == np.shape(ic) and d_b.shape == beta.shape and np.shape(d_ls) == np.shape(ls)
    np.testing.assert_array_equal(np.reshape(logp, -1), raw[:, 0])
    np.testing.assert_array_equal(np.reshape(d_ic, (K, G)), raw[:, 1 : 1 + G])
    np.testing.assert_array_equal(np.reshape(d_b, (K, P)), raw[:, 1 + G : 1 + G + P])
    np.testing.assert_array_equal(np.reshape(d_ls, K), raw[:, -1])


@pytest.mark.parametrize("family", FAMILIES)
def test_glm_batch_fn_splits_theta_with_log_sigma(family):
    from pytensor_federated_b200.sampling import glm_batch_fn

    P, G = 8, 2
    Xs, ts, es, ws, os_ = _case([60, 40], P, family, seed=8, sigma=0.5)
    model = _model(Xs, ts, es, ws, os_, family, groups=[0, 1], n_groups=G, n_chains=2)
    rng = np.random.default_rng(9)
    theta = np.concatenate([0.4 + rng.normal(size=(3, G)) * 0.05, rng.normal(size=(3, P)) * 0.01,
                            np.log(0.5) + rng.normal(size=(3, 1)) * 0.1], axis=1)
    with FederatedEngine(model, backend="collective") as eng:
        logp, grad = glm_batch_fn(eng, G)(theta)
    assert logp.shape == (3,) and grad.shape == theta.shape
    single = _model(Xs, ts, es, ws, os_, family, groups=[0, 1], n_groups=G)
    for i in range(3):
        want = _oracle(single, theta[i, :G], theta[i, G : G + P], theta[i, -1])
        np.testing.assert_allclose(logp[i], want[0], rtol=1e-5)
        np.testing.assert_allclose(grad[i], np.concatenate([want[1], want[2], [want[3]]]), rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("family", FAMILIES)
def test_synth_survival_shard(family):
    import scipy.stats

    n, sigma = 200_000, 0.7
    X, t, ev, beta = synth_survival_shard(n, 16, family=family, sigma=sigma, censor_fraction=0.3, seed=1, device="cpu",
                                          chunk_rows=65536)
    assert X.dtype == torch.bfloat16 and X.shape == (n, 16) and beta.shape == (16,)
    assert t.dtype == torch.float32 and ev.dtype == torch.float32
    assert bool(torch.all(torch.isfinite(t) & (t > 0))) and bool(torch.all((ev == 0) | (ev == 1)))
    assert abs(1.0 - float(ev.mean()) - 0.3) < 0.01
    X2, t2, ev2, _ = synth_survival_shard(n, 16, family=family, sigma=sigma, censor_fraction=0.3, seed=1, device="cpu",
                                          chunk_rows=65536)
    assert torch.equal(X, X2) and torch.equal(t, t2) and torch.equal(ev, ev2)
    # without censoring, at beta* = 0, every time is a draw of the family at scale e^intercept
    _, t0, ev0, _ = synth_survival_shard(50_000, 8, family=family, sigma=sigma, censor_fraction=0.0, seed=2,
                                         device="cpu", beta_scale=0.0, intercept=0.5)
    assert bool(torch.all(ev0 == 1))
    dist = (scipy.stats.weibull_min(c=1.0 / sigma, scale=np.exp(0.5)) if family == "weibull"
            else scipy.stats.lognorm(s=sigma, scale=np.exp(0.5)))
    assert scipy.stats.kstest(t0.double().numpy(), dist.cdf).pvalue > 1e-3
    # and the model the data came from fits it: dLL/ds at the true sigma is ~0 relative to its scale
    m = GlmShards([X], [t], family=family, events=[ev])
    got = _oracle(m, np.float32(0.5), beta.numpy(), np.float32(np.log(sigma)), chunk_rows=1 << 16)
    assert abs(got[3]) < 5 * np.sqrt(n)


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


def _check(got, want, n_rows, K, log_sigma):
    """The dispersion suite's tolerances: LL at rtol 2e-5, the intercept and beta gradients at rtol 1e-4 with
    absolute tolerances scaled per chain by max(1, 1 / sigma^2), d log_sigma at rtol 1e-4 / atol 2e-3 sqrt(n).

    The (hi, lo) bf16 split of R keeps ~2^-17 (7.6e-6) of each |r|, so a gradient component that nearly cancels is
    off by up to about that share of the chain's gradient scale.  Weibull residuals (e^z - delta) / sigma are not
    bounded by 1 / sigma^2 (at sigma = 0.05 a chain's beta gradients reach 3e7), so the absolute tolerances are also
    at least 2e-5 of the chain's largest |gradient|."""
    assert all(np.all(np.isfinite(g)) for g in got)
    for u, v in zip(got, want):
        assert np.shape(u) == np.shape(v)
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)
    lss = np.reshape(log_sigma, -1).astype(np.float64)
    scale = np.maximum(1.0, np.exp(-2.0 * lss))
    atol_b = 2e-3 * np.sqrt(n_rows) if K == 1 else 0.2
    for k in range(K):
        pick = (lambda a: a[k]) if K > 1 else (lambda a: a)
        floor = 2e-5 * max(np.max(np.abs(pick(want[1]))), np.max(np.abs(pick(want[2]))))
        np.testing.assert_allclose(pick(got[1]), pick(want[1]), rtol=1e-4, atol=max(2e-3 * scale[k], floor))
        np.testing.assert_allclose(pick(got[2]), pick(want[2]), rtol=1e-4, atol=max(atol_b * scale[k], floor))
    np.testing.assert_allclose(got[3], want[3], rtol=1e-4, atol=2e-3 * np.sqrt(n_rows))


@pytest.mark.parametrize("censor", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("row_data", [True, False])
@pytest.mark.parametrize("K", [1, 2, 4, 5, 8, 16])
@pytest.mark.parametrize("P", [256, 200, 8])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_matches_oracle(dev, family, P, K, row_data, censor):
    """K <= 1, 4, 8 and 16 select the kernel's four survival buckets; ``row_data`` (offsets and weights, masked rows
    with NaN / negative / zero times and invalid events) its ROWS variant.  The chains cycle through sigma 0.05, 0.5,
    1 and 3; with K = 1 each value is one evaluation."""
    rows = [128 * 37, 77, 4099, 1]
    Xs, ts, es, ws, os_ = _case(rows, P, family, seed=K + P, device=dev, weighted=row_data, offsets=row_data,
                                n_masked=5 if row_data else 0, censor=censor)
    model = _model(Xs, ts, es, ws, os_, family, groups=[0, 1, 0, 1], n_groups=2, n_chains=K, kernel="auto")
    assert model.has_row_data == row_data
    if K == 1:
        inputs = [_theta(2, P, 1, log_sigma=v, seed=5 + i) for i, v in enumerate(LOG_SIGMA)]
    else:
        inputs = [_theta(2, P, K, log_sigma=np.resize(LOG_SIGMA, K))]
    got = _run(model, inputs)
    assert model.selected_kernel == "tc"
    for g, inp in zip(got, inputs):
        _check(g, _oracle(model, *inp, chunk_rows=1 << 20), sum(rows), K, inp[2])


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("K,row_data", [(1, False), (2, True), (5, False), (5, True)])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_with_many_groups_matches_oracle(dev, family, K, row_data):
    G, P = 300, 256
    rows = [128 * 9 + 5, 999, 64, 1, 3000]
    groups = [0, 299, 150, 7, 299]
    Xs, ts, es, ws, os_ = _case(rows, P, family, seed=40 + K, device=dev, weighted=row_data, offsets=row_data,
                                n_masked=5 if row_data else 0)
    model = _model(Xs, ts, es, ws, os_, family, groups=groups, n_groups=G, n_chains=K, kernel="tc")
    inp = _theta(G, P, K, log_sigma=np.resize(LOG_SIGMA[::-1], K) if K > 1 else LOG_SIGMA[0])
    (got,) = _run(model, [inp])
    _check(got, _oracle(model, *inp, chunk_rows=1 << 20), sum(rows), K, inp[2])
    unused = np.ones(G, dtype=bool)
    unused[groups] = False
    assert np.all(got[1][..., unused] == 0.0)


@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("row_data", [False, True])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_weibull_at_unit_sigma_is_poisson_on_the_events(dev, row_data, K):
    wb, po, shift = _weibull_poisson_pair([128 * 30 + 9, 5000, 77], 256, seed=11, device=dev, weighted=row_data,
                                          n_chains=K, kernel="tc")
    ic, beta, ls = _theta(2, 256, K, log_sigma=0.0)
    (a,), (b,) = _run(wb, [(ic, beta, ls)]), _run(po, [(-ic, -beta)])
    np.testing.assert_allclose(a[0], b[0] - shift, rtol=2e-5)
    np.testing.assert_allclose(a[1], -b[1], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(a[2], -b[2], rtol=1e-4, atol=0.2)


@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("row_data", [False, True])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_lognormal_without_censoring_is_gaussian_scale_on_log_times(dev, row_data, K):
    ln, gs, shift = _lognormal_gaussian_pair([128 * 30 + 9, 5000, 77], 256, seed=12, device=dev, weighted=row_data,
                                             n_chains=K, kernel="tc")
    ic, beta, ls = _theta(2, 256, K, log_sigma=-1.0)
    (a,), (b,) = _run(ln, [(ic, beta, ls)]), _run(gs, [(ic, beta, ls)])
    n = 128 * 30 + 9 + 5000 + 77
    np.testing.assert_allclose(a[0], b[0] - shift, rtol=2e-5)
    np.testing.assert_allclose(a[1], b[1], rtol=1e-4, atol=2e-3 * np.exp(2.0))
    np.testing.assert_allclose(a[2], b[2], rtol=1e-4, atol=0.2 * np.exp(2.0))
    np.testing.assert_allclose(a[3], b[3], rtol=1e-4, atol=2e-3 * np.sqrt(n))


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_survival_evaluations_are_bit_reproducible(dev, family):
    rows = [40_000, 25_000, 33_333, 128, 19_999]
    Xs, ts, es, ws, os_ = _case(rows, 256, family, seed=12, device=dev)
    model = _model(Xs, ts, es, ws, os_, family, groups=[0, 1, 2, 1, 0], n_groups=3, n_chains=4, kernel="tc")
    inp = _theta(3, 256, 4, log_sigma=LOG_SIGMA)
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
    Xs, ts, es, ws, os_ = _case(rows, 256, family, seed=13, device=dev)
    model = _model(Xs, ts, es, ws, os_, family, groups=groups, n_groups=2, kernel="tc", node_ids=node_ids, n_nodes=2)
    ic, beta, ls = _theta(2, 256, log_sigma=np.log(0.3))
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
        single = _model([Xs[i] for i in segs], [ts[i] for i in segs], [es[i] for i in segs], [ws[i] for i in segs],
                        [os_[i] for i in segs], family, groups=[groups[i] for i in segs], n_groups=2, kernel="tc")
        (want,) = _run(single, [(ic, beta, ls)])
        np.testing.assert_allclose(blocks[node, 0, 0], want[0], rtol=2e-5)
        np.testing.assert_allclose(blocks[node, 0, 1:3], want[1], rtol=1e-4, atol=2e-2)
        np.testing.assert_allclose(blocks[node, 0, 3:-1], want[2], rtol=1e-4, atol=5.0)
        np.testing.assert_allclose(blocks[node, 0, -1], want[3], rtol=1e-4, atol=2e-3)
        np.testing.assert_allclose(res[node][0], blocks[node, 0, 0], rtol=1e-12)
        assert len(res[node][1]) == 3 and res[node][1][0].shape == (2,) and res[node][1][1].shape == (256,)
        assert np.shape(res[node][1][2]) == ()
        np.testing.assert_allclose(res[node][1][2], want[3], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(total[0], blocks[:, 0, 0].sum(), rtol=1e-12)
    np.testing.assert_allclose(total[1][2], blocks[:, 0, -1].sum(), rtol=1e-12)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_lock_step_hmc_on_a_weibull_engine(dev):
    from pytensor_federated_b200.sampling import glm_batch_fn, hmc_sample_batched

    K, P = 4, 16
    X, t, ev, _ = synth_survival_shard(20_000, P, family="weibull", sigma=0.8, censor_fraction=0.3, seed=3, device=dev)
    model = GlmShards([X], [t], family="weibull", events=[ev], n_chains=K, kernel="tc")
    x0 = np.zeros((K, 1 + P + 1))
    x0[:, 0] = 0.5
    x0[:, -1] = np.log(0.8)
    with FederatedEngine(model) as eng:
        res = hmc_sample_batched(glm_batch_fn(eng, 1), x0, draws=5, tune=5, n_leapfrog=4, step_size=1e-3, seed=1)
        assert eng.n_evals == res.n_batched_evals
    assert res.samples.shape[-1] == 1 + P + 1 and np.all(np.isfinite(res.samples))


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_runtime_rejects_the_survival_families_outside_the_tc_kernel(dev):
    """The C ABI refuses what the Python layer never sends: families 7 and 8 on a CUDA-core kernel (which would take
    an unknown family for the Gaussian one), n_classes != 1, and an output size without the log-sigma gradient."""
    from pytensor_federated_b200.ops import native

    Xs, ts, _, _, _ = _case([256], 16, "weibull", seed=14, device=dev, n_masked=0, weighted=False, offsets=False)
    model = GlmShards(Xs, ts, family="poisson", kernel="simt")
    with FederatedEngine(model) as eng:
        lib, h = eng._lib, eng._handle
        Xp, yp = native.void_p_array([Xs[0].data_ptr()]), native.void_p_array([ts[0].data_ptr()])
        rows, grp = (C.c_longlong * 1)(256), (C.c_int * 1)(0)

        def set_glm(n_chains, family, code, n_classes=1):
            return int(lib.b200_engine_set_glm(h, 1, Xp, yp, None, rows, grp, 16, 16, 1, n_chains, family, code, None, 1,
                                               None, None, n_classes))

        for family, name in ((7, "weibull"), (8, "lognormal")):
            for code in (0, 2, 3, 4):
                assert set_glm(1, family, code) != 0
                assert f"the {name} family runs on the bf16 tensor-core kernel only" in native.last_error()
            assert set_glm(1, family, 1, 2) != 0 and "n_classes must be 1" in native.last_error()
            # this engine's n_vals is 1 + G + P: one value short of the survival families' block
            assert set_glm(1, family, 1) != 0 and "2 + n_groups + n_features" in native.last_error()
        # the engine still evaluates its own model
        ic, beta = np.float32(0.1), np.zeros(16, np.float32)
        got = eng.evaluate(ic, beta)
    want = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)


def _build_weibull_model(rank, world, dev):
    Xs, ts, es, ws, os_ = _case([30_000 + 17 * rank, 999, 77], 256, "weibull", seed=50 + rank, device=dev)
    return _model(Xs, ts, es, ws, os_, "weibull", groups=[rank % 2, 1 - rank % 2, 0], n_groups=2, n_chains=2,
                  kernel="tc")


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.timeout(900)
def test_two_rank_weibull_federation_matches_oracle():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from pytensor_federated_b200.federation import launch_federation

    inp = _theta(2, 256, 2, log_sigma=[np.log(0.1), 0.0])
    dev = torch.device("cuda:0")
    models = [_build_weibull_model(r, 2, dev) for r in range(2)]
    want = models[0].unpack_result(sum(m.reference_partial(list(inp), dtype=torch.float64) for m in models),
                                   models[0].call_context(list(inp)))
    del models
    with launch_federation(_build_weibull_model, 2, timeout=30.0) as eng:
        got = eng.evaluate(*inp)
    _check(got, want, 2 * (31_000 + 77), 2, inp[2])
