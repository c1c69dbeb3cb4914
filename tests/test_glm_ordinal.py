"""Ordinal (cumulative-logit) regression: ``GlmShards(..., family="ordinal", n_classes=C)``.

CPU tests check the fp64 oracle and the collective backend against independent formulas (autograd of the textbook
``log(sigmoid(c_y - eta) - sigmoid(c_{y-1} - eta))``, scipy's logistic CDF, finite differences, the logistic family)
and the model's packing; GPU tests check the tensor-core kernel against that oracle."""
import ctypes as C

import numpy as np
import pytest
import torch

from pytensor_federated_b200.models import Fp8GlmShards, GlmShards, synth_ordinal_shard
from pytensor_federated_b200.parallel import FederatedEngine
from pytensor_federated_b200.parallel.engine import default_inputs_from_words


# ----------------------------------------------------------------------------------------------- fixtures
def _case(rows, P, n_classes, *, seed=0, device="cpu", n_masked=5, weighted=True, offsets=True):
    """Ragged bf16 segments with labels drawn from a cumulative-logit model.  With ``weighted``, every segment but
    the last has weights; the first ``n_masked`` rows of segment 0 have weight 0 and carry a NaN, a negative, a too
    large and a fractional label.  With ``offsets``, every segment but the first has offsets."""
    rng = np.random.default_rng(seed)
    cuts = np.linspace(-1.5, 1.5, n_classes - 1)
    Xs, ys, ws, os_ = [], [], [], []
    for si, n in enumerate(rows):
        X = torch.tensor(rng.normal(size=(n, P)), dtype=torch.float32).to(torch.bfloat16)
        o = rng.normal(size=n) * 0.3
        eta = X.double().numpy() @ (rng.normal(size=P) * 0.1) + (o if offsets and si > 0 else 0.0)
        cdf = 1.0 / (1.0 + np.exp(-(cuts[None, :] - eta[:, None])))
        y = (rng.uniform(size=(n, 1)) > cdf).sum(1).astype(np.float64)
        w = rng.uniform(0.2, 2.0, size=n)
        if si == 0 and n_masked:
            w[:n_masked] = 0.0
            y[:4] = [np.nan, -1.0, n_classes, 0.5][: min(4, n_masked)]
        Xs.append(X.to(device))
        ys.append(torch.tensor(y, dtype=torch.float32, device=device))
        ws.append(torch.tensor(w, dtype=torch.float32, device=device) if weighted and si < len(rows) - 1 else None)
        os_.append(torch.tensor(o, dtype=torch.float32, device=device) if offsets and si > 0 else None)
    return Xs, ys, ws, os_


def _theta(G, P, n_classes, K=1, seed=3, scale=0.03, gaps=(0.05, 4.0)):
    """``(intercept, beta, cutpoints)``; each chain's cutpoint gaps are drawn log-uniformly from ``gaps`` and chain 0
    always has the smallest one."""
    rng = np.random.default_rng(seed)
    lead = (K,) if K > 1 else ()
    ic = (rng.normal(size=lead + (G,)) * 0.2).astype(np.float32)
    beta = (rng.normal(size=lead + (P,)) * scale).astype(np.float32)
    cps = []
    for k in range(K):
        g = np.exp(rng.uniform(np.log(gaps[0]), np.log(gaps[1]), size=n_classes - 2))
        if k == 0 and n_classes > 2:
            g[rng.integers(n_classes - 2)] = gaps[0]
        cps.append(np.concatenate([[rng.normal() * 0.3 - 0.5 * g.sum()], g]).cumsum())
    cp = np.array(cps, dtype=np.float32).reshape(lead + (n_classes - 1,))
    return ic, beta, cp


def _min_gap(cp):
    cp = np.asarray(cp, dtype=np.float64)
    return float(np.diff(cp, axis=-1).min()) if cp.shape[-1] > 1 else np.inf


def _explicit_fp64(Xs, ys, ws, os_, groups, ic, beta, cp):
    """``[LL, dLL/dintercept, dLL/dbeta, dLL/dcutpoints]`` per chain by autograd of the textbook formula."""
    ic, beta, cp = (np.asarray(v, dtype=np.float64) for v in (ic, beta, cp))
    batched = beta.ndim == 2
    if not batched:
        ic, beta, cp = ic.reshape((1, -1)), beta[None], cp[None]
    K = beta.shape[0]
    t_ic, t_b, t_c = (torch.tensor(v, requires_grad=True) for v in (ic.reshape(K, -1), beta, cp))
    total = torch.zeros(K, dtype=torch.float64)
    for X, y, w, o, g in zip(Xs, ys, ws, os_, groups):
        X, y = X.double().cpu(), y.double().cpu()
        keep = torch.ones_like(y, dtype=torch.bool) if w is None else w.cpu() != 0
        lab = torch.where(keep, y, torch.zeros_like(y)).long()
        eta = X @ t_b.T + t_ic[:, g]                                       # [n, K]
        if o is not None:
            eta = eta + o.double().cpu().unsqueeze(1)
        pad = torch.cat([torch.full((K, 1), -torch.inf, dtype=torch.float64), t_c,
                         torch.full((K, 1), torch.inf, dtype=torch.float64)], 1)
        p = torch.sigmoid(pad[:, lab + 1].T - eta) - torch.sigmoid(pad[:, lab].T - eta)
        ll = torch.log(p)
        if w is not None:
            ll = torch.where(keep.unsqueeze(1), w.double().cpu().unsqueeze(1) * ll, torch.zeros_like(ll))
        total = total + ll.sum(0)
    total.sum().backward()
    out = [total.detach().numpy(), t_ic.grad.numpy().reshape(ic.shape), t_b.grad.numpy(), t_c.grad.numpy()]
    return out if batched else [out[0][0], out[1][0], out[2][0], out[3][0]]


def _oracle(model, ic, beta, cp):
    return model.unpack_result(model.reference_partial([ic, beta, cp], dtype=torch.float64, chunk_rows=128),
                               model.call_context([ic, beta, cp]))


def _collective(model, ic, beta, cp):
    with FederatedEngine(model, backend="collective") as eng:
        return [np.asarray(v, dtype=np.float64) for v in eng.evaluate(ic, beta, cp)]


# ----------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("K", [1, 3])
def test_oracle_matches_autograd_of_the_textbook_formula(K):
    rows, P, Cn, groups = [150, 70, 201], 16, 5, [0, 1, 0]
    Xs, ys, ws, os_ = _case(rows, P, Cn, seed=1)
    model = GlmShards(Xs, ys, groups=groups, n_groups=2, family="ordinal", n_classes=Cn, n_chains=K, weights=ws,
                      offsets=os_)
    ic, beta, cp = _theta(2, P, Cn, K, gaps=(0.3, 1.5))
    got = _oracle(model, ic, beta, cp)
    want = _explicit_fp64(Xs, ys, ws, os_, groups, ic, beta, cp)
    assert np.all(np.isfinite(got[0]))
    assert got[1].shape == ic.shape and got[2].shape == beta.shape and got[3].shape == cp.shape
    np.testing.assert_allclose(got[0], want[0], rtol=1e-12)
    for u, v in zip(got[1:], want[1:]):
        np.testing.assert_allclose(u, v, rtol=1e-10, atol=1e-10)


def test_oracle_matches_scipy_logistic_cdf_and_finite_differences():
    from scipy.stats import logistic

    rows, P, Cn = [90, 60], 8, 4
    Xs, ys, ws, os_ = _case(rows, P, Cn, seed=2, n_masked=0)
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family="ordinal", n_classes=Cn, weights=ws, offsets=os_)
    Xn = [X.double().numpy() for X in Xs]
    yn = [y.numpy().astype(int) for y in ys]
    wn = [w.double().numpy() if w is not None else np.ones(len(y)) for w, y in zip(ws, ys)]
    on = [o.double().numpy() if o is not None else np.zeros(len(y)) for o, y in zip(os_, ys)]

    def truth(ic, beta, cp):
        total = 0.0
        pad = np.concatenate([[-np.inf], cp, [np.inf]])
        for g, (X, y, w, o) in enumerate(zip(Xn, yn, wn, on)):
            eta = X @ beta + ic[g] + o
            total += np.sum(w * np.log(logistic.cdf(pad[y + 1] - eta) - logistic.cdf(pad[y] - eta)))
        return total

    ic, beta, cp = [v.astype(np.float64) for v in _theta(2, P, Cn, gaps=(0.5, 2.0))]
    got = _oracle(model, ic, beta, cp)
    np.testing.assert_allclose(got[0], truth(ic, beta, cp), rtol=1e-12)
    eps = 1e-6
    for arr, grad in ((ic, got[1]), (beta, got[2]), (cp, got[3])):
        fd = np.zeros_like(arr)
        for idx in np.ndindex(arr.shape):
            orig = arr[idx]
            arr[idx] = orig + eps
            hi = truth(ic, beta, cp)
            arr[idx] = orig - eps
            lo = truth(ic, beta, cp)
            arr[idx] = orig
            fd[idx] = (hi - lo) / (2 * eps)
        np.testing.assert_allclose(grad, fd, rtol=1e-6, atol=1e-6)


def test_two_categories_are_the_logistic_model_at_intercept_minus_cutpoint():
    rows, P = [130, 77], 16
    Xs, ys, ws, os_ = _case(rows, P, 2, seed=3)
    ordinal = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family="ordinal", n_classes=2, weights=ws, offsets=os_)
    ys_logit = [torch.nan_to_num(y).clamp(0, 1) for y in ys]   # masked rows: any finite response
    logit = GlmShards(Xs, ys_logit, groups=[0, 1], n_groups=2, weights=ws, offsets=os_)
    ic, b, cp = _theta(2, P, 2)
    o = _oracle(ordinal, ic, b, cp)
    lg = logit.unpack_result(logit.reference_partial([ic.astype(np.float64) - cp.astype(np.float64), b],
                                                     dtype=torch.float64))
    np.testing.assert_allclose(o[0], lg[0], rtol=1e-12)
    np.testing.assert_allclose(o[1], lg[1], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(o[2], lg[2], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(o[3], [-lg[1].sum()], rtol=1e-10, atol=1e-12)


def test_tails_stay_finite_and_accurate():
    """|c - eta| of about 30 on both sides and a narrow middle category: the stable formulas keep the log
    probabilities (down to ~-30) and the residuals (~1e-13) to relative accuracy, where sigmoid(a) - sigmoid(b) would
    round to 0 or 1."""
    import mpmath

    n, P = 6, 8
    X = torch.zeros(n, P, dtype=torch.bfloat16)
    y = torch.tensor([0.0, 0.0, 1.0, 1.0, 2.0, 2.0])
    off = torch.tensor([30.0, -30.0, 30.0, -31.0, 30.0, -30.0])
    model = GlmShards([X], [y], family="ordinal", n_classes=3, offsets=[off])
    cp = np.array([0.0, 0.5])
    got = _oracle(model, np.float64(0.0), np.zeros(P), cp)
    assert all(np.all(np.isfinite(g)) for g in got)
    eta = off.double().numpy()
    pad = np.concatenate([[-np.inf], cp, [np.inf]])
    a, b = pad[y.long().numpy() + 1] - eta, pad[y.long().numpy()] - eta
    # the difference of the two CDF values in 50-digit arithmetic
    mpmath.mp.dps = 50
    cdf = lambda v: mpmath.mpf(0) if v == -np.inf else (mpmath.mpf(1) if v == np.inf else 1 / (1 + mpmath.exp(-mpmath.mpf(v))))
    ll = np.array([float(mpmath.log(cdf(ai) - cdf(bi))) for ai, bi in zip(a, b)])
    assert ll.min() < -30
    np.testing.assert_allclose(got[0], ll.sum(), rtol=1e-13)
    # d LL / d eta = sigmoid(a) + sigmoid(b) - 1 per row (a = c_y - eta, b = c_{y-1} - eta), compared row by row
    ic_model = GlmShards([X[i : i + 1] for i in range(n)], [y[i : i + 1] for i in range(n)], groups=list(range(n)),
                         n_groups=n, family="ordinal", n_classes=3, offsets=[off[i : i + 1] for i in range(n)])
    per_row = _oracle(ic_model, np.zeros(n), np.zeros(P), cp)
    from scipy.special import expit

    want = expit(a) + expit(b) - 1.0
    tiny = [0, 5]   # eta = 30 with y = 0, eta = -30 with y = 2: residual ~ -e^-30 and e^-29.5
    np.testing.assert_allclose(per_row[1][tiny], [-expit(-a[0]), expit(b[5])], rtol=1e-12)
    np.testing.assert_allclose(per_row[1], want, rtol=1e-9, atol=1e-15)


@pytest.mark.parametrize("K", [1, 4])
def test_collective_backend_equals_the_oracle(K):
    rows, P, Cn = [300, 45, 129], 24, 4
    Xs, ys, ws, os_ = _case(rows, P, Cn, seed=6)
    model = GlmShards(Xs, ys, groups=[0, 1, 1], n_groups=2, family="ordinal", n_classes=Cn, n_chains=K,
                      weights=ws, offsets=os_)
    ic, beta, cp = _theta(2, P, Cn, K, gaps=(0.2, 2.0))
    got, want = _collective(model, ic, beta, cp), _oracle(model, ic, beta, cp)
    for u, v in zip(got, want):
        assert u.shape == v.shape and np.all(np.isfinite(u))
        np.testing.assert_allclose(u, v, rtol=1e-5, atol=1e-4)


def test_ordinal_validation():
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ys = [torch.zeros(10), torch.full((6,), 2.0)]
    ok = dict(family="ordinal", n_classes=3)
    GlmShards(Xs, ys, **ok)
    GlmShards(Xs, ys, family="ordinal", n_classes=17)
    for n_classes in (None, 1, 18):
        with pytest.raises(ValueError, match="n_classes"):
            GlmShards(Xs, ys, family="ordinal", n_classes=n_classes)
    with pytest.raises(ValueError, match=r"n_chains x \(n_classes - 1\)"):
        GlmShards(Xs, ys, family="ordinal", n_classes=5, n_chains=5)
    GlmShards(Xs, ys, family="ordinal", n_classes=5, n_chains=4)
    for kernel in ("simt", "generic", "fp8"):
        with pytest.raises(ValueError, match="tensor-core kernel only"):
            GlmShards(Xs, ys, kernel=kernel, **ok)
    with pytest.raises(ValueError, match="tensor-core kernel only"):
        Fp8GlmShards.from_dense([torch.randn(10, 32), torch.randn(6, 32)], ys, family="ordinal")
    with pytest.raises(ValueError, match="'ordinal'"):
        GlmShards(Xs, ys, n_classes=3)
    GlmShards(Xs, ys, offsets=[torch.zeros(10), None], **ok)   # offsets shift eta: accepted
    for bad in (3.0, -1.0, 0.5, float("nan")):
        y0 = torch.zeros(10)
        y0[4] = bad
        with pytest.raises(ValueError, match="labels of segment 0"):
            GlmShards(Xs, [y0, ys[1]], **ok)
        w0 = torch.ones(10)
        w0[4] = 0.0
        GlmShards(Xs, [y0, ys[1]], weights=[w0, None], **ok)   # a masked row may carry anything
    for X in (torch.randn(10, 12).to(torch.bfloat16), torch.randn(10, 392).to(torch.bfloat16), torch.randn(10, 16)):
        with pytest.raises(ValueError, match="tensor-core kernel only"):
            GlmShards([X], [torch.zeros(10)], **ok).use_tensor_cores()
    assert GlmShards(Xs, ys, kernel="tc", **ok).use_tensor_cores() == 1


def test_sizes_and_flops():
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ys = [torch.zeros(10), torch.zeros(6)]
    m = GlmShards(Xs, ys, n_groups=2, groups=[0, 1], family="ordinal", n_classes=4, n_chains=2,
                  node_ids=[0, 1], n_nodes=2)
    assert m.n_inputs == 3 and m.kernel_chains == 6
    assert m.n_params == 2 + 16 + 3 and m.n_theta_words == 2 * 3 * 18
    assert m.n_vals == 2 * 2 * 3 * (1 + 2 + 16)
    assert m.flops_per_eval() == 4 * 16 * 16 * 2 * 3
    assert m.bytes_per_eval() == GlmShards(Xs, ys).bytes_per_eval()
    assert m.per_node(np.zeros(m.n_vals)).shape == (2, 2, 1 + 2 + 16 + 3)


@pytest.mark.parametrize("K,G", [(1, 1), (1, 2), (4, 2)])
def test_pack_unpack_and_words_round_trip(K, G):
    P, Cn = 8, 4
    Xs, ys, _, _ = _case([20] * G, P, Cn, seed=7, n_masked=0, weighted=False, offsets=False)
    model = GlmShards(Xs, ys, groups=list(range(G)), n_groups=G, family="ordinal", n_classes=Cn, n_chains=K)
    rng = np.random.default_rng(8)
    lead = (K,) if K > 1 else ()
    # multiples of 2^-8 of moderate size: intercept - c_j is exact in float32, so the words are a faithful image
    ic = (rng.integers(-256, 256, size=lead + (G,)) / 256.0).astype(np.float32)
    cp = np.cumsum(rng.integers(1, 256, size=lead + (Cn - 1,)) / 256.0, axis=-1).astype(np.float32)
    beta = rng.normal(size=lead + (P,)).astype(np.float32)
    if K == 1 and G == 1:
        ic = ic.reshape(())   # a scalar is accepted for one group
    words = np.zeros(model.n_theta_words, dtype=np.uint32)
    ctx = model.pack_theta([ic, beta, cp], words)
    assert ctx == model.call_context([ic, beta, cp]) == (K > 1, ic.shape, cp.shape, ())
    # the kernel's layout: row k (C - 1) + j = (intercept - c_j, beta) of chain k
    th = words.view(np.float32).reshape(K * (Cn - 1), G + P)
    ic_k, b_k, c_k = ic.reshape(K, G), beta.reshape(K, P), cp.reshape(K, Cn - 1)
    for k in range(K):
        for j in range(Cn - 1):
            assert np.array_equal(th[k * (Cn - 1) + j, :G], ic_k[k] - c_k[k, j])
            assert np.array_equal(th[k * (Cn - 1) + j, G:], b_k[k])
    # the words carry only intercept - c_j: they decode to the same model shifted to c_0 = 0
    ic2, b2, c2 = default_inputs_from_words(model, words)
    np.testing.assert_array_equal(np.reshape(ic2, (K, G)), ic_k - c_k[:, :1])
    np.testing.assert_array_equal(np.reshape(c2, (K, Cn - 1)), c_k - c_k[:, :1])
    assert np.array_equal(b2, beta)
    words2 = np.zeros_like(words)
    model.pack_theta([ic2, b2, c2], words2)
    assert np.array_equal(words, words2)
    # unpack: block k (C - 1) + j holds [LL_j, gi_j[G], g_j[P]] of chain k
    raw = np.arange(model.n_vals, dtype=np.float64).reshape(K, Cn - 1, 1 + G + P)
    logp, d_ic, d_b, d_c = model.unpack_result(raw.reshape(-1), ctx)
    assert d_ic.shape == ic.shape and d_b.shape == beta.shape and d_c.shape == cp.shape
    np.testing.assert_array_equal(np.reshape(logp, -1), raw[:, :, 0].sum(1))
    np.testing.assert_array_equal(d_ic.reshape(K, G), raw[:, :, 1 : 1 + G].sum(1))
    np.testing.assert_array_equal(d_b.reshape(K, P), raw[:, :, 1 + G :].sum(1))
    np.testing.assert_array_equal(d_c.reshape(K, Cn - 1), -raw[:, :, 1 : 1 + G].sum(2))
    per = model.per_node(raw.reshape(-1), ctx)
    assert per.shape == (1, K, 1 + G + P + Cn - 1)
    np.testing.assert_array_equal(per[0, :, 1 + G + P :], d_c.reshape(K, Cn - 1))


def test_unordered_cutpoints_give_minus_inf_and_zero_gradients_for_that_chain_only():
    rows, P, Cn, K = [100, 60], 8, 4, 3
    Xs, ys, ws, os_ = _case(rows, P, Cn, seed=9)
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family="ordinal", n_classes=Cn, n_chains=K, weights=ws,
                      offsets=os_)
    ic, beta, cp = _theta(2, P, Cn, K, gaps=(0.3, 1.0))
    good = _oracle(model, ic, beta, cp)
    for bad_cp in ([0.5, 0.5, 1.0], [0.5, 0.2, 1.0], [0.0, np.nan, 1.0]):
        cp2 = cp.copy()
        cp2[1] = bad_cp
        ctx = model.call_context([ic, beta, cp2])
        assert ctx[3] == (1,)
        for got in (_oracle(model, ic, beta, cp2), _collective(model, ic, beta, cp2)):
            assert got[0][1] == -np.inf
            for g in got[1:]:
                assert np.all(g[1] == 0.0)
            for i, g in enumerate(got):
                np.testing.assert_allclose(g[[0, 2]], good[i][[0, 2]], rtol=1e-5, atol=1e-4)
    # the check is on the float32 table: cutpoints that only differ below the rounding of intercept - c are ties
    cp3 = cp.copy()
    cp3[2] = [1.0, 1.0 + 1e-9, 2.0]
    assert model.call_context([ic, beta, cp3])[3] == (2,)


def test_glm_batch_fn_splits_theta_for_the_ordinal_model():
    from pytensor_federated_b200.sampling import glm_batch_fn

    P, Cn, G = 8, 4, 2
    Xs, ys, ws, os_ = _case([60, 40], P, Cn, seed=8)
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=G, family="ordinal", n_classes=Cn, n_chains=2, weights=ws,
                      offsets=os_)
    rng = np.random.default_rng(9)
    theta = np.concatenate([rng.normal(size=(3, G + P)) * 0.1, np.cumsum(rng.uniform(0.3, 1, size=(3, Cn - 1)), 1) - 1],
                           axis=1)
    with FederatedEngine(model, backend="collective") as eng:
        logp, grad = glm_batch_fn(eng, G)(theta)
    assert logp.shape == (3,) and grad.shape == theta.shape
    single = GlmShards(Xs, ys, groups=[0, 1], n_groups=G, family="ordinal", n_classes=Cn, weights=ws, offsets=os_)
    for i in range(3):
        want = _oracle(single, theta[i, :G], theta[i, G : G + P], theta[i, G + P :])
        np.testing.assert_allclose(logp[i], want[0], rtol=1e-5)
        np.testing.assert_allclose(grad[i], np.concatenate([want[1], want[2], want[3]]), rtol=1e-4, atol=1e-4)


def test_synth_ordinal_shard_label_frequencies_match_the_model():
    n, P, Cn = 200_000, 8, 5
    X, y, beta, cuts = synth_ordinal_shard(n, P, Cn, seed=1, device="cpu", chunk_rows=1 << 16, beta_scale=0.3)
    assert X.dtype == torch.bfloat16 and X.shape == (n, P) and beta.shape == (P,) and cuts.shape == (Cn - 1,)
    assert y.dtype == torch.float32 and set(np.unique(y.numpy())) <= set(range(Cn))
    eta = X.double().numpy() @ beta.double().numpy()
    cdf = 1.0 / (1.0 + np.exp(-(np.concatenate([cuts, [np.inf]])[None, :] - eta[:, None])))
    p = np.diff(np.concatenate([np.zeros((n, 1)), cdf], 1), axis=1).mean(0)     # expected category frequencies
    freq = np.bincount(y.numpy().astype(int), minlength=Cn) / n
    np.testing.assert_allclose(freq, p, atol=4 * np.sqrt(p * (1 - p) / n).max())
    X2, y2, _, _ = synth_ordinal_shard(n, P, Cn, seed=1, device="cpu", chunk_rows=1 << 16, beta_scale=0.3)
    assert torch.equal(X, X2) and torch.equal(y, y2)


# ----------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from pytensor_federated_b200.ops import native

    native.load()  # a GPU box without the native library is a failure, not a skip
    return torch.device("cuda:0")


def _run(model, *inputs, repeats=1):
    with FederatedEngine(model) as eng:
        out = [[np.asarray(v).copy() for v in eng.evaluate(*inputs)] for _ in range(repeats)]
    return out[0] if repeats == 1 else out


def _check(got, want, rtol_ll, rtol_g, atol_ic, atol_b, atol_c):
    assert all(np.all(np.isfinite(g)) for g in got)
    for u, v in zip(got, want):
        assert np.shape(u) == np.shape(v)
    np.testing.assert_allclose(got[0], want[0], rtol=rtol_ll)
    np.testing.assert_allclose(got[1], want[1], rtol=rtol_g, atol=atol_ic)
    np.testing.assert_allclose(got[2], want[2], rtol=rtol_g, atol=atol_b)
    np.testing.assert_allclose(got[3], want[3], rtol=rtol_g, atol=atol_c)


def _tolerances(rows, K, cp):
    """The multinomial suite's tolerances, with the absolute ones scaled by max(1, 1 / smallest gap): a row in a
    middle category has residuals of size 1 / gap (r_up, r_lo ~ -/+ 1 / expm1(gap)), and the (hi, lo) bf16 split of
    the residuals keeps a fixed fraction (~2^-17) of |r|, so the kernel's absolute error grows like 1 / gap while its
    relative error does not."""
    s = max(1.0, 1.0 / _min_gap(cp))
    atol_b = 2e-3 * np.sqrt(sum(rows)) if K == 1 else 0.2
    return 2e-5, 1e-4, 2e-3 * s, atol_b * s, 2e-3 * s


@pytest.mark.parametrize("weighted", [True, False])
@pytest.mark.parametrize("K,Cn", [(1, 2), (1, 3), (1, 5), (1, 9), (1, 17), (2, 5), (4, 3), (5, 4), (8, 3)])
@pytest.mark.parametrize("P", [256, 200, 8])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_ordinal_matches_oracle(dev, K, Cn, P, weighted):
    """K (C - 1) = 1, <= 4, <= 8 and <= 16 select the kernel's four ORD buckets; ``weighted`` (weights and offsets)
    its ROWS variant.  Cutpoint gaps range from 0.05 to 4."""
    rows = [128 * 37, 77, 4099, 1]
    Xs, ys, ws, os_ = _case(rows, P, Cn, seed=Cn + K + P, device=dev, weighted=weighted,
                            n_masked=5 if weighted else 0, offsets=weighted)
    model = GlmShards(Xs, ys, groups=[0, 1, 0, 1], n_groups=2, family="ordinal", n_classes=Cn, n_chains=K,
                      kernel="auto", weights=ws, offsets=os_)
    assert model.has_row_data == weighted
    ic, beta, cp = _theta(2, P, Cn, K)
    got = _run(model, ic, beta, cp)
    assert model.selected_kernel == "tc"
    _check(got, _oracle(model, ic, beta, cp), *_tolerances(rows, K, cp))


@pytest.mark.parametrize("Cn,K,weighted", [(2, 1, False), (3, 1, True), (5, 2, False), (4, 4, True)])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_ordinal_with_many_groups_matches_oracle(dev, Cn, K, weighted):
    """A hierarchical model with 300 intercepts: the intercept table is K (C - 1) x G floats, the gap of a row is
    read from two of its rows, and the lanes' columns past K (C - 1) must not index past it."""
    G, P = 300, 256
    rows = [128 * 9 + 5, 999, 64, 1, 3000]
    groups = [0, 299, 150, 7, 299]
    Xs, ys, ws, os_ = _case(rows, P, Cn, seed=40 + Cn + K, device=dev, weighted=weighted,
                            n_masked=5 if weighted else 0, offsets=weighted)
    model = GlmShards(Xs, ys, groups=groups, n_groups=G, family="ordinal", n_classes=Cn, n_chains=K,
                      kernel="tc", weights=ws, offsets=os_)
    ic, beta, cp = _theta(G, P, Cn, K)
    got = _run(model, ic, beta, cp)
    want = _oracle(model, ic, beta, cp)
    _check(got, want, *_tolerances(rows, K, cp))
    unused = np.ones(G, dtype=bool)
    unused[groups] = False
    assert np.all(got[1][..., unused] == 0.0)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_ordinal_tails(dev):
    """Offsets put |c - eta| near 30 on both sides of the cutpoints: the kernel's LL and gradients stay finite and
    match the oracle."""
    n, P, Cn = 128 * 20, 256, 4
    Xs, ys, ws, _ = _case([n], P, Cn, seed=60, device=dev, n_masked=0, weighted=False, offsets=False)
    rng = np.random.default_rng(61)
    off = torch.tensor(rng.choice([-30.0, 30.0], size=n) + rng.normal(size=n), dtype=torch.float32, device=dev)
    model = GlmShards(Xs, ys, family="ordinal", n_classes=Cn, kernel="tc", offsets=[off])
    ic, beta, cp = np.float32(0.0), np.zeros(P, np.float32), np.array([-0.5, 0.0, 0.25], np.float32)
    got = _run(model, ic, beta, cp)
    _check(got, _oracle(model, ic, beta, cp), *_tolerances([n], 1, cp))


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_two_categories_are_the_logistic_kernel(dev):
    rows, P = [128 * 30 + 9, 5000, 77], 256
    Xs, ys, ws, os_ = _case(rows, P, 2, seed=11, device=dev)
    ys_logit = [torch.nan_to_num(y).clamp(0, 1) for y in ys]
    ordinal = GlmShards(Xs, ys, groups=[0, 1, 0], n_groups=2, family="ordinal", n_classes=2, kernel="tc", weights=ws,
                        offsets=os_)
    logit = GlmShards(Xs, ys_logit, groups=[0, 1, 0], n_groups=2, kernel="tc", weights=ws, offsets=os_)
    ic, b, cp = _theta(2, P, 2)
    o, lg = _run(ordinal, ic, b, cp), _run(logit, ic - cp, b)
    np.testing.assert_allclose(o[0], lg[0], rtol=2e-5)
    np.testing.assert_allclose(o[1], lg[1], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(o[2], lg[2], rtol=1e-4, atol=0.2)
    np.testing.assert_allclose(o[3], [-lg[1].sum()], rtol=1e-4, atol=4e-3)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_ordinal_evaluations_are_bit_reproducible(dev):
    rows = [40_000, 25_000, 33_333, 128, 19_999]
    Xs, ys, ws, os_ = _case(rows, 256, 5, seed=12, device=dev)
    model = GlmShards(Xs, ys, groups=[0, 1, 2, 1, 0], n_groups=3, family="ordinal", n_classes=5, n_chains=2,
                      kernel="tc", weights=ws, offsets=os_)
    ic, beta, cp = _theta(3, 256, 5, 2)
    runs = _run(model, ic, beta, cp, repeats=10)
    for run in runs[1:]:
        for u, v in zip(runs[0], run):
            assert np.array_equal(u, v)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_unordered_cutpoints_leave_the_other_chains_alone(dev):
    rows, P, Cn, K = [20_000, 3_000], 256, 4, 3
    Xs, ys, ws, os_ = _case(rows, P, Cn, seed=15, device=dev)
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family="ordinal", n_classes=Cn, n_chains=K, kernel="tc",
                      weights=ws, offsets=os_)
    ic, beta, cp = _theta(2, P, Cn, K, gaps=(0.3, 1.0))
    cp2 = cp.copy()
    cp2[1] = [0.5, 0.5, 1.0]
    with FederatedEngine(model) as eng:
        good = [np.asarray(v).copy() for v in eng.evaluate(ic, beta, cp)]
        got = [np.asarray(v).copy() for v in eng.evaluate(ic, beta, cp2)]
    assert got[0][1] == -np.inf and all(np.all(g[1] == 0.0) for g in got[1:])
    for u, v in zip(got, good):
        assert np.array_equal(u[[0, 2]], v[[0, 2]])


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_node_federation_ordinal_blocks_equal_single_node_models(dev):
    from pytensor_federated_b200.federation import NodeFederation

    rows = [20_000, 128 * 33, 7777]
    node_ids, groups, Cn, P = [0, 1, 1], [0, 1, 0], 4, 256
    Xs, ys, ws, os_ = _case(rows, P, Cn, seed=13, device=dev)
    model = GlmShards(Xs, ys, groups=groups, n_groups=2, family="ordinal", n_classes=Cn, kernel="tc",
                      node_ids=node_ids, n_nodes=2, weights=ws, offsets=os_)
    ic, beta, cp = _theta(2, P, Cn, gaps=(0.3, 2.0))
    with FederatedEngine(model) as eng:
        n0 = eng.kernel_launches
        blocks = model.per_node(eng.evaluate_raw([ic, beta, cp]), model.call_context([ic, beta, cp]))
        assert eng.kernel_launches - n0 == 1
        fed = NodeFederation(eng)
        res = fed.evaluate_nodes({0: (ic, beta, cp), 1: (ic, beta, cp)})
        total = fed.all_nodes_func()(ic, beta, cp)
    for node in (0, 1):
        segs = [i for i, n in enumerate(node_ids) if n == node]
        single = GlmShards([Xs[i] for i in segs], [ys[i] for i in segs], groups=[groups[i] for i in segs], n_groups=2,
                           family="ordinal", n_classes=Cn, kernel="tc", weights=[ws[i] for i in segs],
                           offsets=[os_[i] for i in segs])
        want = _run(single, ic, beta, cp)
        np.testing.assert_allclose(blocks[node, 0, 0], want[0], rtol=2e-5)
        np.testing.assert_allclose(blocks[node, 0, 1:3], want[1], rtol=1e-4, atol=2e-3)
        np.testing.assert_allclose(blocks[node, 0, 3 : 3 + P], want[2], rtol=1e-4, atol=0.5)
        np.testing.assert_allclose(blocks[node, 0, 3 + P :], want[3], rtol=1e-4, atol=4e-3)
        np.testing.assert_allclose(res[node][0], blocks[node, 0, 0], rtol=1e-12)
        assert res[node][1][0].shape == (2,) and res[node][1][1].shape == (P,) and res[node][1][2].shape == (Cn - 1,)
        np.testing.assert_allclose(res[node][1][2], want[3], rtol=1e-4, atol=4e-3)
    np.testing.assert_allclose(total[0], blocks[:, 0, 0].sum(), rtol=1e-12)
    assert total[1][2].shape == (Cn - 1,)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_lock_step_hmc_on_an_ordinal_engine(dev):
    from pytensor_federated_b200.sampling import glm_batch_fn, hmc_sample_batched

    Cn, K, P = 4, 4, 16
    X, y, _, cuts = synth_ordinal_shard(20_000, P, Cn, seed=3, device=dev)
    model = GlmShards([X], [y], family="ordinal", n_classes=Cn, n_chains=K, kernel="tc")
    x0 = np.concatenate([np.zeros((K, 1 + P)), np.tile(cuts.astype(np.float64), (K, 1))], axis=1)
    with FederatedEngine(model) as eng:
        res = hmc_sample_batched(glm_batch_fn(eng, 1), x0, draws=5, tune=5, n_leapfrog=4, step_size=1e-3, seed=1)
        assert eng.n_evals == res.n_batched_evals
    assert res.samples.shape[-1] == 1 + P + Cn - 1 and np.all(np.isfinite(res.samples))
    assert np.all(res.accept_rate > 0)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_runtime_rejects_the_ordinal_family_outside_the_tc_kernel(dev):
    """The C ABI refuses what the Python layer never sends: family 6 on a CUDA-core kernel (which would take an
    unknown family for the Gaussian one), bad category counts, n_chains that are not K (C - 1), and a wrong n_vals;
    each before the engine's model changes."""
    from pytensor_federated_b200.ops import native

    Xs, ys, _, _ = _case([256], 16, 3, seed=14, device=dev, n_masked=0, weighted=False, offsets=False)
    model = GlmShards(Xs, ys, kernel="simt")   # n_vals = 1 + 1 + 16
    with FederatedEngine(model) as eng:
        lib, h = eng._lib, eng._handle
        Xp, yp = native.void_p_array([Xs[0].data_ptr()]), native.void_p_array([ys[0].data_ptr()])
        rows, grp = (C.c_longlong * 1)(256), (C.c_int * 1)(0)

        def set_glm(n_chains, family, code, n_classes):
            return int(lib.b200_engine_set_glm(h, 1, Xp, yp, None, rows, grp, 16, 16, 1, n_chains, family, code, None, 1,
                                               None, None, n_classes))

        for code in (0, 2, 3, 4):
            assert set_glm(1, 6, code, 2) != 0
            assert "tensor-core kernel only" in native.last_error()
        assert set_glm(1, 6, 1, 1) != 0 and "n_classes" in native.last_error()
        assert set_glm(16, 6, 1, 18) != 0 and "n_classes" in native.last_error()
        assert set_glm(3, 6, 1, 3) != 0 and "n_chains" in native.last_error()
        assert set_glm(2, 6, 1, 3) != 0 and "n_vals" in native.last_error()   # needs 2 x 18 values
        assert set_glm(1, 0, 0, 3) != 0 and "n_classes must be 1" in native.last_error()
        # the engine still evaluates its own model
        ic, beta = np.float32(0.1), np.zeros(16, np.float32)
        got = eng.evaluate(ic, beta)
    want = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)
