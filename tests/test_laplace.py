"""Laplace approximation (``sampling.laplace``) and the Hessian assembled from Hessian-vector products
(``sampling.glm_hessian``).

CPU: on a Gaussian linear model with a Gaussian prior the posterior is Gaussian, so the Laplace approximation is
exact: its mean, covariance and evidence must match the closed form.  ``glm_hessian`` on a CPU logistic engine must
match the autograd Hessian of an fp64 log-likelihood.  GPU: standard errors of a 2-shard logistic model from the
kernel's Hessian against an fp64 Hessian of the same data on the CPU.
"""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

from pytensor_federated_b200.models import GlmShards
from pytensor_federated_b200.parallel import FederatedEngine
from pytensor_federated_b200.sampling import glm_batch_fn, glm_hessian, glm_hvp_fn, laplace


def _gaussian_data(n=400, P=8, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, P)).astype(np.float32)
    beta = rng.normal(size=P) * 0.5
    y = (0.3 + X.astype(np.float64) @ beta + rng.normal(size=n)).astype(np.float32)
    return X, y


def test_laplace_exact_on_gaussian_linear_model():
    X, y = _gaussian_data()
    n, P = X.shape
    D, tau2 = 1 + P, 4.0
    m = GlmShards([torch.from_numpy(X)], [torch.from_numpy(y)], family="gaussian", n_chains=2, hvp=True)
    eng = FederatedEngine(m, backend="collective")
    # fp64 oracle path of the collective engine: the model's reference_partial in float64
    m.reference_partial = (lambda f: lambda inputs, **kw: f(inputs, dtype=torch.float64))(m.reference_partial)
    Xt = np.concatenate([np.ones((n, 1)), X.astype(np.float64)], axis=1)
    yd = y.astype(np.float64)

    def logp_dlogp(th):
        r = yd - Xt @ th
        lp = -0.5 * r @ r - n * 0.5 * math.log(2 * math.pi) - th @ th / (2 * tau2) - 0.5 * D * math.log(2 * math.pi * tau2)
        return lp, Xt.T @ r - th / tau2

    def hessian(th):
        return glm_hessian(eng, th)[2] - np.eye(D) / tau2

    res = laplace(logp_dlogp, hessian, np.zeros(D))
    A = Xt.T @ Xt + np.eye(D) / tau2
    cov = np.linalg.inv(A)
    mean = cov @ (Xt.T @ yd)
    S = np.eye(n) + tau2 * Xt @ Xt.T
    sign, logdet = np.linalg.slogdet(S)
    evidence = -0.5 * yd @ np.linalg.solve(S, yd) - 0.5 * logdet - 0.5 * n * math.log(2 * math.pi)
    assert res["converged"]
    np.testing.assert_allclose(res["mean"], mean, rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(res["cov"], cov, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(res["sd"], np.sqrt(np.diag(cov)), rtol=1e-9)
    assert abs(res["log_evidence"] - evidence) <= 1e-9 * abs(evidence)
    assert res["n_evals"] > 0 and res["n_hessian_evals"] == 2


def test_laplace_refuses_a_hessian_that_is_not_negative_definite():
    with pytest.raises(ValueError, match="smallest eigenvalue is -0.5"):
        laplace(lambda th: (-0.5 * th @ th, -th), lambda th: np.diag([-1.0, 0.5]), np.ones(2))


def test_glm_hessian_matches_autograd_on_cpu_logistic():
    rng = np.random.default_rng(1)
    n, P, K = 500, 16, 3
    X = torch.from_numpy(rng.normal(size=(n, P)).astype(np.float32))
    y = torch.from_numpy((rng.uniform(size=n) < 0.4).astype(np.float32))
    m = GlmShards([X], [y], family="logistic", n_chains=K, hvp=True)
    eng = FederatedEngine(m, backend="collective")
    theta = rng.normal(size=1 + P) * 0.3
    logp, grad, H = glm_hessian(eng, theta)
    Xt = torch.cat([torch.ones(n, 1, dtype=torch.float64), X.double()], 1)
    yd = y.double()

    def ll(th):
        eta = Xt @ th
        return (yd * eta - torch.nn.functional.softplus(eta)).sum()

    th = torch.from_numpy(theta)
    want = torch.autograd.functional.hessian(ll, th).numpy()
    # the collective engine's oracle runs in float32
    scale = np.abs(Xt.numpy()).T @ np.abs(Xt.numpy()) * 0.25
    assert np.all(np.abs(H - want) <= 1e-5 * scale + 1e-6)
    np.testing.assert_allclose(logp, float(ll(th)), rtol=1e-5)
    g = torch.autograd.functional.jacobian(ll, th).numpy()
    assert np.all(np.abs(grad - g) <= 1e-5 * np.abs(Xt.numpy()).sum(0))
    # glm_hvp_fn on any n: tiled over K with a padded last tile
    V = rng.normal(size=(7, 1 + P))
    lp, gr, hv = glm_hvp_fn(eng)(np.broadcast_to(theta, (7, 1 + P)), V)
    assert lp.shape == (7,) and gr.shape == (7, 1 + P) and hv.shape == (7, 1 + P)
    assert np.all(np.abs(hv - V @ want.T) <= 1e-5 * np.abs(V) @ scale.T + 1e-6)


def test_glm_hvp_fn_needs_an_hvp_model():
    m = GlmShards([torch.zeros(4, 8)], [torch.zeros(4)], family="logistic")
    with pytest.raises(ValueError, match="hvp=True"):
        glm_hvp_fn(FederatedEngine(m, backend="collective"))


@pytest.mark.gpu
def test_laplace_standard_errors_on_gpu():
    from pytensor_federated_b200.models import synth_logistic_shard

    dev = torch.device("cuda:0")
    P, K, tau2 = 64, 8, 100.0
    Xs, ys = [], []
    for s in range(2):
        X, y, _ = synth_logistic_shard(100_000 + 4099 * s, P, seed=11 + s, device=dev)
        Xs.append(X)
        ys.append(y)
    D = 1 + P
    with FederatedEngine(GlmShards(Xs, ys, n_chains=K)) as grad_eng, \
            FederatedEngine(GlmShards(Xs, ys, n_chains=K, hvp=True)) as hvp_eng:
        batch = glm_batch_fn(grad_eng, 1)

        def logp_dlogp(th):
            lp, g = batch(th[None])
            return float(lp[0]) - th @ th / (2 * tau2), g[0] - th / tau2

        res = laplace(logp_dlogp, lambda th: glm_hessian(hvp_eng, th)[2] - np.eye(D) / tau2, np.zeros(D))
    # fp64 Hessian of the oracle at the same mode, on the CPU
    Xt = torch.cat([torch.cat([torch.ones(X.shape[0], 1, dtype=torch.float64), X.double().cpu()], 1) for X in Xs])
    mu = torch.sigmoid(Xt @ torch.from_numpy(res["mean"]))
    H = -(Xt * (mu * (1 - mu)).unsqueeze(1)).T @ Xt - torch.eye(D, dtype=torch.float64) / tau2
    sd = np.sqrt(np.diag(np.linalg.inv(-H.numpy())))
    # (L-BFGS-B may report a line-search failure this close to the mode, where the kernel's rounded logp is flat to
    # its last bits; laplace's Newton step polishes the mode either way, so `converged` is not asserted here)
    np.testing.assert_allclose(res["sd"], sd, rtol=1e-4)
