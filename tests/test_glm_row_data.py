"""Per-row offsets and observation weights of the GLM models (``GlmShards(..., offsets=, weights=)``).

CPU tests check the fp64 oracle and the collective backend against independent formulas (autograd, scipy);
GPU tests check every fused kernel against that oracle."""
import os
import shutil

import numpy as np
import pytest
import torch

from pytensor_federated_b200.models import CustomFamily, Fp8GlmShards, GlmShards
from pytensor_federated_b200.parallel import FederatedEngine

LOG_2PI_HALF = 0.918938533204672742


# ----------------------------------------------------------------------------------------------- fixtures
def _rows_case(rows, P, *, family="logistic", seed=0, device="cpu", dtype=torch.bfloat16, x_scale=1.0,
               none_segment=1, n_masked=5):
    """Segments with ragged sizes; logistic rows are binomial (``y = k / n``, ``w = n``), Poisson rows carry an
    exposure offset ``log t``; segment ``none_segment`` has neither (``None`` entries).  The first ``n_masked``
    rows of segment 0 have weight 0, and two of them a NaN response and a NaN offset."""
    rng = np.random.default_rng(seed)
    Xs, ys, offs, wts = [], [], [], []
    for si, n in enumerate(rows):
        X = rng.normal(size=(n, P)) * x_scale
        eta = X @ (rng.normal(size=P) * 0.05 / x_scale) + 0.2
        if family == "logistic":
            trials = rng.integers(1, 4, size=n).astype(np.float64)
            k = rng.binomial(trials.astype(int), 1.0 / (1.0 + np.exp(-eta)))
            y, o, w = k / trials, rng.normal(size=n) * 0.3, trials
        elif family == "poisson":
            t = rng.uniform(0.5, 3.0, size=n)
            y, o, w = rng.poisson(t * np.exp(np.clip(eta, None, 2.0))).astype(np.float64), np.log(t), rng.uniform(0.2, 2.0, size=n)
        else:
            y, o, w = eta + rng.normal(size=n), rng.normal(size=n) * 0.5, rng.uniform(0.2, 2.0, size=n)
        if si == 0:
            w[:n_masked] = 0.0
            y[1], o[2] = np.nan, np.nan
        Xs.append(torch.tensor(X, dtype=torch.float32).to(dtype).to(device))
        ys.append(torch.tensor(y, dtype=torch.float32, device=device))
        offs.append(None if si == none_segment else torch.tensor(o, dtype=torch.float32, device=device))
        wts.append(None if si == none_segment else torch.tensor(w, dtype=torch.float32, device=device))
    return Xs, ys, offs, wts


def _theta(G, P, K=1, seed=3):
    rng = np.random.default_rng(seed)
    shape = (K,) if K > 1 else ()
    return (rng.normal(size=shape + (G,)) * 0.2).astype(np.float32), (rng.normal(size=shape + (P,)) * 0.03).astype(np.float32)


def _explicit_fp64(Xs, ys, offs, wts, groups, G, family, ic, beta):
    """``[LL, dLL/dintercept, dLL/dbeta]`` of the weighted, offset model by autograd of the textbook formula."""
    t_ic = torch.tensor(np.asarray(ic, dtype=np.float64), requires_grad=True)
    t_b = torch.tensor(np.asarray(beta, dtype=np.float64), requires_grad=True)
    total = torch.zeros((), dtype=torch.float64)
    for X, y, o, w, g in zip(Xs, ys, offs, wts, groups):
        X, y = X.double().cpu(), y.double().cpu()
        o = o.double().cpu() if o is not None else torch.zeros_like(y)
        if w is not None:   # rows of weight 0 drop out: their y / o may be NaN, which a gradient must not see
            y, o = torch.where(w.cpu() != 0, y, 0.0), torch.where(w.cpu() != 0, o, 0.0)
        eta = X @ t_b + t_ic[g] + o
        if callable(family):
            ll = family(y, eta)[0]
        elif family == "logistic":
            ll = y * eta - torch.nn.functional.softplus(eta)
        elif family == "poisson":
            ll = y * eta - torch.exp(eta)
        else:
            ll = -0.5 * (y - eta) ** 2 - LOG_2PI_HALF
        if w is not None:
            w = w.double().cpu()
            ll = torch.where(w != 0, w * ll, torch.zeros_like(ll))
        total = total + ll.sum()
    total.backward()
    return total.item(), t_ic.grad.numpy(), t_b.grad.numpy()


# ----------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("family", ["logistic", "poisson", "gaussian"])
def test_oracle_matches_autograd_of_the_explicit_formula(family):
    rows, P, groups = [150, 70, 201], 12, [0, 1, 0]
    Xs, ys, offs, wts = _rows_case(rows, P, family=family, seed=1, dtype=torch.float64)
    model = GlmShards(Xs, ys, groups=groups, n_groups=2, family=family, offsets=offs, weights=wts)
    ic, beta = _theta(2, P)
    got = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64, chunk_rows=128))
    want = _explicit_fp64(Xs, ys, offs, wts, groups, 2, family, ic, beta)
    assert np.isfinite(got[0])
    np.testing.assert_allclose(got[0], want[0], rtol=1e-12)
    np.testing.assert_allclose(got[1], want[1], rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(got[2], want[2], rtol=1e-10, atol=1e-10)


def _collective(model, ic, beta):
    with FederatedEngine(model, backend="collective") as eng:
        return [np.asarray(v, dtype=np.float64) for v in eng.evaluate(ic, beta)]


def _central_differences(f, ic, beta, eps=1e-5):
    g_ic, g_b = np.zeros(len(ic)), np.zeros(len(beta))
    for vec, out in ((ic, g_ic), (beta, g_b)):
        for j in range(len(vec)):
            hi, lo = vec.copy(), vec.copy()
            hi[j] += eps
            lo[j] -= eps
            args_hi = (hi, beta) if vec is ic else (ic, hi)
            args_lo = (lo, beta) if vec is ic else (ic, lo)
            out[j] = (f(*args_hi) - f(*args_lo)) / (2 * eps)
    return g_ic, g_b


def test_binomial_rows_as_weighted_logistic_rows_match_scipy():
    import scipy.special
    import scipy.stats

    rng = np.random.default_rng(4)
    rows, P = [120, 90], 6
    Xs = [rng.normal(size=(n, P)) for n in rows]
    ns = [rng.integers(1, 12, size=n) for n in rows]
    ks = [rng.binomial(n, 0.35) for n in ns]
    model = GlmShards([torch.tensor(X) for X in Xs], [torch.tensor(k / n) for k, n in zip(ks, ns)], groups=[0, 1],
                      n_groups=2, weights=[torch.tensor(n, dtype=torch.float64) for n in ns])
    ic, beta = np.array([-0.4, -0.7]), rng.normal(size=P) * 0.2

    def truth(ic, beta):
        total = 0.0
        for g, (X, n, k) in enumerate(zip(Xs, ns, ks)):
            p = scipy.special.expit(X @ beta + ic[g])
            total += scipy.stats.binom.logpmf(k, n, p).sum() - np.log(scipy.special.comb(n, k)).sum()
        return total

    logp, d_ic, d_beta = _collective(model, ic, beta)
    np.testing.assert_allclose(logp, truth(ic, beta), rtol=1e-5)
    fd_ic, fd_b = _central_differences(truth, ic, beta)
    np.testing.assert_allclose(d_ic, fd_ic, rtol=1e-4, atol=1e-3)
    np.testing.assert_allclose(d_beta, fd_b, rtol=1e-4, atol=1e-3)


def test_poisson_rows_with_exposure_offsets_match_scipy():
    import scipy.special
    import scipy.stats

    rng = np.random.default_rng(5)
    rows, P = [100, 140], 5
    Xs = [rng.normal(size=(n, P)) for n in rows]
    ts = [rng.uniform(0.5, 4.0, size=n) for n in rows]
    ys = [rng.poisson(t * 1.5).astype(np.float64) for t in ts]
    model = GlmShards([torch.tensor(X) for X in Xs], [torch.tensor(y) for y in ys], groups=[0, 1], n_groups=2,
                      family="poisson", offsets=[torch.tensor(np.log(t)) for t in ts])
    ic, beta = np.array([0.3, 0.5]), rng.normal(size=P) * 0.1

    def truth(ic, beta):
        return sum(scipy.stats.poisson.logpmf(y, t * np.exp(X @ beta + ic[g])).sum() + scipy.special.gammaln(y + 1).sum()
                   for g, (X, y, t) in enumerate(zip(Xs, ys, ts)))

    logp, d_ic, d_beta = _collective(model, ic, beta)
    np.testing.assert_allclose(logp, truth(ic, beta), rtol=1e-5)
    fd_ic, fd_b = _central_differences(truth, ic, beta)
    np.testing.assert_allclose(d_ic, fd_ic, rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(d_beta, fd_b, rtol=1e-4, atol=2e-3)


@pytest.mark.parametrize("family", ["logistic", "poisson", "gaussian"])
def test_unit_weights_zero_offsets_duplicates_and_masks(family):
    Xs, ys, _, _ = _rows_case([80, 45], 8, family=family, seed=6, dtype=torch.float64, n_masked=0)
    ys = [torch.nan_to_num(y) for y in ys]
    ic, beta = _theta(2, 8)
    plain = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family=family)
    ones = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family=family, offsets=[torch.zeros(len(y)) for y in ys],
                     weights=[torch.ones(len(y)) for y in ys])
    for u, v in zip(_collective(plain, ic, beta), _collective(ones, ic, beta)):
        assert np.array_equal(u, v)
    # integer frequency weights == the rows repeated that often
    rng = np.random.default_rng(7)
    reps = [torch.tensor(rng.integers(0, 4, size=len(y)), dtype=torch.float32) for y in ys]
    freq = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family=family, weights=reps)
    dup = GlmShards([X.repeat_interleave(r.long(), 0) for X, r in zip(Xs, reps)],
                    [y.repeat_interleave(r.long()) for y, r in zip(ys, reps)], groups=[0, 1], n_groups=2, family=family)
    for u, v in zip(_collective(freq, ic, beta), _collective(dup, ic, beta)):
        np.testing.assert_allclose(u, v, rtol=1e-5, atol=1e-4)
    # zero weights == the rows removed, even where the masked response / offset is NaN
    keep = [torch.tensor(rng.random(len(y)) < 0.7) for y in ys]
    bad_y = [torch.where(k, y, torch.full_like(y, float("nan"))) for y, k in zip(ys, keep)]
    bad_o = [torch.where(k, torch.zeros_like(y), torch.full_like(y, float("inf"))) for y, k in zip(ys, keep)]
    masked = GlmShards(Xs, bad_y, groups=[0, 1], n_groups=2, family=family, offsets=bad_o,
                       weights=[k.float() for k in keep])
    cut = GlmShards([X[k] for X, k in zip(Xs, keep)], [y[k] for y, k in zip(ys, keep)], groups=[0, 1], n_groups=2,
                    family=family)
    for u, v in zip(_collective(masked, ic, beta), _collective(cut, ic, beta)):
        assert np.all(np.isfinite(u))
        np.testing.assert_allclose(u, v, rtol=1e-5, atol=1e-4)
    for u, v in zip(masked.unpack_result(masked.reference_partial([ic, beta], dtype=torch.float64)),
                    cut.unpack_result(cut.reference_partial([ic, beta], dtype=torch.float64))):
        np.testing.assert_allclose(u, v, rtol=1e-12, atol=1e-12)


def test_row_data_validation():
    Xs = [torch.randn(10, 4), torch.randn(6, 4)]
    ys = [torch.zeros(10), torch.zeros(6)]
    ok = [torch.ones(10), None]
    GlmShards(Xs, ys, offsets=ok, weights=ok)
    with pytest.raises(ValueError, match="one entry"):
        GlmShards(Xs, ys, weights=[torch.ones(10)])
    with pytest.raises(ValueError, match="rows"):
        GlmShards(Xs, ys, offsets=[torch.ones(10), torch.ones(7)])
    with pytest.raises(ValueError, match="rows"):
        GlmShards(Xs, ys, weights=[torch.ones(10, 1), None])
    with pytest.raises(ValueError, match=">= 0"):
        GlmShards(Xs, ys, weights=[-torch.ones(10), None])
    with pytest.raises(ValueError, match="finite"):
        GlmShards(Xs, ys, weights=[torch.full((10,), float("inf")), None])
    with pytest.raises(ValueError, match="finite"):
        GlmShards(Xs, ys, weights=[torch.full((10,), float("nan")), None])
    with pytest.raises(ValueError, match="finite"):
        GlmShards(Xs, ys, offsets=[torch.full((10,), float("nan")), None])
    # a non-finite offset is allowed on a row of weight 0 only
    o = torch.zeros(10)
    o[3] = float("inf")
    w = torch.ones(10)
    w[3] = 0.0
    GlmShards(Xs, ys, offsets=[o, None], weights=[w, None])
    with pytest.raises(ValueError, match="finite"):
        GlmShards(Xs, ys, offsets=[o, None], weights=[torch.ones(10), None])
    with pytest.raises(ValueError, match="device"):
        GlmShards(Xs, ys, weights=[torch.ones(10, device="meta"), None])
    m = GlmShards(Xs, ys, offsets=[np.zeros(10), None], weights=[None, torch.ones(6, dtype=torch.float64)])
    assert m.offsets[0].dtype == torch.float32 and m.weights[1].dtype == torch.float32 and m.weights[1].is_contiguous()
    assert m.has_row_data and not GlmShards(Xs, ys).has_row_data
    assert m.bytes_per_eval() == GlmShards(Xs, ys).bytes_per_eval() + 4 * (10 + 6)


def test_fp8_shards_pass_row_data_to_the_oracle():
    from pytensor_federated_b200.models import dequantize_block_fp8

    Xs, ys, offs, wts = _rows_case([200, 130, 64], 128, family="poisson", seed=8, dtype=torch.float32)
    fp8 = Fp8GlmShards.from_dense(Xs, ys, groups=[0, 1, 0], n_groups=2, family="poisson", offsets=offs, weights=wts)
    dense = GlmShards([dequantize_block_fp8(X, s) for X, s in zip(fp8.Xs, fp8.scales)], ys, groups=[0, 1, 0], n_groups=2,
                      family="poisson", offsets=offs, weights=wts)
    assert fp8.has_row_data and fp8.bytes_per_eval() > Fp8GlmShards.from_dense(Xs, ys).bytes_per_eval()
    ic, beta = _theta(2, 128)
    with FederatedEngine(fp8, backend="collective") as a, FederatedEngine(dense, backend="collective") as b:
        for u, v in zip(a.evaluate(ic, beta), b.evaluate(ic, beta)):
            assert np.all(np.isfinite(u))
            np.testing.assert_allclose(u, v, rtol=1e-6, atol=1e-6)


STUDENT_T = ("const float d = y - eta; ll = -2.5f * log1pf(d * d * 0.25f); r = 5.f * d / (4.f + d * d);",
             lambda y, eta: (-2.5 * torch.log1p((y - eta) ** 2 / 4), 5 * (y - eta) / (4 + (y - eta) ** 2)))


def test_custom_family_compiles_against_the_row_data_descriptor():
    if shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"):
        pytest.skip("nvcc not available")
    family = CustomFamily(STUDENT_T[0], torch_fn=STUDENT_T[1])
    assert family.launcher_address() != 0
    Xs, ys, offs, wts = _rows_case([60, 40], 4, family="gaussian", seed=9, dtype=torch.float32)
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family=family, offsets=offs, weights=wts)
    ic, beta = _theta(2, 4)
    got = _collective(model, ic, beta)
    want = _explicit_fp64(Xs, ys, offs, wts, [0, 1], 2, STUDENT_T[1], ic, beta)
    np.testing.assert_allclose(got[0], want[0], rtol=1e-5)
    np.testing.assert_allclose(got[1], want[1], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(got[2], want[2], rtol=1e-4, atol=1e-4)


# ----------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from pytensor_federated_b200.ops import native

    native.load()  # a GPU box without the native library is a failure, not a skip
    return torch.device("cuda:0")


def _oracle(model, ic, beta):
    return model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))


def _run(model, ic, beta, repeats=1):
    with FederatedEngine(model) as eng:
        out = [[np.asarray(v).copy() for v in eng.evaluate(ic, beta)] for _ in range(repeats)]
    return out[0] if repeats == 1 else out


def _check(got, want, rtol_ll, rtol_g, atol_ic, atol_b):
    assert all(np.all(np.isfinite(g)) for g in got)
    np.testing.assert_allclose(got[0], want[0], rtol=rtol_ll)
    np.testing.assert_allclose(got[1], want[1], rtol=rtol_g, atol=atol_ic)
    np.testing.assert_allclose(got[2], want[2], rtol=rtol_g, atol=atol_b)


@pytest.mark.parametrize("K", [1, 4, 16])
@pytest.mark.parametrize("P", [256, 200, 8])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_with_row_data_matches_oracle(dev, K, P):
    rows = [128 * 37, 77, 4099, 1]
    Xs, ys, offs, wts = _rows_case(rows, P, seed=K + P, device=dev)
    model = GlmShards(Xs, ys, groups=[0, 1, 0, 1], n_groups=2, n_chains=K, kernel="tc", offsets=offs, weights=wts)
    ic, beta = _theta(2, P, K)
    got = _run(model, ic, beta)
    assert model.selected_kernel == "tc"
    _check(got, _oracle(model, ic, beta), 2e-5, 1e-4, 2e-3, 2e-3 * np.sqrt(sum(rows)) if K == 1 else 0.2)


@pytest.mark.parametrize("family", ["poisson", "gaussian"])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_with_row_data_unbounded_families(dev, family):
    rows = [128 * 20 + 3, 999, 64]
    Xs, ys, offs, wts = _rows_case(rows, 256, family=family, seed=2, device=dev)
    model = GlmShards(Xs, ys, groups=[0, 1, 0], n_groups=2, family=family, kernel="tc", offsets=offs, weights=wts)
    ic, beta = _theta(2, 256)
    want = _oracle(model, ic, beta)
    _check(_run(model, ic, beta), want, 2e-5, 1e-4, 2e-3, 2e-3 * np.sqrt(sum(rows)))


@pytest.mark.parametrize("family", ["logistic", "poisson", "gaussian"])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_simt_kernel_with_row_data_matches_oracle(dev, family):
    rows = [1000, 77, 4099, 8]
    Xs, ys, offs, wts = _rows_case(rows, 256, family=family, seed=3, device=dev)
    model = GlmShards(Xs, ys, groups=[0, 1, 0, 2], n_groups=3, family=family, kernel="simt", offsets=offs, weights=wts)
    ic, beta = _theta(3, 256)
    _check(_run(model, ic, beta), _oracle(model, ic, beta), 2e-5, 1e-4, 2e-3, 2e-3 * np.sqrt(sum(rows)))


@pytest.mark.parametrize("P,dtype", [(200, torch.bfloat16), (37, torch.float32)])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_generic_kernel_with_row_data_matches_oracle(dev, P, dtype):
    rows = [301, 64, 5]
    Xs, ys, offs, wts = _rows_case(rows, P, seed=4, device=dev, dtype=dtype)
    model = GlmShards(Xs, ys, groups=[0, 1, 0], n_groups=2, kernel="generic", offsets=offs, weights=wts)
    ic, beta = _theta(2, P)
    got = _run(model, ic, beta)
    assert model.selected_kernel.startswith("generic")
    _check(got, _oracle(model, ic, beta), 2e-5, 1e-4, 2e-3, 2e-3)


@pytest.mark.parametrize("family", ["logistic", "poisson"])
@pytest.mark.parametrize("K", [1, 3])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_fp8_kernel_with_row_data_matches_oracle(dev, family, K):
    rows = [128 * 35 + 17, 640, 999]
    Xs, ys, offs, wts = _rows_case(rows, 256, family=family, seed=5 + K, device=dev, dtype=torch.float32, x_scale=1.5)
    model = Fp8GlmShards.from_dense(Xs, ys, groups=[0, 1, 0], n_groups=2, n_chains=K, family=family,
                                    offsets=offs, weights=wts)
    ic, beta = _theta(2, 256, K)
    w = _oracle(model, ic, beta)
    _check(_run(model, ic, beta), w, 3e-5, 3e-4, 2e-4 * np.abs(w[1]).max(), 3e-4 * np.abs(w[2]).max())


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_fp8_kernel_with_offsets_only(dev):
    """Offsets without weights keep the logistic residuals bounded: the kernel without residual scaling."""
    Xs, ys, offs, _ = _rows_case([128 * 20 + 5, 300], 128, seed=6, device=dev, dtype=torch.float32, n_masked=0)
    ys = [torch.nan_to_num(y) for y in ys]
    offs = [torch.nan_to_num(o) if o is not None else None for o in offs]
    model = Fp8GlmShards.from_dense(Xs, ys, groups=[0, 1], n_groups=2, offsets=offs)
    ic, beta = _theta(2, 128)
    w = _oracle(model, ic, beta)
    _check(_run(model, ic, beta), w, 2e-5, 1e-4, 5e-3, 2e-4 * np.abs(w[2]).max())


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_custom_family_with_row_data_matches_oracle(dev):
    Xs, ys, offs, wts = _rows_case([3000, 2000], 96, family="gaussian", seed=7, device=dev)
    family = CustomFamily(STUDENT_T[0], torch_fn=STUDENT_T[1])
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family=family, offsets=offs, weights=wts)
    ic, beta = _theta(2, 96)
    _check(_run(model, ic, beta), _oracle(model, ic, beta), 2e-5, 1e-4, 5e-3, 5e-3)


@pytest.mark.parametrize("kernel", ["tc", "simt", "generic", "fp8"])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_unit_weights_and_zero_offsets_reproduce_the_plain_model(dev, kernel):
    """tc, simt, generic: the same bits.  fp8 logistic: close only, because weights switch on the per-row-group
    residual scaling, which rounds the residual operand differently."""
    rows = [128 * 30 + 9, 5000, 77]
    Xs, ys, _, _ = _rows_case(rows, 256, seed=8, device=dev, dtype=torch.float32, n_masked=0)
    ys = [torch.nan_to_num(y) for y in ys]
    zeros, ones = [torch.zeros_like(y) for y in ys], [torch.ones_like(y) for y in ys]
    ic, beta = _theta(2, 256)
    if kernel == "fp8":
        plain = Fp8GlmShards.from_dense(Xs, ys, groups=[0, 1, 0], n_groups=2)
        rows_ = Fp8GlmShards.from_dense(Xs, ys, groups=[0, 1, 0], n_groups=2, offsets=zeros, weights=ones)
    else:
        Xb = [X.to(torch.bfloat16) for X in Xs]
        plain = GlmShards(Xb, ys, groups=[0, 1, 0], n_groups=2, kernel=kernel)
        rows_ = GlmShards(Xb, ys, groups=[0, 1, 0], n_groups=2, kernel=kernel, offsets=zeros, weights=ones)
    a, b = _run(plain, ic, beta), _run(rows_, ic, beta)
    for u, v in zip(a, b):
        if kernel == "fp8":
            np.testing.assert_allclose(u, v, rtol=1e-4, atol=2e-4 * np.abs(a[2]).max())
        else:
            assert np.array_equal(u, v)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_frequency_weights_equal_duplicated_rows_and_masks_equal_truncation(dev):
    rng = np.random.default_rng(9)
    rows = [128 * 25 + 3, 2000]
    Xs, ys, _, _ = _rows_case(rows, 256, seed=9, device=dev, n_masked=0)
    ys = [torch.nan_to_num(y) for y in ys]
    ic, beta = _theta(2, 256)
    reps = [torch.tensor(rng.integers(0, 4, size=n), device=dev) for n in rows]
    freq = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, kernel="tc", weights=[r.float() for r in reps])
    dup = GlmShards([X.repeat_interleave(r, 0) for X, r in zip(Xs, reps)], [y.repeat_interleave(r) for y, r in zip(ys, reps)],
                    groups=[0, 1], n_groups=2, kernel="tc")
    a, b = _run(freq, ic, beta), _run(dup, ic, beta)
    np.testing.assert_allclose(a[0], b[0], rtol=1e-6)
    np.testing.assert_allclose(a[1], b[1], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(a[2], b[2], rtol=1e-4, atol=0.05)
    # rows 1000.. of segment 0 masked (y NaN there) == segment 0 cut at row 1000
    w0 = torch.ones(rows[0], device=dev)
    w0[1000:] = 0.0
    y0 = ys[0].clone()
    y0[1000::7] = float("nan")
    masked = GlmShards(Xs, [y0, ys[1]], groups=[0, 1], n_groups=2, kernel="tc", weights=[w0, None])
    cut = GlmShards([Xs[0][:1000], Xs[1]], [ys[0][:1000], ys[1]], groups=[0, 1], n_groups=2, kernel="tc")
    a, b = _run(masked, ic, beta), _run(cut, ic, beta)
    np.testing.assert_allclose(a[0], b[0], rtol=1e-6)
    np.testing.assert_allclose(a[1], b[1], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(a[2], b[2], rtol=1e-4, atol=0.05)


@pytest.mark.parametrize("kernel", ["tc", "fp8"])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_row_data_evaluations_are_bit_reproducible(dev, kernel):
    rows = [40_000, 25_000, 33_333, 128, 19_999]
    Xs, ys, offs, wts = _rows_case(rows, 256, seed=10, device=dev, dtype=torch.float32)
    if kernel == "fp8":
        model = Fp8GlmShards.from_dense(Xs, ys, groups=[0, 1, 2, 1, 0], n_groups=3, offsets=offs, weights=wts)
    else:
        model = GlmShards([X.to(torch.bfloat16) for X in Xs], ys, groups=[0, 1, 2, 1, 0], n_groups=3, kernel="tc",
                          offsets=offs, weights=wts)
    ic, beta = _theta(3, 256)
    runs = _run(model, ic, beta, repeats=10)
    for run in runs[1:]:
        for u, v in zip(runs[0], run):
            assert np.array_equal(u, v)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_node_federation_blocks_with_weights_equal_single_node_models(dev):
    from pytensor_federated_b200.federation import NodeFederation

    rows = [20_000, 128 * 33, 7777]
    node_ids, groups = [0, 1, 1], [0, 1, 0]
    Xs, ys, offs, wts = _rows_case(rows, 256, seed=11, device=dev)
    model = GlmShards(Xs, ys, groups=groups, n_groups=2, kernel="tc", node_ids=node_ids, n_nodes=2,
                      offsets=offs, weights=wts)
    ic, beta = _theta(2, 256)
    with FederatedEngine(model) as eng:
        n0 = eng.kernel_launches
        blocks = model.per_node(eng.evaluate_raw([ic, beta]))
        assert eng.kernel_launches - n0 == 1
        res = NodeFederation(eng).evaluate_nodes({0: (ic, beta), 1: (ic, beta)})
    for node in (0, 1):
        segs = [i for i, n in enumerate(node_ids) if n == node]
        single = GlmShards([Xs[i] for i in segs], [ys[i] for i in segs], groups=[groups[i] for i in segs], n_groups=2,
                           kernel="tc", offsets=[offs[i] for i in segs], weights=[wts[i] for i in segs])
        want = _run(single, ic, beta)
        np.testing.assert_allclose(blocks[node, 0, 0], want[0], rtol=2e-5)
        np.testing.assert_allclose(blocks[node, 0, 1:3], want[1], rtol=1e-4, atol=2e-3)
        np.testing.assert_allclose(blocks[node, 0, 3:], want[2], rtol=1e-4, atol=0.5)
        np.testing.assert_allclose(res[node][0], blocks[node, 0, 0], rtol=1e-12)


def _build_rows_model(rank, world, dev):
    Xs, ys, offs, wts = _rows_case([30_000 + 17 * rank], 256, seed=50 + rank, device=dev, none_segment=None)
    return GlmShards(Xs, ys, groups=[rank % 2], n_groups=2, kernel="tc", offsets=offs, weights=wts)


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.timeout(900)
def test_two_rank_tc_federation_with_row_data_matches_oracle():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from pytensor_federated_b200.federation import launch_federation

    ic, beta = _theta(2, 256)
    dev = torch.device("cuda:0")
    models = [_build_rows_model(r, 2, dev) for r in range(2)]
    want = models[0].unpack_result(sum(m.reference_partial([ic, beta], dtype=torch.float64) for m in models),
                                   models[0].call_context([ic, beta]))
    del models
    with launch_federation(_build_rows_model, 2, timeout=30.0) as eng:
        got = eng.evaluate(ic, beta)
    _check(got, want, 2e-5, 1e-4, 2e-3, 0.5)
