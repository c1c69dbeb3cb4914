"""Location-scale regression: ``GlmShards(..., family="gaussian_location_scale")`` and ``family="student_t"`` (inputs
``intercept, beta, sigma_intercept, sigma_beta[, log_dispersion = log nu]``).

CPU tests check the fp64 oracle against scipy's and mpmath's densities and derivatives (s from -5 to 5, nu from 0.2 to
1e12, outliers with |z| up to 1e30), the nu -> inf limit, the layout (packing, words, fold, sizes), validation, the
collective backend and a robust fit; GPU tests check the tensor-core kernel against that oracle within a rounding bound
derived from each sum's terms, row by row across the domain, bit for bit against the Gaussian launch where the scale
is 1, and its packed-X, per-node and sampling paths."""
import ctypes as C

import numpy as np
import pytest
import torch

from pytensor_federated_b200.models import Fp8GlmShards, GlmShards, synth_location_scale_shard
from pytensor_federated_b200.models.glm import _location_scale_terms, _student_t_constants
from pytensor_federated_b200.parallel import FederatedEngine
from pytensor_federated_b200.parallel.engine import default_inputs_from_words

FAMILIES = ("gaussian_location_scale", "student_t")
T = "student_t"
#: log nu of the tests' chains: 0.2 .. 1e12
LOG_NU = np.log([0.2, 1.0, 3.0, 30.0, 1e3, 1e5, 1e8, 1e12])
#: sigma intercepts of the tests' chains
SIGMA_ICPT = np.array([-5.0, -1.0, 0.0, 1.5, 5.0])


# ----------------------------------------------------------------------------------------------- fixtures
def _case(rows, P, *, seed=0, device="cpu", n_masked=5, weighted=True, offsets=True, nu=4.0, outliers=(1e2, 1e4, 1e8),
          beta_scale=0.03):
    """Ragged bf16 segments of Student-t (``nu``; None: Gaussian) responses around ``x' beta + 0.4 (+ o)`` with a scale
    that depends on x, plus one gross outlier ``mu +- v`` per value of ``outliers`` in every segment of more than 64
    rows.  With ``weighted``, every segment but the last has weights; the first ``n_masked`` rows of segment 0 have
    weight 0 and carry a NaN, an inf and a -inf.  With ``offsets``, every segment but the second has offsets."""
    rng = np.random.default_rng(seed)
    Xs, ys, ws, os_ = [], [], [], []
    for si, n in enumerate(rows):
        X = torch.tensor(rng.normal(size=(n, P)), dtype=torch.float32).to(torch.bfloat16)
        Xd = X.double().numpy()
        o = rng.uniform(-1.0, 1.0, size=n)
        mu = Xd @ (rng.normal(size=P) * beta_scale) + 0.4 + (o if offsets else 0.0)
        sigma = np.exp(Xd @ (rng.normal(size=P) * 0.03) - 0.2)
        eps = rng.normal(size=n) if nu is None else rng.standard_t(nu, size=n)
        y = mu + sigma * eps
        if n > 64:
            idx = rng.choice(np.arange(n_masked, n), size=len(outliers), replace=False)
            y[idx] = mu[idx] + np.asarray(outliers) * rng.choice([-1.0, 1.0], size=len(outliers))
        w = rng.uniform(0.2, 2.0, size=n)
        if si == 0 and n_masked:
            w[:n_masked] = 0.0
            y[:3] = [np.nan, np.inf, -np.inf][: min(3, n_masked)]
        Xs.append(X.to(device))
        ys.append(torch.tensor(y, dtype=torch.float32, device=device))
        ws.append(torch.tensor(w, dtype=torch.float32, device=device) if weighted and si < len(rows) - 1 else None)
        os_.append(torch.tensor(o, dtype=torch.float32, device=device) if offsets and si != 1 else None)
    return Xs, ys, ws, os_


def _theta(family, G, P, K=1, *, sic=-0.2, log_nu=np.log(4.0), seed=3, scale=0.03):
    """``(intercept, beta, sigma_intercept, sigma_beta[, log_dispersion])``, batched for K > 1 (``sic`` and
    ``log_nu`` may give one value per chain: the sigma intercepts are ``sic`` plus noise)."""
    rng = np.random.default_rng(seed)
    lead = (K,) if K > 1 else ()
    sic = np.asarray(sic, dtype=np.float64)
    out = [(0.4 + rng.normal(size=lead + (G,)) * 0.2).astype(np.float32),
           (rng.normal(size=lead + (P,)) * scale).astype(np.float32),
           ((sic[..., None] if sic.ndim else sic) + rng.normal(size=lead + (G,)) * 0.1).astype(np.float32),
           (rng.normal(size=lead + (P,)) * scale).astype(np.float32)]
    if family == T:
        out.append(np.broadcast_to(np.asarray(log_nu, dtype=np.float32), lead).copy() if K > 1 else np.float32(log_nu))
    return tuple(out)


def _oracle(model, *inputs, chunk_rows=128):
    return model.unpack_result(model.reference_partial(list(inputs), dtype=torch.float64, chunk_rows=chunk_rows))


def _collective(model, *inputs):
    with FederatedEngine(model, backend="collective") as eng:
        return [np.asarray(v, dtype=np.float64) for v in eng.evaluate(*inputs)]


def _terms64(y, mu, s, a=None):
    """The fp64 oracle's per-row ``(ll, dll/dmu, dll/ds[, dll/da])`` of scalars or 1-D arrays, one chain."""
    t = lambda v: torch.as_tensor(np.asarray(v, dtype=np.float64)).reshape(-1, 1)
    out = _location_scale_terms(t(y), t(mu), t(s), None if a is None else torch.tensor([float(a)], dtype=torch.float64))
    ll, r = out[0][:, 0, 0].numpy(), out[1][:, 0].numpy()
    res = [ll, r[:, 0], r[:, 1]]
    if a is not None:
        res.append(out[2][:, 0, 0].numpy())
    return res


# ----------------------------------------------------------------------------------------------- CPU: the oracle
def test_student_t_constants_match_mpmath():
    """C(nu) and Q(nu) from nu = 0.2 to 1e12, both sides of the series switch at 1e3, against 60-digit mpmath."""
    import mpmath as mp

    mp.mp.dps = 60
    nus = np.concatenate([[0.2, 0.5, 1.0, 2.0, 7.9, 16.0, 100.0, 999.0, 1000.0, 1001.0], np.logspace(4, 12, 9)])
    nu, Cn, Q = (v.numpy() for v in _student_t_constants(torch.tensor(np.log(nus))))
    for v, c, q in zip(nu, Cn, Q):
        n = mp.mpf(float(v))
        c_mp = mp.loggamma((n + 1) / 2) - mp.loggamma(n / 2) - mp.log(n * mp.pi) / 2
        q_mp = n / 2 * (mp.digamma((n + 1) / 2) - mp.digamma(n / 2)) - mp.mpf(1) / 2
        # below 1e3 C and Q are differences of lgamma / digamma values of size up to nu log nu: an absolute accuracy of
        # about 1e-13; above, the series are accurate to the last bits
        assert abs(c - float(c_mp)) <= (1e-15 if v >= 1e3 else 1e-12), (v, c, float(c_mp))
        assert abs(q - float(q_mp)) <= (1e-12 * abs(float(q_mp)) if v >= 1e3 else 1e-12), (v, q, float(q_mp))


def _z_grid():
    return np.concatenate([[0.0], np.outer([1.0, -1.0], [1e-4, 0.1, 0.5, 1.0, 2.0, 5.0, 30.0, 1e3, 1e6, 1e10, 1e15,
                                                        1e20, 1e30]).reshape(-1)])


@pytest.mark.parametrize("nu", [0.2, 1.0, 3.0, 30.0, 1e3, 1e4, 1e6, 1e9, 1e12])
def test_student_t_terms_match_mpmath_across_the_domain(nu):
    """ll and its derivatives in mu, s and a = log nu, against their closed forms in 40-digit mpmath (with mpmath's
    loggamma and digamma), for s in [-5, 5] and z from 0 to +-1e30 (z^2 far past the fp32 range); the float32 oracle
    (the collective backend's) stays finite there and within a few hundred ulps of the values' magnitudes."""
    import mpmath as mp

    mp.mp.dps = 40
    a = float(np.log(nu))
    n = mp.exp(mp.mpf(a))
    Cm = mp.loggamma((n + 1) / 2) - mp.loggamma(n / 2) - mp.log(n * mp.pi) / 2
    Qm = n / 2 * (mp.digamma((n + 1) / 2) - mp.digamma(n / 2)) - mp.mpf(1) / 2
    zs = _z_grid()
    for s in (-5.0, 0.0, 5.0):
        mu = 0.3
        y = mu + zs * np.exp(s)
        got = _terms64(y, mu, s, a)
        for i, yi in enumerate(y):
            si = mp.exp(-mp.mpf(s))
            z = (mp.mpf(float(yi)) - mp.mpf(mu)) * si
            q = z * z / n
            want = [Cm - s - (n + 1) / 2 * mp.log1p(q), (n + 1) * z * si / (n + z * z), (n + 1) * z * z / (n + z * z) - 1,
                    Qm + q / (2 * (1 + q)) - n / 2 * (mp.log1p(q) - q / (1 + q))]
            for k, (g, w) in enumerate(zip(got, want)):
                w = float(w)
                # fp64 forms: 1e-12 of the value (dll/da: 1e-10, and 1e-12 absolute for Q's accuracy below nu = 1e3),
                # plus the rounding of y - mu (2^-52 of |y| + |mu|) times the slope
                tol = ((1e-12 if k < 3 else 1e-10) * abs(w) + (1e-13 if k < 3 else 1e-12)
                       + (abs(float(want[1])) + 1) * 2.0 ** -52 * (abs(yi) + mu))
                assert abs(g[i] - w) <= tol, (nu, s, zs[i], k, g[i], w)
        # bounded influence: dll/dmu falls as 1 / z (zs[9] = 1e6, zs[13] = 1e30, zs[26] = -1e30)
        assert abs(got[1][13]) < 1e-20 * abs(got[1][9]) and abs(got[1][26]) < 1e-20 * abs(got[1][9])
        # float32: finite, and within 2^-12 of the magnitudes of the fp64 values at the same (float32) inputs
        y32, mu32, s32, a32 = y.astype(np.float32), np.float32(mu), np.float32(s), np.float32(a)
        t32 = lambda v: torch.as_tensor(np.asarray(v, dtype=np.float32)).reshape(-1, 1)
        out = _location_scale_terms(t32(y32), t32(mu32), t32(s32), torch.tensor([a32], dtype=torch.float32))
        f32 = [out[0][:, 0, 0], out[1][:, 0, 0], out[1][:, 0, 1], out[2][:, 0, 0]]
        ref = _terms64(y32.astype(np.float64), float(mu32), float(s32), float(a32))
        nu32 = float(np.exp(np.float64(a32)))
        z = (y32.astype(np.float64) - float(mu32)) * np.exp(-float(s32))
        L = np.log1p(z * z / nu32)
        mags = (np.abs(ref[0]) + (nu32 + 1) / 2 * L + 1 + abs(s), np.abs(ref[1]), np.abs(ref[2]) + 1,
                np.abs(ref[3]) + nu32 * L + 1)
        for v, w, mag in zip(f32, ref, mags):
            v = v.double().numpy()
            assert np.all(np.isfinite(v)), (nu, s)
            assert np.all(np.abs(v - w) <= 2.0 ** -12 * mag), (nu, s, np.max(np.abs(v - w) / mag))


def test_cauchy_and_the_gaussian_family_match_scipy():
    from scipy import stats

    rng = np.random.default_rng(0)
    y = np.concatenate([rng.normal(size=200) * 3, [1e6, -1e10, 1e20]])
    for s in (-5.0, -0.7, 0.0, 2.0, 5.0):
        mu = 0.25
        sig = np.exp(s)
        ll, rm, rs, qa = _terms64(y, mu, s, 0.0)   # nu = 1
        np.testing.assert_allclose(ll, stats.cauchy(mu, sig).logpdf(y), rtol=1e-13, atol=1e-13)
        np.testing.assert_allclose(ll, stats.t(df=1.0, loc=mu, scale=sig).logpdf(y), rtol=1e-13, atol=1e-13)
        z = (y - mu) / sig
        np.testing.assert_allclose(rm, 2 * z / (1 + z * z) / sig, rtol=1e-13, atol=1e-300)
        np.testing.assert_allclose(rs, 2 * z * z / (1 + z * z) - 1, rtol=1e-13, atol=1e-15)
        for nu in (0.2, 4.0, 300.0):
            ll, *_ = _terms64(y, mu, s, np.log(nu))
            np.testing.assert_allclose(ll, stats.t(df=float(np.exp(np.log(nu))), loc=mu, scale=sig).logpdf(y),
                                       rtol=1e-12, atol=1e-12)
        yg = y[:200]
        ll, rm, rs = _terms64(yg, mu, s)
        zg = (yg - mu) / sig
        np.testing.assert_allclose(ll, stats.norm(mu, sig).logpdf(yg), rtol=1e-13, atol=1e-13)
        np.testing.assert_allclose(rm, zg / sig, rtol=1e-14)
        np.testing.assert_allclose(rs, zg * zg - 1, rtol=1e-13, atol=1e-14)


@pytest.mark.parametrize("nu", [1e6, 1e9, 1e12])
def test_student_t_tends_to_the_gaussian_family(nu):
    """|student_t - gaussian_location_scale| within the O(z^4 / nu) bound: ll and dll/ds differ by at most (1 + z^4) /
    nu, dll/dmu by (1 + |z|^3) e^-s / nu, and dll/da = O(1 / nu) by (1 + z^4) / nu."""
    z = np.linspace(-6, 6, 49)
    for s in (-3.0, 0.0, 3.0):
        y = 1.0 + z * np.exp(s)
        lt, mt, st_, qt = _terms64(y, 1.0, s, np.log(nu))
        lg, mg, sg = _terms64(y, 1.0, s)
        assert np.all(np.abs(lt - lg) <= (1 + z ** 4) / nu)
        assert np.all(np.abs(mt - mg) <= (1 + np.abs(z) ** 3) * np.exp(-s) / nu)
        assert np.all(np.abs(st_ - sg) <= (1 + z ** 4) / nu)
        assert np.all(np.abs(qt) <= (1 + z ** 4) / nu)


def _scipy_truth(family, Xn, yn, wn, on, groups):
    """The log-likelihood as a function of the inputs, from scipy's logpdf."""
    from scipy import stats

    def truth(ic, beta, sic, sbeta, ld=None):
        total = 0.0
        for X, y, w, o, g in zip(Xn, yn, wn, on, groups):
            mu = X @ beta + ic[g] + o
            sig = np.exp(X @ sbeta + sic[g])
            keep = w != 0
            ll = (stats.norm(mu, sig).logpdf(y) if family != T else
                  stats.t(df=np.exp(ld[()]), loc=mu, scale=sig).logpdf(y))
            total += np.sum(w[keep] * ll[keep])
        return total

    return truth


@pytest.mark.parametrize("sic", [-5.0, 0.0, 5.0])
@pytest.mark.parametrize("family,log_nu", [("gaussian_location_scale", 0.0)] + [(T, v) for v in np.log([0.2, 1.0, 5.0, 200.0])])
def test_oracle_matches_scipy_and_finite_differences(family, log_nu, sic):
    rows, P = [90, 60], 8
    Xs, ys, ws, os_ = _case(rows, P, seed=2, nu=None if family != T else 3.0, outliers=(30.0, 1e3))
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, family=family, weights=ws, offsets=os_)
    Xn = [X.double().numpy() for X in Xs]
    yn = [y.double().numpy() for y in ys]
    wn = [w.double().numpy() if w is not None else np.ones(len(y)) for w, y in zip(ws, ys)]
    on = [o.double().numpy() if o is not None else np.zeros(len(y)) for o, y in zip(os_, ys)]
    truth = _scipy_truth(family, Xn, yn, wn, on, [0, 1])
    inputs = [np.asarray(v, dtype=np.float64) for v in _theta(family, 2, P, sic=sic, log_nu=log_nu, scale=0.2)]
    got = _oracle(model, *inputs)
    assert len(got) == len(inputs) + 1
    for g, x in zip(got[1:], inputs):
        assert np.shape(g) == np.shape(x)
    np.testing.assert_allclose(got[0], truth(*inputs), rtol=1e-11)
    eps = 1e-5
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
        np.testing.assert_allclose(grad, fd, rtol=1e-5, atol=1e-5 * (1 + np.abs(got[0])) * np.exp(-min(sic, 0)))


# ----------------------------------------------------------------------------------------------- CPU: layout
@pytest.mark.parametrize("K,G", [(1, 1), (1, 2), (3, 2)])
@pytest.mark.parametrize("family", FAMILIES)
def test_pack_unpack_and_words_round_trip(family, K, G):
    P = 8
    Xs, ys, _, _ = _case([20] * G, P, seed=7, n_masked=0, weighted=False, offsets=False)
    model = GlmShards(Xs, ys, groups=list(range(G)), n_groups=G, family=family, n_chains=K)
    inp = list(_theta(family, G, P, K, log_nu=np.arange(K) - 0.5 if K > 1 else -0.5, scale=1.0))
    if K == 1 and G == 1:
        inp[0], inp[2] = inp[0].reshape(()), inp[2].reshape(())   # scalar intercepts for one group
    t = family == T
    words = np.zeros(model.n_theta_words, dtype=np.uint32)
    ctx = model.pack_theta(inp, words)
    assert ctx == model.call_context(inp) == (K > 1, np.shape(inp[0])) + tuple(np.shape(x) for x in inp[2:])
    # the kernel's layout: rows 2k = (intercept, beta[, log_nu]), 2k + 1 = (sigma_intercept, sigma_beta[, same])
    th = words.view(np.float32).reshape(K, 2, G + P + t)
    np.testing.assert_array_equal(th[:, 0, :G], np.reshape(inp[0], (K, G)))
    np.testing.assert_array_equal(th[:, 0, G : G + P], np.reshape(inp[1], (K, P)))
    np.testing.assert_array_equal(th[:, 1, :G], np.reshape(inp[2], (K, G)))
    np.testing.assert_array_equal(th[:, 1, G : G + P], np.reshape(inp[3], (K, P)))
    if t:
        np.testing.assert_array_equal(th[:, 0, -1], np.reshape(inp[4], K))
        np.testing.assert_array_equal(th[:, 1, -1], np.reshape(inp[4], K))
    back = default_inputs_from_words(model, words)
    assert len(back) == len(inp)
    for u, v in zip(back, inp):
        assert np.array_equal(np.reshape(u, np.shape(v)), v)
    words2 = np.zeros_like(words)
    model.pack_theta(back, words2)
    assert np.array_equal(words, words2)
    # unpack: block 2k holds [LL, gi[G], g[P](, q)] of the mean, block 2k + 1 [0, gi, g(, 0)] of log sigma
    raw = np.arange(model.n_vals, dtype=np.float64).reshape(K, 2, 1 + G + P + t)
    got = model.unpack_result(raw.reshape(-1), ctx)
    assert len(got) == 1 + len(inp)
    for g, x in zip(got[1:], inp):
        assert np.shape(g) == np.shape(x)
    np.testing.assert_array_equal(np.reshape(got[0], -1), raw[:, 0, 0])
    np.testing.assert_array_equal(np.reshape(got[1], (K, G)), raw[:, 0, 1 : 1 + G])
    np.testing.assert_array_equal(np.reshape(got[2], (K, P)), raw[:, 0, 1 + G : 1 + G + P])
    np.testing.assert_array_equal(np.reshape(got[3], (K, G)), raw[:, 1, 1 : 1 + G])
    np.testing.assert_array_equal(np.reshape(got[4], (K, P)), raw[:, 1, 1 + G : 1 + G + P])
    if t:
        np.testing.assert_array_equal(np.reshape(got[5], K), raw[:, 0, -1])


@pytest.mark.parametrize("family", FAMILIES)
def test_sizes_and_flops(family):
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ys = [torch.zeros(10), torch.zeros(6)]
    t = int(family == T)
    m = GlmShards(Xs, ys, n_groups=2, groups=[0, 1], family=family, n_chains=3, node_ids=[0, 1], n_nodes=2)
    assert m.n_inputs == 4 + t and m.kernel_chains == 6
    assert m.input_shapes == [(2,), (16,), (2,), (16,)] + [()] * t
    assert m.n_params == 2 * (2 + 16) + t and m.n_theta_words == 6 * (2 + 16 + t)
    assert m.n_vals == 2 * 6 * (1 + 2 + 16 + t)
    assert m.flops_per_eval() == GlmShards(Xs, ys, n_chains=6).flops_per_eval() == 4 * 16 * 16 * 6
    assert m.bytes_per_eval() == GlmShards(Xs, ys).bytes_per_eval()
    assert m.per_node(np.zeros(m.n_vals)).shape == (2, 3, 1 + m.n_params)


def test_validation():
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ys = [torch.randn(10) * 1e30, torch.full((6,), -2.5)]
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
        for X in (torch.randn(10, 12).to(torch.bfloat16), torch.randn(10, 392).to(torch.bfloat16), torch.randn(10, 16)):
            with pytest.raises(ValueError, match="tensor-core kernel only"):
                GlmShards([X], [torch.zeros(10)], family=family).use_tensor_cores()
        assert GlmShards(Xs, ys, family=family, kernel="tc").use_tensor_cores() == 1
        for bad in (float("nan"), float("inf"), float("-inf")):
            y0 = torch.zeros(10)
            y0[4] = bad
            with pytest.raises(ValueError, match="responses of segment 0 must be finite"):
                GlmShards(Xs, [y0, ys[1]], family=family)
            w0 = torch.ones(10)
            w0[4] = 0.0
            GlmShards(Xs, [y0, ys[1]], weights=[w0, None], family=family)   # a masked row may carry anything


@pytest.mark.parametrize("family", FAMILIES)
def test_too_few_stages_refused_at_attach(family):
    from pytensor_federated_b200.ops import native

    lib = native.load()
    m = GlmShards([torch.zeros(8, 384, dtype=torch.bfloat16)], [torch.zeros(8)], n_chains=8, family=family)
    with pytest.raises(ValueError, match="fewer than two pipeline stages"):
        m.attach(lib, None)   # raises before the engine is touched
    code = 13 if family == "gaussian_location_scale" else 14
    assert lib.b200_glm_tc_stages(384, 16, 1, code, 0) < 2
    assert lib.b200_glm_tc_stages(384, 8, 1, code, 3) >= 2
    assert lib.b200_glm_tc_stages(256, 16, 1, code, 3) >= 2


@pytest.mark.parametrize("K", [1, 4])
@pytest.mark.parametrize("family", FAMILIES)
def test_collective_backend_equals_the_oracle(family, K):
    rows, P = [300, 45, 129], 24
    Xs, ys, ws, os_ = _case(rows, P, seed=6, outliers=(1e2, 1e4))
    model = GlmShards(Xs, ys, groups=[0, 1, 1], n_groups=2, family=family, n_chains=K, weights=ws, offsets=os_)
    inp = _theta(family, 2, P, K, sic=[-1.0, 0.0, 0.5, 1.0][:K] if K > 1 else -0.3,
                 log_nu=np.log([0.5, 3.0, 100.0, 1e9])[:K] if K > 1 else 1.0)
    got, want = _collective(model, *inp), _oracle(model, *inp)
    assert len(got) == len(want) == 1 + len(inp)
    for u, v in zip(got, want):
        assert np.shape(u) == np.shape(v) and np.all(np.isfinite(u))
        np.testing.assert_allclose(u, v, rtol=1e-4, atol=1e-3 * (1 + np.abs(v).max()))


@pytest.mark.parametrize("family", FAMILIES)
def test_glm_batch_fn_splits_theta_in_input_order(family):
    from pytensor_federated_b200.sampling import glm_batch_fn

    P, G = 8, 2
    Xs, ys, ws, os_ = _case([60, 40], P, seed=8, outliers=(20.0,))
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=G, family=family, n_chains=2, weights=ws, offsets=os_)
    rng = np.random.default_rng(9)
    theta = rng.normal(size=(3, model.n_params)) * 0.1
    with FederatedEngine(model, backend="collective") as eng:
        logp, grad = glm_batch_fn(eng, G)(theta)
    assert logp.shape == (3,) and grad.shape == theta.shape
    single = GlmShards(Xs, ys, groups=[0, 1], n_groups=G, family=family, weights=ws, offsets=os_)
    for i in range(3):
        # theta = [intercept[G], beta[P], sigma_intercept[G], sigma_beta[P](, log_dispersion)]
        parts = np.split(theta[i], np.cumsum([G, P, G, P])[: single.n_inputs - 1])
        want = _oracle(single, *[p if p.size > 1 else p.reshape(()) for p in parts])
        np.testing.assert_allclose(logp[i], want[0], rtol=1e-5)
        np.testing.assert_allclose(grad[i], np.concatenate([np.reshape(w, -1) for w in want[1:]]), rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("family,nu", [("gaussian_location_scale", None), (T, 5.0)])
def test_synth_location_scale_shard(family, nu):
    from scipy import stats

    n = 200_000
    X, y, beta, sbeta = synth_location_scale_shard(n, 16, family=family, nu=nu, seed=1, device="cpu", chunk_rows=65536,
                                                   beta_scale=0.0, intercept=0.7, sigma_intercept=0.4,
                                                   sigma_beta_scale=0.0)
    assert X.dtype == torch.bfloat16 and X.shape == (n, 16) and beta.shape == sbeta.shape == (16,)
    assert y.dtype == torch.float32 and bool(torch.all(torch.isfinite(y)))
    e = (y.double().numpy() - 0.7) / np.exp(0.4)
    dist = stats.norm() if nu is None else stats.t(df=nu)
    assert stats.kstest(e, dist.cdf).pvalue > 1e-3
    X2, y2, _, _ = synth_location_scale_shard(n, 16, family=family, nu=nu, seed=1, device="cpu", chunk_rows=65536,
                                              beta_scale=0.0, intercept=0.7, sigma_intercept=0.4, sigma_beta_scale=0.0)
    assert torch.equal(X, X2) and torch.equal(y, y2)
    # the scale follows x: log |y - mu| regresses on x' sigma_beta*
    X, y, beta, sbeta = synth_location_scale_shard(n, 4, family=family, nu=nu, seed=2, device="cpu", beta_scale=0.0,
                                                   intercept=0.0, sigma_beta_scale=0.5)
    lr = np.log(np.abs(y.double().numpy()))
    slope = np.linalg.lstsq(np.c_[np.ones(n), X.double().numpy()], lr, rcond=None)[0][1:]
    np.testing.assert_allclose(slope, sbeta.double().numpy(), atol=0.02)
    with pytest.raises(ValueError, match="nu > 0"):
        synth_location_scale_shard(10, 4, family=T, seed=0, device="cpu")
    with pytest.raises(ValueError, match="family must be"):
        synth_location_scale_shard(10, 4, family="gaussian", seed=0, device="cpu")


def test_student_t_map_resists_gross_outliers():
    """5 % of the rows are gross outliers along x_0.  The MAP of both families through a collective-backend engine
    (``find_map``) matches an fp64 scipy fit of the oracle, and the thresholds come from those fits: the Student-t beta
    is closer to the truth than halfway to the Gaussian fit's, which the outliers pulled."""
    import scipy.optimize

    from pytensor_federated_b200.sampling import find_map, glm_batch_fn

    n, P = 4000, 4
    rng = np.random.default_rng(11)
    X = torch.tensor(rng.normal(size=(n, P)), dtype=torch.float32).to(torch.bfloat16)
    Xd = X.double().numpy()
    beta = np.array([0.8, -0.5, 0.3, 0.0])
    y = Xd @ beta + 0.5 + 0.5 * rng.normal(size=n)
    out = rng.uniform(size=n) < 0.05
    y[out] = 20.0 + 15.0 * Xd[out, 0]
    yt = torch.tensor(y, dtype=torch.float32)
    fits = {}
    for family in FAMILIES:
        model = GlmShards([X], [yt], family=family)
        t = family == T

        def split(x):
            return [x[0], x[1 : 1 + P], x[1 + P], x[2 + P : 2 + 2 * P]] + ([x[-1]] if t else [])

        def oracle_fn(x):
            got = _oracle(model, *split(x), chunk_rows=1 << 20)
            return -float(got[0]), -np.concatenate([np.reshape(g, -1) for g in got[1:]])

        x0 = np.zeros(2 * P + 2 + t)
        if t:
            x0[-1] = np.log(4.0)
        ref = scipy.optimize.minimize(oracle_fn, x0, jac=True, method="L-BFGS-B", options={"maxiter": 2000, "gtol": 1e-9})
        with FederatedEngine(model, backend="collective") as eng:
            fn = glm_batch_fn(eng, 1)
            x_map, _ = find_map(lambda x: (lambda lp, g: (lp[0], g[0]))(*fn(x[None])), x0, maxiter=2000)
        fits[family] = (ref.x[1 : 1 + P], x_map[1 : 1 + P])
        np.testing.assert_allclose(x_map[1 : 1 + P], ref.x[1 : 1 + P], atol=2e-3)
    near = np.linalg.norm(fits[T][0] - beta)
    pulled = np.linalg.norm(fits["gaussian_location_scale"][0] - beta)
    assert pulled > 5 * near, (near, pulled)
    threshold = 0.5 * (near + pulled)
    assert np.linalg.norm(fits[T][1] - beta) < threshold < np.linalg.norm(fits["gaussian_location_scale"][1] - beta)


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


def _row_terms(family, y, mu, s, a):
    """fp64 per-row terms ``[n, K]`` each: ll, dll/dmu, dll/ds and (Student-t) dll/da."""
    out = _location_scale_terms(y, mu, s, a if family == T else None)
    res = [out[0][..., 0], out[1][..., 0], out[1][..., 1]]
    return res + ([out[2][..., 0]] if family == T else [torch.zeros_like(res[0])])


def _magnitudes(family, y, mu, s, a):
    """Per row, the sizes of the values each output is formed from (ll, dll/da), for the rounding part of the bound."""
    z = (y - mu) * torch.exp(-s)
    if family != T:
        return 0.5 * z * z + 1.0 + s.abs(), torch.zeros_like(z)
    nu, Cn, Q = (v.to(z.dtype) for v in _student_t_constants(a))
    L = torch.log1p(z * z / nu)
    return Cn.abs() + s.abs() + 0.5 * (nu + 1) * L + 1.0, Q.abs() + 0.5 * nu * L + 1.0


def _bound(model, ic, beta, sic, sbeta, ld=None):
    """A bound on the kernel's error, per output and in the shapes of the results, from the fp64 magnitudes of the
    terms each one sums.  Per row, the mean and the log scale are each off by at most ``d = 2^-18 (1 + |eta| + sum_j |x_j
    theta_j|)`` (the three-term bf16 split of theta keeps 24 bits, the fp32 MMA sums over P): its effect is the largest
    change of the fp64 terms over the corners ``(mu +- d_mu, s +- d_s)``.  The kernel's own ll and q are off by
    ``2^-16`` of the magnitudes they are formed from (a few fp32 roundings, then per-thread fp32 sums of at most 64
    rows), its gradients by ``2^-14 |r|`` (the (hi, lo) bf16 split of r, then fp32 MMA sums), times ``|x|`` for beta."""
    fam = model.family
    batched = np.ndim(beta) == 2
    K, G, P = model.n_chains, model.n_groups, model.n_features
    dv = model.device
    f64 = lambda v, shape: torch.tensor(np.reshape(v, shape), dtype=torch.float64, device=dv)
    icd, bd, sicd, sbd = f64(ic, (K, G)), f64(beta, (K, P)), f64(sic, (K, G)), f64(sbeta, (K, P))
    ad = f64(ld, (K,)) if ld is not None else None
    t_ll = torch.zeros(K, dtype=torch.float64, device=dv)
    t_q = torch.zeros_like(t_ll)
    t_gi = [torch.zeros(K, G, dtype=torch.float64, device=dv) for _ in range(2)]
    t_g = [torch.zeros(K, P, dtype=torch.float64, device=dv) for _ in range(2)]
    for si, (X, y, g) in enumerate(zip(model.Xs, model.ys, model.groups)):
        w = model.weights[si]
        keep = torch.ones_like(y, dtype=torch.bool) if w is None else w != 0
        ww = (torch.ones_like(y) if w is None else w).double()[keep].unsqueeze(1)
        Xd = X.double()[keep]
        yy = y.double()[keep].unsqueeze(1)
        mu = Xd @ bd.T + icd[:, g]
        if model.offsets[si] is not None:
            mu = mu + model.offsets[si].double()[keep].unsqueeze(1)
        s = Xd @ sbd.T + sicd[:, g]
        d_mu = 2.0 ** -18 * (1.0 + mu.abs() + Xd.abs() @ bd.abs().T)
        d_s = 2.0 ** -18 * (1.0 + s.abs() + Xd.abs() @ sbd.abs().T)
        base = _row_terms(fam, yy, mu, s, ad)
        dev_ = [torch.zeros_like(b) for b in base]
        for sm in (-1.0, 1.0):
            for ss in (-1.0, 1.0):
                for i, (b, c) in enumerate(zip(base, _row_terms(fam, yy, mu + sm * d_mu, s + ss * d_s, ad))):
                    dev_[i] = torch.maximum(dev_[i], (c - b).abs())
        m_ll, m_q = _magnitudes(fam, yy, mu, s, ad)
        t_ll += (ww * (2.0 ** -16 * m_ll + dev_[0])).sum(0)
        t_q += (ww * (2.0 ** -16 * m_q + dev_[3])).sum(0)
        for j in range(2):
            e = ww * (2.0 ** -14 * base[1 + j].abs() + dev_[1 + j])
            t_gi[j][:, g] += e.sum(0)
            t_g[j] += e.T @ Xd.abs()
    out = [t.cpu().numpy() for t in (t_ll, t_gi[0], t_g[0], t_gi[1], t_g[1])]
    if fam == T:
        out.append(t_q.cpu().numpy())
    return out if batched else [o[0] for o in out]


def _check(got, want, tol):
    assert all(np.all(np.isfinite(g)) for g in got)
    assert len(got) == len(want) == len(tol)
    for i, (u, v, t) in enumerate(zip(got, want, tol)):
        assert np.shape(u) == np.shape(v)
        err = np.abs(np.asarray(u, dtype=np.float64) - v)
        assert np.all(err <= t), (i, np.max(err / t), np.max(err))


@pytest.mark.parametrize("row_data", [True, False])
@pytest.mark.parametrize("K", [1, 2, 3, 4, 5, 8])
@pytest.mark.parametrize("P", [256, 200, 8])
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_matches_oracle(dev, family, P, K, row_data):
    """K pairs run 2K columns: K <= 2, <= 4 and <= 8 select the kernel's 4, 8 and 16 buckets; ``row_data`` (offsets
    and weights, masked rows with NaN / +-inf responses) its ROWS variant.  Every segment holds outliers up to 1e8
    (Student-t: 1e30); the chains cycle through the sigma intercepts (-5 .. 5) and nu (0.2 .. 1e12)."""
    rows = [128 * 37, 77, 4099, 1]
    outliers = (1e2, 1e4, 1e8) + ((1e30,) if family == T else ())
    Xs, ys, ws, os_ = _case(rows, P, seed=K + P, device=dev, weighted=row_data, offsets=row_data,
                            n_masked=5 if row_data else 0, outliers=outliers)
    model = GlmShards(Xs, ys, groups=[0, 1, 0, 1], n_groups=2, family=family, n_chains=K, kernel="auto",
                      weights=ws, offsets=os_)
    assert model.has_row_data == row_data
    if K == 1:
        inputs = [_theta(family, 2, P, 1, sic=v, log_nu=a, seed=5 + i)
                  for i, (v, a) in enumerate(zip(SIGMA_ICPT, LOG_NU[[0, 2, 4, 6, 7]]))]
    else:
        inputs = [_theta(family, 2, P, K, sic=np.resize(SIGMA_ICPT, K), log_nu=np.resize(LOG_NU, K))]
    got = _run(model, inputs)
    assert model.selected_kernel == "tc"
    for g, inp in zip(got, inputs):
        _check(g, _oracle(model, *inp, chunk_rows=1 << 20), _bound(model, *inp))


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("K,row_data", [(1, False), (2, True), (5, False), (5, True)])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_with_many_groups_matches_oracle(dev, family, K, row_data):
    """300 intercepts per predictor: the intercept table is KC x G floats, both predictors' rows of it in use."""
    G, P = 300, 256
    rows = [128 * 9 + 5, 999, 64, 1, 3000]
    groups = [0, 299, 150, 7, 299]
    Xs, ys, ws, os_ = _case(rows, P, seed=40 + K, device=dev, weighted=row_data, offsets=row_data,
                            n_masked=5 if row_data else 0)
    model = GlmShards(Xs, ys, groups=groups, n_groups=G, family=family, n_chains=K, kernel="tc", weights=ws,
                      offsets=os_)
    inp = _theta(family, G, P, K, sic=np.resize(SIGMA_ICPT[::-1], K) if K > 1 else 0.5,
                 log_nu=np.resize(LOG_NU[::-1], K) if K > 1 else LOG_NU[0])
    (got,) = _run(model, [inp])
    _check(got, _oracle(model, *inp, chunk_rows=1 << 20), _bound(model, *inp))
    unused = np.ones(G, dtype=bool)
    unused[groups] = False
    assert np.all(got[1][..., unused] == 0.0) and np.all(got[3][..., unused] == 0.0)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_student_t_per_row_values_across_the_domain(dev):
    """The kernel's ll, dll/dmu, dll/ds and dll/da of single rows (one output block each), for 8 chains at nu = 0.2 ..
    1e12 (one launch, 16 columns), s in {-5, 0, 5} and z from 0 to +-1e30: each finite and within 2^-16 of the
    magnitudes it is formed from plus its slope times the rounding of z.  mu and s are exact in the kernel (x = e_0,
    beta = 0, so they are the intercepts)."""
    P, K = 8, 8
    zs = _z_grid()
    pts = [(s, z) for s in (-5.0, 0.0, 5.0) for z in zs]
    mu0 = 0.3
    ys = np.array([mu0 + z * np.exp(s) for s, z in pts], dtype=np.float32)
    svals = np.array([p[0] for p in pts], dtype=np.float32)
    n = len(ys)
    X = torch.zeros(n, P, dtype=torch.bfloat16, device=dev)
    X[:, 0] = 1.0
    Xs = [X[i : i + 1].clone() for i in range(n)]
    yl = [torch.tensor(ys[i : i + 1], device=dev) for i in range(n)]
    model = GlmShards(Xs, yl, groups=list(range(n)), n_groups=n, family=T, n_chains=K, kernel="tc",
                      node_ids=list(range(n)), n_nodes=n)
    a = LOG_NU.astype(np.float32)
    inp = (np.full((K, n), mu0, np.float32), np.zeros((K, P), np.float32), np.broadcast_to(svals, (K, n)).copy(),
           np.zeros((K, P), np.float32), a)
    with FederatedEngine(model) as eng:
        blocks = model.per_node(eng.evaluate_raw(list(inp)))   # [n, K, 1 + 2 (n + P) + 1]
    assert np.all(np.isfinite(blocks))
    idx = np.arange(n)
    ll, rm, rs, qa = blocks[idx, :, 0], blocks[idx, :, 1 + idx], blocks[idx, :, 1 + n + P + idx], blocks[:, :, -1]
    y64 = torch.tensor(ys, dtype=torch.float64).unsqueeze(1)
    s64 = torch.tensor(svals, dtype=torch.float64).unsqueeze(1)
    mu = torch.full_like(y64, float(np.float32(mu0)))
    a64 = torch.tensor(a, dtype=torch.float64)
    want = [t.numpy() for t in _row_terms(T, y64, mu, s64, a64)]
    m_ll, m_q = (t.numpy() for t in _magnitudes(T, y64, mu, s64, a64))
    z = ((y64 - mu) * torch.exp(-s64)).numpy()
    dz = 2.0 ** -21 * (np.abs(z) + np.exp(-svals.astype(np.float64))[:, None] * (abs(mu0) + 1))   # y - mu, e^-s roundings
    # |d value / dz| <= (|value| + 2) (1 + 1 / |z|) covers z ll' = -(nu + 1) q / (1 + q), z rm' and z rs' at every z
    slope = lambda w: (np.abs(w) + 2.0 + np.abs(want[1]) * np.exp(svals)[:, None]) / np.maximum(np.abs(z), 1e-30)
    checks = {"ll": (ll, want[0], m_ll), "dmu": (rm, want[1], np.abs(want[1])), "ds": (rs, want[2], np.abs(want[2]) + 1),
              "da": (qa, want[3], m_q)}
    for name, (g, w, mag) in checks.items():
        tol = 2.0 ** -16 * mag + slope(w) * dz * (np.abs(want[1]) * np.exp(svals)[:, None] + np.abs(w) + 1)
        assert np.all(np.abs(g - w) <= tol), (name, np.max(np.abs(g - w) / tol))
    # bounded influence: dll/dmu falls as 1 / z, from |z| = 1e6 (grid entry 9) to 1e30 (entries 13 and 26)
    nz = len(zs)
    for b0 in range(0, n, nz):
        assert np.all(np.abs(rm[b0 + 13]) < 1e-20 * np.abs(rm[b0 + 9]))
        assert np.all(np.abs(rm[b0 + 26]) < 1e-20 * np.abs(rm[b0 + 9]))


@pytest.mark.parametrize("row_data", [False, True])
@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_unit_scale_is_bit_identical_to_the_gaussian_family(dev, K, row_data):
    """sigma_intercept = 0 and sigma_beta = 0: s is exactly 0 and e^-s exactly 1, so the mean columns of a K-pair
    gaussian_location_scale launch are the even blocks of a 2K-chain gaussian launch (same bucket, same column positions,
    same theta rows)."""
    rows, P = [128 * 30 + 9, 5000, 77], 256
    Xs, ys, ws, os_ = _case(rows, P, seed=11 + K, device=dev, weighted=row_data, offsets=row_data,
                            n_masked=5 if row_data else 0, nu=None)
    ls = GlmShards(Xs, ys, groups=[0, 1, 0], n_groups=2, family="gaussian_location_scale", n_chains=K, kernel="tc",
                   weights=ws, offsets=os_)
    base = GlmShards(Xs, ys, groups=[0, 1, 0], n_groups=2, family="gaussian", n_chains=2 * K, kernel="tc",
                     weights=ws, offsets=os_)
    inp = list(_theta("gaussian_location_scale", 2, P, K))
    inp[2] = np.zeros_like(inp[2])
    inp[3] = np.zeros_like(inp[3])
    lead = lambda x: np.reshape(x, (K, -1))
    b_ic = np.stack([lead(inp[0]), lead(inp[2])], axis=1).reshape(2 * K, 2)
    b_bt = np.stack([lead(inp[1]), lead(inp[3])], axis=1).reshape(2 * K, P)
    (a,), (b,) = _run(ls, [inp], raw=True), _run(base, [[b_ic, b_bt]], raw=True)
    width = 1 + 2 + P
    a, b = a.reshape(2 * K, width), b.reshape(2 * K, width)
    assert np.all(np.isfinite(a))
    assert a[0::2].tobytes() == b[0::2].tobytes()
    assert np.all(a[1::2, 0] == 0.0)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_evaluations_are_bit_reproducible(dev, family):
    rows = [40_000, 25_000, 33_333, 128, 19_999]
    Xs, ys, ws, os_ = _case(rows, 256, seed=12, device=dev)
    model = GlmShards(Xs, ys, groups=[0, 1, 2, 1, 0], n_groups=3, family=family, n_chains=4, kernel="tc",
                      weights=ws, offsets=os_)
    inp = _theta(family, 3, 256, 4, sic=SIGMA_ICPT[:4], log_nu=LOG_NU[:4])
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
    Xs, ys, ws, os_ = _case([3 * 128 + 5, 1000, 128], P, seed=21 + K, device=dev, weighted=rows_data,
                            offsets=rows_data, n_masked=5 if rows_data else 0)
    inp = _theta(family, 1, P, K, sic=np.resize(SIGMA_ICPT, K) if K > 1 else 0.0,
                 log_nu=np.resize(LOG_NU, K) if K > 1 else 1.0)
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
    Xs, ys, ws, os_ = _case(rows, 256, seed=13, device=dev)
    model = GlmShards(Xs, ys, groups=groups, n_groups=2, family=family, kernel="tc", node_ids=node_ids, n_nodes=2,
                      weights=ws, offsets=os_)
    inp = _theta(family, 2, 256, sic=-0.3, log_nu=0.7)
    with FederatedEngine(model) as eng:
        n0 = eng.kernel_launches
        blocks = model.per_node(eng.evaluate_raw(list(inp)))
        assert eng.kernel_launches - n0 == 1
        assert blocks.shape == (2, 1, 1 + model.n_params)
        fed = NodeFederation(eng)
        res = fed.evaluate_nodes({0: inp, 1: inp})
        total = fed.all_nodes_func()(*inp)
    for node in (0, 1):
        segs = [i for i, n in enumerate(node_ids) if n == node]
        single = GlmShards([Xs[i] for i in segs], [ys[i] for i in segs], groups=[groups[i] for i in segs], n_groups=2,
                           family=family, kernel="tc", weights=[ws[i] for i in segs], offsets=[os_[i] for i in segs])
        # the node's block and the single-node model's evaluation, each within the bound of the same oracle
        (one,) = _run(single, [inp])
        want, tol = _oracle(single, *inp, chunk_rows=1 << 20), _bound(single, *inp)
        _check(one, want, tol)
        _check(single.gradients_from_row(blocks[node, 0], [None] * len(inp)), want[1:], tol[1:])
        assert abs(blocks[node, 0, 0] - want[0]) <= tol[0]
        np.testing.assert_allclose(res[node][0], blocks[node, 0, 0], rtol=1e-12)
        assert len(res[node][1]) == len(inp)
        for g, x in zip(res[node][1], inp):
            assert np.shape(g) == np.shape(x)
        np.testing.assert_allclose(np.concatenate([np.reshape(g, -1) for g in res[node][1]]), blocks[node, 0, 1:],
                                   rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(total[0], blocks[:, 0, 0].sum(), rtol=1e-12)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_lock_step_hmc_on_a_student_t_engine(dev):
    from pytensor_federated_b200.sampling import glm_batch_fn, hmc_sample_batched

    K, P = 4, 16
    X, y, _, _ = synth_location_scale_shard(20_000, P, family=T, nu=4.0, seed=3, device=dev)
    model = GlmShards([X], [y], family=T, n_chains=K, kernel="tc")
    x0 = np.zeros((K, model.n_params))
    x0[:, 0] = 0.5             # intercept
    x0[:, -1] = np.log(4.0)    # log_dispersion
    with FederatedEngine(model) as eng:
        res = hmc_sample_batched(glm_batch_fn(eng, 1), x0, draws=5, tune=5, n_leapfrog=4, step_size=1e-3, seed=1)
        assert eng.n_evals == res.n_batched_evals
    assert res.samples.shape[-1] == model.n_params and np.all(np.isfinite(res.samples))
    assert np.all(res.accept_rate > 0)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_runtime_rejects_the_location_scale_families_outside_their_launch(dev):
    """The C ABI refuses what the Python layer never sends: codes 13 and 14 on a CUDA-core kernel, an odd n_chains,
    n_classes != 1, an output size that does not match and the Hessian-vector-product flag, and the engine keeps
    evaluating its own model."""
    from pytensor_federated_b200.ops import native

    Xs, ys, _, _ = _case([256], 16, seed=14, device=dev, n_masked=0, weighted=False, offsets=False)
    model = GlmShards(Xs, ys, kernel="simt", family="gaussian")
    with FederatedEngine(model) as eng:
        lib, h = eng._lib, eng._handle
        Xp, yp = native.void_p_array([Xs[0].data_ptr()]), native.void_p_array([ys[0].data_ptr()])
        rows, grp = (C.c_longlong * 1)(256), (C.c_int * 1)(0)

        def set_glm(n_chains, family, code, n_classes=1):
            return int(lib.b200_engine_set_glm(h, 1, Xp, yp, None, rows, grp, 16, 16, 1, n_chains, family, code, None, 1,
                                               None, None, n_classes))

        for family, name, refused in ((13, "gaussian_location_scale", -34), (14, "student_t", -39)):
            for code in (0, 2, 3, 4):
                assert set_glm(2, family, code) == refused
                assert f"the {name} family runs on the bf16 tensor-core kernel only" in native.last_error()
            assert set_glm(2, family, 1, 2) == -38 and "n_classes must be 1" in native.last_error()
            for n_chains in (1, 3, 18):
                assert set_glm(n_chains, family, 1) == -44 and "even n_chains in [2, 16]" in native.last_error()
            # this engine's n_vals is 1 + G + P: a 2-column launch needs twice that (plus the dispersion words)
            assert set_glm(2, family, 1) == -33 and "n_vals does not match" in native.last_error()
            assert set_glm(2, family | 16, 1) != 0   # no Hessian-vector products of these families
        ic, beta = np.float32(0.1), np.zeros(16, np.float32)
        got = eng.evaluate(ic, beta)
    want = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)


def _build_student_t_model(rank, world, dev):
    Xs, ys, ws, os_ = _case([30_000 + 17 * rank, 999], 256, seed=50 + rank, device=dev)
    return GlmShards(Xs, ys, groups=[rank % 2, 1 - rank % 2], n_groups=2, family=T, n_chains=2, kernel="tc",
                     weights=ws, offsets=os_)


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.timeout(900)
def test_two_rank_student_t_federation_matches_oracle():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from pytensor_federated_b200.federation import launch_federation

    inp = _theta(T, 2, 256, 2, sic=[-1.0, 0.5], log_nu=np.log([2.0, 50.0]))
    dev = torch.device("cuda:0")
    models = [_build_student_t_model(r, 2, dev) for r in range(2)]
    want = models[0].unpack_result(sum(m.reference_partial(list(inp), dtype=torch.float64) for m in models),
                                   models[0].call_context(list(inp)))
    tol = [sum(v) for v in zip(*(_bound(m, *inp) for m in models))]
    del models
    with launch_federation(_build_student_t_model, 2, timeout=30.0) as eng:
        got = eng.evaluate(*inp)
    _check(got, want, tol)
