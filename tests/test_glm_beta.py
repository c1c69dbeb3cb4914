"""Beta regression for proportions in (0, 1): ``GlmShards(Xs, ys, family="beta")``, logit link to the mean,
``log_dispersion`` = the log of the precision phi.

CPU tests check the fp64 oracle against 60-digit mpmath and against scipy (its density and central differences of
it), an fp32 emulation of the kernel's per-row code against the per-row bound of the GPU domain sweep (and two naive
variants against the same bound, which they must break), the collective backend, ``NodeFederation``, validation, the
model's packing and the synthetic data.  GPU tests check the tensor-core kernel against the oracle within a rounding
bound derived from the magnitudes of each sum's terms, per row across the family's domain, bit for bit against itself,
and a MAP fit end to end."""
import ctypes as C

import numpy as np
import pytest
import torch

from pytensor_federated_b200.models import Fp8GlmShards, GlmShards, synth_beta_shard
from pytensor_federated_b200.models.glm import FAMILIES as CODES
from pytensor_federated_b200.models.glm import _DISPERSION_TERMS, _beta_constants, _beta_tails
from pytensor_federated_b200.parallel import FederatedEngine
from pytensor_federated_b200.parallel.engine import default_inputs_from_words

FAMILY = "beta"
TERMS = _DISPERSION_TERMS[FAMILY]
# log precision of the GPU tests: phi from 0.05 to 1e6
LOG_PHI = np.log([0.05, 0.3, 1.0, 3.0, 8.0, 30.0, 300.0, 1e4, 1e6])
# the (eta, y, a) domain: a from -5 to 14 (phi 0.0067 to 1.2e6), eta from -30 to 30, y from 1e-6 to 1 - 2^-24
DOMAIN_A = np.array([-5.0, -2.0, 0.0, 1.0, np.log(8.0), 3.0, 5.0, 7.0, np.log(1e4), 11.0, 14.0])
Y_MAX = 1.0 - 2.0 ** -24


# ----------------------------------------------------------------------------------------------- fixtures
def _beta_true(P):
    return np.random.default_rng(1000 + P).normal(size=P) * 0.01


def _case(rows, P, *, seed=0, device="cpu", n_masked=5, weighted=True, offsets=True, phi=20.0, icpt=(0.4, -1.0)):
    """Ragged bf16 segments with responses drawn from Beta(mu phi, (1 - mu) phi) at ``intercept = icpt[segment %
    2]`` and ``beta = _beta_true(P)``, clipped into (0, 1) in float32.  With ``weighted``, every segment but the last
    has weights; the first ``n_masked`` rows of segment 0 have weight 0 and carry NaN, 0, 1, a negative and an
    infinite y.  With ``offsets``, every segment but the second has offsets.  Returns ``(Xs, ys, weights, offsets)``."""
    rng = np.random.default_rng(seed)
    Xs, ys, ws, os_ = [], [], [], []
    for si, n in enumerate(rows):
        X = torch.tensor(rng.normal(size=(n, P)), dtype=torch.float32).to(torch.bfloat16)
        o = rng.uniform(-0.5, 0.5, size=n)
        eta = X.double().numpy() @ _beta_true(P) + icpt[si % 2] + (o if offsets else 0.0)
        mu = 1.0 / (1.0 + np.exp(-eta))
        y = np.clip(rng.beta(mu * phi, (1.0 - mu) * phi), 1e-30, Y_MAX)
        w = rng.uniform(0.2, 2.0, size=n)
        if si == 0 and n_masked:
            w[:n_masked] = 0.0
            y[:5] = [np.nan, 0.0, 1.0, -0.5, np.inf][: min(5, n_masked)]
        Xs.append(X.to(device))
        ys.append(torch.tensor(y, dtype=torch.float32, device=device))
        ws.append(torch.tensor(w, dtype=torch.float32, device=device) if weighted and si < len(rows) - 1 else None)
        os_.append(torch.tensor(o, dtype=torch.float32, device=device) if offsets and si != 1 else None)
    return Xs, ys, ws, os_


def _theta(G, P, K=1, log_phi=np.log(20.0), seed=3, scale=0.002):
    """``(intercept, beta, log_phi)`` near the parameters the data were drawn at; batched (``[K, G]``, ``[K, P]``,
    ``[K]``) for K > 1, where ``log_phi`` may give one value per chain."""
    rng = np.random.default_rng(seed)
    b0 = _beta_true(P)
    base = np.resize([0.4, -1.0], G)
    if K == 1:
        return ((base + rng.normal(size=G) * 0.02).astype(np.float32),
                (b0 + rng.normal(size=P) * scale).astype(np.float32), np.float32(log_phi))
    return ((base + rng.normal(size=(K, G)) * 0.02).astype(np.float32),
            (b0 + rng.normal(size=(K, P)) * scale).astype(np.float32),
            np.broadcast_to(np.asarray(log_phi, dtype=np.float32), (K,)).copy())


def _model(Xs, ys, ws, os_, **kw):
    return GlmShards(Xs, ys, family=FAMILY, weights=ws, offsets=os_, **kw)


def _oracle(model, *inputs, chunk_rows=128):
    return model.unpack_result(model.reference_partial(list(inputs), dtype=torch.float64, chunk_rows=chunk_rows))


def _collective(model, *inputs):
    with FederatedEngine(model, backend="collective") as eng:
        return [np.asarray(v, dtype=np.float64) for v in eng.evaluate(*inputs)]


def _t64(v):
    return torch.as_tensor(np.asarray(v, dtype=np.float64))


def _terms64(y, eta, a):
    """The fp64 oracle's ``(ll, r, q)`` as numpy arrays, ``y`` and ``eta`` ``[n]``, ``a`` ``[K]`` -> ``[n, K]``."""
    return [t.numpy() for t in TERMS(_t64(y)[:, None], _t64(eta)[:, None], _t64(a))]


def _parts(y, eta, a):
    """Per row and chain, the fp64 magnitudes of the terms the grouped form adds to make ll, r and q (the shifts below
    z = 8 included), ``[n, K]`` each: what a relative rounding error of the parts makes of each value."""
    y, eta, a = _t64(y)[:, None], _t64(eta)[:, None], _t64(a)
    phi, Cp, Qp = _beta_constants(a)
    ly, l1y = torch.log(y).abs(), torch.log1p(-y).abs()
    lmu, l1mu = -torch.nn.functional.softplus(-eta), -torch.nn.functional.softplus(eta)
    mu, nmu = torch.sigmoid(eta), torch.sigmoid(-eta)
    lA, lB = lmu + a, l1mu + a
    A, B = torch.exp(lA), torch.exp(lB)
    d = y - mu
    su, sv = (d / mu).abs() < 0.5, (d / nmu).abs() < 0.5
    D = torch.log(y / mu).abs() + torch.log((1 - y) / nmu).abs()   # |log1p(u)| + |log1p(v)|
    kl_u = A * torch.log(y / mu).abs()
    kl_v = B * torch.log((1 - y) / nmu).abs()
    # the log-ratio branch takes log1p(u) as log y - log mu: its parts are the two logs (times A where A multiplies)
    lr_u = torch.where(su, torch.zeros_like(A), ly + lmu.abs())
    lr_v = torch.where(sv, torch.zeros_like(B), l1y + l1mu.abs())
    SA, tA = _beta_tails(A, lA)
    SB, tB = _beta_tails(B, lB)

    def shift(z, lz):   # the recurrence's terms below z = 8: (z' - 1/2) log z', (z + 1/2) log z, m, the product's log
        return torch.where(z < 8.0, 45.0 + (z + 0.5) * lz.abs(), torch.zeros_like(z)), \
            torch.where(z < 8.0, 1.0 + z * (3.0 + lz.abs() + 2.0), torch.zeros_like(z))

    shA, stA = shift(A, lA)
    shB, stB = shift(B, lB)
    kl = phi * d.abs() + kl_u + kl_v + A * lr_u + B * lr_v
    ll = Cp.abs() + lmu.abs() + l1mu.abs() + ly + l1y + kl + SA.abs() + SB.abs() + shA + shB
    r = A * nmu * (D + lr_u + lr_v) + nmu * (tA.abs() + stA) + mu * (tB.abs() + stB)
    q = Qp.abs() + kl + tA.abs() + tB.abs() + stA + stB
    return ll.numpy(), r.numpy(), q.numpy()


def _slopes(y, eta, a):
    """|d/deta| of the oracle's ll, r and q per row and chain (central differences in fp64)."""
    h = 1e-5 * np.maximum(1.0, np.abs(eta))
    up, dn = _terms64(y, eta + h, a), _terms64(y, eta - h, a)
    return [np.abs(u - v) / (2 * h[:, None]) for u, v in zip(up, dn)]


# ----------------------------------------------------------------------------------------------- the domain
def _domain_rows(a=DOMAIN_A):
    """(eta, y) rows of the domain sweep, float32: eta on a grid from -30 to 30 plus the etas at which A = mu phi or
    B = (1 - mu) phi is just below and above the shift threshold 8 for one of the chains ``a``; y on a grid from 1e-6
    to 1 - 2^-24, y within 1, 2 and 4 ulp of mu, and y at relative distances 1e-4 .. 0.6 of mu on both sides (across
    the series switch of the relative differences at 1/2)."""
    etas = [-30.0, -20.0, -10.0, -5.0, -2.0, -0.7, 0.0, 0.3, 2.0, 5.0, 10.0, 20.0, 30.0]
    for phi in np.exp(a):
        if phi > 16:
            for z in (7.9, 8.1):
                etas += [np.log(z / (phi - z)), -np.log(z / (phi - z))]   # A = z, B = z
    grid = [1e-6, 1e-4, 0.01, 0.1, 0.3, 0.5, 0.7, 0.9, 0.99, 1 - 1e-4, Y_MAX]
    rows = []
    for e in np.float32(etas):
        mu = np.float32(1.0 / (1.0 + np.exp(-np.float64(e))))
        near = [mu]
        for k in (1, 2, 4):
            near += [np.nextafter(mu, np.float32(0)), np.nextafter(mu, np.float32(1))]
            for _ in range(k - 1):
                near[-2], near[-1] = np.nextafter(near[-2], np.float32(0)), np.nextafter(near[-1], np.float32(1))
        rel = [mu * (1 + s * t) for t in (1e-4, 1e-3, 0.01, 0.1, 0.3, 0.49, 0.51, 0.6) for s in (1, -1)]
        for y in grid + near + rel:
            y32 = np.float32(np.clip(np.float64(y), 1e-6, Y_MAX))
            if 0 < y32 < 1:
                rows.append((e, y32))
    rows = sorted(set(rows))
    return np.array([r[0] for r in rows], np.float32), np.array([r[1] for r in rows], np.float32)


# ----------------------------------------------------------------------------------------------- CPU: the oracle
def _mp_terms(y, eta, a):
    """ll, r and q at 60 digits from lgamma and digamma (the ungrouped closed forms)."""
    import mpmath

    with mpmath.workdps(60):
        y, eta, a = mpmath.mpf(float(y)), mpmath.mpf(float(eta)), mpmath.mpf(float(a))
        phi = mpmath.exp(a)
        mu = 1 / (1 + mpmath.exp(-eta))
        nmu = 1 / (1 + mpmath.exp(eta))
        A, B = mu * phi, nmu * phi
        ly, l1y = mpmath.log(y), mpmath.log(1 - y)
        ll = mpmath.loggamma(phi) - mpmath.loggamma(A) - mpmath.loggamma(B) + (A - 1) * ly + (B - 1) * l1y
        r = phi * mu * nmu * (mpmath.digamma(B) - mpmath.digamma(A) + ly - l1y)
        q = phi * (mpmath.digamma(phi) - mu * mpmath.digamma(A) - nmu * mpmath.digamma(B) + mu * ly + nmu * l1y)
        return float(ll), float(r), float(q)


def test_oracle_matches_mpmath_over_the_domain():
    """The fp64 oracle's ll, r and q agree with 60-digit mpmath to 1e-8 of the sum of the magnitudes of their grouped
    terms, on a from -5 to 14, eta from -30 to 30 and y from 1e-6 to 1 - 2^-24, y within a few ulp of mu, A or B below
    1e-6 and near the shift threshold 8."""
    a = DOMAIN_A[::2].copy()
    etas, ys = _domain_rows(a)
    rng = np.random.default_rng(0)
    pick = rng.choice(len(ys), size=min(len(ys), 140), replace=False)
    etas, ys = etas[pick], ys[pick]
    got = _terms64(ys, etas, a)
    parts = _parts(ys, etas, a)
    n_small = 0
    for i in range(len(ys)):
        for k in range(len(a)):
            want = _mp_terms(ys[i], etas[i], a[k])
            A = np.exp(a[k]) / (1 + np.exp(-np.float64(etas[i])))
            n_small += A < 1e-6
            for g, w, p in zip(got, want, parts):
                assert abs(g[i, k] - w) <= 1e-8 * p[i, k], (ys[i], etas[i], a[k], g[i, k], w, p[i, k])
    assert n_small > 0


def test_constants_and_tails_match_mpmath():
    """C(phi), Q(phi) and the per-row S and z tau(z) against mpmath, on both sides of the series switch at 8."""
    import mpmath

    a = np.log([0.0067, 0.05, 1.0, 7.999999, 8.0, 8.000001, 50.0, 1e3, 1.2e6])
    phi, Cp, Qp = (t.numpy() for t in _beta_constants(_t64(a)))
    for i, ph in enumerate(phi):
        with mpmath.workdps(60):
            z = mpmath.mpf(float(ph))
            S = mpmath.loggamma(z) - ((z - 0.5) * mpmath.log(z) - z + 0.5 * mpmath.log(2 * mpmath.pi))
            Cw = float(0.5 * (mpmath.log(z) - mpmath.log(2 * mpmath.pi)) + S)
            Qw = float(z * (mpmath.digamma(z) - mpmath.log(z)))
        assert abs(Cp[i] - Cw) <= 1e-13 * max(1.0, abs(Cw)) and abs(Qp[i] - Qw) <= 1e-13 * max(1.0, abs(Qw))
    assert abs(Qp[-1] + 0.5) < 1e-7


@pytest.mark.parametrize("log_phi", [-3.0, 0.0, 2.0, 4.0])
def test_oracle_matches_scipy_and_finite_differences(log_phi):
    """Three groups at mu ~ 0.01, 0.5 and 0.99, offsets, weights with masked NaN / 0 / 1 rows, and two nodes: each
    node's LL is the weighted sum of scipy's beta logpdf, and its gradients are central differences of it."""
    import scipy.stats

    P, G = 8, 3
    rows, groups, node_ids = [60, 45, 50, 33], [0, 1, 2, 1], [0, 1, 1, 0]
    rng = np.random.default_rng(int(log_phi * 10) + 100)
    ic = np.array([-4.6, 0.0, 4.6]) + rng.normal(size=G) * 0.1
    beta = rng.normal(size=P) * 0.1
    phi = np.exp(log_phi)
    Xs, ys, ws, os_ = [], [], [], []
    for si, n in enumerate(rows):
        X = torch.tensor(rng.normal(size=(n, P)), dtype=torch.float32).to(torch.bfloat16)
        o = rng.uniform(-0.3, 0.3, size=n)
        mu = 1 / (1 + np.exp(-(X.double().numpy() @ beta + ic[groups[si]] + o)))
        y = np.clip(rng.beta(mu * phi, (1 - mu) * phi), 1e-6, Y_MAX)
        w = rng.uniform(0.2, 2.0, size=n)
        if si == 0:
            w[:3] = 0.0
            y[:3] = [np.nan, 0.0, 1.0]
        Xs.append(X)
        ys.append(torch.tensor(y, dtype=torch.float32))
        ws.append(torch.tensor(w, dtype=torch.float32))
        os_.append(torch.tensor(o, dtype=torch.float32))
    model = GlmShards(Xs, ys, groups=groups, n_groups=G, family=FAMILY, weights=ws, offsets=os_, node_ids=node_ids,
                      n_nodes=2)
    Xn, yn, wn, on = ([t.double().numpy() for t in v] for v in (Xs, ys, ws, os_))

    def truth(ic, beta, lp, node):
        total = 0.0
        for si in range(len(rows)):
            if node_ids[si] != node:
                continue
            keep = wn[si] != 0
            mu = 1 / (1 + np.exp(-(Xn[si] @ beta + ic[groups[si]] + on[si])))[keep]
            ph = np.exp(lp[()])
            total += np.sum(wn[si][keep] * scipy.stats.beta(a=mu * ph, b=(1 - mu) * ph).logpdf(yn[si][keep]))
        return total

    lp = np.asarray(log_phi)
    blocks = model.per_node(model.reference_partial([ic, beta, lp], dtype=torch.float64, chunk_rows=128))
    assert blocks.shape == (2, 1, 2 + G + P)
    for node in (0, 1):
        got = blocks[node, 0]
        np.testing.assert_allclose(got[0], truth(ic, beta, lp, node), rtol=1e-10)
        for arr, sl in ((ic, slice(1, 1 + G)), (beta, slice(1 + G, 1 + G + P)), (lp, slice(1 + G + P, None))):
            fd = np.zeros(arr.size)
            for i, idx in enumerate(np.ndindex(arr.shape)):
                orig = arr[idx].copy()
                h = 1e-6
                arr[idx] = orig + h
                hi = truth(ic, beta, lp, node)
                arr[idx] = orig - h
                lo = truth(ic, beta, lp, node)
                arr[idx] = orig
                fd[i] = (hi - lo) / (2 * h)
            np.testing.assert_allclose(got[sl], fd, rtol=1e-5, atol=1e-6 * np.max(np.abs(fd)))


def test_fp32_terms_stay_near_the_fp64_ones():
    """The collective backend evaluates the same grouped terms in float32; on |eta| <= 10 and phi up to 1e6 they stay
    within 2^-16 of the parts' magnitudes of the fp64 values (plus the slope times the inputs' rounding)."""
    etas, ys = _domain_rows(DOMAIN_A)
    keep = np.abs(etas) <= 10
    etas, ys = etas[keep], ys[keep]
    a = DOMAIN_A.astype(np.float32)
    got = [t.double().numpy() for t in TERMS(torch.tensor(ys)[:, None], torch.tensor(etas)[:, None], torch.tensor(a))]
    want = _terms64(ys, etas, a)
    parts, slopes = _parts(ys, etas, a), _slopes(ys, etas, a)
    for g, w, p, s in zip(got, want, parts, slopes):
        assert np.all(np.isfinite(g))
        assert np.all(np.abs(g - w) <= 2.0 ** -16 * p + s * 2.0 ** -18 * (1 + np.abs(etas))[:, None])


# ----------------------------------------------------------------------------------------------- CPU: the emulation
def _emulate(etas, ys, a, variant=None):
    """The kernel's ``beta_loglik`` (with ``beta_constants`` and ``beta_tails``) in fp32 numpy, ``(ll, r, q)`` of each
    row and chain.  ``variant="lgamma"``: ll as ``lgamma(phi) - lgamma(A) - lgamma(B) + (A - 1) log y + (B - 1) log(1 -
    y)`` with each lgamma correctly rounded to fp32; ``"logs"``: ``log y - log mu`` and ``log(1 - y) - log(1 - mu)``
    in place of the relative differences on every row."""
    from scipy.special import gammaln

    f = np.float32
    with np.errstate(all="ignore"):
        a32 = a.astype(f)
        ld = a32.astype(np.float64)
        phi64, C64, Q64 = (t.numpy() for t in _beta_constants(_t64(ld)))
        phi, Cp, Qp = phi64.astype(f), C64.astype(f), Q64.astype(f)
        y = ys.astype(f)[:, None]
        eta = etas.astype(f)[:, None]
        ly, l1y = np.log(y), np.log1p(-y)
        e = np.exp(-np.abs(eta))
        l1e = np.log1p(e)
        inv, ie = f(1) / (f(1) + e), f(1) / e
        pos = eta >= 0
        mu, nmu = np.where(pos, inv, e * inv), np.where(pos, e * inv, inv)
        lmu, l1mu = np.where(pos, -l1e, eta - l1e), np.where(pos, -eta - l1e, -l1e)
        imu, inmu = np.where(pos, f(1) + e, f(1) + ie), np.where(pos, f(1) + ie, f(1) + e)
        A, B = mu * phi, nmu * phi
        d = np.where(pos, nmu - (f(1) - y), y - mu)
        u, v = d * imu, -d * inmu

        def kser(x):
            s = x * (f(1) / (f(2) + x))
            s2 = s * s
            p = s2 * f(1 / 15) + f(1 / 13)
            for c in (1 / 11, 1 / 9, 1 / 7, 1 / 5, 1 / 3):
                p = s2 * p + f(c)
            return x * s - f(2) * (s * s2) * p

        su, sv = np.abs(u) < f(0.5), np.abs(v) < f(0.5)
        if variant == "logs":
            su = sv = np.zeros_like(su)
        ku, kv = kser(u), kser(v)
        lu, lv = np.where(su, u - ku, ly - lmu), np.where(sv, v - kv, l1y - l1mu)
        pd = phi * d
        kl = np.where(su, A * ku, pd - A * lu) + np.where(sv, B * kv, -pd - B * lv)

        def tails(z, lz):
            m = np.where(z < f(8), np.ceil(f(8) - z), f(0)).astype(f)
            lp = np.zeros_like(z)
            sr = np.zeros_like(z)
            for g in range(2):
                pr, nu = np.ones_like(z), np.zeros_like(z)
                for j in range(4 * g + 1, min(4 * g + 5, 8)):
                    fj = z + f(j)
                    take = f(j) < m
                    nu = np.where(take, nu * fj + pr, nu)
                    pr = np.where(take, pr * fj, pr)
                lp = lp + np.log(pr)
                sr = sr + nu / pr
            zp = z + m
            iz = f(1) / zp
            iz2 = iz * iz
            Sz = iz * (f(1 / 12) - iz2 * (f(1 / 360) - iz2 * f(1 / 1260)))
            Tz = f(-0.5) * iz - iz2 * (f(1 / 12) - iz2 * (f(1 / 120) - iz2 * f(1 / 252)))
            lzp = np.log(zp)
            sh = m > 0
            S = np.where(sh, Sz + (((zp - f(0.5)) * lzp - m) - lp - (z + f(0.5)) * lz), Sz)
            zt = np.where(sh, z * ((Tz - sr) + (lzp - lz)) - f(1), z * Tz)
            return S, zt

        SA, tA = tails(A, lmu + a32)
        SB, tB = tails(B, l1mu + a32)
        # each tail folded into ll, r and q in turn, as the kernel does
        ll = ((((Cp + f(0.5) * (lmu + l1mu)) - (ly + l1y)) - kl) - SA) - SB
        if variant == "lgamma":
            g32 = lambda z: gammaln(z.astype(np.float64)).astype(f)
            ll = ((g32(phi) - g32(A)) - g32(B)) + ((A - f(1)) * ly + (B - f(1)) * l1y)
        r = ((A * nmu) * (lu - lv) - nmu * tA) + mu * tB
        q = ((Qp - kl) - tA) - tB
    return [v.astype(np.float64) for v in (ll, r, q)]


def _sweep_failures(etas, ys, a, ll, r, g0, q):
    """The per-row checks of the domain sweep that some row fails, for values ``[rows, chains]``: each of ll, r, the
    MMA-path gradient g0 and q may be off by 16 fp32 roundings (``2^-20``) of the magnitudes of its grouped terms
    (:func:`_parts`; g0 by ``2^-16``, the (hi, lo) bf16 split of r and MMA #2), plus its slope in eta times ``2^-20``:
    mu and 1 - mu carry a few roundings of expf and the reciprocal, which act as an error of that size in eta."""
    want = _terms64(ys, etas, a)
    parts = _parts(ys, etas, a)
    sl = _slopes(ys, etas, a)
    u, de = 2.0 ** -20, 2.0 ** -20
    ok = {
        "finite": all(np.all(np.isfinite(v)) for v in (ll, r, g0, q)),
        "ll": np.all(np.abs(ll - want[0]) <= u * parts[0] + sl[0] * de),
        "r": np.all(np.abs(r - want[1]) <= u * parts[1] + sl[1] * de),
        "g0": np.all(np.abs(g0 - want[1]) <= 2.0 ** -16 * parts[1] + sl[1] * de),
        "q": np.all(np.abs(q - want[2]) <= u * parts[2] + sl[2] * de),
    }
    return sorted(k for k, v in ok.items() if not v)


#: the chains of the domain sweep: 16 log precisions from -5 to 14 (phi 0.0067 to 1.2e6)
SWEEP_A = np.concatenate([DOMAIN_A, [-1.0, 2.5, 4.0, 6.0, 12.5]]).astype(np.float32)


def test_sweep_bound_tells_the_grouped_form_from_naive_ones():
    """The per-row bound of the domain sweep holds for an fp32 emulation of the kernel's code, and breaks for direct
    lgamma differences (at phi >= 1e4) and for log differences in place of the relative ones (at y ~ mu)."""
    etas, ys = _domain_rows(SWEEP_A)
    ll, r, q = _emulate(etas, ys, SWEEP_A)
    assert _sweep_failures(etas, ys, SWEEP_A, ll, r, r, q) == []
    big = SWEEP_A >= np.log(1e4)
    ll, r, q = _emulate(etas, ys, SWEEP_A[big], variant="lgamma")
    assert "ll" in _sweep_failures(etas, ys, SWEEP_A[big], ll, r, r, q)
    near = np.abs(ys / (1 / (1 + np.exp(-etas.astype(np.float64)))) - 1) < 1e-3
    ll, r, q = _emulate(etas[near], ys[near], SWEEP_A, variant="logs")
    failed = _sweep_failures(etas[near], ys[near], SWEEP_A, ll, r, r, q)
    assert "ll" in failed and "q" in failed


# ----------------------------------------------------------------------------------------------- CPU: the model
@pytest.mark.parametrize("K", [1, 4])
def test_collective_backend_equals_the_oracle(K):
    rows, P = [300, 45, 129], 24
    Xs, ys, ws, os_ = _case(rows, P, seed=6)
    model = _model(Xs, ys, ws, os_, groups=[0, 1, 1], n_groups=2, n_chains=K)
    ic, beta, lp = _theta(2, P, K, log_phi=[-0.5, 2.0, 5.0, 9.0][:K] if K > 1 else 3.0)
    got, want = _collective(model, ic, beta, lp), _oracle(model, ic, beta, lp)
    for u, v in zip(got, want):
        assert np.shape(u) == np.shape(v) and np.all(np.isfinite(u))
        np.testing.assert_allclose(u, v, rtol=1e-4, atol=1e-3 * max(1.0, np.max(np.abs(v))))


def test_node_federation_on_the_collective_backend_equals_single_node_models():
    from pytensor_federated_b200.federation import NodeFederation

    rows, node_ids, groups = [200, 128, 77], [0, 1, 1], [0, 1, 0]
    Xs, ys, ws, os_ = _case(rows, 16, seed=13)
    model = _model(Xs, ys, ws, os_, groups=groups, n_groups=2, node_ids=node_ids, n_nodes=2)
    ic, beta, lp = _theta(2, 16, log_phi=np.log(20.0))
    with FederatedEngine(model, backend="collective") as eng:
        blocks = model.per_node(eng.evaluate_raw([ic, beta, lp]))
        res = NodeFederation(eng).evaluate_nodes({0: (ic, beta, lp), 1: (ic, beta, lp)})
    assert blocks.shape == (2, 1, 2 + 2 + 16)
    for node in (0, 1):
        segs = [i for i, n in enumerate(node_ids) if n == node]
        single = _model([Xs[i] for i in segs], [ys[i] for i in segs], [ws[i] for i in segs], [os_[i] for i in segs],
                        groups=[groups[i] for i in segs], n_groups=2)
        want = _oracle(single, ic, beta, lp)
        got = [blocks[node, 0, 0], blocks[node, 0, 1:3], blocks[node, 0, 3:-1], blocks[node, 0, -1]]
        for u, v in zip(got, want):
            np.testing.assert_allclose(u, v, rtol=1e-4, atol=1e-3 * max(1.0, np.max(np.abs(v))))
        np.testing.assert_allclose(res[node][0], blocks[node, 0, 0], rtol=1e-12)


def test_validation():
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ys = [torch.full((10,), 0.25), torch.full((6,), 0.5)]
    GlmShards(Xs, ys, family=FAMILY)
    GlmShards(Xs, ys, family=FAMILY, n_chains=16, offsets=[torch.zeros(10), None], weights=[None, torch.ones(6)])
    for kernel in ("simt", "generic", "fp8"):
        with pytest.raises(ValueError, match="tensor-core kernel only"):
            GlmShards(Xs, ys, family=FAMILY, kernel=kernel)
    with pytest.raises(ValueError, match="tensor-core kernel only"):
        Fp8GlmShards.from_dense([torch.randn(10, 32), torch.randn(6, 32)], ys, family=FAMILY)
    with pytest.raises(ValueError, match="n_classes"):
        GlmShards(Xs, ys, family=FAMILY, n_classes=2)
    with pytest.raises(ValueError, match="events="):
        GlmShards(Xs, ys, family=FAMILY, events=[None, None])
    with pytest.raises(ValueError, match="hvp=True is for family"):
        GlmShards(Xs, ys, family=FAMILY, hvp=True)
    for X in (torch.randn(10, 12).to(torch.bfloat16), torch.randn(10, 392).to(torch.bfloat16), torch.randn(10, 16)):
        with pytest.raises(ValueError, match="tensor-core kernel only"):
            GlmShards([X], [torch.full((10,), 0.5)], family=FAMILY).use_tensor_cores()
    assert GlmShards(Xs, ys, family=FAMILY, kernel="tc").use_tensor_cores() == 1
    for bad in (0.0, -0.0, 1.0, -0.5, 1.5, float("nan"), float("inf"), float("-inf")):
        y1 = torch.full((6,), 0.5)
        y1[2] = bad
        with pytest.raises(ValueError, match="responses of segment 1 must be finite with 0 < y < 1"):
            GlmShards(Xs, [ys[0], y1], family=FAMILY)
        w1 = torch.ones(6)
        w1[2] = 0.0
        GlmShards(Xs, [ys[0], y1], family=FAMILY, weights=[None, w1])   # a masked row may carry anything
    y0 = torch.full((10,), 0.5)
    y0[3], y0[4] = 1e-38, Y_MAX   # the ends of the open interval in float32 are valid responses
    GlmShards(Xs, [y0, ys[1]], family=FAMILY)


def test_sizes_and_flops():
    Xs = [torch.randn(10, 16).to(torch.bfloat16), torch.randn(6, 16).to(torch.bfloat16)]
    ys = [torch.full((10,), 0.5), torch.full((6,), 0.5)]
    m = GlmShards(Xs, ys, n_groups=2, groups=[0, 1], family=FAMILY, n_chains=3, node_ids=[0, 1], n_nodes=2)
    assert m.n_inputs == 3 and m.input_shapes == [(2,), (16,), ()]
    assert m.n_params == 2 + 16 + 1 and m.n_theta_words == 3 * 19
    assert m.n_vals == 2 * 3 * (2 + 2 + 16)
    assert m.flops_per_eval() == GlmShards(Xs, ys, n_chains=3).flops_per_eval()
    assert m.bytes_per_eval() == GlmShards(Xs, ys).bytes_per_eval()


@pytest.mark.parametrize("K,G", [(1, 1), (1, 2), (4, 2)])
def test_pack_unpack_and_words_round_trip(K, G):
    P = 8
    Xs, ys, _, _ = _case([20] * G, P, seed=7, n_masked=0, weighted=False, offsets=False)
    model = GlmShards(Xs, ys, groups=list(range(G)), n_groups=G, family=FAMILY, n_chains=K)
    ic, beta, lp = _theta(G, P, K, log_phi=np.arange(K) - 0.5 if K > 1 else -0.5, scale=1.0)
    if K == 1 and G == 1:
        ic = ic.reshape(())   # a scalar intercept for one group
    words = np.zeros(model.n_theta_words, dtype=np.uint32)
    ctx = model.pack_theta([ic, beta, lp], words)
    assert ctx == model.call_context([ic, beta, lp]) == (K > 1, ic.shape, np.shape(lp))
    th = words.view(np.float32).reshape(K, G + P + 1)
    np.testing.assert_array_equal(th[:, :G], np.reshape(ic, (K, G)))
    np.testing.assert_array_equal(th[:, G : G + P], np.reshape(beta, (K, P)))
    np.testing.assert_array_equal(th[:, G + P], np.reshape(lp, K))
    ic2, b2, lp2 = default_inputs_from_words(model, words)
    assert np.array_equal(ic2.reshape(ic.shape), ic) and np.array_equal(b2, beta) and np.array_equal(lp2, lp)
    theta = np.concatenate([np.reshape(ic, (K, G)), np.reshape(beta, (K, P)), np.reshape(lp, (K, 1))], axis=1)
    for u, v in zip(model.inputs_from_theta(theta), (ic, beta, lp)):
        assert np.array_equal(np.reshape(u, np.shape(v)), v)
    raw = np.arange(model.n_vals, dtype=np.float64).reshape(K, 2 + G + P)
    logp, d_ic, d_b, d_lp = model.unpack_result(raw.reshape(-1), ctx)
    assert d_ic.shape == np.shape(ic) and d_b.shape == beta.shape and np.shape(d_lp) == np.shape(lp)
    np.testing.assert_array_equal(np.reshape(logp, -1), raw[:, 0])
    np.testing.assert_array_equal(np.reshape(d_ic, (K, G)), raw[:, 1 : 1 + G])
    np.testing.assert_array_equal(np.reshape(d_b, (K, P)), raw[:, 1 + G : 1 + G + P])
    np.testing.assert_array_equal(np.reshape(d_lp, K), raw[:, -1])


def test_glm_batch_fn_splits_theta_with_log_precision():
    from pytensor_federated_b200.sampling import glm_batch_fn

    P, G = 8, 2
    Xs, ys, ws, os_ = _case([60, 40], P, seed=8)
    model = _model(Xs, ys, ws, os_, groups=[0, 1], n_groups=G, n_chains=2)
    rng = np.random.default_rng(9)
    theta = np.concatenate([np.array([0.4, -1.0]) + rng.normal(size=(3, G)) * 0.05, rng.normal(size=(3, P)) * 0.01,
                            np.log(20.0) + rng.normal(size=(3, 1)) * 0.1], axis=1)
    with FederatedEngine(model, backend="collective") as eng:
        logp, grad = glm_batch_fn(eng, G)(theta)
    assert logp.shape == (3,) and grad.shape == theta.shape
    single = _model(Xs, ys, ws, os_, groups=[0, 1], n_groups=G)
    for i in range(3):
        want = _oracle(single, theta[i, :G], theta[i, G : G + P], theta[i, -1])
        np.testing.assert_allclose(logp[i], want[0], rtol=1e-5)
        np.testing.assert_allclose(grad[i], np.concatenate([want[1], want[2], [want[3]]]), rtol=1e-4, atol=1e-3)


def test_tc_stages_are_the_dispersion_layouts():
    from pytensor_federated_b200.ops import native

    lib = native.load()
    for P, K, G, rows in ((8, 1, 1, 0), (256, 4, 2, 3), (256, 16, 300, 1), (384, 8, 1, 0), (384, 16, 1, 3)):
        assert lib.b200_glm_tc_stages(P, K, G, CODES[FAMILY], rows) == \
            lib.b200_glm_tc_stages(P, K, G, CODES["negative_binomial"], rows)


def test_synth_beta_shard():
    import scipy.stats

    n, phi = 200_000, 30.0
    X, y, beta = synth_beta_shard(n, 16, phi=phi, seed=1, device="cpu", chunk_rows=65536)
    assert X.dtype == torch.bfloat16 and X.shape == (n, 16) and beta.shape == (16,)
    assert y.dtype == torch.float32 and bool(torch.all((y > 0) & (y < 1)))
    X2, y2, _ = synth_beta_shard(n, 16, phi=phi, seed=1, device="cpu", chunk_rows=65536)
    assert torch.equal(X, X2) and torch.equal(y, y2)
    # at beta* = 0 every y is a draw at mean sigmoid(intercept): its moments and distribution
    mu = 1 / (1 + np.exp(-0.5))
    _, y0, _ = synth_beta_shard(n, 8, phi=phi, seed=2, device="cpu", beta_scale=0.0, intercept=0.5)
    v = y0.double().numpy()
    var = mu * (1 - mu) / (1 + phi)
    assert abs(v.mean() - mu) < 5 * np.sqrt(var / n)
    assert scipy.stats.kstest(v[:50_000], scipy.stats.beta(a=mu * phi, b=(1 - mu) * phi).cdf).pvalue > 1e-3
    # a tiny precision puts most of the mass at the ends: every y stays inside the open interval in float32
    _, yt, _ = synth_beta_shard(20_000, 8, phi=0.01, seed=3, device="cpu", intercept=-3.0)
    assert bool(torch.all((yt > 0) & (yt < 1)))
    # ... and at the end the draw picked, not at the centre: P(y > 1/2) is about mu there
    assert abs(float((yt > 0.5).double().mean()) - 1 / (1 + np.exp(3.0))) < 0.01
    assert float(((yt > 0.01) & (yt < 0.99)).double().mean()) < 0.05
    # and the model the data came from fits it: dLL/da at the true precision is ~0 relative to its scale
    m = GlmShards([X], [y], family=FAMILY)
    got = _oracle(m, np.float32(0.5), beta.numpy(), np.float32(np.log(phi)), chunk_rows=1 << 16)
    assert abs(got[3]) < 5 * np.sqrt(n)
    with pytest.raises(ValueError, match="phi must be > 0"):
        synth_beta_shard(10, 8, phi=0.0, seed=0, device="cpu")


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


def _bound(model, ic, beta, lp):
    """A bound on the kernel's error, per output and in the shapes of the results, from the fp64 magnitudes of the
    terms each one sums.  Per row, eta is off by at most ``d_eta = 2^-18 (1 + |eta| + sum_j |x_j beta_j|)`` (the
    three-term bf16 split of beta keeps 24 bits, the fp32 MMA sums over P), and the kernel's ll, r and q by a few fp32
    roundings of the parts they are formed from (:func:`_parts`).  The per-thread fp32 sums of a chunk add at most 64
    rows, so LL and q get ``2^-16`` of the summed parts plus ``slope d_eta``; the gradients get ``2^-14`` of ``sum w
    (parts of r) |x|`` (the (hi, lo) bf16 split of r keeps ~2^-17 of it, then fp32 MMA sums) plus ``sum w |dr/deta|
    d_eta |x|``."""
    batched = np.ndim(beta) == 2
    K, G, P = model.n_chains, model.n_groups, model.n_features
    icd = np.reshape(ic, (K, G)).astype(np.float64)
    bd = np.reshape(beta, (K, P)).astype(np.float64)
    ad = np.reshape(lp, (K,)).astype(np.float64)
    t_ll, t_q = np.zeros(K), np.zeros(K)
    t_gi, t_g = np.zeros((K, G)), np.zeros((K, P))
    for si, (X, y, g) in enumerate(zip(model.Xs, model.ys, model.groups)):
        w = model.weights[si]
        keep = torch.ones_like(y, dtype=torch.bool) if w is None else w != 0
        ww = (torch.ones_like(y) if w is None else w).double()[keep].cpu().numpy()[:, None]
        Xd = X.double()[keep].cpu().numpy()
        yy = y.double()[keep].cpu().numpy()
        eta = Xd @ bd.T + icd[:, g]
        if model.offsets[si] is not None:
            eta = eta + model.offsets[si].double()[keep].cpu().numpy()[:, None]
        d_eta = 2.0 ** -18 * (1.0 + np.abs(eta) + np.abs(Xd) @ np.abs(bd).T)
        cols = [[], [], [], [], [], []]
        for k in range(K):   # per chain: eta differs per chain
            p = _parts(yy, eta[:, k], ad[k : k + 1])
            s = _slopes(yy, eta[:, k], ad[k : k + 1])
            for c, v in zip(cols, list(p) + list(s)):
                c.append(v[:, 0])
        (p_ll, p_r, p_q, s_ll, s_r, s_q) = (np.stack(c, axis=1) for c in cols)
        t_ll += (ww * (2.0 ** -16 * p_ll + s_ll * d_eta)).sum(0)
        t_q += (ww * (2.0 ** -16 * p_q + s_q * d_eta)).sum(0)
        e = ww * (2.0 ** -14 * p_r + s_r * d_eta)
        t_gi[:, g] += e.sum(0)
        t_g += e.T @ np.abs(Xd)
    out = [t_ll, t_gi, t_g, t_q]
    return out if batched else [out[0][0], out[1][0], out[2][0], out[3][0]]


def _check(got, want, tol):
    assert all(np.all(np.isfinite(g)) for g in got)
    for u, v, t in zip(got, want, tol):
        assert np.shape(u) == np.shape(v)
        err = np.abs(np.asarray(u, dtype=np.float64) - v)
        assert np.all(err <= t), (np.max(err / t), np.max(err))


@pytest.mark.parametrize("row_data", [True, False])
@pytest.mark.parametrize("P,K", [(8, 1), (256, 1), (256, 2), (128, 3), (256, 4), (256, 8), (200, 13), (256, 16)])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_matches_oracle(dev, P, K, row_data):
    """K = 1, 2, 3, 4, 8, 13 and 16 cover the kernel's four buckets, full and partial; ``row_data`` (offsets and
    weights, masked rows with NaN / 0 / 1 / negative / inf responses) its ROWS variant.  The chains cycle through phi
    from 0.05 to 1e6; with K = 1 three of them are evaluated, one launch each."""
    rows = [128 * 37, 77, 4099, 1]
    Xs, ys, ws, os_ = _case(rows, P, seed=K + P, device=dev, weighted=row_data, offsets=row_data,
                            n_masked=5 if row_data else 0)
    model = _model(Xs, ys, ws, os_, groups=[0, 1, 0, 1], n_groups=2, n_chains=K, kernel="auto")
    assert model.has_row_data == row_data
    if K == 1:
        inputs = [_theta(2, P, 1, log_phi=v, seed=5 + i) for i, v in enumerate(LOG_PHI[[0, 5, 8]])]
    else:
        inputs = [_theta(2, P, K, log_phi=np.resize(LOG_PHI, K))]
    got = _run(model, inputs)
    assert model.selected_kernel == "tc"
    for g, inp in zip(got, inputs):
        _check(g, _oracle(model, *inp, chunk_rows=1 << 20), _bound(model, *inp))


@pytest.mark.parametrize("K,row_data", [(1, False), (4, True), (16, True)])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_kernel_with_many_groups_and_nodes_matches_oracle(dev, K, row_data):
    """300 groups, ragged segments of 1 to 3000 rows and three output blocks (one per node)."""
    G, P = 300, 256
    rows = [128 * 9 + 5, 999, 64, 1, 3000]
    groups, node_ids = [0, 299, 150, 7, 299], [0, 2, 1, 0, 2]
    Xs, ys, ws, os_ = _case(rows, P, seed=40 + K, device=dev, weighted=row_data, offsets=row_data,
                            n_masked=5 if row_data else 0)
    model = _model(Xs, ys, ws, os_, groups=groups, n_groups=G, n_chains=K, kernel="tc", node_ids=node_ids, n_nodes=3)
    inp = _theta(G, P, K, log_phi=np.resize(LOG_PHI[::-1], K) if K > 1 else LOG_PHI[4])
    (raw,) = _run(model, [inp], raw=True)
    blocks = model.per_node(raw)
    for node in range(3):
        segs = [i for i, n in enumerate(node_ids) if n == node]
        single = _model([Xs[i] for i in segs], [ys[i] for i in segs], [ws[i] for i in segs], [os_[i] for i in segs],
                        groups=[groups[i] for i in segs], n_groups=G, n_chains=K, kernel="tc")
        want = _oracle(single, *inp, chunk_rows=1 << 20)
        b = blocks[node] if K > 1 else blocks[node, 0]
        got = [b[..., 0], b[..., 1 : 1 + G], b[..., 1 + G : 1 + G + P], b[..., -1]]
        _check(got, want, _bound(single, *inp))
    unused = np.ones(G, dtype=bool)
    unused[groups] = False
    assert np.all(blocks[..., 1 : 1 + G][..., unused] == 0.0)


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_tc_per_row_values_across_the_domain(dev):
    """The kernel's ll, r = dll/deta (intercept gradient), the MMA-path gradient and q = dll/da of single rows (one
    segment, group and output block each, eta = the intercept exactly: beta = 0, x = e_0) at 16 precisions from
    0.0067 to 1.2e6 (one launch per 128 rows, K = 16), within the per-row bound of :func:`_sweep_failures`, with no
    value NaN or inf."""
    P, K = 8, 16
    etas, ys = _domain_rows(SWEEP_A)
    lls, rs, g0s, qs = [], [], [], []
    for c0 in range(0, len(ys), 128):
        e, yv = etas[c0 : c0 + 128], ys[c0 : c0 + 128]
        n = len(yv)
        X = torch.zeros(n, P, dtype=torch.bfloat16, device=dev)
        X[:, 0] = 1.0
        Xs = [X[i : i + 1].clone() for i in range(n)]
        yl = [torch.tensor(yv[i : i + 1], device=dev) for i in range(n)]
        model = GlmShards(Xs, yl, groups=list(range(n)), n_groups=n, family=FAMILY, n_chains=K, kernel="tc",
                          node_ids=list(range(n)), n_nodes=n)
        inp = (np.broadcast_to(e, (K, n)).copy(), np.zeros((K, P), np.float32), SWEEP_A)
        with FederatedEngine(model) as eng:
            blocks = model.per_node(eng.evaluate_raw(list(inp)))   # [n, K, 2 + n + P]
        idx = np.arange(n)
        lls.append(blocks[idx, :, 0])
        rs.append(blocks[idx, :, 1 + idx])
        g0s.append(blocks[:, :, 1 + n])
        qs.append(blocks[:, :, -1])
    ll, r, g0, q = (np.concatenate(v) for v in (lls, rs, g0s, qs))
    assert _sweep_failures(etas, ys, SWEEP_A, ll, r, g0, q) == []


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_tc_evaluations_are_reproducible_over_grids_and_transports(dev):
    """The same bits whatever the grid, and in both result transports: 8 chains x (2 + 3 + 256) values > 2048, and
    one chain at P = 16 (20 values)."""
    rows = [40_000, 25_000, 33_333, 128, 19_999]
    for P, K in ((256, 8), (16, 1)):
        Xs, ys, ws, os_ = _case(rows, P, seed=12, device=dev)
        model = _model(Xs, ys, ws, os_, groups=[0, 1, 2, 1, 0], n_groups=3, n_chains=K, kernel="tc")
        assert (model.n_vals > 2048) == (K == 8)
        inp = _theta(3, P, K, log_phi=np.resize(LOG_PHI, K) if K > 1 else LOG_PHI[4])
        outs = []
        for grid in (None, 7, 200):
            outs += _run(model, [inp] * 2, raw=True, grid=grid)
        for o in outs[1:]:
            assert o.tobytes() == outs[0].tobytes()


@pytest.mark.parametrize("rows_data", [False, True])
@pytest.mark.parametrize("K", [1, 2, 4])
@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_packed_launch_is_bitwise_the_unpacked_one(dev, K, rows_data, monkeypatch):
    """P = 200 and 256 with at most 4 columns are packed by default."""
    for P in (200, 256):
        Xs, ys, ws, os_ = _case([3 * 128 + 5, 1000, 128], P, seed=21 + K, device=dev, weighted=rows_data,
                                offsets=rows_data, n_masked=5 if rows_data else 0)
        inp = _theta(2, P, K, log_phi=np.resize(LOG_PHI, K) if K > 1 else 3.0)
        outs = {}
        for packed in (True, False):
            if packed:
                monkeypatch.delenv("B200FED_NO_PACKED_X", raising=False)
            else:
                monkeypatch.setenv("B200FED_NO_PACKED_X", "1")
            model = _model(Xs, ys, ws, os_, groups=[0, 1, 0], n_groups=2, n_chains=K, kernel="tc")
            (outs[packed],) = _run(model, [inp], raw=True)
            assert model.packed_x is packed
        assert np.all(np.isfinite(outs[True]))
        assert outs[True].tobytes() == outs[False].tobytes()


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_node_federation_blocks_equal_single_node_models(dev):
    from pytensor_federated_b200.federation import NodeFederation

    rows = [20_000, 128 * 33, 7777]
    node_ids, groups = [0, 1, 1], [0, 1, 0]
    Xs, ys, ws, os_ = _case(rows, 256, seed=13, device=dev)
    model = _model(Xs, ys, ws, os_, groups=groups, n_groups=2, kernel="tc", node_ids=node_ids, n_nodes=2)
    ic, beta, lp = _theta(2, 256, log_phi=np.log(20.0))
    with FederatedEngine(model) as eng:
        n0 = eng.kernel_launches
        blocks = model.per_node(eng.evaluate_raw([ic, beta, lp]))
        assert eng.kernel_launches - n0 == 1
        fed = NodeFederation(eng)
        res = fed.evaluate_nodes({0: (ic, beta, lp), 1: (ic, beta, lp)})
        total = fed.all_nodes_func()(ic, beta, lp)
    for node in (0, 1):
        segs = [i for i, n in enumerate(node_ids) if n == node]
        single = _model([Xs[i] for i in segs], [ys[i] for i in segs], [ws[i] for i in segs], [os_[i] for i in segs],
                        groups=[groups[i] for i in segs], n_groups=2, kernel="tc")
        want = _oracle(single, ic, beta, lp, chunk_rows=1 << 20)
        got = [blocks[node, 0, 0], blocks[node, 0, 1:3], blocks[node, 0, 3:-1], blocks[node, 0, -1]]
        _check(got, want, _bound(single, ic, beta, lp))
        np.testing.assert_allclose(res[node][0], blocks[node, 0, 0], rtol=1e-12)
        np.testing.assert_allclose(res[node][1][2], blocks[node, 0, -1], rtol=1e-12)
    np.testing.assert_allclose(total[0], blocks[:, 0, 0].sum(), rtol=1e-12)


@pytest.mark.gpu
@pytest.mark.timeout(1200)
def test_map_recovers_the_parameters(dev):
    """On 2M synthetic rows x 64 features (phi = 30), L-BFGS through ``glm_batch_fn`` on the kernel finds beta*, the
    intercept and log phi, each within 4 standard errors; the standard errors come from the Hessian of the fp64
    oracle's LL at the MAP (central differences of its gradient), on the CPU."""
    from pytensor_federated_b200.sampling import find_map, glm_batch_fn

    n, P, phi = 2_000_000, 64, 30.0
    X, y, beta = synth_beta_shard(n, P, phi=phi, seed=7, device=dev, beta_scale=0.2)
    model = GlmShards([X], [y], family=FAMILY, kernel="tc")
    truth = np.concatenate([[0.5], beta.cpu().numpy(), [np.log(phi)]])
    with FederatedEngine(model) as eng:
        fn = glm_batch_fn(eng, 1)

        def logp_dlogp(x):
            lp, g = fn(x[None])
            return lp[0], g[0]

        x_map, info = find_map(logp_dlogp, np.zeros_like(truth), maxiter=500)
    cpu = GlmShards([X.cpu()], [y.cpu()], family=FAMILY)

    def grad64(x):
        out = _oracle(cpu, x[0], x[1 : 1 + P], x[-1], chunk_rows=1 << 18)
        return np.concatenate([np.atleast_1d(out[1]), out[2], [out[3]]])

    D = len(truth)
    H = np.zeros((D, D))
    for i in range(D):
        e = np.zeros(D)
        e[i] = 1e-4
        H[i] = (grad64(x_map + e) - grad64(x_map - e)) / 2e-4
    se = np.sqrt(np.diag(np.linalg.inv(-0.5 * (H + H.T))))
    assert np.all(np.isfinite(se)) and np.all(se > 0)
    assert np.all(np.abs(x_map - truth) < 4 * se), (x_map - truth) / se


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_runtime_rejects_the_beta_family_outside_the_tc_kernel(dev):
    """The C ABI refuses what the Python layer never sends: family 15 on a CUDA-core or fp8 kernel, n_classes != 1,
    an output size without the log-precision gradient, and the Hessian-vector-product flag.  The engine keeps its
    model after each refusal."""
    from pytensor_federated_b200.ops import native

    Xs, ys, _, _ = _case([256], 16, seed=14, device=dev, n_masked=0, weighted=False, offsets=False)
    model = GlmShards(Xs, ys, family="poisson", kernel="simt")
    ic, beta = np.float32(0.1), np.zeros(16, np.float32)
    want = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    code = CODES[FAMILY]
    with FederatedEngine(model) as eng:
        lib, h = eng._lib, eng._handle
        Xp, yp = native.void_p_array([Xs[0].data_ptr()]), native.void_p_array([ys[0].data_ptr()])
        rows, grp = (C.c_longlong * 1)(256), (C.c_int * 1)(0)

        def set_glm(n_chains, family, kernel, n_classes=1):
            return int(lib.b200_engine_set_glm(h, 1, Xp, yp, None, rows, grp, 16, 16, 1, n_chains, family, kernel,
                                               None, 1, None, None, n_classes))

        def still_poisson():
            got = eng.evaluate(ic, beta)
            np.testing.assert_allclose(got[0], want[0], rtol=2e-5)

        for kernel in (0, 2, 3, 4):
            assert set_glm(1, code, kernel) == -39
            assert "the beta family runs on the bf16 tensor-core kernel only" in native.last_error()
            still_poisson()
        assert set_glm(1, code, 1, 2) == -38 and "n_classes must be 1" in native.last_error()
        still_poisson()
        # this engine's n_vals is 1 + G + P: one value short of this family's block
        assert set_glm(1, code, 1) == -33 and "2 + n_groups + n_features" in native.last_error()
        still_poisson()
        assert set_glm(2, code | 16, 1) == -40 and "Hessian-vector products exist for" in native.last_error()
        still_poisson()


def _build_beta_model(rank, world, dev):
    Xs, ys, ws, os_ = _case([30_000 + 17 * rank, 999, 77], 256, seed=50 + rank, device=dev)
    return _model(Xs, ys, ws, os_, groups=[rank % 2, 1 - rank % 2, 0], n_groups=2, n_chains=2, kernel="tc")


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.timeout(900)
def test_two_rank_beta_federation_matches_oracle():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from pytensor_federated_b200.federation import launch_federation

    inp = _theta(2, 256, 2, log_phi=[np.log(0.5), 6.0])
    dev = torch.device("cuda:0")
    models = [_build_beta_model(r, 2, dev) for r in range(2)]
    want = models[0].unpack_result(sum(m.reference_partial(list(inp), dtype=torch.float64) for m in models),
                                   models[0].call_context(list(inp)))
    tol = [sum(v) for v in zip(*(_bound(m, *inp) for m in models))]
    del models
    with launch_federation(_build_beta_model, 2, timeout=30.0) as eng:
        got = eng.evaluate(*inp)
    _check(got, want, tol)
