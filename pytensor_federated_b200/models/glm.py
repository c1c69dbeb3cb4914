"""Generalised linear model shards with a low-precision, HBM-resident design matrix.

Workloads from ``BASELINE.json`` (not present in the reference, whose only model is
the 10-point linear regression): *federated logistic GLM, 10M rows x 256 features per shard,
bf16 design matrix* and *hierarchical GLM, 8 partial-pooling groups, fp8 block-scaled design
matrix*.  ``theta = [intercept[G], beta[P]]`` (float32) per chain; a segment (shard) uses
``intercept[group]``, so G = 1 is the pooled GLM and G = #shards the partial-pooling one.
Result per chain: ``[LL, dLL/dintercept[G], dLL/dbeta[P]]`` (float64).

How a family's inputs map to the kernel (the input shapes, the theta words, the kernel's output blocks and the
oracle's per-row terms) is decided by one layout object per family (``_Scalar``, ``_Softmax``, ``_Dispersion``,
``_Ordinal``, ``_Survival``, ``_Positive``, ``_Beta``, ``_Hvp``, ``_ZeroInflated``, ``_LocationScale`` below); :class:`GlmShards` and its callers are generic over it.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence

import numpy as np

from .base import ShardModel

FAMILIES = {"logistic": 0, "poisson": 1, "gaussian": 2, "multinomial": 3, "gaussian_scale": 4, "negative_binomial": 5,
            "ordinal": 6, "weibull": 7, "lognormal": 8, "zero_inflated_poisson": 9, "zero_inflated_negative_binomial": 10,
            "gamma": 11, "inverse_gaussian": 12, "gaussian_location_scale": 13, "student_t": 14, "beta": 15}


#: dynamic shared memory one CTA may opt in to on the H100 (227 KB), less 256 bytes for a kernel's static variables
CTA_SMEM_LIMIT = 227 * 1024 - 256


def _family_code(family) -> int:
    return family.code_id if hasattr(family, "code_id") else FAMILIES[family]


def _aligned16(t):
    """``t``, or a copy of it when its storage does not start on a 16-byte boundary (a view such as ``y[1:]``): the
    tensor-core kernel streams per-row arrays with TMA, which reads from 16-byte aligned addresses only."""
    return t.clone() if t.data_ptr() % 16 != 0 else t


def _split(rows: np.ndarray, shapes) -> List[np.ndarray]:
    """``rows[..., n]`` cut into consecutive pieces, piece i reshaped to ``rows.shape[:-1] + shapes[i]`` (views where
    the reshape allows; never a cast)."""
    lead, out, a = rows.shape[:-1], [], 0
    for s in shapes:
        n = int(np.prod(s))
        out.append(rows[..., a : a + n].reshape(lead + tuple(s)))
        a += n
    return out


class GlmShards(ShardModel):
    """The GLM segments that live on ONE GPU.

    Parameters
    ----------
    Xs, ys
        Per-segment design matrices ``[n_rows, P]`` (bf16, row-major) and responses ``[n_rows]``
        (float32).
    groups
        Intercept index of every segment.
    n_groups
        Total number of intercepts G in the federation.
    n_chains
        Parameter vectors evaluated per call (K).  ``K > 1`` needs the tensor-core kernel.
    kernel
        ``"simt"`` (one chain, any P % 8 == 0 up to 512), ``"tc"`` (wgmma + TMA: bf16, any P % 8 == 0 up to
        384 — the tile is padded to whole 128-feature blocks by TMA's zero fill —, up to 16 chains) or ``"auto"``.
    node_ids, n_nodes
        Keep the result PER NODE instead of summed: segment ``s`` is (part of) node ``node_ids[s]`` of
        an ``n_nodes`` federation and the reduced vector holds one ``[K][1 + G + P]`` block per node
        (every kernel: the tensor-core kernels route a chunk's sums to its node's block, the CUDA-core kernels flush
        at node boundaries into fixed-point accumulators).  ``evaluate`` still returns the sum; :meth:`per_node` and
        :class:`~pytensor_federated_b200.federation.NodeFederation` expose the blocks — the reference's
        one-Op-per-node pattern (``demo_model.py:28-36``) answered by one launch.
    offsets, weights
        Per-row data, ``None`` or one entry per segment: ``None`` (no offset / weight 1 for that segment) or a 1-D
        tensor of the segment's ``n_rows`` (converted once to contiguous, 16-byte aligned float32, as ``ys`` are; a
        tensor must already live on the device of X).  Every kernel evaluates

            eta_i = intercept[group] + x_i' beta + o_i,     LL = sum_i w_i ll(y_i, eta_i),
            dLL/dbeta = sum_i w_i r_i x_i,   dLL/dintercept[g] = sum_{i in g} w_i r_i,   r_i = dll/deta at eta_i,

        the family constants weighted with the rest: Gaussian rows give ``w (-d^2 / 2 - log(2 pi) / 2)``, Poisson
        rows still omit ``-lgamma(y + 1)``.  Offsets carry exposures (``log t`` for Poisson rates) and known
        per-row terms; weights carry binomial trial counts (``y = k / n``, ``w = n``), frequency and survey
        weights.  A row of weight 0 contributes exactly nothing, even if its ``y`` or offset is not finite (its X
        row must be finite), which masks rows (held-out folds, bad rows) without copying X.  Weights must be
        finite and >= 0, offsets finite wherever the weight is not 0.  ``w = 1, o = 0`` reproduces the plain
        model bit for bit on the ``tc``, ``simt`` and general-shape kernels.  The kernels read the tensors given
        here on every evaluation, as they read X and y.
    family, n_classes
        ``"logistic"``, ``"poisson"``, ``"gaussian"``, a :class:`CustomFamily`, or ``"multinomial"`` with
        ``n_classes=C``: softmax (categorical) regression over C classes.  ``ys`` then holds class labels
        ``0 .. C-1`` (stored as float32, so exact up to 2^24); every row of non-zero weight must carry an integer
        label in ``[0, C)``, a row of weight 0 may carry anything.  The inputs per call are ``intercept[G, C]`` (also
        ``[C]`` when G = 1) and ``beta[P, C]``, batched ``[K, G, C]`` and ``[K, P, C]``; gradients come back in the
        shapes of the inputs, and

            eta_ic = intercept[group, c] + x_i' beta[:, c],     LL = sum_i w_i (eta_{i, y_i} - logsumexp_c eta_ic).

        ``2 <= C <= 16`` and ``K * C <= 16``.  Only the bf16 tensor-core kernel evaluates this family (bf16 X,
        P % 8 == 0, 8 <= P <= 384, 16-byte aligned rows): ``kernel="simt"`` / ``"generic"``, :class:`Fp8GlmShards`
        and shapes outside these raise a ValueError, and so do ``offsets`` (an offset common to all classes
        cancels in the softmax).  The kernel runs the C classes of chain k as columns ``k C + c`` of a K C-chain
        launch, so a C-class model reads X once, like a C-chain logistic one.

        This full parameterisation is not identified without priors: adding one vector to every class column of
        ``(intercept, beta)`` leaves LL unchanged (its gradients sum to 0 over the classes).  A reference-category
        model is obtained by fixing one column (say class 0) at 0 and ignoring its gradient.

        ``"gaussian_scale"`` and ``"negative_binomial"`` learn a dispersion parameter: the inputs per call are
        ``(intercept, beta, log_dispersion)`` — ``intercept[G]`` (a scalar when G = 1), ``beta[P]`` and a scalar, batched
        ``[K, G]``, ``[K, P]`` and ``[K]`` — and the gradients come back in the same shapes.  With
        ``eta = intercept[group] + x' beta + o``:

            gaussian_scale, s = log sigma:   ll = -(d / sigma)^2 / 2 - s - log(2 pi) / 2,      d = y - eta
            negative_binomial, a = log alpha (NB2: mean mu = exp(eta), variance mu + mu^2 / alpha):
                ll = lgamma(y + alpha) - lgamma(alpha) + alpha log(alpha / (alpha + mu)) + y log(mu / (alpha + mu))

        The negative-binomial LL omits ``-lgamma(y + 1)``, as the Poisson family does, so as alpha -> inf it tends to
        the Poisson family's ``y eta - mu`` exactly (the Gaussian one keeps ``-log(2 pi) / 2`` like ``"gaussian"``,
        which it equals at s = 0).  Offsets (``log t`` exposures of count models) and weights work as for every family.
        Counts must be integers in ``[0, 2^24]`` on every row of non-zero weight.  Only the bf16 tensor-core kernel
        evaluates these families, with the shape limits of the multinomial one; ``n_classes`` is rejected.

        ``"ordinal"`` with ``n_classes=C`` is cumulative-logit (proportional-odds) regression over C ordered categories
        (PyMC's ``OrderedLogistic``, brms' ``cumulative("logit")``): Likert scales, severity grades, ratings.  ``ys``
        holds the categories ``0 .. C-1`` as float32, with the same label rules as the multinomial family.  The inputs
        per call are ``(intercept, beta, cutpoints)`` — ``intercept[G]`` (a scalar when G = 1), ``beta[P]`` and
        ``cutpoints[C-1]``, batched ``[K, G]``, ``[K, P]`` and ``[K, C-1]`` — and the gradients come back in the same
        shapes.  With ``eta = intercept[group] + x' beta + o``, ``c_{-1} = -inf`` and ``c_{C-1} = +inf``:

            P(y <= j) = sigmoid(c_j - eta),     LL = sum_i w_i log(sigmoid(c_{y_i} - eta_i) - sigmoid(c_{y_i - 1} - eta_i)).

        ``2 <= C <= 17`` and ``K * (C - 1) <= 16``; the kernel and shape limits are those of the multinomial family.
        Offsets and weights work as for every family (an offset shifts eta and does not cancel).  The intercepts and
        the cutpoints are not identified together: adding one number to all of them leaves LL unchanged, so with
        G = 1 one normally fixes ``intercept = 0``.  The kernel sees only ``intercept[g] - c_j``, rounded to float32:
        a chain whose rounded values are not strictly decreasing in j for every group (cutpoints that are not
        strictly increasing, or NaN) gets ``LL = -inf`` and zero gradients, and the other chains of the call are
        unaffected.  Nothing is raised, so a sampler can step there and reject the proposal.  To sample, use an
        ordered transform such as ``c = cumsum([c0, exp(d_1), ..., exp(d_{C-2})])`` and apply the chain rule to the
        cutpoint gradient on the host: ``dLL/dc0 = sum_j dLL/dc_j``, ``dLL/dd_m = exp(d_m) sum_{j >= m} dLL/dc_j``.

        ``"weibull"`` and ``"lognormal"`` are right-censored survival regression (accelerated failure time, as
        ``survreg`` and lifelines fit them, PyMC's ``pm.Censored`` and brms' ``y | cens(c)``): ``ys`` holds the
        times ``t > 0`` and ``events`` whether each row's event was observed.  With ``eta = intercept[group] + x' beta
        + o``, ``log T = eta + sigma eps`` and ``s = log sigma`` learned, the inputs and gradients are those of
        ``gaussian_scale``: ``(intercept, beta, log_dispersion)`` with ``log_dispersion = s``.  With ``z = (log t -
        eta) / sigma`` and ``delta`` = 1 for an event, 0 for a censored row (the event had not happened by ``t``):

            weibull (eps standard minimum-Gumbel):   ll = delta (z - s - log t) - e^z
            lognormal (eps ~ N(0, 1)):               ll = delta (-z^2 / 2 - s - log(2 pi) / 2 - log t)
                                                          + (1 - delta) log Phi(-z)

        The event rows' LL is the density of T, ``-log t`` included, so it equals ``scipy.stats.weibull_min(c=1 /
        sigma, scale=e^eta)`` and ``lognorm(s=sigma, scale=e^eta)``, ``logpdf`` for events and ``logsf`` for censored
        rows.  The Weibull shape is ``k = e^{-s}`` and its scale ``e^eta``; as a proportional-hazards model its
        coefficients are ``-beta / sigma``.  An offset shifts the location of log T; weights work as for every
        family, and a row of weight 0 may carry any time and event.  Times must be finite and > 0 and events 0 or 1
        on every row of non-zero weight.  ``events`` takes one entry per segment: ``None`` (every row an event) or a
        1-D tensor or array of 0 / 1 of the segment's rows (on the device of X, like ``offsets``); it is rejected
        for every other family.  The model keeps a float32 copy of the times with censored rows negated, which is
        what the kernel reads (the tensors passed in are not modified).  Only the bf16 tensor-core kernel evaluates
        these families, with the shape limits of the multinomial one; ``n_classes`` is rejected.

        ``"zero_inflated_poisson"`` and ``"zero_inflated_negative_binomial"`` are count models with excess zeros
        (brms' ``zero_inflated_poisson`` / ``zero_inflated_negbinomial``, PyMC's ``ZeroInflatedPoisson`` /
        ``ZeroInflatedNegativeBinomial``, R's ``pscl::zeroinfl``): insurance claims, species counts, visits, defects.
        Two linear predictors share the covariates: the count predictor ``eta = intercept[group] + x' beta + o`` (the
        offset goes into eta only, as in brms and pscl) and the zero-inflation logit ``zeta = zi_intercept[group] + x'
        zi_beta``.  ``pi = sigmoid(zeta)`` is the probability of a structural zero (brms' ``zi``; PyMC's ``psi`` is
        ``1 - pi``), and with f the Poisson(``mu = e^eta``) or NB2(``mu``, ``alpha = e^a``) pmf of the plain families:

            P(y = 0) = pi + (1 - pi) f(0),     P(y > 0) = (1 - pi) f(y).

        LL omits ``-lgamma(y + 1)`` on the rows with y > 0, as ``"poisson"`` and ``"negative_binomial"`` do; that
        constant is 0 at y = 0, so the plain families' per-row LL at y = 0 is exactly ``log f(0)`` and the mixture
        is exact.  The inputs per call are ``(intercept, beta, zi_intercept, zi_beta)``, shapes ``[G]``, ``[P]``,
        ``[G]`` and ``[P]`` (a scalar intercept when G = 1), and for the negative binomial a trailing scalar
        ``log_dispersion = log alpha``; batched with a leading K (at most 8).  Gradients come back in the shapes of
        the inputs.  Chain k runs as the kernel columns 2k (eta) and 2k + 1 (zeta) of a 2K-column launch, so X is
        read once for both predictors.  An intercept-only zero part (brms' ``zi ~ 1``) is ``zi_beta = 0``, held
        fixed (its gradient ignored); it costs the same launch.  Both parts are identified by the data only through
        the zeros: with few zeros or a zeta far below 0 the zero part is weakly identified, so give it a prior.
        Counts must be integers in ``[0, 2^24]`` on every row of non-zero weight; offsets and weights work as for
        every family.  Only the bf16 tensor-core kernel evaluates these families, with the shape limits of the
        multinomial one; ``n_classes``, ``events`` and ``hvp`` are rejected, and so is a shape whose 2K-column
        launch gets fewer than two pipeline stages (checked when an engine attaches the model).

        ``"gamma"`` and ``"inverse_gaussian"`` are regression for positive, right-skewed continuous responses with a
        model for the MEAN (R's ``Gamma(link="log")`` / ``inverse.gaussian(link="log")``, brms' ``Gamma`` /
        ``inverse.gaussian``, PyMC's ``Gamma`` / ``Wald``): claim severities, costs, incomes, amounts, concentrations,
        durations.  The inputs and gradients are those of ``negative_binomial``: ``(intercept, beta,
        log_dispersion)``, one chain or batched.  With ``eta = intercept[group] + x' beta + o``, ``mu = e^eta`` is the
        mean of y, and ``a = log_dispersion`` is the log of the SHAPE (a larger shape, less dispersion, as ``log
        alpha`` of the negative binomial).  With ``z = log y - eta``:

            gamma, nu = e^a, Var(y) = mu^2 / nu:
                ll = nu (1 + z - e^z) + nu log nu - nu - lgamma(nu) - log y
            inverse_gaussian, lambda = e^a, Var(y) = mu^3 / lambda:
                ll = a / 2 - log(2 pi) / 2 - (3/2) log y - lambda (y - mu)^2 / (2 mu^2 y)

        LL is the full density, ``-log y`` terms included, so it equals ``scipy.stats.gamma(a=nu, scale=mu /
        nu).logpdf(y)`` and ``scipy.stats.invgauss(mu=mu / lambda, scale=lambda).logpdf(y)``.  At ``a = 0`` the gamma
        family is the exponential distribution with mean mu.  Responses must be finite and > 0 on every row of
        non-zero weight (a row of weight 0 may carry any y); offsets and weights work as for every family.  Only the
        bf16 tensor-core kernel evaluates these families, with the shape limits of the multinomial one;
        ``n_classes``, ``events`` and ``hvp`` are rejected.

        ``"gaussian_location_scale"`` and ``"student_t"`` are location-scale (distributional) regression for a
        continuous response on the real line: the scale gets its own linear predictor (brms' ``bf(y ~ x, sigma ~
        x)``, GAMLSS, per-group variances), and ``student_t`` is robust regression with learned degrees of freedom
        (PyMC's robust linear regression, brms' ``student()``), whose bounded influence keeps gross outliers from
        pulling beta.  The mean ``mu = intercept[group] + x' beta + o`` (identity link; the offset goes into mu only)
        and ``s = log sigma = sigma_intercept[group] + x' sigma_beta``.  With ``z = (y - mu) e^-s``:

            gaussian_location_scale:   ll = -z^2 / 2 - s - log(2 pi) / 2
            student_t, nu = e^a:       ll = lgamma((nu + 1) / 2) - lgamma(nu / 2) - log(nu pi) / 2 - s
                                            - (nu + 1) / 2 log1p(z^2 / nu)

        LL is the full density: it equals ``scipy.stats.norm(mu, sigma).logpdf(y)`` and ``scipy.stats.t(df=nu,
        loc=mu, scale=sigma).logpdf(y)``.  At nu = 1 Student-t is the Cauchy distribution, and as nu grows it tends to
        the Gaussian family.  The inputs per call are ``(intercept, beta, sigma_intercept, sigma_beta)``, shapes
        ``[G]``, ``[P]``, ``[G]`` and ``[P]`` (a scalar intercept when G = 1), and for Student-t a trailing scalar
        ``log_dispersion = log nu``; batched with a leading K (at most 8).  Gradients come back in the shapes of the
        inputs.  Chain k runs as the kernel columns 2k (mu) and 2k + 1 (s) of a 2K-column launch, so X is read once
        for both predictors.  A constant scale is ``sigma_beta = 0``, held fixed (its gradient ignored); it costs the
        same launch.  Responses must be finite on every row of non-zero weight (a row of weight 0 may carry any y);
        offsets and weights work as for every family.  Only the bf16 tensor-core kernel evaluates these families, with
        the shape limits of the multinomial one; ``n_classes``, ``events`` and ``hvp`` are rejected, and so is a shape
        whose 2K-column launch gets fewer than two pipeline stages (checked when an engine attaches the model).

        ``"beta"`` is beta regression for continuous proportions strictly between 0 and 1 (Ferrari and Cribari-Neto;
        R's ``betareg``, brms' ``Beta()``, statsmodels' ``BetaModel``): market shares, budget fractions, percent
        cover, pass rates, allele frequencies.  The family name is not the coefficient input ``beta``.  The inputs and
        gradients are those of ``negative_binomial``: ``(intercept, beta, log_dispersion)``, one chain or batched.
        With ``eta = intercept[group] + x' beta + o``, the mean is ``mu = sigmoid(eta)`` (logit link), and ``a =
        log_dispersion`` is the log of the PRECISION phi (a larger phi, less dispersion: ``Var(y) = mu (1 - mu) / (1 +
        phi)``, as the log shape of ``gamma``).  With ``A = mu phi`` and ``B = (1 - mu) phi``:

            ll = lgamma(phi) - lgamma(A) - lgamma(B) + (A - 1) log y + (B - 1) log(1 - y)

        LL is the full density: it equals ``scipy.stats.beta(a=A, b=B).logpdf(y)``.  Unlike logistic regression on
        fractional y (quasi-binomial), it is a density with a learned dispersion, so the posterior's width follows the
        data.  Responses must be finite with ``0 < y < 1`` on every row of non-zero weight (a row of weight 0 may carry
        any y, 0 and 1 included); offsets and weights work as for every family.  Only the bf16 tensor-core kernel
        evaluates this family, with the shape limits of the multinomial one; ``n_classes``, ``events`` and ``hvp``
        are rejected.
    events
        Per-row event indicators of the survival families (see ``family``).
    hvp
        Hessian-vector products of the ``"logistic"``, ``"poisson"`` and ``"gaussian"`` families.  The inputs per
        call are ``(intercept, beta, v_intercept, v_beta)``: the parameters and a direction ``v``, shapes ``[G]``,
        ``[P]``, ``[G]`` and ``[P]`` (a scalar intercept when G = 1), batched with a leading ``K = n_chains`` (at most
        8).  ``evaluate`` returns ``[LL, d_intercept, d_beta, Hv_intercept, Hv_beta]``: the last two are NOT gradients
        with respect to ``v`` but the product ``H v`` of the Hessian of LL (negative semidefinite for these families)
        at ``(intercept, beta)`` with ``v``.  With ``h = ll''(eta)`` (logistic ``-mu (1 - mu)``, Poisson ``-mu``,
        Gaussian ``-1``) and ``u_i = v_intercept[group] + x_i' v_beta`` (no offset: u is linear in v),

            (H v)_intercept[g] = sum_{i in g} w_i h_i u_i,     (H v)_beta = sum_i w_i h_i u_i x_i.

        Pair k runs as the kernel columns 2k (the parameters) and 2k + 1 (the direction) of a 2K-column launch, so
        X is read once for K products.  Offsets and weights work as for every family (a row of weight 0 gives exactly
        0).  Only the bf16 tensor-core kernel evaluates products: any other family, ``kernel`` other than ``"auto"``
        or ``"tc"``, :class:`Fp8GlmShards`, shapes outside that kernel's limits, ``n_chains > 8`` and a shape whose
        2K-column launch gets fewer than two pipeline stages (checked when an engine attaches the model) raise a
        ValueError.  :func:`~pytensor_federated_b200.sampling.glm_hessian` assembles the full Hessian from
        ``ceil((G + P) / K)`` launches.
    """

    def __init__(
        self,
        Xs: Sequence,
        ys: Sequence,
        *,
        groups: Optional[Sequence[int]] = None,
        n_groups: int = 1,
        family: str = "logistic",
        n_chains: int = 1,
        kernel: str = "auto",
        scales: Optional[Sequence] = None,
        node_ids: Optional[Sequence[int]] = None,
        n_nodes: Optional[int] = None,
        offsets: Optional[Sequence] = None,
        weights: Optional[Sequence] = None,
        n_classes: Optional[int] = None,
        events: Optional[Sequence] = None,
        hvp: bool = False,
    ) -> None:
        import torch

        if len(Xs) != len(ys):
            raise ValueError("Xs and ys must have the same length")
        self.Xs = list(Xs)
        self.ys = [_aligned16(y.to(torch.float32).contiguous()) for y in ys]
        self.weights = self._row_data(weights, "weights")
        self.offsets = self._row_data(offsets, "offsets")
        for si, (o, w) in enumerate(zip(self.offsets, self.weights)):
            if w is not None and not bool(torch.all(torch.isfinite(w) & (w >= 0))):
                raise ValueError(f"weights of segment {si} must be finite and >= 0")
            if o is not None:
                bad = ~torch.isfinite(o)
                if w is not None:
                    bad &= w != 0   # a masked row may carry anything
                if bool(torch.any(bad)):
                    raise ValueError(f"offsets of segment {si} must be finite on every row of non-zero weight")
        self.scales = list(scales) if scales is not None else None
        self.groups = list(groups) if groups is not None else [0] * len(Xs)
        self.n_groups = int(n_groups)
        self.family = family
        self.n_chains = int(n_chains)
        self.kernel = kernel
        X0 = self.Xs[0]
        self.n_features = int(X0.shape[1])
        self.ld = int(X0.stride(0))
        for X in self.Xs:
            if X.dim() != 2 or X.shape[1] != self.n_features or X.stride(1) != 1 or X.stride(0) != self.ld:
                raise ValueError("all design matrices must be row-major [n, P] with one row stride")
        self.device = X0.device
        if (node_ids is None) != (n_nodes is None):
            raise ValueError("node_ids and n_nodes come together")
        self.node_ids = list(node_ids) if node_ids is not None else None
        self.n_nodes = int(n_nodes) if n_nodes is not None else 1
        if self.node_ids is not None and (len(self.node_ids) != len(self.Xs) or not all(0 <= i < self.n_nodes for i in self.node_ids)):
            raise ValueError("node_ids needs one node index in [0, n_nodes) per segment")
        #: Hessian-vector products: every call also takes a direction per chain (see ``hvp``)
        self.hvp = bool(hvp)
        layout = _Hvp if self.hvp else (_LAYOUTS.get(family, _Scalar) if isinstance(family, str) else _Scalar)
        if events is not None and not layout.takes_events:
            raise ValueError(f"events= is for family='weibull' or 'lognormal' only, not {family!r}")
        #: per-row event indicators of the survival families (one float32 tensor or None per segment)
        self.events = self._row_data(events, "events")
        self._layout = lay = layout(self, n_classes)
        #: classes per chain (multinomial and ordinal families; 1 for every other family)
        self.n_classes = lay.n_classes
        #: per-chain shapes of the inputs, in order: ``(intercept, beta)`` or ``(intercept, beta, third)``
        self.input_shapes = lay.shapes
        self.n_inputs = len(lay.shapes)
        self.n_params = sum(int(np.prod(s)) for s in lay.shapes)
        #: columns of one launch: K, times C for the multinomial family, times C - 1 for the ordinal one
        self.kernel_chains = self.n_chains * lay.columns
        self.n_theta_words = self.kernel_chains * lay.words
        self.n_vals = self.n_nodes * self.kernel_chains * (1 + lay.words)

    def _row_data(self, entries, name: str) -> list:
        """One contiguous float32 tensor (or None) per segment, on the device of the segment's X."""
        import torch

        if entries is None:
            return [None] * len(self.Xs)
        entries = list(entries)
        if len(entries) != len(self.Xs):
            raise ValueError(f"{name} needs one entry (None or a tensor) per segment: got {len(entries)} for {len(self.Xs)}")
        out = []
        for si, (v, X) in enumerate(zip(entries, self.Xs)):
            if v is None:
                out.append(None)
                continue
            if isinstance(v, torch.Tensor):
                if v.device != X.device:
                    raise ValueError(f"{name} of segment {si} are on device {v.device}, its X on {X.device}")
            else:
                v = torch.as_tensor(np.asarray(v), device=X.device)
            if v.dim() != 1 or v.shape[0] != X.shape[0]:
                raise ValueError(f"{name} of segment {si} must be 1-D with {X.shape[0]} rows, got shape {tuple(v.shape)}")
            out.append(_aligned16(v.to(torch.float32).contiguous()))
        return out

    @property
    def has_row_data(self) -> bool:
        """Whether some segment has offsets or weights."""
        return any(v is not None for v in self.offsets + self.weights)

    @property
    def n_rows(self) -> int:
        return int(sum(X.shape[0] for X in self.Xs))

    # -- packing ---------------------------------------------------------------------------
    #: call context of the most recent single-threaded ``pack_theta`` / ``reference_partial`` / ``eager_partial``
    #: (before any: unbatched, scalar shapes, no unordered chains); the engine passes the context explicitly instead
    _last_ctx = (False, (), (), ())

    def call_context(self, inputs):
        """``(batched, intercept shape)`` of one call: ``beta`` with one more axis than its per-chain shape means one
        row per chain.  Three-input families add the shape of the third input; the ordinal family then adds the
        chains whose cutpoints are not ordered."""
        return self._layout.call_context(inputs)

    def pack_theta(self, inputs, out: np.ndarray):
        ctx = self._last_ctx = self._layout.pack(inputs, out)
        return ctx

    def inputs_from_words(self, words: np.ndarray):
        """Theta words -> inputs of one call (the peers of the collective backend).  The ordinal family's words carry
        only ``intercept - c_j``, so its inputs come back shifted to ``c_0 = 0`` (the likelihood does not see the
        shift; they pack back to the same words)."""
        return self._layout.inputs_from_words(words)

    def inputs_from_theta(self, theta: np.ndarray) -> List[np.ndarray]:
        """The inputs held in flat parameter rows ``theta[..., n_params]`` (each input flattened row-major, in
        order): input i gets shape ``theta.shape[:-1] + input_shapes[i]``, so ``[K, n_params]`` gives a batched
        call and ``[n_params]`` an unbatched one.  Views where possible; the dtype is kept."""
        return _split(np.asarray(theta), self.input_shapes)

    def gradients_from_row(self, row: np.ndarray, shapes) -> List[np.ndarray]:
        """The gradients in result rows ``[..., 1 + n_params]`` (``[LL, gradients]`` as :meth:`per_node` gives
        them), in the order of the inputs and as fresh arrays: gradient i gets ``shapes[i]``, or where that is None
        the rows' leading axes and the input's per-chain shape."""
        return [(g if s is None else g.reshape(s)).copy() for g, s in zip(_split(row[..., 1:], self.input_shapes), shapes)]

    def per_node(self, vals: np.ndarray, ctx=None) -> np.ndarray:
        """The reduced vector as ``[n_nodes, n_chains, 1 + n_params]``: ``[LL, gradients]`` per node and chain, the
        gradients flattened row-major in the order of the inputs (multinomial: ``[LL, d intercept (G, C), d beta
        (P, C)]``, summed from the kernel's blocks of the chain's C classes; ordinal: ``[LL, d intercepts, d beta,
        d cutpoints]`` from the kernel's blocks ``[LL_j, gi_j[G], g_j[P]]`` of the chain's C - 1 cutpoints, with
        ``d c_j = -sum_g gi_j[g]``).  Ordinal chains that ``ctx`` (the call context, by default that of the last
        ``pack_theta``) marks as unordered get ``LL = -inf`` and zero gradients."""
        raw = np.asarray(vals, dtype=np.float64).reshape(self.n_nodes, self.kernel_chains, 1 + self._layout.words)
        return self._layout.fold(raw, self._last_ctx if ctx is None else ctx)

    def unpack_result(self, vals: np.ndarray, ctx=None) -> List[np.ndarray]:
        ctx = self._last_ctx if ctx is None else ctx
        batched, icpt_shape = ctx[0], ctx[1]
        v = self.per_node(vals, ctx).sum(axis=0)                    # [K, 1 + n_params]
        if not batched:
            v = v[0]
        # the intercept's gradient in the shape it was passed (chains leading when batched), beta's in the model's
        # shape, a third input's in its shape
        shapes = [(self.n_chains,) + tuple(icpt_shape[1:]) if batched else icpt_shape, None, *ctx[2 : self.n_inputs]]
        return [np.array(v[..., 0]), *self.gradients_from_row(v, shapes)]

    # -- native ----------------------------------------------------------------------------
    def use_tensor_cores(self):
        """Kernel selector passed to the runtime: 0 = SIMT, 1 = tensor cores (bf16), 2 = block-scaled fp8,
        3 / 4 = general-shape fallback (bf16 / fp32 design matrix).  Raises ValueError for a CUDA-core model whose
        shared memory would exceed what one CTA can have."""
        code = self._select_kernel()
        if code in (0, 3, 4) and self.cuda_core_smem_bytes(code) > CTA_SMEM_LIMIT:
            fits, too_many = 0, self.n_groups   # the most groups that fit (bytes grow with the group count)
            while too_many - fits > 1:
                mid = (fits + too_many) // 2
                fits, too_many = (mid, too_many) if self.cuda_core_smem_bytes(code, mid) <= CTA_SMEM_LIMIT else (fits, mid)
            raise ValueError(
                f"the CUDA-core GLM kernels keep theta and one accumulator per group in shared memory: {self.n_groups} "
                f"groups with {self.n_features} features need {self.cuda_core_smem_bytes(code)} bytes, more than the "
                f"{CTA_SMEM_LIMIT} a CTA can have; at most {fits} groups fit")
        return code

    def cuda_core_smem_bytes(self, code: int, n_groups: Optional[int] = None) -> int:
        """Dynamic shared memory of one CTA of the SIMT (``code`` 0) or general-shape (3, 4) kernel, by the
        formulas of ``b200_glm_simt_smem`` (csrc/glm_simt.cu) and ``launch_generic`` (csrc/glm_generic.cu),
        for this model or for the same model with ``n_groups`` groups."""
        G = self.n_groups if n_groups is None else int(n_groups)
        n_theta = self.n_theta_words + (G - self.n_groups) * self.kernel_chains
        P = self.n_features
        if code == 0:
            per_warp = ((P + 255) // 256) * 256
        else:
            j = (P + 31) // 32
            per_warp = (8 if j <= 8 else 16 if j <= 16 else 32) * 32
        return ((n_theta + 3) & ~3) * 4 + 8 * per_warp * 4 + ((G + 1) & ~1) * 8 + 32 * 8

    def _select_kernel(self) -> int:
        import torch

        X0 = self.Xs[0]
        if hasattr(self.family, "code_id"):  # user-compiled likelihood: general-shape kernel
            if X0.dtype not in (torch.bfloat16, torch.float32) or self.n_chains != 1 or self.n_features > 1024:
                raise ValueError("custom likelihoods need a bf16/fp32 design matrix, one chain and P <= 1024")
            return 3 if X0.dtype == torch.bfloat16 else 4
        bf16 = X0.dtype == torch.bfloat16
        tc_ok = (bf16 and self.n_features % 8 == 0 and 8 <= self.n_features <= 384 and self.n_chains <= 16
                 and all(X.data_ptr() % 16 == 0 for X in self.Xs) and self.ld % 8 == 0)
        if self._layout.tc_only:   # the bf16 tensor-core kernel or nothing: no other kernel has these families
            if not tc_ok:
                raise ValueError(f"the {self.family} family runs on the bf16 tensor-core kernel only, which needs a bf16 "
                                 f"design matrix with P % 8 == 0, 8 <= P <= 384 and 16-byte aligned rows (got "
                                 f"{X0.dtype}, P = {self.n_features}, row stride {self.ld}) and at most 16 chains")
            return 1
        if self.kernel == "fp8":
            return 2
        if self.kernel == "tc":
            return 1
        if self.kernel == "simt":
            return 0
        generic = 3 if X0.dtype == torch.bfloat16 else (4 if X0.dtype == torch.float32 else None)
        if self.kernel == "generic":
            if generic is None:
                raise ValueError("the general-shape kernel needs a bf16 or fp32 design matrix")
            return generic
        # auto: the tensor-core kernel wherever its shape constraints hold (it is faster even for one chain:
        # TMA streaming + the X tile reused from smem for both GEMMs), then SIMT, then the general kernel
        if tc_ok:
            return 1
        if self.n_chains > 1:
            raise ValueError("multi-chain evaluation needs the tensor-core kernel (bf16, P % 8 == 0, P <= 384, K <= 16)")
        simt_ok = (bf16 and self.n_features % 8 == 0 and self.n_features <= 512 and self.ld % 8 == 0
                   and all(X.data_ptr() % 16 == 0 for X in self.Xs))
        if simt_ok:
            return 0
        if generic is not None and self.n_features <= 1024:
            return generic
        raise ValueError(f"no fused GLM kernel for dtype {X0.dtype} with {self.n_features} features; "
                         "serve this model through ArraysToArraysService instead")

    def attach(self, lib, handle) -> None:
        from ..ops import native

        n = len(self.Xs)
        Xp = native.void_p_array([X.data_ptr() for X in self.Xs])
        yp = native.void_p_array([y.data_ptr() for y in self._layout.kernel_ys])
        kernel_scales = getattr(self, "_kernel_scales", None) or self.scales   # fp8: packed per tile
        sp = native.void_p_array([s.data_ptr() for s in kernel_scales]) if kernel_scales else None
        rows = (C.c_longlong * n)(*[X.shape[0] for X in self.Xs])
        grp = (C.c_int * n)(*self.groups)
        code = int(self.use_tensor_cores())
        if self._layout.pairs:
            # the 2K-column launch must get two TMA stages; refused here, before the engine's model changes
            row_data = (1 if any(o is not None for o in self.offsets) else 0) | (2 if any(w is not None for w in self.weights) else 0)
            fam = _family_code(self.family) | (HVP_FLAG if self.hvp else 0)
            if int(lib.b200_glm_tc_stages(self.n_features, self.kernel_chains, self.n_groups, fam, row_data)) < 2:
                what = "hvp=True" if self.hvp else f"family={self.family!r}"
                raise ValueError(f"{what} with {self.n_chains} pairs at P = {self.n_features}: the tensor-core kernel's "
                                 f"{self.kernel_chains}-column launch gets fewer than two pipeline stages in shared memory; "
                                 f"use fewer pairs per launch")
        #: which fused kernel serves this model ("tc" / "fp8" = wgmma tensor cores, else CUDA cores)
        self.selected_kernel = {0: "simt", 1: "tc", 2: "fp8", 3: "generic-bf16", 4: "generic-fp32"}[code]
        if self.kernel == "auto" and code not in (1, 2) and not hasattr(self.family, "code_id"):
            import logging

            logging.getLogger(__name__).warning(
                "GLM with %d features (%s, row stride %d) is outside the tensor-core kernel's shapes (bf16, P %% 8 == 0, "
                "P <= 384, 16-byte aligned rows): using the %s CUDA-core kernel — single pass, but slower",
                self.n_features, self.Xs[0].dtype, self.ld, self.selected_kernel)
        out_grp = (C.c_int * n)(*self.node_ids) if self.node_ids is not None else None
        op = native.void_p_array([o.data_ptr() if o is not None else 0 for o in self.offsets]) \
            if any(o is not None for o in self.offsets) else None
        wp = native.void_p_array([w.data_ptr() if w is not None else 0 for w in self.weights]) \
            if any(w is not None for w in self.weights) else None
        native.check(
            lib.b200_engine_set_glm(
                handle, n, Xp, yp, sp, rows, grp, self.n_features, self.ld, self.n_groups,
                self.kernel_chains, _family_code(self.family) | (HVP_FLAG if self.hvp else 0), code, out_grp, self.n_nodes, op, wp,
                self.n_classes,
            ),
            "set_glm",
        )
        if hasattr(self.family, "code_id"):
            lib.b200_engine_set_custom_launcher(handle, C.c_void_p(self.family.launcher_address()))
        #: whether the tensor-core kernel reads X in its packed 12-bit form (see :func:`pack_x12`)
        self.packed_x = False
        if code == 1 and os.environ.get("B200FED_NO_PACKED_X", "0") in ("", "0"):
            row_data = (1 if any(o is not None for o in self.offsets) else 0) | (2 if any(w is not None for w in self.weights) else 0)
            fam = _family_code(self.family) | (HVP_FLAG if self.hvp else 0)
            slots = int(lib.b200_glm_tc_packed_slots(self.n_features, self.kernel_chains, self.n_groups, fam, row_data,
                                                     self.n_theta_words))
            if slots >= 2 and self._packing_pays(row_data):
                packs = self._packed()
                if packs is not None:
                    tabs = (C.c_uint * (4 * n))(*[w for _, _, t in packs for w in t])
                    native.check(lib.b200_engine_set_glm_packed(
                        handle, n, native.void_p_array([p.data_ptr() for p, _, _ in packs]),
                        native.void_p_array([f.data_ptr() for _, f, _ in packs]), tabs), "set_glm_packed")
                    self.packed_x = True

    _packs = None            # the packed X, once made
    _packs_refused = False   # some tile of X has more exceptions than its footer holds: X never packs

    def _packing_pays(self, row_data: int) -> bool:
        """Whether packed X is faster for this launch shape, as measured (docs/KERNELS.md, "Packed X"): launches of up to
        4 kernel columns with the tile padded to 256 features (129 <= P <= 256).  At 16 columns the consumer chain binds
        and at P <= 128 the bf16 layout has 4 stages to the packed one's 2: both were measured slower packed, and 8
        columns were not measured, so those launches read X as bf16."""
        return (self.n_features + 127) // 128 == 2 and self.kernel_chains <= X12_MAX_COLUMNS

    def _packed(self):
        """The packed form of every segment's X (made once, kept with the model), or None where some segment's X does
        not pack (a tile with more exceptions than its footer holds: remembered, X does not change) or the device
        lacks the memory for it now (tried again at the next attach); the kernel then reads X itself."""
        import logging

        import torch

        if self._packs is not None or self._packs_refused:
            return self._packs
        log = logging.getLogger(__name__)
        need = sum(x12_packed_bytes(X.shape[0], self.n_features) for X in self.Xs)
        free, _ = torch.cuda.mem_get_info(self.device)
        if need + (2 << 30) > free:   # headroom for the packing's temporaries
            log.warning("not packing X: it needs %.1f GB and %.1f GB are free; the kernel reads the bf16 matrix",
                        need / 1e9, free / 1e9)
            return None
        packs = []
        for si, X in enumerate(self.Xs):
            p = pack_x12(X[:, : self.n_features])
            if p is None:
                log.warning("not packing X: a tile of segment %d has more than %d values outside its table", si,
                            X12_MAX_EXCEPTIONS)
                self._packs_refused = True
                return None
            packs.append(p)
        self._packs = packs
        return packs

    # -- eager oracle (also the compute step of the NCCL baseline) ---------------------------
    def reference_partial(self, inputs, *, dtype=None, chunk_rows: int = 1 << 20) -> np.ndarray:
        """This node's partial with stock PyTorch ops (oracle of the kernels, compute step of the CPU / gloo
        path), in the kernel's layout (:meth:`per_node` folds it).  Rows are processed ``chunk_rows`` at a time (a
        multiple of 128), so an fp64 oracle of a 10M-row shard needs 2 GB of scratch, not 20."""
        import torch

        self._last_ctx = self.call_context(inputs)
        return self._partial(inputs, dtype=dtype or torch.float32, chunk_rows=chunk_rows)

    def eager_partial(self, inputs) -> np.ndarray:
        """Stock-PyTorch evaluation as a practitioner would write it: two bf16 GEMMs (X @ beta, then
        r @ X) plus elementwise ops — the compute step of the NCCL baseline ("baseline B").  Reads the
        design matrix twice; no custom kernels."""
        import torch

        if self.Xs[0].dtype != torch.bfloat16:
            return self.reference_partial(inputs)
        self._last_ctx = self.call_context(inputs)
        return self._layout.baseline(self, inputs)

    def _partial(self, inputs, *, dtype, chunk_rows: int, bf16_gemms: bool = False) -> np.ndarray:
        """The partial in the kernel's layout ``[n_nodes][kernel_chains][1 + G + P (+ 1)]``, from the family's
        per-row terms (``_Layout.oracle``) in ``dtype``.  ``bf16_gemms``: the collective baseline, eta and the beta
        gradient from bf16 GEMMs of the stored matrix (one per column of eta: the ordinal family puts
        ``X' (sum_j r_j)`` in the block of cutpoint 0 and the host sums the blocks); else the oracle, from the
        dequantised rows."""
        import torch

        lay = self._layout
        icpt, beta, terms = lay.oracle(inputs, self.device, dtype)   # [G, E], [P, E]: E columns of eta
        icpt = icpt.to(self.device, dtype)
        B = beta.to(self.device, torch.bfloat16 if bf16_gemms else dtype)
        G, P = self.n_groups, self.n_features
        step = self.kernel_chains // B.shape[1]   # kernel columns per column of eta
        full = torch.zeros(self.n_nodes, self.kernel_chains, 1 + lay.words, dtype=torch.float64, device=self.device)
        for si, (X, y, g) in enumerate(zip(self.Xs, lay.kernel_ys, self.groups)):
            out = full[self.node_ids[si] if self.node_ids is not None else 0]
            w = self.weights[si]
            for r0 in range(0, X.shape[0], chunk_rows):
                r1 = min(X.shape[0], r0 + chunk_rows)
                if bf16_gemms:
                    Xf = X[r0:r1]
                    eta = (Xf @ B).to(dtype)
                else:
                    Xf = self._dequant_rows(si, r0, r1).to(dtype)
                    eta = Xf @ B
                eta = eta + icpt[g]
                if self.offsets[si] is not None:
                    cols = lay.offset_columns
                    eta[:, cols] = eta[:, cols] + self.offsets[si][r0:r1].to(dtype).unsqueeze(1)
                # ll, r (and the dispersion families' q = dll/dlog_dispersion), [n, K] or [n, K, columns]
                ll, r, *q = self._weigh(si, r0, r1, *terms(y[r0:r1], None if w is None else w[r0:r1], eta))
                out[:, 0] += ll.double().sum(0).reshape(-1)
                out[:, 1 + g] += r.double().sum(0).reshape(-1)
                if not bf16_gemms:
                    out[:, 1 + G : 1 + G + P] += (r.reshape(r1 - r0, -1).T @ Xf).double()
                elif step == 1:
                    out[:, 1 + G : 1 + G + P] += (r.reshape(r1 - r0, -1).T.to(torch.bfloat16) @ Xf).double()
                else:
                    out[::step, 1 + G : 1 + G + P] += (r.sum(2).T.to(torch.bfloat16) @ Xf).double()
                for t in q:
                    out[:, 1 + G + P] += t.double().sum(0).reshape(-1)
        return full.reshape(-1).cpu().numpy()

    def _weigh(self, seg: int, r0: int, r1: int, *terms):
        """``w t`` for each per-row term ``t`` of rows ``[r0, r1)`` of segment ``seg``; rows of weight 0 give exactly 0
        (a select, not a product: their terms may be NaN)."""
        import torch

        w = self.weights[seg]
        if w is None:
            return terms
        ww = w[r0:r1].to(terms[0].dtype).reshape((-1,) + (1,) * (terms[0].dim() - 1))   # broadcast over chains
        keep = ww != 0
        return [torch.where(keep, ww * t, torch.zeros_like(t)) for t in terms]

    def _dequant_rows(self, seg: int, r0: int, r1: int):
        """Rows ``[r0, r1)`` of segment ``seg`` as stored values (dense kernels: the matrix itself)."""
        return self.Xs[seg][r0:r1]

    def _dequant(self, X):
        return X

    def _row_data_bytes(self) -> int:
        """Bytes of offsets and weights read per evaluation (4 per row per vector present)."""
        return int(sum(4 * v.shape[0] for v in self.offsets + self.weights if v is not None))

    def bytes_per_eval(self) -> int:
        """Bytes the kernel reads per evaluation: X (or its packed form, blocks and footers of every tile the kernel
        visits), y and the row data."""
        if getattr(self, "packed_x", False):
            xb = sum(x12_packed_bytes(X.shape[0], self.n_features) for X in self.Xs)
            return int(xb + sum(4 * X.shape[0] for X in self.Xs)) + self._row_data_bytes()
        return int(sum(X.shape[0] * (self.n_features * X.element_size() + 4) for X in self.Xs)) + self._row_data_bytes()

    def flops_per_eval(self) -> int:
        return int(4 * self.n_rows * self.n_features * self.kernel_chains)


# -- packed X: a lossless 12-bit form of a bf16 design matrix (csrc/glm_tc.cu, "Packed X") ----------------------
X12_BLOCK = 128 * 64 * 3 // 2   # bytes per (128-row tile, 64-feature panel): 8192 low bytes + 8192 4-bit codes
X12_FOOT = 256                  # bytes of a tile's exception footer: count, then (position << 8 | high byte) words
X12_MAX_EXCEPTIONS = X12_FOOT // 4 - 1
X12_MAX_COLUMNS = 4             # kernel columns up to which a launch reads X packed (GlmShards._packing_pays)


def x12_tiles(n_rows: int) -> int:
    """Tiles the packed form of an n-row segment holds: the tensor-core kernel's chunks visit an even number."""
    t = (n_rows + 127) // 128
    return t + (t & 1)


def x12_packed_bytes(n_rows: int, n_features: int) -> int:
    return x12_tiles(n_rows) * (((n_features + 127) // 128 * 2) * X12_BLOCK + X12_FOOT)


def pack_x12(X, chunk_rows: int = 1 << 17):
    """The packed form of one segment's bf16 matrix ``X[n, P]``, on its device: ``(blocks, footers, table)``.

    The 16-entry table of high bytes (sign and upper 7 exponent bits) holds 0x00 in entry 0 (padding: rows past n
    and features past P are +0), the 14 most frequent other high bytes of X in entries 1-14, and code 15 marks an
    exception.  ``blocks`` is uint8 ``[tiles, panels, 12288]``: per 128-row tile and 64-feature panel the low bytes
    in row-major order, then the codes two per byte (the even feature in the low nibble).  ``footers`` is int32
    ``[tiles, 64]``: the tile's exception count, then ``position << 8 | high byte`` with position = panel * 8192 +
    row * 64 + feature, in increasing order.  ``table`` is the 4 little-endian words of the table.  Returns None
    when a tile has more than 63 exceptions.  Works through ``chunk_rows`` rows (a multiple of 128) at a time."""
    import torch

    n, P = X.shape
    PP = (P + 127) // 128 * 128
    panels = PP // 64
    tiles = x12_tiles(n)
    dev = X.device
    hist = torch.zeros(256, dtype=torch.long, device=dev)
    for r0 in range(0, n, chunk_rows):
        hb = (X[r0 : r0 + chunk_rows].contiguous().view(torch.int16) >> 8) & 0xFF
        hist += torch.bincount(hb.reshape(-1).long(), minlength=256)
    hist[0] = -1   # entry 0 is 0x00 whatever its count
    order = torch.argsort(hist, descending=True, stable=True)[:14].tolist()
    counts = hist.tolist()
    entries = [0] + [b for b in order if counts[b] > 0]
    entries += [0] * (16 - len(entries))
    lut = torch.full((256,), 15, dtype=torch.uint8, device=dev)
    for code in range(15 - 1, -1, -1):   # entries past the used ones repeat 0x00, which keeps code 0
        lut[entries[code]] = code
    table = [int.from_bytes(bytes(entries[4 * q : 4 * q + 4]), "little") for q in range(4)]

    blocks = torch.empty(tiles, panels, X12_BLOCK, dtype=torch.uint8, device=dev)
    foot = torch.zeros(tiles, X12_FOOT // 4, dtype=torch.int32, device=dev)
    for r0 in range(0, tiles * 128, chunk_rows):
        rows = min(chunk_rows, tiles * 128 - r0)
        nt = rows // 128
        t0 = r0 // 128
        v = torch.zeros(rows, PP, dtype=torch.int16, device=dev)
        valid = max(0, min(n, r0 + rows) - r0)
        if valid:
            v[:valid, :P] = X[r0 : r0 + valid].view(torch.int16)
        v = v.view(nt, 128, panels, 64).permute(0, 2, 1, 3)                    # [tile, panel, row, feature]
        hb = ((v >> 8) & 0xFF).to(torch.uint8)
        code = lut[hb.long()]
        blocks[t0 : t0 + nt, :, : 8192] = (v & 0xFF).to(torch.uint8).reshape(nt, panels, 8192)
        blocks[t0 : t0 + nt, :, 8192 :] = (code[..., 0::2] | (code[..., 1::2] << 4)).reshape(nt, panels, 4096)
        ex = (code == 15).reshape(nt, panels * 8192)
        cnt = ex.sum(1)
        if int(cnt.max()) > X12_MAX_EXCEPTIONS:
            return None
        foot[t0 : t0 + nt, 0] = cnt.to(torch.int32)
        tile, pos = ex.nonzero(as_tuple=True)                                   # row-major: by tile, then position
        if tile.numel():
            start = torch.cumsum(cnt, 0) - cnt
            rank = torch.arange(tile.numel(), device=dev) - start[tile]
            word = (pos << 8) | hb.reshape(nt, panels * 8192)[tile, pos].long()
            foot[t0 + tile, 1 + rank] = word.to(torch.int32)
    return blocks, foot, table


# -- family layouts ------------------------------------------------------------------------------
def _f64(x):
    import torch

    return torch.as_tensor(np.asarray(x, dtype=np.float64))


def _tc_kernel_only(m) -> None:
    if m.kernel not in ("auto", "tc"):
        raise ValueError(f"kernel={m.kernel!r}: the {m.family} family runs on the bf16 tensor-core kernel only "
                         "(kernel='tc' or 'auto')")


def _check_classes(m, n_classes, most: int, per_chain: int, columns_text: str) -> int:
    """``n_classes`` as an int once it is in ``[2, most]`` and ``per_chain`` kernel columns of it fit K times."""
    if n_classes is None or not 2 <= int(n_classes) <= most:
        raise ValueError(f"the {m.family} family needs n_classes in [2, {most}], got {n_classes}")
    cols = per_chain(int(n_classes))
    if m.n_chains * cols > 16:
        raise ValueError(f"n_chains x {columns_text} must be <= 16 (the tensor-core kernel's columns per launch), got "
                         f"{m.n_chains} x {cols}")
    return int(n_classes)


def _check_integers(m, what: str, valid: str, below) -> None:
    """Every row of non-zero weight holds an integer ``y >= 0`` with ``below(y)`` (``valid`` says so in words)."""
    import torch

    for si, (y, w) in enumerate(zip(m.ys, m.weights)):
        bad = ~((y == torch.floor(y)) & (y >= 0) & below(y))   # NaN fails every comparison
        if w is not None:
            bad &= w != 0   # a masked row may carry anything
        if bool(torch.any(bad)):
            raise ValueError(f"{what} of segment {si} must be integers in {valid} on every row of non-zero weight")


def _check_positive(m, what: str) -> None:
    """Every row of non-zero weight holds a finite y > 0."""
    import torch

    for si, (y, w) in enumerate(zip(m.ys, m.weights)):
        bad = ~(torch.isfinite(y) & (y > 0))   # NaN fails the comparison
        if w is not None:
            bad &= w != 0   # a masked row may carry anything
        if bool(torch.any(bad)):
            raise ValueError(f"{what} of segment {si} must be finite and > 0 on every row of non-zero weight")


def _check_finite(m, what: str) -> None:
    """Every row of non-zero weight holds a finite y."""
    import torch

    for si, (y, w) in enumerate(zip(m.ys, m.weights)):
        bad = ~torch.isfinite(y)
        if w is not None:
            bad &= w != 0   # a masked row may carry anything
        if bool(torch.any(bad)):
            raise ValueError(f"{what} of segment {si} must be finite on every row of non-zero weight")


def _check_unit_interval(m, what: str) -> None:
    """Every row of non-zero weight holds a finite y with 0 < y < 1."""
    import torch

    for si, (y, w) in enumerate(zip(m.ys, m.weights)):
        bad = ~((y > 0) & (y < 1))   # NaN fails the comparisons
        if w is not None:
            bad &= w != 0   # a masked row may carry anything
        if bool(torch.any(bad)):
            raise ValueError(f"{what} of segment {si} must be finite with 0 < y < 1 on every row of non-zero weight")


def _labels(y, w):
    """Integer labels of a chunk; masked rows may carry NaN or out-of-range labels: any valid class will do."""
    import torch

    if w is not None:
        y = torch.where(w != 0, y, torch.zeros_like(y))
    return y.long()


class _Layout:
    """How one family's inputs map to the kernel.  A layout owns the per-chain input shapes, ``columns`` (kernel
    columns per chain) and ``words`` (theta words per column), and converts inputs -> theta words (:meth:`pack`),
    words -> inputs, the kernel's output blocks ``[n_nodes, kernel_chains, 1 + words]`` -> ``[n_nodes, K,
    1 + n_params]`` (:meth:`fold`), and gives the oracle's per-row terms (:meth:`oracle`).  This base is the identity
    layout: one column per chain whose theta row is the chain's inputs flattened in order."""

    columns = 1
    n_classes = 1
    tc_only = True   # no kernel but the bf16 tensor-core one evaluates the family
    offset_columns = slice(None)   # the columns of eta that take the per-row offset (all of them)
    takes_events = False   # the survival families' per-row event indicators
    pairs = False   # two kernel columns per chain (2k, 2k + 1), at most 8 chains, checked for two stages at attach

    def __init__(self, m) -> None:
        self.family, self.K, self.G, self.P = m.family, m.n_chains, m.n_groups, m.n_features
        #: the per-row values the kernel and the oracle read as y (the model's ``ys`` but for the survival families)
        self.kernel_ys = m.ys
        self.shapes = [(self.G,), (self.P,)]
        self.words = self.G + self.P
        self._views = None

    @staticmethod
    def _no_classes(n_classes) -> None:
        if n_classes is not None:
            raise ValueError("n_classes is for family='multinomial' or 'ordinal' only")

    def call_context(self, inputs):
        batched = np.ndim(inputs[1]) == 1 + len(self.shapes[1])
        return (batched, np.shape(inputs[0])) + tuple(np.shape(x) for x in inputs[2:])

    def pack(self, inputs, out: np.ndarray):
        views = self._views
        if views is None or views[0] is not out:
            # float32 windows into the staging buffer, built once per buffer (this runs on every evaluation)
            th = out.view(np.float32).reshape(self.K, -1)
            views = self._views = (out, _split(th, [(n,) for n in (int(np.prod(s)) for s in self.shapes)]))
        xs = [x if type(x) is np.ndarray else np.asarray(x) for x in inputs]
        for view, x in zip(views[1], xs):
            view[...] = x.reshape(view.shape)   # converts to float32 while it copies
        return self.call_context(xs)

    def _theta_rows(self, words: np.ndarray) -> np.ndarray:
        """Words -> ``[K, n_params]``, each chain's inputs flattened in order."""
        return words.view(np.float32).reshape(self.K, -1)

    def inputs_from_words(self, words: np.ndarray):
        th = self._theta_rows(words)
        return [x.copy() for x in _split(th if self.K > 1 else th[0], self.shapes)]

    def fold(self, raw: np.ndarray, ctx) -> np.ndarray:
        return raw

    def _matrices(self, inputs):
        """``(intercepts [G, K], beta [P, K])`` of one call as float64 host tensors."""
        return _f64(inputs[0]).reshape(self.K, self.G).T, _f64(inputs[1]).reshape(self.K, self.P).T

    def oracle(self, inputs, device, dtype):
        """``(intercepts [G, E], beta [P, E], terms)`` of one call, the first two float64 on the host, with E the
        columns of eta; ``terms(y, w, eta)`` gives a chunk's per-row terms ``(ll, dll/deta)`` (dispersion families:
        and ``dll/dlog_dispersion``) as ``[n, K]`` tensors, or ``[n, K, columns]`` where a chain has several kernel
        columns, unweighted."""
        raise NotImplementedError

    def baseline(self, m, inputs) -> np.ndarray:
        """The partial of the collective baseline (:meth:`GlmShards.eager_partial`)."""
        import torch

        return m._partial(inputs, dtype=torch.float32, chunk_rows=1 << 62, bf16_gemms=True)


class _Scalar(_Layout):
    """The logistic, Poisson and Gaussian families and :class:`CustomFamily`: inputs ``(intercept[G], beta[P])``."""

    tc_only = False

    def __init__(self, m, n_classes) -> None:
        self._no_classes(n_classes)
        super().__init__(m)

    def oracle(self, inputs, device, dtype):
        return (*self._matrices(inputs), self._terms)

    def _terms(self, y, w, eta):
        import torch

        yy = y.to(eta.dtype).unsqueeze(1)
        if hasattr(self.family, "code_id"):
            if self.family.torch_fn is None:
                raise ValueError("this CustomFamily has no torch_fn oracle")
            return self.family.torch_fn(yy, eta)
        if self.family == "logistic":
            return yy * eta - torch.nn.functional.softplus(eta), yy - torch.sigmoid(eta)
        if self.family == "poisson":
            mu = torch.exp(eta)
            return yy * eta - mu, yy - mu
        d = yy - eta
        return -0.5 * d * d - _LOG_SQRT_2PI, d

    def baseline(self, m, inputs) -> np.ndarray:
        """Whole segments at once, fp32 elementwise work and fp32 sums."""
        import torch

        ic = torch.as_tensor(np.asarray(inputs[0], dtype=np.float32)).reshape(self.K, -1).to(m.device)
        bt = torch.as_tensor(np.asarray(inputs[1], dtype=np.float32)).reshape(self.K, self.P).to(m.device)
        out = torch.zeros(self.K, 1 + m.n_params, dtype=torch.float64, device=m.device)
        for si, (X, y, g) in enumerate(zip(m.Xs, m.ys, m.groups)):
            eta = (X @ bt.T.to(torch.bfloat16)).float() + ic[:, g]          # [n, K]
            if m.offsets[si] is not None:
                eta = eta + m.offsets[si].unsqueeze(1)
            ll, r = m._weigh(si, 0, X.shape[0], *self._terms(y, None, eta))
            out[:, 0] += ll.sum(0).double()
            out[:, 1 + g] += r.sum(0).double()
            out[:, 1 + self.G :] += (r.T.to(torch.bfloat16) @ X).double()
        return out.reshape(-1).cpu().numpy()


class _Hvp(_Scalar):
    """Hessian-vector products (``GlmShards(..., hvp=True)``): inputs ``(intercept[G], beta[P], v_intercept[G],
    v_beta[P])``; pair k runs as kernel columns 2k, with the theta row ``(intercept, beta)`` and the output block
    ``[LL, d intercept[G], d beta[P]]``, and 2k + 1, with the theta row ``(v_intercept, v_beta)`` and the output block
    ``[0, (H v)_intercept[G], (H v)_beta[P]]``.  Only the parameter columns take the offset."""

    columns = 2
    tc_only = True
    offset_columns = slice(0, None, 2)
    pairs = True

    def __init__(self, m, n_classes) -> None:
        if m.family not in ("logistic", "poisson", "gaussian"):
            raise ValueError(f"hvp=True is for family='logistic', 'poisson' or 'gaussian', not {m.family!r}")
        _tc_kernel_only(m)
        if not 1 <= m.n_chains <= 8:
            raise ValueError(f"hvp=True takes n_chains in [1, 8] (each pair of parameters and direction is two of the "
                             f"tensor-core kernel's 16 columns per launch), got {m.n_chains}")
        super().__init__(m, n_classes)
        self.shapes = self.shapes * 2

    def fold(self, raw: np.ndarray, ctx) -> np.ndarray:
        n = raw.shape[0]
        raw = raw.reshape(n, self.K, 2, 1 + self.words)
        return np.concatenate([raw[:, :, 0], raw[:, :, 1, 1:]], axis=2)

    def oracle(self, inputs, device, dtype):
        import torch

        ic, bt = self._matrices(inputs[:2])
        vic, vbt = self._matrices(inputs[2:])
        pairs = lambda a, b: torch.stack([a, b], dim=2).reshape(a.shape[0], -1)   # column 2k: theta, 2k + 1: v

        def terms(y, w, eta):
            et, u = eta[:, 0::2], eta[:, 1::2]
            ll, r = self._terms(y, w, et)
            if self.family == "logistic":
                h = -torch.sigmoid(et) * torch.sigmoid(-et)
            elif self.family == "poisson":
                h = -torch.exp(et)
            else:
                h = -torch.ones_like(et)
            return torch.stack([ll, torch.zeros_like(ll)], dim=2), torch.stack([r, h * u], dim=2)

        return pairs(ic, vic), pairs(bt, vbt), terms

    baseline = _Layout.baseline


class _Dispersion(_Layout):
    """``gaussian_scale`` and ``negative_binomial``: inputs ``(intercept[G], beta[P], log_dispersion)``, one kernel
    column per chain with the theta row ``[intercept, beta, log_dispersion]`` and the output block ``[LL,
    d intercept[G], d beta[P], d log_dispersion]``."""

    def __init__(self, m, n_classes) -> None:
        self._no_classes(n_classes)
        _tc_kernel_only(m)
        if m.family == "negative_binomial":
            _check_integers(m, "counts", "[0, 2^24]", lambda y: y <= 2.0 ** 24)
        super().__init__(m)
        self.shapes.append(())
        self.words += 1

    def oracle(self, inputs, device, dtype):
        ld = _f64(inputs[2]).reshape(self.K).to(device, dtype)
        fn = _DISPERSION_TERMS[self.family]
        return (*self._matrices(inputs), lambda y, w, eta: fn(y.to(eta.dtype).unsqueeze(1), eta, ld))


class _Survival(_Dispersion):
    """``weibull`` and ``lognormal``: the layout of :class:`_Dispersion` with ``log_dispersion = log sigma``.  The
    event indicator travels in the sign of the kernel's y: ``kernel_ys`` is a float32 copy of the times, negated on
    censored rows (times are > 0, so negation is exact and frees the sign bit); the oracle decodes it the same way."""

    takes_events = True

    def __init__(self, m, n_classes) -> None:
        import torch

        super().__init__(m, n_classes)
        _check_positive(m, "times")
        signed = []
        for si, (t, ev, w) in enumerate(zip(m.ys, m.events, m.weights)):
            if ev is None:
                signed.append(t)
                continue
            keep = torch.ones_like(t, dtype=torch.bool) if w is None else w != 0   # a masked row may carry anything
            if bool(torch.any(keep & ~((ev == 0) | (ev == 1)))):
                raise ValueError(f"events of segment {si} must be 0 or 1 on every row of non-zero weight")
            signed.append(_aligned16(torch.where(ev == 0, -t, t).contiguous()))
        self.kernel_ys = signed


class _Positive(_Dispersion):
    """``gamma`` and ``inverse_gaussian``: the layout of :class:`_Dispersion` with ``log_dispersion`` the log of the
    shape (nu, lambda).  Every row of non-zero weight must hold a finite y > 0."""

    def __init__(self, m, n_classes) -> None:
        super().__init__(m, n_classes)
        _check_positive(m, "responses")


class _Beta(_Dispersion):
    """``beta``: the layout of :class:`_Dispersion` with ``log_dispersion`` the log of the precision phi.  Every row
    of non-zero weight must hold a finite y with 0 < y < 1."""

    def __init__(self, m, n_classes) -> None:
        super().__init__(m, n_classes)
        _check_unit_interval(m, "responses")


class _Softmax(_Layout):
    """``multinomial``: inputs ``(intercept[G, C], beta[P, C])``; chain k runs as kernel columns ``k C + c`` with the
    theta rows ``(intercept[:, c], beta[:, c])``, one ``[LL, gi[G], g[P]]`` block per chain and class."""

    def __init__(self, m, n_classes) -> None:
        _tc_kernel_only(m)
        C = _check_classes(m, n_classes, 16, lambda c: c, "n_classes")
        if any(o is not None for o in m.offsets):
            raise ValueError("offsets are not supported by the multinomial family: an offset common to all classes "
                             "cancels in the softmax")
        _check_integers(m, "labels", f"[0, {C})", lambda y: y < C)
        super().__init__(m)
        self.n_classes = self.columns = C
        self.shapes = [(self.G, C), (self.P, C)]

    def pack(self, inputs, out: np.ndarray):
        K, C, G, P = self.K, self.n_classes, self.G, self.P
        th = out.view(np.float32).reshape(K, C, G + P)
        ic, bt = np.asarray(inputs[0]), np.asarray(inputs[1])
        th[:, :, :G] = ic.reshape(K, G, C).transpose(0, 2, 1)
        th[:, :, G:] = bt.reshape(K, P, C).transpose(0, 2, 1)
        return self.call_context([ic, bt])

    def _theta_rows(self, words: np.ndarray) -> np.ndarray:
        th = words.view(np.float32).reshape(self.K, self.n_classes, self.G + self.P)
        return th.transpose(0, 2, 1).reshape(self.K, -1)

    def fold(self, raw: np.ndarray, ctx) -> np.ndarray:
        n, K, C, G, P = raw.shape[0], self.K, self.n_classes, self.G, self.P
        raw = raw.reshape(n, K, C, 1 + G + P)
        return np.concatenate([raw[..., 0].sum(axis=2)[..., None],
                               raw[..., 1 : 1 + G].transpose(0, 1, 3, 2).reshape(n, K, G * C),
                               raw[..., 1 + G :].transpose(0, 1, 3, 2).reshape(n, K, P * C)], axis=2)

    def oracle(self, inputs, device, dtype):
        import torch

        K, C, G, P = self.K, self.n_classes, self.G, self.P
        icpt = _f64(inputs[0]).reshape(K, G, C).permute(1, 0, 2).reshape(G, K * C)   # column k C + c
        beta = _f64(inputs[1]).reshape(K, P, C).permute(1, 0, 2).reshape(P, K * C)

        def terms(y, w, eta):
            n = eta.shape[0]
            hit = torch.nn.functional.one_hot(_labels(y, w), C).bool().unsqueeze(1)   # [n, 1, C]
            logp = torch.log_softmax(eta.reshape(n, K, C), dim=-1)
            ll = torch.where(hit, logp, torch.zeros_like(logp))
            r = hit.to(eta.dtype) - torch.exp(logp)
            return ll, r

        return icpt, beta, terms


class _Ordinal(_Layout):
    """``ordinal``: inputs ``(intercept[G], beta[P], cutpoints[C - 1])``; chain k runs as kernel columns
    ``k (C - 1) + j`` with the theta rows ``(intercept - c_j, beta)``, one ``[LL_j, gi_j[G], g_j[P]]`` block per chain
    and cutpoint."""

    def __init__(self, m, n_classes) -> None:
        _tc_kernel_only(m)
        C = _check_classes(m, n_classes, 17, lambda c: c - 1, "(n_classes - 1)")
        _check_integers(m, "labels", f"[0, {C})", lambda y: y < C)
        super().__init__(m)
        self.n_classes, self.columns = C, C - 1
        self.shapes.append((C - 1,))

    def _table(self, inputs):
        """``(T, ctx)``: the kernel's intercept table ``T[K, C - 1, G] = float32(intercept[g] - c_j)`` (the difference
        taken in double, rounded once) and the call context ``(batched, intercept shape, cutpoints shape, bad)``, with
        ``bad`` the chains whose table is not strictly decreasing in j for every group."""
        intercept, beta, cutpoints = inputs
        ic = np.asarray(intercept, dtype=np.float64).reshape(self.K, self.G)
        cp = np.asarray(cutpoints, dtype=np.float64).reshape(self.K, self.columns)
        T = (ic[:, None, :] - cp[:, :, None]).astype(np.float32)
        ordered = np.all(T[:, 1:, :] < T[:, :-1, :], axis=(1, 2))   # NaN fails the comparison
        bad = tuple(int(k) for k in np.flatnonzero(~ordered))
        return T, (np.ndim(beta) == 2, np.shape(intercept), np.shape(cutpoints), bad)

    def call_context(self, inputs):
        return self._table(inputs)[1]

    def pack(self, inputs, out: np.ndarray):
        T, ctx = self._table(inputs)
        th = out.view(np.float32).reshape(self.K, self.columns, self.G + self.P)
        th[:, :, : self.G] = T
        th[:, :, self.G :] = np.asarray(inputs[1]).reshape(self.K, 1, self.P)
        return ctx

    def inputs_from_words(self, words: np.ndarray):
        # only the differences travel: intercept[g] = T[0, g], c_j = T[0, 0] - T[j, 0], in double (which packs back
        # to the same words)
        G = self.G
        th = words.view(np.float32).reshape(self.K, self.columns, G + self.P)
        ic = th[:, 0, :G].copy()
        cp = th[:, 0, :1].astype(np.float64) - th[:, :, 0].astype(np.float64)
        bt = th[:, 0, G:].copy()
        if self.K == 1:
            return ic[0], bt[0], cp[0]
        return ic, bt, cp

    def fold(self, raw: np.ndarray, ctx) -> np.ndarray:
        n, K, C1, G = raw.shape[0], self.K, self.columns, self.G
        raw = raw.reshape(n, K, C1, 1 + G + self.P)
        out = np.concatenate([raw[..., 0].sum(axis=2)[..., None], raw[..., 1:].sum(axis=2),
                              -raw[..., 1 : 1 + G].sum(axis=3)], axis=2)
        bad = list(ctx[3])
        out[:, bad, 0] = -np.inf
        out[:, bad, 1:] = 0.0
        return out

    def oracle(self, inputs, device, dtype):
        import torch

        K, C1 = self.K, self.columns
        cp = _f64(inputs[2]).reshape(K, C1).to(device, dtype)
        inf = torch.full((K, 1), float("inf"), dtype=dtype, device=device)
        cpad = torch.cat([-inf, cp, inf], dim=1)                     # [K, C + 1]: c_{-1} = -inf, ..., c_{C-1} = +inf

        def terms(y, w, eta):
            # r_j = dll / dz_j at z_j = eta - c_j, non-zero only for j = y and j = y - 1; each row's ll is credited to
            # j = min(y, C - 2), as the kernel does
            dt = eta.dtype
            lab = _labels(y, w)
            a = cpad[:, lab + 1].T - eta                          # c_y - eta = -z_up
            b = cpad[:, lab].T - eta                              # c_{y-1} - eta = -z_lo
            t = 1.0 / torch.expm1(a - b)                          # 1 / expm1(gap), 0 at the infinite ends
            ll = torch.nn.functional.logsigmoid(a) + torch.nn.functional.logsigmoid(-b) + torch.log(-torch.expm1(b - a))
            r_up = -torch.sigmoid(-a) - t
            r_lo = torch.sigmoid(b) + t
            hot = lambda j: torch.nn.functional.one_hot(j.clamp(0, C1 - 1), C1).to(dt).unsqueeze(1)   # [n, 1, C1]
            up, lo = (lab <= C1 - 1).to(dt), (lab >= 1).to(dt)
            ll = ll.unsqueeze(2) * hot(torch.clamp(lab, max=C1 - 1))
            r = (r_up * up.unsqueeze(1)).unsqueeze(2) * hot(lab) + (r_lo * lo.unsqueeze(1)).unsqueeze(2) * hot(lab - 1)
            return ll, r

        return (*self._matrices(inputs), terms)


class _Pair(_Layout):
    """Two linear predictors per chain over one read of X: inputs ``(intercept[G], beta[P], intercept2[G], beta2[P])``
    and, where ``disp``, a trailing ``log_dispersion``.  Chain k runs as kernel columns 2k, with the theta row
    ``(intercept, beta[, log_dispersion])`` and the output block ``[LL, d intercept[G], d beta[P](, d log_dispersion)]``,
    and 2k + 1, with the theta row ``(intercept2, beta2[, log_dispersion])`` and the output block ``[0, d intercept2[G],
    d beta2[P](, 0)]``.  Only the first predictor takes the offset.  Subclasses give the validation and
    :meth:`_pair_terms`, the oracle's per-row terms."""

    columns = 2
    offset_columns = slice(0, None, 2)
    pairs = True

    def __init__(self, m, n_classes, predictors: str, disp: bool) -> None:
        self._no_classes(n_classes)
        _tc_kernel_only(m)
        if not 1 <= m.n_chains <= 8:
            raise ValueError(f"the {m.family} family takes n_chains in [1, 8] (each chain's {predictors} predictors are "
                             f"two of the tensor-core kernel's 16 columns per launch), got {m.n_chains}")
        super().__init__(m)
        self.disp = disp
        self.shapes = self.shapes * 2 + ([()] if disp else [])
        self.words += int(disp)

    def pack(self, inputs, out: np.ndarray):
        G, P = self.G, self.P
        xs = [np.asarray(x) for x in inputs]
        th = out.view(np.float32).reshape(self.K, 2, self.words)
        th[:, 0, :G] = xs[0].reshape(self.K, G)
        th[:, 0, G : G + P] = xs[1].reshape(self.K, P)
        th[:, 1, :G] = xs[2].reshape(self.K, G)
        th[:, 1, G : G + P] = xs[3].reshape(self.K, P)
        if self.disp:
            th[:, :, G + P] = xs[4].reshape(self.K, 1)   # both rows: every column's table is built from its own row
        return self.call_context(xs)

    def _theta_rows(self, words: np.ndarray) -> np.ndarray:
        th = words.view(np.float32).reshape(self.K, 2, self.words)
        GP = self.G + self.P
        return np.concatenate([th[:, 0, :GP], th[:, 1, :GP], th[:, 0, GP:]], axis=1)

    def fold(self, raw: np.ndarray, ctx) -> np.ndarray:
        n, GP = raw.shape[0], self.G + self.P
        raw = raw.reshape(n, self.K, 2, 1 + self.words)
        return np.concatenate([raw[:, :, 0, : 1 + GP], raw[:, :, 1, 1 : 1 + GP], raw[:, :, 0, 1 + GP :]], axis=2)

    def oracle(self, inputs, device, dtype):
        import torch

        ic, bt = self._matrices(inputs[:2])
        ic2, bt2 = self._matrices(inputs[2:4])
        pairs = lambda a, b: torch.stack([a, b], dim=2).reshape(a.shape[0], -1)   # column 2k: first, 2k + 1: second
        ld = _f64(inputs[4]).reshape(self.K).to(device, dtype) if self.disp else None

        def terms(y, w, eta):
            return self._pair_terms(y.to(eta.dtype).unsqueeze(1), eta[:, 0::2], eta[:, 1::2], ld)

        return pairs(ic, ic2), pairs(bt, bt2), terms

    @staticmethod
    def _pair_terms(y, first, second, a):
        """The per-row terms ``[n, K, 2]`` of :meth:`_Layout.oracle` from both predictors (and log_dispersion)."""
        raise NotImplementedError


class _ZeroInflated(_Pair):
    """``zero_inflated_poisson`` and ``zero_inflated_negative_binomial``: the pair layout with the count predictor
    ``(intercept, beta)``, the zero-inflation logit ``(zi_intercept, zi_beta)`` and, for the negative binomial,
    ``log_dispersion = log alpha``."""

    def __init__(self, m, n_classes) -> None:
        super().__init__(m, n_classes, "count and zero-inflation", m.family == "zero_inflated_negative_binomial")
        _check_integers(m, "counts", "[0, 2^24]", lambda y: y <= 2.0 ** 24)

    @staticmethod
    def _pair_terms(y, eta, zeta, a):
        return _zero_inflated_terms(y, eta, zeta, a)


class _LocationScale(_Pair):
    """``gaussian_location_scale`` and ``student_t``: the pair layout with the mean ``(intercept, beta)``, the log scale
    ``(sigma_intercept, sigma_beta)`` and, for Student-t, ``log_dispersion = log nu``.  Every row of non-zero weight
    must hold a finite y."""

    def __init__(self, m, n_classes) -> None:
        super().__init__(m, n_classes, "mean and log-scale", m.family == "student_t")
        _check_finite(m, "responses")

    @staticmethod
    def _pair_terms(y, mu, s, a):
        return _location_scale_terms(y, mu, s, a)


_LAYOUTS = {"multinomial": _Softmax, "gaussian_scale": _Dispersion, "negative_binomial": _Dispersion,
            "ordinal": _Ordinal, "weibull": _Survival, "lognormal": _Survival,
            "zero_inflated_poisson": _ZeroInflated, "zero_inflated_negative_binomial": _ZeroInflated,
            "gamma": _Positive, "inverse_gaussian": _Positive, "gaussian_location_scale": _LocationScale,
            "student_t": _LocationScale, "beta": _Beta}


_LOG_SQRT_2PI = 0.918938533204672742
#: flag bit on the family code of a Hessian-vector-product launch (csrc/models.h: kGlmHvp)
HVP_FLAG = 16


def _gaussian_scale_terms(y, eta, s):
    """``(ll, dll/deta, dll/ds)`` of the Gaussian with ``sigma = exp(s)`` (``s`` per chain, broadcast over rows)."""
    import torch

    dn = (y - eta) * torch.exp(-s)
    return -0.5 * dn * dn - s - _LOG_SQRT_2PI, dn * torch.exp(-s), dn * dn - 1.0


def _negative_binomial_terms(y, eta, a):
    """``(ll, dll/deta, dll/da)`` of the NB2 negative binomial with ``alpha = exp(a)``, ``mu = exp(eta)``, without
    ``-lgamma(y + 1)``.  ``lgamma(y + alpha) - lgamma(alpha) - y a`` and ``psi(y + alpha) - psi(alpha)`` are taken
    from their Stirling-series differences (written with ``log1p(y / alpha)``) where alpha is large, so that the
    y log alpha terms and the lgamma values of size alpha log alpha cancel analytically, not in floating point."""
    import torch

    alpha = torch.exp(a)
    x = eta - a
    sp = torch.nn.functional.softplus(x)
    big = alpha >= (8.0 if eta.dtype == torch.float32 else 1e3)   # the series' error: < 1e-9 (fp32), < 1e-25 (fp64)
    yb = torch.where(torch.isfinite(y) & (y >= 0), y, torch.zeros_like(y))   # masked rows: keep every branch finite
    ab = torch.where(big, alpha, torch.full_like(alpha, 1e3))
    z = yb + ab
    l1 = torch.log1p(yb / ab)

    def stirling(v):   # lgamma(v) - ((v - 1/2) log v - v + log(2 pi) / 2)
        return (1.0 / 12 - (1.0 / 360 - 1.0 / (1260 * v * v)) / (v * v)) / v

    def psi_tail(v):   # psi(v) - log v
        i2 = 1.0 / (v * v)
        return -0.5 / v - i2 * (1.0 / 12 - i2 * (1.0 / 120 - i2 / 252))

    d_big = (z - 0.5) * l1 - yb + stirling(z) - stirling(ab)
    dpsi_big = l1 + psi_tail(z) - psi_tail(ab)
    d_small = torch.lgamma(y + alpha) - torch.lgamma(alpha) - y * a
    dpsi_small = torch.digamma(y + alpha) - torch.digamma(alpha)
    D = torch.where(big, d_big, d_small)
    dpsi = torch.where(big, dpsi_big, dpsi_small)
    ll = D + y * eta - (alpha + y) * sp
    r = y - (alpha + y) * torch.sigmoid(x)
    return ll, r, alpha * (dpsi - sp) - r


def _survival_split(y, eta, s):
    """``(delta, log t, z, 1 / sigma)`` of rows whose times carry the event in their sign (+t event, -t censored)."""
    import torch

    event = ~torch.signbit(y)
    lt = torch.log(y.abs())
    sinv = torch.exp(-s)
    return event, lt, (lt - eta) * sinv, sinv


def _weibull_terms(y, eta, s):
    """``(ll, dll/deta, dll/ds)`` of the right-censored Weibull AFT model, ``sigma = exp(s)``: shape ``1 / sigma``,
    scale ``exp(eta)``; ``y`` = +t for an event, -t for a censored row."""
    import torch

    event, lt, z, sinv = _survival_split(y, eta, s)
    ez = torch.exp(z)
    d = event.to(eta.dtype)
    ll = torch.where(event, z - ez - s - lt, -ez)
    return ll, (ez - d) * sinv, z * (ez - d) - d


def _lognormal_terms(y, eta, s):
    """``(ll, dll/deta, dll/ds)`` of the right-censored log-normal AFT model, ``sigma = exp(s)``; ``y`` as in
    :func:`_weibull_terms`.  Censored rows use ``log_ndtr``, relatively accurate far into the upper tail, and the
    inverse Mills ratio ``phi(z) / Phi(-z)`` as the exponential of a difference of logs."""
    import torch

    event, lt, z, sinv = _survival_split(y, eta, s)
    log_sf = torch.special.log_ndtr(-z)
    lam = torch.exp(-0.5 * z * z - _LOG_SQRT_2PI - log_sf)
    ll = torch.where(event, -0.5 * z * z - s - _LOG_SQRT_2PI - lt, log_sf)
    r = torch.where(event, z, lam) * sinv
    q = torch.where(event, z * z - 1.0, z * lam)
    return ll, r, q


#: 1 / k! for k = 2 .. 16: the series of -g(z) / z^2, g(z) = 1 + z - e^z, to a truncation error below 1e-17 of g at
#: |z| < 1/2
_G_SERIES = [1.0 / float(np.prod(np.arange(1, k + 1))) for k in range(2, 17)]


def _gamma_g(z):
    """``g(z) = 1 + z - e^z``, relatively accurate near z = 0 (where ``z - expm1(z)`` loses ``2 eps / |z|``): a power
    series below |z| = 1/2, ``z - expm1(z)`` above."""
    import torch

    small = z.abs() < 0.5
    zs = torch.where(small, z, torch.zeros_like(z))
    acc = torch.full_like(z, _G_SERIES[-1])
    for c in reversed(_G_SERIES[:-1]):
        acc = acc * zs + c
    return torch.where(small, -(zs * zs) * acc, z - torch.expm1(z))


def _gamma_shape_terms(a):
    """``(nu, C(nu), Q(nu))`` per chain in float64: ``C = nu log nu - nu - lgamma(nu)`` and ``Q = nu (log nu -
    psi(nu))``, from their Stirling series at nu >= 1e3 (truncation error < 1e-24), where the direct forms would
    subtract values of size nu log nu.  Both stay O(1): ``C -> (a - log 2 pi) / 2``, ``Q -> 1/2``."""
    import torch

    a = a.double()
    nu = torch.exp(a)
    big = nu >= 1e3
    nb = torch.where(big, nu, torch.full_like(nu, 1e3))
    ns = torch.where(big, torch.ones_like(nu), nu)
    i2 = 1.0 / (nb * nb)
    S = (1.0 / 12 - i2 * (1.0 / 360 - i2 / 1260)) / nb
    T = -0.5 / nb - i2 * (1.0 / 12 - i2 * (1.0 / 120 - i2 / 252))
    C = torch.where(big, 0.5 * a - _LOG_SQRT_2PI - S, ns * torch.log(ns) - ns - torch.lgamma(ns))
    Q = torch.where(big, -nb * T, ns * (torch.log(ns) - torch.digamma(ns)))
    return nu, C, Q


def _gamma_terms(y, eta, a):
    """``(ll, dll/deta, dll/da)`` of the gamma family with mean ``mu = exp(eta)`` and shape ``nu = exp(a)``:
    ``ll = nu g(z) + C(nu) - log y``, ``dll/deta = nu expm1(z)``, ``dll/da = nu g(z) + Q(nu)`` with ``z = log y -
    eta`` (:func:`_gamma_g`, :func:`_gamma_shape_terms`; the shape's terms in float64 whatever the dtype)."""
    import torch

    nu, C, Q = (v.to(eta.dtype) for v in _gamma_shape_terms(a))
    lt = torch.log(y)
    z = lt - eta
    ng = nu * _gamma_g(z)
    return ng + C - lt, nu * torch.expm1(z), ng + Q


def _inverse_gaussian_terms(y, eta, a):
    """``(ll, dll/deta, dll/da)`` of the inverse Gaussian family with mean ``mu = exp(eta)`` and shape ``lambda =
    exp(a)``: with ``h = lambda expm1(z)^2 / (2 y)`` (= lambda (y - mu)^2 / (2 mu^2 y)), ``ll = a / 2 - log(2 pi) / 2 -
    (3/2) log y - h``, ``dll/deta = lambda e^-eta expm1(z)``, ``dll/da = 1/2 - h``."""
    import torch

    lam = torch.exp(a)
    lt = torch.log(y)
    em = torch.expm1(lt - eta)
    h = 0.5 * lam * em * (em / y)
    return 0.5 * a - _LOG_SQRT_2PI - 1.5 * lt - h, lam * torch.exp(-eta) * em, 0.5 - h


def _zero_inflated_terms(y, eta, zeta, a=None):
    """The per-row terms of a zero-inflated count model, ``[n, K, 2]`` (column 0: eta, 1: zeta): ``ll`` (in column 0,
    0 in column 1), ``(dll/deta, dll/dzeta)`` and, with ``a = log alpha`` (negative binomial; ``None``: Poisson),
    ``dll/da`` (in column 0).  ``(l, r, q)`` are the plain family's terms, ``l = log f(y)`` without
    ``-lgamma(y + 1)``:

        y > 0:  ll = l - softplus(zeta),       dll/deta = r,       dll/dzeta = -sigmoid(zeta)
        y = 0:  ll = logaddexp(zeta, l) - softplus(zeta),  dll/deta = w0 r,  w0 = sigmoid(l - zeta),
                dll/dzeta = -sigmoid(zeta - l) sigmoid(-zeta) expm1(l)

    and ``dll/da = q`` (y > 0) or ``w0 q`` (y = 0)."""
    import torch

    if a is None:
        mu = torch.exp(eta)
        l, r, q = y * eta - mu, y - mu, None
    else:
        l, r, q = _negative_binomial_terms(y, eta, a)
    zero = y == 0
    sp = torch.logaddexp(zeta, torch.zeros_like(zeta))
    w0 = torch.where(zero, torch.sigmoid(l - zeta), torch.ones_like(l))
    ll = torch.where(zero, torch.logaddexp(zeta, l), l) - sp
    rz = torch.where(zero, -torch.sigmoid(zeta - l) * torch.sigmoid(-zeta) * torch.expm1(l), -torch.sigmoid(zeta))
    pair = lambda u, v: torch.stack([u, v], dim=2)
    out = [pair(ll, torch.zeros_like(ll)), pair(w0 * r, rz)]
    if q is not None:
        out.append(pair(w0 * q, torch.zeros_like(q)))
    return out


_LOG_PI = 1.1447298858494002


def _student_t_constants(a):
    """``(nu, C(nu), Q(nu))`` per chain in float64 for ``nu = exp(a)``: ``C = lgamma((nu + 1) / 2) - lgamma(nu / 2) -
    log(nu pi) / 2`` and ``Q = (nu / 2) [psi((nu + 1) / 2) - psi(nu / 2)] - 1/2``, from their asymptotic series at
    nu >= 1e3 (truncation error < 1e-20), where the direct forms subtract values of size nu log nu: ``C = -log(2 pi) / 2
    - 1 / (4 nu) + 1 / (24 nu^3) - 1 / (20 nu^5)``, ``Q = 1 / (4 nu) - 1 / (8 nu^3) + 1 / (4 nu^5)``."""
    import torch

    a = a.double()
    nu = torch.exp(a)
    big = nu >= 1e3
    ns = torch.where(big, torch.ones_like(nu), nu)
    x = 1.0 / torch.where(big, nu, torch.full_like(nu, 1e3))
    x2 = x * x
    c_small = torch.lgamma(0.5 * (ns + 1)) - torch.lgamma(0.5 * ns) - 0.5 * (torch.log(ns) + _LOG_PI)
    q_small = 0.5 * ns * (torch.digamma(0.5 * (ns + 1)) - torch.digamma(0.5 * ns)) - 0.5
    C = torch.where(big, -_LOG_SQRT_2PI - x * (0.25 - x2 * (1.0 / 24 - x2 / 20)), c_small)
    Q = torch.where(big, x * (0.25 - x2 * (0.125 - x2 * 0.25)), q_small)
    return nu, C, Q


#: 1 / k for k = 2 .. 30: the series h = sum_k p^k / k of h(q) = log1p(q) - q / (1 + q) in p = q / (1 + q), to a
#: truncation error below 1e-19 of h at q < 1/4
_H_SERIES = [1.0 / k for k in range(2, 31)]


def _location_scale_terms(y, mu, s, a=None):
    """The per-row terms of a location-scale model, ``[n, K, 2]`` (column 0: the mean mu, 1: s = log sigma), with ``z =
    (y - mu) e^-s``: ``ll`` (in column 0, 0 in column 1), ``(dll/dmu, dll/ds)`` and, with ``a = log nu`` (Student-t;
    ``None``: Gaussian), ``dll/da`` (in column 0).  Gaussian: ``ll = -z^2 / 2 - s - log(2 pi) / 2``, ``dll/dmu = z
    e^-s``, ``dll/ds = z^2 - 1``.  Student-t, with ``q = z^2 / nu``, ``p = q / (1 + q)`` and :func:`_student_t_constants`:

        ll = C - s - (nu + 1) / 2 log1p(q),   dll/dmu = (nu + 1) z e^-s / (nu + z^2),   dll/ds = (nu + 1) p - 1,
        dll/da = Q + p / 2 - (nu / 2) h(q),   h(q) = log1p(q) - p.

    From ``u = |z| nu^-1/2 = 2^12`` up, where z^2 may overflow float32, ``log1p(q) = 2 log u + log1p(1 / q)`` and
    ``z / (nu + z^2) = p / z`` with ``1 / q = (nu / z) / z``; below q = 1/4, h is its series in p (``h = p^2 / 2 + p^3 /
    3 + ...``), since the difference loses about ``2 eps / q``.  Valid in float64 and float32."""
    import torch

    sinv = torch.exp(-s)
    z = (y - mu) * sinv
    pair = lambda u, v: torch.stack([u, v], dim=2)
    if a is None:
        ll = -0.5 * z * z - s - _LOG_SQRT_2PI
        return [pair(ll, torch.zeros_like(ll)), pair(z * sinv, z * z - 1.0)]
    nu, C, Q = (v.to(z.dtype) for v in _student_t_constants(a))
    u = z.abs() / torch.sqrt(nu)
    big = u >= 4096.0
    zb = torch.where(big, z, torch.ones_like(z))          # every branch finite where it is not taken
    q = torch.where(big, torch.zeros_like(u), u * u)
    iq = torch.where(big, (nu / zb) / zb, torch.ones_like(z))
    p = torch.where(big, 1.0 / (1.0 + iq), q / (1.0 + q))
    L = torch.where(big, 2.0 * torch.log(torch.where(big, u, torch.ones_like(u))) + torch.log1p(iq), torch.log1p(q))
    zr = torch.where(big, p / zb, z / (nu * (1.0 + q)))   # z / (nu + z^2)
    ps = torch.where(q < 0.25, p, torch.zeros_like(p))
    acc = torch.full_like(ps, _H_SERIES[-1])
    for c in reversed(_H_SERIES[:-1]):
        acc = acc * ps + c
    h = torch.where(big | (q >= 0.25), L - p, ps * ps * acc)
    ll = C - s - 0.5 * (nu + 1.0) * L
    qa = Q + 0.5 * p - 0.5 * nu * h
    return [pair(ll, torch.zeros_like(ll)), pair((nu + 1.0) * zr * sinv, (nu + 1.0) * p - 1.0), pair(qa, torch.zeros_like(qa))]


#: the Stirling tail S(z) = lgamma(z) - [(z - 1/2) log z - z + log(2 pi) / 2] = sum_k c_k z^(1 - 2k) and z (psi(z) -
#: log z) = -1/2 + sum_k d_k z^(1 - 2k): truncation errors below 1e-15 from z = 8 up
_S_SERIES = [1.0 / 12, -1.0 / 360, 1.0 / 1260, -1.0 / 1680, 1.0 / 1188, -691.0 / 360360, 1.0 / 156]
_T_SERIES = [-1.0 / 12, 1.0 / 120, -1.0 / 252, 1.0 / 240, -1.0 / 132, 691.0 / 32760, -1.0 / 12]
#: 1 / (2 j + 3), j = 0 .. 17: the series of k(x) = x - log1p(x) in s = x / (2 + x) (see :func:`_kl_series`), to a
#: truncation error below 1e-17 of k at |x| < 1/2
_K_SERIES = [1.0 / (2 * j + 3) for j in range(18)]


def _poly(x, coeffs):
    """``sum_k coeffs[k] x^k`` by Horner's rule."""
    import torch

    acc = torch.full_like(x, coeffs[-1])
    for c in reversed(coeffs[:-1]):
        acc = acc * x + c
    return acc


def _beta_tails(z, lz):
    """``(S(z), z tau(z))`` with ``S`` the Stirling tail of lgamma and ``tau(z) = psi(z) - log z``, ``lz = log z``
    given: their asymptotic series from z = 8 up, ``lgamma`` and ``digamma`` below (where neither is large)."""
    import torch

    big = z >= 8.0
    zb = torch.where(big, z, torch.full_like(z, 8.0))
    zs = torch.where(big, torch.ones_like(z), z)
    ls = torch.where(big, torch.zeros_like(z), lz)
    i1 = 1.0 / zb
    i2 = i1 * i1
    S = torch.where(big, i1 * _poly(i2, _S_SERIES), torch.lgamma(zs) - (zs - 0.5) * ls + zs - _LOG_SQRT_2PI)
    zt = torch.where(big, -0.5 + i1 * _poly(i2, _T_SERIES), zs * (torch.digamma(zs) - ls))
    return S, zt


def _beta_constants(a):
    """``(phi, C(phi), Q(phi))`` per chain in float64 for ``phi = exp(a)``: ``C = (a - log 2 pi) / 2 + S(phi)`` and
    ``Q = phi tau(phi)`` (:func:`_beta_tails`), both O(1) however large phi is: ``Q -> -1/2``."""
    import torch

    a = a.double()
    phi = torch.exp(a)
    S, Q = _beta_tails(phi, a)
    return phi, 0.5 * a - _LOG_SQRT_2PI + S, Q


def _kl_series(x):
    """``k(x) = x - log1p(x)`` for |x| < 1/2, relatively accurate near 0 (where the difference loses ``2 eps / |x|``):
    with ``s = x / (2 + x)``, ``log1p(x) = 2 atanh(s)`` and ``k = x s - 2 s^3 (1/3 + s^2 / 5 + s^4 / 7 + ...)``."""
    s = x / (2.0 + x)
    s2 = s * s
    return x * s - 2.0 * s * s2 * _poly(s2, _K_SERIES)


def _beta_terms(y, eta, a):
    """``(ll, dll/deta, dll/da)`` of beta regression, ``mu = sigmoid(eta)``, precision ``phi = exp(a)``, ``A = mu
    phi``, ``B = (1 - mu) phi``, in the grouped form that has no large cancellation (valid in float64 and float32):

        ll = C(phi) + (log mu + log(1 - mu)) / 2 - log y - log(1 - y) - phi KL - S(A) - S(B),
        dll/deta = phi mu (1 - mu) (logit y - logit mu) - (1 - mu) A tau(A) + mu B tau(B),
        dll/da = Q(phi) - phi KL - A tau(A) - B tau(B),

    with ``KL = mu log(mu / y) + (1 - mu) log((1 - mu) / (1 - y))`` (:func:`_beta_constants`, :func:`_beta_tails`).
    ``logit y - logit mu = log1p(u) - log1p(v)`` and ``phi KL = A k(u) + B k(v)`` come from the relative differences
    ``u = (y - mu) / mu`` and ``v = (mu - y) / (1 - mu)``: below |x| = 1/2 from :func:`_kl_series`, above from the logs
    (``log1p(u) = log y - log mu``).  ``log mu = -softplus(-eta)``, ``1 - mu = sigmoid(-eta)``.  In float32 (the
    collective backend) ``A`` and ``B`` underflow once ``|eta| + |a|`` nears 87; every test of that path stays inside."""
    import torch

    phi, C, Q = (v.to(eta.dtype) for v in _beta_constants(a))
    a = a.to(eta.dtype)
    ly, l1y = torch.log(y), torch.log1p(-y)
    lmu, l1mu = -torch.nn.functional.softplus(-eta), -torch.nn.functional.softplus(eta)
    mu, nmu = torch.sigmoid(eta), torch.sigmoid(-eta)
    d = torch.where(eta >= 0, nmu - (1.0 - y), y - mu)   # y - mu, exact where y ~ mu
    u, v = d / mu, -d / nmu
    su, sv = u.abs() < 0.5, v.abs() < 0.5
    ku = _kl_series(torch.where(su, u, torch.zeros_like(u)))
    kv = _kl_series(torch.where(sv, v, torch.zeros_like(v)))
    lu = torch.where(su, u - ku, ly - lmu)
    lv = torch.where(sv, v - kv, l1y - l1mu)
    lA, lB = lmu + a, l1mu + a
    A, B = torch.exp(lA), torch.exp(lB)
    kl = torch.where(su, A * ku, phi * d - A * lu) + torch.where(sv, B * kv, -phi * d - B * lv)
    SA, tA = _beta_tails(A, lA)
    SB, tB = _beta_tails(B, lB)
    ll = C + 0.5 * (lmu + l1mu) - ly - l1y - kl - SA - SB
    r = A * nmu * (lu - lv) - nmu * tA + mu * tB
    return ll, r, Q - kl - tA - tB


_DISPERSION_TERMS = {"gaussian_scale": _gaussian_scale_terms, "negative_binomial": _negative_binomial_terms,
                     "weibull": _weibull_terms, "lognormal": _lognormal_terms, "gamma": _gamma_terms,
                     "inverse_gaussian": _inverse_gaussian_terms, "beta": _beta_terms}


def quantize_block_fp8(X, block: int = 32):
    """Block-scaled FP8 quantisation of a design matrix (MX-style, 32 x 32 blocks).

    Returns ``(Xq, scales)``: ``Xq`` e4m3 bytes ``[n, P]`` (``torch.float8_e4m3fn``) and UE8M0 scale
    bytes ``[4 * ceil(n / 128), P / 32]`` (rows padded to whole 128-row tiles with 2^0), with
    ``X[r, f] ~= float(Xq[r, f]) * 2 ** (scales[r // 32, f // 32] - 127)``.
    """
    import torch

    n, P = X.shape
    if P % block:
        raise ValueError("P must be a multiple of 32")
    n_rb = (n + block - 1) // block
    n_rb_pad = ((n + 127) // 128) * 4
    Xf = X.float()
    pad = n_rb * block - n
    if pad:
        Xf = torch.cat([Xf, torch.zeros(pad, P, device=X.device)], 0)
    blocks = Xf.view(n_rb, block, P // block, block)
    amax = blocks.abs().amax(dim=(1, 3))                                  # [n_rb, P/32]
    # power-of-two scale such that amax / scale <= 448 (e4m3 max)
    exp = torch.ceil(torch.log2(torch.clamp(amax, min=2.0**-100) / 448.0)).clamp(-127, 127)
    exp = torch.where(amax > 0, exp, torch.zeros_like(exp))
    scale = torch.exp2(exp)
    q = (blocks / scale[:, None, :, None]).reshape(n_rb * block, P)[:n].to(torch.float8_e4m3fn)
    scales = torch.full((n_rb_pad, P // block), 127, dtype=torch.uint8, device=X.device)
    scales[:n_rb] = (exp + 127).to(torch.uint8)
    return q.contiguous(), scales.contiguous()


def dequantize_block_fp8(Xq, scales, block: int = 32):
    """Inverse of :func:`quantize_block_fp8` (fp32 result); the oracle of the fp8 kernel tests."""
    import torch

    n, P = Xq.shape
    s = torch.exp2(scales.float() - 127.0)                                 # [n_rb_pad, P/32]
    s_full = s.repeat_interleave(block, 0)[:n].repeat_interleave(block, 1)
    return Xq.float() * s_full


def pack_tile_scales(scales, n_features: int):
    """Re-orders the UE8M0 block scales ``[4 * tiles, P / 32]`` into 16 words per 128-row tile: words 0-7
    feature-block-major per row group (word ``4g + q`` = row group ``q``, feature blocks ``4g..4g+3``),
    words 8-15 row-group-major per feature block (word ``4h + qq`` = row groups 0..3 of feature block
    ``4h + qq``).  ``csrc/glm_fp8.cu`` reads words 8-15: byte ``32 + 4 fb + q`` is the scale of (row group
    ``q``, feature block ``fb``) of the tile, one 32-byte line per tile.  Returns ``uint8 [tiles, 64]``."""
    import torch

    nfb = n_features // 32
    if nfb not in (4, 8) or scales.shape[0] % 4 or scales.shape[1] != nfb:
        raise ValueError("the fp8 kernel takes P in {128, 256} and scales padded to whole 128-row tiles")
    tiles, g2 = scales.shape[0] // 4, nfb // 4
    s4 = scales.contiguous().view(tiles, 4, g2, 4)                       # [tile, q, g, j]
    packed = torch.full((tiles, 2, 2, 4, 4), 127, dtype=torch.uint8, device=scales.device)
    packed[:, 0, :g2] = s4.permute(0, 2, 1, 3)                           # [tile, g, q, byte j]
    packed[:, 1, :g2] = s4.permute(0, 2, 3, 1)                           # [tile, h, qq, byte q]
    return packed.reshape(tiles, 64).contiguous()


class Fp8GlmShards(GlmShards):
    """GLM shards whose design matrices are block-scaled FP8 (``quantize_block_fp8``).

    The hierarchical-GLM configuration of BASELINE.json: one partial-pooling group (intercept) per
    shard/GPU, e4m3 design matrix with 32 x 32 UE8M0 block scales, evaluated by ``csrc/glm_fp8.cu``
    (e4m3 wgmma, block scales applied in fp32 registers per 32-deep K step).  Up to 3 chains per launch.
    The residuals of the Poisson and Gaussian families are unbounded, so the kernel scales them too (one
    power of two per 32-row group and chain); so are weighted residuals, of any family.  ``offsets`` and
    ``weights`` are those of :class:`GlmShards`.
    """

    def __init__(self, Xqs, scales, ys, *, groups=None, n_groups: int = 1, n_chains: int = 1,
                 family: str = "logistic", node_ids=None, n_nodes=None, offsets=None, weights=None,
                 hvp: bool = False) -> None:
        if hvp:
            raise ValueError("hvp=True runs on the bf16 tensor-core kernel only, not on the block-scaled fp8 kernel")
        if not 1 <= n_chains <= 3:
            raise ValueError("the fp8 kernel batches at most 3 chains per launch")
        super().__init__(Xqs, ys, groups=groups, n_groups=n_groups, family=family, n_chains=n_chains, kernel="fp8",
                         scales=scales, node_ids=node_ids, n_nodes=n_nodes, offsets=offsets, weights=weights)
        self._kernel_scales = [pack_tile_scales(s, self.n_features) for s in self.scales]

    @classmethod
    def from_dense(cls, Xs, ys, **kw):
        pairs = [quantize_block_fp8(X) for X in Xs]
        return cls([p[0] for p in pairs], [p[1] for p in pairs], ys, **kw)

    def _dequant(self, X):
        idx = next(i for i, Xi in enumerate(self.Xs) if Xi is X)
        return dequantize_block_fp8(X, self.scales[idx])

    def _dequant_rows(self, seg: int, r0: int, r1: int):
        if r0 % 32:
            raise ValueError("row chunks of block-scaled matrices start on a 32-row boundary")
        return dequantize_block_fp8(self.Xs[seg][r0:r1], self.scales[seg][r0 // 32 : (r1 + 31) // 32])

    def bytes_per_eval(self) -> int:
        return int(sum(X.shape[0] * (self.n_features + 4) + s.numel() for X, s in zip(self.Xs, self._kernel_scales))) + \
            self._row_data_bytes()


def synth_logistic_shard(n_rows: int, n_features: int, *, seed: int, device, chunk_rows: int = 1 << 20,
                         beta_scale: float = 0.05):
    """Synthetic logistic-regression shard generated on the device in chunks
    (bf16 ``X ~ N(0,1)``, ``y ~ Bernoulli(sigmoid(X beta* + 0.3))``)."""
    import torch

    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    beta_true = (torch.randn(n_features, generator=gen, device=device) * beta_scale).float()
    X = torch.empty(n_rows, n_features, dtype=torch.bfloat16, device=device)
    y = torch.empty(n_rows, dtype=torch.float32, device=device)
    for r0 in range(0, n_rows, chunk_rows):
        r1 = min(n_rows, r0 + chunk_rows)
        xb = torch.randn(r1 - r0, n_features, generator=gen, device=device, dtype=torch.float32).to(torch.bfloat16)
        X[r0:r1] = xb
        p = torch.sigmoid(xb.float() @ beta_true + 0.3)
        y[r0:r1] = (torch.rand(r1 - r0, generator=gen, device=device) < p).float()
    return X, y, beta_true


def synth_multinomial_shard(n_rows: int, n_features: int, n_classes: int, *, seed: int, device,
                            chunk_rows: int = 1 << 20, beta_scale: float = 0.05):
    """Synthetic softmax-regression shard generated on the device in chunks (bf16 ``X ~ N(0,1)``,
    ``y ~ Categorical(softmax(X beta* + b*))`` as float32 labels ``0 .. C-1``).  Returns ``(X, y, beta* [P, C])``."""
    import torch

    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    beta_true = (torch.randn(n_features, n_classes, generator=gen, device=device) * beta_scale).float()
    b_true = (torch.randn(n_classes, generator=gen, device=device) * 0.3).float()
    X = torch.empty(n_rows, n_features, dtype=torch.bfloat16, device=device)
    y = torch.empty(n_rows, dtype=torch.float32, device=device)
    for r0 in range(0, n_rows, chunk_rows):
        r1 = min(n_rows, r0 + chunk_rows)
        xb = torch.randn(r1 - r0, n_features, generator=gen, device=device, dtype=torch.float32).to(torch.bfloat16)
        X[r0:r1] = xb
        p = torch.softmax(xb.float() @ beta_true + b_true, dim=1)
        y[r0:r1] = torch.multinomial(p, 1, generator=gen).squeeze(1).float()
    return X, y, beta_true


def synth_negative_binomial_shard(n_rows: int, n_features: int, *, alpha: float, seed: int, device,
                                  chunk_rows: int = 1 << 20, beta_scale: float = 0.05, intercept: float = 0.5):
    """Synthetic over-dispersed count shard generated on the device in chunks: bf16 ``X ~ N(0,1)``,
    ``y ~ NegativeBinomial(mean mu = exp(X beta* + intercept), variance mu + mu^2 / alpha)`` drawn as a gamma-Poisson
    mixture (``lambda ~ Gamma(alpha, scale mu / alpha)``, ``y ~ Poisson(lambda)``), stored as float32.
    Returns ``(X, y, beta*)``."""
    import torch

    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    beta_true = (torch.randn(n_features, generator=gen, device=device) * beta_scale).float()
    X = torch.empty(n_rows, n_features, dtype=torch.bfloat16, device=device)
    y = torch.empty(n_rows, dtype=torch.float32, device=device)
    for r0 in range(0, n_rows, chunk_rows):
        r1 = min(n_rows, r0 + chunk_rows)
        xb = torch.randn(r1 - r0, n_features, generator=gen, device=device, dtype=torch.float32).to(torch.bfloat16)
        X[r0:r1] = xb
        mu = torch.exp(xb.float() @ beta_true + intercept).double()
        lam = torch._standard_gamma(torch.full_like(mu, float(alpha)), generator=gen) * (mu / alpha)
        y[r0:r1] = torch.poisson(lam, generator=gen).float()
    return X, y, beta_true


def synth_zero_inflated_shard(n_rows: int, n_features: int, *, seed: int, device, alpha: Optional[float] = None,
                              chunk_rows: int = 1 << 20, beta_scale: float = 0.05, intercept: float = 0.5,
                              zi_intercept: float = -1.0, zi_beta_scale: float = 0.05):
    """Synthetic zero-inflated count shard generated on the device in chunks: bf16 ``X ~ N(0,1)``, a structural zero
    with probability ``pi = sigmoid(X zi_beta* + zi_intercept)``, else a count from ``Poisson(mu)`` (``alpha`` None)
    or ``NegativeBinomial(mean mu, variance mu + mu^2 / alpha)`` (a gamma-Poisson mixture), ``mu = exp(X beta* +
    intercept)``, stored as float32.  Returns ``(X, y, beta*, zi_beta*)``."""
    import torch

    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    beta_true = (torch.randn(n_features, generator=gen, device=device) * beta_scale).float()
    zi_true = (torch.randn(n_features, generator=gen, device=device) * zi_beta_scale).float()
    X = torch.empty(n_rows, n_features, dtype=torch.bfloat16, device=device)
    y = torch.empty(n_rows, dtype=torch.float32, device=device)
    for r0 in range(0, n_rows, chunk_rows):
        r1 = min(n_rows, r0 + chunk_rows)
        xb = torch.randn(r1 - r0, n_features, generator=gen, device=device, dtype=torch.float32).to(torch.bfloat16)
        X[r0:r1] = xb
        xf = xb.float()
        lam = torch.exp(xf @ beta_true + intercept).double()
        if alpha is not None:
            lam = torch._standard_gamma(torch.full_like(lam, float(alpha)), generator=gen) * (lam / alpha)
        counts = torch.poisson(lam, generator=gen)
        zero = torch.rand(r1 - r0, generator=gen, device=device) < torch.sigmoid(xf @ zi_true + zi_intercept)
        y[r0:r1] = torch.where(zero, torch.zeros_like(counts), counts).float()
    return X, y, beta_true, zi_true


def synth_ordinal_shard(n_rows: int, n_features: int, n_classes: int, *, seed: int, device, chunk_rows: int = 1 << 20,
                        beta_scale: float = 0.05, cutpoints=None):
    """Synthetic ordinal (cumulative-logit) shard generated on the device in chunks: bf16 ``X ~ N(0,1)`` and labels
    ``y = #{j : U > sigmoid(c_j - X beta*)}`` with ``U ~ Uniform(0, 1)``, so ``P(y <= j) = sigmoid(c_j - X beta*)``,
    stored as float32 ``0 .. C-1``.  ``cutpoints`` (increasing, ``C - 1`` of them) default to evenly spaced values
    in [-1.5, 1.5].  Returns ``(X, y, beta*, cutpoints)``."""
    import torch

    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    beta_true = (torch.randn(n_features, generator=gen, device=device) * beta_scale).float()
    cuts = np.linspace(-1.5, 1.5, n_classes - 1) if cutpoints is None else np.asarray(cutpoints, dtype=np.float64)
    if cuts.shape != (n_classes - 1,) or not np.all(np.diff(cuts) > 0):
        raise ValueError(f"cutpoints must be {n_classes - 1} strictly increasing values")
    c = torch.as_tensor(cuts, dtype=torch.float32, device=device)
    X = torch.empty(n_rows, n_features, dtype=torch.bfloat16, device=device)
    y = torch.empty(n_rows, dtype=torch.float32, device=device)
    for r0 in range(0, n_rows, chunk_rows):
        r1 = min(n_rows, r0 + chunk_rows)
        xb = torch.randn(r1 - r0, n_features, generator=gen, device=device, dtype=torch.float32).to(torch.bfloat16)
        X[r0:r1] = xb
        cdf = torch.sigmoid(c[None, :] - (xb.float() @ beta_true)[:, None])   # [n, C - 1], P(y <= j)
        u = torch.rand(r1 - r0, 1, generator=gen, device=device)
        y[r0:r1] = (u > cdf).sum(1).float()
    return X, y, beta_true, cuts.astype(np.float32)


def synth_survival_shard(n_rows: int, n_features: int, *, family: str, sigma: float, censor_fraction: float, seed: int,
                         device, chunk_rows: int = 1 << 20, beta_scale: float = 0.05, intercept: float = 0.5):
    """Synthetic right-censored survival shard generated on the device in chunks: bf16 ``X ~ N(0,1)``, event times
    ``log T = X beta* + intercept + sigma eps`` with ``eps`` standard minimum-Gumbel (``family="weibull"``) or
    N(0, 1) (``"lognormal"``), and censoring times ``C`` drawn independently of T from the same family with the
    location shifted by one constant, chosen (for the marginal of ``X beta*``) so that about ``censor_fraction`` of
    the rows are censored.  The observed time is ``min(T, C)`` and the event ``T <= C``.  ``censor_fraction`` = 0
    gives no censoring.  Returns ``(X, time, event, beta*)``, time and event float32."""
    import torch

    if family not in ("weibull", "lognormal"):
        raise ValueError(f"family must be 'weibull' or 'lognormal', got {family!r}")
    if not 0.0 <= censor_fraction < 1.0:
        raise ValueError(f"censor_fraction must be in [0, 1), got {censor_fraction}")
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    beta_true = (torch.randn(n_features, generator=gen, device=device) * beta_scale).float()

    def eps(n):
        u = torch.rand(n, generator=gen, device=device, dtype=torch.float64).clamp(1e-300, 1.0)
        return torch.log(-torch.log(u)) if family == "weibull" else torch.randn(n, generator=gen, device=device,
                                                                                 dtype=torch.float64)

    shift = float("inf")
    if censor_fraction > 0:
        # log C - log T = shift + sigma (eps_c - eps_t), with x' beta* cancelled: P(C < T) is censor_fraction when
        # -shift is that quantile of sigma (eps_c - eps_t), estimated from 2^20 pairs
        diff = sigma * (eps(1 << 20) - eps(1 << 20))
        shift = -float(torch.quantile(diff.cpu().float(), censor_fraction))
    X = torch.empty(n_rows, n_features, dtype=torch.bfloat16, device=device)
    time = torch.empty(n_rows, dtype=torch.float32, device=device)
    event = torch.empty(n_rows, dtype=torch.float32, device=device)
    for r0 in range(0, n_rows, chunk_rows):
        r1 = min(n_rows, r0 + chunk_rows)
        xb = torch.randn(r1 - r0, n_features, generator=gen, device=device, dtype=torch.float32).to(torch.bfloat16)
        X[r0:r1] = xb
        loc = (xb.float() @ beta_true + intercept).double()
        log_t = loc + sigma * eps(r1 - r0)
        log_c = loc + shift + sigma * eps(r1 - r0)
        ev = log_t <= log_c
        time[r0:r1] = torch.exp(torch.where(ev, log_t, log_c)).float()
        event[r0:r1] = ev.float()
    return X, time, event, beta_true


def _check_positive_args(family: str, shape: float) -> None:
    if family not in ("gamma", "inverse_gaussian"):
        raise ValueError(f"family must be 'gamma' or 'inverse_gaussian', got {family!r}")
    if not shape > 0:
        raise ValueError(f"shape must be > 0, got {shape}")


def draw_positive(mu, *, family: str, shape: float, generator):
    """float32 draws with mean ``mu`` (a float64 tensor) and shape ``shape``: ``Gamma(shape, scale mu / shape)``
    (``family="gamma"``) or inverse Gaussian ``IG(mu, lambda = shape)`` (``"inverse_gaussian"``, Michael-Schucany-Haas:
    with ``n ~ N(0, 1)`` and ``c = mu n^2 / (2 lambda)``, the smaller root ``x = mu / (1 + c + sqrt(c (2 + c)))``, free
    of cancellation, taken with probability ``mu / (mu + x)``, else ``mu^2 / x``), drawn in float64 and clamped into
    the positive finite float32 range."""
    import torch

    _check_positive_args(family, shape)
    if family == "gamma":
        v = torch._standard_gamma(torch.full_like(mu, float(shape)), generator=generator) * (mu / shape)
    else:
        n = torch.randn(mu.shape, generator=generator, device=mu.device, dtype=torch.float64)
        c = mu * n * n / (2.0 * shape)
        x = mu / (1.0 + c + torch.sqrt(c * (2.0 + c)))
        u = torch.rand(mu.shape, generator=generator, device=mu.device, dtype=torch.float64)
        v = torch.where(u * (mu + x) <= mu, x, mu * mu / x)
    fi = torch.finfo(torch.float32)
    return v.clamp(fi.tiny, fi.max).float()


def synth_positive_shard(n_rows: int, n_features: int, *, family: str, shape: float, seed: int, device,
                         chunk_rows: int = 1 << 20, beta_scale: float = 0.05, intercept: float = 0.5):
    """Synthetic positive-response shard generated on the device in chunks: bf16 ``X ~ N(0,1)`` and y with mean
    ``mu = exp(X beta* + intercept)`` and shape ``shape``: ``Gamma(shape, scale mu / shape)`` (``family="gamma"``) or
    inverse Gaussian ``IG(mu, lambda = shape)`` (``"inverse_gaussian"``, Michael-Schucany-Haas in a cancellation-free
    form), drawn in float64 by :func:`draw_positive` and stored as float32 > 0.  Returns ``(X, y, beta*)``."""
    import torch

    _check_positive_args(family, shape)
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    beta_true = (torch.randn(n_features, generator=gen, device=device) * beta_scale).float()
    X = torch.empty(n_rows, n_features, dtype=torch.bfloat16, device=device)
    y = torch.empty(n_rows, dtype=torch.float32, device=device)
    for r0 in range(0, n_rows, chunk_rows):
        r1 = min(n_rows, r0 + chunk_rows)
        xb = torch.randn(r1 - r0, n_features, generator=gen, device=device, dtype=torch.float32).to(torch.bfloat16)
        X[r0:r1] = xb
        mu = torch.exp(xb.float() @ beta_true + intercept).double()
        y[r0:r1] = draw_positive(mu, family=family, shape=shape, generator=gen)
    return X, y, beta_true


def synth_beta_shard(n_rows: int, n_features: int, *, phi: float, seed: int, device, chunk_rows: int = 1 << 20,
                     beta_scale: float = 0.05, intercept: float = 0.5):
    """Synthetic proportion shard generated on the device in chunks: bf16 ``X ~ N(0,1)`` and ``y ~ Beta(mu phi, (1 -
    mu) phi)`` with ``mu = sigmoid(X beta* + intercept)``, drawn in float64 as ``sigmoid(log G_A - log G_B)`` from two
    standard gamma draws taken in log space (``log G(c) = log G(c + 1) + log(U) / c``, which does not underflow at a
    tiny shape c), and clamped into the open interval ``(0, 1)`` of float32 (``[2^-126, 1 - 2^-24]``).  Returns
    ``(X, y, beta*)``."""
    import torch

    if not phi > 0:
        raise ValueError(f"phi must be > 0, got {phi}")
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    beta_true = (torch.randn(n_features, generator=gen, device=device) * beta_scale).float()
    X = torch.empty(n_rows, n_features, dtype=torch.bfloat16, device=device)
    y = torch.empty(n_rows, dtype=torch.float32, device=device)
    lo, hi = torch.finfo(torch.float32).tiny, 1.0 - 2.0 ** -24
    for r0 in range(0, n_rows, chunk_rows):
        r1 = min(n_rows, r0 + chunk_rows)
        xb = torch.randn(r1 - r0, n_features, generator=gen, device=device, dtype=torch.float32).to(torch.bfloat16)
        X[r0:r1] = xb
        mu = torch.sigmoid(xb.float() @ beta_true + intercept).double()

        def log_gamma_draw(c):
            u = torch.rand(c.shape, generator=gen, device=device, dtype=torch.float64).clamp(min=1e-300)
            return torch.log(torch._standard_gamma(c + 1.0, generator=gen)) + torch.log(u) / c

        d = log_gamma_draw(mu * phi) - log_gamma_draw((1.0 - mu) * phi)
        y[r0:r1] = torch.sigmoid(d).clamp(lo, hi).float()
    return X, y, beta_true


def synth_location_scale_shard(n_rows: int, n_features: int, *, family: str, seed: int, device, nu: Optional[float] = None,
                               chunk_rows: int = 1 << 20, beta_scale: float = 0.05, intercept: float = 0.5,
                               sigma_intercept: float = 0.0, sigma_beta_scale: float = 0.05):
    """Synthetic location-scale shard generated on the device in chunks: bf16 ``X ~ N(0,1)`` and ``y = mu + sigma
    eps`` with ``mu = X beta* + intercept`` and ``log sigma = X sigma_beta* + sigma_intercept``, ``eps ~ N(0, 1)``
    (``family="gaussian_location_scale"``) or Student-t with ``nu`` degrees of freedom (``"student_t"``, drawn as
    ``N(0, 1) / sqrt(chi2_nu / nu)`` with the chi-square a ``Gamma(nu / 2, scale 2)`` draw), in float64 and stored as
    float32 (clamped into its finite range).  Returns ``(X, y, beta*, sigma_beta*)``."""
    import torch

    if family not in ("gaussian_location_scale", "student_t"):
        raise ValueError(f"family must be 'gaussian_location_scale' or 'student_t', got {family!r}")
    if (family == "student_t") != (nu is not None) or (nu is not None and not nu > 0):
        raise ValueError(f"nu > 0 is for family='student_t' only, got nu={nu} for {family!r}")
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    beta_true = (torch.randn(n_features, generator=gen, device=device) * beta_scale).float()
    sigma_true = (torch.randn(n_features, generator=gen, device=device) * sigma_beta_scale).float()
    fmax = torch.finfo(torch.float32).max
    X = torch.empty(n_rows, n_features, dtype=torch.bfloat16, device=device)
    y = torch.empty(n_rows, dtype=torch.float32, device=device)
    for r0 in range(0, n_rows, chunk_rows):
        r1 = min(n_rows, r0 + chunk_rows)
        xb = torch.randn(r1 - r0, n_features, generator=gen, device=device, dtype=torch.float32).to(torch.bfloat16)
        X[r0:r1] = xb
        xd = xb.double()
        mu = xd @ beta_true.double() + intercept
        sigma = torch.exp(xd @ sigma_true.double() + sigma_intercept)
        eps = torch.randn(r1 - r0, generator=gen, device=device, dtype=torch.float64)
        if nu is not None:
            chi2 = 2.0 * torch._standard_gamma(torch.full_like(eps, 0.5 * nu), generator=gen)
            eps = eps / torch.sqrt(chi2 / nu)
        y[r0:r1] = (mu + sigma * eps).clamp(-fmax, fmax).float()   # a heavy tail at a small nu stays finite
    return X, y, beta_true, sigma_true


def synth_logistic_shard_fp8(n_rows: int, n_features: int, *, seed: int, device, chunk_rows: int = 1 << 20):
    """Like :func:`synth_logistic_shard` but quantised chunk-wise to block-scaled FP8 (never holds
    the fp32 matrix): returns ``(Xq e4m3 [n, P], scales uint8 [4*ceil(n/128), P/32], y)``."""
    import torch

    assert chunk_rows % 128 == 0
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    beta_true = (torch.randn(n_features, generator=gen, device=device) * 0.05).float()
    col_scale = torch.exp(torch.randn(n_features, generator=gen, device=device) * 0.5)  # heterogeneous feature scales
    Xq = torch.empty(n_rows, n_features, dtype=torch.float8_e4m3fn, device=device)
    scales = torch.full((((n_rows + 127) // 128) * 4, n_features // 32), 127, dtype=torch.uint8, device=device)
    y = torch.empty(n_rows, dtype=torch.float32, device=device)
    for r0 in range(0, n_rows, chunk_rows):
        r1 = min(n_rows, r0 + chunk_rows)
        xb = torch.randn(r1 - r0, n_features, generator=gen, device=device) * col_scale
        q, s = quantize_block_fp8(xb)
        Xq[r0:r1] = q
        scales[r0 // 32 : r0 // 32 + s.shape[0]] = s
        xd = dequantize_block_fp8(q, s)
        p = torch.sigmoid(xd @ (beta_true / col_scale) + 0.3)
        y[r0:r1] = (torch.rand(r1 - r0, generator=gen, device=device) < p).float()
    return Xq, scales, y
