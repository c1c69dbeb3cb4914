"""The linear-regression kernel (csrc/linreg.cu) against an exact oracle, and the federation's transport modes.

Exact cases hold integer x (|x| <= 2^6), intercepts and slopes on a 2^-4 grid, y such that every residual
r = y - (a + b x) is a multiple of 2^-4 with |r| <= 2^6, and power-of-two sigmas.  :func:`budget` proves that every
partial sum the kernel forms is then exact in fp64, in any order and with or without FMA contraction, so dLL/da and
dLL/db must equal the integer oracle bit for bit on every grid and in every transport mode.  LL adds the constant
``n_here * (-log sigma - log sqrt(2 pi))`` once per CTA and is held to a bound that a count off by one row breaks.

Inexact cases (normal data, large offsets that cancel) are held to a first-order error bound against exact rational
arithmetic on the stored values.  A NumPy emulation of the kernel shows that each of a list of plausible kernel bugs
would break one of these checks.

The GPU cases run the kernel at the shapes where its indexing changes (warp per shard, CTA-stride boundaries, the
automatic grid thresholds, several reduction groups) and run every case through each transport mode of the runtime:
tagged-word ("LL") or fence-and-flag theta, tagged-word or flag results, the single-CTA latency path, speculative
launches and device-resident theta.  The other kernels run through the same modes and must keep their bits.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from fractions import Fraction
from typing import List, Optional, Tuple

import numpy as np
import pytest

LOG_SQRT_2PI = 0.91893853320467274178   # log(sqrt(2 pi)) as the kernel spells it
U = 2.0 ** -53
BLOCK = 256                              # threads per CTA of the linreg kernel
GROUP = 16                               # CTAs per level-1 reduction group (fed_comm.cuh: kReduceGroup)
LL_VARS = ("B200FED_NO_LL", "B200FED_LL_MAX_VALS", "B200FED_LL_MAX_THETA")


# ---------------------------------------------------------------------------------------------------------------------
# cases


@dataclass
class Case:
    name: str
    xs: List[np.ndarray]              # stored values as float64 (float32 storage: already rounded)
    ys: List[np.ndarray]
    sigmas: List[float]
    local_ids: List[int]
    n_total: int
    thetas: List[Tuple[np.ndarray, np.ndarray]]   # two (a[n_total], b[n_total])
    exact: bool
    grid: Optional[int] = None        # explicit engine grid, or None for the automatic one
    want_grid: Optional[int] = None   # grid the engine must run (-1 = one CTA, one warp per shard)
    dtype: str = "f64"                # storage type of x and y

    def as_f32(self) -> "Case":
        f = lambda v: v.astype(np.float32).astype(np.float64)   # noqa: E731
        return Case(self.name + "-f32", [f(x) for x in self.xs], [f(y) for y in self.ys], self.sigmas, self.local_ids,
                    self.n_total, self.thetas, self.exact, self.grid, self.want_grid, "f32")


def exact_case(name, sizes, *, seed, n_total=None, local_ids=None, grid=None, want_grid=None) -> Case:
    rng = np.random.default_rng(seed)
    n_total = len(sizes) if n_total is None else n_total
    local_ids = list(range(len(sizes))) if local_ids is None else list(local_ids)
    a1 = rng.integers(-64, 65, n_total) / 16.0          # |a| <= 4
    b1 = rng.integers(-32, 33, n_total) / 16.0          # |b| <= 2
    a2 = a1 + rng.integers(-32, 33, n_total) / 16.0
    b2 = b1 + rng.integers(-8, 9, n_total) / 16.0
    xs, ys = [], []
    for s, n in zip(local_ids, sizes):
        x = rng.integers(-64, 65, n).astype(np.float64)
        ys.append(a1[s] + b1[s] * x + rng.integers(-128, 129, n) / 16.0)   # |r| <= 8 at theta 1, <= 42 at theta 2
        xs.append(x)
    sigmas = [2.0 ** int(k) for k in rng.integers(-2, 3, len(sizes))]
    return Case(name, xs, ys, sigmas, local_ids, n_total, [(a1, b1), (a2, b2)], True, grid, want_grid)


def inexact_case(name, sizes, *, seed, offset, grid=None, want_grid=None) -> Case:
    """Normal data; with ``offset`` x sits around 1e4 and y around 1e6, so that a + b x and y cancel."""
    rng = np.random.default_rng(seed)
    n_total = len(sizes)
    x0, b0 = (1e4, 100.0) if offset else (0.0, 0.5)
    a1 = rng.normal(size=n_total) + 1.0
    b1 = b0 + 0.01 * rng.normal(size=n_total)
    a2, b2 = a1 + 0.3 * rng.normal(size=n_total), b1 * (1 + 1e-6 * rng.normal(size=n_total))
    sigmas = list(0.3 + rng.random(n_total))
    xs = [x0 + rng.normal(size=n) * (50.0 if offset else 1.0) for n in sizes]
    ys = [a1[s] + b1[s] * x + sigmas[s] * rng.normal(size=x.size) for s, x in enumerate(xs)]
    return Case(name, xs, ys, sigmas, list(range(n_total)), n_total, [(a1, b1), (a2, b2)], False, grid, want_grid)


def budget(case: Case, limit: int = 2 ** 53) -> None:
    """Raises ValueError unless every operation of the kernel is exact on ``case`` at both of its thetas: every
    value sits on its grid, and the sums of |r^2|, |r| and |r x| in grid units stay below ``limit`` (2^53), so that
    every partial sum is an integer number of grid units that fp64 holds exactly."""
    if not case.exact:
        raise ValueError(f"{case.name} is not an exact case")
    for a, b in case.thetas:
        for name, v in (("a", a), ("b", b)):
            if not (np.all(v * 16 == np.round(v * 16)) and np.all(np.abs(v) <= 64)):
                raise ValueError(f"{case.name}: {name} must be multiples of 2^-4 with |{name}| <= 2^6")
        for x, y, sigma, s in zip(case.xs, case.ys, case.sigmas, case.local_ids):
            if not (np.all(x == np.round(x)) and np.all(np.abs(x) <= 64)):
                raise ValueError(f"{case.name}: x must be integers with |x| <= 2^6")
            if not np.all(y * 16 == np.round(y * 16)):
                raise ValueError(f"{case.name}: y must be multiples of 2^-4")
            m, e = math.frexp(sigma)
            if m != 0.5:
                raise ValueError(f"{case.name}: sigma {sigma} is not a power of two")
            R = residual_units(x, y, a[s], b[s])
            if R.size and np.abs(R).max() > 64 * 16:
                raise ValueError(f"{case.name}: |r| exceeds 2^6")
            X = x.astype(np.int64)
            # in grid units (r^2: 2^-8; r and r x: 2^-4) every partial sum is an integer below 2^53
            for what, total in (("r^2", int((R * R).sum())), ("|r|", int(np.abs(R).sum())),
                                ("|r x|", int(np.abs(R * X).sum()))):
                if total >= limit:
                    raise ValueError(f"{case.name}: sum of {what} leaves the exact range")


def residual_units(x, y, a, b) -> np.ndarray:
    """16 r as int64 (exact cases)."""
    return np.round(y * 16).astype(np.int64) - int(round(a * 16)) - int(round(b * 16)) * x.astype(np.int64)


def log_norm(sigma: float) -> float:
    return -math.log(sigma) - LOG_SQRT_2PI


# ---------------------------------------------------------------------------------------------------------------------
# oracles and tolerances


@dataclass
class Expected:
    vals: np.ndarray                  # [n_total, 3] rounded to fp64
    ll: List[Optional[Fraction]]      # exact LL per shard (local shards)
    tol: np.ndarray                   # [n_total, 3] absolute tolerance (exact cases: LL only)


def chain_length(n: int, grid: int) -> int:
    """Longest chain of additions that forms one output: rows per thread, 5 shuffle levels, then the block, the
    reduction group and the node."""
    if grid < 0:
        return -(-n // 32) + 5
    return -(-n // (grid * BLOCK)) + 5 + 5 + min(GROUP, grid) + -(-grid // GROUP)


def _dyadic(v) -> Tuple[List[int], int]:
    """Integers N and an exponent k with v == N / 2^k exactly."""
    fr = [float(t).as_integer_ratio() for t in v]
    k = max([d.bit_length() - 1 for _, d in fr] + [0])
    return [n << (k - d.bit_length() + 1) for n, d in fr], k


def expected(case: Case, theta, grid: int) -> Expected:
    """Exact results: integer arithmetic for exact cases, exact rational arithmetic on the stored values otherwise.
    Independent of models/linreg.py."""
    a, b = theta
    vals = np.zeros((case.n_total, 3))
    tol = np.zeros((case.n_total, 3))
    ll: List[Optional[Fraction]] = [None] * case.n_total
    for x, y, sigma, s in zip(case.xs, case.ys, case.sigmas, case.local_ids):
        n = x.size
        inv_var = 1 / Fraction(sigma) ** 2
        L = log_norm(sigma)
        if case.exact:
            R = residual_units(x, y, a[s], b[s])
            srr, sr, srx = Fraction(int((R * R).sum()), 256), Fraction(int(R.sum()), 16), Fraction(int((R * x.astype(np.int64)).sum()), 16)
        else:
            X, kx = _dyadic(x)
            Y, ky = _dyadic(y)
            (A,), ka = _dyadic([a[s]])
            (B,), kb = _dyadic([b[s]])
            K = max(ky, ka, kb + kx)
            R = [(Yi << (K - ky)) - (A << (K - ka)) - ((B * Xi) << (K - kb - kx)) for Xi, Yi in zip(X, Y)]
            srr = Fraction(sum(r * r for r in R), 1 << (2 * K))
            sr = Fraction(sum(R), 1 << K)
            srx = Fraction(sum(r * xi for r, xi in zip(R, X)), 1 << (K + kx))
        q = -srr / 2 * inv_var
        ll[s] = q + n * Fraction(L)
        vals[s] = [float(ll[s]), float(sr * inv_var), float(srx * inv_var)]
        m = chain_length(n, grid)
        g = 1 if grid < 0 else grid
        if case.exact:
            tol[s, 0] = (g + 70) * 2.0 ** -52 * (abs(float(q)) + n * abs(L))
        else:
            r = y - (a[s] + b[s] * x)
            T = np.abs(r) + np.abs(y) + abs(a[s]) + np.abs(b[s] * x)
            iv = float(inv_var)
            tol[s] = (m + 8) * U * np.array([(2 * np.abs(r) * T).sum() * iv + n * abs(L), T.sum() * iv,
                                             (np.abs(x) * T).sum() * iv])
    return Expected(vals, ll, tol)


def deviation(case: Case, exp: Expected, got: np.ndarray) -> float:
    """Largest error of one evaluation's ``[n_total, 3]`` results in tolerances; inf where an exact bit is wrong."""
    got = np.asarray(got, dtype=np.float64).reshape(case.n_total, 3)
    others = np.setdiff1d(np.arange(case.n_total), case.local_ids)
    if np.any(got[others] != 0.0) or np.any(np.signbit(got[others])):
        return math.inf
    loc = np.asarray(case.local_ids, dtype=np.int64)
    if case.exact:
        if not np.array_equal(got[loc, 1:], exp.vals[loc, 1:]):
            return math.inf
        worst = 0.0
        for s in case.local_ids:
            if not np.isfinite(got[s, 0]):
                return math.inf
            err = abs(Fraction(float(got[s, 0])) - exp.ll[s])
            if err:
                worst = max(worst, float(err) / exp.tol[s, 0] if exp.tol[s, 0] else math.inf)
        return worst
    if not np.all(np.isfinite(got[loc])):
        return math.inf
    err = np.abs(got[loc] - exp.vals[loc])
    with np.errstate(divide="ignore"):
        return float(np.max(np.where(err == 0, 0.0, err / exp.tol[loc]), initial=0.0))


# ---------------------------------------------------------------------------------------------------------------------
# NumPy emulation of the kernel (self-tests of the checks above)

BUGS = ["r_fp32", "drop_last_row", "n_here_off_by_one", "sigma_for_var", "log_var_in_constant", "slot_shift",
        "swap_ab", "x_fp32", "stale_cta_partial", "group_counted_twice"]


def _butterfly(v: np.ndarray) -> np.ndarray:
    """xor-shuffle sum over the last axis (32 lanes); every lane ends with the total."""
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., idx ^ o]
    return v


def _cta_rows(case: Case, theta, grid: int, bug: Optional[str]) -> np.ndarray:
    a, b = theta
    g = 1 if grid < 0 else grid
    rows = np.zeros((g, case.n_total * 3))
    for x, y, sigma, s in zip(case.xs, case.ys, case.sigmas, case.local_ids):
        slot = (s + 1) % case.n_total if bug == "slot_shift" else s
        aa, bb = (b[s], a[s]) if bug == "swap_ab" else (a[s], b[s])
        xx = x.astype(np.float32).astype(np.float64) if bug == "x_fp32" else x
        if bug == "r_fp32":
            f = np.float32
            r = (y.astype(f) - (f(aa) + f(bb) * xx.astype(f))).astype(np.float64)
        else:
            r = y - (aa + bb * xx)
        n = x.size
        if bug == "drop_last_row" and n:
            r, xx = r[:-1], xx[:-1]
        terms = np.stack([r * r, r, r * xx])                       # [3, rows]
        inv_var = 1.0 / sigma if bug == "sigma_for_var" else 1.0 / (sigma * sigma)
        L = -math.log(sigma * sigma if bug == "log_var_in_constant" else sigma) - LOG_SQRT_2PI
        n_count = n + 1 if bug == "n_here_off_by_one" else n
        if grid < 0:
            per = -(-terms.shape[1] // 32) * 32
            lanes = np.pad(terms, ((0, 0), (0, per - terms.shape[1]))).reshape(3, -1, 32).sum(axis=1)
            sums = _butterfly(lanes)[:, :1]                          # [3, 1]
            n_here = np.array([n_count])
        else:
            stride = g * BLOCK
            per = max(1, -(-terms.shape[1] // stride)) * stride
            th = np.pad(terms, ((0, 0), (0, per - terms.shape[1]))).reshape(3, -1, g, BLOCK).sum(axis=1)
            warps = _butterfly(th.reshape(3, g, BLOCK // 32, 32))[..., 0]                       # [3, g, 8]
            sums = _butterfly(np.pad(warps, ((0, 0), (0, 0), (0, 32 - BLOCK // 32))))[..., 0]   # [3, g]
            first = np.arange(g) * BLOCK
            left = np.maximum(n_count - first, 0)
            n_here = np.where(left > 0, left // stride * BLOCK + np.minimum(left % stride, BLOCK), 0)
        rows[:, slot * 3 + 0] = -0.5 * sums[0] * inv_var + n_here * L
        rows[:, slot * 3 + 1] = sums[1] * inv_var
        rows[:, slot * 3 + 2] = sums[2] * inv_var
    return rows


def emulate(case: Case, theta, grid: int, bug: Optional[str] = None, previous=None) -> np.ndarray:
    """The kernel's per-CTA partials and its fixed-order two-level reduction, in fp64."""
    rows = _cta_rows(case, theta, grid, bug)
    if bug == "stale_cta_partial" and previous is not None:
        rows[-1] = _cta_rows(case, previous, grid, None)[-1]
    if rows.shape[0] == 1:
        return rows[0].reshape(-1, 3)
    groups = []
    for first in range(0, rows.shape[0], GROUP):
        acc = np.zeros(rows.shape[1])
        for row in rows[first:first + GROUP]:
            acc = acc + row
        groups.append(acc)
    if bug == "group_counted_twice":
        groups.append(groups[0])
    node = np.zeros(rows.shape[1])
    for grp in groups:
        node = node + grp
    return node.reshape(-1, 3)


def _self_cases() -> List[Tuple[Case, int]]:
    small = [0, 1, 31, 32, 33, 4096, 7, 100, 2]
    return [
        (exact_case("exact-small9", small, seed=1), -1),
        (exact_case("exact-grid2", [2 * BLOCK - 1, 2 * BLOCK + 1, 5], seed=2), 2),
        (exact_case("exact-grid17", [17 * BLOCK * 2 + 1, 17 * BLOCK - 1, 40], seed=3), 17),
        (exact_case("exact-ids-3-7", [300, 2000], seed=4, n_total=10, local_ids=[3, 7]), 2),
        (inexact_case("inexact-offset-grid33", [30_001, 3], seed=5, offset=True), 33),
        (inexact_case("inexact-offset-small", [4000, 33], seed=6, offset=True), -1),
        (inexact_case("inexact-plain-grid3", [5000], seed=7, offset=False), 3),
    ]


SELF_CASES = _self_cases()


# ---------------------------------------------------------------------------------------------------------------------
# CPU tests


@pytest.mark.parametrize("i", range(sum(c.exact for c, _ in SELF_CASES)))
def test_exact_case_is_inside_its_budget(i):
    budget([c for c, _ in SELF_CASES if c.exact][i])


def test_budget_rejects_cases_outside_it():
    base = exact_case("base", [50, 60], seed=11)
    budget(base)
    bad_x = exact_case("x65", [50, 60], seed=11)
    bad_x.xs[0] = bad_x.xs[0].copy()
    bad_x.xs[0][3] = 65.0
    bad_sigma = exact_case("sigma3", [50, 60], seed=11)
    bad_sigma.sigmas[1] = 3.0
    bad_y = exact_case("yfine", [50, 60], seed=11)
    bad_y.ys[0] = bad_y.ys[0] + 2.0 ** -6
    bad_r = exact_case("rbig", [50, 60], seed=11)
    bad_r.ys[1] = bad_r.ys[1] + 100.0
    for case in (bad_x, bad_sigma, bad_y, bad_r):
        with pytest.raises(ValueError):
            budget(case)
    with pytest.raises(ValueError):
        budget(inexact_case("normal", [10], seed=1, offset=False))
    # the sum bound: 2^53 grid units would take some 2^33 rows, so it is shown at a smaller limit
    with pytest.raises(ValueError, match="exact range"):
        budget(exact_case("long", [5000], seed=12), limit=2 ** 20)


@pytest.mark.parametrize("case,grid", SELF_CASES, ids=[c.name for c, _ in SELF_CASES])
def test_oracle_agrees_with_the_model_reference(case, grid):
    """``LinregShards.reference_partial`` (torch, fp64): dLL/da and dLL/db bit for bit on exact cases; otherwise
    every output within 1e-14 of its error scale."""
    from pytensor_federated_b200.models import LinregShards

    model = LinregShards(case.xs, case.ys, case.sigmas, local_ids=case.local_ids, n_shards_total=case.n_total)
    for theta in case.thetas:
        exp = expected(case, theta, grid)
        ref = model.reference_partial(list(theta)).reshape(-1, 3)
        loc = case.local_ids
        if case.exact:
            assert np.array_equal(ref[loc, 1:], exp.vals[loc, 1:])
            assert deviation(case, exp, ref) <= 1.0
        else:
            m = np.array([chain_length(x.size, grid) + 8 for x in case.xs])[:, None]
            scale = exp.tol[loc] / (m * U)
            assert np.all(np.abs(ref[loc] - exp.vals[loc]) <= 1e-14 * scale)


@pytest.mark.parametrize("case,grid", SELF_CASES, ids=[c.name for c, _ in SELF_CASES])
def test_emulated_kernel_passes_the_checks(case, grid):
    if case.exact:
        budget(case)
    prev = case.thetas[1]
    for theta in case.thetas:
        got = emulate(case, theta, grid, previous=prev)
        assert deviation(case, expected(case, theta, grid), got) <= 1.0
        prev = theta


@pytest.mark.parametrize("bug", BUGS)
def test_each_injected_kernel_bug_is_detected(bug):
    """Every bug changes an exact bit or moves some output by more than 4 tolerances."""
    worst = 0.0
    for case, grid in SELF_CASES:
        prev = case.thetas[1]
        for theta in case.thetas:
            got = emulate(case, theta, grid, bug=bug, previous=prev)
            worst = max(worst, deviation(case, expected(case, theta, grid), got))
            prev = theta
    assert worst > 4.0, f"{bug} stays within {worst:.3g} tolerances"


def test_linreg_shards_validate_their_data():
    from pytensor_federated_b200.models import LinregShards

    x = np.arange(10.0)
    with pytest.raises(ValueError, match="same length"):
        LinregShards([x], [x[:9]], [1.0])
    with pytest.raises(ValueError, match="1-D"):
        LinregShards([x.reshape(2, 5)], [x.reshape(2, 5)], [1.0])
    for sigma in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="sigma"):
            LinregShards([x], [x], [sigma])
    with pytest.raises(ValueError, match="local_ids"):
        LinregShards([x, x], [x, x], [1.0, 1.0], local_ids=[2, 2], n_shards_total=4)
    with pytest.raises(ValueError, match="local_ids"):
        LinregShards([x], [x], [1.0], local_ids=[4], n_shards_total=4)
    top = LinregShards.MAX_SHARDS_TOTAL
    assert 16 * top + 256 <= 227 * 1024 - 256 < 16 * (top + 1) + 256
    LinregShards([x], [x], [1.0], local_ids=[top - 1], n_shards_total=top)
    with pytest.raises(ValueError, match="shared memory"):
        LinregShards([x], [x], [1.0], local_ids=[0], n_shards_total=top + 1)


@pytest.mark.parametrize("kernel,P,dtype", [("simt", 256, "bf16"), ("simt", 512, "bf16"), ("generic", 100, "f32"),
                                            ("generic", 1000, "bf16")])
def test_cuda_core_glm_refuses_more_groups_than_shared_memory_holds(kernel, P, dtype):
    import torch

    from pytensor_federated_b200.models import GlmShards
    from pytensor_federated_b200.models.glm import CTA_SMEM_LIMIT

    X = torch.zeros(16, P, dtype=torch.bfloat16 if dtype == "bf16" else torch.float32)

    def model(G):
        return GlmShards([X], [torch.zeros(16)], groups=[0], n_groups=G, kernel=kernel)

    code = model(1).use_tensor_cores()
    assert code == (0 if kernel == "simt" else 3 if dtype == "bf16" else 4)
    # the largest group count that fits runs; one more is refused with that count in the message
    fits = max(G for G in range(1, 60_000) if model(1).cuda_core_smem_bytes(code, G) <= CTA_SMEM_LIMIT)
    assert model(fits).use_tensor_cores() == code
    with pytest.raises(ValueError, match=f"at most {fits} groups fit"):
        model(fits + 1).use_tensor_cores()
    if kernel == "simt" and P == 256:
        assert 18_000 < fits < 19_000   # about 12 bytes per group next to 9.5 KB of fixed cost


def test_raise_maps_every_native_code(monkeypatch):
    """Status bits of the completion flag, the host-side timeout and a failed launch each get their own error."""
    from pytensor_federated_b200.ops import native
    from pytensor_federated_b200.parallel import engine as engine_mod
    from pytensor_federated_b200.parallel.engine import FederatedEngine, FederationError, FederationTimeout

    monkeypatch.setattr(native, "last_error", lambda: "kernel launch failed: invalid argument")
    eng = FederatedEngine.__new__(FederatedEngine)
    eng.timeout = 3.0
    cases = [(1, FederationTimeout, "theta broadcast never arrived"),
             (2, FederationTimeout, "did not deliver its partial"),
             (3, FederationTimeout, "never arrived; a peer node"),
             (4, FederationError, "mbarrier pipeline stalled"),
             (-5, FederationTimeout, "invalid argument"),
             (engine_mod.RC_LAUNCH_FAILED, FederationError, "could not be launched .*invalid argument"),
             (-8, FederationError, "rc=-8")]
    for rc, exc, msg in cases:
        with pytest.raises(exc, match=msg) as info:
            eng._raise(rc)
        if rc == engine_mod.RC_LAUNCH_FAILED:
            assert not isinstance(info.value, TimeoutError)
    assert engine_mod.RC_LAUNCH_FAILED == -10


# ---------------------------------------------------------------------------------------------------------------------
# GPU


@pytest.fixture(scope="module")
def dev():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from pytensor_federated_b200.ops import native

    native.load()   # a GPU box without the native library is a failure, not a skip
    return torch.device("cuda:0")


def _engine(model, monkeypatch, env=None, grid=None):
    from pytensor_federated_b200.parallel import FederatedEngine

    for k in LL_VARS:
        monkeypatch.delenv(k, raising=False)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    return FederatedEngine(model, grid=grid)


def _linreg_model(case: Case, dev):
    import torch

    from pytensor_federated_b200.models import LinregShards

    return LinregShards(case.xs, case.ys, case.sigmas, local_ids=case.local_ids, n_shards_total=case.n_total,
                        device=dev, dtype=torch.float32 if case.dtype == "f32" else torch.float64)


def _alternate(eng, thetas, evaluate) -> List[Tuple[int, np.ndarray]]:
    """Six evaluations alternating two thetas, ``reset()``, then two more (theta 2 first)."""
    out = [(i % 2, evaluate(thetas[i % 2])) for i in range(6)]
    eng.reset()
    out += [((i + 1) % 2, evaluate(thetas[(i + 1) % 2])) for i in range(2)]
    return out


def _run_mode(eng, inputs_of, thetas, how: str):
    if how == "spec":
        assert eng.set_speculative(300.0) and eng.speculative

    def evaluate(theta):
        if how == "device":
            eng.set_device_theta(inputs_of(theta))
            return np.array(eng.wait(eng.launch()), copy=True)
        return eng.evaluate_raw(inputs_of(theta))

    return _alternate(eng, thetas, evaluate)


def _check_linreg(case: Case, results, grid: int) -> None:
    exps = [expected(case, th, grid) for th in case.thetas]
    for which, vals in results:
        d = deviation(case, exps[which], vals)
        assert d <= 1.0, f"{case.name} theta {which + 1}: {d:.3g} tolerances"


def _kernel_cases() -> List[Case]:
    k = []
    edge = [0, 1, 31, 32, 33, 4096]
    k.append(exact_case("small-1", [10], seed=20, want_grid=-1))
    k.append(exact_case("small-8", edge + [5, 64], seed=21, want_grid=-1))
    k.append(exact_case("small-9", edge + [5, 64, 2], seed=22, want_grid=-1))
    k.append(exact_case("small-33", (edge[:-1] * 7)[:32] + [4096], seed=23, want_grid=-1))
    k.append(exact_case("small-257", [(3 * i) % 40 for i in range(256)] + [4096], seed=24, want_grid=-1))
    k.append(exact_case("auto-16384-small", [4096] * 4, seed=25, want_grid=-1))
    k.append(exact_case("auto-4097-grid1", [4097], seed=26, want_grid=1))
    k.append(exact_case("auto-16385-grid2", [4096] * 4 + [1], seed=27, want_grid=2))
    for g in (2, 15, 16, 17, 33):
        sizes = [j * g * BLOCK + d for j in (1, 2) for d in (-1, 0, 1)] + [g * BLOCK // 2 + 3]
        k.append(exact_case(f"grid{g}-stride-edges", sizes, seed=30 + g, grid=g, want_grid=g))
    k.append(exact_case("grid1050-66-groups", [2 * 1050 * BLOCK + 1, 1050 * BLOCK - 1, 77], seed=40, grid=1050,
                        want_grid=1050))
    k.append(exact_case("auto-9M-rows-528", [3_000_001, 3_000_000, 2_999_999, 5], seed=41, want_grid=528))
    k.append(exact_case("ids-3-7-of-10", [5000, 300], seed=42, n_total=10, local_ids=[3, 7], grid=4, want_grid=4))
    k.append(exact_case("ids-3-7-of-10-small", [50, 3], seed=43, n_total=10, local_ids=[3, 7], want_grid=-1))
    k.append(exact_case("max-shards", [2] * 40, seed=44, n_total=14496, local_ids=range(0, 14496, 371), grid=3,
                        want_grid=3))
    k.append(inexact_case("inexact-offset-auto", [60_000, 20_000, 7], seed=45, offset=True, want_grid=5))
    k.append(inexact_case("inexact-offset-grid33", [40_000, 1], seed=46, offset=True, grid=33, want_grid=33))
    k.append(inexact_case("inexact-offset-small", [4000, 33, 0], seed=47, offset=True, want_grid=-1))
    k.append(inexact_case("inexact-plain-grid17", [50_000], seed=48, offset=False, grid=17, want_grid=17))
    return k


KERNEL_CASES = _kernel_cases()


@pytest.mark.parametrize("case", [c for c in KERNEL_CASES if c.exact], ids=lambda c: c.name)
def test_kernel_case_is_inside_its_budget(case):
    budget(case)
    if case.name == "max-shards":
        from pytensor_federated_b200.models import LinregShards

        assert case.n_total == LinregShards.MAX_SHARDS_TOTAL


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", KERNEL_CASES, ids=lambda c: c.name)
def test_linreg_kernel_matches_the_exact_oracle(dev, case, monkeypatch):
    """fp64 storage, then float32 storage: exact cases give the same bits either way."""
    bits = {}
    for c in (case, case.as_f32()):
        with _engine(_linreg_model(c, dev), monkeypatch, grid=c.grid) as eng:
            grid = eng.grid
            print(f"{c.name}: grid={grid}")
            assert grid == case.want_grid
            res = _run_mode(eng, lambda th: list(th), c.thetas, "eval")
        _check_linreg(c, res, grid)
        bits[c.dtype] = [v for _, v in res]
    if case.exact:
        for u, v in zip(bits["f64"], bits["f32"]):
            assert np.array_equal(u, v)


# transport modes: (name, environment, grid, how); grid None = the automatic choice (small mode for these models)
MODES = [
    ("auto", {}, None, "eval"),
    ("grid8", {}, 8, "eval"),
    ("grid8-no-ll", {"B200FED_NO_LL": "1"}, 8, "eval"),
    ("grid8-flag-results", {"B200FED_LL_MAX_VALS": "0"}, 8, "eval"),
    ("grid1", {}, 1, "eval"),
    ("grid1-no-ll", {"B200FED_NO_LL": "1"}, 1, "eval"),
    ("auto-speculative", {}, None, "spec"),
    ("grid8-speculative", {}, 8, "spec"),
    ("grid8-device-theta", {}, 8, "device"),
]


def transport(n_theta: int, n_vals: int, env: dict) -> str:
    """Which protocol the runtime picks (csrc/runtime.cu, b200_engine_create)."""
    ll_theta = n_theta <= int(env.get("B200FED_LL_MAX_THETA", 4096)) and "B200FED_NO_LL" not in env
    ll_vals = ll_theta and n_vals <= int(env.get("B200FED_LL_MAX_VALS", 2048))
    return f"theta={'LL' if ll_theta else 'flag'} results={'LL' if ll_vals else 'flag'}" + \
        (" root-cached" if not ll_vals and n_vals <= 1024 else "")


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("n_shards", [256, 257, 341, 342, 682, 683, 1024, 1025, 3056, 3057, 5000])
def test_linreg_transport_modes_give_the_same_bits(dev, n_shards, monkeypatch):
    rng = np.random.default_rng(n_shards)
    case = exact_case(f"matrix-{n_shards}", list(rng.integers(0, 40, n_shards)), seed=n_shards)
    budget(case)
    model = _linreg_model(case, dev)
    per_grid, reference = {}, None
    for name, env, grid, how in MODES:
        if how == "spec" and model.n_theta_words > 1024:
            with _engine(model, monkeypatch, env, grid) as eng:
                assert eng.set_speculative(300.0) is False   # theta too large for tagged host words
            continue
        with _engine(model, monkeypatch, env, grid) as eng:
            g = eng.grid
            print(f"{case.name} {name}: grid={g} {transport(model.n_theta_words, model.n_vals, env)}")
            res = _run_mode(eng, lambda th: list(th), case.thetas, how)
        _check_linreg(case, res, g)
        vals = [v for _, v in res]
        if g in per_grid:   # same grid: every bit, LL included
            for u, v in zip(per_grid[g], vals):
                assert np.array_equal(u, v), f"{name} differs from the other modes on grid {g}"
        per_grid.setdefault(g, vals)
        if reference is None:
            reference = vals
        for u, v in zip(reference, vals):   # any grid: the exact gradients
            assert np.array_equal(u.reshape(-1, 3)[:, 1:], v.reshape(-1, 3)[:, 1:])
    assert {1, 8} <= set(per_grid) and len(per_grid) == 3   # the automatic grid, 8 and 1


_FRESH_PROCESS = """
import numpy as np, torch
from pytensor_federated_b200.models import LinregShards
from pytensor_federated_b200.parallel import FederatedEngine
for n in (3055, 3056, 3057):
    m = LinregShards([np.arange(5.0)], [np.arange(5.0) + 1.0], [1.0], local_ids=[n - 1], n_shards_total=n, device="cuda:0")
    with FederatedEngine(m, grid=2) as eng:
        v = eng.evaluate_raw([np.zeros(n), np.ones(n)]).reshape(-1, 3)
    assert np.array_equal(v[n - 1, 1:], [5.0, 10.0]) and not np.any(v[: n - 1]), n
print("ok")
"""


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_shared_memory_opt_in_in_a_fresh_process(dev):
    """The shared-memory limit a launch raises stays raised for the rest of the process, so the models just past
    the 48 KB default run first thing in a process of their own."""
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, "-c", _FRESH_PROCESS], cwd=root, capture_output=True, text=True, timeout=240,
                         env={**os.environ, "PYTHONPATH": root})
    assert res.returncode == 0 and res.stdout.strip().endswith("ok"), res.stdout + res.stderr


def _other_kernel(which: str, dev):
    """A model of another kernel, its input builder and two thetas."""
    import torch

    from pytensor_federated_b200.models import Fp8GlmShards, GlmShards, OdeShards, synth_lv_shard

    torch.manual_seed(5)
    rng = np.random.default_rng(6)
    if which == "ode":
        shards = [synth_lv_shard(n, 8, seed=s, device=dev) for s, n in enumerate([300, 129])]
        model = OdeShards(*[[s[i] for s in shards] for i in range(4)])
        thetas = [[np.array([1.0, 0.4, 0.8, 0.2]) * (1 + 0.05 * rng.normal(size=4))] for _ in range(2)]
        return model, thetas
    P, K = (256, 16) if which == "tc-k16" else ((100 if which == "generic" else 256), 1)
    rows = [30_000 + 5, 5_000]
    dtype = torch.float32 if which == "generic" else torch.bfloat16
    Xs = [torch.randn(n, P, device=dev).to(dtype) for n in rows]
    ys = [(torch.rand(n, device=dev) < 0.5).float() for n in rows]
    if which == "fp8":
        model = Fp8GlmShards.from_dense(Xs, ys, groups=[0, 1], n_groups=2)
    else:
        model = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, n_chains=K, kernel=which.split("-")[0])
    shape = (K, 2) if K > 1 else (2,)
    bshape = (K, P) if K > 1 else (P,)
    thetas = [[(rng.normal(size=shape) * 0.1).astype(np.float32), (rng.normal(size=bshape) * 0.03).astype(np.float32)]
              for _ in range(2)]
    return model, thetas


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("which", ["tc-k1", "tc-k16", "simt", "generic", "fp8", "ode"])
def test_other_kernels_keep_their_bits_in_every_transport_mode(dev, which, monkeypatch):
    """Within a grid every mode gives the same bits.  The tensor-core and fp8 kernels sum double-double partials,
    so their bits do not depend on the grid either."""
    model, thetas = _other_kernel(which, dev)
    if which == "tc-k16":
        assert model.n_theta_words > 4096 and model.n_vals > 2048   # beyond both tagged-word thresholds
    per_grid, default_grid, reference = {}, None, None
    for name, env, grid, how in MODES:
        grid = None if grid == 8 else grid   # this kernel's own grid
        if how == "spec" and (model.n_theta_words > 1024 or "NO_LL" in str(env)):
            continue
        with _engine(model, monkeypatch, env, grid) as eng:
            g = eng.grid
            print(f"{which} {name}: grid={g} {transport(model.n_theta_words, model.n_vals, env)}")
            res = _run_mode(eng, lambda th: th, thetas, how)
        first = {}
        for which_theta, v in res:   # each theta gives one result, before and after reset()
            if which_theta in first:
                assert np.array_equal(first[which_theta], v), f"{name}: theta {which_theta + 1} changed its bits"
            first.setdefault(which_theta, v)
        assert not np.array_equal(first[0], first[1])
        vals = [first[0], first[1]]
        if grid is None:
            default_grid = g if default_grid is None else default_grid
            assert g == default_grid
        if g in per_grid:
            for u, v in zip(per_grid[g], vals):
                assert np.array_equal(u, v), f"{name} differs from the other modes on grid {g}"
        per_grid.setdefault(g, vals)
        reference = vals if reference is None else reference
        if which in ("tc-k1", "tc-k16", "fp8"):
            for u, v in zip(reference, vals):
                assert np.array_equal(u, v), f"{name} (grid {g}) differs from the default grid"
    assert 1 in per_grid and len(per_grid) == (1 if default_grid == 1 else 2)
