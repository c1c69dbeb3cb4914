"""Every GLM kernel's data path, bit for bit, on inputs where the Gaussian families are exact.

In the Gaussian family (and ``gaussian_scale`` at ``log_dispersion = 0``, where 1 / sigma = 1 exactly) the residual
is ``r = y - eta``: no transcendental.  With small integer X (or e4m3 integers times power-of-two block scales),
coefficients, responses, offsets and intercepts on one dyadic grid and small integer weights, every product and
every partial sum the kernels form is exact: the wgmma and FMA chains in fp32, the (hi, mid, lo) bf16 split of
theta, the (hi, lo) bf16 split and the radix-16 e4m3 expansion of ``w r``, the double-double totals and the 40.24
fixed point of the CUDA-core kernels.  So every intercept, beta and dispersion gradient the kernels return equals
an int64 computation from the integer inputs, and any row, tile, chunk, group, node, chain column or row-data
element that goes astray shows up as a difference, however few rows it touches.

CPU: :func:`budget` asserts that each case stays inside that exact range for its kernel; :func:`oracle` computes
the expected gradients in int64 without ``models/glm.py``, and ``GlmShards.reference_partial`` in fp64 must agree
with it bit for bit; plausible data-path bugs applied to the oracle each change an expected gradient bit.
GPU: each case against the oracle with ``np.array_equal``; the log-likelihood, which rounds per row (the fp32
constant log(2 pi) / 2), within the fp32 summation bound of the kernel's longest accumulation.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import pytest
import torch

from pytensor_federated_b200.models import CustomFamily, Fp8GlmShards, GlmShards

LIMIT = 1 << 21        # |partial sums| in grid units: 3 bits of margin under fp32's 24 for aligning accumulators
KSTEP_LIMIT = 1 << 10  # one 32-row e4m3 wgmma K step, in units of its finest product (fewer bits than fp32)
SM_H100 = 132          # SMs of an H100 SXM: the chunk tables of the CPU checks
TC_CHUNKS = (2, 32, 4)   # chunk table of csrc/glm_tc.cu: tiles a multiple of 2, kMaxChunk, kMinChunk
FP8_CHUNKS = (3, 30, 6)  # csrc/glm_fp8.cu: kChunkMultiple, kMaxChunkF, kMinChunkF
TILE = 128
LOG_SQRT_2PI_F32 = np.float32(0.918938533204672742)
# Longest fp32 accumulation of per-row log-likelihoods, in additions per running sum:
#   tc:      2 rows per thread per tile x kMaxChunk = 32 tiles, then double (glm_tc.cu, ll_acc)
#   fp8:     2 rows per thread per tile x kMaxChunkF = 30 tiles (glm_fp8.cu, ll_acc)
#   simt:    one row per lane per 8-row batch, flushed to double every 256 batches (glm_simt.cu, flush_count)
#   generic: lane 0 adds the 8 rows of a batch, flushed every 64 batches (glm_generic.cu, flush)
LL_TERMS = {"tc": 64, "fp8": 60, "simt": 256, "generic": 512}


# ------------------------------------------------------------------------------------------------ cases
@dataclass
class Seg:
    X: np.ndarray               # int64 or int16 [n, P]: the stored design matrix times 2^xs
    y: np.ndarray               # int64 [n], grid units (0 where the row is NaN)
    o: Optional[np.ndarray]     # int64 [n] grid units, or None
    w: Optional[np.ndarray]     # int64 [n], or None (weight 1)
    nan: np.ndarray             # bool [n]: rows of weight 0 whose y (and offset) are NaN
    group: int
    node: int
    xq: Optional[np.ndarray] = None   # fp8: e4m3 integers [n, P]
    sc: Optional[np.ndarray] = None   # fp8: UE8M0 scale bytes [4 ceil(n / 128), P / 32]
    nz: Optional[np.ndarray] = None   # [m, 2] (row, feature) of zeros of X stored as -0.0


@dataclass
class Case:
    name: str
    kernel: str            # "tc", "fp8", "simt", "generic" or "custom" (CustomFamily on the general-shape kernel)
    family: str            # "gaussian", "gaussian_scale" or "gaussian_location_scale" (its scale at 0)
    P: int
    K: int
    G: int
    n_nodes: int
    xs: int                # X = X_int 2^-xs
    ts: int                # beta = beta_int 2^-ts; the grid unit of eta, y, offsets and intercepts is 2^-(xs + ts)
    segs: List[Seg]
    ic: np.ndarray         # int64 [K, G] grid units
    beta: np.ndarray       # int64 [K, P] units 2^-ts
    storage: str = "bf16"  # design matrix: "bf16", "fp32" or "fp8"
    ld: int = 0            # row stride of the stored matrix (0: P)
    misalign: bool = False # the matrix starts one element past a 16-byte boundary

    @property
    def e(self) -> int:
        return self.xs + self.ts

    @property
    def disp(self) -> bool:
        return self.family == "gaussian_scale"

    @property
    def pair(self) -> bool:
        """Chain k runs as kernel columns 2k (the mean: ic, beta) and 2k + 1 (the log scale: all coefficients 0)."""
        return self.family == "gaussian_location_scale"

    @property
    def columns(self) -> int:
        return 2 * self.K if self.pair else self.K

    @property
    def n_rows(self) -> List[int]:
        return [s.X.shape[0] for s in self.segs]

    def inputs(self):
        ic = (self.ic * 2.0 ** -self.e).astype(np.float32)
        beta = (self.beta * 2.0 ** -self.ts).astype(np.float32)
        out = [ic[0], beta[0]] if self.K == 1 else [ic, beta]
        if self.pair:
            out += [np.zeros_like(v) for v in out]
        if self.disp:
            out.append(np.float32(0.0) if self.K == 1 else np.zeros(self.K, np.float32))
        return out


def make_case(name, kernel, *, P, rows, K=1, G=1, groups=None, nodes=None, n_nodes=1, offsets=False, weights=False,
              family="gaussian", storage="bf16", ld=0, misalign=False, seed=0) -> Case:
    """A case on the dyadic grid.  y is eta of chain 0 plus a residual d, so the other chains (beta and intercepts
    shifted by a few units) see residuals d - x' delta_beta - delta_intercept.  Some coefficients are odd multiples
    of the grid above 256 (they need the mid bf16 term); on the bf16 kernels about a fifth of the rows have |w r| >
    256 units (they need the lo term of the residual split).  Offsets and weights, where present, skip one segment
    (absent for that segment); weights include 0, and half of the weight-0 rows carry NaN y and offsets."""
    rng = np.random.default_rng(seed)
    if kernel == "fp8":
        xs, ts, d_max, big, dbeta, dic = 1, 5, 10, 0.0, 1, 2   # small residuals: the e4m3 K-step budget
    elif family == "gaussian_scale":
        xs, ts, d_max, big, dbeta, dic = 0, 3, 12, 0.0, 1, 2   # q = d^2 - 1 on the grid's square: small d
    elif kernel == "custom":
        xs, ts, d_max, big, dbeta, dic = 0, 3, 6, 0.0, 0, 0    # the custom LL -d^2 / 2 is exact too: small d
    else:
        xs, ts, d_max, big, dbeta, dic = 0, 6, 40, 0.2, 2, 4
    groups = list(groups) if groups is not None else [0] * len(rows)
    nodes = list(nodes) if nodes is not None else [0] * len(rows)
    beta0 = rng.integers(-8, 9, P)
    wide = rng.choice(P, max(1, P // 8), replace=False)
    beta0[wide] = rng.choice([-1, 1], wide.size) * (2 * rng.integers(129, 256, wide.size) + 1)   # 9 significant bits
    beta = np.repeat(beta0[None], K, axis=0)
    ic0 = rng.integers(-200, 201, G)
    ic = np.repeat(ic0[None], K, axis=0)
    for k in range(1, K):
        f = rng.choice(P, min(P, 4 if kernel != "fp8" else 1), replace=False)
        beta[k, f] += rng.choice([-1, 1], f.size) * rng.integers(1, max(dbeta, 1) + 1, f.size)
        ic[k] += rng.integers(-dic, dic + 1, G)
    segs = []
    for si, (n, g, nd) in enumerate(zip(rows, groups, nodes)):
        xq = sc = None
        if kernel == "fp8":
            xq = rng.integers(-2, 3, (n, P))
            n_rb = 4 * -(-n // TILE)
            sc = np.full((n_rb, P // 32), 127, dtype=np.int64)
            sc[: -(-n // 32)] = rng.integers(126, 129, (-(-n // 32), P // 32))   # 2^-1, 2^0, 2^1 per 32 x 32 block
            X = xq << np.repeat(np.repeat(sc[: -(-n // 32)] - 126, 32, 0)[:n], 32, 1)
        else:
            X = rng.integers(-3, 4, (n, P))
        skip = len(rows) >= 3 and si == 1          # one segment without the row arrays the model has
        o = rng.integers(-600, 601, n) if offsets and not skip else None
        w = rng.choice(4, n, p=[0.15, 0.35, 0.25, 0.25]) if weights and not skip else None
        nan = (w == 0) & (rng.random(n) < 0.5) if w is not None else np.zeros(n, bool)
        d = rng.integers(-d_max, d_max + 1, n)
        wide_r = rng.random(n) < big
        d[wide_r] = rng.choice([-1, 1], int(wide_r.sum())) * rng.integers(260, 701, int(wide_r.sum()))
        eta0 = X @ beta0 + ic0[g] + (o if o is not None else 0)
        y = np.where(nan, 0, eta0 + d)
        segs.append(Seg(X, y, o, w, nan, g, nd, xq, sc))
    return Case(name, kernel, family, P, K, G, n_nodes, xs, ts, segs, ic, beta, storage, ld, misalign)


# ------------------------------------------------------------------------------------------------ emulation
def bf16_split(v: np.ndarray, n: int) -> List[np.ndarray]:
    """``v`` (float32-exact values) as the kernels split it: n bf16 terms, hi first (as test_numerics_emulation.py)."""
    terms, rem = [], torch.from_numpy(np.asarray(v, dtype=np.float32))
    for _ in range(n):
        t = rem.to(torch.bfloat16).float()
        terms.append(t.double().numpy())
        rem = rem - t
    return terms


def e4m3_digits(wr: np.ndarray, unit: float):
    """``w r`` of one segment and chain (grid units) as csrc/glm_fp8.cu's DYN path stores it: per 32-row group a power
    of two 2^ex with max |w r| / 2^ex in [0.5, 1), then ``expand16(w r / 2^ex * 256)``.  Returns the four e4m3 terms
    ``[4, n]`` (raw e4m3 values, as MMA #2 multiplies them) and each term's value ``t_k 16^-k 2^ex / 256`` in grid
    units ``[4, n]`` (float64)."""
    n = wr.size
    ng = -(-n // 32)
    r = np.zeros(ng * 32, np.float32)
    r[:n] = wr * unit
    m = np.abs(r.reshape(ng, 32)).max(1)
    ex = np.where(m > 0, np.frexp(m)[1], 0).clip(-126, 126)
    scale = np.repeat(np.ldexp(np.float32(1), ex).astype(np.float32), 32)
    rem = torch.from_numpy(r / scale * np.float32(256))
    raw = []
    for _ in range(4):
        t = rem.clamp(-448, 448).to(torch.float8_e4m3fn).float()
        raw.append(t.double().numpy()[:n])
        rem = (rem - t) * 16.0
    raw = np.stack(raw)
    vals = raw * (16.0 ** -np.arange(4))[:, None] * (scale[:n] / 256.0) / unit
    return raw, vals


def imatmul(A: np.ndarray, B: np.ndarray, block: int = 1 << 16) -> np.ndarray:
    """``A @ B`` of integer matrices as int64, through fp64 BLAS in blocks of ``block`` rows of A and of the inner
    dimension.  fp64 is exact here: every partial sum of a block is an integer of magnitude at most inner x max|a| x
    max|b|, asserted below 2^53, and the blocks add in int64."""
    n, m = A.shape
    out = np.zeros((n, B.shape[1]), np.int64)
    for i in range(0, n, block):
        for j in range(0, m, block):
            a = A[i : i + block, j : j + block].astype(np.float64)
            b = B[j : j + block].astype(np.float64)
            assert np.abs(a).max(initial=0) * np.abs(b).max(initial=0) * a.shape[1] < 2.0 ** 53
            out[i : i + block] += (a @ b).astype(np.int64)
    return out


def _eta(case: Case, seg: Seg, beta: np.ndarray, o: Optional[np.ndarray]) -> np.ndarray:
    """eta [n, K] in grid units from integer coefficients [K, P] (units 2^-ts)."""
    eta = imatmul(seg.X, beta.T) + case.ic[:, seg.group][None, :]
    return eta + (o[:, None] if o is not None else 0)


def _wr(case: Case, seg: Seg, beta=None, o="seg", w="seg"):
    """(d, w, w d) [n, K] in grid units; rows of weight 0 give 0 (their y and offset may be NaN)."""
    o = seg.o if isinstance(o, str) else o
    w = seg.w if isinstance(w, str) else w
    d = seg.y[:, None] - _eta(case, seg, case.beta if beta is None else beta, o)
    ww = np.ones(seg.X.shape[0], np.int64) if w is None else w
    d = np.where(ww[:, None] == 0, 0, d)
    return d, ww, ww[:, None] * d


def chunk_table(n_rows, sm_count, multiple, max_chunk, min_chunk) -> np.ndarray:
    """``[n_chunks, 3]`` = (segment, first tile, tiles) from the runtime's own chunk builder (csrc/chunks.h)."""
    from pytensor_federated_b200.ops import native

    lib = native.load()
    rows = (C.c_longlong * len(n_rows))(*n_rows)
    cap = 1 << 16
    out = (C.c_int * (3 * cap))()
    n = lib.b200_glm_tc_chunk_table(rows, len(n_rows), sm_count, multiple, max_chunk, min_chunk, out, cap)
    assert 0 < n <= cap
    return np.frombuffer(out, dtype=np.int32, count=3 * n).reshape(n, 3).copy()


def _window_sums(A: np.ndarray, bounds) -> int:
    """max over the row windows [a, b) of the column sums of ``A [n, ...]``."""
    cs = np.concatenate([np.zeros((1,) + A.shape[1:], A.dtype), np.cumsum(A, axis=0)])
    return max(np.abs(cs[b] - cs[a]).max() for a, b in bounds) if bounds else 0


def _window_xsums(absX: np.ndarray, col: np.ndarray, bounds) -> int:
    """``_window_sums(absX * |col|[:, None], bounds)`` without forming the product: one window per row of a matrix
    product."""
    if not bounds:
        return 0
    M = np.zeros((len(bounds), absX.shape[0]), np.int64)
    for j, (a, b) in enumerate(bounds):
        M[j, a:b] = np.abs(col[a:b])
    return int(imatmul(M, absX).max())


def _row_blocks(n: int, starts, rows: int = 1 << 16):
    """``[r0, r1)`` covering ``[0, n)`` in blocks of about ``rows`` rows, cut only at the given window starts (a
    window, a chunk of the segment, stays in the block its start is in)."""
    cuts = [0]
    for a in sorted(starts):
        if a - cuts[-1] >= rows:
            cuts.append(a)
    if not starts:
        cuts = list(range(0, n, rows)) or [0]
    return list(zip(cuts, cuts[1:] + [n]))


def seg_rows(s: Seg, r0: int, r1: int) -> Seg:
    """Rows ``[r0, r1)`` of a segment, as a segment (views)."""
    cut = lambda v: None if v is None else v[r0:r1]
    return Seg(s.X[r0:r1], s.y[r0:r1], cut(s.o), cut(s.w), s.nan[r0:r1], s.group, s.node, cut(s.xq), s.sc,
               None if s.nz is None else s.nz[(s.nz[:, 0] >= r0) & (s.nz[:, 0] < r1)] - [r0, 0])


def _lowbit(v: np.ndarray) -> np.ndarray:
    return v & -v


# ------------------------------------------------------------------------------------------------ budget
def budget(case: Case, sm_count: int = SM_H100) -> None:
    """Asserts that every value the case's kernel forms is exact, in grid units (see the module docstring)."""
    k8 = case.kernel == "fp8"
    split = case.kernel in ("tc", "fp8")        # theta as (hi, mid, lo) bf16 terms for the wgmma of eta
    unit = 2.0 ** -case.e
    # the stored values are exact in their format
    if split:
        terms = bf16_split(case.beta * 2.0 ** -case.ts, 3)
        assert np.array_equal(sum(terms), case.beta * 2.0 ** -case.ts), "beta is not the sum of its three bf16 terms"
        assert all(np.array_equal(t * 2.0 ** case.ts, np.rint(t * 2.0 ** case.ts)) for t in terms)
        beta_terms = [np.rint(t * 2.0 ** case.ts).astype(np.int64) for t in terms]
    else:
        beta_terms = [case.beta]
    table = None
    if case.kernel in ("tc", "fp8"):
        table = chunk_table(case.n_rows, sm_count, *(FP8_CHUNKS if k8 else TC_CHUNKS))
    tot_xwr = np.zeros((case.K, case.P), np.int64)
    tot_wr = np.zeros(case.K, np.int64)
    tot_ll = 0
    for si, seg in enumerate(case.segs):
        bounds = []
        if table is not None:
            bounds = sorted((f * TILE, min(seg.X.shape[0], (f + t) * TILE)) for sg, f, t in table if sg == si)
        # a long segment in blocks of whole chunks: every check below is per row or per chunk
        for r0, r1 in _row_blocks(seg.X.shape[0], [a for a, _ in bounds]):
            s = seg_rows(seg, r0, r1)
            win = [(a - r0, b - r0) for a, b in bounds if r0 <= a < r1]
            Xv = s.X * 2.0 ** -case.xs
            if case.storage == "bf16":
                assert np.array_equal(torch.from_numpy(Xv).to(torch.bfloat16).double().numpy(), Xv), "X is not bf16"
            if k8:
                assert np.all(np.abs(s.xq) <= 16), "e4m3 integers are exact up to 16"
            absX = np.abs(s.X)
            # eta: every partial dot product of every term, then the intercept and the offset
            for bt in beta_terms:
                assert imatmul(absX, np.abs(bt).T).max() < LIMIT, f"{case.name}: x' beta term exceeds the eta budget"
            eta_abs = imatmul(absX, np.abs(case.beta).T) + np.abs(case.ic[:, s.group])[None, :]
            if s.o is not None:
                eta_abs = eta_abs + np.abs(s.o)[:, None]
            assert eta_abs.max() < LIMIT and np.abs(s.y).max() < LIMIT, f"{case.name}: |eta| or |y| over budget"
            d, w, wr = _wr(case, s)
            assert np.abs(d).max() < LIMIT
            for k in range(case.K):
                if case.kernel == "tc":
                    hi, lo = (np.rint(t / unit).astype(np.int64) for t in bf16_split(wr[:, k] * unit, 2))
                    assert np.array_equal(hi + lo, wr[:, k]), f"{case.name}: w r is not hi + lo in bf16"
                    cols = [hi, lo, wr[:, k]]
                elif k8:
                    raw, vals = e4m3_digits(wr[:, k], unit)
                    assert np.array_equal(vals, np.rint(vals)), f"{case.name}: an e4m3 term of w r is off the grid"
                    vals = vals.astype(np.int64)
                    assert np.array_equal(vals.sum(0), wr[:, k]), f"{case.name}: w r is not its 4-term e4m3 expansion"
                    cols = [*vals, wr[:, k]]
                    # MMA #2: one wgmma K step = 32 rows of x_q . t_k, accumulated with fewer bits than fp32
                    n = s.X.shape[0]
                    ng = -(-n // 32)
                    xq = np.zeros((ng * 32, case.P), np.int64)
                    xq[:n] = s.xq
                    for t in raw:
                        ti = np.zeros(ng * 32, np.int64)
                        ti[:n] = np.rint(t * 512)                      # e4m3 values are multiples of 2^-9
                        p = np.abs(xq.reshape(ng, 32, case.P) * ti.reshape(ng, 32, 1))
                        lb = np.where(p > 0, _lowbit(p), np.int64(1) << 62).min(1)   # finest product per column
                        tot = p.sum(1)
                        assert np.all((tot == 0) | (tot < KSTEP_LIMIT * lb)), f"{case.name}: e4m3 K step over budget"
                else:
                    cols = [wr[:, k]]
                if table is not None:   # fp32 accumulation windows: the chunks
                    for col in cols:
                        assert _window_xsums(absX, col, win) < LIMIT, f"{case.name}: x r over budget"
                    assert _window_sums(np.abs(wr[:, k]), win) < LIMIT, f"{case.name}: sum w r over budget"
                    if case.disp:
                        q = w * np.abs(d[:, k] ** 2 - (1 << 2 * case.e))
                        assert _window_sums(q, win) < LIMIT, f"{case.name}: sum w q over budget"
                if case.pair:
                    # column 2k + 1 at s = 0: the residual w (d^2 - 1), units 2^-2e, through the same (hi, lo) split
                    # and chunk sums as the mean's (d^2 - 1 is exact in fp32 below 2^24)
                    assert (d[:, k] ** 2).max() < 1 << 24, f"{case.name}: d^2 over budget"
                    ws = w * (d[:, k] ** 2 - (1 << 2 * case.e))
                    u2 = 2.0 ** (-2 * case.e)
                    hi, lo = (np.rint(t / u2).astype(np.int64) for t in bf16_split(ws * u2, 2))
                    assert np.array_equal(hi + lo, ws), f"{case.name}: w (d^2 - 1) is not hi + lo in bf16"
                    for col in (hi, lo, ws):
                        assert _window_xsums(absX, col, win) < LIMIT, f"{case.name}: x w (d^2 - 1) over budget"
                    assert _window_sums(np.abs(ws), win) < LIMIT, f"{case.name}: sum w (d^2 - 1) over budget"
                tot_xwr[k] += imatmul(np.abs(wr[:, k])[None, :], absX)[0]
                tot_wr[k] += np.abs(wr[:, k]).sum()
            tot_ll += int((w[:, None] * d * d).sum())
    if table is None:   # CUDA-core kernels: a warp's fp32 sums may run over the whole model
        assert tot_xwr.max() < LIMIT and tot_wr.max() < LIMIT, f"{case.name}: model-wide sums over budget"
        if case.kernel == "custom":   # -w d^2 / 2 in units of half the grid's square
            assert tot_ll < LIMIT, f"{case.name}: the custom log-likelihood's sum over budget"


# ------------------------------------------------------------------------------------------------ oracles
BUGS = ["r_hi", "theta_hi", "offset_bf16", "weight_shift", "drop_last", "stale_tile", "swap_chains", "wrong_group",
        "wrong_node", "drop_q"]


def oracle(case: Case, bug: Optional[str] = None):
    """The expected gradients in int64, in the kernel's layout: ``(gi [n_nodes, K, G] grid units, gb [n_nodes, K, P]
    units 2^-xs of the grid, q [n_nodes, K] units of the grid squared)``.  ``bug`` applies one of :data:`BUGS`.  A
    pair case has 2K columns: 2k the mean's, as above, and 2k + 1 the scale's, in units of the grid squared (gi) and
    2^-xs of it (gb)."""
    K, G, P = case.K, case.G, case.P
    gi = np.zeros((case.n_nodes, case.columns, G), np.int64)
    gb = np.zeros((case.n_nodes, case.columns, P), np.int64)
    q = np.zeros((case.n_nodes, case.columns), np.int64)
    mean = slice(0, None, 2) if case.pair else slice(None)
    unit = 2.0 ** -case.e
    beta = case.beta
    if bug == "theta_hi":
        beta = np.rint(bf16_split(beta * 2.0 ** -case.ts, 1)[0] * 2.0 ** case.ts).astype(np.int64)
    for si, s in enumerate(case.segs):
        o, w = s.o, s.w
        if bug == "offset_bf16" and o is not None:
            o = np.rint(bf16_split(o * unit, 1)[0] / unit).astype(np.int64)
        if bug == "weight_shift" and w is not None:
            w = np.roll(w, 1)
        if bug == "drop_last":
            w = (np.ones(s.X.shape[0], np.int64) if w is None else w.copy())
            w[-1] = 0
        d, ww, wr = _wr(case, s, beta, o, w)
        if bug in ("weight_shift", "drop_last"):   # a shifted weight may land on a NaN row: the select keeps it out
            wr = np.where(s.nan[:, None] & (ww[:, None] != 0), 0, wr)
        wr_b = wr
        if bug == "r_hi":
            wr_b = np.stack([np.rint(bf16_split(wr[:, k] * unit, 1)[0] / unit) for k in range(K)], 1).astype(np.int64)
        if bug == "stale_tile" and s.X.shape[0] > TILE:
            wr_b = wr.copy()
            m = min(TILE, s.X.shape[0] - TILE)
            wr_b[TILE : TILE + m] = wr[:m]   # tile 1 multiplied with tile 0's residuals
        node = (s.node + 1) % case.n_nodes if bug == "wrong_node" and si == 0 else s.node
        grp = (s.group + 1) % G if bug == "wrong_group" and si == 0 else s.group
        gi[node, mean, grp] += wr.sum(0)
        gb[node, mean] += imatmul(wr_b.T, s.X)
        if case.pair:   # the scale column at s = 0: dll/ds = z^2 - 1 with z = d
            ws = ww[:, None] * (d * d - (1 << 2 * case.e))
            gi[node, 1::2, grp] += ws.sum(0)
            gb[node, 1::2] += imatmul(ws.T, s.X)
        if case.disp and bug != "drop_q":
            q[node] += (ww[:, None] * (d * d - (1 << 2 * case.e))).sum(0)
    if bug == "swap_chains":
        gi[:, [0, 1]], gb[:, [0, 1]], q[:, [0, 1]] = gi[:, [1, 0]], gb[:, [1, 0]], q[:, [1, 0]]
    return gi, gb, q


def expected_raw(case: Case, ints, ll: np.ndarray) -> np.ndarray:
    """``[n_nodes, K, 1 + G + P (+ 1)]`` float64 (exact) from the oracle's integers and a log-likelihood per block
    (pair cases: ``[n_nodes, 2K, 1 + G + P]``)."""
    gi, gb, q = ints
    e = np.tile([case.e, 2 * case.e], case.K)[None, :, None] if case.pair else case.e
    parts = [ll[..., None], gi * 2.0 ** -e, gb * 2.0 ** -(e + case.xs)]
    if case.disp:
        parts.append((q * 2.0 ** (-2 * case.e))[..., None])
    return np.concatenate(parts, axis=2)


def row_loglik(case: Case):
    """``(sum_i w_i ll_i, sum_i |w_i ll_i|)`` per block ``[n_nodes, K]``: each row's ``w ll`` in float32 with the
    kernels' operations (``-0.5f * d * d`` is exact, so FMA contraction does not matter; minus the fp32 constant, one
    rounding; ``gaussian_scale`` then subtracts s = 0; times the weight, one rounding), summed exactly."""
    vals = [[[] for _ in range(case.K)] for _ in range(case.n_nodes)]
    for s in case.segs:
        d, ww, _ = _wr(case, s)
        df = (d * 2.0 ** -case.e).astype(np.float32)
        if case.kernel == "custom":
            ll = np.float32(-0.5) * df * df
        else:
            ll = np.float32(-0.5) * df * df - LOG_SQRT_2PI_F32
        wll = np.where(ww[:, None] == 0, np.float32(0), ww[:, None].astype(np.float32) * ll).astype(np.float64)
        for k in range(case.K):
            vals[s.node][k].append(wll[:, k])
    tot = np.zeros((case.n_nodes, case.K))
    mag = np.zeros((case.n_nodes, case.K))
    for n in range(case.n_nodes):
        for k in range(case.K):
            v = np.concatenate(vals[n][k]) if vals[n][k] else np.zeros(0)
            tot[n, k], mag[n, k] = math.fsum(v), math.fsum(np.abs(v))
    return tot, mag


# ------------------------------------------------------------------------------------------------ models
CUSTOM_GAUSSIAN = ("const float d = y - eta; ll = -0.5f * d * d; r = d;",
                   lambda y, eta: (-0.5 * (y - eta) ** 2, y - eta))


def build_model(case: Case, device) -> GlmShards:
    unit = 2.0 ** -case.e
    Xs, ys, os_, ws = [], [], [], []
    for s in case.segs:
        n = s.X.shape[0]
        y = torch.tensor(s.y * unit, dtype=torch.float32)
        y[torch.from_numpy(s.nan)] = float("nan")
        ys.append(y.to(device))
        if s.o is None:
            os_.append(None)
        else:
            o = torch.tensor(s.o * unit, dtype=torch.float32)
            o[torch.from_numpy(s.nan)] = float("nan")
            os_.append(o.to(device))
        ws.append(None if s.w is None else torch.tensor(s.w, dtype=torch.float32, device=device))
        if case.storage == "fp8":
            Xs.append(torch.tensor(s.xq, dtype=torch.float32).to(torch.float8_e4m3fn).to(device))
            continue
        dt = torch.bfloat16 if case.storage == "bf16" else torch.float32
        ld = case.ld or case.P
        buf = torch.zeros(n * ld + 1, dtype=dt, device=device)
        first = 1 if case.misalign else 0
        X = buf[first : first + n * ld].view(n, ld)[:, : case.P]
        X.copy_((torch.from_numpy(s.X).to(device, torch.float32) * 2.0 ** -case.xs).to(dt))
        if s.nz is not None and len(s.nz):
            X[torch.from_numpy(s.nz[:, 0]).to(device), torch.from_numpy(s.nz[:, 1]).to(device)] = -0.0
        Xs.append(X)
    kw = dict(groups=[s.group for s in case.segs], n_groups=case.G, n_chains=case.K,
              offsets=os_ if any(o is not None for o in os_) else None,
              weights=ws if any(w is not None for w in ws) else None)
    if case.n_nodes > 1:
        kw.update(node_ids=[s.node for s in case.segs], n_nodes=case.n_nodes)
    if case.kernel == "fp8":
        scales = [torch.tensor(s.sc, dtype=torch.uint8, device=device) for s in case.segs]
        return Fp8GlmShards(Xs, scales, ys, family=case.family, **kw)
    if case.kernel == "custom":
        return GlmShards(Xs, ys, family=CustomFamily(CUSTOM_GAUSSIAN[0], torch_fn=CUSTOM_GAUSSIAN[1]), **kw)
    return GlmShards(Xs, ys, family=case.family, kernel=case.kernel, **kw)


# ------------------------------------------------------------------------------------------------ the matrix
def _cases() -> List[Case]:
    c = []
    tc = lambda name, **kw: c.append(make_case(name, "tc", seed=len(c), **kw))
    tc("tc_k1_p8_short_segments", P=8, rows=[1, 2, 127, 128, 129])
    tc("tc_k2_p64_offsets_g7", P=64, K=2, G=7, rows=[255, 257, 4095, 4096], groups=[6, 2, 4, 0], offsets=True)
    tc("tc_k4_p72_weights_g7", P=72, K=4, G=7, rows=[4097, 389, 1, 128], groups=[3, 3, 1, 5], weights=True)
    tc("tc_k5_p128_both_g300", P=128, K=5, G=300, rows=[129, 4096, 2000], groups=[299, 17, 150], offsets=True,
       weights=True)
    tc("tc_k8_p200_both", P=200, K=8, G=7, rows=[127, 3000, 4097], groups=[5, 0, 5], offsets=True, weights=True)
    tc("tc_k9_p256", P=256, K=9, rows=[2, 5000, 641])
    tc("tc_k13_p256_offsets", P=256, K=13, G=7, rows=[4095, 129], groups=[1, 0], offsets=True)
    tc("tc_k16_p256_both_g300", P=256, K=16, G=300, rows=[1000, 257], groups=[7, 255], offsets=True, weights=True)
    tc("tc_smem_boundary_p384_k8_g238", P=384, K=8, G=238, rows=[3000, 1, 700], groups=[237, 0, 100], offsets=True,
       weights=True)
    tc("tc_nodes", P=128, K=4, G=7, rows=[300, 4097, 129, 50, 1000], groups=[2, 0, 6, 2, 1], nodes=[0, 2, 0, 1, 2],
       n_nodes=4, offsets=True, weights=True)
    tc("tc_1m_rows", P=8, K=2, G=2, rows=[1_100_003, 5], groups=[1, 0], offsets=True, weights=True)
    sc = lambda name, **kw: c.append(make_case(name, "tc", family="gaussian_scale", seed=len(c), **kw))
    sc("scale_k1_both", P=64, rows=[500, 4097, 3], G=2, groups=[1, 0, 1], offsets=True, weights=True)
    sc("scale_k4_nodes", P=128, K=4, G=3, rows=[129, 2000, 77], groups=[2, 0, 1], nodes=[1, 0, 1], n_nodes=2)
    sc("scale_k16_both", P=256, K=16, G=5, rows=[3000, 257], groups=[4, 2], offsets=True, weights=True)
    simt = lambda name, **kw: c.append(make_case(name, "simt", seed=len(c), **kw))
    simt("simt_p64", P=64, G=3, rows=[1000, 77, 8], groups=[2, 0, 1])
    simt("simt_p256_nodes", P=256, G=2, rows=[3, 40, 3, 40, 500, 3, 40], groups=[0, 1, 0, 1, 0, 1, 1],
         nodes=[0, 1, 0, 1, 2, 1, 0], n_nodes=3, offsets=True, weights=True)
    simt("simt_p504_both", P=504, rows=[700, 1300], G=2, groups=[1, 0], offsets=True, weights=True)
    gen = lambda name, **kw: c.append(make_case(name, "generic", seed=len(c), **kw))
    gen("generic_bf16_p37_strided", P=37, G=2, rows=[300, 41, 900], groups=[1, 0, 1], nodes=[1, 0, 1], n_nodes=2,
        ld=40, misalign=True, offsets=True, weights=True)
    gen("generic_fp32_p100", P=100, rows=[1500, 3], storage="fp32")
    gen("generic_fp32_p700_both", P=700, G=2, rows=[800, 33, 400], groups=[0, 1, 0], storage="fp32", offsets=True,
        weights=True)
    c.append(make_case("custom_gaussian", "custom", P=48, G=2, rows=[1200, 801, 5], groups=[1, 0, 0], offsets=True,
                       weights=True, seed=len(c)))
    f8 = lambda name, **kw: c.append(make_case(name, "fp8", storage="fp8", seed=len(c), **kw))
    f8("fp8_p128_k1_weights", P=128, G=2, rows=[4000, 129, 1], groups=[1, 0, 1], weights=True)
    f8("fp8_p256_k3_nodes", P=256, K=3, G=3, rows=[2000, 385, 3000, 100], groups=[2, 0, 1, 2], nodes=[1, 0, 1, 2],
       n_nodes=3, offsets=True, weights=True)
    f8("fp8_p128_k2", P=128, K=2, rows=[5000, 31])
    return c


CASES = {c.name: c for c in _cases()}
NAMES = list(CASES)


# ------------------------------------------------------------------------------------------------ CPU tests
@pytest.mark.parametrize("name", NAMES)
def test_case_is_inside_its_exact_budget(name):
    cs = CASES[name]
    budget(cs)
    unit = 2.0 ** -cs.e
    wide = bf16_split(cs.beta * 2.0 ** -cs.ts, 1)[0] != cs.beta * 2.0 ** -cs.ts
    assert wide.any(), "no coefficient needs the mid bf16 term"
    assert (cs.beta != cs.beta[0]).any(axis=1)[1:].all(), "every chain has its own beta"
    if cs.kernel == "tc" and cs.family == "gaussian":
        wr = np.concatenate([_wr(cs, s)[2].ravel() for s in cs.segs])
        assert (bf16_split(wr * unit, 1)[0] != wr * unit).mean() > 0.05, "too few rows need the lo term of w r"
    if cs.kernel == "fp8":
        raw = [e4m3_digits(_wr(cs, s)[2][:, k], unit)[0] for s in cs.segs for k in range(cs.K)]
        assert any((r[1] != 0).any() for r in raw), "no row needs a second e4m3 term"
        bytes_ = np.concatenate([s.sc[: -(-s.X.shape[0] // 32)].ravel() for s in cs.segs])
        assert len(set(bytes_.tolist())) == 3, "block scales must differ between blocks"
    if any(s.w is not None for s in cs.segs):
        assert any(((s.w == 0) & s.nan).any() for s in cs.segs if s.w is not None), "no NaN row of weight 0"
    if cs.kernel == "tc":
        from pytensor_federated_b200.ops import native

        has = lambda field: any(getattr(s, field) is not None for s in cs.segs)
        row_data = (1 if has("o") else 0) | (2 if has("w") else 0)   # kGlmRowOffsets | kGlmRowWeights
        code = 4 if cs.disp else 2
        assert native.load().b200_glm_tc_stages(cs.P, cs.K, cs.G, code, row_data) >= 2, "a shape the runtime refuses"


def test_million_row_case_has_full_chunks_several_per_cta_and_a_small_tail():
    cs = CASES["tc_1m_rows"]
    table = chunk_table(cs.n_rows, SM_H100, *TC_CHUNKS)
    big = table[table[:, 0] == 0, 2]
    assert (big[:4] == 32).all() and len(table) > 3 * SM_H100     # full chunks first, several chunks per CTA
    assert big[-1] <= 4 and (big[-100:] <= 4).all()                 # the small tail


def test_budget_refuses_a_case_outside_it():
    cs = make_case("wide", "tc", P=64, rows=[4096], seed=1)
    cs.segs[0].y = cs.segs[0].y + (1 << 13)      # residuals of ~2^13 units over 2-tile chunks: the sums overflow
    with pytest.raises(AssertionError, match="over budget"):
        budget(cs)
    cs = make_case("fine", "tc", P=64, rows=[300], seed=2)
    seg = cs.segs[0]
    seg.y[0] += (1 << 20) + 1025 - _wr(cs, seg)[0][0, 0]   # r = 2^20 + 2^10 + 1: hi = 2^20, lo needs 11 bits
    with pytest.raises(AssertionError, match="hi \\+ lo"):
        budget(cs)


@pytest.mark.parametrize("name", NAMES)
def test_fp64_oracle_equals_the_integer_oracle(name):
    """``reference_partial`` in fp64 on CPU tensors reproduces the int64 gradients bit for bit (which also pins each
    family layout's ``fold`` of the kernel blocks on these inputs)."""
    cs = CASES[name]
    model = build_model(cs, torch.device("cpu"))
    inputs = cs.inputs()
    ref = model.reference_partial(inputs, dtype=torch.float64).reshape(cs.n_nodes, cs.K, -1)
    want = expected_raw(cs, oracle(cs), ref[..., 0])
    assert np.array_equal(ref[..., 1:], want[..., 1:])
    assert np.array_equal(model.per_node(ref.reshape(-1)), model.per_node(want.reshape(-1)))


SENSITIVITY = {"r_hi": "tc_k4_p72_weights_g7", "theta_hi": "tc_k2_p64_offsets_g7", "offset_bf16": "tc_k8_p200_both",
               "weight_shift": "fp8_p128_k1_weights", "drop_last": "simt_p256_nodes", "stale_tile": "tc_k9_p256",
               "swap_chains": "tc_k16_p256_both_g300", "wrong_group": "tc_k5_p128_both_g300",
               "wrong_node": "tc_nodes", "drop_q": "scale_k4_nodes"}


@pytest.mark.parametrize("bug", BUGS)
def test_each_data_path_bug_changes_an_expected_gradient_bit(bug):
    cs = CASES[SENSITIVITY[bug]]
    good, bad = oracle(cs), oracle(cs, bug)
    assert any(not np.array_equal(a, b) for a, b in zip(good, bad)), f"{bug} leaves every gradient of {cs.name} intact"


# ------------------------------------------------------------------------------------------------ GPU tests
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from pytensor_federated_b200.ops import native

    native.load()  # a GPU box without the native library is a failure, not a skip
    return torch.device("cuda:0")


SELECTED = {"tc": "tc", "fp8": "fp8", "simt": "simt", "custom": "generic-bf16"}


@pytest.mark.gpu
@pytest.mark.timeout(600)
@pytest.mark.parametrize("name", NAMES)
def test_kernel_gradients_are_exact(dev, name):
    from pytensor_federated_b200.parallel import FederatedEngine

    cs = CASES[name]
    sm_count = torch.cuda.get_device_properties(dev).multi_processor_count
    budget(cs, sm_count)
    model = build_model(cs, dev)
    inputs = cs.inputs()
    with FederatedEngine(model) as eng:
        raw = eng.evaluate_raw(inputs)
        folded = eng.evaluate(*inputs)
        again = eng.evaluate_raw(inputs)
    want_kernel = SELECTED.get(cs.kernel, "generic-" + cs.storage)
    assert model.selected_kernel == want_kernel
    got = raw.reshape(cs.n_nodes, cs.K, -1)
    want = expected_raw(cs, oracle(cs), got[..., 0])
    bad = np.argwhere(got[..., 1:] != want[..., 1:])
    assert bad.size == 0, (f"{len(bad)} gradient values differ; first (node, chain, value index): {bad[:8].tolist()}, "
                           f"got {got[..., 1:][tuple(bad[0])]!r}, want {want[..., 1:][tuple(bad[0])]!r}")
    assert np.array_equal(raw, again), "a second evaluation changed bits"
    for u, v in zip(folded, model.unpack_result(want.reshape(-1), model.call_context(inputs))):
        assert np.array_equal(u, v)
    # log-likelihood: each row's w ll rounds; the sums are fp32 runs of at most m terms, then double
    ll, mag = row_loglik(cs)
    if cs.kernel == "custom":
        assert np.array_equal(got[..., 0], ll)   # -d^2 / 2 and its sums are exact as well
        return
    m = LL_TERMS["generic" if cs.kernel == "generic" else cs.kernel]
    gamma = (m - 1) * 2.0 ** -24 / (1 - (m - 1) * 2.0 ** -24)
    bound = gamma * mag + 2.0 ** -40 * mag   # 2^-40: the double-precision stages
    if cs.n_nodes > 1 and cs.kernel in ("simt", "generic"):
        # per-node blocks of the CUDA-core kernels: every flush of a warp rounds to the 40.24 fixed point
        bound = bound + (8 * 2 * sm_count + len(cs.segs)) * 2.0 ** -25
    err = np.abs(got[..., 0] - ll)
    assert np.all(err <= bound), (err, bound)
