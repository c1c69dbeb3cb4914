"""Hessian-vector products of the logistic, Poisson and Gaussian families (``GlmShards(..., hvp=True)``).

CPU: the fp64 oracle (``reference_partial`` / ``per_node``) against ``torch.autograd.functional.hvp`` of an
independent fp64 log-likelihood; the layout's round trips; the collective engine and ``NodeFederation``; every
validation rule.  An exact Gaussian (and Poisson at theta = 0, where h = -exp(0) = -1 exactly) case family: integer
X, dyadic parameters and directions, integer weights.  :func:`budget` proves that u = v_intercept + x'v_beta and
s = w h u stay exact through the kernel's 3-way bf16 split of theta, the (hi, lo) bf16 split of the residual column
and every fp32 accumulation window of the chunk table, so the kernel's Hv must equal an int64 oracle bit for bit;
plausible bugs applied to that oracle each change an expected bit.

GPU: the exact cases bit for bit over every column bucket; the parameter columns of an HVP launch bit-identical to a
plain 2K-column launch; logistic and Poisson against the fp64 oracle within a rounding bound; the whole Hessian;
reproducibility and both result transports; two GPUs.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import pytest
import torch

from pytensor_federated_b200.federation import NodeFederation
from pytensor_federated_b200.models import CustomFamily, Fp8GlmShards, GlmShards
from pytensor_federated_b200.parallel import FederatedEngine

T = 6                  # grid of the exact cases: parameters, directions, y and offsets are integers times 2^-T
LIMIT = 1 << 21        # |partial sums| in grid units: 3 bits of margin under fp32's 24
TILE, MAX_CHUNK = 128, 32   # csrc/glm_tc.cu: rows per tile, tiles per chunk at most (one fp32 accumulation window)


# ------------------------------------------------------------------------------------------------ fp64 oracle
def _ll_rows(family, y, eta):
    if family == "logistic":
        return y * eta - torch.nn.functional.softplus(eta)
    if family == "poisson":
        return y * eta - torch.exp(eta)
    return -0.5 * (y - eta) ** 2 - 0.5 * math.log(2 * math.pi)


def _loglik(m, node=None):
    """``theta -> LL`` in fp64 written from the model's data (not from models/glm.py's oracle): masked rows are
    cleaned before use, so that no NaN reaches autograd."""
    G = m.n_groups
    segs = []
    for si, (X, y, g) in enumerate(zip(m.Xs, m.ys, m.groups)):
        if node is not None and m.node_ids[si] != node:
            continue
        w = m.weights[si].double() if m.weights[si] is not None else torch.ones(X.shape[0], dtype=torch.float64)
        keep = w != 0
        o = m.offsets[si].double() if m.offsets[si] is not None else torch.zeros_like(w)
        segs.append((X.double(), torch.where(keep, y.double(), 0.0), torch.where(keep, o, 0.0), w, g))

    def ll(theta):
        tot = theta.new_zeros(())
        for X, y, o, w, g in segs:
            eta = theta[g] + X @ theta[G:] + o
            tot = tot + (w * _ll_rows(m.family, y, eta)).sum()
        return tot

    return ll, segs


def _scale(m, theta, v, node=None):
    """S_j = sum_i w_i |h_i| (|u_i| + sum_l |x_il v_l|) |x~_ij| over the node's rows (float64 [G + P])."""
    G = m.n_groups
    _, segs = _loglik(m, node)
    S = torch.zeros(G + m.n_features, dtype=torch.float64)
    th, vv = torch.as_tensor(theta, dtype=torch.float64), torch.as_tensor(v, dtype=torch.float64)
    for X, y, o, w, g in segs:
        eta = th[g] + X @ th[G:] + o
        h = {"logistic": torch.sigmoid(eta) * torch.sigmoid(-eta), "poisson": torch.exp(eta),
             "gaussian": torch.ones_like(eta)}[m.family]
        u = vv[g] + X @ vv[G:]
        a = w * h * (u.abs() + X.abs() @ vv[G:].abs())
        S[g] += a.sum()
        S[G:] += X.abs().T @ a
    return S.numpy()


def _random_model(family, G, K, *, rows=True, n_nodes=1, P=16, seed=0):
    rng = np.random.default_rng(seed)
    Xs, ys, offs, ws, groups, nodes = [], [], [], [], [], []
    for s in range(max(3, G)):
        n = 60 + 17 * s
        X = torch.from_numpy(rng.normal(size=(n, P)).astype(np.float32))
        eta = X.double().numpy() @ (rng.normal(size=P) * 0.2)
        y = {"logistic": (rng.uniform(size=n) < 0.5) * 1.0, "poisson": rng.poisson(np.exp(0.3 * eta)) * 1.0,
             "gaussian": eta + rng.normal(size=n)}[family]
        o = rng.normal(size=n) * 0.3 if rows and s % 2 == 0 else None
        w = rng.integers(0, 3, size=n).astype(np.float64) if rows and s != 1 else None
        if w is not None:
            y[w == 0] = np.nan
            if o is not None:
                o[w == 0] = np.nan
        Xs.append(X)
        ys.append(torch.from_numpy(y.astype(np.float32)))
        offs.append(None if o is None else torch.from_numpy(o.astype(np.float32)))
        ws.append(None if w is None else torch.from_numpy(w.astype(np.float32)))
        groups.append(s % G)
        nodes.append(s % n_nodes)
    kw = dict(node_ids=nodes, n_nodes=n_nodes) if n_nodes > 1 else {}
    return GlmShards(Xs, ys, groups=groups, n_groups=G, family=family, n_chains=K, hvp=True, offsets=offs,
                     weights=ws, **kw)


def _inputs(m, rng, scale=0.2):
    K, G, P = m.n_chains, m.n_groups, m.n_features
    th = rng.normal(size=(K, G + P)) * scale
    v = rng.normal(size=(K, G + P))
    return th, v, m.inputs_from_theta(np.concatenate([th, v], axis=1).astype(np.float32) if K > 1 else
                                      np.concatenate([th, v], axis=1)[0].astype(np.float32))


# ------------------------------------------------------------------------------------------------ CPU: oracle
@pytest.mark.parametrize("family", ["logistic", "poisson", "gaussian"])
@pytest.mark.parametrize("G", [1, 3])
@pytest.mark.parametrize("K,n_nodes", [(1, 1), (3, 1), (2, 2)])
def test_oracle_matches_autograd_hvp(family, G, K, n_nodes):
    m = _random_model(family, G, K, n_nodes=n_nodes, seed=G * 10 + K)
    rng = np.random.default_rng(5)
    _, _, inputs = _inputs(m, rng)
    per = m.per_node(m.reference_partial(inputs, dtype=torch.float64))   # [n_nodes, K, 1 + 2 (G + P)]
    D = G + m.n_features
    flat = [np.asarray(x, dtype=np.float64).reshape(K, -1) for x in inputs]
    for node in range(n_nodes):
        ll, _ = _loglik(m, node if n_nodes > 1 else None)
        for k in range(K):
            th = torch.from_numpy(np.concatenate([flat[0][k], flat[1][k]]))
            v = torch.from_numpy(np.concatenate([flat[2][k], flat[3][k]]))
            lp, hv = torch.autograd.functional.hvp(ll, th, v)
            g = torch.autograd.functional.jacobian(ll, th)
            S = _scale(m, th, v, node if n_nodes > 1 else None)
            got = per[node, k]
            assert abs(got[0] - float(lp)) <= 1e-12 * max(1.0, abs(float(lp)))
            assert np.all(np.abs(got[1 : 1 + D] - g.numpy()) <= 1e-12 * (np.abs(got[1 : 1 + D]) + S + 1))
            assert np.all(np.abs(got[1 + D :] - hv.numpy()) <= 1e-12 * S), (node, k)


def test_unbatched_and_batched_calls_agree():
    m1 = _random_model("logistic", 3, 1, seed=2)
    m2 = _random_model("logistic", 3, 2, seed=2)
    rng = np.random.default_rng(0)
    th, v, _ = _inputs(m2, rng)
    one = m1.unpack_result(m1.reference_partial(m1.inputs_from_theta(np.concatenate([th[1], v[1]])), dtype=torch.float64))
    both = m2.unpack_result(m2.reference_partial(m2.inputs_from_theta(np.concatenate([th, v], 1)), dtype=torch.float64))
    assert [a.shape for a in one] == [(), (3,), (16,), (3,), (16,)]
    assert [a.shape for a in both] == [(2,), (2, 3), (2, 16), (2, 3), (2, 16)]
    for a, b in zip(one, both):
        np.testing.assert_allclose(a, b[1], rtol=1e-12, atol=1e-12)


def test_layout_round_trips():
    m = _random_model("poisson", 3, 4, seed=1)
    rng = np.random.default_rng(1)
    _, _, inputs = _inputs(m, rng)
    words = np.zeros(m.n_theta_words, dtype=np.uint32)
    m.pack_theta(inputs, words)
    again = np.zeros_like(words)
    m.pack_theta(m.inputs_from_words(words), again)
    assert np.array_equal(words, again)
    # column 2k holds (intercept, beta) of pair k, column 2k + 1 its direction
    th = words.view(np.float32).reshape(8, 3 + 16)
    assert np.array_equal(th[2, :3], np.asarray(inputs[0], np.float32)[1])
    assert np.array_equal(th[3, 3:], np.asarray(inputs[3], np.float32)[1])
    assert [x.shape for x in m.inputs_from_theta(np.zeros((4, m.n_params)))] == [(4, 3), (4, 16), (4, 3), (4, 16)]
    assert [x.shape for x in m.inputs_from_theta(np.zeros(m.n_params))] == [(3,), (16,), (3,), (16,)]
    row = np.arange(4 * (1 + m.n_params), dtype=np.float64).reshape(4, -1)
    gr = m.gradients_from_row(row, [None] * 4)
    assert [g.shape for g in gr] == [(4, 3), (4, 16), (4, 3), (4, 16)]
    assert gr[2][0, 0] == row[0, 1 + 19]


def test_collective_engine_and_node_federation_on_cpu():
    m = _random_model("logistic", 3, 2, n_nodes=2, seed=3)
    rng = np.random.default_rng(3)
    _, _, inputs = _inputs(m, rng)
    want = m.unpack_result(m.reference_partial(inputs))
    eng = FederatedEngine(m, backend="collective")
    got = eng.evaluate(*inputs)
    for a, b in zip(got, want):
        np.testing.assert_array_equal(a, b)
    fed = NodeFederation(eng)
    one = [np.asarray(x)[1] for x in inputs]
    res = fed.evaluate_nodes({0: one, 1: one})
    per = m.per_node(m.reference_partial([np.stack([x, x]) for x in one]))
    for node in (0, 1):
        lp, grads = res[node]
        assert float(lp) == per[node, 0, 0]
        assert np.array_equal(np.concatenate([g.reshape(-1) for g in grads]), per[node, 0, 1:])
    lp, grads = fed.evaluate_node(1, *one)
    assert len(grads) == 4
    assert len(fed.compute_func(0)(*one)) == 5
    for build in (fed.node_ops, fed.all_nodes_op, fed.all_nodes_func, lambda: fed.logp_grad_func(0)):
        with pytest.raises(ValueError, match="Hessian-vector products"):
            build()


def test_validation():
    X, y = [torch.zeros(8, 16, dtype=torch.bfloat16)], [torch.zeros(8)]
    for fam in ("multinomial", "gaussian_scale", "ordinal", CustomFamily("ll = 0.f; r = 0.f;")):
        with pytest.raises(ValueError, match="hvp=True is for family"):
            GlmShards(X, y, family=fam, hvp=True, n_classes=3 if fam in ("multinomial", "ordinal") else None)
    for kernel in ("simt", "generic", "fp8"):
        with pytest.raises(ValueError, match="tensor-core kernel only"):
            GlmShards(X, y, kernel=kernel, hvp=True)
    with pytest.raises(ValueError, match="fp8"):
        Fp8GlmShards([torch.zeros(8, 128, dtype=torch.float8_e4m3fn)], [torch.full((4, 4), 127, dtype=torch.uint8)],
                     y, hvp=True)
    with pytest.raises(ValueError, match=r"n_chains in \[1, 8\]"):
        GlmShards(X, y, n_chains=9, hvp=True)
    with pytest.raises(ValueError, match="tensor-core kernel only"):
        GlmShards([torch.zeros(8, 12, dtype=torch.bfloat16)], y, hvp=True).use_tensor_cores()
    with pytest.raises(ValueError, match="tensor-core kernel only"):
        GlmShards([torch.zeros(8, 16)], y, hvp=True).use_tensor_cores()   # fp32 X


def test_too_few_stages_refused_at_attach():
    from pytensor_federated_b200.ops import native

    lib = native.load()
    m = GlmShards([torch.zeros(8, 384, dtype=torch.bfloat16)], [torch.zeros(8)], n_chains=8, hvp=True)
    with pytest.raises(ValueError, match="fewer than two pipeline stages"):
        m.attach(lib, None)   # raises before the engine is touched
    assert lib.b200_glm_tc_stages(384, 8, 1, 16, 3) >= 2   # 4 pairs with offsets and weights fit


# ------------------------------------------------------------------------------------------------ exact cases
@dataclass
class Seg:
    X: np.ndarray              # int64 [n, P]
    y: np.ndarray              # int64 [n] grid units (0 where NaN)
    o: Optional[np.ndarray]    # int64 [n] grid units or None
    w: Optional[np.ndarray]    # int64 [n] or None
    nan: np.ndarray            # bool [n]: weight-0 rows with NaN y and offset
    group: int
    node: int


@dataclass
class Case:
    name: str
    family: str                # "gaussian", or "poisson" at theta = 0 without offsets (h = -1 exactly)
    P: int
    K: int
    G: int
    n_nodes: int
    segs: List[Seg]
    th: np.ndarray             # int64 [K, G + P] grid units
    v: np.ndarray              # int64 [K, G + P] grid units


def make_case(name, *, P, K, G=1, lens=(300,), n_nodes=1, rows="both", family="gaussian", seed=0, xmax=2, vmax=4):
    rng = np.random.default_rng(seed)
    segs = []
    for s, n in enumerate(lens):
        X = rng.integers(-xmax, xmax + 1, size=(n, P))
        X[rng.uniform(size=(n, P)) < 0.3] = 0
        w = rng.integers(0, 4, size=n) if rows in ("both", "weights") and s % 3 != 1 else None
        o = rng.integers(-64, 65, size=n) if rows in ("both", "offsets") and family == "gaussian" and s % 2 == 0 else None
        y = rng.integers(0, 9, size=n) if family == "poisson" else rng.integers(-200, 201, size=n)
        nan = (w == 0) & (rng.uniform(size=n) < 0.5) if w is not None else np.zeros(n, bool)
        y[nan] = 0
        if o is not None:
            o[nan] = 0
        segs.append(Seg(X, y, o, w, nan, (s * 7) % G, s % n_nodes))
    th = rng.integers(-4, 5, size=(K, G + P)) if family == "gaussian" else np.zeros((K, G + P), np.int64)
    v = rng.integers(-vmax, vmax + 1, size=(K, G + P))
    return Case(name, family, P, K, G, n_nodes, segs, th, v)


def oracle(case: Case, bug: Optional[str] = None) -> np.ndarray:
    """Expected kernel blocks ``[n_nodes, 2K, G + P]`` (the gradients of column 2k and the Hv of column 2k + 1, LL
    left out) in grid units 2^-T: int64 arithmetic, except for the bug ``h_from_v`` (Poisson: h = -exp(u))."""
    K, G, P = case.K, case.G, case.P
    th, v = (case.v, case.th) if bug == "swap" else (case.th, case.v)
    out = np.zeros((case.n_nodes, 2 * K, G + P), dtype=object if bug == "h_from_v" else np.int64)
    for sg in case.segs:
        w = sg.w if sg.w is not None and bug != "no_weight" else np.ones(len(sg.y), np.int64)
        wr = sg.w if sg.w is not None else np.ones(len(sg.y), np.int64)
        o = sg.o if sg.o is not None else np.zeros(len(sg.y), np.int64)
        for k in range(K):
            eta = th[k, sg.group] + sg.X @ th[k, G:] + o   # grid units
            vg = (sg.group + 1) % G if bug == "wrong_group" else sg.group
            u = v[k, vg] + sg.X @ v[k, G:] + (o if bug == "offset_in_u" else 0)
            if case.family == "gaussian":
                r = wr * (sg.y - eta)
            else:   # poisson at eta = 0: r = y - 1, in grid units
                r = wr * (sg.y - (1 << T))
            if bug == "h_from_v":
                s = np.array([-float(wi) * math.exp(ui * 2.0 ** -T) * ui for wi, ui in zip(w, u)], dtype=object)
            else:
                s = -w * u
            blk = out[sg.node]
            blk[2 * k, sg.group] += r.sum()
            blk[2 * k, G:] += sg.X.T @ r
            blk[2 * k + 1, sg.group] += s.sum()
            blk[2 * k + 1, G:] += sg.X.T @ s
    return out


def _bf16_exact(a: np.ndarray) -> bool:
    """Whether every value (integers < 2^24) is the sum of its bf16 (hi, lo) split, as the kernel forms it."""
    f = torch.from_numpy(a.astype(np.float32))
    hi = f.to(torch.bfloat16).float()
    lo = (f - hi).to(torch.bfloat16).float()
    return bool(torch.all(hi.double() + lo.double() == f.double()))


def budget(case: Case) -> None:
    """Asserts that every value the kernel forms for this case is exact (see the module docstring)."""
    K, G = case.K, case.G
    for sg in case.segs:
        n = len(sg.y)
        w = sg.w if sg.w is not None else np.ones(n, np.int64)
        o = sg.o if sg.o is not None else np.zeros(n, np.int64)
        absX = np.abs(sg.X)
        for k in range(K):
            for vec in (case.th[k], case.v[k]):
                assert np.all(np.abs(vec) < 1 << 8)   # 8 significant bits: the bf16 hi term alone
                assert np.all(absX @ np.abs(vec[G:]) + abs(vec[sg.group]) + np.abs(o) < LIMIT)   # eta / u in fp32
            eta = case.th[k, sg.group] + sg.X @ case.th[k, G:] + o
            u = case.v[k, sg.group] + sg.X @ case.v[k, G:]
            r = w * (sg.y - eta) if case.family == "gaussian" else w * (sg.y - (1 << T))
            s = -w * u
            for col in (r, s):
                assert np.all(np.abs(col) < LIMIT)
                assert _bf16_exact(col), case.name            # the (hi, lo) residual split
                # every fp32 accumulation window: a chunk of at most MAX_CHUNK tiles, gradient and intercept sums
                a = np.abs(col)[:, None] * np.concatenate([np.ones((n, 1), np.int64), absX], axis=1)
                pad = (-n) % TILE
                tiles = np.concatenate([a, np.zeros((pad, a.shape[1]), np.int64)]).reshape(-1, TILE, a.shape[1]).sum(1)
                c = np.concatenate([np.zeros((1, a.shape[1]), np.int64), np.cumsum(tiles, 0)])
                win = c[min(MAX_CHUNK, len(tiles)):] - c[: len(c) - min(MAX_CHUNK, len(tiles))]
                assert win.max() < LIMIT, (case.name, int(win.max()))
    # the int64 results fit fp64 exactly
    assert np.abs(oracle(case)).max() < 1 << 52


def build_model(case: Case, device, *, hvp=True):
    """The case as a GlmShards on ``device`` (X bf16, y, offsets, weights float32 with NaN on the masked rows)."""
    u = 2.0 ** -T
    Xs, ys, offs, ws = [], [], [], []
    for sg in case.segs:
        Xs.append(torch.from_numpy(sg.X.astype(np.float32)).to(torch.bfloat16).to(device))
        y = sg.y.astype(np.float64) * u
        y[sg.nan] = np.nan
        ys.append(torch.from_numpy(y.astype(np.float32)).to(device))
        if sg.o is not None:
            o = sg.o.astype(np.float64) * u
            o[sg.nan] = np.nan
            offs.append(torch.from_numpy(o.astype(np.float32)).to(device))
        else:
            offs.append(None)
        ws.append(torch.from_numpy(sg.w.astype(np.float32)).to(device) if sg.w is not None else None)
    kw = dict(node_ids=[sg.node for sg in case.segs], n_nodes=case.n_nodes) if case.n_nodes > 1 else {}
    return GlmShards(Xs, ys, groups=[sg.group for sg in case.segs], n_groups=case.G, family=case.family,
                     n_chains=case.K, hvp=hvp, offsets=offs if any(o is not None for o in offs) else None,
                     weights=ws if any(w is not None for w in ws) else None, **kw)


def case_inputs(case: Case, m):
    rows = np.concatenate([case.th, case.v], axis=1).astype(np.float64) * 2.0 ** -T
    return m.inputs_from_theta(rows.astype(np.float32) if case.K > 1 else rows[0].astype(np.float32))


def kernel_blocks(case: Case, vals: np.ndarray) -> np.ndarray:
    """The raw result as ``[n_nodes, 2K, G + P]`` in grid units (LL left out)."""
    raw = np.asarray(vals).reshape(case.n_nodes, 2 * case.K, 1 + case.G + case.P)
    return raw[..., 1:] * 2.0 ** T


CPU_CASES = [
    make_case("plain", P=16, K=1, rows="none"),
    make_case("rows_g3", P=32, K=3, G=3, lens=(200, 129, 75, 300)),
    make_case("nodes", P=24, K=2, G=2, lens=(130, 40, 257, 3), n_nodes=3),
    make_case("poisson", P=16, K=2, G=2, lens=(200, 150), family="poisson"),
]


@pytest.mark.parametrize("case", CPU_CASES, ids=lambda c: c.name)
def test_exact_oracle_and_budget(case):
    budget(case)
    m = build_model(case, torch.device("cpu"))
    got = kernel_blocks(case, m.reference_partial(case_inputs(case, m), dtype=torch.float64))
    want = oracle(case)
    assert np.array_equal(got, want.astype(np.float64))


@pytest.mark.parametrize("bug", ["offset_in_u", "h_from_v", "no_weight", "swap", "wrong_group"])
def test_exact_oracle_catches_bugs(bug):
    cases = {"h_from_v": CPU_CASES[3], "wrong_group": CPU_CASES[1]}
    case = cases.get(bug, CPU_CASES[1])
    good, bad = oracle(case).astype(np.float64), oracle(case, bug).astype(np.float64)
    assert not np.array_equal(good[:, 1::2], bad[:, 1::2]) or not np.array_equal(good, bad)


# ------------------------------------------------------------------------------------------------ GPU
GPU_CASES = [
    make_case("k1_p8", P=8, K=1, rows="none", lens=(1000,)),
    make_case("k2_p128_rows", P=128, K=2, G=3, lens=(700, 129, 4000)),
    make_case("k3_p256_offsets", P=256, K=3, G=2, lens=(3000, 255), rows="offsets"),
    make_case("k4_p384_weights", P=384, K=4, lens=(2000,), rows="weights", vmax=2),
    make_case("k5_p64_g300", P=64, K=5, G=300, lens=tuple(50 + 3 * i for i in range(300))),
    make_case("k8_p200_nodes", P=200, K=8, G=4, lens=(1000, 77, 513, 2049, 9), n_nodes=3),
    make_case("k2_p96_poisson", P=96, K=2, G=2, lens=(5000, 33), family="poisson"),
    make_case("k4_p128_1.1M", P=128, K=4, lens=(1_100_000,), rows="both", xmax=1, vmax=2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=lambda c: c.name)
def test_exact_hvp_on_gpu(case):
    budget(case)
    m = build_model(case, torch.device("cuda:0"))
    inputs = case_inputs(case, m)
    with FederatedEngine(m) as eng:
        first = eng.evaluate_raw(inputs)
        again = eng.evaluate_raw(inputs)
    assert np.array_equal(first, again)
    got = kernel_blocks(case, first)
    want = oracle(case).astype(np.float64)
    assert np.array_equal(got[:, 1::2], want[:, 1::2]), case.name       # Hv
    assert np.array_equal(got[:, 0::2], want[:, 0::2]), case.name       # the gradients of the parameter columns
    raw = np.asarray(first).reshape(case.n_nodes, 2 * case.K, -1)
    assert np.all(raw[:, 1::2, 0] == 0.0)                                # the direction columns' LL


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["logistic", "poisson", "gaussian"])
@pytest.mark.parametrize("rows", [False, True])
def test_parameter_columns_match_a_plain_launch(family, rows):
    dev = torch.device("cuda:0")
    K = 3
    m = _random_model(family, 2, K, rows=rows, P=64, seed=7)
    m.Xs = [X.to(torch.bfloat16).to(dev) for X in m.Xs]
    hv = GlmShards(m.Xs, [y.to(dev) for y in m.ys], groups=m.groups, n_groups=2, family=family, n_chains=K, hvp=True,
                   offsets=[None if o is None else o.to(dev) for o in m.offsets] if rows else None,
                   weights=[None if w is None else w.to(dev) for w in m.weights] if rows else None)
    plain = GlmShards(hv.Xs, hv.ys, groups=m.groups, n_groups=2, family=family, n_chains=2 * K, offsets=hv.offsets
                      if rows else None, weights=hv.weights if rows else None)
    rng = np.random.default_rng(1)
    th, v, inputs = _inputs(hv, rng)
    rows2 = np.stack([th, v], axis=1).reshape(2 * K, -1).astype(np.float32)   # row 2k = theta_k, 2k + 1 = v_k
    with FederatedEngine(hv) as e1:
        a = np.asarray(e1.evaluate_raw(inputs)).reshape(2 * K, -1)
    with FederatedEngine(plain) as e2:
        b = np.asarray(e2.evaluate_raw(plain.inputs_from_theta(rows2))).reshape(2 * K, -1)
    assert np.array_equal(a[0::2], b[0::2])


def _fp64_check(m, inputs, got_per, c):
    """The largest error of the kernel's Hv (``got_per``, as ``per_node`` gives it) against the fp64 oracle of the CPU
    model ``m``, in units of the bound ``c 2^-16 S_j``."""
    want = m.per_node(m.reference_partial(inputs, dtype=torch.float64))
    D = m.n_groups + m.n_features
    flat = [np.asarray(x, dtype=np.float64).reshape(m.n_chains, -1) for x in inputs]
    worst = 0.0
    for k in range(m.n_chains):
        S = _scale(m, np.concatenate([flat[0][k], flat[1][k]]), np.concatenate([flat[2][k], flat[3][k]]))
        err = np.abs(got_per[0, k, 1 + D :] - want[0, k, 1 + D :])
        worst = max(worst, float(np.max(err / (c * 2.0 ** -16 * S))))
    return worst


# Rounding bound of the kernel's Hv against the exact value, in units of 2^-16 S_j:
# - MMA #2 accumulates s x in fp32 over a chunk of at most 32 tiles x 128 rows = 256 wgmma K steps; each step rounds
#   the running sum once inside the tensor core and once on accumulation: 2 x 256 x 2^-24 = 2^-15 = 2 units;
# - s is carried as its bf16 (hi, lo) split: relative error 2^-17 = 0.5 units;
# - u: the 3-way split of v is exact to 2^-24 and eta's fp32 wgmma chain over P <= 384 features (24 K steps, 3 terms)
#   adds 2 x 24 x 2^-24 of sum_l |x_l v_l| (< 0.01 units); h from expf and one division, a few ulps (< 0.01 units);
# - the intercept sums: 64 fp32 additions per thread and chunk (< 0.01 units); chunks combine in double-double.
# 2.53 units in all, so c = 3.
C_HV = 3.0


@pytest.mark.gpu
@pytest.mark.parametrize("family,scale", [("logistic", 1.0), ("logistic", 8.0), ("poisson", 0.35)])
def test_hvp_against_fp64(family, scale):
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(3)
    P, K, n = 128, 4, 50_000
    X = torch.from_numpy(rng.normal(size=(n, P)).astype(np.float32)).to(torch.bfloat16)
    eta = X.float().numpy() @ (rng.normal(size=P) * scale / math.sqrt(P))
    if family == "logistic":   # |eta| up to about 30 at scale 8
        y = (rng.uniform(size=n) < 1 / (1 + np.exp(-eta))) * 1.0
    else:                      # mu up to about e^10
        eta = np.clip(eta * 10 / max(1e-9, np.abs(eta).max()), -10, 10)
        y = rng.poisson(np.exp(np.minimum(eta, 9.5))) * 1.0
    w = rng.integers(0, 3, size=n).astype(np.float32)
    m = GlmShards([X.to(dev)], [torch.from_numpy(y.astype(np.float32)).to(dev)], family=family, n_chains=K, hvp=True,
                  weights=[torch.from_numpy(w).to(dev)])
    th = np.zeros((K, 1 + P))
    beta = np.linalg.lstsq(X.float().numpy()[:2000], eta[:2000], rcond=None)[0] if family == "poisson" else \
        rng.normal(size=P) * scale / math.sqrt(P)
    th[:, 1:] = beta
    v = rng.normal(size=(K, 1 + P))
    inputs = m.inputs_from_theta(np.concatenate([th, v], 1).astype(np.float32))
    with FederatedEngine(m) as eng:
        got = m.per_node(eng.evaluate_raw(inputs))
    cpu = GlmShards([X], [torch.from_numpy(y.astype(np.float32))], family=family, n_chains=K, hvp=True,
                    weights=[torch.from_numpy(w)])
    assert _fp64_check(cpu, inputs, got, C_HV) <= 1.0


@pytest.mark.gpu
def test_whole_hessian_and_finite_differences():
    from pytensor_federated_b200.sampling import glm_batch_fn, glm_hessian, glm_hvp_fn

    dev = torch.device("cuda:0")
    rng = np.random.default_rng(4)
    P, n = 64, 40_000
    X = torch.from_numpy(rng.normal(size=(n, P)).astype(np.float32)).to(torch.bfloat16).to(dev)
    y = (torch.rand(n, device=dev) < 0.4).float()
    theta = rng.normal(size=1 + P) * 0.1
    with FederatedEngine(GlmShards([X], [y], n_chains=8, hvp=True)) as eng, \
            FederatedEngine(GlmShards([X], [y], n_chains=2)) as geng:
        D = 1 + P
        _, _, cols = glm_hvp_fn(eng)(np.broadcast_to(theta, (D, D)), np.eye(D))
        _, _, H = glm_hessian(eng, theta)
        cpu = GlmShards([X.cpu()], [y.cpu()], n_chains=1, hvp=True)
        S = np.stack([_scale(cpu, theta, np.eye(D)[j]) for j in range(D)])   # S[j] bounds column j
        assert np.all(np.abs(cols.T - cols) <= C_HV * 2.0 ** -16 * (S + S.T))
        assert np.allclose(H, H.T)
        v = rng.normal(size=D)
        epsv = 1e-3
        _, g = glm_batch_fn(geng, 1)(np.stack([theta + epsv * v, theta - epsv * v]))
        fd = (g[0] - g[1]) / (2 * epsv)
        np.testing.assert_allclose(fd, H @ v, rtol=2e-2, atol=2e-2 * np.abs(H @ v).max())


@pytest.mark.gpu
def test_reproducible_over_grids_and_transports():
    dev = torch.device("cuda:0")
    big = make_case("flag_results", P=256, K=8, lens=(6000, 3000), rows="both")      # 16 x 258 values > 2048
    small = make_case("tagged", P=16, K=1, lens=(500,), rows="none")                  # 2 x 18 values
    for case in (big, small):
        budget(case)
        m = build_model(case, dev)
        inputs = case_inputs(case, m)
        outs = []
        for grid in (None, 7):
            with FederatedEngine(m, grid=grid) as eng:
                outs.append(eng.evaluate_raw(inputs))
                outs.append(eng.evaluate_raw(inputs))
        for o in outs[1:]:
            assert np.array_equal(o, outs[0])
        want = oracle(case).astype(np.float64)
        assert np.array_equal(kernel_blocks(case, outs[0]), want)
    assert build_model(big, dev).n_vals > 2048 and build_model(small, dev).n_vals <= 2048


TWO_GPU_CASE = make_case("two_gpus", P=64, K=2, G=2, lens=(3000, 2000), n_nodes=2)


def _two_gpu_model(rank, world, dev):
    sg = TWO_GPU_CASE.segs[rank]
    one = Case("rank", TWO_GPU_CASE.family, TWO_GPU_CASE.P, TWO_GPU_CASE.K, TWO_GPU_CASE.G, 1, [sg],
               TWO_GPU_CASE.th, TWO_GPU_CASE.v)
    m = build_model(one, dev)
    return GlmShards(m.Xs, m.ys, groups=m.groups, n_groups=m.n_groups, family=m.family, n_chains=m.n_chains, hvp=True,
                     offsets=m.offsets if any(o is not None for o in m.offsets) else None,
                     weights=m.weights if any(w is not None for w in m.weights) else None,
                     node_ids=[rank], n_nodes=world)


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_match_one():
    from pytensor_federated_b200.federation import launch_federation

    case = TWO_GPU_CASE
    m1 = build_model(case, torch.device("cuda:0"))
    with FederatedEngine(m1) as eng:
        one = eng.evaluate_raw(case_inputs(case, m1))
    with launch_federation(_two_gpu_model, 2) as eng:
        two = eng.evaluate_raw(case_inputs(case, eng.model))
    assert np.array_equal(one, two)
    assert np.array_equal(kernel_blocks(case, one), oracle(case).astype(np.float64))
