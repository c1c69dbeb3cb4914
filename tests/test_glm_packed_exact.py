"""The packed (12-bit) design matrix of the bf16 tensor-core GLM kernel, bit for bit against the integer oracle.

The kernel reads X packed by default where the tile pads to 256 features and a launch has at most 4 kernel columns:
the flagship shape.  Here X is a small integer matrix on the exact grid of ``test_glm_exact.py`` whose high bytes
(sign and top 7 exponent bits) take 16 values: 0x00, +-1, +-2..7, +-8..31, +-32..127, +-128..511, +-512..2047, -0.0
and +2048..8191 in a segment's table, and -2048..-8191, the rarest, as the exceptions its tiles' footers patch.  The
exceptions sit where a pipelined decoder goes wrong: a tile with a full footer of 63, the first and last rows of a
tile, the first and last feature of a panel and of X, a segment's tail tile; adjacent segments have different
tables.  The large values sit on rows of small residual and features of small coefficient, so every sum stays on the
exact grid (:func:`budget`).

CPU: every case is inside its exact budget; ``reference_partial`` in fp64 equals the integer oracle; the packing and
chunk properties each case is for are read back from ``pack_x12`` and the runtime's chunk table; each plausible
fault of the packed path, emulated with the kernel's own tile decoder, changes an expected gradient bit.
GPU: each case packed and with ``B200FED_NO_PACKED_X=1``, each against the oracle with ``np.array_equal``.
"""
from __future__ import annotations

import functools
from dataclasses import replace
from typing import Dict, List, Tuple

import numpy as np
import pytest
import torch

from test_glm_exact import (LL_TERMS, SM_H100, TC_CHUNKS, TILE, Case, Seg, _wr, budget, build_model, chunk_table,
                            expected_raw, imatmul, oracle, row_loglik)
from test_glm_packed import _decode

from pytensor_federated_b200.models.glm import X12_MAX_EXCEPTIONS, pack_x12

FAMILY_CODE = {"gaussian": 2, "gaussian_scale": 4, "gaussian_location_scale": 13}
N_SMALL = 100   # resolution of the small values' distribution


def _bf16_ints(rng, lo: int, hi: int, size) -> np.ndarray:
    """Integers in [lo, hi) (lo a power of two) with at most 8 significant bits: exact in bf16."""
    m = rng.integers(lo, hi, size)
    shift = np.maximum(np.floor(np.log2(m)).astype(np.int64) + 1 - 8, 0)
    return (m >> shift) << shift


# the table's rare buckets (value ranges; one high byte each) and the exceptions' bucket
SPRINKLE = [(1, 8, 32), (-1, 8, 32), (1, 32, 128), (-1, 32, 128), (1, 128, 512), (-1, 128, 512), (1, 512, 2048),
            (-1, 512, 2048), (1, 2048, 8192)]


def make_packed_case(name, *, family="gaussian", P, rows, K=1, G=1, groups=None, nodes=None, n_nodes=1,
                     offsets=(), weights=(), dominant=None, exceptions=None, full=None, seed=0) -> Case:
    """A case on the exact grid whose packed X has controlled statistics.

    ``offsets`` / ``weights``: the segments that carry them.  ``dominant[s]``: ``"one"`` (mostly +-1) or ``"two"``
    (mostly +-2..3), alternating by default, so adjacent segments' tables differ in order.  ``exceptions[s]``: (row,
    feature) positions of exception values; ``full[s]``: tiles that get 63 of them (a full footer), on 63 distinct rows
    (0 and 127 among them) and features.  Every other position keeps a small value, apart from the rare buckets,
    sprinkled on random rows, more often than the exceptions so that they keep their table entries.  Rows that carry a
    large value get a small residual and weight 1; their features have coefficients +-1 and no per-chain change."""
    rng = np.random.default_rng(seed)
    scale = family != "gaussian"
    xs, ts, d_max, big, dbeta, dic = (0, 3, 12, 0.0, 1, 2) if scale else (0, 6, 40, 0.2, 2, 4)
    exc_hi = 4096 if scale else 8192   # the scale column's w (d^2 - 1) is larger than the mean's w d on quiet rows
    groups = list(groups) if groups is not None else [0] * len(rows)
    nodes = list(nodes) if nodes is not None else [0] * len(rows)
    dominant = dominant or ["one" if si % 2 == 0 else "two" for si in range(len(rows))]
    exceptions, full = exceptions or {}, full or {}
    edges = {f for f in (0, 63, 64, 127, 128, 191, 192, 255, P - 1) if f < P}
    free = np.array([f for f in range(P) if f not in edges])
    small_f = rng.choice(free, max(2, P // 4), replace=False)      # wide coefficients and per-chain changes
    big_f = np.setdiff1d(np.arange(P), small_f)                    # where large values may go
    beta0 = rng.choice([-1, 1], P)
    beta0[small_f] = rng.integers(-8, 9, small_f.size)
    wide = small_f[: max(1, P // 8)]
    beta0[wide] = rng.choice([-1, 1], wide.size) * (2 * rng.integers(129, 256, wide.size) + 1)   # 9 significant bits
    beta = np.repeat(beta0[None], K, axis=0)
    ic0 = rng.integers(-200, 201, G)
    ic = np.repeat(ic0[None], K, axis=0)
    for k in range(1, K):
        f = rng.choice(small_f, min(small_f.size, 4), replace=False)
        beta[k, f] += rng.choice([-1, 1], f.size) * rng.integers(1, dbeta + 1, f.size)
        ic[k] += rng.integers(-dic, dic + 1, G)
    luts = {   # 100 draws: 0 x 20, then the dominant magnitude's values most often
        "one": np.array([0] * 20 + [1] * 25 + [-1] * 25 + [2] * 8 + [-2] * 8 + [3] * 7 + [-3] * 7, np.int16),
        "two": np.array([0] * 20 + [1] * 8 + [-1] * 8 + [2] * 17 + [-2] * 17 + [3] * 15 + [-3] * 15, np.int16)}
    segs = []
    for si, (n, g, nd) in enumerate(zip(rows, groups, nodes)):
        X = np.empty((n, P), np.int16)
        lut = luts[dominant[si]]
        for r0 in range(0, n, 1 << 16):
            r1 = min(n, r0 + (1 << 16))
            X[r0:r1] = lut[rng.integers(0, N_SMALL, (r1 - r0, P), dtype=np.uint8)]
        exc = [tuple(p) for p in exceptions.get(si, [])]
        for t in full.get(si, []):
            r = np.concatenate([[0, 127], rng.choice(np.arange(1, 127), 61, replace=False)])
            f = rng.choice(big_f, 63, replace=False)
            exc += [(t * TILE + int(a), int(b)) for a, b in zip(r, f)]
        assert len(set(exc)) == len(exc)
        # the rare buckets: each more often than the exceptions, on rows and features the exceptions leave alone
        count = len(exc) + 3
        taken = set(exc)
        quiet = {r for r, _ in exc}
        for sign, lo, hi in SPRINKLE + [(0, 0, 0)]:
            placed = 0
            while placed < count:
                pos = (int(rng.integers(0, n)), int(rng.choice(big_f)))
                if pos in taken:
                    continue
                taken.add(pos)
                quiet.add(pos[0])
                X[pos] = 0 if sign == 0 else sign * _bf16_ints(rng, lo, hi, 1)[0]
                placed += 1
        nz = np.array(sorted(p for p in taken if X[p] == 0 and p not in exc), np.int64).reshape(-1, 2)
        for p in exc:
            assert p[1] in big_f, f"{name}: exception at feature {p[1]}, whose coefficient is wide or changes per chain"
            X[p] = -_bf16_ints(rng, 2048, exc_hi, 1)[0]
        quiet = np.array(sorted(quiet), np.int64)
        o = rng.integers(-600, 601, n) if si in offsets else None
        w = rng.choice(4, n, p=[0.15, 0.35, 0.25, 0.25]) if si in weights else None
        if w is not None:
            w[quiet] = 1
        nan = (w == 0) & (rng.random(n) < 0.5) if w is not None else np.zeros(n, bool)
        d = rng.integers(-d_max, d_max + 1, n)
        wide_r = rng.random(n) < big
        d[wide_r] = rng.choice([-1, 1], int(wide_r.sum())) * rng.integers(260, 701, int(wide_r.sum()))
        d[quiet] = rng.integers(-2, 3, quiet.size)
        eta0 = imatmul(X, beta0[:, None])[:, 0] + ic0[g] + (o if o is not None else 0)
        y = np.where(nan, 0, eta0 + d)
        segs.append(Seg(X, y, o, w, nan, g, nd, nz=nz))
    return Case(name, "tc", family, P, K, G, n_nodes, xs, ts, segs, ic, beta)


# ------------------------------------------------------------------------------------------------ the matrix
FORCED = {"forced_k8_p256", "forced_k16_p128", "forced_pairs_p64"}   # packed although it is not the default there


def _cases() -> List[Case]:
    c = []
    add = lambda name, **kw: c.append(make_packed_case(name, seed=len(c), **kw))
    n0 = 1_100_003   # 8594 tiles, the last of 99 rows
    add("flagship_long", P=256, rows=[n0, 129, 4133], G=3, groups=[2, 0, 1], offsets={0, 2}, weights={0, 1, 2},
        full={0: [4000]}, exceptions={0: [(0, 0), (127, 255), (5 * 128 + 3, 64), (200 * 128 + 50, 191),
                                          (300 * 128 + 60, 192), (n0 - 99, 0), (n0 - 1, 255)],
                                      1: [(128, 128)], 2: [(4132, 63)]})
    add("k4_both_p200", P=200, K=4, G=7, rows=[5000, 127, 4097, 1], groups=[5, 0, 3, 6], offsets={0, 2},
        weights={0, 1, 2}, full={0: [10]},
        exceptions={0: [(0, 199), (127, 0), (1000, 63), (1001, 64), (2000, 127), (2001, 128), (4999, 199)],
                    1: [(0, 0), (126, 199)], 2: [(128, 0), (255, 199), (4096, 199)], 3: [(0, 199)]})
    rng = np.random.default_rng(7)
    rows = rng.integers(1, 401, 3000).tolist()
    rows[:4] = [1, 128, 256, 400]
    exc = {si: [(int(rng.integers(0, n)), int(f))] for si, (n, f) in enumerate(zip(rows, rng.choice([0, 63, 64, 135], 3000)))
           if si % 2 == 0}
    add("many_segments_p136", P=136, K=3, G=300, rows=rows, groups=rng.integers(0, 300, 3000).tolist(),
        nodes=rng.integers(0, 3, 3000).tolist(), n_nodes=3, weights=set(range(0, 3000, 2)), exceptions=exc)
    add("scale_k2_p256", family="gaussian_scale", P=256, K=2, G=2, rows=[3000, 257, 129], groups=[1, 0, 1],
        offsets={0, 2}, weights={0, 1, 2}, full={0: [3]}, exceptions={0: [(0, 0), (2999, 255)], 1: [(256, 255)]})
    add("location_scale_k1_p256", family="gaussian_location_scale", P=256, rows=[2000, 300, 129], offsets={0},
        exceptions={0: [(0, 0), (1999, 255)], 1: [(128, 64)], 2: [(128, 255)]})
    add("location_scale_k2_p200", family="gaussian_location_scale", P=200, K=2, G=3, rows=[1500, 129, 640],
        groups=[2, 0, 1], offsets={1}, weights={0, 1, 2}, exceptions={0: [(0, 199), (127, 0)], 1: [(128, 199)],
                                                                      2: [(639, 0)]})
    add("forced_k8_p256", P=256, K=8, rows=[3000, 1, 700, 129], exceptions={0: [(0, 0), (2999, 255)], 1: [(0, 255)],
                                                                           2: [(699, 64)], 3: [(128, 0)]})
    add("forced_k16_p128", P=128, K=13, G=2, rows=[2000, 300, 129], groups=[1, 0, 1], offsets={0, 2},
        weights={0, 1, 2}, exceptions={0: [(0, 0), (1999, 127), (700, 63), (701, 64)], 2: [(128, 127)]})
    add("forced_pairs_p64", family="gaussian_location_scale", P=64, K=8, rows=[1000, 129, 300],
        exceptions={0: [(0, 0), (999, 63)], 1: [(128, 63)], 2: [(127, 0)]})
    return c


CASES: Dict[str, Case] = {c.name: c for c in _cases()}
NAMES = list(CASES)


@functools.lru_cache(maxsize=None)
def _oracle(name: str):
    return oracle(CASES[name])


def _bf16(s: Seg) -> torch.Tensor:
    X = torch.from_numpy(s.X).to(torch.float32).to(torch.bfloat16)
    if s.nz is not None and len(s.nz):
        X[torch.from_numpy(s.nz[:, 0]), torch.from_numpy(s.nz[:, 1])] = -0.0
    return X


@functools.lru_cache(maxsize=None)
def _packs(name: str):
    """``pack_x12`` of every segment of the case on CPU tensors: (blocks, footers, table) as numpy."""
    cs = CASES[name]
    out = []
    for s in cs.segs:
        p = pack_x12(_bf16(s))
        assert p is not None, f"{name}: a tile has more than {X12_MAX_EXCEPTIONS} exceptions"
        out.append((p[0].numpy(), p[1].numpy(), tuple(p[2])))
    return out


def _exception_positions(foot: np.ndarray):
    """(tile, panel, row, feature in the panel) of every exception in the footers ``[tiles, 64]``."""
    t = np.repeat(np.arange(foot.shape[0]), foot[:, 0])
    rank = np.concatenate([np.arange(c) for c in foot[:, 0]]) if foot.shape[0] else np.zeros(0, int)
    pos = foot[t, 1 + rank].astype(np.int64) >> 8
    return t, pos >> 13, (pos >> 6) & 127, pos & 63


# ------------------------------------------------------------------------------------------------ CPU tests
@pytest.mark.parametrize("name", NAMES)
def test_case_is_inside_its_exact_budget(name):
    budget(CASES[name])


@pytest.mark.parametrize("name", NAMES)
def test_fp64_oracle_equals_the_integer_oracle(name):
    """``reference_partial`` in fp64 on CPU tensors reproduces the int64 gradients bit for bit, and ``per_node`` folds
    both alike (for the pairs: the ``_Pair.fold`` interleaving of the two columns' blocks)."""
    cs = CASES[name]
    model = build_model(cs, torch.device("cpu"))
    inputs = cs.inputs()
    ref = model.reference_partial(inputs, dtype=torch.float64, chunk_rows=1 << 16).reshape(cs.n_nodes, cs.columns, -1)
    want = expected_raw(cs, _oracle(name), ref[..., 0])
    assert np.array_equal(ref[..., 1:], want[..., 1:])
    if cs.pair:
        assert np.array_equal(ref[:, 1::2, 0], np.zeros((cs.n_nodes, cs.K)))
    assert np.array_equal(model.per_node(ref.reshape(-1)), model.per_node(want.reshape(-1)))


@pytest.mark.parametrize("name", NAMES)
def test_packed_form_has_the_exceptions_the_case_places(name):
    """The footers hold exactly the values below -2047 (the rarest high byte, 0xC5), every other value is in its
    segment's table, and the decoder's image of each tile with exceptions is X's."""
    cs = CASES[name]
    PP = (cs.P + 127) // 128 * 128
    for s, (blocks, foot, table) in zip(cs.segs, _packs(name)):
        t, pnl, r, f = _exception_positions(foot)
        got = sorted(zip((t * TILE + r).tolist(), (pnl * 64 + f).tolist()))
        assert got == sorted(map(tuple, np.argwhere(s.X <= -2048).tolist()))
        entries = b"".join(w.to_bytes(4, "little") for w in table)
        assert 0xC5 not in entries[:15] and entries[0] == 0
        for tile in np.flatnonzero(foot[:, 0])[:3].tolist() + [(s.X.shape[0] - 1) // TILE]:
            rc, _ = _decode(blocks[tile], foot[tile], table, PP // 64)
            assert rc == foot[tile, 0]
            assert np.array_equal(_decoded_tile(blocks[tile], foot[tile], table, PP)[: s.X.shape[0] - tile * TILE,
                                  : cs.P], s.X[tile * TILE : (tile + 1) * TILE])


def test_the_cases_put_exceptions_at_every_edge():
    found = set()
    for name, cs in CASES.items():
        for s, (_, foot, _) in zip(cs.segs, _packs(name)):
            t, pnl, r, f = _exception_positions(foot)
            feat = pnl * 64 + f
            n_panels = (cs.P + 127) // 128 * 2
            found |= {"full footer"} if (foot[:, 0] == 63).any() else set()
            found |= {"empty tile"} if (foot[: (s.X.shape[0] + 127) // 128, 0] == 0).any() else set()
            found |= {"panel 0"} if (pnl == 0).any() else set()
            found |= {"last panel"} if ((pnl == n_panels - 1) & (feat < cs.P)).any() else set()
            found |= {"last real panel"} if (pnl == (cs.P - 1) // 64).any() else set()
            found |= {"row 0"} if (r == 0).any() else set()
            found |= {"row 127"} if (r == 127).any() else set()
            found |= {"panel feature 0"} if ((f == 0) & (pnl > 0)).any() else set()
            found |= {"panel feature 63"} if ((f == 63) & (pnl > 0)).any() else set()
            found |= {"feature 0"} if (feat == 0).any() else set()
            if cs.P % 64:
                found |= {"feature P - 1"} if (feat == cs.P - 1).any() else set()
            if s.X.shape[0] % TILE:
                found |= {"tail tile"} if (t == (s.X.shape[0] - 1) // TILE).any() else set()
    want = {"full footer", "empty tile", "panel 0", "last panel", "last real panel", "row 0", "row 127",
            "panel feature 0", "panel feature 63", "feature 0", "feature P - 1", "tail tile"}
    assert want <= found, want - found
    # the flagship: the full footer and an exception in the tail tile of its long segment
    foot = _packs("flagship_long")[0][1]
    n0 = CASES["flagship_long"].segs[0].X.shape[0]
    assert (foot[:, 0] == 63).any() and foot[(n0 - 1) // TILE, 0] > 0


@pytest.mark.parametrize("name", NAMES)
def test_adjacent_segments_have_different_tables(name):
    tabs = [p[2] for p in _packs(name)]
    pairs = [a != b for a, b in zip(tabs, tabs[1:])]
    assert all(pairs) if len(tabs) < 10 else np.mean(pairs) > 0.9, pairs


def test_chunk_tables():
    """The flagship's long segment runs in full 32-tile chunks, several per CTA; the many-segment case gives every
    CTA at least 20 chunks, more than its chunk ring's 16 slots."""
    cs = CASES["flagship_long"]
    table = chunk_table(cs.n_rows, SM_H100, *TC_CHUNKS)
    long = table[table[:, 0] == 0, 2]
    assert (long[:4] == TC_CHUNKS[1]).all() and len(long) > 2 * SM_H100
    cs = CASES["many_segments_p136"]
    assert len(chunk_table(cs.n_rows, SM_H100, *TC_CHUNKS)) >= 20 * SM_H100


@pytest.mark.parametrize("name", sorted(FORCED))
def test_forced_shapes_run_packed(name):
    """A forced case must not fall back to the bf16 read: its shape gets at least two compressed slots."""
    from pytensor_federated_b200.ops import native

    cs = CASES[name]
    model = build_model(cs, torch.device("cpu"))
    row_data = (1 if any(s.o is not None for s in cs.segs) else 0) | (2 if any(s.w is not None for s in cs.segs) else 0)
    lib = native.load()
    assert lib.b200_glm_tc_packed_slots(cs.P, cs.columns, cs.G, FAMILY_CODE[cs.family], row_data,
                                        model.n_theta_words) >= 2
    assert not model._packing_pays(row_data)   # not the default: the test forces it


@pytest.mark.parametrize("name", sorted(set(NAMES) - FORCED))
def test_default_cases_pack_by_default(name):
    cs = CASES[name]
    assert build_model(cs, torch.device("cpu"))._packing_pays(3)


# ------------------------------------------------------------------------------------------------ faults
def _untma(img: np.ndarray, PP: int) -> np.ndarray:
    """The inverse of ``test_glm_packed._tma_image``: the decoder's 128B-swizzled tile -> uint16 [128, PP]."""
    panels = PP // 64
    sw = img.view(np.uint16).reshape(panels, 128, 8, 8)
    rows = np.arange(128)[:, None]
    sub = sw[:, rows, np.arange(8)[None, :] ^ (rows % 8)]   # [panel, row, chunk, element]
    return sub.transpose(1, 0, 2, 3).reshape(128, PP)


def _decoded_tile(blocks, foot, table, PP: int) -> np.ndarray:
    """One tile through the kernel's decoder, as X_int [128, PP].  Values off the grid (an unpatched exception decodes
    with high byte 0x00 to a tiny number) round to it: the fault still moves X by about the exception's value."""
    rc, img = _decode(blocks, foot, table, PP // 64)
    assert rc >= 0
    bits = _untma(img, PP).astype(np.int16)
    v = torch.from_numpy(bits).view(torch.bfloat16).double().numpy()
    return np.rint(v).astype(np.int64)


def _with_x(cs: Case, si: int, tiles, foot_of=lambda t, foot: foot[t], table=None) -> Case:
    """The case with the given tiles of segment si decoded from its packed form, with footer ``foot_of(t, footers)``
    and the given table (default: the segment's own)."""
    blocks, foot, tab = _packs(cs.name)[si]
    s = cs.segs[si]
    n, PP = s.X.shape[0], (cs.P + 127) // 128 * 128
    X = s.X.astype(np.int64)
    for t in tiles:
        rows = min(TILE, n - t * TILE)
        X[t * TILE : t * TILE + rows] = _decoded_tile(blocks[t], foot_of(t, foot), table or tab, PP)[:rows, : cs.P]
    segs = list(cs.segs)
    segs[si] = replace(s, X=X)
    return replace(cs, segs=segs)


def _tiles(s: Seg) -> range:
    return range((s.X.shape[0] + TILE - 1) // TILE)


def _fault(fault: str) -> Tuple[Case, tuple]:
    """(case, expected gradients) with one fault of the packed path emulated."""
    cs = CASES[FAULTS[fault]]
    if fault in ("wrong_table", "no_exceptions", "exception_cap", "stale_footer"):
        si = 2 if fault == "wrong_table" else 0
        s, (_, foot, _) = cs.segs[si], _packs(cs.name)[si]
        if fault == "wrong_table":
            bad = _with_x(cs, si, _tiles(s), table=_packs(cs.name)[si - 1][2])
        elif fault == "no_exceptions":
            bad = _with_x(cs, si, _tiles(s), lambda t, f: np.zeros_like(f[t]))
        elif fault == "exception_cap":
            full = int(np.flatnonzero(foot[:, 0] == 63)[0])
            bad = _with_x(cs, si, [full], lambda t, f: np.concatenate([[62], f[t, 1:]]).astype(f.dtype))
        else:   # tile t patched with the footer of tile t - 2, the same parity of the footer double buffer
            t = int(np.flatnonzero(foot[2:, 0] != foot[:-2, 0])[0]) + 2
            bad = _with_x(cs, si, [t], lambda t, f: f[t - 2])
        return bad, oracle(bad)
    if fault == "row_slot_shift":   # tile 1 of segment 0 takes tile 0's y, offset and weight
        s = cs.segs[0]
        mv = lambda v: None if v is None else np.concatenate([v[:TILE], v[:TILE], v[2 * TILE :]])
        bad = replace(cs, segs=[replace(s, y=mv(s.y), o=mv(s.o), w=mv(s.w), nan=mv(s.nan))] + cs.segs[1:])
        return bad, oracle(bad)
    gi, gb, q = (a.copy() for a in oracle(cs))
    if fault == "pair_swap":
        return cs, (gi[:, _swap(cs)], gb[:, _swap(cs)], q)
    assert fault == "offset_on_scale"   # s = offset on column 2k + 1: z = d e^-s, in fp64 (no longer on the grid)
    gi, gb = gi.astype(np.float64), gb.astype(np.float64)
    for s in cs.segs:
        if s.o is None:
            continue
        d, ww, _ = _wr(cs, s)
        f = np.exp(-2.0 * s.o * 2.0 ** -cs.e)[:, None]
        rm, rs = ww[:, None] * d * f, ww[:, None] * (d * d * f - (1 << 2 * cs.e))
        exact = ww[:, None] * d, ww[:, None] * (d * d - (1 << 2 * cs.e))
        for col, r, r0 in ((slice(0, None, 2), rm, exact[0]), (slice(1, None, 2), rs, exact[1])):
            gi[s.node, col, s.group] += (r - r0).sum(0)
            gb[s.node, col] += (r - r0).T @ s.X.astype(np.float64)
    return cs, (gi, gb, q)


def _swap(cs: Case) -> np.ndarray:
    return np.arange(cs.columns).reshape(-1, 2)[:, ::-1].reshape(-1)

FAULTS = {"wrong_table": "k4_both_p200", "no_exceptions": "k4_both_p200", "exception_cap": "k4_both_p200",
          "stale_footer": "k4_both_p200", "row_slot_shift": "k4_both_p200",
          "offset_on_scale": "location_scale_k2_p200", "pair_swap": "forced_pairs_p64"}


@pytest.mark.parametrize("fault", list(FAULTS))
def test_each_packed_path_fault_changes_an_expected_gradient_bit(fault):
    good = _oracle(FAULTS[fault])
    _, bad = _fault(fault)
    assert any(not np.array_equal(a, b) for a, b in zip(good, bad)), f"{fault} leaves every gradient intact"


# ------------------------------------------------------------------------------------------------ GPU tests
@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from pytensor_federated_b200.ops import native

    native.load()  # a GPU box without the native library is a failure, not a skip
    return torch.device("cuda:0")


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("packed", [True, False], ids=["packed", "bf16"])
@pytest.mark.parametrize("name", NAMES)
def test_kernel_gradients_are_exact(dev, name, packed, monkeypatch):
    from pytensor_federated_b200.parallel import FederatedEngine

    if packed:
        monkeypatch.delenv("B200FED_NO_PACKED_X", raising=False)
    else:
        monkeypatch.setenv("B200FED_NO_PACKED_X", "1")
    cs = CASES[name]
    sm_count = torch.cuda.get_device_properties(dev).multi_processor_count
    budget(cs, sm_count)
    model = build_model(cs, dev)
    if name in FORCED:
        model._packing_pays = lambda row_data: True
    inputs = cs.inputs()
    with FederatedEngine(model) as eng:
        assert model.packed_x is packed and model.selected_kernel == "tc"
        raw = eng.evaluate_raw(inputs)
        folded = eng.evaluate(*inputs)
        again = eng.evaluate_raw(inputs)
    got = np.asarray(raw, dtype=np.float64).reshape(cs.n_nodes, cs.columns, -1)
    want = expected_raw(cs, _oracle(name), got[..., 0])
    bad = np.argwhere(got[..., 1:] != want[..., 1:])
    assert bad.size == 0, (f"{len(bad)} gradient values differ; first (node, chain, value index): {bad[:8].tolist()}, "
                           f"got {got[..., 1:][tuple(bad[0])]!r}, want {want[..., 1:][tuple(bad[0])]!r}")
    assert np.array_equal(raw, again), "a second evaluation changed bits"
    for u, v in zip(folded, model.unpack_result(want.reshape(-1), model.call_context(inputs))):
        assert np.array_equal(u, v)
    ll, mag = row_loglik(cs)
    m = LL_TERMS["tc"]
    gamma = (m - 1) * 2.0 ** -24 / (1 - (m - 1) * 2.0 ** -24)
    bound = gamma * mag + 2.0 ** -40 * mag   # 2^-40: the double-precision stages
    got_ll = got[:, 0::2, 0] if cs.pair else got[..., 0]
    if cs.pair:
        assert np.array_equal(got[:, 1::2, 0], np.zeros((cs.n_nodes, cs.K))), "the scale column's LL is not 0"
    err = np.abs(got_ll - ll)
    assert np.all(err <= bound), (err, bound)
