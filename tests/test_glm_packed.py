"""The packed (12-bit) design matrix of the bf16 tensor-core GLM kernel.

CPU: the packer (``pack_x12``) and the kernel's tile decoder (``b200_glm_x12_decode_tile``, the same
``__host__ __device__`` code the decoder warps run) reproduce TMA's 128B-swizzled image of the bf16 tile byte for
byte: over every one of the 65 536 bf16 bit patterns, on N(0, 1) data, on tail tiles and the empty padding tile, and at
P in {8, 72, 136, 256}.  A tile with more exceptions than its footer holds is refused.
GPU: every epilogue in every K bucket, with and without row data, computes the same bits packed and unpacked.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from pytensor_federated_b200.models.glm import X12_BLOCK, X12_FOOT, pack_x12, x12_tiles


def _lib():
    from pytensor_federated_b200.ops import native

    return native.load()


def _tma_image(bits: np.ndarray) -> np.ndarray:
    """What TMA writes for one tile: bits is uint16 [128, PP]; per 64-feature panel, row r's 16-byte chunk j lands at
    r * 128 + (j ^ (r % 8)) * 16."""
    panels = bits.shape[1] // 64
    out = np.zeros((panels, 128, 8, 8), dtype=np.uint16)
    sub = bits.reshape(128, panels, 8, 8).transpose(1, 0, 2, 3)              # [panel, row, chunk, element]
    rows = np.arange(128)[:, None]
    out[:, rows, np.arange(8)[None, :] ^ (rows % 8)] = sub
    return out.reshape(-1).view(np.uint8)


def _decode(blocks: np.ndarray, foot: np.ndarray, table, panels: int) -> tuple:
    out = np.zeros(panels * 16384, dtype=np.uint8)
    tab = (C.c_uint * 4)(*table)
    blocks = np.ascontiguousarray(blocks)
    foot = np.ascontiguousarray(foot, dtype=np.int32)
    rc = _lib().b200_glm_x12_decode_tile(blocks.ctypes.data, foot.ctypes.data, C.cast(tab, C.c_void_p), panels,
                                         out.ctypes.data)
    return rc, out


def _check_packed(X: torch.Tensor) -> int:
    """Packs X and decodes every tile, against TMA's image of the zero-padded matrix; returns the exceptions seen."""
    n, P = X.shape
    PP = (P + 127) // 128 * 128
    packed = pack_x12(X)
    assert packed is not None
    blocks, foot, table = packed
    tiles = x12_tiles(n)
    assert blocks.shape == (tiles, PP // 64, X12_BLOCK) and foot.shape == (tiles, X12_FOOT // 4)
    padded = np.zeros((tiles * 128, PP), dtype=np.uint16)
    padded[:n, :P] = X.view(torch.int16).numpy().view(np.uint16)
    seen = 0
    for t in range(tiles):
        rc, got = _decode(blocks[t].numpy(), foot[t].numpy(), table, PP // 64)
        assert rc >= 0
        seen += rc
        want = _tma_image(padded[128 * t : 128 * (t + 1)])
        assert np.array_equal(got, want), f"tile {t} of {tiles}: {np.count_nonzero(got != want)} bytes differ"
    return seen


@pytest.mark.parametrize("P", [8, 72, 136, 256])
def test_normal_data_tail_tiles_and_padding(P):
    g = torch.Generator().manual_seed(P)
    n = 3 * 128 + 37   # 4 tiles with a tail, padded to 4; and 5 tiles -> 6 (an empty padding tile)
    for rows in (n, n + 128):
        _check_packed(torch.randn(rows, P, generator=g).to(torch.bfloat16))


def test_every_bf16_bit_pattern():
    """Each high byte in turn is in the table (14 at a time, each with all 256 low bytes) and, for a few low bytes,
    an exception of a tile whose table does not hold it."""
    patterns = np.arange(65536, dtype=np.uint32)
    high = patterns >> 8
    covered = np.zeros(65536, dtype=bool)
    others = [h for h in range(1, 256)]
    for g0 in range(0, len(others), 14):
        group = others[g0 : g0 + 14]
        vals = patterns[np.isin(high, [0] + group)]                             # 256 (15 high bytes) values
        # the remaining high bytes as exceptions, at most 63 per 128 x 256 tile: a few low bytes of each
        rest = [h for h in range(256) if h not in group and h != 0]
        exc = np.array([(h << 8) | ((h * 37 + g0) & 0xFF) for h in rest], dtype=np.uint32)
        tiles = []
        body = np.resize(vals, (128 * 256,))
        for k in range(0, len(exc), 60):
            t = body.copy()
            t[np.linspace(0, t.size - 1, len(exc[k : k + 60])).astype(int)] = exc[k : k + 60]
            tiles.append(t)
        # the group's values outnumber everything else, so the table holds the group
        X = torch.from_numpy(np.concatenate(tiles).astype(np.uint16).view(np.int16)).view(torch.bfloat16)
        X = X.reshape(-1, 256)
        seen = _check_packed(X)
        assert seen > 0
        covered[np.concatenate(tiles)] = True
        covered[vals] = True
    assert covered.all()


def test_special_values_decode():
    specials = [0x0000, 0x8000, 0x7F80, 0xFF80, 0x7FC0, 0x7F81, 0xFFFF, 0x0001, 0x807F, 0x3F80, 0xBF80]
    bits = np.resize(np.array(specials, dtype=np.uint16), 130 * 72)
    X = torch.from_numpy(bits.view(np.int16)).view(torch.bfloat16).reshape(130, 72)
    _check_packed(X)


def test_tile_with_too_many_exceptions_is_refused():
    X = torch.zeros(256, 64, dtype=torch.bfloat16)
    X[:, 0] = 1.0   # the one frequent high byte
    flat = X.view(torch.int16).reshape(-1)
    rare = torch.tensor([(h << 8) | 1 for h in range(16, 16 + 64 + 15)], dtype=torch.int32).to(torch.int16)
    flat[1 : 1 + rare.numel()] = rare   # 79 distinct rare high bytes in tile 0: at least 64 exceptions
    assert pack_x12(X) is None
    ok = torch.zeros(256, 64, dtype=torch.bfloat16)
    ok.view(torch.int16).reshape(-1)[1 : 1 + 63 + 14] = rare[: 63 + 14]
    assert pack_x12(ok) is not None


def test_decoder_refuses_a_bad_footer():
    blocks = np.zeros(4 * X12_BLOCK, dtype=np.uint8)
    foot = np.zeros(X12_FOOT // 4, dtype=np.int32)
    foot[0] = X12_FOOT // 4
    assert _decode(blocks, foot, (0, 0, 0, 0), 4)[0] == -1


def test_packed_layout_fits_the_flagship_shape():
    lib = _lib()
    assert lib.b200_glm_tc_packed_slots(256, 1, 1, 0, 0, 257) >= 4
    for K in (1, 4, 8, 16):
        for row_data in (0, 3):
            assert lib.b200_glm_tc_packed_slots(256, K, 1, 0, row_data, K * 257) >= 2
            assert lib.b200_glm_tc_packed_slots(128, K, 1, 0, row_data, K * 129) >= 2
    assert lib.b200_glm_tc_packed_slots(384, 1, 1, 0, 0, 385) < 2   # P = 384 keeps reading X itself


@pytest.mark.parametrize("P", [72, 128, 256])
def test_theta_larger_than_the_two_packed_stages_refuses_packing(P):
    """fp32 theta is staged in the bf16 stages; the packed layout has two, so a theta of more than 2 stages' bytes
    (many groups and chains) must keep the shape on the bf16 read, whose 3 or 4 stages hold it."""
    lib = _lib()
    stage_bytes = (P + 127) // 128 * 2 * 16384
    fits = 2 * stage_bytes // 4
    assert lib.b200_glm_tc_packed_slots(P, 16, 1, 0, 0, fits) >= 2
    assert lib.b200_glm_tc_packed_slots(P, 16, 1, 0, 0, fits + 1) < 2
    G = 1000   # 16 chains x (G + P) floats: more than 64 KB at P = 72 and 128
    if 16 * (G + P) > fits:
        assert lib.b200_glm_tc_packed_slots(P, 16, G, 0, 0, 16 * (G + P)) < 2
        assert lib.b200_glm_tc_stages(P, 16, G, 0, 0) >= 2   # the bf16 read still runs it


def test_packing_is_the_default_only_where_it_was_measured_faster():
    from pytensor_federated_b200.models import GlmShards

    def pays(P, K, **kw):
        return GlmShards([torch.zeros(128, P, dtype=torch.bfloat16)], [torch.zeros(128)], n_chains=K, **kw)._packing_pays(0)

    assert pays(256, 1) and pays(256, 4) and pays(136, 1) and pays(200, 2, family="multinomial", n_classes=2)
    assert not pays(128, 1) and not pays(72, 4) and not pays(256, 8) and not pays(256, 16)
    assert not pays(256, 2, family="multinomial", n_classes=3)   # 6 kernel columns: the K = 8 bucket
    assert not pays(256, 4, hvp=True)                           # 8 kernel columns


# ---------------------------------------------------------------------------------------------------------------- GPU
CASES = [  # (family, model kwargs, K): every epilogue, every K bucket
    ("logistic", {}, 1),
    ("logistic", {}, 4),
    ("poisson", {}, 8),
    ("gaussian", {}, 16),
    ("multinomial", {"n_classes": 3}, 2),
    ("gaussian_scale", {}, 4),
    ("ordinal", {"n_classes": 4}, 2),
    ("weibull", {}, 8),
    ("logistic", {"hvp": True}, 4),
]


def _inputs(model, K, rng):
    return [rng.normal(size=(K,) + tuple(s)).astype(np.float32) * 0.05 for s in model.input_shapes]


@pytest.mark.gpu
@pytest.mark.parametrize("rows_data", [False, True])
@pytest.mark.parametrize("P", [72, 256])
@pytest.mark.parametrize("family,kw,K", CASES)
def test_packed_launch_is_bitwise_the_unpacked_one(family, kw, K, P, rows_data, monkeypatch):
    from pytensor_federated_b200.parallel import FederatedEngine

    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(11)
    sizes = [3 * 128 + 5, 1000, 128]
    Xs = [torch.randn(n, P, generator=g, device=dev).to(torch.bfloat16) for n in sizes]
    if family == "multinomial" or family == "ordinal":
        ys = [torch.randint(0, kw["n_classes"], (n,), generator=g, device=dev).float() for n in sizes]
    elif family in ("poisson",):
        ys = [torch.randint(0, 5, (n,), generator=g, device=dev).float() for n in sizes]
    elif family == "weibull":
        ys = [torch.rand(n, generator=g, device=dev) + 0.5 for n in sizes]
    else:
        ys = [(torch.rand(n, generator=g, device=dev) < 0.5).float() for n in sizes]
    extra = {}
    if rows_data:
        extra["weights"] = [torch.rand(n, generator=g, device=dev) + 0.5 for n in sizes]
        if family != "multinomial":
            extra["offsets"] = [None, 0.1 * torch.randn(sizes[1], generator=g, device=dev), None]
    outs = {}
    for packed in (True, False):
        if packed:
            monkeypatch.delenv("B200FED_NO_PACKED_X", raising=False)
        else:
            monkeypatch.setenv("B200FED_NO_PACKED_X", "1")
        model = GlmShardsFactory(Xs, ys, family, K, kw, extra)
        # every shape the packed layout fits, also those where packing is not the default (it does not pay there)
        model._packing_pays = lambda row_data: True
        with FederatedEngine(model) as eng:
            assert model.packed_x is packed
            outs[packed] = np.asarray(eng.evaluate_raw(_inputs(model, K, np.random.default_rng(5))), dtype=np.float64)
    assert outs[True].tobytes() == outs[False].tobytes()


def GlmShardsFactory(Xs, ys, family, K, kw, extra):
    from pytensor_federated_b200.models import GlmShards

    return GlmShards(Xs, ys, family=family, n_chains=K, kernel="tc", **kw, **extra)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [72, 128])
def test_many_groups_and_chains_stay_correct(P, monkeypatch):
    """16 chains x 1000 groups: theta (72 KB and more) does not fit in the packed layout's two stages, so the launch
    reads X itself, and computes what the bf16 read computes."""
    from pytensor_federated_b200.models import GlmShards
    from pytensor_federated_b200.parallel import FederatedEngine

    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(3)
    G, K, n = 1000, 16, 300
    Xs = [torch.randn(n, P, generator=g, device=dev).to(torch.bfloat16) for _ in range(4)]
    ys = [(torch.rand(n, generator=g, device=dev) < 0.5).float() for _ in range(4)]
    rng = np.random.default_rng(1)
    inputs = [rng.normal(size=(K, G)).astype(np.float32) * 0.1, rng.normal(size=(K, P)).astype(np.float32) * 0.05]
    outs = {}
    for packed in (True, False):
        if packed:
            monkeypatch.delenv("B200FED_NO_PACKED_X", raising=False)
        else:
            monkeypatch.setenv("B200FED_NO_PACKED_X", "1")
        model = GlmShards(Xs, ys, groups=[0, 1, 998, 999], n_groups=G, n_chains=K, kernel="tc")
        with FederatedEngine(model) as eng:
            assert model.packed_x is False
            outs[packed] = np.asarray(eng.evaluate_raw(inputs), dtype=np.float64)
    assert outs[True].tobytes() == outs[False].tobytes()
    want = model.reference_partial(inputs, dtype=torch.float64)
    assert np.allclose(outs[True], want, rtol=1e-4, atol=1e-2)


@pytest.mark.gpu
def test_unpackable_matrix_falls_back():
    from pytensor_federated_b200.models import GlmShards
    from pytensor_federated_b200.parallel import FederatedEngine

    dev = torch.device("cuda:0")
    X = torch.zeros(256, 64, dtype=torch.bfloat16)
    X[:, 0] = 1.0
    X.view(torch.int16).reshape(-1)[1 : 1 + 79] = torch.tensor([(h << 8) | 1 for h in range(16, 95)],
                                                                dtype=torch.int32).to(torch.int16)
    model = GlmShards([X.to(dev)], [torch.ones(256, device=dev)], kernel="tc")
    for _ in range(2):   # the refusal is remembered, and a second engine attaches the model as the first did
        with FederatedEngine(model) as eng:
            assert model.packed_x is False
            got = np.asarray(eng.evaluate_raw([np.zeros(1, np.float32), np.zeros(64, np.float32)]))
            want = model.reference_partial([np.zeros(1, np.float32), np.zeros(64, np.float32)], dtype=torch.float64)
            assert np.allclose(got, want, rtol=1e-5, atol=1e-3)
