"""Numerics of the fused sm_90a kernels vs plain PyTorch references (needs an H100)."""
import numpy as np
import pytest
import torch

from pytensor_federated_b200.models import (
    CustomFamily,
    Fp8GlmShards,
    GlmShards,
    LinregShards,
    OdeShards,
    make_demo_data,
    synth_logistic_shard,
    synth_lv_shard,
)
from pytensor_federated_b200.parallel import FederatedEngine

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from pytensor_federated_b200.ops import native

    native.load()  # a GPU box without the native library is a failure, not a skip
    return torch.device("cuda:0")


def test_linreg_demo_model_matches_float64_oracle(dev):
    import scipy.stats

    x, y, sigma = make_demo_data()
    model = LinregShards([x], [y], [sigma], device=dev)
    with FederatedEngine(model) as eng:
        assert eng.backend == "fused"
        for a, b in [(0.4, 1.2), (1.5, 0.5), (-3.0, 2.0)]:
            logp, da, db = eng.evaluate(np.array(a), np.array(b))
            expected = scipy.stats.norm.logpdf(y, loc=a + b * x, scale=sigma).sum()
            np.testing.assert_allclose(logp, expected, rtol=1e-12)
            r = y - (a + b * x)
            np.testing.assert_allclose(da, r.sum() / sigma**2, rtol=1e-11, atol=1e-11)
            np.testing.assert_allclose(db, (r * x).sum() / sigma**2, rtol=1e-11, atol=1e-11)
        assert eng.kernel_launches == 3


def test_linreg_many_shards_large_and_float32(dev):
    rng = np.random.default_rng(0)
    sizes = [10, 1000, 70001, 333]
    xs = [rng.normal(size=n) for n in sizes]
    ys = [1.0 + 0.5 * x + rng.normal(scale=0.3, size=x.size) for x in xs]
    sig = [0.3, 0.5, 0.7, 1.1]
    a = np.array([0.9, 1.0, 1.1, 1.2])
    for dtype, rtol in ((torch.float64, 1e-11), (torch.float32, 1e-5)):
        model = LinregShards(xs, ys, sig, device=dev, dtype=dtype)
        with FederatedEngine(model) as eng:
            got = eng.evaluate(a, np.array(0.45))
            want = model.reference([a, np.array(0.45)])
            for g, w in zip(got, want):
                np.testing.assert_allclose(g, w, rtol=rtol, atol=1e-6)
            per = LinregShards.per_shard(eng.evaluate_raw([a, np.array(0.45)]))
            assert per.shape == (4, 3)


@pytest.mark.parametrize("family", ["logistic", "poisson", "gaussian"])
@pytest.mark.parametrize("P", [256, 64, 512])
def test_glm_simt_matches_reference(dev, family, P):
    torch.manual_seed(1)
    rows = [1000, 77, 4099, 8]
    Xs, ys = [], []
    for i, n in enumerate(rows):
        X, y, _ = synth_logistic_shard(n, P, seed=i, device=dev, beta_scale=0.05)
        Xs.append(X)
        ys.append(y)
    model = GlmShards(Xs, ys, groups=[0, 1, 0, 2], n_groups=3, family=family, kernel="simt")
    ic = np.array([0.3, -0.2, 0.1])
    beta = (np.random.default_rng(2).normal(size=P) * 0.03).astype(np.float32)
    with FederatedEngine(model) as eng:
        logp, d_ic, d_beta = eng.evaluate(ic, beta)
    w_logp, w_ic, w_beta = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(logp, w_logp, rtol=2e-5)
    np.testing.assert_allclose(d_ic, w_ic, rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(d_beta, w_beta, rtol=1e-4, atol=2e-3 * np.sqrt(sum(rows)))


def _glm_case(dev, rows, P, groups, n_groups, seed=0):
    Xs, ys = [], []
    for i, n in enumerate(rows):
        X, y, _ = synth_logistic_shard(n, P, seed=seed + i, device=dev, beta_scale=0.05)
        Xs.append(X)
        ys.append(y)
    return Xs, ys


@pytest.mark.parametrize("P", [256, 128, 384, 72, 200, 8])
@pytest.mark.parametrize("family", ["logistic", "gaussian"])
def test_glm_tensor_core_matches_reference(dev, family, P):
    rows = [128 * 37, 77, 4099, 128, 1]
    Xs, ys = _glm_case(dev, rows, P, None, 3)
    model = GlmShards(Xs, ys, groups=[0, 1, 0, 2, 1], n_groups=3, family=family, kernel="tc")
    ic = np.array([0.3, -0.2, 0.1])
    beta = (np.random.default_rng(2).normal(size=P) * 0.03).astype(np.float32)
    with FederatedEngine(model) as eng:
        logp, d_ic, d_beta = eng.evaluate(ic, beta)
        again = eng.evaluate(ic, beta)
    w_logp, w_ic, w_beta = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(logp, w_logp, rtol=2e-5)
    np.testing.assert_allclose(d_ic, w_ic, rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(d_beta, w_beta, rtol=1e-4, atol=2e-3 * np.sqrt(sum(rows)))
    for u, v in zip((logp, d_ic, d_beta), again):
        assert np.array_equal(u, v)


@pytest.mark.parametrize("K", [2, 3, 4, 8, 13, 16])
def test_glm_tensor_core_batches_chains(dev, K):
    rows = [128 * 50 + 5, 3000]
    Xs, ys = _glm_case(dev, rows, 256, None, 2, seed=9)
    model = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, n_chains=K, kernel="tc")
    rng = np.random.default_rng(4)
    ic = rng.normal(size=(K, 2)).astype(np.float32) * 0.2
    beta = rng.normal(size=(K, 256)).astype(np.float32) * 0.03
    with FederatedEngine(model) as eng:
        logp, d_ic, d_beta = eng.evaluate(ic, beta)
    assert logp.shape == (K,) and d_ic.shape == (K, 2) and d_beta.shape == (K, 256)
    w = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(logp, w[0], rtol=2e-5)
    np.testing.assert_allclose(d_ic, w[1], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(d_beta, w[2], rtol=1e-4, atol=0.2)


def test_glm_tensor_core_many_tiles_flushes_accumulator(dev):
    """> kFlush tiles per CTA so the register -> fp64 flush is exercised on every CTA."""
    X, y, _ = synth_logistic_shard(132 * 128 * 70 + 13, 256, seed=21, device=dev)
    model_tc = GlmShards([X], [y], kernel="tc")
    model_simt = GlmShards([X], [y], kernel="simt")
    beta = (np.random.default_rng(3).normal(size=256) * 0.02).astype(np.float32)
    with FederatedEngine(model_tc) as eng:
        a = eng.evaluate(np.array([0.1]), beta)
    with FederatedEngine(model_simt) as eng:
        b = eng.evaluate(np.array([0.1]), beta)
    np.testing.assert_allclose(a[0], b[0], rtol=1e-6)
    np.testing.assert_allclose(a[1], b[1], rtol=1e-4, atol=0.05)
    np.testing.assert_allclose(a[2], b[2], rtol=1e-4, atol=0.05)


@pytest.mark.parametrize("P", [256, 128])
def test_glm_fp8_block_scaled_matches_dequantised_reference(dev, P):
    """kind::mxf8f6f4.block_scale kernel vs fp64 maths on the dequantised matrix."""
    torch.manual_seed(3)
    rows = [128 * 40 + 7, 999, 128]
    Xs, ys = [], []
    for i, n in enumerate(rows):
        # heterogeneous row/feature magnitudes so that the block scales really differ
        X = torch.randn(n, P, device=dev) * torch.exp(torch.randn(P, device=dev)) * torch.exp(
            0.5 * torch.randn(n, 1, device=dev))
        Xs.append(X)
        ys.append((torch.rand(n, device=dev) < 0.4).float())
    model = Fp8GlmShards.from_dense(Xs, ys, groups=[0, 1, 2], n_groups=3)
    assert len({int(v) for s in model.scales for v in s.flatten().tolist()}) > 3
    ic = np.array([0.2, -0.3, 0.05])
    beta = (np.random.default_rng(5).normal(size=P) * 0.02).astype(np.float32)
    with FederatedEngine(model) as eng:
        logp, d_ic, d_beta = eng.evaluate(ic, beta)
        again = eng.evaluate(ic, beta)
    w_logp, w_ic, w_beta = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(logp, w_logp, rtol=2e-5)
    np.testing.assert_allclose(d_ic, w_ic, rtol=1e-4, atol=5e-3)
    np.testing.assert_allclose(d_beta, w_beta, rtol=2e-4, atol=2e-4 * np.abs(w_beta).max())
    for u, v in zip((logp, d_ic, d_beta), again):
        assert np.array_equal(u, v)


@pytest.mark.parametrize("K", [2, 3])
def test_glm_fp8_batches_chains(dev, K):
    torch.manual_seed(5)
    rows = [128 * 33 + 9, 700]
    Xs = [torch.randn(n, 256, device=dev) * torch.exp(0.7 * torch.randn(256, device=dev)) for n in rows]
    ys = [(torch.rand(n, device=dev) < 0.45).float() for n in rows]
    model = Fp8GlmShards.from_dense(Xs, ys, groups=[0, 1], n_groups=2, n_chains=K)
    rng = np.random.default_rng(8)
    ic = (rng.normal(size=(K, 2)) * 0.2).astype(np.float32)
    beta = (rng.normal(size=(K, 256)) * np.array([0.02, 0.2, 0.002])[:K, None]).astype(np.float32)  # different scales per chain
    with FederatedEngine(model) as eng:
        logp, d_ic, d_beta = eng.evaluate(ic, beta)
    assert logp.shape == (K,) and d_beta.shape == (K, 256)
    w = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(logp, w[0], rtol=2e-5)
    np.testing.assert_allclose(d_ic, w[1], rtol=1e-4, atol=5e-3)
    np.testing.assert_allclose(d_beta, w[2], rtol=2e-4, atol=2e-4 * np.abs(w[2]).max())


@pytest.mark.parametrize("family,K", [("gaussian", 1), ("poisson", 1), ("gaussian", 3), ("poisson", 2)])
def test_glm_fp8_unbounded_residual_families(dev, family, K):
    """Poisson / Gaussian on the fp8 kernel: residuals are block-scaled per 32-row group (scale-factor-B)."""
    torch.manual_seed(11)
    rows = [128 * 35 + 17, 640]
    P = 256
    Xs = [torch.randn(n, P, device=dev) * torch.exp(0.5 * torch.randn(P, device=dev)) for n in rows]
    beta_true = torch.randn(P, device=dev) * 0.02
    ys = []
    for X in Xs:
        eta = X @ beta_true
        if family == "poisson":
            ys.append(torch.poisson(torch.exp(eta.clamp(max=3.0) + 0.5)))
        else:
            # residual magnitudes spanning orders of magnitude between row groups
            noise = torch.exp(2.0 * torch.randn(X.shape[0], device=dev)) * torch.randn(X.shape[0], device=dev)
            ys.append(40.0 * eta + 25.0 * noise)
    model = Fp8GlmShards.from_dense(Xs, ys, groups=[0, 1], n_groups=2, n_chains=K, family=family)
    rng = np.random.default_rng(12)
    shape = (K,) if K > 1 else ()
    ic = (rng.normal(size=shape + (2,)) * 0.2).astype(np.float32)
    beta = (rng.normal(size=shape + (P,)) * 0.02).astype(np.float32)
    with FederatedEngine(model) as eng:
        logp, d_ic, d_beta = eng.evaluate(ic, beta)
        again = eng.evaluate(ic, beta)
    w = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(logp, w[0], rtol=3e-5)
    np.testing.assert_allclose(d_ic, w[1], rtol=2e-4, atol=2e-4 * np.abs(w[1]).max())
    np.testing.assert_allclose(d_beta, w[2], rtol=3e-4, atol=3e-4 * np.abs(w[2]).max())
    for u, v in zip((logp, d_ic, d_beta), again):
        assert np.array_equal(u, v)


@pytest.mark.parametrize("P,dtype", [(37, torch.float32), (200, torch.bfloat16), (700, torch.float32), (1000, torch.bfloat16)])
def test_glm_general_shape_fallback(dev, P, dtype):
    """Shapes none of the fast kernels accept (odd P, fp32 X, non-contiguous rows) still run fused."""
    torch.manual_seed(7)
    rows = [301, 64, 5]
    Xs, ys = [], []
    for n in rows:
        big = torch.randn(n, P + 3, device=dev).to(dtype)
        Xs.append(big[:, 1 : 1 + P])            # row stride P + 3, misaligned start
        ys.append((torch.rand(n, device=dev) < 0.5).float())
    model = GlmShards(Xs, ys, groups=[0, 1, 0], n_groups=2, family="logistic")
    assert model.use_tensor_cores() in (3, 4)
    ic = np.array([0.1, -0.2])
    beta = (np.random.default_rng(1).normal(size=P) * 0.05).astype(np.float32)
    with FederatedEngine(model) as eng:
        logp, d_ic, d_beta = eng.evaluate(ic, beta)
    w = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(logp, w[0], rtol=2e-5)
    np.testing.assert_allclose(d_ic, w[1], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(d_beta, w[2], rtol=1e-4, atol=2e-3)


def test_custom_likelihood_runs_inside_the_fused_kernel(dev):
    """A user-supplied likelihood (Student-t regression), compiled with nvcc at runtime."""
    family = CustomFamily(
        "const float d = y - eta; ll = -2.5f * log1pf(d * d * 0.25f); r = 5.f * d / (4.f + d * d);",
        torch_fn=lambda y, eta: (-2.5 * torch.log1p((y - eta) ** 2 / 4), 5 * (y - eta) / (4 + (y - eta) ** 2)),
    )
    torch.manual_seed(11)
    X = torch.randn(5000, 96, device=dev).to(torch.bfloat16)
    y = (X.float() @ torch.randn(96, device=dev) * 0.1 + torch.distributions.StudentT(4.0).sample((5000,)).to(dev)).float()
    model = GlmShards([X[:3000], X[3000:]], [y[:3000], y[3000:]], groups=[0, 1], n_groups=2, family=family)
    beta = (np.random.default_rng(3).normal(size=96) * 0.05).astype(np.float32)
    ic = np.array([0.05, -0.1])
    with FederatedEngine(model) as eng:
        logp, d_ic, d_beta = eng.evaluate(ic, beta)
    w = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(logp, w[0], rtol=2e-5)
    np.testing.assert_allclose(d_ic, w[1], rtol=1e-4, atol=5e-3)
    np.testing.assert_allclose(d_beta, w[2], rtol=1e-4, atol=5e-3)


@pytest.mark.parametrize("kernel", ["tc", "simt", "fp8", "generic"])
def test_glm_kernels_are_bit_reproducible_with_many_groups(dev, kernel):
    """Fixed-order reductions + fixed-point intercept accumulation: 10 repeats, identical bits."""
    torch.manual_seed(13)
    rows = [40_000, 25_000, 33_333, 128, 19_999]
    Xs = [torch.randn(n, 256, device=dev) for n in rows]
    ys = [(torch.rand(n, device=dev) < 0.5).float() for n in rows]
    if kernel == "fp8":
        model = Fp8GlmShards.from_dense(Xs, ys, groups=[0, 1, 2, 1, 0], n_groups=3)
    else:
        model = GlmShards([X.to(torch.bfloat16) for X in Xs], ys, groups=[0, 1, 2, 1, 0], n_groups=3, kernel=kernel)
    ic = np.array([0.3, -0.2, 0.1])
    beta = (np.random.default_rng(1).normal(size=256) * 0.03).astype(np.float32)
    with FederatedEngine(model) as eng:
        first = [v.copy() for v in eng.evaluate(ic, beta)]
        for _ in range(9):
            for u, v in zip(first, eng.evaluate(ic, beta)):
                assert np.array_equal(u, v)


def test_glm_simt_is_deterministic(dev):
    X, y, _ = synth_logistic_shard(50_000, 256, seed=5, device=dev)
    model = GlmShards([X], [y], kernel="simt")
    beta = np.full(256, 0.01, dtype=np.float32)
    with FederatedEngine(model) as eng:
        a = [v.copy() for v in eng.evaluate(np.array([0.0]), beta)]
        for _ in range(3):
            b = eng.evaluate(np.array([0.0]), beta)
            for u, v in zip(a, b):
                assert np.array_equal(u, v)  # fixed-order reductions: bit-identical


def test_ode_matches_float64_oracle(dev):
    shards = [synth_lv_shard(300, 12, seed=s, device=dev) for s in range(2)]
    model = OdeShards([s[0] for s in shards], [s[1] for s in shards], [s[2] for s in shards], [s[3] for s in shards])
    th = np.array([0.95, 0.42, 0.78, 0.21])
    with FederatedEngine(model) as eng:
        logp, grad = eng.evaluate(th)
    w_logp, w_grad = model.reference([th.astype(np.float32).astype(np.float64)])
    np.testing.assert_allclose(logp, w_logp, rtol=2e-4)
    np.testing.assert_allclose(grad, w_grad, rtol=5e-3, atol=1.0)


def test_user_defined_ode_systems_on_the_fused_kernel(dev):
    """csrc/ode_generic.cu (dual-number RK4): the Lotka-Volterra instance reproduces the hand-written
    kernel, and a user-supplied SIR system matches its float64 autograd oracle."""
    from pytensor_federated_b200.models import LOTKA_VOLTERRA, OdeSystem, synth_ode_shard

    shards = [synth_lv_shard(300, 12, seed=s, device=dev) for s in range(2)]
    args = ([s[0] for s in shards], [s[1] for s in shards], [s[2] for s in shards], [s[3] for s in shards])
    th = np.array([0.95, 0.42, 0.78, 0.21])
    with FederatedEngine(OdeShards(*args)) as eng:
        hand = eng.evaluate(th)
    with FederatedEngine(OdeShards(*args, system=LOTKA_VOLTERRA)) as eng:
        dual = eng.evaluate(th)
    np.testing.assert_allclose(dual[0], hand[0], rtol=1e-5)
    np.testing.assert_allclose(dual[1], hand[1], rtol=1e-3, atol=0.5)

    sir = OdeSystem(
        "const auto inf = th[0] * y[0] * y[1]; dy[0] = -inf; dy[1] = inf - th[1] * y[1]; dy[2] = th[1] * y[1];",
        lambda y, th, t: (-th[0] * y[0] * y[1], th[0] * y[0] * y[1] - th[1] * y[1], th[1] * y[1]),
        n_states=3, n_params=2, name="sir",
    )
    rng = np.random.default_rng(2)
    n = 500
    i0 = rng.uniform(0.02, 0.2, size=n)
    y0 = np.stack([1.0 - i0, i0, np.zeros(n)])
    theta = np.array([1.8, 0.5])
    t, y0_t, obs, sigma = synth_ode_shard(sir, theta, y0, 10, seed=4, device=dev, sigma=0.02, t_end=6.0)
    model = OdeShards([t], [y0_t], [obs], [sigma], system=sir)
    probe = np.array([1.7, 0.55])
    with FederatedEngine(model) as eng:
        logp, grad = eng.evaluate(probe)
        again = eng.evaluate(probe)
    w_logp, w_grad = model.reference([probe.astype(np.float32).astype(np.float64)])
    np.testing.assert_allclose(logp, w_logp, rtol=2e-4)
    np.testing.assert_allclose(grad, w_grad, rtol=5e-3, atol=1.0)
    assert np.array_equal(logp, again[0]) and np.array_equal(grad, again[1])


def test_service_client_reaches_gpu_node_through_local_registry(dev):
    """ArraysToArraysServiceClient("gpu", 0) -> fused engine, no sockets, no codec."""
    from pytensor_federated_b200 import LogpGradServiceClient, service

    x, y, sigma = make_demo_data()
    model = LinregShards([x], [y], [sigma], device=dev)
    with FederatedEngine(model) as eng:
        service.register_local_node("gpu", 0, eng.evaluate)
        try:
            client = LogpGradServiceClient("gpu", 0)
            logp, grads = client.evaluate(np.array(0.4), np.array(1.2))
            want = model.reference([np.array(0.4), np.array(1.2)])
            np.testing.assert_allclose(logp, want[0], rtol=1e-12)
            np.testing.assert_allclose(grads, want[1:], rtol=1e-11)
            del client
        finally:
            service.unregister_local_node("gpu", 0)


def test_device_timer_trace_orders_the_phases(dev):
    """Tracing subsystem: %globaltimer stamps of theta release -> node partial -> result release."""
    x, y, sigma = make_demo_data()
    with FederatedEngine(LinregShards([x], [y], [sigma], device=dev)) as eng:
        for i in range(5):
            eng.evaluate(np.array(0.1 * i), np.array(0.5))
        t_theta, t_partial, t_result = eng.trace(5)
        assert 0 < t_theta <= t_partial <= t_result
        assert (t_result - t_theta) < 5_000_000  # the whole fused evaluation is far below 5 ms


@pytest.mark.parametrize("kernel, P, dtype", [("simt", 256, torch.bfloat16), ("simt", 504, torch.bfloat16),
                                              ("generic", 37, torch.bfloat16), ("generic", 100, torch.float32)])
def test_glm_cuda_core_kernels_keep_per_node_output_blocks(dev, kernel, P, dtype):
    """The SIMT and general-shape kernels flush a warp's sums at node boundaries into fixed-point accumulators:
    per-node blocks for every GLM shape, bit-identical across repeats although several warps share a block."""
    torch.manual_seed(5)
    rows = [9_001, 128 * 7, 3, 12_345, 40]      # a 3-row and a 40-row segment: warps cross several boundaries
    node_ids = [0, 1, 1, 2, 3]
    groups = [0, 1, 0, 1, 1]
    Xs = [torch.randn(n, P, device=dev).to(dtype) for n in rows]
    ys = [(torch.rand(n, device=dev) < 0.5).float() for n in rows]
    model = GlmShards(Xs, ys, groups=groups, n_groups=2, kernel=kernel, node_ids=node_ids, n_nodes=4)
    rng = np.random.default_rng(8)
    ic = rng.normal(size=2) * 0.1
    beta = (rng.normal(size=P) * 0.03).astype(np.float32)
    with FederatedEngine(model) as eng:
        assert model.selected_kernel.startswith(kernel)
        raw = eng.evaluate_raw([ic, beta])
        assert np.array_equal(raw, eng.evaluate_raw([ic, beta]))
        blocks = model.per_node(raw)
        want = model.per_node(model.reference_partial([ic, beta], dtype=torch.float64))
        for n in range(4):
            np.testing.assert_allclose(blocks[n, :, 0], want[n, :, 0], rtol=2e-5)
            np.testing.assert_allclose(blocks[n, :, 1:], want[n, :, 1:], rtol=1e-4, atol=2e-2)
        assert np.all(blocks[0, :, 2] == 0) and np.all(blocks[3, :, 1] == 0)   # a node only touches its own intercept
        summed = eng.evaluate(ic, beta)
        np.testing.assert_allclose(summed[0], want[:, :, 0].sum(), rtol=2e-5)
        np.testing.assert_allclose(summed[2], want[:, 0, 3:].sum(0), rtol=1e-4, atol=5e-2)


@pytest.mark.parametrize("K", [1, 4])
def test_glm_tc_keeps_per_node_output_blocks(dev, K):
    """GlmShards(node_ids=...): one [K][1+G+P] block per node from ONE launch; the blocks equal the nodes'
    own models and add up to the pooled evaluation bit for bit across repeats."""
    from pytensor_federated_b200.federation import NodeFederation

    torch.manual_seed(21)
    rows = [20_000, 128 * 33, 7777, 15_000]
    node_ids = [0, 1, 1, 2]           # node 1 owns two segments
    Xs = [torch.randn(n, 256, device=dev).to(torch.bfloat16) for n in rows]
    ys = [(torch.rand(n, device=dev) < 0.5).float() for n in rows]
    groups = [0, 1, 1, 0]
    model = GlmShards(Xs, ys, groups=groups, n_groups=2, n_chains=K, kernel="tc", node_ids=node_ids, n_nodes=3)
    rng = np.random.default_rng(3)
    ic = rng.normal(size=(K, 2) if K > 1 else 2) * 0.1
    beta = (rng.normal(size=(K, 256) if K > 1 else 256) * 0.03).astype(np.float32)
    with FederatedEngine(model) as eng:
        raw = eng.evaluate_raw([ic, beta])
        again = eng.evaluate_raw([ic, beta])
        assert np.array_equal(raw, again)
        blocks = model.per_node(raw)
        want = model.per_node(model.reference_partial([ic, beta], dtype=torch.float64))
        for n in range(3):
            np.testing.assert_allclose(blocks[n, :, 0], want[n, :, 0], rtol=2e-5)
            np.testing.assert_allclose(blocks[n, :, 1:3], want[n, :, 1:3], rtol=1e-4, atol=2e-3)
            np.testing.assert_allclose(blocks[n, :, 3:], want[n, :, 3:], rtol=1e-4, atol=0.5)
        assert np.all(blocks[0, :, 2] == 0) and np.all(blocks[1, :, 1] == 0)   # a node only touches its own intercept
        summed = eng.evaluate(ic, beta)
        np.testing.assert_allclose(summed[0], want[:, :, 0].sum(0).reshape(np.shape(summed[0])), rtol=2e-5)
        if K == 1:
            fed = NodeFederation(eng)
            res = fed.evaluate_nodes({1: (ic, beta), 2: (ic, beta)})
            np.testing.assert_allclose(res[1][0], blocks[1, 0, 0], rtol=1e-12)
            np.testing.assert_allclose(res[2][1][1], blocks[2, 0, 3:], rtol=1e-12)


def test_ode_nodes_with_their_own_parameters_on_the_gpu(dev):
    shards = [synth_lv_shard(200, 10, seed=s, device=dev) for s in range(3)]
    model = OdeShards([s[0] for s in shards], [s[1] for s in shards], [s[2] for s in shards], [s[3] for s in shards],
                      node_ids=[0, 1, 2], n_nodes=3)
    th = np.array([[0.95, 0.42, 0.78, 0.21], [1.0, 0.4, 0.8, 0.2], [1.05, 0.38, 0.82, 0.19]])
    with FederatedEngine(model) as eng:
        logp, grads = eng.evaluate(th)
        assert grads.shape == (3, 4)
        blocks = model.per_node(eng.evaluate_raw([th]))
    want = model.per_node(model.reference_partial([th.astype(np.float32).astype(np.float64)]))
    np.testing.assert_allclose(blocks[:, 0], want[:, 0], rtol=2e-4)
    np.testing.assert_allclose(blocks[:, 1:], want[:, 1:], rtol=5e-3, atol=1.0)
    np.testing.assert_allclose(logp, want[:, 0].sum(), rtol=2e-4)


def test_glm_tensor_core_takes_many_segments_and_tiny_shards(dev):
    """100 segments (round 1 stopped at 64), some of a single row, some empty-tile padded, 7 groups."""
    torch.manual_seed(31)
    rng = np.random.default_rng(31)
    rows = [int(r) for r in rng.integers(1, 700, size=100)]
    rows[3], rows[50], rows[99] = 1, 128, 129
    Xs = [torch.randn(n, 128, device=dev).to(torch.bfloat16) for n in rows]
    ys = [(torch.rand(n, device=dev) < 0.5).float() for n in rows]
    groups = [i % 7 for i in range(100)]
    model = GlmShards(Xs, ys, groups=groups, n_groups=7, kernel="tc")
    ic = rng.normal(size=7) * 0.1
    beta = (rng.normal(size=128) * 0.05).astype(np.float32)
    with FederatedEngine(model) as eng:
        got = eng.evaluate(ic, beta)
        again = eng.evaluate(ic, beta)
    want = model.unpack_result(model.reference_partial([ic, beta], dtype=torch.float64))
    np.testing.assert_allclose(got[0], want[0], rtol=2e-5)
    np.testing.assert_allclose(got[1], want[1], rtol=1e-4, atol=2e-3)
    np.testing.assert_allclose(got[2], want[2], rtol=1e-4, atol=0.05)
    assert all(np.array_equal(a, b) for a, b in zip(got, again))


def test_glm_fp8_keeps_per_node_output_blocks(dev):
    """The hierarchical configuration as the reference would model it: one group AND one node per shard."""
    torch.manual_seed(9)
    rows = [128 * 50 + 3, 9000, 128 * 7]
    Xs = [torch.randn(n, 256, device=dev) * torch.exp(0.3 * torch.randn(256, device=dev)) for n in rows]
    ys = [(torch.rand(n, device=dev) < 0.4).float() for n in rows]
    model = Fp8GlmShards.from_dense(Xs, ys, groups=[0, 1, 2], n_groups=3, node_ids=[0, 1, 2], n_nodes=3)
    ic = np.array([0.2, -0.3, 0.05])
    beta = (np.random.default_rng(5).normal(size=256) * 0.02).astype(np.float32)
    with FederatedEngine(model) as eng:
        raw = eng.evaluate_raw([ic, beta])
        assert np.array_equal(raw, eng.evaluate_raw([ic, beta]))
        summed = eng.evaluate(ic, beta)
    blocks = model.per_node(raw)
    want = model.per_node(model.reference_partial([ic, beta], dtype=torch.float64))
    for n in range(3):
        np.testing.assert_allclose(blocks[n, 0, 0], want[n, 0, 0], rtol=2e-5)
        np.testing.assert_allclose(blocks[n, 0, 4:], want[n, 0, 4:], rtol=2e-4, atol=2e-4 * np.abs(want[n, 0, 4:]).max())
        assert np.count_nonzero(blocks[n, 0, 1:4]) == 1          # only the node's own intercept gradient
    np.testing.assert_allclose(summed[0], want[:, 0, 0].sum(), rtol=2e-5)


@pytest.mark.parametrize("which", ["glm-tc", "glm-fp8", "glm-simt", "linreg-1cta", "linreg-multi"])
def test_speculative_root_launches_give_the_same_results(dev, which):
    """`set_speculative`: the next evaluation's kernel is enqueued before theta exists and picks it up as tagged
    words from host memory.  Same bits as one launch per evaluation; kernels that wait in vain give up (idle
    tick) and the next evaluate launches afresh; explicit launches and toggling keep the epochs in step."""
    import time

    torch.manual_seed(4)
    rng = np.random.default_rng(2)
    if which.startswith("glm"):
        rows = [30_000, 5_000]
        Xs = [torch.randn(n, 256, device=dev).to(torch.bfloat16) for n in rows]
        ys = [(torch.rand(n, device=dev) < 0.5).float() for n in rows]
        if which == "glm-fp8":
            model = Fp8GlmShards.from_dense(Xs, ys, groups=[0, 1], n_groups=2)
        else:
            model = GlmShards(Xs, ys, groups=[0, 1], n_groups=2, kernel=which.split("-")[1])
        thetas = [[rng.normal(size=2) * 0.1, (rng.normal(size=256) * 0.03).astype(np.float32)] for _ in range(12)]
    else:
        sizes = [10] if which == "linreg-1cta" else [10, 70001, 333]
        xs = [rng.normal(size=n) for n in sizes]
        ys_ = [1.0 + 0.5 * x + rng.normal(scale=0.3, size=x.size) for x in xs]
        model = LinregShards(xs, ys_, [0.3 + 0.1 * i for i in range(len(sizes))], device=dev)
        thetas = [[rng.normal(size=len(sizes)), np.array(rng.normal())] for _ in range(12)]
    with FederatedEngine(model) as eng:
        want = [eng.evaluate_raw(th) for th in thetas]
        assert eng.set_speculative(300.0) and eng.speculative
        n0 = eng.kernel_launches
        got = [eng.evaluate_raw(th) for th in thetas[:6]]
        time.sleep(0.01)                                  # both kernels in the stream give up: idle ticks
        got += [eng.evaluate_raw(th) for th in thetas[6:9]]
        # explicit launch + wait while speculation is on (drains the speculative kernels first)
        e = eng.launch()
        np.testing.assert_array_equal(eng.wait(e), want[8])
        got += [eng.evaluate_raw(th) for th in thetas[9:]]
        for g, w in zip(got, want):
            np.testing.assert_array_equal(g, w)
        assert eng.kernel_launches - n0 >= len(thetas) + 1
        assert eng.set_speculative(0.0) is False
        np.testing.assert_array_equal(eng.evaluate_raw(thetas[0]), want[0])
        assert eng.set_speculative(300.0)
        np.testing.assert_array_equal(eng.evaluate_raw(thetas[1]), want[1])
    # a speculative engine that is closed right after an evaluation drains its waiting kernels
    with FederatedEngine(model, speculative_us=200.0) as eng:
        assert eng.speculative
        np.testing.assert_array_equal(eng.evaluate_raw(thetas[2]), want[2])
