"""CPU: the numpy restatement of RLlib's ES update in tests/es_reference.py, which the device ES learner is checked against."""
import numpy as np

from es_reference import (Adam, compute_centered_ranks, compute_ranks, es_gradient, es_gradient64, global_grad, mix64, noise_indices,
                          perturbed, training_step)


def test_ranks_equal_rllibs_default_argsort_without_ties():
    rng = np.random.default_rng(0)
    x = rng.standard_normal((40, 2)).astype(np.float32)
    default = compute_ranks(x.ravel(), None)
    np.testing.assert_array_equal(compute_ranks(x.ravel(), 'stable'), default)
    want = (default.astype(np.float32) / np.float32(x.size - 1) - np.float32(0.5)).reshape(x.shape)
    np.testing.assert_array_equal(compute_centered_ranks(x), want)


def test_ties_go_to_index_order():
    x = np.array([[1.0, 1.0], [0.0, 1.0], [0.0, -1.0]], np.float32)
    r = compute_ranks(x.ravel(), 'stable')
    np.testing.assert_array_equal(r, [3, 4, 1, 5, 2, 0])
    y = compute_centered_ranks(np.full((5, 2), 3.0, np.float32))
    np.testing.assert_array_equal(y.ravel(), np.arange(10, dtype=np.float32) / np.float32(9) - np.float32(0.5))


def test_centered_ranks_sum_to_zero_within_half():
    rng = np.random.default_rng(1)
    for n in (1, 2, 7, 500):
        x = rng.integers(-3, 4, (n, 2)).astype(np.float32)
        y = compute_centered_ranks(x)
        assert y.dtype == np.float32
        assert abs(float(y.astype(np.float64).sum())) < 1e-5
        assert y.min() == -0.5 and y.max() == 0.5


def test_adam_follows_optimizers_py():
    """the float32 restatement against optimizers.py's statements in float64, step by step, and its dtypes"""
    rng = np.random.default_rng(2)
    n = 64
    theta = rng.standard_normal(n).astype(np.float32)
    ad = Adam(n, 0.01)
    m64, v64, th64 = np.zeros(n), np.zeros(n), theta.astype(np.float64)
    for t in range(1, 4):
        g = rng.standard_normal(n).astype(np.float32)
        gg = global_grad(theta, g, 0.005)
        new, ratio = ad.update(theta, gg)
        assert new.dtype == ad.m.dtype == ad.v.dtype == np.float32 and ad.t == t
        a = 0.01 * (np.sqrt(1 - 0.999 ** t) / (1 - 0.99 ** t))
        gg64 = -g.astype(np.float64) + 0.005 * th64
        m64 = 0.99 * m64 + (1 - 0.99) * gg64
        v64 = 0.999 * v64 + (1 - 0.999) * (gg64 * gg64)
        step64 = -a * m64 / (np.sqrt(v64) + 1e-08)
        np.testing.assert_allclose(ad.m, m64, rtol=1e-5, atol=1e-9)
        np.testing.assert_allclose(ad.v, v64, rtol=1e-5, atol=1e-12)
        np.testing.assert_allclose(new - theta, step64, rtol=1e-3, atol=1e-7)
        assert abs(ratio - np.linalg.norm(step64) / np.linalg.norm(th64)) < 1e-3 * ratio
        theta, th64 = new, new.astype(np.float64)


def test_gradient_batches_match_float64():
    rng = np.random.default_rng(3)
    n, N = 50, 1200                                           # three batches of batched_weighted_sum
    noise = rng.standard_normal(5000).astype(np.float32)
    idx = rng.integers(0, len(noise) - n + 1, N)
    ranks = compute_centered_ranks(rng.standard_normal((N, 2)).astype(np.float32))
    g, g64 = es_gradient(ranks, noise, idx, n), es_gradient64(ranks, noise, idx, n)
    assert np.linalg.norm(g - g64) <= 1e-6 * np.linalg.norm(g64)


def test_linear_return_estimate_aligns_with_its_slope():
    """R(theta) = c . theta with a small sigma: the ES estimate points along c"""
    rng = np.random.default_rng(4)
    n, N, sigma = 16, 400, 1e-3
    noise = rng.standard_normal(20000).astype(np.float32)
    c = rng.standard_normal(n)
    theta = rng.standard_normal(n).astype(np.float32)
    idx = noise_indices(7, 0, 0, N, len(noise), n)
    R = np.array([[c @ perturbed(theta, noise, i, sigma, +1), c @ perturbed(theta, noise, i, sigma, -1)] for i in idx], np.float32)
    new, ranks, g, info = training_step(theta, R, idx, noise, Adam(n, 0.01), 0.0)
    cos = float(g @ c) / (np.linalg.norm(g) * np.linalg.norm(c))
    assert cos > 0.9, cos
    assert float((new - theta) @ c) > 0                       # Adam on -g climbs the return
    assert info['episodes_this_iter'] == 2 * N


def test_splitmix64_and_noise_indices():
    assert mix64(0) == 0xE220A8397B1DCDAF                      # splitmix64's first output from state 0
    idx = noise_indices(3, 1, 2, 1000, 100, 40)
    assert idx.min() >= 0 and idx.max() <= 60 and len(np.unique(idx)) == 61
    np.testing.assert_array_equal(idx, noise_indices(3, 1, 2, 1000, 100, 40))
    assert (idx != noise_indices(3, 1, 3, 1000, 100, 40)).any()
