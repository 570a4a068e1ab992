"""CPU: the numpy restatement of RLlib's ES update in tests/es_reference.py, which the device ES learner is checked against."""
import numpy as np

from es_reference import (Adam, compute_centered_ranks, compute_ranks, coverage_sets, episodes_of_set, es_gradient, es_gradient64,
                          global_grad, mix64, noise_indices, perturbed, population_loops, reward_mean, set_of_episode, training_step,
                          update_loops)


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


def test_reward_mean_is_es_finishs_window():
    assert np.isnan(reward_mean([], 10))
    assert reward_mean([1.0, 3.0], 10) == 2.0
    assert reward_mean(np.arange(12.0), 10) == np.arange(2.0, 12.0).mean()


def test_population_loops_on_a_132_sm_part():
    """the trip counts the GPU tests assert, for the H100's 132 SMs: gnn.yaml at 8,704 episodes, three job types"""
    k = population_loops(8704, 2, 3, 132)
    assert (k['n_pairs'], k['n_sets'], k['items'], k['embed_grid']) == (4351, 8703, 26109, 264)
    assert k['items_per_cta'] == 99 and k['head_warps'] == 4224 and k['episodes_per_warp'] == 3
    k = population_loops(16, 2, 2, 132)                       # the twin-environment test: one item per CTA, one episode per warp
    assert k['embed_grid'] == k['items'] == 30 and k['items_per_cta'] == 1 and k['episodes_per_warp'] == 1
    assert update_loops(1024, 10)['pair_chunks'] == 1 and update_loops(1025, 10)['pair_chunks'] == 2
    u = update_loops(1100, 305_187)
    assert (u['pair_chunks'], u['max_weight_passes'], u['min_weight_passes']) == (2, 5, 4)
    assert update_loops(1, 21_920)['max_weight_passes'] == 1


def test_coverage_sets_reach_every_loop():
    B, E, M, sm = 8704, 2, 3, 132
    k = population_loops(B, E, M, sm)
    N, G, W = k['n_pairs'], k['embed_grid'], k['head_warps']
    cov = coverage_sets(B, E, M, sm)
    sets = sorted({s for v in cov.values() for s in v})
    assert 20 <= len(sets) <= 40 and all(0 <= s <= 2 * N for s in sets)
    items = {it for s in sets for it in range(s * M, (s + 1) * M)}
    for c in (0, G - 1):
        passes = {it // G for it in items if it % G == c}
        assert {1, 2, (k['items'] - 1 - c) // G} <= passes, c
    assert k['items'] - 1 in items
    eps = {b for s in sets for b in episodes_of_set(s, B, N)}
    assert {b // W for b in eps} == {0, 1, 2} and B - 1 in eps and {0, 1, 2 * N - 2, 2 * N - 1} <= eps
    assert [set_of_episode(b, N) for b in (2 * N - 1, 2 * N, B - 1)] == [2 * N - 1, 2 * N, 2 * N]
    assert episodes_of_set(2 * N, B, N) == [B - 2, B - 1]
    assert 'eval set' not in coverage_sets(16, 0, 2, sm)          # n_eval = 0: every episode runs its own set
