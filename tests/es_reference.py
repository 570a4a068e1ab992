"""A numpy restatement of RLlib's evolution strategies training step (ray/rllib/algorithms/es: utils.py compute_ranks /
compute_centered_ranks / batched_weighted_sum, optimizers.py Adam, es.py training_step), for the tests of the device ES learner
(ddls_b200/csrc/ramp_es.cuh).  RLlib is not installed; the functions are restated from the published sources.

Every scalar RLlib mixes into a float32 array is cast to float32 here explicitly, so that the float32 results do not depend on
numpy's promotion rules (numpy 2 would promote optimizers.Adam's float64 step size to float64)."""
import numpy as np

M64 = 2 ** 64 - 1


def mix64(x: int) -> int:
    """splitmix64, as the kernels' splitmix64"""
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def es_key(seed: int, iteration: int, rnd: int, x: int) -> int:
    k = mix64(seed & M64)
    k = mix64(k ^ iteration)
    k = mix64(k ^ rnd)
    return mix64(k ^ x)


def noise_indices(seed, iteration, rnd, n_pairs, noise_size, n):
    """pair i's noise index of round rnd: uniform on [0, noise_size - n] (RLlib's SharedNoiseTable.sample_index range)"""
    rng = noise_size - n + 1
    return np.array([(es_key(seed, iteration, rnd, 2 * i) * rng) >> 64 for i in range(n_pairs)], dtype=np.int64)


def act_seed(seed, iteration, rnd, t):
    """the draw seed of env-step t of round rnd (ramp_policy_decide's seed for the same decisions)"""
    return es_key(seed, iteration, rnd, 2 * t + 1)


def perturbed(theta, noise, index, sigma, sign):
    """fl(theta +- fl(sigma eps)), eps = noise[index : index + n] (es.py do_rollouts)"""
    eps = noise[index:index + len(theta)]
    d = np.float32(sigma) * eps
    return (theta + d if sign > 0 else theta - d).astype(np.float32)


def compute_ranks(x, kind=None):
    """utils.compute_ranks: ranks in [0, len(x) - 1]; kind='stable' gives ties to index order"""
    assert x.ndim == 1
    ranks = np.empty(len(x), dtype=int)
    ranks[x.argsort(kind=kind)] = np.arange(len(x))
    return ranks


def compute_centered_ranks(x, kind='stable'):
    """utils.compute_centered_ranks in float32: rank / (size - 1) - 0.5"""
    y = compute_ranks(x.ravel(), kind).reshape(x.shape).astype(np.float32)
    y /= np.float32(x.size - 1)
    y -= np.float32(0.5)
    return y


def itergroups(items, group_size):
    group = []
    for x in items:
        group.append(x)
        if len(group) == group_size:
            yield tuple(group)
            del group[:]
    if group:
        yield tuple(group)


def batched_weighted_sum(weights, vecs, batch_size=500):
    """utils.batched_weighted_sum: float32 dot products over batches of batch_size"""
    total, num = 0, 0
    for bw, bv in zip(itergroups(weights, batch_size), itergroups(vecs, batch_size)):
        assert len(bw) == len(bv) <= batch_size
        total += np.dot(np.asarray(bw, dtype=np.float32), np.asarray(bv, dtype=np.float32))
        num += len(bw)
    return total, num


def es_gradient(ranks, noise, idx, n):
    """es.py: g = batched_weighted_sum(rank+ - rank-, eps_i) / returns.size, float32 as RLlib forms it"""
    w = ranks[:, 0] - ranks[:, 1]
    g, count = batched_weighted_sum(w, (noise[i:i + n] for i in idx), batch_size=500)
    assert count == len(idx)
    return (np.asarray(g, np.float32) / np.float32(ranks.size)).astype(np.float32)


def es_gradient64(ranks, noise, idx, n):
    """the same sum in float64"""
    w = ranks[:, 0].astype(np.float64) - ranks[:, 1].astype(np.float64)
    g = np.zeros(n, np.float64)
    for wi, i in zip(w, idx):
        g += wi * noise[i:i + n].astype(np.float64)
    return g / ranks.size


class Adam:
    """optimizers.Adam, every operation float32 (the step size a = stepsize sqrt(1 - b2^t) / (1 - b1^t) formed in float64, then
    cast, as numpy's value-based casting did for the ray the reference pins)"""

    def __init__(self, n, stepsize, beta1=0.99, beta2=0.999, epsilon=1e-08):
        self.stepsize, self.beta1, self.beta2, self.epsilon = stepsize, beta1, beta2, epsilon
        self.t = 0
        self.m = np.zeros(n, dtype=np.float32)
        self.v = np.zeros(n, dtype=np.float32)

    def update(self, theta, globalg):
        """(theta + step, ||step|| / ||theta||)"""
        self.t += 1
        a = self.stepsize * (np.sqrt(1 - self.beta2 ** self.t) / (1 - self.beta1 ** self.t))
        f = np.float32
        self.m = f(self.beta1) * self.m + f(1 - self.beta1) * globalg
        self.v = f(self.beta2) * self.v + f(1 - self.beta2) * (globalg * globalg)
        step = f(-a) * self.m / (np.sqrt(self.v) + f(self.epsilon))
        ratio = np.linalg.norm(step.astype(np.float64)) / np.linalg.norm(theta.astype(np.float64))
        return (theta + step).astype(np.float32), ratio


def global_grad(theta, g, l2_coeff):
    """es.py: -g + l2_coeff * theta, float32"""
    return (-g + np.float32(l2_coeff) * theta).astype(np.float32)


def training_step(theta, returns, idx, noise, adam, l2_coeff, g=None):
    """es.py training_step after the rollouts, given the noisy returns [N, 2] and their noise indices: ranks, g (or the given g),
    Adam.  Returns (theta', ranks, g, info)."""
    n = len(theta)
    ranks = compute_centered_ranks(np.asarray(returns, np.float32))
    if g is None:
        g = es_gradient(ranks, noise, idx, n)
    new, ratio = adam.update(theta, global_grad(theta, g, l2_coeff))
    info = dict(weights_norm=float(np.square(new.astype(np.float64)).sum()), grad_norm=float(np.square(g.astype(np.float64)).sum()),
                update_ratio=float(ratio), episodes_this_iter=2 * len(idx))
    return new, ranks, g, info
