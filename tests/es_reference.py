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


def reward_mean(eval_means, report_length):
    """es_finish's episode_reward_mean: the mean of the last report_length steps' eval return means (steps without eval episodes
    add none), NaN before the first"""
    last = list(eval_means)[-report_length:]
    return float(np.mean(last)) if last else float('nan')


# ---- the launch rules of the population and update kernels (ramp_es.cuh), so that a test can say which of their loops it runs

ES_GRID, ES_THREADS, ES_PAIR_CHUNK = 264, 256, 1024     # ramp_es_update_kernel: CTAs, threads, pairs staged per chunk
EMBED_CTAS_PER_SM = 2          # ramp_es_embed_kernel: 256 threads at 80 registers fit 3 CTAs per SM; es_scratch caps it at 2
HEAD_WARPS, HEAD_CTAS_PER_SM = 8, 4                     # ramp_es_act: 8-warp CTAs, at most 4 per SM


def population_loops(B, n_eval, n_models, sm_count):
    """the trip counts of one round's population kernels on a device of sm_count SMs: pairs, sets, (set, job type) items, the
    embed grid and its largest items per CTA, head warps and their largest episodes per warp"""
    n_pairs = (B - n_eval) // 2
    n_sets = 2 * n_pairs + 1
    items = n_sets * n_models
    grid = min(EMBED_CTAS_PER_SM * sm_count, items)
    warps = HEAD_WARPS * max(1, min(-(-B // HEAD_WARPS), HEAD_CTAS_PER_SM * sm_count))
    return dict(n_pairs=n_pairs, n_sets=n_sets, items=items, embed_grid=grid, items_per_cta=-(-items // grid), head_warps=warps,
                episodes_per_warp=-(-B // warps))


def update_loops(n_pairs, n):
    """ramp_es_update_kernel's trip counts: pair chunks, and the weight passes of CTA 0 and of the last CTA"""
    stride = ES_GRID * ES_THREADS
    passes = [len(range(c * ES_THREADS, n, stride)) for c in (0, ES_GRID - 1)]
    return dict(pair_chunks=-(-n_pairs // ES_PAIR_CHUNK), max_weight_passes=passes[0], min_weight_passes=passes[1])


def set_of_episode(b, n_pairs):
    """episode b < 2 n_pairs runs set b; the eval episodes run theta, set 2 n_pairs"""
    return b if b < 2 * n_pairs else 2 * n_pairs


def episodes_of_set(s, B, n_pairs):
    return [s] if s < 2 * n_pairs else list(range(2 * n_pairs, B))


def coverage_sets(B, n_eval, n_models, sm_count, n_random=12, seed=0):
    """{path: weight sets} covering every loop of the population kernels that the round runs: the first and last pair, the eval
    set, the last (set, job type) item, items on the 2nd, 3rd and last pass of CTA 0, of a middle CTA and of the last CTA (item k
    runs on CTA k mod grid), episodes on the 2nd and 3rd pass of the first and last head warp (episode b on warp b mod warps),
    and n_random sets drawn with seed.  The last episode stands for the last warp's last pass.  Paths a round does not reach are
    left out."""
    k = population_loops(B, n_eval, n_models, sm_count)
    N, G, W, items = k['n_pairs'], k['embed_grid'], k['head_warps'], k['items']
    out = {'first and last pair': [0, 1, 2 * N - 2, 2 * N - 1], 'eval set': [2 * N] if n_eval else [],
           'last item': [(items - 1) // n_models]}
    for c in (0, G // 2, G - 1):
        last = (items - 1 - c) // G
        out[f'CTA {c}, passes 2, 3, last'] = sorted({(p * G + c) // n_models for p in (1, 2, last) if 1 <= p <= last})
    for p in (1, 2):
        if p * W < B:
            out[f'warp pass {p + 1}'] = sorted({set_of_episode(b, N) for b in (p * W, min(p * W + W - 1, B - 1))})
    rng = np.random.default_rng(seed)
    out['random'] = sorted(int(s) for s in rng.choice(2 * N, min(n_random, 2 * N), replace=False))
    return {path: sets for path, sets in out.items() if sets}


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
