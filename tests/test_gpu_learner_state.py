"""-m gpu: checkpoint and resume.  Three collect -> learn calls straight through equal, byte for byte, one call, training_state()
saved with np.savez, fresh learner and policy objects that load it, then two calls: every call's statistics, and at the end the
weights, the Adam state, kl_coeff and the call and act counts (ES: its step records, ES Adam state, iteration count and eval
means).  For DevicePPOLearner, DeviceIMPALALearner, DevicePGLearner, DeviceESLearner and each population learner at K = 4."""
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

A = 17
H, J = 8, 6


def _script(B, J, seed):
    rng = np.random.default_rng(seed)
    gap = rng.exponential(1000.0, size=(B, J))
    gap[:, J - 1] = np.inf
    return {'model': np.zeros((B, J), np.int64), 'gap': gap, 'frac': np.ones((B, J))}


def _env(B, J, script):
    from ddls_b200 import workload
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    return DeviceRampJobPartitioningEnvironment((4, 4, 4), [workload.make_graph('resnet')], n_episodes=B, jobs_per_episode=J,
                                                script=script)


def _bits(stats):
    return np.array([stats[k] for k in sorted(stats)], np.float64).view(np.uint64)


def _same_state(a, b):
    assert a.keys() == b.keys()
    for key in a:
        x, y = np.asarray(a[key]), np.asarray(b[key])
        assert x.shape == y.shape and x.tobytes() == y.astype(x.dtype).tobytes(), key


def _reload(state, tmp_path):
    """the state through its checkpoint file"""
    path = tmp_path / 'ckpt.npz'
    np.savez(path, **state)
    with np.load(path) as f:
        return {k: f[k] for k in f.files}


def _configs(algo, K):
    from ddls_b200 import learn
    if algo == 'ppo':
        return [learn.PPOConfig(sgd_minibatch_size=16, num_sgd_iter=2, seed=5 + k, lr=[3e-4, 1e-3, 5e-5, 2e-3][k % 4]) for k in range(K)]
    if algo == 'impala':
        return [learn.IMPALAConfig(rollout_fragment_length=4, train_batch_size=8, lr=[3e-4, 1e-3, 5e-5, 2e-3][k % 4]) for k in range(K)]
    if algo == 'pg':
        return [learn.PGConfig(lr=[3e-4, 1e-3, 5e-5, 2e-3][k % 4], gamma=0.9) for k in range(K)]
    return [learn.ESConfig(noise_stdev=0.05, n_eval=2, episodes_per_batch=1, train_batch_size=0, seed=9 + 13 * k) for k in range(K)]


def _single(algo, cfg, sd_seed, noise=None):
    from ddls_b200 import learn
    from ddls_b200 import policy as P
    from ddls_b200 import workload
    pol = P.DeviceGNNPolicy([workload.make_graph('resnet')], A, None, P.random_state_dict(P.DEFAULT_CONFIG, A, seed=sd_seed))
    cls = {'ppo': learn.DevicePPOLearner, 'impala': learn.DeviceIMPALALearner, 'pg': learn.DevicePGLearner}.get(algo)
    lrn = cls(pol, dataclasses.replace(cfg)) if cls else learn.DeviceESLearner(pol, dataclasses.replace(cfg), noise=noise)
    return pol, lrn


def _call(algo, pol, lrn, env, it, K=None):
    """one training call: collect -> learn (ES: one step); its statistics and, for ES, the step records"""
    if algo == 'es':
        stats = lrn.learn(env)
        recs = [lrn.last_step(k) for k in range(K)] if K else [lrn.last_step()]
        return stats, recs
    seed = [100 * it + k for k in range(K)] if K else 100 * it
    pol.collect(env, H, seed=seed)
    return lrn.learn(env, H), []


def _same_call(a, b):
    (sa, ra), (sb, rb) = a, b
    for x, y in zip(sa if isinstance(sa, list) else [sa], sb if isinstance(sb, list) else [sb]):
        assert np.array_equal(_bits(x), _bits(y)), (x, y)
    for x, y in zip(ra, rb):
        for key in x:
            assert np.array_equal(x[key], y[key]), key


@pytest.mark.parametrize('algo', ['ppo', 'impala', 'pg', 'es'])
def test_single_resume_equals_uninterrupted(algo, tmp_path):
    b = 6 if algo == 'es' else 4
    env = _env(b, 4 if algo == 'es' else J, _script(b, 4 if algo == 'es' else J, seed=7))
    cfg = _configs(algo, 1)[0]
    noise = np.random.default_rng(1).standard_normal(200_000).astype(np.float32)
    pol, lrn = _single(algo, cfg, 3, noise)
    straight = [_call(algo, pol, lrn, env, it) for it in range(3)]
    want = lrn.training_state()
    pol.close()
    pol, lrn = _single(algo, cfg, 3, noise)
    first = _call(algo, pol, lrn, env, 0)
    _same_call(first, straight[0])
    state = _reload(lrn.training_state(), tmp_path)
    pol.close()
    pol, lrn = _single(algo, cfg, 44, noise)                              # other weights: the state replaces them
    lrn.load_training_state(state)
    for it in (1, 2):
        _same_call(_call(algo, pol, lrn, env, it), straight[it])
    _same_state(lrn.training_state(), want)
    if algo == 'ppo':
        assert want['calls'] == 3 and want['kl_coeff'] != cfg.kl_coeff
    if algo == 'es':
        assert want['iteration'] == 3 and len(want['eval_means']) == 3 and want['t'] == 3
    else:
        assert want['step'] > 0 and want['act_count'] == 3 * H
    pol.close()


def _population(algo, K, sd_seed, noise):
    from ddls_b200 import learn
    from ddls_b200 import policy as P
    from ddls_b200 import workload
    sds = [P.random_state_dict(P.DEFAULT_CONFIG, A, seed=sd_seed + k) for k in range(K)]
    pop = P.DeviceGNNPolicyPopulation([workload.make_graph('resnet')], A, None, sds)
    cls = {'ppo': learn.DevicePopulationPPOLearner, 'impala': learn.DevicePopulationIMPALALearner, 'pg': learn.DevicePopulationPGLearner}.get(algo)
    cfgs = _configs(algo, K)
    lrn = cls(pop, cfgs) if cls else learn.DevicePopulationESLearner(pop, cfgs, noise=noise)
    return pop, lrn


@pytest.mark.parametrize('algo', ['ppo', 'impala', 'pg', 'es'])
def test_population_resume_equals_uninterrupted(algo, tmp_path):
    K = 4
    b = 6 if algo == 'es' else 4
    jobs = 4 if algo == 'es' else J
    env = _env(K * b, jobs, _script(K * b, jobs, seed=8))
    noise = np.random.default_rng(1).standard_normal(200_000).astype(np.float32)
    pop, lrn = _population(algo, K, 30, noise)
    straight = [_call(algo, pop, lrn, env, it, K) for it in range(3)]
    want = [lrn.training_state(k) for k in range(K)]
    pop.close()
    pop, lrn = _population(algo, K, 30, noise)
    _same_call(_call(algo, pop, lrn, env, 0, K), straight[0])
    states = [_reload(lrn.training_state(k), tmp_path) for k in range(K)]
    pop.close()
    pop, lrn = _population(algo, K, 70, noise)
    for k in range(K):
        lrn.load_training_state(k, states[k])
    for it in (1, 2):
        _same_call(_call(algo, pop, lrn, env, it, K), straight[it])
    for k in range(K):
        _same_state(lrn.training_state(k), want[k])
    assert len({want[k]['weights'].tobytes() for k in range(K)}) == K
    pop.close()


def test_load_refuses_a_state_of_another_shape():
    from ddls_b200 import learn
    pol, lrn = _single('pg', learn.PGConfig(), 3)
    state = lrn.training_state()
    bad = dict(state, exp_avg=state['exp_avg'][:-1])
    with pytest.raises(ValueError, match='training state: exp_avg has'):
        lrn.load_training_state(bad)
    pol.close()
