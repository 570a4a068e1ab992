"""-m gpu: population-based training on the device.  DeviceGNNPolicyPopulation.copy_sets and DevicePopulationESLearner.copy_sets
copy training state bit for bit and touch no other set; their refusals name the pair; after a PopulationBasedTraining step that
copies set j onto set i and perturbs i's learning rate, set i trains as a single learner that loaded j's training_state with i's
new config on i's twin environment, bit for bit; two runs from one seed decide and train alike; and every byte is given back."""
import dataclasses
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

A = 17
SMALL = dict(out_features_msg=8, out_features_hidden=16, out_features_node=8, out_features_graph=4, num_rounds=2, fcnet_hiddens=(A,),
             vf_share_layers=True)


def _script(B, J, n_models, seed):
    rng = np.random.default_rng(seed)
    gap = rng.exponential(1000.0, size=(B, J))
    gap[:, J - 1] = np.inf
    return {'model': rng.integers(0, n_models, size=(B, J)), 'gap': gap, 'frac': np.ones((B, J))}


def _rows(script, lo, hi):
    return {k: v[lo:hi] for k, v in script.items()}


def _env(graphs, B, J, script):
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    return DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=B, jobs_per_episode=J, script=script)


def _graphs():
    from ddls_b200 import workload
    return [workload.make_graph('resnet')]


def _population(K, configs=None, seed=30):
    from ddls_b200 import policy as P
    cfgs = configs or [None] * K
    sds = [P.random_state_dict(dict(P.DEFAULT_CONFIG, **(c or {})), A, seed=seed + k) for k, c in enumerate(cfgs)]
    return P.DeviceGNNPolicyPopulation(_graphs(), A, configs, sds), sds


def _random_states(lrn, pop, seed=0):
    """give every set distinct weights, Adam moments and step counts through load_training_state"""
    rng = np.random.default_rng(seed)
    for k in range(pop.K):
        n = pop.weight_count(k)
        lrn.load_training_state(k, dict(weights=rng.standard_normal(n).astype(np.float32) * 0.1,
                                        exp_avg=rng.standard_normal(n).astype(np.float32), exp_avg_sq=rng.random(n).astype(np.float32),
                                        step=10 + 3 * k, act_count=0, kl_coeff=0.01, calls=0))


def _snapshot(lrn, pop):
    return [(pop.get_weights(k),) + tuple(lrn.adam_state(k)) for k in range(pop.K)]


def _check_copy(before, after, dst, src):
    moved = dict(zip(dst, src))
    for k in range(len(before)):
        want = before[moved.get(k, k)]
        for a, b in zip(after[k], want):
            if isinstance(a, np.ndarray):
                assert a.dtype == b.dtype and a.tobytes() == b.tobytes(), k
            else:
                assert a == b, k


@pytest.mark.parametrize('K', [4, 272])
def test_copy_sets_bit_for_bit(K):
    """K = 272: 2 K n_models CTAs-worth of pairs, so the copy's grid strides over each slice"""
    from ddls_b200 import learn
    pop, _ = _population(K)
    lrn = learn.DevicePopulationPPOLearner(pop, [learn.PPOConfig(seed=k) for k in range(K)])
    _random_states(lrn, pop)
    before = _snapshot(lrn, pop)
    if K == 4:
        dst, src = [0, 2], [3, 3]                                          # one source, two destinations
    else:
        dst, src = list(range(0, 68)), [200 + i % 72 for i in range(68)]
    pop.copy_sets(dst, src)
    _check_copy(before, _snapshot(lrn, pop), dst, src)
    assert len(set(before[k][3] for k in range(K))) == K                  # the step counts were distinct, so they moved too
    pop.copy_sets([], [])                                                  # no pair: nothing happens
    pop.close()


def test_copy_sets_in_a_mixed_shape_population():
    from ddls_b200 import learn
    cfgs = [SMALL, None, SMALL, None]
    pop, _ = _population(4, cfgs)
    lrn = learn.DevicePopulationPGLearner(pop, [learn.PGConfig() for _ in range(4)])
    _random_states(lrn, pop)
    before = _snapshot(lrn, pop)
    pop.copy_sets([2, 1], [0, 3])
    _check_copy(before, _snapshot(lrn, pop), [2, 1], [0, 3])
    with pytest.raises(Exception, match=r'pair 0 \(set 1 <- set 0\): the sets differ in shape'):
        pop.copy_sets([1], [0])
    pop.close()


def test_copy_refusals_name_the_pair():
    from ddls_b200 import learn
    pop, _ = _population(4)
    lrn = learn.DevicePopulationPGLearner(pop, [learn.PGConfig() for _ in range(4)])
    _random_states(lrn, pop)
    before = _snapshot(lrn, pop)
    for dst, src, msg in [([0, 4], [1, 1], r'pair 1 \(set 4 <- set 1\): a set outside \[0, 4\)'),
                          ([-1], [1], r'pair 0 \(set -1 <- set 1\): a set outside'),
                          ([0, 0], [1, 2], r'pair 1 \(set 0 <- set 2\): set 0 is already the destination of pair 0'),
                          ([0, 1], [1, 2], r'pair 0 \(set 0 <- set 1\): set 1 is both a source and a destination'),
                          ([2], [2], r'pair 0 \(set 2 <- set 2\): set 2 is both a source and a destination')]:
        with pytest.raises(Exception, match=msg):
            pop.copy_sets(dst, src)
    with pytest.raises(ValueError, match='2 destinations for 1 sources'):
        pop.copy_sets([0, 1], [2])
    _check_copy(before, _snapshot(lrn, pop), [], [])                     # a refused copy changes nothing
    pop.close()


def test_es_copy_sets_bit_for_bit():
    from ddls_b200 import learn
    K = 4
    pop, _ = _population(K)
    noise = np.random.default_rng(1).standard_normal(pop.weight_count(0) + 1000).astype(np.float32)
    es = learn.DevicePopulationESLearner(pop, [learn.ESConfig(n_eval=2, seed=k) for k in range(K)], noise=noise)
    torch_adam = learn.DevicePopulationPGLearner(pop, [learn.PGConfig() for _ in range(K)])
    _random_states(torch_adam, pop, seed=1)
    rng = np.random.default_rng(2)
    for k in range(K):
        n = pop.weight_count(k)
        es.load_training_state(k, dict(weights=pop.get_weights(k), m=rng.standard_normal(n).astype(np.float32),
                                       v=rng.random(n).astype(np.float32), t=5 + k, iteration=7, eval_means=rng.standard_normal(k + 1)))
    before = [es.training_state(k) for k in range(K)]
    torch_before = _snapshot(torch_adam, pop)
    es.copy_sets([1, 0], [3, 3])
    for k in range(K):
        got, want = es.training_state(k), before[{1: 3, 0: 3}.get(k, k)]
        for key in ('m', 'v', 'eval_means'):
            assert got[key].tobytes() == want[key].tobytes(), (k, key)
        assert got['t'] == want['t'] and got['iteration'] == 7, k
    _check_copy(torch_before, _snapshot(torch_adam, pop), [], [])         # the weights and torch-Adam state are the population's
    with pytest.raises(Exception, match=r'pair 0 \(set 0 <- set 0\): set 0 is both'):
        es.copy_sets([0], [0])
    es.close()
    pop.close()


def _pbt_case(algo):
    from ddls_b200 import learn, pbt
    K, b, H, J = 4, 4, 8, 6
    if algo == 'ppo':
        cfgs = [learn.PPOConfig(sgd_minibatch_size=16, num_sgd_iter=2, seed=11 + k, lr=[1e-4, 3e-4, 1e-3, 2e-4][k]) for k in range(K)]
        Single, Pop, field = learn.DevicePPOLearner, learn.DevicePopulationPPOLearner, 'lr'
    elif algo == 'impala':
        cfgs = [learn.IMPALAConfig(rollout_fragment_length=4, train_batch_size=8, lr=[1e-4, 3e-4, 1e-3, 2e-4][k]) for k in range(K)]
        Single, Pop, field = learn.DeviceIMPALALearner, learn.DevicePopulationIMPALALearner, 'lr'
    else:
        cfgs = [learn.PGConfig(lr=[1e-4, 3e-4, 1e-3, 2e-4][k], gamma=[0.99, 0.9, 0.95, 0.5][k]) for k in range(K)]
        Single, Pop, field = learn.DevicePGLearner, learn.DevicePopulationPGLearner, 'lr'
    return K, b, H, J, cfgs, Single, Pop, {field: pbt.log_uniform(1e-5, 1e-2)}


def _bits(stats):
    return np.array([stats[k] for k in sorted(stats)], np.float64).view(np.uint64)


@pytest.mark.parametrize('algo', ['ppo', 'impala', 'pg'])
def test_exploit_and_explore_match_a_twin(algo):
    """collect -> learn; a PBT step on scores that make set 0 the worst and set 3 the best; then set 0 over two collect -> learn
    calls equals a fresh single learner that loaded set 3's training_state, with set 0's new config, on group 0's twin environment"""
    from ddls_b200 import policy as P
    from ddls_b200 import pbt
    K, b, H, J, cfgs, Single, Pop, mutations = _pbt_case(algo)
    graphs = _graphs()
    script = _script(K * b, J, 1, seed=5)
    env = _env(graphs, K * b, J, script)
    pop, _ = _population(K)
    lrn = Pop(pop, cfgs)
    sched = pbt.PopulationBasedTraining(lrn, mutations, seed=3)
    pop.collect(env, H, seed=[1, 2, 3, 4])
    lrn.learn(env, H)
    recs = sched.step([0.0, 1.0, 1.0, 2.0])
    (field,) = mutations
    assert [(r['set'], r['donor']) for r in recs] == [(0, 3)]
    assert recs[0]['old'][field] == cfgs[0].__dict__[field] and recs[0]['new'][field] != cfgs[3].__dict__[field]
    assert getattr(lrn.configs[0], field) == recs[0]['new'][field]
    if algo == 'ppo':
        assert lrn.configs[0].seed == cfgs[0].seed and lrn.configs[0].kl_coeff == lrn.configs[3].kl_coeff
    state = lrn.training_state(3)
    mine = lrn.training_state(0)
    for key in ('weights', 'exp_avg', 'exp_avg_sq', 'step'):
        assert np.array_equal(mine[key], state[key]), key
    tenv = _env(graphs, b, J, _rows(script, 0, b))
    tpol = P.DeviceGNNPolicy(graphs, A, None, P.random_state_dict(P.DEFAULT_CONFIG, A, seed=99))
    twin = Single(tpol, dataclasses.replace(lrn.configs[0]))
    twin.load_training_state(state)
    for it in range(2):
        seeds = [10 * it + k for k in range(K)]
        traj = pop.collect(env, H, seed=seeds)
        actions = np.array(traj['action'][:, :b])
        stats = lrn.learn(env, H)
        tt = tpol.collect(tenv, H, seed=seeds[0])
        assert np.array_equal(actions, tt['action']), it
        ts = twin.learn(tenv, H)
        assert np.array_equal(_bits(stats[0]), _bits(ts)), (it, stats[0], ts)
    got, want = lrn.training_state(0), twin.training_state()
    for key in want:
        assert np.array_equal(np.asarray(got[key]), np.asarray(want[key])), key
    tpol.close()
    pop.close()


def test_es_exploit_and_explore_match_a_twin():
    from ddls_b200 import policy as P
    from ddls_b200 import learn, pbt
    K, b, J = 4, 6, 4
    graphs = _graphs()
    script = _script(K * b, J, 1, seed=5)
    env = _env(graphs, K * b, J, script)
    pop, _ = _population(K)
    noise = np.random.default_rng(1).standard_normal(pop.weight_count(0) + 4000).astype(np.float32)
    cfgs = [learn.ESConfig(noise_stdev=0.05, n_eval=2, episodes_per_batch=1, train_batch_size=0, seed=9 + 13 * k,
                           stepsize=[0.01, 0.02, 0.005, 0.03][k]) for k in range(K)]
    lrn = learn.DevicePopulationESLearner(pop, cfgs, noise=noise)
    sched = pbt.PopulationBasedTraining(lrn, {'stepsize': pbt.log_uniform(1e-3, 1e-1)}, seed=4)
    lrn.learn(env)
    lrn.learn(env)
    recs = sched.step([-1.0, 0.0, 0.0, 5.0])
    assert [(r['set'], r['donor']) for r in recs] == [(0, 3)] and recs[0]['new']['stepsize'] != cfgs[3].stepsize
    assert lrn.configs[0].seed == cfgs[0].seed and lrn.configs[0].stepsize == recs[0]['new']['stepsize']
    state = lrn.training_state(3)
    got0 = lrn.training_state(0)
    for key in state:
        assert np.array_equal(np.asarray(got0[key]), np.asarray(state[key])), key
    assert len(state['eval_means']) == 2 and state['iteration'] == 2
    tenv = _env(graphs, b, J, _rows(script, 0, b))
    tpol = P.DeviceGNNPolicy(graphs, A, None, P.random_state_dict(P.DEFAULT_CONFIG, A, seed=99))
    twin = learn.DeviceESLearner(tpol, dataclasses.replace(lrn.configs[0]), noise=noise)
    twin.load_training_state(state)
    for it in range(2):
        stats = lrn.learn(env)
        ts = twin.learn(tenv)
        assert np.array_equal(_bits(stats[0]), _bits(ts)), (it, stats[0], ts)
        mine, want = lrn.last_step(0), twin.last_step()
        for key in want:
            assert np.array_equal(mine[key], want[key]), (it, key)
    got, want = lrn.training_state(0), twin.training_state()
    for key in want:
        assert np.array_equal(np.asarray(got[key]), np.asarray(want[key])), key
    twin.close()
    tpol.close()
    lrn.close()
    pop.close()


def _pbt_run(seed):
    from ddls_b200 import learn, pbt
    K, b, H, J = 8, 3, 8, 6
    env = _env(_graphs(), K * b, J, _script(K * b, J, 1, seed=7))
    pop, _ = _population(K)
    lrn = learn.DevicePopulationPGLearner(pop, [learn.PGConfig(lr=1e-4 * (k + 1), gamma=0.9) for k in range(K)])
    sched = pbt.PopulationBasedTraining(lrn, {'lr': pbt.log_uniform(1e-5, 1e-2), 'gamma': [0.5, 0.9, 0.99]}, interval=2, seed=seed)
    decisions = []
    for it in range(6):
        traj = pop.collect(env, H, seed=[it * 100 + k for k in range(K)])
        scores = pbt.group_returns(traj, K)
        lrn.learn(env, H)
        decisions.append(sched.step(scores))
    out = decisions, [pop.get_weights(k) for k in range(K)], [dataclasses.asdict(c) for c in lrn.configs]
    pop.close()
    return out


def test_two_runs_from_one_seed_agree():
    d1, w1, c1 = _pbt_run(seed=21)
    d2, w2, c2 = _pbt_run(seed=21)
    assert d1 == d2 and c1 == c2
    assert sum(len(d) for d in d1) == 6                                   # three PBT steps of 2 recipients
    assert all(a.tobytes() == b.tobytes() for a, b in zip(w1, w2))


def test_pbt_gives_back_every_byte():
    from ddls_b200 import engine, learn, pbt

    def lifecycle(check):
        K = 4
        env = _env(_graphs(), K * 2, 4, _script(K * 2, 4, 1, seed=3))
        pop, _ = _population(K)
        lrn = learn.DevicePopulationPGLearner(pop, [learn.PGConfig() for _ in range(K)])
        noise = np.random.default_rng(1).standard_normal(pop.weight_count(0) + 100).astype(np.float32)
        es = learn.DevicePopulationESLearner(pop, [learn.ESConfig(n_eval=0) for _ in range(K)], noise=noise)
        sched = pbt.PopulationBasedTraining(lrn, {'lr': [1e-4, 1e-3]})
        pop.collect(env, 4, seed=[1, 2, 3, 4])
        lrn.learn(env, 4)
        sched.step([0.0, 1.0, 2.0, 3.0])
        es.copy_sets([0], [1])
        lrn.load_training_state(2, lrn.training_state(1))
        check()
        es.close()
        pop.close()

    lifecycle(lambda: None)
    gc.collect()
    base = engine.device_bytes()
    lifecycle(lambda: engine.device_bytes()[0] > base[0] or pytest.fail('the population holds no device memory'))
    gc.collect()
    assert engine.device_bytes() == base
