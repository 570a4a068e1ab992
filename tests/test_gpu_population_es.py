"""-m gpu: DevicePopulationESLearner (ramp_population_es_*) against twins.

As in test_gpu_population_ppo.py, ``script=`` gives group k of the population's K b episodes and a b-episode twin environment
identical episode streams.  The twin is one DeviceGNNPolicy with set k's configuration and weights and a DeviceESLearner with ES
config k on the same noise table.  Over three learn() steps every comparison is bit for bit: each step's statistics (NaNs
included), the step record (noise indices, returns, lengths, act seeds, ranks, g, eval returns and lengths), the last act's
outputs of the groups whose twin ran the population's last round, and after the steps every compared set's weights and ES Adam
state.  The number of rounds each group ran is held to the numpy round rule (es_population_reference.es_rounds)."""
import ctypes as C
import dataclasses
import gc

import numpy as np
import pytest

from es_population_reference import es_rounds

pytestmark = pytest.mark.gpu

A = 17
MIXED = [
    dict(out_features_msg=8, out_features_hidden=16, out_features_node=8, out_features_graph=4, num_rounds=2, fcnet_hiddens=(A,),
         aggregator_activation='relu', fcnet_activation='relu', vf_share_layers=True),
    dict(out_features_msg=32, out_features_hidden=64, out_features_node=16, out_features_graph=8, num_rounds=3, fcnet_hiddens=(32,),
         aggregator_activation='leaky_relu', fcnet_activation='tanh', vf_share_layers=False),
    dict(out_features_msg=64, out_features_hidden=32, out_features_node=32, out_features_graph=16, num_rounds=4, fcnet_hiddens=(256,),
         aggregator_activation='relu', fcnet_activation='tanh', vf_share_layers=False),
    dict(out_features_msg=16, out_features_hidden=128, out_features_node=48, out_features_graph=24, num_rounds=2, fcnet_hiddens=(512,),
         aggregator_activation='leaky_relu', fcnet_activation='relu', vf_share_layers=True),
]
# more weights than one pass of the update kernel's grid covers (264 CTAs x 256 threads)
LARGEST = dict(out_features_msg=128, out_features_hidden=128, out_features_node=64, out_features_graph=8, num_rounds=8,
               fcnet_hiddens=(512,), vf_share_layers=True)
RECORD_KEYS = ('noise_index', 'returns', 'lengths', 'seeds', 'ranks', 'g', 'eval_returns', 'eval_lengths')


def phase3_grid():
    """scripts/wandb_sweep_config.yaml's PHASE 3 widths and round counts at gnn.yaml's other settings: 128 shapes"""
    return [dict(out_features_msg=m, out_features_hidden=h, out_features_node=n, num_rounds=r)
            for m in (8, 16, 32, 64) for h in (8, 16, 32, 64) for n in (8, 16, 32, 64) for r in (2, 4)]


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


def _es(K, **per_set):
    """K ES configs: n_eval 2, one episode and no env-step asked (one round), a seed per set; per_set: field -> list of K"""
    from ddls_b200.learn import ESConfig
    cfgs = [ESConfig(noise_stdev=0.05, n_eval=2, episodes_per_batch=1, train_batch_size=0, seed=9 + 13 * k) for k in range(K)]
    for field, values in per_set.items():
        for c, v in zip(cfgs, values):
            setattr(c, field, v)
    return cfgs


def _noise(n, extra=4000, seed=11):
    return np.random.default_rng(seed).standard_normal(n + extra).astype(np.float32)


def _bits(stats):
    return np.array([stats[k] for k in sorted(stats)], np.float64).view(np.uint64)


def _same_stats(a, b):
    return a.keys() == b.keys() and np.array_equal(_bits(a), _bits(b))


def _population(graphs, pcfgs, seed=30):
    from ddls_b200 import policy as P
    sds = [P.random_state_dict(dict(P.DEFAULT_CONFIG, **(c or {})), A, seed=seed + k) for k, c in enumerate(pcfgs)]
    return P.DeviceGNNPolicyPopulation(graphs, A, pcfgs, sds), sds


def _twin_run(pcfgs, ecfgs, b=6, J=4, kinds=('resnet',), compare=None, iters=3, graphs=None):
    """iters learn() steps of a population with policy configs pcfgs and ES configs ecfgs, and of its twins; every comparison is
    asserted here.  Returns per compared set its rounds per step, and the last round's embedding launch (CTAs, items)."""
    from ddls_b200 import workload
    from ddls_b200 import policy as P
    from ddls_b200.learn import DeviceESLearner, DevicePopulationESLearner
    K = len(pcfgs)
    graphs = graphs or [workload.make_graph(k) for k in kinds]
    script = _script(K * b, J, len(graphs), seed=11)
    pop, sds = _population(graphs, pcfgs)
    noise = _noise(max(pop.weight_count(k) for k in range(K)))
    env = _env(graphs, K * b, J, script)
    lrn = DevicePopulationESLearner(pop, ecfgs, noise=noise)
    compare = list(range(K)) if compare is None else compare
    twins = {}
    for k in compare:
        tenv = _env(graphs, b, J, _rows(script, k * b, (k + 1) * b))
        tpol = P.DeviceGNNPolicy(graphs, A, pcfgs[k], sds[k])
        twins[k] = (tenv, tpol, DeviceESLearner(tpol, ecfgs[k], noise=noise))
    seen = dict(rounds={k: [] for k in compare})
    for it in range(iters):
        stats = lrn.learn(env)
        logits, logp, actions = lrn.act_read(env)
        last = max(int(s['rounds']) for s in stats)
        lengths, n_pairs = [], []
        for k, (tenv, tpol, tl) in twins.items():
            ts = tl.learn(tenv)
            assert _same_stats(stats[k], ts), (it, k, stats[k], ts)
            mine, want = lrn.last_step(k), tl.last_step()
            for key in RECORD_KEYS:
                assert mine[key].dtype == want[key].dtype and np.array_equal(mine[key], want[key]), (it, k, key)
            if int(ts['rounds']) == last:                      # the twin ran the population's last round
                cols = slice(k * b, (k + 1) * b)
                tlog, tlp, tact = tl.act_read(tenv)
                assert np.array_equal(logits[cols], tlog) and np.array_equal(logp[cols], tlp) and np.array_equal(actions[cols], tact), (it, k)
            seen['rounds'][k].append(int(stats[k]['rounds']))
            n_pairs.append(len(mine['noise_index']) // int(stats[k]['rounds']))
            lengths.append(mine['lengths'].reshape(int(stats[k]['rounds']), -1))
        # the population's round counts against the numpy round rule on the lengths the population recorded (the twin
        # comparisons above hold those lengths and counts to the single learner's); its eval episodes do not count
        R = max(len(l) for l in lengths)
        padded = np.zeros((R, len(twins), 2 * max(n_pairs)), np.int64)
        for j, l in enumerate(lengths):
            padded[:len(l), j, :l.shape[1]] = l
            padded[len(l):, j, :l.shape[1]] = 10 ** 6         # rounds the twin did not run: any length ends the rule
        cfg = [ecfgs[k] for k in twins]
        _, r_k, rounds = es_rounds(padded, n_pairs, [c.episodes_per_batch for c in cfg], [c.train_batch_size for c in cfg])
        assert list(r_k) == [seen['rounds'][k][-1] for k in twins], (it, r_k)
        if compare == list(range(K)):
            assert rounds == last
    seen['embed'] = lrn.embed_ctas()
    for k, (tenv, tpol, tl) in twins.items():
        assert np.array_equal(pop.get_weights(k), tpol.get_weights()), k
        m, v, t = lrn.adam_state(k)
        tm, tv, tt = tl.adam_state()
        assert np.array_equal(m, tm) and np.array_equal(v, tv) and t == tt == iters, (k, t, tt)
        tl.close()
        tpol.close()
    lrn.close()
    pop.close()
    return seen


def test_one_set():
    _twin_run([None], _es(1))


@pytest.mark.parametrize('K', [2, 4])
def test_sets_with_their_own_hyperparameters(K):
    ecfgs = _es(K, noise_stdev=[0.05, 0.2, 0.01, 0.1][:K], stepsize=[0.01, 0.05, 0.002, 0.02][:K], l2_coeff=[0.005, 0.0, 0.05, 0.01][:K],
                n_eval=[2, 4, 0, 2][:K], adam_beta1=[0.99, 0.9, 0.99, 0.5][:K])
    _twin_run([None] * K, ecfgs, b=8)


def test_two_job_types():
    _twin_run([None] * 2, _es(2), kinds=('resnet', 'gpt2'))


def test_groups_run_different_numbers_of_rounds():
    """b = 6, n_eval 2: 4 noisy episodes a round.  Set 0 stops after one round, set 1 after two (episodes), set 2 after three
    (episodes), set 3 on its env-steps; in the later rounds the stopped groups run theta and record nothing"""
    J = 4
    ecfgs = _es(4, episodes_per_batch=[4, 8, 12, 1], train_batch_size=[0, 0, 0, 3 * 4 * J])
    seen = _twin_run([None] * 4, ecfgs, J=J)
    for it in range(3):
        r = [seen['rounds'][k][it] for k in range(4)]
        assert r[:3] == [1, 2, 3] and r[3] >= 1, r
    print('rounds per step and set:', seen['rounds'])


def test_a_set_without_eval_episodes():
    ecfgs = _es(3, n_eval=[0, 2, 0], report_length=[1, 3, 10])
    _twin_run([None] * 3, ecfgs)


def test_sets_of_different_shapes():
    ecfgs = _es(4, noise_stdev=[0.05, 0.1, 0.02, 0.2], n_eval=[2, 0, 4, 2])
    _twin_run(MIXED, ecfgs, b=8)


def test_phase3_grid_loops_the_embedding_grid():
    """the sweep's 128 shapes with two job types and b = 2 (one pair, no eval episode): 3 ES weight sets per group, 768 embedding
    items, more than the resident CTAs run at once.  Twins at the ends and the middle of the grid"""
    grid = phase3_grid()
    K = len(grid)
    seen = _twin_run(grid, _es(K, n_eval=[0] * K), b=2, kinds=('resnet', 'gpt2'), compare=[0, K // 2, K - 1], iters=3)
    ctas, items = seen['embed']
    print(f'embedding launch: {items} items on {ctas} CTAs, {-(-items // ctas)} trips for the busiest CTA')
    assert items == K * 3 * 2 and ctas < items, seen['embed']


def test_update_on_host_inputs_per_set():
    """update() per set across 1,024 / 1,025 pairs (one and two pair chunks) and several passes of the weight loop, against the
    single learner's update() with the same inputs"""
    from ddls_b200 import workload
    from ddls_b200 import policy as P
    from ddls_b200.learn import DeviceESLearner, DevicePopulationESLearner
    graphs = [workload.make_graph('resnet')]
    pcfgs = [MIXED[0], LARGEST, MIXED[2]]
    K = len(pcfgs)
    pop, sds = _population(graphs, pcfgs)
    n = [pop.weight_count(k) for k in range(K)]
    assert n[1] > 2 * 264 * 256, n                                   # the largest set takes three passes of the weight loop
    noise = _noise(max(n))
    ecfgs = _es(K, stepsize=[0.02, 0.01, 0.05], l2_coeff=[0.005, 0.0, 0.01])
    lrn = DevicePopulationESLearner(pop, ecfgs, noise=noise)
    twins = [P.DeviceGNNPolicy(graphs, A, pcfgs[k], sds[k]) for k in range(K)]
    tls = [DeviceESLearner(twins[k], ecfgs[k], noise=noise) for k in range(K)]
    rng = np.random.default_rng(5)
    for pairs in ([1024, 1025, 3], [1, 1024, 1025], [2048, 7, 1]):
        idx = [rng.integers(0, len(noise) - n[k] + 1, p).astype(np.int32) for k, p in enumerate(pairs)]
        idx[0][::5] = len(noise) - n[0]
        ret = [np.round(rng.normal(0, 3, (p, 2))).astype(np.float32) for p in pairs]      # ties: the stable rank order
        got = lrn.update(idx, ret)
        for k in range(K):
            s, ranks, g = got[k]
            ts, tranks, tg = tls[k].update(idx[k], ret[k])
            assert _same_stats(s, ts) and np.array_equal(ranks, tranks) and np.array_equal(g, tg), (pairs, k)
            assert np.array_equal(pop.get_weights(k), twins[k].get_weights()), (pairs, k)
            m, v, t = lrn.adam_state(k)
            tm, tv, tt = tls[k].adam_state()
            assert np.array_equal(m, tm) and np.array_equal(v, tv) and t == tt, (pairs, k)
    with pytest.raises(Exception, match='set 1: es: noise index'):
        lrn.update([idx[0], np.array([len(noise)], np.int32), idx[2]], [ret[0], np.zeros((1, 2), np.float32), ret[2]])
    with pytest.raises(ValueError, match='set 2: an update needs at least one pair'):
        lrn.update([idx[0], idx[1], np.zeros(0, np.int32)], [ret[0], ret[1], np.zeros((0, 2), np.float32)])
    lrn.reset()
    assert all(lrn.adam_state(k)[2] == 0 and not lrn.adam_state(k)[0].any() for k in range(K))
    for x in tls + twins:
        x.close()
    lrn.close()
    pop.close()


def test_torch_adam_untouched_and_ppo_after_es():
    """PPO, then two ES steps, then PPO on one population: the ES steps leave the population's torch-Adam state as it was, and
    the second PPO call still equals its twin's"""
    from ddls_b200 import workload
    from ddls_b200 import policy as P
    from ddls_b200.learn import DeviceESLearner, DevicePopulationESLearner, DevicePopulationPPOLearner, DevicePPOLearner, PPOConfig
    graphs = [workload.make_graph('resnet')]
    K, b, J, H = 2, 6, 4, 4
    pcfgs = [MIXED[0], MIXED[1]]
    script = _script(K * b, J, 1, seed=21)
    pop, sds = _population(graphs, pcfgs)
    noise = _noise(max(pop.weight_count(k) for k in range(K)))
    env = _env(graphs, K * b, J, script)
    pcfg = [PPOConfig(sgd_minibatch_size=8, num_sgd_iter=2, seed=3 + k) for k in range(K)]
    ecfgs = _es(K)
    ppo, es = DevicePopulationPPOLearner(pop, pcfg), DevicePopulationESLearner(pop, ecfgs, noise=noise)
    tw = []
    for k in range(K):
        tenv = _env(graphs, b, J, _rows(script, k * b, (k + 1) * b))
        tpol = P.DeviceGNNPolicy(graphs, A, pcfgs[k], sds[k])
        tw.append((tenv, tpol, DevicePPOLearner(tpol, pcfg[k]), DeviceESLearner(tpol, ecfgs[k], noise=noise)))

    def ppo_step(it):
        pop.collect(env, H, seed=[10 * it + k for k in range(K)])
        stats = ppo.learn(env, H)
        for k, (tenv, tpol, tp, _) in enumerate(tw):
            tpol.collect(tenv, H, seed=10 * it + k)
            assert stats[k] == tp.learn(tenv, H), (it, k)

    ppo_step(0)
    before = [ppo.adam_state(k) for k in range(K)]
    assert all(s[2] > 0 for s in before)
    for _ in range(2):
        stats = es.learn(env)
        for k, (tenv, _, _, te) in enumerate(tw):
            assert _same_stats(stats[k], te.learn(tenv)), k
    for k in range(K):
        m, v, step = ppo.adam_state(k)
        assert np.array_equal(m, before[k][0]) and np.array_equal(v, before[k][1]) and step == before[k][2], k
    ppo_step(1)
    for k, (tenv, tpol, tp, te) in enumerate(tw):
        assert np.array_equal(pop.get_weights(k), tpol.get_weights()), k
        m, v, step = ppo.adam_state(k)
        tm, tv, tstep = tp.adam_state()
        assert np.array_equal(m, tm) and np.array_equal(v, tv) and step == tstep, k
        te.close()
        tpol.close()
    es.close()
    pop.close()


def test_one_seed_gives_the_same_bits():
    from ddls_b200 import workload
    from ddls_b200.learn import DevicePopulationESLearner
    graphs = [workload.make_graph('resnet')]
    K, b, J = 3, 6, 4
    script = _script(K * b, J, 1, seed=4)
    ecfgs = _es(K, episodes_per_batch=[4, 8, 1])
    runs = []
    for _ in range(2):
        pop, _ = _population(graphs, MIXED[:K])
        env = _env(graphs, K * b, J, script)
        lrn = DevicePopulationESLearner(pop, ecfgs, noise=_noise(max(pop.weight_count(k) for k in range(K))))
        out = [[_bits(s) for s in lrn.learn(env)] for _ in range(2)]
        out.append([(pop.get_weights(k), *lrn.adam_state(k)[:2], *[lrn.last_step(k)[key] for key in RECORD_KEYS]) for k in range(K)])
        runs.append(out)
        lrn.close()
        pop.close()
    for a, b_ in zip(runs[0][:2], runs[1][:2]):
        assert all(np.array_equal(x, y) for x, y in zip(a, b_))
    for a, b_ in zip(runs[0][2], runs[1][2]):
        assert all(np.array_equal(x, y) for x, y in zip(a, b_))


def test_errors_name_the_set():
    from ddls_b200 import engine, workload
    from ddls_b200.learn import DevicePopulationESLearner, _CESConfig, _c_struct
    graphs = [workload.make_graph('resnet')]
    pop, _ = _population(graphs, MIXED[:3])
    noise = _noise(max(pop.weight_count(k) for k in range(3)))
    lrn = DevicePopulationESLearner(pop, _es(3), noise=noise)
    env = _env(graphs, 12, 4, _script(12, 4, 1, seed=2))
    with pytest.raises(ValueError, match='10 episodes do not split into 3 groups'):
        lrn.learn(_env(graphs, 10, 4, _script(10, 4, 1, seed=2)))
    # the C checks, reached past the Python ones
    bad = [_c_struct(_CESConfig, c, n_eval=2) for c in _es(3)]
    bad[2].report_length = 0
    with pytest.raises(Exception, match='population: set 2: es: episodes_per_batch'):
        engine._check(lrn._L.ramp_population_es_round_begin(lrn._h, env.eng._h, (_CESConfig * 3)(*bad), 0))
    bad[2].report_length = 10
    bad[1].n_eval = 3
    with pytest.raises(Exception, match='population: set 1: es: 4 episodes of its group less 3 eval episodes leave 1'):
        engine._check(lrn._L.ramp_population_es_round_begin(lrn._h, env.eng._h, (_CESConfig * 3)(*bad), 0))
    with pytest.raises(Exception, match='set 0: es: no complete round'):
        lrn.step()
    h = C.c_void_p()
    small = np.zeros(pop.weight_count(0), np.float32)
    first = next(k for k in range(3) if pop.weight_count(k) > len(small))
    with pytest.raises(Exception, match=f"smaller than set {first}'s"):
        engine._check(lrn._L.ramp_population_es_create(pop._h, small.ctypes.data, len(small), C.byref(h)))
    assert not h.value
    # a round after every group stopped is refused
    lrn.learn(env)
    env.reset()
    with pytest.raises(Exception, match='round 1 does not follow'):
        lrn.begin_round(env, 1)
    lrn.begin_round(env, 0)
    for t in range(env.J):
        lrn.act(env, t)
        env.step_device()
    assert not lrn.end_round(env)
    with pytest.raises(Exception, match='every set has collected'):
        lrn.begin_round(env, 1)
    lrn.close()
    pop.close()


def test_gives_back_every_byte():
    from ddls_b200 import engine, workload
    from ddls_b200.learn import DevicePopulationESLearner
    graphs = [workload.make_graph('resnet')]
    env = _env(graphs, 12, 4, _script(12, 4, 1, seed=3))

    def lifecycle(check):
        pop, _ = _population(graphs, MIXED[:2])
        lrn = DevicePopulationESLearner(pop, _es(2, episodes_per_batch=[4, 8]), noise=_noise(max(pop.weight_count(k) for k in range(2))))
        lrn.learn(env)
        lrn.update([np.zeros(3, np.int32), np.ones(2, np.int32)], [np.ones((3, 2), np.float32), np.ones((2, 2), np.float32)])
        check()
        lrn.close()
        pop.close()

    lifecycle(lambda: None)
    gc.collect()
    base = engine.device_bytes()
    lifecycle(lambda: engine.device_bytes()[0] > base[0] or pytest.fail('the learner holds no device memory'))
    gc.collect()
    assert engine.device_bytes() == base
    # the population closed before its learner: the learner refuses every call, and closing it gives back its bytes
    pop, _ = _population(graphs, MIXED[:2])
    lrn = DevicePopulationESLearner(pop, _es(2), noise=_noise(max(pop.weight_count(k) for k in range(2))))
    lrn.learn(env)
    pop.close()
    with pytest.raises(RuntimeError, match='population was closed before its ES learner'):
        lrn.learn(env)
    lrn.close()
    gc.collect()
    assert engine.device_bytes() == base
    # refused creations keep nothing: a table smaller than a set, and one whose noise indices do not fit int32 (refused before
    # the table is read)
    pop, _ = _population(graphs, MIXED[:2])
    before = engine.device_bytes()
    noise = np.zeros(pop.weight_count(1) - 1, np.float32)
    for size, match in ((len(noise), "smaller than set 1's"), ((1 << 31) + pop.weight_count(1), 'must fit in int32')):
        h = C.c_void_p()
        with pytest.raises(Exception, match=match):
            engine._check(pop._L.ramp_population_es_create(pop._h, noise.ctypes.data, size, C.byref(h)))
        assert not h.value and engine.device_bytes() == before
    pop.close()


def test_evaluate_a_population():
    """agents.evaluate(env, population) equals evaluate(twin, population.policy(k)) for every group, after ES steps"""
    from ddls_b200 import agents, workload
    from ddls_b200.learn import DevicePopulationESLearner
    graphs = [workload.make_graph('resnet')]
    K, b, J = 4, 6, 4
    script = _script(K * b, J, 1, seed=8)
    pop, _ = _population(graphs, MIXED)
    env = _env(graphs, K * b, J, script)
    lrn = DevicePopulationESLearner(pop, _es(K), noise=_noise(max(pop.weight_count(k) for k in range(K))))
    lrn.learn(env)
    got = agents.evaluate(env, pop)
    for k in range(K):
        tenv = _env(graphs, b, J, _rows(script, k * b, (k + 1) * b))
        tpol = pop.policy(k)
        want = agents.evaluate(tenv, tpol)
        assert got.keys() == want.keys()
        for key, v in want.items():
            mine = got[key][k * b:(k + 1) * b]
            assert len(mine) == len(v) and all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(mine, v)), (k, key)
        tpol.close()
    agents.evaluate(env, pop, sample=True, seed=5)
    lrn.close()
    pop.close()
