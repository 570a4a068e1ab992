"""-m gpu: populations whose weight sets differ in shape (DeviceGNNPolicyPopulation with one configuration per set) against twins.

As in test_gpu_population_ppo.py, ``script=`` gives group k of the population's K b episodes and a b-episode twin environment
identical episode streams.  The twin is one DeviceGNNPolicy with set k's configuration and weights, and the single learner with
learner config k.  Over three collect -> learn iterations every comparison is bit for bit: the trajectory, the last act's outputs,
each learn call's statistics, IMPALA's V-trace arrays, and after the calls every compared set's weights, Adam moments and step
count, and PPO's kl_coeff."""
import ctypes as C
import dataclasses
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

A = 17
TRAJ_KEYS = ('graph_features_dynamic', 'model', 'action_mask', 'action', 'logp', 'value', 'reward', 'done')

# K = 4 sets differing in every field the environment does not fix
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
# the smallest admitted shape, and the largest whose read-out fits the head kernel's 200 KiB of shared memory: the sweep's widest
# embedding (64), 8 rounds, 512 hidden units (196,024 B staged)
SMALLEST = dict(out_features_msg=2, out_features_hidden=1, out_features_node=1, out_features_graph=1, num_rounds=2, fcnet_hiddens=(A,),
                vf_share_layers=False)
LARGEST = dict(out_features_msg=128, out_features_hidden=128, out_features_node=64, out_features_graph=8, num_rounds=8,
               fcnet_hiddens=(512,), vf_share_layers=True)


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


def _learner_configs(algo, K):
    from ddls_b200 import learn
    if algo == 'ppo':
        return [learn.PPOConfig(sgd_minibatch_size=12, num_sgd_iter=2, seed=7 * k + 1, lr=[3e-4, 1e-3, 5e-5, 2e-4][k % 4],
                                entropy_coeff=[0.003, 0.02, 0.0, 0.01][k % 4]) for k in range(K)]
    if algo == 'impala':
        return [learn.IMPALAConfig(rollout_fragment_length=4, train_batch_size=8, lr=[3e-4, 1e-3, 5e-5, 2e-3][k % 4],
                                   gamma=[0.99, 0.9, 0.999, 0.5][k % 4]) for k in range(K)]
    return [learn.PGConfig(lr=[3e-4, 1e-3, 5e-5, 2e-3][k % 4], gamma=[0.99, 0.9, 0.5, 1.0][k % 4]) for k in range(K)]


def _learners(algo):
    from ddls_b200 import learn
    return {'ppo': (learn.DevicePopulationPPOLearner, learn.DevicePPOLearner),
            'impala': (learn.DevicePopulationIMPALALearner, learn.DeviceIMPALALearner),
            'pg': (learn.DevicePopulationPGLearner, learn.DevicePGLearner)}[algo]


def _twin_run(algos, configs, b=3, H=8, J=6, kinds=('resnet',), compare=None, iters=3, graphs=None):
    """iters collect -> learn iterations of a population with one configuration per set and of its twins, the population's
    learner of iteration i being algos[i % len(algos)]; every comparison is asserted here.  The job types are `graphs`
    (synth.ForwardGraph) or else the workload graphs `kinds`.  Returns the population's embedding CTAs and, per compared set, its
    weight count."""
    from ddls_b200 import workload
    from ddls_b200 import policy as P
    K = len(configs)
    graphs = graphs or [workload.make_graph(k) for k in kinds]
    script = _script(K * b, J, len(graphs), seed=11)
    sds = [P.random_state_dict(dict(P.DEFAULT_CONFIG, **c), A, seed=30 + k) for k, c in enumerate(configs)]
    compare = list(range(K)) if compare is None else compare
    env = _env(graphs, K * b, J, script)
    pop = P.DeviceGNNPolicyPopulation(graphs, A, configs, sds)
    lcfg = {a: _learner_configs(a, K) for a in algos}
    plrn = {a: _learners(a)[0](pop, lcfg[a]) for a in algos}
    twins = {}
    for k in compare:
        tenv = _env(graphs, b, J, _rows(script, k * b, (k + 1) * b))
        tpol = P.DeviceGNNPolicy(graphs, A, configs[k], sds[k])
        twins[k] = (tenv, tpol, {a: _learners(a)[1](tpol, lcfg[a][k]) for a in algos})
    for it in range(iters):
        algo = algos[it % len(algos)]
        seeds = [1000 * it + 3 * k for k in range(K)]
        traj = {key: np.array(v) for key, v in pop.collect(env, H, seed=seeds).items()}
        last = pop.read(env)
        stats = plrn[algo].learn(env, H)
        for k, (tenv, tpol, tl) in twins.items():
            tt = tpol.collect(tenv, H, seed=seeds[k])
            cols = slice(k * b, (k + 1) * b)
            for key in TRAJ_KEYS:
                assert np.array_equal(traj[key][:, cols], tt[key]), (it, k, key)
            tr = tpol.read(tenv)
            for key in ('logits', 'value', 'logp', 'actions'):
                assert np.array_equal(last[key][cols], tr[key]), (it, k, key)
            ts = tl[algo].learn(tenv, H)
            assert stats[k] == ts, (algo, it, k, stats[k], ts)
            if algo == 'impala':
                mine, want = plrn[algo].vtrace(k), tl[algo].vtrace()
                assert mine.keys() == want.keys()
                for key in want:
                    assert np.array_equal(mine[key], want[key]), (it, k, key)
    seen = dict(ctas=pop.embed_ctas(), n_w={})
    for k, (tenv, tpol, tl) in twins.items():
        w = pop.get_weights(k)
        assert np.array_equal(w, tpol.get_weights()), k
        seen['n_w'][k] = len(w)
        for a in algos:                                                   # one Adam state per set, whichever learner reads it
            m, v, step = plrn[a].adam_state(k)
            tm, tv, tstep = tl[algos[0]].adam_state()
            assert np.array_equal(m, tm) and np.array_equal(v, tv) and step == tstep, (k, step, tstep)
        if 'ppo' in algos:
            assert plrn['ppo'].configs[k].kl_coeff == tl['ppo'].config.kl_coeff, k
        tpol.close()
    pop.close()
    return seen


@pytest.mark.parametrize('algo', ['ppo', 'impala', 'pg'])
def test_mixed_shapes_match_their_twins(algo):
    from ddls_b200 import policy as P
    n_w = _twin_run([algo], MIXED)['n_w']
    assert len(set(n_w.values())) == len(MIXED)
    assert [len(P.weight_keys(dict(P.DEFAULT_CONFIG, **c))) for c in MIXED] != [len(P.weight_keys(P.DEFAULT_CONFIG))] * len(MIXED)


def test_smallest_next_to_largest():
    """staging, records and the read-out's shared memory sized for the largest set carry the smallest"""
    from ddls_b200 import policy as P
    cfgs = [SMALLEST, LARGEST, SMALLEST]
    n_w = _twin_run(['ppo'], cfgs)['n_w']
    assert n_w[0] == n_w[2] < 1000 < 100_000 < n_w[1], n_w
    assert all(P.weight_count(dict(P.DEFAULT_CONFIG, **c), A) == n_w[k] for k, c in enumerate(cfgs))


def test_two_job_types_mixed_shapes():
    _twin_run(['ppo'], MIXED, kinds=('resnet', 'gpt2'))


def test_ppo_then_impala_then_pg_mixed_shapes():
    _twin_run(['ppo', 'impala', 'pg'], MIXED)


def test_phase3_grid_loops_the_embedding_grid():
    """the sweep's 128 shapes with two job types: K n_models items loop over the resident embedding CTAs.  Twins: the first,
    middle and last sets and the sets with the fewest and the most weights"""
    from ddls_b200 import policy as P
    grid = phase3_grid()
    K = len(grid)
    n_w = [P.weight_count(dict(P.DEFAULT_CONFIG, **c), A) for c in grid]
    compare = sorted({0, K // 2, K - 1, int(np.argmin(n_w)), int(np.argmax(n_w))})       # the grid's order puts them first and last
    seen = _twin_run(['ppo'], grid, b=1, kinds=('resnet', 'gpt2'), compare=compare)
    assert K * 2 > seen['ctas'], (K, seen['ctas'])
    assert seen['n_w'][int(np.argmin(n_w))] == min(n_w) < max(n_w) == seen['n_w'][int(np.argmax(n_w))]


def test_configs_list_of_one_config_equals_config():
    """configs=[c] * K runs the same bits as config=c"""
    from ddls_b200 import workload
    from ddls_b200 import policy as P
    from ddls_b200.learn import DevicePopulationPPOLearner
    K, b, H, J = 3, 4, 8, 6
    c = MIXED[1]
    graphs = [workload.make_graph('resnet')]
    script = _script(K * b, J, 1, seed=9)
    sds = [P.random_state_dict(dict(P.DEFAULT_CONFIG, **c), A, seed=50 + k) for k in range(K)]
    runs = []
    for config in (c, [c] * K):
        env = _env(graphs, K * b, J, script)
        pop = P.DeviceGNNPolicyPopulation(graphs, A, config, sds)
        lrn = DevicePopulationPPOLearner(pop, _learner_configs('ppo', K))
        out = []
        for it in range(2):
            traj = {key: np.array(v) for key, v in pop.collect(env, H, seed=[10 * it + k for k in range(K)]).items()}
            out.append((traj, lrn.learn(env, H)))
        out.append([(pop.get_weights(k), *lrn.adam_state(k)) for k in range(K)])
        runs.append(out)
        pop.close()
    for (ta, sa), (tb, sb) in zip(runs[0][:2], runs[1][:2]):
        assert all(np.array_equal(ta[key], tb[key]) for key in TRAJ_KEYS) and sa == sb
    for (wa, ma, va, na), (wb, mb, vb, nb) in zip(runs[0][2], runs[1][2]):
        assert np.array_equal(wa, wb) and np.array_equal(ma, mb) and np.array_equal(va, vb) and na == nb


def test_policy_and_state_dict_of_a_set():
    """policy(k) evaluates as its twin; gnn_state_dict(k) has set k's shapes and loads back unchanged"""
    from ddls_b200 import agents, workload
    from ddls_b200 import policy as P
    graphs = [workload.make_graph('resnet')]
    K, b, J = len(MIXED), 3, 5
    cfgs = [dict(P.DEFAULT_CONFIG, **c) for c in MIXED]
    sds = [P.random_state_dict(c, A, seed=60 + k) for k, c in enumerate(cfgs)]
    pop = P.DeviceGNNPolicyPopulation(graphs, A, MIXED, sds)
    for k in range(K):
        sd = pop.gnn_state_dict(k)
        assert {key: v.shape for key, v in sd.items()} == P.weight_shapes(cfgs[k], A)
        assert all(np.array_equal(sd[key], sds[k][key]) for key in sd)
        pop.set_weights(k, sd)
        assert np.array_equal(pop.get_weights(k), P.pack_weights(sds[k], cfgs[k], A))
        env = _env(graphs, b, J, _script(b, J, 1, seed=3))
        mine, twin = pop.policy(k), P.DeviceGNNPolicy(graphs, A, MIXED[k], sds[k])
        try:
            assert mine.config == twin.config
            assert _same(agents.evaluate(env, mine), agents.evaluate(env, twin))
        finally:
            mine.close()
            twin.close()
    pop.close()


def _same(a, b):
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return np.array_equal(np.asarray(a), np.asarray(b))


def _template(graphs, config=None):
    from ddls_b200 import policy as P
    tpl = P.DeviceGNNPolicy(graphs, A, config)
    P._bind_population(tpl._L)
    return tpl


def test_errors_name_the_set():
    from ddls_b200 import engine, workload
    from ddls_b200 import policy as P
    graphs = [workload.make_graph('resnet')]
    pop = P.DeviceGNNPolicyPopulation(graphs, A, MIXED[:2], [P.random_state_dict(dict(P.DEFAULT_CONFIG, **c), A) for c in MIXED[:2]])
    with pytest.raises(Exception, match='for set 1, its configuration has'):
        pop.set_weights(1, np.zeros(pop.weight_count(0), np.float32))
    pop.close()
    tpl = _template(graphs)
    cfgs = [P.c_config(dict(P.DEFAULT_CONFIG, **c), A, 1) for c in MIXED[:3]]
    # created from configurations alone, no set has weights: act refuses, naming the first set without
    h = C.c_void_p()
    engine._check(tpl._L.ramp_population_create_configs(tpl._h, 3, (P._Config * 3)(*cfgs), C.byref(h)))
    env = _env(graphs, 6, 4, _script(6, 4, 1, seed=2))
    seeds = np.zeros(3, np.uint64)
    with pytest.raises(Exception, match='set 0 has no weights'):
        engine._check(tpl._L.ramp_population_act(h, env.eng._h, 0, seeds.ctypes.data))
    blobs = [P.pack_weights(P.random_state_dict(dict(P.DEFAULT_CONFIG, **c), A), dict(P.DEFAULT_CONFIG, **c), A) for c in MIXED[:3]]
    for k in (0, 2):
        engine._check(tpl._L.ramp_population_set_weights(h, k, blobs[k].ctypes.data, len(blobs[k])))
    with pytest.raises(Exception, match='set 1 has no weights'):
        engine._check(tpl._L.ramp_population_act(h, env.eng._h, 0, seeds.ctypes.data))
    engine._check(tpl._L.ramp_population_set_weights(h, 1, blobs[1].ctypes.data, len(blobs[1])))
    engine._check(tpl._L.ramp_population_act(h, env.eng._h, 0, seeds.ctypes.data))
    tpl._L.ramp_population_destroy(h)
    # the fields the environment fixes, and each configuration's own checks
    for field, value in (('n_actions', A + 1), ('n_models', 2), ('in_features_edge', 3)):
        bad = list(cfgs)
        setattr(bad[2], field, value)
        h = C.c_void_p()
        with pytest.raises(Exception, match=f'set 2: {field} differs'):
            engine._check(tpl._L.ramp_population_create_configs(tpl._h, 3, (P._Config * 3)(*bad), C.byref(h)))
        assert not h.value
        setattr(bad[2], field, getattr(cfgs[0], field))
    bad = [P.c_config(dict(P.DEFAULT_CONFIG, **c), A, 1) for c in MIXED[:3]]
    bad[1].out_features_msg = 7
    with pytest.raises(Exception, match='set 1: policy: out_features_msg must be even'):
        engine._check(tpl._L.ramp_population_create_configs(tpl._h, 3, (P._Config * 3)(*bad), C.byref(h)))
    assert not h.value
    tpl.close()


def test_mixed_population_gives_back_every_byte():
    from ddls_b200 import engine, learn, workload
    from ddls_b200 import policy as P
    graphs = [workload.make_graph('resnet')]
    env = _env(graphs, 4, 4, _script(4, 4, 1, seed=3))
    cfgs = [MIXED[0], MIXED[3]]

    def lifecycle(check):
        pop = P.DeviceGNNPolicyPopulation(graphs, A, cfgs, [P.random_state_dict(dict(P.DEFAULT_CONFIG, **c), A, seed=s)
                                                            for s, c in enumerate(cfgs)])
        ppo = learn.DevicePopulationPPOLearner(pop, _learner_configs('ppo', 2))
        imp = learn.DevicePopulationIMPALALearner(pop, [dataclasses.replace(c, rollout_fragment_length=2, train_batch_size=4)
                                                        for c in _learner_configs('impala', 2)])
        pop.collect(env, 4, seed=[5, 6])
        ppo.learn(env, 4)
        pop.collect(env, 4, seed=[7, 8])
        imp.learn(env, 4)
        check()
        pop.close()

    lifecycle(lambda: None)
    gc.collect()
    base = engine.device_bytes()
    lifecycle(lambda: engine.device_bytes()[0] > base[0] or pytest.fail('the population holds no device memory'))
    gc.collect()
    assert engine.device_bytes() == base
    # a mixed population too large for the card: the creation fails naming the allocation and keeps nothing
    import torch
    tpl = _template(graphs)
    ccfgs = [P.c_config(dict(P.DEFAULT_CONFIG, **c), A, 1) for c in cfgs]
    n_w = sum(P.weight_count(dict(P.DEFAULT_CONFIG, **c), A) for c in cfgs) / 2
    K = int(2 * torch.cuda.get_device_properties(0).total_memory // (4 * n_w) + 1)
    before = engine.device_bytes()
    h = C.c_void_p()
    arr = (P._Config * K)()
    rows = np.array([np.frombuffer(bytes(c), dtype=np.int32) for c in ccfgs])
    np.frombuffer(arr, dtype=np.int32).reshape(K, -1)[:] = rows[np.arange(K) % 2]
    with pytest.raises(Exception, match='d_w'):
        engine._check(tpl._L.ramp_population_create_configs(tpl._h, K, arr, C.byref(h)))
    assert not h.value and engine.device_bytes() == before
    tpl.close()
