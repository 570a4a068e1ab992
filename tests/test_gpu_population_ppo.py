"""-m gpu: K PPO trainings in one environment batch (DeviceGNNPolicyPopulation, DevicePopulationPPOLearner) against K twins.

Twin environments get identical episode streams through ``script=``: group k of the population's K b episodes replays the script
rows of a b-episode environment driven by one DeviceGNNPolicy holding set k's weights and one DevicePPOLearner with config k.
Every comparison is bit for bit: the trajectory each collect() records, the last act's logits, every learn call's statistics,
and after the calls every set's weights, Adam moments and step count, and kl_coeff.  Each case asserts the situation it exists for
(rows past the last full minibatch, a group with no row in the later minibatches, the embedding grid looping)."""
import dataclasses
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

A = 17
TRAJ_KEYS = ('graph_features_dynamic', 'model', 'action_mask', 'action', 'logp', 'value', 'reward', 'done')


def _script(B, J, n_models, seed, early=()):
    """per-episode job types, gaps and fractions; an episode in `early` gets no job after its first"""
    rng = np.random.default_rng(seed)
    gap = rng.exponential(1000.0, size=(B, J))
    gap[:, J - 1] = np.inf
    for b in early:
        gap[b, 0] = np.inf
    return {'model': rng.integers(0, n_models, size=(B, J)), 'gap': gap, 'frac': np.ones((B, J))}


def _rows(script, lo, hi):
    return {k: v[lo:hi] for k, v in script.items()}


def _env(graphs, B, J, script):
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    return DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=B, jobs_per_episode=J, script=script)


def _configs(K, mb, iters, vary):
    from ddls_b200.learn import PPOConfig
    out = []
    for k in range(K):
        c = PPOConfig(sgd_minibatch_size=mb, num_sgd_iter=iters, seed=7 * k + 1)
        if vary:
            c = dataclasses.replace(c, lr=[3e-4, 1e-3, 5e-5, 2e-4][k % 4], clip_param=[0.18, 0.3, 0.1, 0.25][k % 4],
                                    entropy_coeff=[0.003, 0.02, 0.0, 0.01][k % 4], grad_clip=[1.5, 0.5, 0.0, 4.0][k % 4])
        out.append(c)
    return out


CASES = {
    # name: K, b, horizon, jobs per episode, job types, minibatch, passes, vary hyperparameters, early groups, twins compared
    'k1': dict(K=1, b=6, H=8, J=6, kinds=('resnet',), mb=16, iters=3, vary=False),
    'k2_hparams': dict(K=2, b=5, H=8, J=6, kinds=('resnet',), mb=16, iters=3, vary=True),
    'k4_two_types': dict(K=4, b=4, H=8, J=6, kinds=('resnet', 'gpt2'), mb=12, iters=3, vary=True),
    'k2_early_end_one_pass': dict(K=2, b=6, H=8, J=6, kinds=('resnet',), mb=8, iters=1, vary=True, early=1),
    'k3_short_last_minibatch': dict(K=3, b=5, H=9, J=8, kinds=('resnet',), mb=16, iters=3, vary=True),
    'grid_loops': dict(K=None, b=1, H=8, J=6, kinds=('resnet',), mb=8, iters=1, vary=True, compare='ends'),
}


def _same(a, b):
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return np.array_equal(np.asarray(a), np.asarray(b))


@pytest.mark.parametrize('name', list(CASES))
def test_population_matches_its_twins(name):
    import torch
    from ddls_b200 import agents, workload
    from ddls_b200 import policy as P
    from ddls_b200.learn import DevicePopulationPPOLearner, DevicePPOLearner
    case = dict(CASES[name])
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    K = case['K'] or 2 * sms + 8                                         # K n_models > 2 SMs: the embedding CTAs loop
    b, H, J, mb, iters = case['b'], case['H'], case['J'], case['mb'], case['iters']
    graphs = [workload.make_graph(k) for k in case['kinds']]
    early = range(case.get('early', K) * b, (case.get('early', K) + 1) * b) if 'early' in case else ()
    script = _script(K * b, J, len(graphs), seed=11, early=early)
    cfgs = _configs(K, mb, iters, case['vary'])
    sds = [P.random_state_dict(P.DEFAULT_CONFIG, A, seed=30 + k) for k in range(K)]
    compare = [0, K // 2, K - 1] if case.get('compare') == 'ends' else list(range(K))
    env = _env(graphs, K * b, J, script)
    pop = P.DeviceGNNPolicyPopulation(graphs, A, None, sds)
    lrn = DevicePopulationPPOLearner(pop, cfgs)
    twins = {}
    for k in compare:
        tenv = _env(graphs, b, J, _rows(script, k * b, (k + 1) * b))
        tpol = P.DeviceGNNPolicy(graphs, A, None, sds[k])
        twins[k] = (tenv, tpol, DevicePPOLearner(tpol, cfgs[k]))
    ctas = pop.embed_ctas()
    if case.get('compare') == 'ends':
        assert K * len(graphs) > 2 * sms and K * len(graphs) > ctas, (K, ctas, sms)
    rows_seen = {k: [] for k in compare}
    for it in range(3):
        seeds = [1000 * it + 3 * k for k in range(K)]
        traj = {key: np.array(v) for key, v in pop.collect(env, H, seed=seeds).items()}
        last = pop.read(env)
        stats = lrn.learn(env, H)
        for k, (tenv, tpol, tlrn) in twins.items():
            tt = tpol.collect(tenv, H, seed=seeds[k])
            cols = slice(k * b, (k + 1) * b)
            for key in TRAJ_KEYS:
                assert np.array_equal(traj[key][:, cols], tt[key]), (name, it, k, key)
            tl = tpol.read(tenv)
            for key in ('logits', 'value', 'logp', 'actions'):
                assert np.array_equal(last[key][cols], tl[key]), (name, it, k, key)
            ts = tlrn.learn(tenv, H)
            assert stats[k] == ts, (name, it, k, stats[k], ts)
            rows_seen[k].append(int(ts['rows']))
    for k, (tenv, tpol, tlrn) in twins.items():
        assert np.array_equal(pop.get_weights(k), tpol.get_weights()), (name, k)
        m, v, step = lrn.adam_state(k)
        tm, tv, tstep = tlrn.adam_state()
        assert np.array_equal(m, tm) and np.array_equal(v, tv) and step == tstep, (name, k, step, tstep)
        assert lrn.configs[k].kl_coeff == tlrn.config.kl_coeff, (name, k)
    n_mb = -(-H * b // mb)
    if name == 'k3_short_last_minibatch':
        assert (H * b) % mb, 'the last minibatch must be short'
    if 'early' in case:
        g = case['early']
        assert max(rows_seen[g]) <= mb < min(rows_seen[1 - g]) and n_mb > 1, (rows_seen, n_mb)   # its later minibatches: no-ops
    if name == 'k2_hparams':
        w = [pop.get_weights(k) for k in range(K)]
        assert not np.array_equal(w[0], w[1])
    if name == 'k1':
        # evaluation: policy(k) is a standalone policy holding set k's weights
        tenv, tpol, _ = twins[0]
        mine = pop.policy(0)
        try:
            got, want = agents.evaluate(tenv, mine), agents.evaluate(tenv, tpol)
            assert _same(got, want)
        finally:
            mine.close()
    for tenv, tpol, _ in twins.values():
        tpol.close()
    pop.close()


def test_population_gives_back_every_byte():
    from ddls_b200 import engine, workload
    from ddls_b200 import policy as P
    from ddls_b200.learn import DevicePopulationPPOLearner
    graphs = [workload.make_graph('resnet')]
    env = _env(graphs, 4, 4, _script(4, 4, 1, seed=3))

    def lifecycle(check):
        pop = P.DeviceGNNPolicyPopulation(graphs, A, None, [P.random_state_dict(P.DEFAULT_CONFIG, A, seed=s) for s in (1, 2)])
        lrn = DevicePopulationPPOLearner(pop, _configs(2, 4, 2, True))
        pop.collect(env, 4, seed=[5, 6])
        lrn.learn(env, 4)
        check()
        pop.close()

    # the first run grows the environment's own tables (the placements its steps meet); the second takes the same steps
    lifecycle(lambda: None)
    gc.collect()
    base = engine.device_bytes()
    lifecycle(lambda: engine.device_bytes()[0] > base[0] or pytest.fail('the population holds no device memory'))
    gc.collect()
    assert engine.device_bytes() == base
    # a population too large for the card: the creation fails naming the allocation and keeps nothing
    import ctypes as C
    import torch
    tpl = P.DeviceGNNPolicy(graphs, A, None, P.random_state_dict(P.DEFAULT_CONFIG, A, seed=1))
    n_w = len(tpl.get_weights())
    K = int(2 * torch.cuda.get_device_properties(0).total_memory // (4 * n_w) + 1)
    assert K < 2 ** 31
    before = engine.device_bytes()
    P._bind_population(tpl._L)
    h = C.c_void_p()
    with pytest.raises(Exception, match='d_w'):
        engine._check(tpl._L.ramp_population_create(tpl._h, K, C.byref(h)))
    assert not h.value and engine.device_bytes() == before
    tpl.close()
