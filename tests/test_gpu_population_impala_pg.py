"""-m gpu: K IMPALA and K PG trainings in one environment batch (DevicePopulationIMPALALearner, DevicePopulationPGLearner) against
K twins.

As in test_gpu_population_ppo.py, ``script=`` gives group k of the population's K b episodes and a b-episode twin environment
identical episode streams; the twin is one DeviceGNNPolicy holding set k's weights with one DeviceIMPALALearner / DevicePGLearner
with config k.  Over three collect -> learn iterations every comparison is bit for bit: each learn call's statistics, IMPALA's
V-trace arrays, and after the calls every compared set's weights, Adam moments and step count.  Each case asserts the situation it
exists for."""
import dataclasses
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

A = 17


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


def _impala_configs(K, L, tbs, vary):
    from ddls_b200.learn import IMPALAConfig
    out = []
    for k in range(K):
        c = IMPALAConfig(rollout_fragment_length=L, train_batch_size=tbs, lr=3e-4)
        if vary:
            c = dataclasses.replace(c, lr=[3e-4, 1e-3, 5e-5, 2e-3][k % 4], vtrace_clip_rho_threshold=[1.0, 0.8, 1.5, 0.9][k % 4],
                                    vtrace_clip_pg_rho_threshold=[1.0, 0.7, 2.0, 1.2][k % 4], entropy_coeff=[0.01, 0.05, 0.0, 0.02][k % 4],
                                    vf_loss_coeff=[0.5, 1.0, 0.25, 0.1][k % 4], grad_clip=[40.0, 0.5, 0.0, 4.0][k % 4],
                                    gamma=[0.99, 0.9, 0.999, 0.5][k % 4])
        out.append(c)
    return out


def _pg_configs(K, vary):
    from ddls_b200.learn import PGConfig
    out = []
    for k in range(K):
        c = PGConfig(lr=3e-4)
        if vary:
            c = dataclasses.replace(c, gamma=[0.99, 0.9, 0.5, 1.0][k % 4], lr=[3e-4, 1e-3, 5e-5, 2e-3][k % 4], grad_clip=[0.0, 0.5, 4.0, 1e-3][k % 4])
        out.append(c)
    return out


def _twin_run(algo, K, b, H, J, kinds, cfgs, early=None, compare=None):
    """three collect -> learn iterations of the population and its twins; every comparison asserted here.  Returns what the
    cases assert about: per iteration the population's trajectory and statistics, and per compared set its V-trace arrays."""
    from ddls_b200 import workload
    from ddls_b200 import policy as P
    from ddls_b200 import learn
    graphs = [workload.make_graph(k) for k in kinds]
    early_eps = range(early * b, (early + 1) * b) if early is not None else ()
    script = _script(K * b, J, len(graphs), seed=11, early=early_eps)
    sds = [P.random_state_dict(P.DEFAULT_CONFIG, A, seed=30 + k) for k in range(K)]
    compare = list(range(K)) if compare is None else compare
    Pop, Single = {'impala': (learn.DevicePopulationIMPALALearner, learn.DeviceIMPALALearner),
                   'pg': (learn.DevicePopulationPGLearner, learn.DevicePGLearner)}[algo]
    env = _env(graphs, K * b, J, script)
    pop = P.DeviceGNNPolicyPopulation(graphs, A, None, sds)
    lrn = Pop(pop, cfgs)
    twins = {}
    for k in compare:
        tenv = _env(graphs, b, J, _rows(script, k * b, (k + 1) * b))
        tpol = P.DeviceGNNPolicy(graphs, A, None, sds[k])
        twins[k] = (tenv, tpol, Single(tpol, cfgs[k]))
    seen = dict(traj=[], stats=[], vtrace=[], ctas=pop.embed_ctas())
    for it in range(3):
        seeds = [1000 * it + 3 * k for k in range(K)]
        traj = {key: np.array(v) for key, v in pop.collect(env, H, seed=seeds).items()}
        stats = lrn.learn(env, H)
        vts = {}
        for k, (tenv, tpol, tlrn) in twins.items():
            tt = tpol.collect(tenv, H, seed=seeds[k])
            for key in ('action', 'reward', 'done', 'logp'):
                assert np.array_equal(traj[key][:, k * b:(k + 1) * b], tt[key]), (algo, it, k, key)
            ts = tlrn.learn(tenv, H)
            assert stats[k] == ts, (algo, it, k, stats[k], ts)
            if algo == 'impala':
                mine, want = lrn.vtrace(k), tlrn.vtrace()
                assert mine.keys() == want.keys()
                for key in want:
                    assert np.array_equal(mine[key], want[key]), (algo, it, k, key)
                vts[k] = mine
        seen['traj'].append(traj)
        seen['stats'].append(stats)
        seen['vtrace'].append(vts)
    for k, (tenv, tpol, tlrn) in twins.items():
        assert np.array_equal(pop.get_weights(k), tpol.get_weights()), (algo, k)
        m, v, step = lrn.adam_state(k)
        tm, tv, tstep = tlrn.adam_state()
        assert np.array_equal(m, tm) and np.array_equal(v, tv) and step == tstep, (algo, k, step, tstep)
        seen.setdefault('steps', {})[k] = step
    for tenv, tpol, _ in twins.values():
        tpol.close()
    pop.close()
    return seen


IMPALA_CASES = {
    # name: K, b, horizon, jobs per episode, job types, rollout_fragment_length, train_batch_size, vary hyperparameters, early group
    'L_is_horizon': dict(K=2, b=4, H=8, J=6, kinds=('resnet',), L=0, tbs=200, vary=False),
    'L_divides_horizon': dict(K=3, b=4, H=8, J=6, kinds=('resnet',), L=4, tbs=8, vary=False),
    'short_last_batch': dict(K=2, b=5, H=8, J=6, kinds=('resnet',), L=4, tbs=12, vary=True),
    'one_fragment_per_step': dict(K=2, b=3, H=6, J=5, kinds=('resnet',), L=2, tbs=3, vary=True),
    'ends_mid_fragment': dict(K=2, b=4, H=8, J=6, kinds=('resnet',), L=4, tbs=8, vary=True, early=0),
    'two_types': dict(K=4, b=3, H=8, J=6, kinds=('resnet', 'gpt2'), L=4, tbs=12, vary=True),
    'hparams_rho_clipped': dict(K=4, b=4, H=8, J=6, kinds=('resnet',), L=4, tbs=8, vary=True),
    'grid_loops': dict(K=None, b=1, H=8, J=6, kinds=('resnet',), L=4, tbs=4, vary=True, compare='ends'),
}


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize('name', list(IMPALA_CASES))
def test_impala_population_matches_its_twins(name):
    c = dict(IMPALA_CASES[name])
    K = c['K'] or 2 * _sms() + 8                                          # K n_models > 2 SMs: the embedding CTAs loop
    b, H = c['b'], c['H']
    cfgs = _impala_configs(K, c['L'], c['tbs'], c['vary'])
    compare = [0, K // 2, K - 1] if c.get('compare') == 'ends' else None
    seen = _twin_run('impala', K, b, H, c['J'], c['kinds'], cfgs, early=c.get('early'), compare=compare)
    L = c['L'] or H
    n_frag = (H // L) * b
    F = min(c['tbs'] // L, n_frag)
    n_sgd = -(-n_frag // F)
    assert all(s['sgd_steps'] == n_sgd for st in seen['stats'] for s in st)
    if name == 'L_is_horizon':
        assert L == H and n_sgd == 1
    if name == 'L_divides_horizon':
        assert L < H and H % L == 0 and n_frag % F == 0 and n_sgd > 1
    if name == 'short_last_batch':
        assert n_frag % F, 'the last train batch must be short'
    if name == 'one_fragment_per_step':
        assert F == 1 and n_sgd == n_frag
    if name == 'ends_mid_fragment':
        done = np.concatenate([t['done'][:, :b] for t in seen['traj']], axis=1)    # the early group's columns
        t_end = [int(np.argmax(done[:, e])) for e in range(done.shape[1]) if done[:, e].any()]
        assert any(t % L != L - 1 for t in t_end), t_end
    if name == 'two_types':
        assert len(np.unique(np.concatenate([t['model'][t['model'] >= 0] for t in seen['traj']]))) == 2
    if name == 'hparams_rho_clipped':
        # set 1's clip_rho 0.8: on a later SGD step (rows past the first train batch) the weights moved and some rho exceeds it
        mb = F * L
        clipped = [np.exp(vt[1]['log_rho'][mb:]) > 0.8 for vt in seen['vtrace']]
        assert any(c.any() for c in clipped)
    if name == 'grid_loops':
        assert K > 2 * _sms() and K > seen['ctas'], (K, seen['ctas'])


PG_CASES = {
    'hparams': dict(K=3, b=4, H=8, J=6, kinds=('resnet',), vary=True),
    'one_group_ends_early': dict(K=3, b=4, H=8, J=6, kinds=('resnet',), vary=True, early=1),
    'two_types': dict(K=4, b=3, H=8, J=6, kinds=('resnet', 'gpt2'), vary=True),
    'grid_loops': dict(K=None, b=1, H=8, J=6, kinds=('resnet',), vary=True, compare='ends'),
}


@pytest.mark.parametrize('name', list(PG_CASES))
def test_pg_population_matches_its_twins(name):
    c = dict(PG_CASES[name])
    K = c['K'] or 2 * _sms() + 8
    cfgs = _pg_configs(K, c['vary'])
    compare = [0, K // 2, K - 1] if c.get('compare') == 'ends' else None
    seen = _twin_run('pg', K, c['b'], c['H'], c['J'], c['kinds'], cfgs, early=c.get('early'), compare=compare)
    if name == 'hparams':
        assert len({s['grad_gnorm'] for s in seen['stats'][0]}) == K
    if name == 'one_group_ends_early':
        g = c['early']
        for st in seen['stats']:
            rows = [int(s['rows']) for s in st]
            assert all(rows[g] < rows[k] for k in range(K) if k != g), rows          # its loss is averaged over fewer rows
    if name == 'two_types':
        assert len(np.unique(np.concatenate([t['model'][t['model'] >= 0] for t in seen['traj']]))) == 2
    if name == 'grid_loops':
        assert K > 2 * _sms() and K > seen['ctas'], (K, seen['ctas'])


def test_ppo_then_impala_then_pg_continue_one_adam_state():
    """one population runs a PPO, an IMPALA and a PG learn call; each twin runs the three single learners on one policy, whose
    Adam state they share"""
    from ddls_b200 import workload
    from ddls_b200 import policy as P
    from ddls_b200 import learn
    K, b, H, J = 3, 4, 8, 6
    graphs = [workload.make_graph('resnet')]
    script = _script(K * b, J, 1, seed=5)
    sds = [P.random_state_dict(P.DEFAULT_CONFIG, A, seed=40 + k) for k in range(K)]
    ppo = [learn.PPOConfig(sgd_minibatch_size=16, num_sgd_iter=2, seed=k, lr=[3e-4, 1e-3, 5e-5][k]) for k in range(K)]
    imp = _impala_configs(K, 4, 8, True)
    pg = _pg_configs(K, True)
    env = _env(graphs, K * b, J, script)
    pop = P.DeviceGNNPolicyPopulation(graphs, A, None, sds)
    plrn = [learn.DevicePopulationPPOLearner(pop, ppo), learn.DevicePopulationIMPALALearner(pop, imp), learn.DevicePopulationPGLearner(pop, pg)]
    twins = []
    for k in range(K):
        tenv = _env(graphs, b, J, _rows(script, k * b, (k + 1) * b))
        tpol = P.DeviceGNNPolicy(graphs, A, None, sds[k])
        twins.append((tenv, tpol, [learn.DevicePPOLearner(tpol, ppo[k]), learn.DeviceIMPALALearner(tpol, imp[k]), learn.DevicePGLearner(tpol, pg[k])]))
    steps = []
    for i in range(3):
        seeds = [100 * i + k for k in range(K)]
        pop.collect(env, H, seed=seeds)
        stats = plrn[i].learn(env, H)
        steps.append(plrn[0].adam_state(0)[2])
        for k, (tenv, tpol, tl) in enumerate(twins):
            tpol.collect(tenv, H, seed=seeds[k])
            assert stats[k] == tl[i].learn(tenv, H), (i, k)
    for k, (tenv, tpol, tl) in enumerate(twins):
        assert np.array_equal(pop.get_weights(k), tpol.get_weights()), k
        for lr in plrn:                                                   # one Adam state per set, whichever learner reads it
            m, v, step = lr.adam_state(k)
            tm, tv, tstep = tl[0].adam_state()
            assert np.array_equal(m, tm) and np.array_equal(v, tv) and step == tstep, (k, step, tstep)
        tpol.close()
    # set 0's count: PPO's minibatch steps, then IMPALA's 4 SGD steps (8 fragments, 2 per train batch), then PG's one step
    assert steps[0] > 0 and steps[1] == steps[0] + 4 and steps[2] == steps[1] + 1, steps
    pop.close()


def test_population_impala_pg_give_back_every_byte():
    from ddls_b200 import engine, workload
    from ddls_b200 import policy as P
    from ddls_b200 import learn
    graphs = [workload.make_graph('resnet')]
    env = _env(graphs, 4, 4, _script(4, 4, 1, seed=3))

    def lifecycle(check):
        pop = P.DeviceGNNPolicyPopulation(graphs, A, None, [P.random_state_dict(P.DEFAULT_CONFIG, A, seed=s) for s in (1, 2)])
        imp = learn.DevicePopulationIMPALALearner(pop, _impala_configs(2, 2, 4, True))
        pg = learn.DevicePopulationPGLearner(pop, _pg_configs(2, True))
        pop.collect(env, 4, seed=[5, 6])
        imp.learn(env, 4)
        imp.vtrace(1)
        pop.collect(env, 4, seed=[7, 8])
        pg.learn(env, 4)
        check()
        pop.close()

    lifecycle(lambda: None)
    gc.collect()
    base = engine.device_bytes()
    lifecycle(lambda: engine.device_bytes()[0] > base[0] or pytest.fail('the population holds no device memory'))
    gc.collect()
    assert engine.device_bytes() == base
