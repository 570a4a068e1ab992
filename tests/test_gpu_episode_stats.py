"""-m gpu: ``episode_stats()`` of both batched environments -- RampClusterEnvironment.episode_stats (RCE:1086-1167, 1466-1540)
accumulated on the device over every cluster step, fused ones included -- against the reference's own evaluation runs: the 16
golden episodes replayed with their recorded actions must give the episode statistics the reference recorded (es_* keys)."""
import numpy as np
import pytest

from golden_io import Golden
from test_gpu_batched_env import BATCHES, SHAPES, _decisions, _graphs

pytestmark = pytest.mark.gpu

SCALARS = ['episode_start_time', 'episode_end_time', 'episode_time', 'mean_load_rate', 'blocking_rate', 'acceptance_rate',
           'compute_info_processed', 'dep_info_processed', 'flow_info_processed', 'cluster_info_processed',
           'demand_compute_info_processed', 'demand_dep_info_processed', 'demand_total_info_processed',
           'mean_compute_throughput', 'mean_dep_throughput', 'mean_flow_throughput', 'mean_cluster_throughput',
           'mean_demand_compute_throughput', 'mean_demand_dep_throughput', 'mean_demand_total_throughput',
           'mean_compute_overhead_frac', 'mean_communication_overhead_frac', 'mean_num_jobs_running', 'mean_num_mounted_workers']
LISTS = ['job_completion_time', 'job_completion_time_speedup', 'job_communication_overhead_time', 'job_computation_overhead_time',
         'jobs_completed_mean_mounted_worker_utilisation_frac', 'jobs_completed_num_mounted_workers', 'jobs_completed_num_mounted_channels',
         'jobs_completed_max_acceptable_job_completion_time']


def golden_env(names, where, max_partitions_per_op=16):
    """The environment replaying golden episodes `names` side by side (tests/test_gpu_batched_env.py's set-up), with every job's
    max acceptable JCT as the reference computed it: from the recorded mount rows for mounted jobs, from the recorded
    episode_stats for the blocked ones that never mounted.  The arrival rows are the environment's own: the load rates (RCE:364)
    and the demand_* sums read the original job's total op memory and dep size from them.  Returns (env, goldens, per-episode
    decisions)."""
    from ddls_b200 import batched
    from ddls_b200.template_builder import original_job_totals
    cls = batched.BatchedRampJobPartitioningEnvironment if where == 'host' else batched.DeviceRampJobPartitioningEnvironment
    goldens = [Golden(n) for n in names]
    catalogue = _graphs()
    graphs, seen = [], {}
    for n in names:
        for gr in catalogue[n]:
            if gr.name not in seen:
                seen[gr.name] = len(graphs)
                graphs.append(gr)
    totals = [original_job_totals(gr)[0] for gr in graphs]
    B, J = len(goldens), max(len(g.d['arrivals']) for g in goldens)
    model, gap, macc = np.zeros((B, J), dtype=np.int64), np.full((B, J), np.inf), np.full((B, J), np.nan)
    decisions = []
    for b, (n, g) in enumerate(zip(names, goldens)):
        arr = g.d['arrivals']
        for k in range(len(arr)):
            model[b, k] = [seen[gr.name] for gr in catalogue[n] if abs(totals[seen[gr.name]] - arr[k, 1]) <= 1e-9 * abs(arr[k, 1])][0]
            gap[b, k] = arr[k, 0]
        for i, k in enumerate(g.d['es_blocked_job_idxs']):
            macc[b, k] = g.d['es_jobs_blocked_max_acceptable_job_completion_time'][i]
        dec = _decisions(g)
        decisions.append(dec)
        for e, (s, a) in enumerate(dec):
            if a > 0 and int(g.d['step_tid'][s]) >= 0:
                macc[b, e] = g.d['step_mount'][s][0]
    env = cls(SHAPES[goldens[0].n_cluster_workers], graphs, n_episodes=B, jobs_per_episode=J, max_partitions_per_op=max_partitions_per_op,
              max_simulation_run_time=goldens[0].max_sim_time, script={'model': model, 'gap': gap, 'max_acceptable_jct': macc},
              apply_action_mask=False)
    return env, goldens, decisions


def set_job_counts(env, goldens):
    for b, g in enumerate(goldens):
        env.eng.set_job_count(b, len(g.d['arrivals']))


def check_against_golden(es, b, g, name):
    from ddls_b200.engine import SS
    for k in ('num_jobs_arrived', 'num_jobs_completed', 'num_jobs_blocked'):
        assert es[k][b] == int(g.d['es_' + k]), (name, k)
    assert bool(es['done'][b]), name
    for k in SCALARS:
        assert es[k][b] == pytest.approx(float(g.d['es_' + k]), rel=1e-12, abs=0), (name, k, es[k][b], float(g.d['es_' + k]))
    assert list(es['completed_job_idxs'][b]) == list(g.d['es_completed_job_idxs']), name
    assert sorted(es['blocked_job_idxs'][b]) == sorted(g.d['es_blocked_job_idxs']), name
    for k in LISTS:
        np.testing.assert_allclose(es[k][b], g.d['es_' + k], rtol=1e-6, atol=0, err_msg=f'{name} {k}')
    ref_blocked = dict(zip(g.d['es_blocked_job_idxs'].tolist(), g.d['es_jobs_blocked_max_acceptable_job_completion_time'].tolist()))
    ours = dict(zip(es['blocked_job_idxs'][b].tolist(), es['jobs_blocked_max_acceptable_job_completion_time'][b].tolist()))
    assert ours.keys() == ref_blocked.keys(), name
    for k in ours:
        assert ours[k] == pytest.approx(ref_blocked[k], rel=1e-6, abs=0), (name, k)
    # the mean over every per-tick utilisation entry of the episode, from the recorded per-step list sums and lengths
    st = g.d['step_stats']
    n_ticks = st[:, SS['num_ticks']].sum()
    for k, col in (('mean_mounted_worker_utilisation_frac', 'util_mounted_sum'), ('mean_cluster_worker_utilisation_frac', 'util_cluster_sum')):
        assert es[k][b] == pytest.approx(st[:, SS[col]].sum() / n_ticks, rel=1e-12, abs=0), (name, k)
    assert es['num_cluster_steps'][b] == g.n_steps and es['num_ticks'][b] == n_ticks, name


@pytest.mark.parametrize('where', ['host', 'device'])
@pytest.mark.parametrize('names', BATCHES, ids=lambda n: '+'.join(n))
def test_episode_stats_equal_the_reference_on_golden_episodes(names, where):
    env, goldens, decisions = golden_env(names, where)
    env.reset()
    set_job_counts(env, goldens)
    B = len(goldens)
    for e in range(max(len(d) for d in decisions)):
        env.step(np.array([decisions[b][e][1] if e < len(decisions[b]) else 0 for b in range(B)], dtype=np.int64))
    assert env.done.all()
    es = env.episode_stats()
    for b, (n, g) in enumerate(zip(names, goldens)):
        check_against_golden(es, b, g, n)
    env.close()


def _random_envs(B=512, J=7, seed=11):
    from ddls_b200 import synth
    from ddls_b200.batched import BatchedRampJobPartitioningEnvironment, DeviceRampJobPartitioningEnvironment
    graphs = [synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3), synth.chain_graph(6, 'chain6'),
              synth.transformer_like_graph(n_layers=1, name='tfm1', seed=4)]
    kw = dict(n_episodes=B, jobs_per_episode=J, seed=seed, interarrival=('exponential', 600.0))
    return BatchedRampJobPartitioningEnvironment((4, 4, 4), graphs, **kw), DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, **kw)


def _rollout(envs, J, seed=5):
    rng = np.random.default_rng(seed)
    cand = np.array([0, 1, 2, 4, 8, 16])
    obs = [e.reset() for e in envs]
    for _ in range(J):
        ok = obs[0]['action_mask'][:, cand].astype(bool)
        actions = cand[(rng.random(ok.shape) * ok).argmax(axis=1)]
        obs = [e.step(actions)[0] for e in envs]
    return [e.episode_stats() for e in envs]


def _assert_identical(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], list):
            assert len(a[k]) == len(b[k])
            for x, y in zip(a[k], b[k]):
                np.testing.assert_array_equal(x, y, err_msg=k)
        else:
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_host_and_device_episode_stats_are_identical_and_reset_clears_them():
    host, dev = _random_envs()
    es_h, es_d = _rollout([host, dev], 7)
    assert es_h['done'].all() and es_d['done'].all()
    _assert_identical(es_h, es_d)
    assert (es_h['num_jobs_completed'] > 0).any() and (es_h['num_jobs_blocked'] > 0).any()
    # a second reset and the same rollout: the accumulators, the job tables and the return start from zero again
    host.rng, dev.rng = np.random.default_rng(11), np.random.default_rng(11)
    es_h2, es_d2 = _rollout([host, dev], 7)
    _assert_identical(es_h, es_h2)
    _assert_identical(es_d, es_d2)
    host.close(); dev.close()


@pytest.mark.parametrize('where', ['host', 'device'])
def test_an_episode_whose_only_job_is_declined(where):
    """One job, declined: blocked, nothing ever runs -- every throughput, step mean and utilisation mean is 0."""
    from ddls_b200 import batched, synth
    from ddls_b200.engine import EP
    cls = batched.BatchedRampJobPartitioningEnvironment if where == 'host' else batched.DeviceRampJobPartitioningEnvironment
    env = cls((2, 2, 2), [synth.chain_graph(6, 'chain6')], n_episodes=4, jobs_per_episode=1, seed=0)
    env.reset()
    _, reward, done, _ = env.step(np.zeros(4, dtype=np.int64))
    assert done.all()
    es = env.episode_stats()
    assert (es['num_jobs_arrived'] == 1).all() and (es['num_jobs_blocked'] == 1).all() and (es['num_jobs_completed'] == 0).all()
    assert (es['blocking_rate'] == 1.0).all() and (es['acceptance_rate'] == 0.0).all()
    np.testing.assert_array_equal(es['episode_end_time'], env.eng.episode_state()[:, EP['time']])
    for k in SCALARS[6:] + ['mean_mounted_worker_utilisation_frac', 'mean_cluster_worker_utilisation_frac']:
        assert (es[k] == 0.0).all(), k
    np.testing.assert_array_equal(es['return'], reward)
    assert all(len(x) == 0 for x in es['job_completion_time']) and all(list(x) == [0] for x in es['blocked_job_idxs'])
    env.close()


def test_step_stats_and_job_records_do_not_depend_on_reading_episode_stats():
    _, dev_a = _random_envs(B=256, seed=3)
    _, dev_b = _random_envs(B=256, seed=3)
    rng = np.random.default_rng(1)
    cand = np.array([0, 1, 2, 4, 8, 16])
    oa, ob = dev_a.reset(), dev_b.reset()
    for _ in range(7):
        ok = oa['action_mask'][:, cand].astype(bool)
        actions = cand[(rng.random(ok.shape) * ok).argmax(axis=1)]
        oa, ra, _, _ = dev_a.step(actions)
        dev_a.episode_stats()
        ob, rb, _, _ = dev_b.step(actions)
        np.testing.assert_array_equal(ra, rb)
        np.testing.assert_array_equal(dev_a.last_stats, dev_b.last_stats)
        np.testing.assert_array_equal(dev_a.eng.episode_state(), dev_b.eng.episode_state())
        a, b = dev_a.eng.job_records(), dev_b.eng.job_records()
        for f in a.dtype.names:
            np.testing.assert_array_equal(a[f], b[f], err_msg=f)
    dev_a.close(); dev_b.close()
