"""CPU: the oracle's batch driver in the form the GPU tests compare the bench's workloads against
(orc_run_scripted_rjpe_full_batch), and the host restatement of the episode-end finalisation.

- The full driver equals the bench's driver (orc_run_scripted_rjpe_batch) on the rows both write, and equals OracleEnv stepped from
  Python one RampJobPartitioningEnvironment.step at a time (the action step, then Action() until a job is queued or the episode is
  done): every cluster step's row, the cluster-step counts, every job record and the final episode state.
- tests/episode_stats_reference.py applied to the oracle's rows of the 16 golden episodes gives the reference's recorded es_*
  statistics, so that the GPU tests can hold ramp_get_episode_stats to it bit for bit."""
import numpy as np
import pytest

from episode_stats_reference import ES_FIELDS, episode_stats
from golden_io import Golden
from test_gpu_episode_stats import SCALARS

FILES = ['chain8', 'chain8_busy', 'chain8_maxtime', 'residual8_deg4', 'mixed16', 'res16_flood', 'tfm32_acceptable', 'residual32_deg16',
         'resnet32_cfg2', 'mixed64_busy', 'resnet64_deg2_full', 'resnet64_deg4_full', 'resnet64_deg8_full', 'resnet64_deg16_full',
         'mix128_exp', 'bert256_shard']


def oracle_script(wl):
    """A workload's [L, B] action rows as the oracle driver's [B, L] template ids (indices into wl.templates) and mount rows."""
    from oracle import oracle
    tid = np.ascontiguousarray(wl.actions['template_id'].T, dtype=np.int32)
    mount = np.zeros(tid.shape, dtype=oracle.MOUNT_DTYPE)
    for f in oracle.MOUNT_DTYPE.names:
        mount[f] = wl.actions[f].T
    return tid, mount


def run_oracle(wl, n_threads=None):
    """Every episode of a workload through orc_run_scripted_rjpe_full_batch, as bench.py's CPU arm sets it up."""
    from oracle import oracle
    tid, mount = oracle_script(wl)
    return oracle.run_scripted_episodes(wl.templates, tid, mount, wl.arrivals, wl.shape.n_workers, max(wl.template_model) + 1,
                                        n_threads=n_threads)


def oracle_jcts(templates):
    from oracle import oracle
    return [oracle.run_lookahead(t, trace_cap=0)['jct'] for t in templates]


@pytest.mark.parametrize('config,B', [('cfg1-chain-8w', 384), ('cfg3-resnet50-64w', 256)])
def test_full_driver_equals_the_bench_driver_and_python_stepping(config, B, oracle_lib):
    from ddls_b200 import workload
    from oracle.oracle import MOUNT_DTYPE, SS, STEP_STATS_LEN, CLoweredJob, lib, to_c
    import copy
    from ddls_b200.lowered import MountScalars
    wl = workload.generate(config, oracle_jcts, n_episodes=B, n_steps=8, seed=3, run_times='one_to_one')
    L = wl.n_steps
    out = run_oracle(wl, n_threads=4)

    # the bench's driver on the same script: the same action-step rows (done after the whole env-step) and job records
    tid, mount = oracle_script(wl)
    stats = np.zeros((B, L, STEP_STATS_LEN))
    rec = np.zeros((B, L), dtype=oracle_lib.JOB_RECORD_DTYPE)
    ctemps = (CLoweredJob * len(wl.templates))(*[to_c(t) for t in wl.templates])
    assert lib().orc_run_scripted_rjpe_batch(ctemps, len(wl.templates), B, L, tid.ctypes.data, mount.ctypes.data,
                                             np.ascontiguousarray(wl.arrivals).ctypes.data, L, float('inf'), wl.shape.n_workers,
                                             max(wl.template_model) + 1, 1025, stats.ctypes.data, rec.ctypes.data, 4) == 0
    assert np.array_equal(out['stats'], stats)
    assert np.array_equal(out['records'], rec)

    # OracleEnv stepped from Python, one env-step at a time
    n_multi = n_unplaced = 0
    for b in range(B):
        env = oracle_lib.OracleEnv(wl.shape.n_workers, max_jobs=L, memo_models=max(wl.template_model) + 1)
        env.reset(wl.arrivals[b])
        rows, done = [], False
        for s in range(L):
            if done:
                assert out['n_cluster_steps'][b, s] == 0 and out['stats'][b, s, SS['done']] == 1.0
                continue
            t = int(tid[b, s])
            job = None
            if t >= 0 and env.queued_job >= 0:
                job = copy.copy(wl.templates[t])
                m = mount[b, s]
                job.mount = MountScalars(*[m[f].item() for f in MOUNT_DTYPE.names])
            n_unplaced += t < 0
            first = env.step(job)
            rows.append(first)
            last = first
            while env.queued_job < 0 and last[SS['done']] == 0.0:
                last = env.step(None)
                rows.append(last)
            n = len(rows) - int(out['n_cluster_steps'][b, :s].sum())
            assert out['n_cluster_steps'][b, s] == n, (b, s)
            n_multi += n > 1
            want = first.copy()
            want[SS['done']] = last[SS['done']]
            assert np.array_equal(out['stats'][b, s], want), (b, s)
            done = last[SS['done']] != 0.0
        assert done, b
        assert out['n_cluster_stats'][b] == len(rows)
        assert np.array_equal(out['cluster_stats'][b, :len(rows)], np.array(rows)), b
        assert np.array_equal(out['records'][b], env.job_records()), b
        assert np.array_equal(out['episode_state'][b], env.episode_state()), b
    # the script reaches fused Action() steps, and its first-fit allocator leaves decisions unplaced
    assert n_multi > 0 and n_unplaced > 0


def test_full_driver_does_not_step_a_finished_episode(oracle_lib):
    """Env-steps past the end of the episode run no cluster step and leave the state as it was."""
    from ddls_b200 import workload
    from oracle.oracle import EP, SS
    wl = workload.generate('cfg1-chain-8w', oracle_jcts, n_episodes=32, n_steps=4, seed=1, run_times='one_to_one')
    short = run_oracle(wl)
    tid, mount = oracle_script(wl)
    tid2 = np.concatenate([tid, np.full_like(tid, -1)], axis=1)
    mount2 = np.concatenate([mount, mount], axis=1)
    from oracle import oracle
    long = oracle.run_scripted_episodes(wl.templates, tid2, mount2, wl.arrivals, wl.shape.n_workers, 1)
    assert (short['episode_state'][:, EP['done']] == 1).all()
    assert np.array_equal(long['stats'][:, :4], short['stats'])
    assert (long['n_cluster_steps'][:, 4:] == 0).all()
    tail = long['stats'][:, 4:]
    assert (tail[..., SS['done']] == 1).all()
    assert np.array_equal(tail[..., SS['step_counter']], np.repeat(short['episode_state'][:, None, EP['step_counter']], 4, axis=1))
    rest = np.delete(tail, [SS['done'], SS['step_counter'], SS['job_queue_length']], axis=2)
    assert (rest == 0).all()
    for k in ('episode_state', 'records', 'n_cluster_stats'):
        assert np.array_equal(long[k], short[k]), k
    cap = short['cluster_stats'].shape[1]
    assert np.array_equal(long['cluster_stats'][:, :cap], short['cluster_stats']) and (long['cluster_stats'][:, cap:] == 0).all()


def test_full_driver_fails_when_its_cluster_step_capacity_is_exceeded(oracle_lib):
    from ddls_b200 import workload
    wl = workload.generate('cfg1-chain-8w', oracle_jcts, n_episodes=8, n_steps=8, seed=0, run_times='one_to_one')
    tid, mount = oracle_script(wl)
    with pytest.raises(Exception, match='status 2'):
        oracle_lib.run_scripted_episodes(wl.templates, tid, mount, wl.arrivals, wl.shape.n_workers, 1, cs_cap=7)


@pytest.mark.parametrize('fname', FILES)
def test_finalisation_equals_the_reference_episode_stats(fname, oracle_lib):
    """episode_stats_reference on the oracle's cluster-step rows of a golden episode against the es_* statistics the reference
    recorded, with tests/test_gpu_episode_stats.py::check_against_golden's tolerances and definitions."""
    from oracle.oracle import SS
    g = Golden(fname)
    env = oracle_lib.OracleEnv(g.n_cluster_workers, max_jobs=len(g.arrivals()), memo_models=max(g.n_models, 1))
    env.reset(g.arrivals(), max_simulation_run_time=g.max_sim_time)
    rows = np.array([env.step(g.step_job(s)) for s in range(g.n_steps)])
    es = episode_stats(rows, g.arrivals())
    assert list(es) == ES_FIELDS
    for k in ('num_jobs_arrived', 'num_jobs_completed', 'num_jobs_blocked'):
        assert es[k] == int(g.d['es_' + k]), (fname, k)
    assert es['done'] == 1.0, fname
    for k in SCALARS:
        assert es[k] == pytest.approx(float(g.d['es_' + k]), rel=1e-12, abs=0), (fname, k, es[k], float(g.d['es_' + k]))
    st = g.d['step_stats']
    n_ticks = st[:, SS['num_ticks']].sum()
    for k, col in (('mean_mounted_worker_utilisation_frac', 'util_mounted_sum'), ('mean_cluster_worker_utilisation_frac', 'util_cluster_sum')):
        assert es[k] == pytest.approx(st[:, SS[col]].sum() / n_ticks, rel=1e-12, abs=0), (fname, k)
    assert es['num_cluster_steps'] == g.n_steps and es['num_ticks'] == n_ticks, fname
    # the oracle's own load-rate bookkeeping agrees with the restatement's, bit for bit
    ep = env.episode_state()
    from oracle.oracle import EP
    assert es['mean_load_rate'] == ep[EP['load_rate_sum']] / ep[EP['load_rate_n']]
    assert es['episode_end_time'] == ep[EP['time']] == env.time
