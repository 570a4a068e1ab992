"""-m gpu: the step kernel's on-chip episode state, and the reset that does not drain the stream.

ramp_reset copies the caller's arrivals into a pinned staging buffer and returns without waiting for the device; the step kernel
copies each episode's scalars and running-job table into shared memory, runs the cluster steps there and writes them back.
These tests pin what a caller can observe of that:
  - a reset whose host arrivals are overwritten as soon as reset() returns, with steps enqueued right after, gives the results of
    an untouched copy; so do two resets back to back;
  - memo_stats() counts from the last reset, whether read right after it or after steps;
  - episodes that fill every row of the on-chip running-job table run against the CPU oracle, cluster step for cluster step;
  - the bench workload with every lookahead on the non-resident (warp / CTA) kernels equals the oracle.
"""
import numpy as np
import pytest

from test_gpu_bench_workloads import L, _device_actions, _oracle, _segment, _workload

pytestmark = pytest.mark.gpu

CONFIG, B, SEED = 'cfg2-resnet50-32w', 256, 0


def _run_steps(eng, on_dev):
    """L device steps enqueued back to back after whatever the caller enqueued; the host copies of what they returned."""
    import torch
    from ddls_b200 import engine
    stats = torch.full((L, B, engine.STEP_STATS_LEN), float('nan'), dtype=torch.float64, device='cuda')
    ncs = torch.full((L, B), -1, dtype=torch.int32, device='cuda')
    for p in range(L):
        eng.step_device(on_dev[p].data_ptr(), True, stats[p].data_ptr(), ncs[p].data_ptr())
    eng.sync()
    eng.check_status()
    return dict(stats=stats.cpu().numpy(), ncs=ncs.cpu().numpy(), ep=eng.episode_state(), records=eng.job_records(),
                es=eng.episode_stats(), memo=eng.memo_stats_ex())


def _assert_same(a, b):
    for k in ('stats', 'ncs', 'ep', 'es'):
        assert np.array_equal(a[k], b[k], equal_nan=True), k
    for f in a['records'].dtype.names:
        assert np.array_equal(a['records'][f], b['records'][f]), f
    assert a['memo'] == b['memo']


@pytest.fixture(scope='module')
def bench_case():
    eng, wl, tmap = _workload(CONFIG, B, SEED, 'reference')
    on_dev = _device_actions(wl, tmap)
    eng.reset(np.array(wl.arrivals))
    want = _run_steps(eng, on_dev)
    yield eng, wl, on_dev, want
    eng.close()


def _garbage(arr):
    g = np.array(arr)
    for f in g.dtype.names:
        g[f] = 12345.0 + np.arange(g.size).reshape(g.shape)
    return g


def test_reset_arrivals_overwritten_after_return(bench_case):
    eng, wl, on_dev, want = bench_case
    arr = np.array(wl.arrivals)                    # contiguous ARRIVAL_DTYPE: reset() hands this very buffer to the library
    eng.reset(arr)
    arr[...] = _garbage(arr)                       # before any step is even enqueued
    _assert_same(_run_steps(eng, on_dev), want)


def test_two_resets_back_to_back(bench_case):
    eng, wl, on_dev, want = bench_case
    eng.reset(_garbage(wl.arrivals))
    eng.reset(np.array(wl.arrivals))
    _assert_same(_run_steps(eng, on_dev), want)


def test_memo_stats_since_the_last_reset(bench_case):
    eng, wl, on_dev, want = bench_case
    _run_steps(eng, on_dev)                        # counters keep counting past the end of a segment
    eng.reset(np.array(wl.arrivals))
    assert eng.memo_stats() == dict(lookups=0, hits=0, lookaheads=0)
    assert eng.memo_stats_ex() == dict(lookups=0, hits=0, shared_hits=0, lookaheads=0)
    got = _run_steps(eng, on_dev)
    assert got['memo'] == want['memo'] and want['memo']['lookups'] > 0 and want['memo']['lookaheads'] > 0
    m = eng.memo_stats()
    assert m == {k: want['memo'][k] for k in ('lookups', 'hits', 'lookaheads')}


@pytest.mark.parametrize('lookahead_mode', ['warp', 'cta'])
def test_non_resident_route_equals_the_oracle(lookahead_mode):
    """Every lookahead on the round-1 kernels (the warp kernel, the CTA kernel): the on-chip step kernel must see their results."""
    from ddls_b200 import engine
    from ddls_b200.engine import EP
    eng, wl, tmap = _workload(CONFIG, B, SEED, 'reference', lookahead_mode=lookahead_mode)
    assert all(eng.template_info(tmap[i])['size_class'] != 2 for i in tmap)
    ref = _oracle(CONFIG, B, SEED, 'reference', wl)
    got = _segment(eng, wl, tmap, _device_actions(wl, tmap), host=False)
    keep = np.arange(engine.STEP_STATS_LEN)
    for p in range(L):
        assert np.array_equal(got['stats'][p][:, keep], ref['stats'].transpose(1, 0, 2)[p][:, keep]), p
    assert np.array_equal(got['ncs'], ref['n_cluster_steps'].T)
    assert np.array_equal(got['ep'][:, :EP['status']], ref['episode_state'][:, :EP['status']])
    assert np.array_equal(got['es'], ref['es'])
    eng.close()


@pytest.mark.parametrize('max_jobs,max_running', [(6, 0), (8, 6)])
def test_full_running_table_equals_the_oracle(max_jobs, max_running):
    """Six jobs arrive faster than any completes, so every episode ends up with six running jobs: all rows of the on-chip table
    (min(max_running, max_jobs) = 6 rows in both shapes).  Then the jobs complete one cluster step at a time, each completion
    sliding the rows after it down."""
    from ddls_b200 import engine, synth
    from ddls_b200.engine import EP, action_row
    from ddls_b200.template_builder import RampShape, build_template, original_job_totals
    from oracle import oracle
    shape = RampShape(2, 2, 2)
    g = synth.residual_small_graph()
    t = build_template(g, 4, shape)
    jct = oracle.run_lookahead(t)['jct']
    Bt, n_jobs = 64, 6
    eng = engine.RampEngine(n_episodes=Bt, n_cluster_workers=shape.n_workers, max_jobs=max_jobs, max_running=max_running)
    tid = eng.register_template(t)
    om, od = original_job_totals(g)
    arr = np.zeros((Bt, n_jobs), dtype=engine.ARRIVAL_DTYPE)
    # episode b's jobs arrive jct / (50 + b) apart: every episode stacks all six, each at its own times
    arr['interarrival'] = (jct / (50.0 + np.arange(Bt)))[:, None]
    arr['interarrival'][:, -1] = np.inf
    arr['orig_op_mem'], arr['orig_dep_size'] = om, od
    eng.reset(arr)
    envs = [oracle.OracleEnv(shape.n_workers, max_jobs=n_jobs) for _ in range(4)]
    watched = [0, 1, Bt // 2, Bt - 1]
    for env, b in zip(envs, watched):
        env.reset(arr[b])
    running, completed = [], []
    for step in range(4 * n_jobs):
        actions = eng.make_actions()
        job = t if step < n_jobs else None
        if job is not None:
            for b in range(Bt):
                action_row(actions, b, tid, t.mount)
        stats = eng.step(actions)
        eng.check_status()
        ep = eng.episode_state()
        running.append(ep[:, EP['num_running']].copy())
        completed.append(ep[:, EP['num_completed']].copy())
        for env, b in zip(envs, watched):
            ref = env.step(job)
            assert np.array_equal(stats[b], ref), (step, b, stats[b], ref)
        if (ep[:, EP['done']] == 1).all():
            break
    # five jobs run after the fifth mount; the sixth mount fills the sixth row and, with no arrival left, the same cluster step
    # runs on to the first completion
    assert (running[n_jobs - 2] == n_jobs - 1).all() and (completed[n_jobs - 2] == 0).all()
    assert (running[n_jobs - 1] == n_jobs - 1).all() and (completed[n_jobs - 1] == 1).all()
    assert (ep[:, EP['done']] == 1).all() and (ep[:, EP['num_completed']] == n_jobs).all()
    eng.close()
