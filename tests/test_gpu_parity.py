"""-m gpu: the CUDA path (through the C ABI, ddls_b200/libramp_b200.so) against

  (1) the committed golden fixtures produced by the unmodified reference (tests/golden/*.npz), and
  (2) the CPU oracle on the same seeded inputs, including BASELINE.json-sized templates.

Bars: integer state (tick counts, per-tick active-worker counts, job statuses, counters) bit-exact;
float timings asserted bit-exact too (np.array_equal on f64), which is stricter than the 1e-6 relative
tolerance BASELINE.json's north_star states.
"""
import numpy as np
import pytest

from conftest import golden_files
from golden_io import Golden

pytestmark = pytest.mark.gpu

FILES = golden_files()


@pytest.fixture(scope='module')
def eng_mod():
    import torch
    assert torch.cuda.is_available(), 'these tests need a CUDA device'
    from ddls_b200 import engine
    engine.load_library()
    return engine


# every lookahead kernel: one THREAD per lookahead on the symmetry quotient (the default whenever the quotient fits shared
# memory), the same kernel on the unfolded job, one CTA per lookahead
MODES = ['thread', 'thread_unfolded', 'cta']
THREAD_MODES = ['thread', 'thread_unfolded']
# every mode on a template's first launch, and the thread kernel's second route too: a later launch of a template reads the
# TemplateHints the first one recorded, keeps every list in shared memory, writes its trace in place and sums the utilisation
# inside the tick loop (the CTA kernel keeps no hints)
MODE_LAUNCHES = [pytest.param(m, 'first', id=m) for m in MODES] + [pytest.param(m, 'hinted', id=f'{m}-hinted') for m in THREAD_MODES]


def _run_all_templates(engine, templates, n_cluster_workers=64, repeat=1, mode='auto', launch='first', trace_cap=1 << 16,
                       want_info=False):
    """launch='first': one run_lookaheads (every template's first run); 'hinted': the same run once without a trace, which
    records the hints, then again with the trace -- the second run's results.  want_info: also each template's
    engine.template_info after the runs."""
    import os
    os.environ['RAMP_LOOKAHEAD_MODE'] = mode
    try:
        eng = engine.RampEngine(n_episodes=1, n_cluster_workers=n_cluster_workers, max_jobs=1, trace_cap=trace_cap)
    finally:
        os.environ.pop('RAMP_LOOKAHEAD_MODE', None)
    tids = [eng.register_template(t) for t in templates]
    ids = np.repeat(tids, repeat)
    if launch == 'hinted':
        eng.run_lookaheads(ids)
    else:
        assert launch == 'first', launch
    res, ms, tn, tt = eng.run_lookaheads(ids, want_trace=True)
    info = [eng.template_info(t) for t in tids] if want_info else None
    eng.close()
    return (res, tn, tt, info) if want_info else (res, tn, tt)


@pytest.mark.parametrize('mode,launch', MODE_LAUNCHES)
@pytest.mark.parametrize('fname', FILES)
def test_lookahead_vs_reference_golden(fname, mode, launch, eng_mod):
    """_run_lookahead RCE:379-467: (jct, comm, comp) and the whole tick trace equal the reference's, bit for bit."""
    g = Golden(fname)
    res, tn, tt = _run_all_templates(eng_mod, g.templates, g.n_cluster_workers, mode=mode, launch=launch)
    assert (res['status'] == 0).all()
    for i in range(g.n_lookaheads):
        la = g.lookahead(i)
        k = la['tid']
        T = len(la['trace_n'])
        assert res['n_ticks'][k] == T
        np.testing.assert_array_equal(tn[k, :T], la['trace_n'])
        np.testing.assert_array_equal(tt[k, :T], la['trace_tick'])
        assert res['jct'][k] == la['jct'] and res['comm'][k] == la['comm'] and res['comp'][k] == la['comp']


@pytest.mark.parametrize('mode,launch', MODE_LAUNCHES)
@pytest.mark.parametrize('fname', FILES)
def test_lookahead_vs_oracle_all_templates(fname, mode, launch, eng_mod, oracle_lib):
    """Every lowered Action in the fixtures (not only the un-memoised ones) against the CPU oracle."""
    g = Golden(fname)
    res, tn, tt = _run_all_templates(eng_mod, g.templates, g.n_cluster_workers, repeat=3, mode=mode, launch=launch)
    for k, t in enumerate(g.templates):
        o = oracle_lib.run_lookahead(t)
        for rep in range(3):
            r = res[3 * k + rep]
            assert r['status'] == o['status'] and r['n_ticks'] == o['n_ticks']
            assert r['jct'] == o['jct'] and r['comm'] == o['comm'] and r['comp'] == o['comp']
            np.testing.assert_array_equal(tn[3 * k + rep, :o['n_ticks']], o['trace_n_active'])
            np.testing.assert_array_equal(tt[3 * k + rep, :o['n_ticks']], o['trace_tick'])


@pytest.mark.parametrize('fname', FILES)
@pytest.mark.parametrize('memo_mode', [0, 1, 2, 3])
def test_episode_replay_vs_reference_golden(fname, memo_mode, eng_mod):
    """RampClusterEnvironment.step RCE:894-1179 replayed for a batch of 5 identical episodes: step_stats,
    job records and counters against the reference's own run."""
    from ddls_b200.engine import SS, STEP_STATS, JS_COMPLETED, JS_BLOCKED, action_row
    g = Golden(fname)
    B = 5
    arr = g.arrivals()
    eng = eng_mod.RampEngine(n_episodes=B, n_cluster_workers=g.n_cluster_workers, max_jobs=len(arr),
                             memo_mode=memo_mode, max_simulation_run_time=g.max_sim_time, trace_cap=1 << 16)
    tids = [eng.register_template(t) for t in g.templates]
    arrivals = np.zeros((B, len(arr)), dtype=eng_mod.ARRIVAL_DTYPE)
    for b in range(B):
        arrivals[b] = arr
    eng.reset(arrivals)
    ref = g.d['step_stats']
    exact = ['step_counter', 'num_jobs_completed', 'num_jobs_arrived', 'num_jobs_blocked', 'job_queue_length',
             'num_ticks', 'done']
    # with memo_mode != reference, results are identical only if the memoised (model, degree) lookahead equals
    # the job's own lookahead; the reference memo is lossy (RCE:271-277), so compare floats only in reference mode
    # and structure (counters) otherwise when the fixture has memo-hit steps with a different template
    for s in range(g.n_steps):
        actions = eng.make_actions()
        job = g.step_job(s)
        if job is not None:
            for b in range(B):
                action_row(actions, b, tids[int(g.d['step_tid'][s])], job.mount)
        stats = eng.step(actions)
        eng.check_status()
        if memo_mode in (0, 3):          # 3 = reference semantics + batch-wide result cache: same results, fewer lookaheads
            for b in range(B):
                for k in exact + (['lookahead_ran'] if memo_mode == 0 else []):
                    assert stats[b, SS[k]] == ref[s, SS[k]], (fname, s, b, k)
                for k in STEP_STATS:
                    if memo_mode == 3 and k == 'lookahead_ran':
                        continue
                    a, c = stats[b, SS[k]], ref[s, SS[k]]
                    assert a == pytest.approx(c, rel=1e-6, abs=0), (fname, s, b, k, a, c)
        else:
            cols = [i for k, i in SS.items() if k != 'lookahead_ran']   # in exact mode one episode per key runs it
            assert (stats[:, cols] == stats[0, cols]).all()
    if memo_mode == 3:
        m = eng.memo_stats_ex()
        assert m['lookaheads'] <= g.n_lookaheads            # 5 episodes share what one reference env ran
        assert m['shared_hits'] >= (B - 1) * m['lookaheads']
    if memo_mode not in (0, 3):
        eng.close()
        return
    rec = eng.job_records()
    st = eng.episode_state()
    for b in range(B):
        r = rec[b]
        order = np.argsort(r['event_seq'], kind='stable')
        completed = [int(i) for i in order if r['status'][i] == JS_COMPLETED]
        blocked = [int(i) for i in order if r['status'][i] == JS_BLOCKED]
        assert completed == list(g.d['es_completed_job_idxs'])
        assert sorted(blocked) == sorted(g.d['es_blocked_job_idxs'])
        jct = r['time_completed'][completed] - r['time_arrived'][completed]
        np.testing.assert_allclose(jct, g.d['es_job_completion_time'], rtol=1e-6, atol=0)
        np.testing.assert_allclose(r['comm'][completed], g.d['es_job_communication_overhead_time'], rtol=1e-6, atol=0)
        np.testing.assert_allclose(r['comp'][completed], g.d['es_job_computation_overhead_time'], rtol=1e-6, atol=0)
        np.testing.assert_allclose(r['util'][completed], g.d['es_jobs_completed_mean_mounted_worker_utilisation_frac'],
                                   rtol=1e-6, atol=0)
        assert st[b, eng_mod.EP['num_arrived']] == int(g.d['es_num_jobs_arrived'])
        assert st[b, eng_mod.EP['num_completed']] == int(g.d['es_num_jobs_completed'])
        assert st[b, eng_mod.EP['num_blocked']] == int(g.d['es_num_jobs_blocked'])
        mlr = st[b, eng_mod.EP['load_rate_sum']] / st[b, eng_mod.EP['load_rate_n']]
        assert mlr == pytest.approx(float(g.d['es_mean_load_rate']), rel=1e-6)
    eng.close()


@pytest.mark.parametrize('shape', ['roomy', 'cta'])
@pytest.mark.parametrize('fname', FILES)
def test_episode_replay_vs_oracle_bit_exact(fname, shape, eng_mod, oracle_lib):
    """Same replay, CUDA vs CPU oracle: every step_stats entry and job record identical (bit-exact f64).  'cta' makes no
    template resident, so every step's lookaheads take the non-resident route: the work-count read-back and the CTA kernel."""
    import os
    from ddls_b200.engine import action_row
    g = Golden(fname)
    arr = g.arrivals()
    env = oracle_lib.OracleEnv(g.n_cluster_workers, max_jobs=len(arr), memo_models=max(g.n_models, 1))
    env.reset(arr, max_simulation_run_time=g.max_sim_time)
    if shape == 'cta':
        os.environ['RAMP_LOOKAHEAD_MODE'] = 'cta'
    try:
        eng = eng_mod.RampEngine(n_episodes=2, n_cluster_workers=g.n_cluster_workers, max_jobs=len(arr),
                                 max_simulation_run_time=g.max_sim_time, trace_cap=1 << 16)
    finally:
        os.environ.pop('RAMP_LOOKAHEAD_MODE', None)
    tids = [eng.register_template(t) for t in g.templates]
    eng.reset(np.stack([arr, arr]))
    for s in range(g.n_steps):
        job = g.step_job(s)
        o = env.step(job)
        actions = eng.make_actions()
        if job is not None:
            for b in range(2):
                action_row(actions, b, tids[int(g.d['step_tid'][s])], job.mount)
        stats = eng.step(actions)
        np.testing.assert_array_equal(stats[0], o)
        np.testing.assert_array_equal(stats[1], o)
    rec = eng.job_records()
    orec = env.job_records()
    for f in orec.dtype.names:
        np.testing.assert_array_equal(rec[0][f], orec[f])
    eng.close()


def test_fused_empty_steps_match_separate_steps(eng_mod):
    """RJPE:394-395 loop fused on the device == issuing Action() steps one by one."""
    from ddls_b200.engine import action_row, SS, EP
    g = Golden('chain8')
    arr = g.arrivals()
    B = 3
    def make():
        e = eng_mod.RampEngine(n_episodes=B, n_cluster_workers=g.n_cluster_workers, max_jobs=len(arr),
                               max_simulation_run_time=g.max_sim_time, trace_cap=1 << 16)
        t = [e.register_template(x) for x in g.templates]
        e.reset(np.stack([arr] * B))
        return e, t
    e1, t1 = make()
    e2, t2 = make()
    s = 0
    while s < g.n_steps:
        job = g.step_job(s)
        a = e1.make_actions()
        if job is not None:
            for b in range(B):
                action_row(a, b, t1[int(g.d['step_tid'][s])], job.mount)
        st1 = e1.step(a)
        s += 1
        n_empty = 0
        while s < g.n_steps and g.step_job(s) is None and int(g.d['step_tid'][s]) < 0 and \
                st1[0, SS['job_queue_length']] == 0 and st1[0, SS['done']] == 0:
            st1 = e1.step(e1.make_actions())
            s += 1
            n_empty += 1
        st2, ncs = e2.step(a, fuse_empty_steps=True, want_cluster_steps=True)
        assert (ncs == 1 + n_empty).all()
        np.testing.assert_array_equal(e1.episode_state(), e2.episode_state())
    for f in e1.job_records().dtype.names:
        np.testing.assert_array_equal(e1.job_records()[f], e2.job_records()[f])
    e1.close(); e2.close()


def zero_jct_template():
    """Every op zero-cost and every flow zero-time: jct == 0, so hint_jct == 0 and a hinted launch sums no utilisation
    in its tick loop (the reference would divide by zero computing it, RCE:832; only the lookahead is run here)."""
    from ddls_b200.lowered import LoweredJob, MountScalars
    # op 0 -> op 1 (flow on channel 0, run time 0) and op 0 -> op 2 (non-flow), op 1 -> op 2 (flow); two workers
    return LoweredJob(n_ops=3, n_deps=3, n_workers=2, n_channels=1, num_training_steps=2, model_id=0, degree=1,
                      op_cost=np.zeros(3), op_prio=np.array([2, 1, 0]), op_worker=np.array([0, 1, 0]),
                      op_n_parents=np.array([0, 1, 2]), row_ptr=np.array([0, 2, 3, 3]), dep_dst=np.array([1, 2, 2]),
                      dep_run_time=np.zeros(3), dep_prio=np.array([0, 1, 2]), dep_channel=np.array([0, 0xFFFF, 0]),
                      dep_is_flow=np.array([1, 0, 1]), mount=MountScalars(n_mounted_workers=2)).canonicalise()


@pytest.mark.parametrize('mode,launch', MODE_LAUNCHES)
def test_random_templates_vs_oracle(mode, launch, eng_mod, oracle_lib):
    """Adversarial random lowered jobs: priority ties, zero-cost ops, zero-time flows, flows without a channel,
    mutual edges, deadlocks (status INFINITE_TICK must match too), and a job whose completion time is 0."""
    from ddls_b200.template_builder import random_dag_template
    rng = np.random.default_rng(1234)
    templates = [random_dag_template(rng, int(n), n_workers=int(w)) for n, w in
                 zip(rng.integers(2, 400, size=60), rng.integers(1, 9, size=60))]
    templates.append(zero_jct_template())
    res, tn, tt = _run_all_templates(eng_mod, templates, mode=mode, launch=launch)
    assert res['jct'][-1] == 0.0 and res['status'][-1] == 0
    n_err = 0
    for k, t in enumerate(templates):
        o = oracle_lib.run_lookahead(t)
        assert res['status'][k] == o['status'], k
        assert res['n_ticks'][k] == o['n_ticks'], k
        np.testing.assert_array_equal(tn[k, :o['n_ticks']], o['trace_n_active'])
        np.testing.assert_array_equal(tt[k, :o['n_ticks']], o['trace_tick'])
        if o['status'] == 0:
            assert res['jct'][k] == o['jct'] and res['comm'][k] == o['comm'] and res['comp'][k] == o['comp']
        else:
            n_err += 1
    assert n_err < len(templates)


@pytest.mark.parametrize('mode,launch', MODE_LAUNCHES)
@pytest.mark.parametrize('degree', [2, 4, 8, 16])
def test_baseline_sized_template_vs_oracle(degree, mode, launch, eng_mod, oracle_lib):
    """BASELINE.json config 2/3 shape: ResNet-50-like job partitioned to `degree` on a 64-worker RAMP."""
    from ddls_b200 import synth
    from ddls_b200.template_builder import build_template, RampShape
    t = build_template(synth.resnet_like_graph(), degree, RampShape(4, 4, 4))
    o = oracle_lib.run_lookahead(t)
    res, tn, tt = _run_all_templates(eng_mod, [t], repeat=8, mode=mode, launch=launch)
    for rep in range(8):
        assert res['status'][rep] == 0 and res['n_ticks'][rep] == o['n_ticks']
        assert res['jct'][rep] == o['jct'] and res['comm'][rep] == o['comm'] and res['comp'][rep] == o['comp']
        np.testing.assert_array_equal(tn[rep, :o['n_ticks']], o['trace_n_active'])
        np.testing.assert_array_equal(tt[rep, :o['n_ticks']], o['trace_tick'])


def test_infinite_tick_raises_like_reference(eng_mod):
    """A deadlocked job graph raises the reference's message (RCE:462) through the C ABI."""
    from ddls_b200.lowered import LoweredJob, MountScalars
    from ddls_b200.engine import action_row
    # op 1 waits for a parent dep that can never start because op 0 -> 1 and 1 -> 0 are mutual edges and 1 has no other parent
    t = LoweredJob(n_ops=2, n_deps=2, n_workers=1, n_channels=0, num_training_steps=1, model_id=0, degree=2,
                   op_cost=np.array([1.0, 1.0]), op_prio=np.array([0, 1]), op_worker=np.array([0, 0]),
                   op_n_parents=np.array([0, 0]), row_ptr=np.array([0, 1, 2]), dep_dst=np.array([1, 0]),
                   dep_run_time=np.array([0.0, 0.0]), dep_prio=np.array([0, 0]), dep_channel=np.array([0xFFFF, 0xFFFF]),
                   dep_is_flow=np.array([0, 0]), mount=MountScalars(n_mounted_workers=1)).canonicalise()
    eng = eng_mod.RampEngine(n_episodes=1, n_cluster_workers=8, max_jobs=2)
    tid = eng.register_template(t)
    arr = np.zeros((1, 2), dtype=eng_mod.ARRIVAL_DTYPE)
    arr['interarrival'] = [[10.0, np.inf]]
    eng.reset(arr)
    a = eng.make_actions()
    action_row(a, 0, tid, t.mount)
    eng.step(a)
    with pytest.raises(Exception, match='Last tick was infinite'):
        eng.check_status()
    eng.close()


@pytest.mark.parametrize('mode,cta_threads', [('cta', '0'), ('cta', '64'), ('cta', '128'), ('cta', '256'), ('auto', '0'),
                                               ('thread_unfolded', '0')])
def test_many_mixed_items_per_launch(mode, cta_threads, eng_mod, oracle_lib):
    """Hundreds of lookaheads of four very different sizes in one launch, persistent CTAs processing several items each:
    every result equals the oracle's (this configuration once exposed a shared-memory race in the CTA kernel).  ('cta', '0')
    leaves the thread count to the launch rule: 6,000 items are more than one wave, so they run on persistent 64-thread CTAs."""
    import os
    from ddls_b200 import synth
    from ddls_b200.template_builder import build_template, RampShape
    g = synth.resnet_like_graph(n_blocks=4, name='res4')
    ts = [build_template(g, d, RampShape(4, 4, 4)) for d in (2, 4, 8, 16)]
    want = [oracle_lib.run_lookahead(t) for t in ts]
    os.environ['RAMP_LOOKAHEAD_MODE'] = mode
    if cta_threads != '0':
        os.environ['RAMP_LOOKAHEAD_CTA_THREADS'] = cta_threads
    try:
        eng = eng_mod.RampEngine(n_episodes=1, n_cluster_workers=64, max_jobs=1, trace_cap=4096)
    finally:
        os.environ.pop('RAMP_LOOKAHEAD_MODE', None)
        os.environ.pop('RAMP_LOOKAHEAD_CTA_THREADS', None)
    tids = [eng.register_template(t) for t in ts]
    rng = np.random.default_rng(7)
    for n in (700, 2500, 6000):
        pick = rng.integers(0, 4, size=n)
        res, _ = eng.run_lookaheads(np.array(tids, dtype=np.int32)[pick])
        assert (res['status'] == 0).all()
        for d in range(4):
            sel = pick == d
            assert (res['jct'][sel] == want[d]['jct']).all() and (res['comm'][sel] == want[d]['comm']).all()
            assert (res['comp'][sel] == want[d]['comp']).all() and (res['n_ticks'][sel] == want[d]['n_ticks']).all()
    eng.close()


@pytest.mark.parametrize('mode', ['warp', 'dense'])
def test_unknown_lookahead_mode_fails_engine_creation(mode, eng_mod):
    """RAMP_LOOKAHEAD_MODE names a route (auto or thread, thread_unfolded, cta); any other value, such as warp, fails
    engine creation instead of quietly running the automatic route."""
    import os
    os.environ['RAMP_LOOKAHEAD_MODE'] = mode
    try:
        with pytest.raises(Exception, match='RAMP_LOOKAHEAD_MODE'):
            eng_mod.RampEngine(n_episodes=1, n_cluster_workers=8, max_jobs=1)
    finally:
        os.environ.pop('RAMP_LOOKAHEAD_MODE', None)


def test_shared_memo_survives_reset_and_matches_reference_mode(eng_mod):
    """RAMP_MEMO_SHARED: second episode after ramp_reset re-uses the batch-wide cache (no lookahead runs) and every
    step-stats entry still equals the per-episode reference mode."""
    from ddls_b200.engine import action_row, SS
    g = Golden('mixed16')
    arr = g.arrivals()
    B = 4
    runs = {}
    for mode in (0, 3):
        eng = eng_mod.RampEngine(n_episodes=B, n_cluster_workers=g.n_cluster_workers, max_jobs=len(arr), memo_mode=mode,
                                 max_simulation_run_time=g.max_sim_time, trace_cap=1 << 16)
        tids = [eng.register_template(t) for t in g.templates]
        out = []
        for episode in range(2):
            eng.reset(np.stack([arr] * B))
            for s in range(g.n_steps):
                a = eng.make_actions()
                job = g.step_job(s)
                if job is not None:
                    for b in range(B):
                        action_row(a, b, tids[int(g.d['step_tid'][s])], job.mount)
                st = eng.step(a)
                out.append(np.delete(st, SS['lookahead_ran'], axis=1))
            out.append(eng.job_records()['jct'].copy())
            if mode == 3:
                m = eng.memo_stats_ex()
                if episode == 1:
                    assert m['lookaheads'] == 0 and m['lookups'] > 0
        runs[mode] = out
        eng.close()
    for a, b in zip(runs[0], runs[3]):
        np.testing.assert_array_equal(a, b)


def _fan_template(M, W, seed):
    """source -> M children -> sink on W workers: every shared-memory list of the kernels overflows into HBM when M is in
    the thousands (flow frontier, one-tick non-flow list, op frontier, readied-op queue), and the sink's in-degree M > 255
    forces the global parent counters."""
    from ddls_b200.lowered import LoweredJob, MountScalars
    rng = np.random.default_rng(seed)
    N, E = M + 2, 2 * M
    worker = np.concatenate([[0], rng.integers(0, W, size=M), [0]]).astype(np.int64)
    cost = np.concatenate([[1.0], np.round(rng.uniform(0.0, 3.0, size=M), 2), [0.5]])
    cost[1:M + 1][rng.random(M) < 0.1] = 0.0                                   # zero-cost ops complete in zero-length ticks
    row_ptr = np.concatenate([[0, M], M + 1 + np.arange(M), [E]]).astype(np.int64)   # op 0: M deps; child i: 1 dep; sink: 0
    dst = np.concatenate([1 + np.arange(M), np.full(M, M + 1)]).astype(np.int64)
    src_w = np.concatenate([np.zeros(M, dtype=np.int64), worker[1:M + 1]])
    dst_w = worker[dst]
    is_flow = (src_w != dst_w).astype(np.uint8)
    pair = src_w * W + dst_w
    chans = {p: i for i, p in enumerate(np.unique(pair[is_flow == 1]))}
    channel = np.array([chans[p] if f else 0xFFFF for p, f in zip(pair, is_flow)], dtype=np.int64)
    rt = np.where(is_flow == 1, np.round(rng.uniform(0.01, 2.0, size=E), 3), 0.0)
    rt[(is_flow == 1) & (rng.random(E) < 0.3)] = 0.25                            # many equal run times: completions in bulk
    n_par = np.concatenate([[0], np.ones(M), [M]]).astype(np.int64)
    return LoweredJob(n_ops=N, n_deps=E, n_workers=W, n_channels=len(chans), num_training_steps=3, model_id=0, degree=2,
                      op_cost=cost, op_prio=rng.integers(0, 50, size=N), op_worker=worker, op_n_parents=n_par, row_ptr=row_ptr,
                      dep_dst=dst, dep_run_time=rt, dep_prio=rng.integers(0, 20, size=E), dep_channel=channel, dep_is_flow=is_flow,
                      mount=MountScalars(n_mounted_workers=W)).canonicalise()


@pytest.mark.parametrize('mode,cta_threads,launch',
                         [pytest.param(m, c, 'first', id=f'{m}-{c}') for m, c in
                          [('cta', '64'), ('cta', '128'), ('cta', '256'), ('thread', '0'), ('thread_unfolded', '0')]]
                         + [pytest.param(m, '0', 'hinted', id=f'{m}-0-hinted') for m in THREAD_MODES])
@pytest.mark.parametrize('M,W', [(200, 4), (3000, 6)])
def test_wide_fan_overflows_every_shared_memory_list(M, W, mode, cta_threads, launch, eng_mod, oracle_lib):
    """Frontiers far beyond shared memory.  Hinted: the recorded frontiers do not fit, so the second launch must spill too."""
    import os
    t = _fan_template(M, W, seed=M)
    want = oracle_lib.run_lookahead(t)
    os.environ['RAMP_LOOKAHEAD_MODE'] = mode
    if cta_threads != '0':
        os.environ['RAMP_LOOKAHEAD_CTA_THREADS'] = cta_threads
    try:
        eng = eng_mod.RampEngine(n_episodes=1, n_cluster_workers=8, max_jobs=1, trace_cap=1 << 15)
    finally:
        os.environ.pop('RAMP_LOOKAHEAD_MODE', None)
        os.environ.pop('RAMP_LOOKAHEAD_CTA_THREADS', None)
    tid = eng.register_template(t)
    if launch == 'hinted':
        eng.run_lookaheads(np.full(5, tid, dtype=np.int32))
        h = eng.template_info(tid)
        assert (h['size_class'] == 2) == (M == 200)             # M = 3000: the quotient blob exceeds 96 KB (CTA kernel)
        if M == 200:
            assert h['n_ticks'] == want['n_ticks'] and h['max_f'] > 16
    res, _, tn, tt = eng.run_lookaheads(np.full(5, tid, dtype=np.int32), want_trace=True)
    assert (res['status'] == 0).all() and (res['n_ticks'] == want['n_ticks']).all()
    for i in range(5):
        T = int(res['n_ticks'][i])
        np.testing.assert_array_equal(tn[i, :T], want['trace_n_active'])
        np.testing.assert_array_equal(tt[i, :T], want['trace_tick'])
    assert (res['jct'] == want['jct']).all() and (res['comm'] == want['comm']).all() and (res['comp'] == want['comp']).all()
    eng.close()


def test_register_rejects_non_flow_dep_with_run_time(eng_mod):
    """RCE:542-560 zeroes every non-flow run time; with a non-zero one the reference's zero-length ticks never end."""
    t = _fan_template(20, 3, seed=1)
    k = int(np.nonzero(np.asarray(t.dep_is_flow) == 0)[0][0])
    t.dep_run_time = np.array(t.dep_run_time, dtype=np.float64)
    t.dep_run_time[k] = 0.5
    eng = eng_mod.RampEngine(n_episodes=1, n_cluster_workers=8, max_jobs=1)
    with pytest.raises(Exception, match='non-flow dep'):
        eng.register_template(t)
    eng.close()


@pytest.mark.parametrize('cta_threads,M', [('128', 4500), ('256', 9000)])
def test_op_frontier_larger_than_a_cta_can_mask(cta_threads, M, eng_mod, oracle_lib):
    """More ready ops than 32 per thread of the CTA (the per-thread winner bit mask runs out: the kernel falls back to
    re-reading the per-worker arg-max slots and clears them with an extra pass)."""
    import os
    t = _fan_template(M, 6, seed=M)
    want = oracle_lib.run_lookahead(t)
    os.environ['RAMP_LOOKAHEAD_MODE'] = 'cta'
    os.environ['RAMP_LOOKAHEAD_CTA_THREADS'] = cta_threads
    try:
        eng = eng_mod.RampEngine(n_episodes=1, n_cluster_workers=8, max_jobs=1, trace_cap=1 << 15)
    finally:
        os.environ.pop('RAMP_LOOKAHEAD_MODE', None)
        os.environ.pop('RAMP_LOOKAHEAD_CTA_THREADS', None)
    tid = eng.register_template(t)
    res, _ = eng.run_lookaheads(np.full(3, tid, dtype=np.int32))
    assert (res['status'] == 0).all() and (res['n_ticks'] == want['n_ticks']).all()
    assert (res['jct'] == want['jct']).all() and (res['comm'] == want['comm']).all() and (res['comp'] == want['comp']).all()
    eng.close()
