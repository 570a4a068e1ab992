"""-m gpu: the workloads bench.py times, run the way it runs them, against the CPU oracle episode for episode.

Scripted arm: each config's templates, JCTs and scripts are built as ``run_b200_arm`` builds them (the engine created with
``max_jobs=L, trace_cap=4096``, the JCTs from its own ``run_lookaheads``), then two segments run as ``device_step`` runs them:
``reset``, L x ``step_device`` with device-resident action rows, fused empty steps and the statistics written to device buffers with
no host synchronisation in between, then ``export_episode_state_to``.  Every env-step's statistics row, the cluster-step counts,
the job records, the episode-state rows and ``ramp_get_episode_stats`` must be bit-identical to
``orc_run_scripted_rjpe_full_batch`` on the same templates, script and arrivals, and to tests/episode_stats_reference.py's
finalisation of the oracle's cluster-step rows.  The second segment runs on the hints the first recorded and must reproduce it.

Batched-environment arm: DeviceRampJobPartitioningEnvironment (prewarmed) and BatchedRampJobPartitioningEnvironment with the bench's
arguments and its stand-in agent, side by side for two segments; the host environment's lowered jobs and action rows are replayed
through the same oracle driver."""
import os

import numpy as np
import pytest

from episode_stats_reference import as_row, episode_stats
from test_oracle_bench_driver import oracle_script

pytestmark = pytest.mark.gpu

L = 8
SEGMENTS = 2
_ORACLE = {}


def _workload(config, B, seed, run_times, memo_mode=0, lookahead_mode=None):
    """The engine and workload exactly as bench.py's run_b200_arm builds them, plus the template ids in engine numbering."""
    from ddls_b200 import engine, workload
    from oracle import oracle
    cfg = workload.CONFIGS[config]
    if lookahead_mode:
        os.environ['RAMP_LOOKAHEAD_MODE'] = lookahead_mode
    try:
        eng = engine.RampEngine(n_episodes=B, n_cluster_workers=int(np.prod(cfg['shape'])), max_jobs=L, memo_mode=memo_mode,
                                trace_cap=4096)
    finally:
        os.environ.pop('RAMP_LOOKAHEAD_MODE', None)
    tmap = {}

    def engine_jcts(templates):
        for i, t in enumerate(templates):
            tmap[i] = eng.register_template(t)
        res, _ = eng.run_lookaheads([tmap[i] for i in range(len(templates))])
        assert (res['status'] == 0).all()
        return res['jct']
    wl = workload.generate(config, engine_jcts, n_episodes=B, n_steps=L, seed=seed, run_times=run_times)
    jct_dev = eng.run_lookaheads([tmap[i] for i in range(len(wl.templates))])[0]['jct']
    jct_orc = np.array([oracle.run_lookahead(t, trace_cap=0)['jct'] for t in wl.templates])
    assert np.array_equal(jct_dev, jct_orc), (config, jct_dev, jct_orc)
    return eng, wl, tmap


def _oracle(config, B, seed, run_times, wl):
    """The oracle's run of a workload; cached, since engine settings do not change the script (its JCTs are asserted equal)."""
    from test_oracle_bench_driver import run_oracle
    key = (config, B, seed, run_times)
    if key not in _ORACLE:
        out = run_oracle(wl)
        out['es'] = np.array([as_row(episode_stats(out['cluster_stats'][b, :out['n_cluster_stats'][b]], wl.arrivals[b]))
                              for b in range(B)])
        out['tid'], _ = oracle_script(wl)
        _ORACLE[key] = out
    out = _ORACLE[key]
    assert np.array_equal(out['tid'], oracle_script(wl)[0]), 'the workload changed between engine settings'
    return out


def _segment(eng, wl, tmap, on_dev, host):
    """One bench segment.  Returns the host copies of what the step path handed back."""
    import torch
    from ddls_b200 import engine
    B = wl.n_episodes
    eng.reset(wl.arrivals)
    if host:
        stats = np.zeros((L, B, engine.STEP_STATS_LEN))
        ncs = np.zeros((L, B), np.int32)
        for p in range(L):
            a = wl.actions[p].copy()
            placed = a['template_id'] >= 0
            a['template_id'][placed] = [tmap[int(t)] for t in a['template_id'][placed]]
            stats[p], ncs[p] = eng.step(a, fuse_empty_steps=True, want_cluster_steps=True)
        ep = torch.empty((B, engine.EP_LEN), dtype=torch.float64, device='cuda')
        eng.export_episode_state_to(ep.data_ptr())
        eng.sync()
        ep = ep.cpu().numpy()
    else:
        stats_dev = torch.full((L, B, engine.STEP_STATS_LEN), float('nan'), dtype=torch.float64, device='cuda')
        ncs_dev = torch.full((L, B), -1, dtype=torch.int32, device='cuda')
        ep_dev = torch.empty((B, engine.EP_LEN), dtype=torch.float64, device='cuda')
        torch.cuda.synchronize()
        for p in range(L):
            eng.step_device(on_dev[p].data_ptr(), True, stats_dev[p].data_ptr(), ncs_dev[p].data_ptr())
        eng.export_episode_state_to(ep_dev.data_ptr())
        eng.sync()
        stats, ncs, ep = stats_dev.cpu().numpy(), ncs_dev.cpu().numpy(), ep_dev.cpu().numpy()
    eng.check_status()
    return dict(stats=stats, ncs=ncs, ep=ep, records=eng.job_records(), es=eng.episode_stats(), memo=eng.memo_stats_ex())


CASES = [
    ('cfg1-chain-8w', 1, 0, 'reference', 0, None, False),
    ('cfg1-chain-8w', 1024, 0, 'reference', 0, None, False),
    ('cfg2-resnet50-32w', 256, 0, 'reference', 0, None, False),
    ('cfg3-resnet50-64w', 4096, 0, 'reference', 0, None, False),
    ('cfg4-bert-256w', 4096, 0, 'reference', 0, None, False),
    ('cfg5-mix-128w', 16384, 0, 'reference', 0, None, False),
    ('cfg3-resnet50-64w', 4096, 1000, 'reference', 0, None, False),
    ('cfg3-resnet50-64w', 4096, 0, 'one_to_one', 0, None, False),
    ('cfg3-resnet50-64w', 4096, 0, 'reference', 0, None, True),
] + [(c, 4096, 0, 'reference', m, None, False) for c in ('cfg3-resnet50-64w', 'cfg4-bert-256w') for m in (1, 2, 3)] \
  + [(c, 4096, 0, 'reference', 0, lm, False) for c in ('cfg3-resnet50-64w', 'cfg4-bert-256w') for lm in ('warp', 'cta', 'thread_unfolded')]


def _case_id(c):
    config, B, seed, run_times, memo, la, host = c
    return '-'.join([config.split('-')[0], f'B{B}', f's{seed}', run_times] + ([f'memo{memo}'] if memo else []) + ([la] if la else [])
                    + (['host_step'] if host else []))


@pytest.mark.parametrize('case', CASES, ids=[_case_id(c) for c in CASES])
def test_bench_workload_equals_the_oracle(case):
    from ddls_b200 import engine
    from ddls_b200.engine import EP, SS
    config, B, seed, run_times, memo_mode, lookahead_mode, host = case
    eng, wl, tmap = _workload(config, B, seed, run_times, memo_mode, lookahead_mode)
    ref = _oracle(config, B, seed, run_times, wl)
    on_dev = _device_actions(wl, tmap)
    size_class = {i: eng.template_info(tmap[i])['size_class'] for i in tmap}

    # bench.py's rows are [B][STEP_STATS_LEN] per env-step; the oracle's [B][L][...]
    want_stats = ref['stats'].transpose(1, 0, 2)
    want_ncs = ref['n_cluster_steps'].T
    exempt = [] if memo_mode == engine.MEMO_REFERENCE else [SS['lookahead_ran']]
    keep = np.setdiff1d(np.arange(engine.STEP_STATS_LEN), exempt)
    want_ep = ref['episode_state']
    segs = []
    for seg in range(SEGMENTS if not host else 1):
        got = _segment(eng, wl, tmap, on_dev, host)
        segs.append(got)
        for p in range(L):
            bad = ~(got['stats'][p][:, keep] == want_stats[p][:, keep]).all(axis=1)
            assert not bad.any(), (seg, p, int(np.nonzero(bad)[0][0]), got['stats'][p][bad][0], want_stats[p][bad][0])
        assert np.array_equal(got['ncs'], want_ncs), seg
        for f in got['records'].dtype.names:
            assert np.array_equal(got['records'][f], ref['records'][f]), (seg, f)
        assert np.array_equal(got['ep'][:, :EP['status']], want_ep[:, :EP['status']]), seg
        assert (got['ep'][:, EP['status']] == 0).all()
        assert np.array_equal(got['es'], ref['es']), (seg, np.nonzero((got['es'] != ref['es']).any(axis=0))[0])
        if seg == 0 and not lookahead_mode:
            # the second segment runs the thread kernel's hinted route: every resident template mounted has its hints now
            mounted = np.unique(ref['tid'][ref['tid'] >= 0])
            for i in mounted:
                if size_class[int(i)] == 2:
                    assert eng.template_info(tmap[int(i)])['n_ticks'] > 0, i
    if len(segs) > 1:
        a, b = segs
        for k in ('ncs', 'ep', 'es'):
            assert np.array_equal(a[k], b[k]), k
        assert np.array_equal(a['stats'][..., keep], b['stats'][..., keep])
        if memo_mode == engine.MEMO_SHARED:
            assert b['memo']['lookaheads'] == 0, b['memo']

    # what the workload reached
    tid = ref['tid']                                                    # [B, L], -1 = left out of the action
    jct = np.array([eng.run_lookaheads([tmap[i]])[0]['jct'][0] for i in range(len(wl.templates))])
    macc = wl.actions['max_acceptable_jct'].T
    placed = tid >= 0
    blocked_by_lookahead = int((placed & (jct[np.maximum(tid, 0)] > macc)).sum())
    unplaced = int((~placed).sum())
    multi = int((ref['n_cluster_steps'] > 1).sum())
    mixed = 0
    if memo_mode == engine.MEMO_REFERENCE:
        ran = ref['stats'][..., SS['lookahead_ran']] == 1                # [B, L]: memo misses
        for p in range(L):
            classes = {size_class[int(t)] == 2 for t in tid[ran[:, p], p]}
            mixed += classes == {True, False}
    print(_case_id(case), dict(episodes=B, env_steps=B * L, cluster_steps=int(ref['n_cluster_steps'].sum()),
                               blocked_by_lookahead=blocked_by_lookahead, unplaced=unplaced, multi_cluster_step_env_steps=multi,
                               mixed_size_class_steps=mixed))
    assert multi > 0 and blocked_by_lookahead > 0
    if config.startswith(('cfg1', 'cfg2', 'cfg3')):
        assert unplaced > 0
    if config.startswith('cfg4') and memo_mode == engine.MEMO_REFERENCE and lookahead_mode is None:
        assert mixed > 0, 'no step mixed resident and non-resident memo misses'
    eng.close()


def _device_actions(wl, tmap):
    import torch
    out = []
    for p in range(L):
        a = wl.actions[p].copy()
        placed = a['template_id'] >= 0
        a['template_id'][placed] = np.array([tmap[int(t)] for t in a['template_id'][placed]], dtype=np.int32)
        out.append(torch.from_numpy(a.view(np.uint8).reshape(wl.n_episodes, -1).copy()).cuda())
    return out


def test_engines_in_one_process_step_alternately():
    """A kernel's dynamic shared memory limit is shared by every engine of the process.  An engine whose templates need less of it
    (cfg1's chains) must not break the launches of one that needs more (cfg4's BERT jobs, resident and not) stepped after it."""
    import torch
    from ddls_b200 import engine
    runs = []
    for config, B in (('cfg4-bert-256w', 512), ('cfg1-chain-8w', 64)):
        eng, wl, tmap = _workload(config, B, 0, 'reference')
        runs.append((eng, wl, _device_actions(wl, tmap), _oracle(config, B, 0, 'reference', wl)))
    for eng, wl, _, _ in runs:
        eng.reset(wl.arrivals)
    bufs = [torch.empty((L, wl.n_episodes, engine.STEP_STATS_LEN), dtype=torch.float64, device='cuda') for _, wl, _, _ in runs]
    for p in range(L):
        for (eng, _, on_dev, _), buf in zip(runs, bufs):
            eng.step_device(on_dev[p].data_ptr(), True, buf[p].data_ptr(), None)
    for (eng, _, _, ref), buf in zip(runs, bufs):
        eng.sync()
        eng.check_status()
        assert np.array_equal(buf.cpu().numpy(), ref['stats'].transpose(1, 0, 2))
        assert np.array_equal(eng.episode_stats(), ref['es'])
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------------------
ENV_CONFIGS = [('cfg2-resnet50-32w', 256), ('cfg3-resnet50-64w', 4096), ('cfg4-bert-256w', 4096), ('cfg5-mix-128w', 16384)]


@pytest.mark.parametrize('config,B', ENV_CONFIGS, ids=[c.split('-')[0] for c, _ in ENV_CONFIGS])
def test_batched_environments_equal_each_other_and_the_oracle(config, B):
    from ddls_b200 import batched, workload
    from ddls_b200.engine import SS
    from oracle import oracle
    cfg = workload.CONFIGS[config]
    seed = 0
    envs = {}
    for label, cls in (('device', batched.DeviceRampJobPartitioningEnvironment), ('host', batched.BatchedRampJobPartitioningEnvironment)):
        graphs = [workload.make_graph(kind, **kw) for kind, kw in cfg['graphs']]
        envs[label] = cls(tuple(cfg['shape']), graphs, n_episodes=B, jobs_per_episode=L, seed=seed, run_times='reference',
                          interarrival=('exponential', 1000.0) if cfg.get('exponential') else ('fixed', 1000.0),
                          **({'prewarm': True} if label == 'device' else {}))
    dev, host = envs['device'], envs['host']
    print(config, 'device env decides everything on the device (no synchronisation path):', dev._device_decides_everything)
    # the host environment's lowered jobs, by engine template id, and the action rows it hands its engine
    jobs, rows = {}, []
    reg, step = host.eng.register_template, host.eng.step

    def register(job):
        t = reg(job)
        jobs[t] = job
        return t

    def capture(actions, **kw):
        rows.append(actions.copy())
        return step(actions, **kw)
    host.eng.register_template, host.eng.step = register, capture

    degs = np.array([d for d in cfg['degrees'] if d <= dev.W])
    prng = np.random.default_rng(99)

    def policy(obs, noise):                                       # bench.py's stand-in agent: a random valid degree, else 0
        am = obs['action_mask']
        best = np.where(am[:, degs[0]] != 0, noise[0], np.float32(0))
        act = np.where(best > 0, degs[0], 0)
        for j in range(1, len(degs)):
            v = np.where(am[:, degs[j]] != 0, noise[j], np.float32(0))
            act = np.where(v > best, degs[j], act)
            np.maximum(best, v, out=best)
        return act

    n_fail = 0
    for seg in range(SEGMENTS):
        od, oh = dev.reset(), host.reset()
        np.testing.assert_array_equal(dev.arrivals, host.arrivals)
        rows.clear()
        host_stats, dev_stats = [], []
        for s in range(L):
            live = ~oh['done']
            np.testing.assert_array_equal(od['done'], oh['done'])
            np.testing.assert_array_equal(od['action_mask'], oh['action_mask'])
            np.testing.assert_array_equal(od['model'][live], oh['model'][live])
            assert np.array_equal(od['graph_features_dynamic'][live], oh['graph_features_dynamic'][live]), (seg, s)
            assert np.array_equal(od['graph_features_dynamic'][:, 9:], oh['graph_features_dynamic'][:, 9:]), (seg, s)
            noise = prng.random((len(degs), B), dtype=np.float32) + np.float32(1e-3)
            actions = policy(oh, noise)
            od, rd, dd, _ = dev.step(actions)
            oh, rh, dh, _ = host.step(actions)
            np.testing.assert_array_equal(rd, rh)
            np.testing.assert_array_equal(dd, dh)
            n_fail += int((rh < 0).sum())
            host_stats.append(host.last_stats.copy())
            dev_stats.append(dev.last_stats)
        assert dh.all()
        rec_d, rec_h = dev.eng.job_records(), host.eng.job_records()
        for f in rec_h.dtype.names:
            np.testing.assert_array_equal(rec_d[f], rec_h[f], err_msg=f)
        es_d, es_h = dev.episode_stats(), host.episode_stats()
        assert es_d.keys() == es_h.keys()
        for k in es_h:
            if isinstance(es_h[k], list):
                assert len(es_d[k]) == len(es_h[k]) and all(np.array_equal(x, y) for x, y in zip(es_d[k], es_h[k])), k
            else:
                np.testing.assert_array_equal(es_d[k], es_h[k], err_msg=k)
        # the host environment's segment replayed through the oracle driver
        ids = sorted(jobs)
        assert ids == list(range(len(ids)))
        script = np.stack([r['template_id'] for r in rows], axis=1)                        # [B, L]
        mount = np.zeros(script.shape, dtype=oracle.MOUNT_DTYPE)
        for f in oracle.MOUNT_DTYPE.names:
            mount[f] = np.stack([r[f] for r in rows], axis=1)
        ref = oracle.run_scripted_episodes([jobs[i] for i in ids], script, mount, host.arrivals, host.W, len(host.models))
        for s in range(L):
            assert np.array_equal(host_stats[s], ref['stats'][:, s]), (seg, s)
            assert np.array_equal(dev_stats[s], ref['stats'][:, s]), (seg, s)
        for f in rec_h.dtype.names:
            np.testing.assert_array_equal(rec_h[f], ref['records'][f], err_msg=f)
        fin = np.array([as_row(episode_stats(ref['cluster_stats'][b, :ref['n_cluster_stats'][b]], host.arrivals[b])) for b in range(B)])
        np.testing.assert_array_equal(host.eng.episode_stats(), fin)
        print(config, f'segment {seg}: {B} episodes, {B * L} env-steps, {int(ref["n_cluster_steps"].sum())} cluster steps, '
              f'{len(jobs)} templates, {n_fail} rewards of fail_reward so far')
    dev.close(); host.close()
