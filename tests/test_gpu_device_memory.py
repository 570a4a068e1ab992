"""GPU: the engine and the policy give back every byte they allocate, on success and on failure.

Each case compares the library's own count of the device and page-locked host bytes it holds (engine.device_bytes(), process-wide)
before and after, within the test: unlike cudaMemGetInfo it does not move with other work on the card."""
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

L = 8


def _bytes():
    from ddls_b200 import engine
    return engine.device_bytes()


def _baseline():
    """the count with every engine and policy of earlier tests that only a reference cycle still holds freed first"""
    gc.collect()
    return _bytes()


def _templates(config):
    from ddls_b200 import workload
    return workload.build_templates(config, run_times='reference')[3]


def test_engine_lifecycle_gives_back_every_byte():
    """Resident and non-resident templates, a prewarmed device environment with its host mirror and per-tick lists, steps, and
    standalone lookaheads with traces at two growing sizes (their buffers and private trace pools grow): close() frees all of it."""
    from ddls_b200 import batched, workload
    base = _baseline()
    cfg = workload.CONFIGS['cfg3-resnet50-64w']
    graphs = [workload.make_graph(kind, **kw) for kind, kw in cfg['graphs']]
    env = batched.DeviceRampJobPartitioningEnvironment(tuple(cfg['shape']), graphs, n_episodes=64, jobs_per_episode=L, seed=0,
                                                       run_times='reference', prewarm=True)
    eng = env.eng
    eng.enable_tick_lists(64)
    eng.enable_tick_lists(128)                                       # replaces the lists
    ids = [eng.register_template(t) for t in _templates('cfg3-resnet50-64w') + _templates('cfg4-bert-256w')]
    classes = {eng.template_info(t)['size_class'] for t in ids}
    assert 2 in classes and classes - {2}, classes                  # resident and not
    obs = env.reset()
    degs = np.arange(1, obs['action_mask'].shape[1])
    for _ in range(3):
        am = obs['action_mask']
        actions = np.where(am[:, degs].any(1), degs[np.argmax(am[:, degs] != 0, axis=1)], 0)
        obs, _, _, _ = env.step(actions)
    held = _bytes()
    assert held[0] > base[0] and held[1] > base[1]
    for n in (len(ids) // 2, 2 * len(ids)):
        res = eng.run_lookaheads((ids * 2)[:n], want_trace=True)[0]
        assert (res['status'] == 0).all()
    env.close()
    assert _bytes() == base


def test_policy_lifecycle_gives_back_every_byte():
    from ddls_b200 import policy as P
    from ddls_b200.engine import _check
    from test_gpu_policy_kernels import _env
    env, gs = _env(B=256)
    env.reset()
    base = _baseline()
    pol = P.DeviceGNNPolicy(gs, 17, None, P.random_state_dict(P.DEFAULT_CONFIG, 17, seed=2))
    st = pol.static[0]
    for _ in range(2):                                               # replaces model 0's arrays
        pol.set_model(0, st['node_features'], st['edge_features'], st['edges_src'], st['edges_dst'], st['graph_static'])
    rng = np.random.default_rng(0)
    for n in (8, 512):
        pol.forward(rng.integers(0, len(gs), n), rng.standard_normal((n, 17)), np.ones((n, 17), dtype=np.uint8))
    pol.act(env)
    for horizon in (2, 4):                                           # the second replaces the trajectory buffers
        _check(pol._L.ramp_policy_trajectory_begin(pol._h, env.eng._h, horizon))
    assert _bytes()[0] > base[0]
    pol.close()
    assert _bytes() == base
    env.close()


def test_failed_engine_creation_gives_back_every_byte():
    """An engine whose job-record table is over twice the card's memory: the driver refuses that allocation before it reserves
    anything.  Creation raises naming the allocation, nothing stays allocated, and an engine created afterwards steps correctly."""
    import torch
    from ddls_b200 import engine
    from test_gpu_bench_workloads import _device_actions, _oracle, _workload
    B, record_bytes = 2, engine.JOB_RECORD_DTYPE.itemsize
    max_jobs = 2 * torch.cuda.get_device_properties(0).total_memory // (record_bytes * B) + 1
    assert max_jobs < 2 ** 31
    base = _baseline()
    with pytest.raises(Exception, match='ep_rec'):
        engine.RampEngine(n_episodes=B, n_cluster_workers=8, max_jobs=int(max_jobs))
    assert _bytes() == base
    eng, wl, tmap = _workload('cfg1-chain-8w', 64, 0, 'reference')
    ref = _oracle('cfg1-chain-8w', 64, 0, 'reference', wl)
    on_dev = _device_actions(wl, tmap)
    eng.reset(wl.arrivals)
    buf = torch.empty((L, wl.n_episodes, engine.STEP_STATS_LEN), dtype=torch.float64, device='cuda')
    for p in range(L):
        eng.step_device(on_dev[p].data_ptr(), True, buf[p].data_ptr(), None)
    eng.sync()
    eng.check_status()
    assert np.array_equal(buf.cpu().numpy(), ref['stats'].transpose(1, 0, 2))
    assert np.array_equal(eng.episode_stats(), ref['es'])
    eng.close()


def test_a_smaller_policy_leaves_a_larger_ones_shared_memory_alone():
    """The read-out kernel's dynamic shared memory limit belongs to the kernel in the process: a gnn.yaml policy (about 71 KB of it)
    created after the widest configuration (174,852 B) must not lower it under the wider one's launches."""
    from ddls_b200 import policy as P
    from test_gpu_policy_kernels import CONFIGS, SEED, _cfg, graphs, head_smem_bytes, raw_policy
    over, A, smem, _ = CONFIGS['max']
    c = _cfg(over)
    assert head_smem_bytes(c, A) == smem
    rng = np.random.default_rng(5)
    gs = [g.features(c, rng) for g in graphs(False)]
    sd = P.random_state_dict(c, A, seed=SEED)
    n = 300
    model = rng.integers(0, len(gs), n)
    gf = rng.standard_normal((n, c['in_features_graph'])).astype(np.float32)
    mask = (rng.random((n, A)) < 0.7).astype(np.uint8)
    wide = raw_policy(c, A, gs, sd)
    small = P.DeviceGNNPolicy(_env_graphs(), 17)
    assert head_smem_bytes(small.config, 17) < smem
    got = wide.forward(model, gf, mask)
    fresh = raw_policy(c, A, gs, sd)
    want = fresh.forward(model, gf, mask)
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g, w)
    for p in (wide, small, fresh):
        p.close()


def _env_graphs():
    from ddls_b200 import synth
    return [synth.chain_graph(6, 'chain6'), synth.transformer_like_graph(n_layers=1, name='tfm1', seed=4)]
