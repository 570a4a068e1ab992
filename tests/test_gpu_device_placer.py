"""-m gpu: ``place_on_device=True`` -- jobs whose ops split unevenly placed by ramp_env_place_kernel and looked up by canonical mask
-- against the host's placer: the host environment and the device environment without the option, stepped with the same
masked-random actions, give the same rewards, done flags, observations and job records at every step, and the same decisions and
episode statistics at the end."""
import gc
import warnings

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _workload(kind):
    from ddls_b200 import synth
    if kind == 'host_placer':
        graphs = [synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3), synth.chain_graph(6, 'chain6'),
                  synth.transformer_like_graph(n_layers=1, name='tfm1', seed=4)]
        return (4, 4, 4), graphs, dict(n_episodes=768, jobs_per_episode=7, seed=11, interarrival=('exponential', 600.0))
    if kind == 'bert16':            # BASELINE config 4's job on its cluster; at degree 16 one op splits 10 ways
        return (8, 8, 4), [synth.transformer_like_graph(n_layers=12, name='bert_base_like', seed=2)], \
            dict(n_episodes=4096, jobs_per_episode=6, seed=4, interarrival=('exponential', 800.0), max_partitions_per_op=16)
    if kind == 'mix128_exp':
        return (8, 4, 4), [synth.resnet_like_graph(), synth.transformer_like_graph(n_layers=12, name='gpt2_small_like', seed=5, gpt=True)], \
            dict(n_episodes=512, jobs_per_episode=8, seed=5, interarrival=('exponential', 1000.0))
    raise KeyError(kind)


def _actions(mask, rng):
    """masked uniform: one allowed action per episode"""
    r = rng.random(mask.shape) * mask.astype(bool)
    return r.argmax(axis=1)


def _assert_same(a, b, where):
    assert type(a) is type(b), where
    if isinstance(a, dict):
        assert sorted(a) == sorted(b), where
        for k in a:
            _assert_same(a[k], b[k], f'{where}.{k}')
    elif isinstance(a, list):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same(x, y, f'{where}[{i}]')
    else:
        np.testing.assert_array_equal(a, b, err_msg=where)


def _assert_records_equal(a, b, where):
    for f in a.dtype.names:
        np.testing.assert_array_equal(a[f], b[f], err_msg=f'{where}: {f}')


def _rollout(envs, seed, max_steps=64, loose=()):
    """Resets every environment to the same arrival streams and steps them with the same masked-random actions; checks them
    against envs[0] at every step.  The `loose` ones (the host environment) are checked on everything but the float32 features,
    which agree to 1e-6."""
    rng = np.random.default_rng(seed)
    for e in list(envs) + list(loose):
        e.rng = np.random.default_rng(seed)
    obs = [e.reset() for e in envs]
    lobs = [e.reset() for e in loose]
    for n in range(max_steps):
        for o in lobs:
            np.testing.assert_array_equal(o['action_mask'], obs[0]['action_mask'], err_msg=f'host, step {n}')
            np.testing.assert_allclose(o['graph_features_dynamic'], obs[0]['graph_features_dynamic'], rtol=1e-6, atol=0)
        for e, o in zip(envs[1:], obs[1:]):
            np.testing.assert_array_equal(o['action_mask'], obs[0]['action_mask'], err_msg=f'step {n}')
            live = ~obs[0]['done']
            np.testing.assert_array_equal(o['model'][live], obs[0]['model'][live], err_msg=f'step {n}')
            np.testing.assert_array_equal(o['graph_features_dynamic'].view(np.uint32), obs[0]['graph_features_dynamic'].view(np.uint32),
                                          err_msg=f'step {n}')
        a = _actions(obs[0]['action_mask'], rng)
        out = [e.step(a) for e in envs]
        lout = [e.step(a) for e in loose]
        obs, lobs = [o[0] for o in out], [o[0] for o in lout]
        for e, o in zip(list(envs[1:]) + list(loose), out[1:] + lout):
            np.testing.assert_array_equal(o[1], out[0][1], err_msg=f'reward, step {n}')
            np.testing.assert_array_equal(o[2], out[0][2], err_msg=f'done, step {n}')
            _assert_records_equal(e.eng.job_records(), envs[0].eng.job_records(), f'step {n}')
        if out[0][2].all():
            return n + 1
    raise AssertionError('episodes did not finish')


@pytest.mark.parametrize('kind', ['host_placer', 'bert16', 'mix128_exp'])
def test_device_placer_gives_the_host_placers_episodes(kind):
    from ddls_b200.batched import BatchedRampJobPartitioningEnvironment, DeviceRampJobPartitioningEnvironment
    shape, graphs, kw = _workload(kind)
    ref = DeviceRampJobPartitioningEnvironment(shape, graphs, **kw)
    dev = DeviceRampJobPartitioningEnvironment(shape, graphs, place_on_device=True, **kw)
    host = BatchedRampJobPartitioningEnvironment(shape, graphs, **kw)
    # the host environment's features are float32 of float64 numpy: the device ones agree to 1e-6 (test_gpu_batched_env), so
    # the bit-for-bit comparison is against the device environment without the option
    assert dev.place_on_device
    _rollout([ref, dev], seed=1, loose=[host])
    np.testing.assert_array_equal(dev.decisions(), ref.decisions())
    _assert_same(dev.episode_stats(), ref.episode_stats(), 'episode_stats')
    if kind == 'bert16':
        assert not dev._uniform[0, 16] and dev._geom_mask_set          # the device placed uneven jobs
    ref.close(); dev.close(); host.close()


@pytest.mark.parametrize('kind', ['host_placer', 'bert16'])
def test_torch_env_with_device_placer(kind):
    import torch
    from ddls_b200.torch_env import TorchRampJobPartitioningEnvironment
    shape, graphs, kw = _workload(kind)
    kw = dict(kw, n_episodes=min(kw['n_episodes'], 1024))
    a_env = TorchRampJobPartitioningEnvironment(shape, graphs, place_on_device=True, **kw)
    b_env = TorchRampJobPartitioningEnvironment(shape, graphs, **kw)
    assert a_env.env.place_on_device and not b_env.env.place_on_device
    gen = torch.Generator(device=a_env.device).manual_seed(3)
    oa, ob = a_env.reset(), b_env.reset()
    for n in range(64):
        for k in oa:
            assert torch.equal(oa[k], ob[k]), (n, k)
        act = torch.multinomial(oa['action_mask'].to(torch.float32), 1, generator=gen).reshape(-1)
        oa, ra, da, _ = a_env.step(act)
        ob, rb, db, _ = b_env.step(act)
        assert torch.equal(ra, rb) and torch.equal(da, db), n
        if bool(da.all()):
            break
    a_env.check()
    assert bool(da.all())
    np.testing.assert_array_equal(a_env.decisions(), b_env.decisions())
    _assert_same(a_env.episode_stats(), b_env.episode_stats(), 'episode_stats')
    a_env.close(); b_env.close()


def test_goldens_with_device_placer(monkeypatch):
    """The 16 recorded golden episodes give their recorded step statistics with the option on.  None of them takes a decision on a
    job whose ops split unevenly (every recorded action splits every op of its job `degree` ways), so they pin that the option
    leaves uniform jobs as they were; the uneven ones are pinned by the twins above, against the host placer."""
    from ddls_b200 import batched
    from ddls_b200.batched import _Model
    from ddls_b200.template_builder import original_job_totals
    import test_gpu_batched_env as replay
    from golden_io import Golden

    class _Placing(batched.DeviceRampJobPartitioningEnvironment):
        def __init__(self, *a, **k):
            super().__init__(*a, place_on_device=True, **k)
            assert self.place_on_device
    monkeypatch.setattr(batched, 'DeviceRampJobPartitioningEnvironment', _Placing)
    catalogue, uneven = replay._graphs(), []
    for names in replay.BATCHES:
        replay.test_batched_env_replays_reference_episodes_in_lock_step(names, 'device')
        for n in names:
            g = Golden(n)
            totals = [original_job_totals(x)[0] for x in catalogue[n]]
            for e, (_, a) in enumerate(replay._decisions(g)):
                if a == 0:
                    continue
                x = catalogue[n][[i for i, t in enumerate(totals) if abs(t - g.d['arrivals'][e, 1]) <= 1e-9 * abs(g.d['arrivals'][e, 1])][0]]
                if len(set(_Model(x, 0.01, 50).splits(a))) > 1:
                    uneven.append(n)
    assert uneven == []


def test_warm_environment_reads_back_only_the_count():
    """A second reset-and-rollout with the same streams and actions calls the host's placer 0 times, and its decisions copy nothing
    from the device but the count and the error word (page-locked); a cold rollout's host placements copy lists and rows."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    shape, graphs, kw = _workload('bert16')
    kw = dict(kw, n_episodes=1024)
    env = DeviceRampJobPartitioningEnvironment(shape, graphs, place_on_device=True, **kw)

    def rollout():
        rng = np.random.default_rng(9)
        env.rng = np.random.default_rng(9)                              # the same arrival streams every time
        obs = env.reset()
        steps = 0
        while not obs['done'].all():
            env._actions_pinned[:] = _actions(obs['action_mask'], rng)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:               # the decision half of DeviceRamp...step
                _engine._check(env.eng._L.ramp_env_decide(env.eng._h, env._actions_pinned.ctypes.data, C.byref(n_need), env._need.ctypes.data))
                if n_need.value > 0:
                    env._decide_on_host(env._need[:n_need.value].copy(), env._actions_pinned)
                torch.cuda.synchronize()
            copies.append(sum(1 for ev in prof.events() if 'Memcpy DtoH' in ev.name and 'Pageable' in ev.name))
            _engine._check(env.eng._L.ramp_env_advance(env.eng._h))
            obs = env._read()
            steps += 1
        return steps
    import ctypes as C
    from ddls_b200 import engine as _engine
    n_need = C.c_int32(0)
    copies = []
    rollout()
    cold_calls, cold_copies = env.stats['placer_calls'], sum(copies)
    assert cold_calls > 0 and cold_copies > 0
    copies.clear()
    rollout()
    assert env.stats['placer_calls'] == cold_calls
    assert sum(copies) == 0, copies
    env.close()


def test_geometry_table_grows_and_keeps_its_entries():
    """Hundreds of extra entries grow the table several times over; the entries a rollout registered still decide the next one."""
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    shape, graphs, kw = _workload('bert16')
    kw = dict(kw, n_episodes=512)
    ref = DeviceRampJobPartitioningEnvironment(shape, graphs, **kw)
    env = DeviceRampJobPartitioningEnvironment(shape, graphs, place_on_device=True, **kw)
    _rollout([ref, env], seed=3)
    calls = env.stats['placer_calls']
    L, h = env.eng._L, env.eng._h
    mt = np.zeros(6)
    mt[:] = env._t_mount[0]
    for k in range(600):                                               # masks no placement makes: model 0, degree 2, one server
        cm = np.zeros(env.n_words, dtype=np.uint64)
        cm[k % env.n_words] = np.uint64(1) << np.uint64(k // env.n_words % 64)
        cm[(k + 1) % env.n_words] |= np.uint64(1) << np.uint64(63 - k // (64 * env.n_words) % 64)
        assert L.ramp_env_set_geometry_template(h, 0, 2, cm.ctypes.data, 0, mt.ctypes.data) == 0
    _rollout([ref, env], seed=3)
    assert env.stats['placer_calls'] == calls
    ref.close(); env.close()


def _limit_graph(n):
    """a chain of n ops, every other one small enough to split 2 ways at degree 4"""
    from ddls_b200.synth import ForwardGraph
    g = ForwardGraph(name=f'chain{n}')
    for i in range(1, n + 1):
        g.add('Linear', 0.015 if i % 2 else 0.3, 0.01, 1e6, 1e3)
        if i > 1:
            g.edges.append((i - 1, i))
    return g


def test_shared_memory_limit_both_sides():
    """At the limit the library takes the tables (it checks the same bound); one op past it the environment warns and keeps the
    host's placer.  A job of 3,000 ops is not simulated here: its lookahead outgrows the engine's tick trace."""
    from ddls_b200.batched import PLACE_SMEM_PER_WARP, DeviceRampJobPartitioningEnvironment, place_smem_per_warp
    shape = (2, 2, 4)
    n_max = (PLACE_SMEM_PER_WARP - 8 * (16 + 8)) // 4
    assert place_smem_per_warp(16, n_max) == PLACE_SMEM_PER_WARP
    kw = dict(n_episodes=32, jobs_per_episode=3, seed=1, max_partitions_per_op=4, interarrival=('fixed', 1e9))
    with warnings.catch_warnings():
        warnings.simplefilter('error')
        env = DeviceRampJobPartitioningEnvironment(shape, [_limit_graph(n_max)], place_on_device=True, **kw)
    assert env.place_on_device and not env._uniform[0, 4]
    env.close()
    with pytest.warns(UserWarning, match='shared memory'):
        env = DeviceRampJobPartitioningEnvironment(shape, [_limit_graph(n_max + 1)], place_on_device=True, **kw)
    assert not env.place_on_device
    env.close()


@pytest.mark.parametrize('apply_action_mask', [True, False])
def test_action_mask_errors_unchanged(apply_action_mask):
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    shape, graphs, kw = _workload('host_placer')
    kw = dict(kw, n_episodes=64, apply_action_mask=apply_action_mask)
    msgs = []
    for place in (False, True):
        env = DeviceRampJobPartitioningEnvironment(shape, graphs, place_on_device=place, **kw)
        obs = env.reset()
        a = np.zeros(64, dtype=np.int64)
        a[5] = 3                                                        # odd: never in the mask
        try:
            _, r, _, _ = env.step(a)
            msgs.append(('ok', r.tolist()))
        except Exception as e:                                          # noqa: BLE001
            msgs.append(('raised', str(e)))
        env.close()
    assert msgs[0] == msgs[1]
    assert (msgs[0][0] == 'raised') == apply_action_mask


def test_every_byte_returned():
    from ddls_b200 import engine
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    gc.collect()
    base = engine.device_bytes()
    shape, graphs, kw = _workload('bert16')
    env = DeviceRampJobPartitioningEnvironment(shape, graphs, place_on_device=True, **dict(kw, n_episodes=256))
    rng = np.random.default_rng(0)
    obs = env.reset()
    for _ in range(3):
        obs, _, _, _ = env.step(_actions(obs['action_mask'], rng))
    assert engine.device_bytes()[0] > base[0]
    env.close()
    assert engine.device_bytes() == base
    # a failed construction: the placer tables are refused after the engine allocated its environment
    from ddls_b200 import batched

    def boom(self, cand_ptr):
        raise RuntimeError('refused')
    orig = batched.DeviceRampJobPartitioningEnvironment._set_placer_tables
    batched.DeviceRampJobPartitioningEnvironment._set_placer_tables = boom
    try:
        from ddls_b200.torch_env import TorchRampJobPartitioningEnvironment
        with pytest.raises(RuntimeError, match='refused'):
            TorchRampJobPartitioningEnvironment(shape, graphs, place_on_device=True, **dict(kw, n_episodes=256))
    finally:
        batched.DeviceRampJobPartitioningEnvironment._set_placer_tables = orig
    gc.collect()
    assert engine.device_bytes() == base
