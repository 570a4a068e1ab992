"""-m gpu: the device environment stepped with PyTorch CUDA tensors (ddls_b200/torch_env.py: ramp_env_ingest / ramp_env_export on the
caller's stream).  The observation it hands out is the reference's, bit for bit, on the 16 golden episodes; its episodes are the
host-array path's, step for step, with and without the host's placer, at config 3's 4,096 episodes and on two models; errors are
the host path's; results are ordered on the caller's stream without a synchronisation; a torch GNNPolicy reads it as the device
policy does; and it gives back every byte it took."""
import numpy as np
import pytest

from golden_io import Golden
from test_env_observation_model import CASES, DYNAMIC, OBS, model_of_arrivals, recorded_jobs_params
from test_gpu_batched_env import SHAPES, _graphs
from test_gpu_episode_stats import set_job_counts

pytestmark = pytest.mark.gpu


def replay_env(name):
    """The torch environment replaying case `name` in one episode: recorded models, gaps and fracs, the reference's jobs_params and
    no max-acceptable-JCT override (tests/test_gpu_env_observation.py's setup)."""
    from ddls_b200.torch_env import TorchRampJobPartitioningEnvironment
    g = Golden(name)
    graphs = _graphs()[name]
    model = model_of_arrivals(name, graphs)
    J = len(model)
    frac = np.ones(J)
    frac[OBS[name + '_job_idx']] = OBS[name + '_frac']
    script = {'model': model[None, :], 'gap': g.d['arrivals'][None, :, 0], 'frac': frac[None, :]}
    env = TorchRampJobPartitioningEnvironment(SHAPES[g.n_cluster_workers], graphs, n_episodes=1, jobs_per_episode=J,
                                              max_partitions_per_op=int(OBS[name + '_max_partitions_per_op']),
                                              max_simulation_run_time=g.max_sim_time, script=script,
                                              machine_epsilon=float(OBS[name + '_machine_epsilon']), jobs_params=recorded_jobs_params(name))
    return env, g


@pytest.mark.parametrize('name', CASES)
def test_replay_observation_is_the_references_bit_for_bit(name):
    import torch
    env, g = replay_env(name)
    obs = env.reset()
    set_job_counts(env.env, [g])
    gf, mask, actions = OBS[name + '_graph_features'], OBS[name + '_action_mask'], OBS[name + '_actions']
    for e in range(len(actions)):
        got = obs['graph_features'][0].cpu().numpy()
        assert got.dtype == np.float32 and got.shape == gf[e].shape
        bad = np.flatnonzero(got.view(np.uint32) != gf[e].view(np.uint32))
        assert not len(bad), (name, e, bad, got[bad], gf[e][bad])
        np.testing.assert_array_equal(obs['action_mask'][0].cpu().numpy(), mask[e].astype(bool), err_msg=f'{name} step {e}')
        obs, reward, done, _ = env.step(torch.tensor([int(actions[e])], dtype=torch.int64, device=env.device))
    env.check()
    assert bool(done.all()), name
    env.close()


# ---- the torch path against the host-array path ----------------------------------------------------------------------------

def _workload(kind):
    from ddls_b200 import synth
    if kind == 'cfg3':          # bench.py's config 3: 4,096 episodes, the 64-worker cluster, ResNet-50, 8 jobs per episode
        return (4, 4, 4), [synth.resnet_like_graph()], dict(n_episodes=4096, jobs_per_episode=8, seed=3), True
    if kind == 'host_placer':   # tfm1 splits its ops unevenly at some degrees: those placements go to the host's placer
        graphs = [synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3), synth.chain_graph(6, 'chain6'),
                  synth.transformer_like_graph(n_layers=1, name='tfm1', seed=4)]
        return (4, 4, 4), graphs, dict(n_episodes=768, jobs_per_episode=7, seed=11, interarrival=('exponential', 600.0)), False
    if kind == 'mix128_exp':
        return (8, 4, 4), _graphs()['mix128_exp'], dict(n_episodes=512, jobs_per_episode=8, seed=5, interarrival=('exponential', 1000.0)), True
    raise KeyError(kind)


def _twins(kind, **extra):
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    from ddls_b200.torch_env import TorchRampJobPartitioningEnvironment
    shape, graphs, kw, prewarm = _workload(kind)
    kw = dict(kw, **extra)
    return (TorchRampJobPartitioningEnvironment(shape, graphs, prewarm=prewarm, **kw),
            DeviceRampJobPartitioningEnvironment(shape, graphs, prewarm=prewarm, **kw))


def _draw(mask, gen):
    """masked uniform categorical: one action per episode among those its mask allows"""
    import torch
    return torch.multinomial(mask.to(torch.float32), 1, generator=gen).reshape(-1)


def _assert_obs_equal(obs, host, where):
    gf = obs['graph_features'].cpu().numpy()
    np.testing.assert_array_equal(obs['model'].cpu().numpy(), host['model'].astype(np.int64), err_msg=where)
    np.testing.assert_array_equal(gf[:, DYNAMIC].view(np.uint32), host['graph_features_dynamic'].view(np.uint32), err_msg=where)
    np.testing.assert_array_equal(obs['action_mask'].cpu().numpy(), host['action_mask'].astype(bool), err_msg=where)
    np.testing.assert_array_equal(gf[:, 17:], host['action_mask'].astype(np.float32), err_msg=where)


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


def _run_twins(t_env, h_env, gen, dtype, strided, max_steps=64):
    import torch
    obs, host = t_env.reset(), h_env.reset()
    n = 0
    for n in range(max_steps):
        _assert_obs_equal(obs, host, f'step {n}')
        a = _draw(obs['action_mask'], gen).to(dtype)
        if strided:
            a = torch.stack([a, torch.zeros_like(a)], dim=1)[:, 0]
            assert not a.is_contiguous()
        obs, reward, done, _ = t_env.step(a)
        host, h_reward, h_done, _ = h_env.step(a.cpu().numpy())
        np.testing.assert_array_equal(reward.cpu().numpy(), h_reward, err_msg=f'step {n}')
        np.testing.assert_array_equal(done.cpu().numpy(), h_done, err_msg=f'step {n}')
        if h_done.all():
            break
    t_env.check()
    assert h_done.all() and n > 0
    np.testing.assert_array_equal(t_env.decisions(), h_env.decisions())
    _assert_same(t_env.episode_stats(), h_env.episode_stats(), 'episode_stats')


@pytest.mark.parametrize('kind,dtype,strided', [('cfg3', 'int64', False), ('cfg3', 'int32', True), ('host_placer', 'int32', False),
                                                ('host_placer', 'int64', True), ('mix128_exp', 'int64', False)])
def test_torch_path_gives_the_host_paths_episodes(kind, dtype, strided):
    import torch
    t_env, h_env = _twins(kind)
    if kind != 'mix128_exp':
        assert t_env.env._device_decides_everything == (kind == 'cfg3')
    gen = torch.Generator(device=t_env.device).manual_seed(17)
    _run_twins(t_env, h_env, gen, getattr(torch, dtype), strided)
    if kind == 'host_placer':
        assert t_env.env.stats['placer_calls'] > 0
    t_env.close(); h_env.close()


# ---- errors ------------------------------------------------------------------------------------------------------------------

def _small(apply_action_mask=True, prewarm=True):
    from ddls_b200 import synth
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    from ddls_b200.torch_env import TorchRampJobPartitioningEnvironment
    args = ((4, 4, 4), [synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3)])
    kw = dict(n_episodes=64, jobs_per_episode=6, seed=2, apply_action_mask=apply_action_mask)
    return TorchRampJobPartitioningEnvironment(*args, prewarm=prewarm, **kw), DeviceRampJobPartitioningEnvironment(*args, prewarm=prewarm, **kw)


def test_an_action_the_mask_forbids_raises_at_check_with_the_host_paths_message():
    import torch
    t_env, h_env = _small(apply_action_mask=True)
    obs = t_env.reset(); h_env.reset()
    assert not bool(obs['action_mask'][:, 3].any())               # an odd degree above 1 has no RAMP-symmetric block
    a = torch.zeros(t_env.B, dtype=torch.int64, device=t_env.device)
    a[5] = 3
    with pytest.raises(Exception) as host_err:
        h_env.step(a.cpu().numpy())
    t_env.step(a)                                                  # prewarmed: the error waits for a synchronising call
    with pytest.raises(Exception) as err:
        t_env.check()
    assert str(err.value) == str(host_err.value) and str(err.value).startswith('episode 5: the action is invalid given its action mask')
    t_env.check()                                                  # raised once
    t_env.close(); h_env.close()


def test_an_action_the_mask_forbids_is_placed_as_0_without_the_mask():
    import torch
    t_env, h_env = _small(apply_action_mask=False)
    obs, host = t_env.reset(), h_env.reset()
    gen = torch.Generator(device=t_env.device).manual_seed(4)
    for n in range(12):
        _assert_obs_equal(obs, host, f'step {n}')
        a = _draw(obs['action_mask'], gen)
        a[::3] = 3                                                 # masked for every episode
        obs, reward, done, _ = t_env.step(a)
        host, h_reward, h_done, _ = h_env.step(a.cpu().numpy())
        np.testing.assert_array_equal(reward.cpu().numpy(), h_reward)
        np.testing.assert_array_equal(done.cpu().numpy(), h_done)
        if h_done.all():
            break
    t_env.check()
    np.testing.assert_array_equal(t_env.decisions(), h_env.decisions())
    _assert_same(t_env.episode_stats(), h_env.episode_stats(), 'episode_stats')
    t_env.close(); h_env.close()


@pytest.mark.parametrize('apply_action_mask', [True, False])
@pytest.mark.parametrize('prewarm', [True, False])
@pytest.mark.parametrize('bad,dtype', [(-1, 'int32'), (17, 'int32'), (17, 'int64'), (2 ** 40, 'int64')])
def test_an_action_outside_the_set_raises_whatever_the_mask_setting(bad, dtype, apply_action_mask, prewarm):
    import torch
    t_env, _ = _small(apply_action_mask=apply_action_mask, prewarm=prewarm)
    t_env.reset()
    a = torch.zeros(t_env.B, dtype=getattr(torch, dtype), device=t_env.device)
    a[40], a[7] = bad, bad
    with pytest.raises(Exception) as err:
        t_env.step(a)
        t_env.check()
    want = f'Action {bad} not in action set {list(range(17))}.'      # RJPE:314-316, BatchedRampJobPartitioningEnvironment.step
    assert str(err.value).startswith(f'episode 7: {want}'), str(err.value)
    t_env.check()                                                  # raised once
    t_env.close()


# ---- stream order ------------------------------------------------------------------------------------------------------------

def test_actions_made_on_a_side_stream_behind_a_sleep_give_the_twins_results():
    import torch
    t_env, h_env = _small()
    obs, host = t_env.reset(), h_env.reset()
    gen = torch.Generator(device=t_env.device).manual_seed(8)
    side = torch.cuda.Stream(device=t_env.device)
    for n in range(6):
        side.wait_stream(torch.cuda.current_stream(t_env.device))
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)
            a = _draw(obs['action_mask'], gen)
        torch.cuda.current_stream(t_env.device).wait_stream(side)
        a.record_stream(torch.cuda.current_stream(t_env.device))
        obs, reward, done, _ = t_env.step(a)
        host, h_reward, h_done, _ = h_env.step(a.cpu().numpy())
        _assert_obs_equal(obs, host, f'step {n}')
        np.testing.assert_array_equal(reward.cpu().numpy(), h_reward)
        np.testing.assert_array_equal(done.cpu().numpy(), h_done)
    t_env.check()
    t_env.close(); h_env.close()


def test_a_prewarmed_step_does_not_wait_for_the_callers_stream():
    import torch
    t_env, h_env = _small()
    obs, host = t_env.reset(), h_env.reset()
    assert t_env.env._device_decides_everything
    gen = torch.Generator(device=t_env.device).manual_seed(1)
    a = _draw(obs['action_mask'], gen)                             # the first step sizes the engine's scratch, which synchronises
    obs = t_env.step(a)[0]
    h_env.step(a.cpu().numpy())
    a = _draw(obs['action_mask'], gen)
    cur = torch.cuda.current_stream(t_env.device)
    cur.synchronize()
    torch.cuda._sleep(500_000_000)                                 # a few hundred ms queued ahead of the step
    obs, reward, done, _ = t_env.step(a)
    assert not cur.query()                                         # step() returned while the stream was still asleep
    cur.synchronize()
    host, h_reward, h_done, _ = h_env.step(a.cpu().numpy())
    _assert_obs_equal(obs, host, 'after the sleep')
    np.testing.assert_array_equal(reward.cpu().numpy(), h_reward)
    np.testing.assert_array_equal(done.cpu().numpy(), h_done)
    t_env.check()
    t_env.close(); h_env.close()


def test_observations_kept_across_steps_hold_their_own_steps_values_and_out_slices_equal_fresh_tensors():
    import torch
    t_env, h_env = _small()
    o_env, _ = _small()
    obs, host = t_env.reset(), h_env.reset()
    o_env.reset()
    gen = torch.Generator(device=t_env.device).manual_seed(6)
    T, B, A = 3, t_env.B, t_env.n_actions
    buf = {'model': torch.full((T, B), -7, dtype=torch.int64, device=t_env.device),
           'graph_features': torch.full((T, B, 17 + A), -7.0, device=t_env.device),
           'action_mask': torch.zeros((T, B, A), dtype=torch.bool, device=t_env.device),
           'reward': torch.full((T, B), -7.0, dtype=torch.float64, device=t_env.device),
           'done': torch.zeros((T, B), dtype=torch.bool, device=t_env.device)}
    kept, hosts = [], []
    for t in range(T):
        a = _draw(obs['action_mask'], gen)
        obs, reward, done, _ = t_env.step(a)
        o_obs, o_reward, o_done, _ = o_env.step(a, out={k: v[t] for k, v in buf.items()})
        assert o_reward.data_ptr() == buf['reward'][t].data_ptr() and o_obs['graph_features'].data_ptr() == buf['graph_features'][t].data_ptr()
        kept.append((obs, reward, done))
        hosts.append(tuple(np.copy(x) if isinstance(x, np.ndarray) else {k: np.copy(v) for k, v in x.items()}
                           for x in h_env.step(a.cpu().numpy())[:3]))
    torch.cuda.synchronize()
    for t, ((obs, reward, done), (host, h_reward, h_done)) in enumerate(zip(kept, hosts)):
        _assert_obs_equal(obs, host, f'kept step {t}')
        np.testing.assert_array_equal(reward.cpu().numpy(), h_reward)
        np.testing.assert_array_equal(done.cpu().numpy(), h_done)
        for k, v in list(obs.items()) + [('reward', reward), ('done', done)]:
            assert torch.equal(buf[k][t], v), (t, k)
    t_env.check(); o_env.check()
    t_env.close(); h_env.close(); o_env.close()


# ---- a torch policy on the environment ------------------------------------------------------------------------------------

def test_the_torch_gnn_policy_reads_the_observation_as_the_device_policy_does():
    import torch
    from ddls_b200 import policy as P
    from ddls_b200 import synth
    from ddls_b200.torch_env import TorchRampJobPartitioningEnvironment
    from test_gpu_policy import ATOL, RTOL, _torch_policy
    graphs = [synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3), synth.chain_graph(6, 'chain6')]
    env = TorchRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=256, jobs_per_episode=6, seed=9, prewarm=True)
    A = env.n_actions
    cfg = dict(P.DEFAULT_CONFIG)
    sd = P.random_state_dict(cfg, A, seed=7)
    pol = P.DeviceGNNPolicy(graphs, A, cfg, sd)
    ref = _torch_policy(cfg, A, sd).to(env.device)
    with torch.no_grad():
        emb = torch.stack([ref.embed(st['node_features'], st['edge_features'], st['edges_src'], st['edges_dst']) for st in env.static])
    obs = env.reset()
    n_rows = 0
    for n in range(8):
        pol.act(env.env, sample=True, seed=n)
        got = pol.read(env.env)
        live = obs['model'] >= 0
        with torch.no_grad():
            wl, wv = ref(emb[obs['model'].clamp(min=0)], obs['graph_features'], obs['action_mask'].to(torch.float32))
        live_np, valid = live.cpu().numpy(), obs['action_mask'].cpu().numpy()
        rows = np.flatnonzero(live_np)
        np.testing.assert_allclose(got['logits'][rows][valid[rows]], wl.cpu().numpy()[rows][valid[rows]], atol=ATOL, rtol=RTOL, err_msg=f'step {n}')
        np.testing.assert_allclose(got['value'][rows], wv.cpu().numpy()[rows], atol=ATOL, rtol=RTOL, err_msg=f'step {n}')
        n_rows += len(rows)
        obs, reward, done, _ = env.step(torch.from_numpy(got['actions']).to(env.device))
        if bool(done.all()):
            break
    env.check()
    assert n_rows > 256
    pol.close(); env.close()


# ---- memory ----------------------------------------------------------------------------------------------------------------

def test_every_byte_comes_back_a_failed_creation_included():
    import torch
    from ddls_b200 import engine, synth
    from ddls_b200.torch_env import TorchRampJobPartitioningEnvironment
    args = ((4, 4, 4), [synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3)])
    before = engine.device_bytes()
    env = TorchRampJobPartitioningEnvironment(*args, n_episodes=128, jobs_per_episode=6, seed=1, prewarm=True)
    obs = env.reset()
    gen = torch.Generator(device=env.device).manual_seed(3)
    for _ in range(4):
        obs = env.step(_draw(obs['action_mask'], gen))[0]
    env.check()
    assert engine.device_bytes()[0] > before[0]
    env.close()
    assert engine.device_bytes() == before
    with pytest.raises(Exception, match='bad environment shape'):
        TorchRampJobPartitioningEnvironment(*args, n_episodes=128, jobs_per_episode=6, max_partitions_per_op=0)
    assert engine.device_bytes() == before
