"""-m gpu: the torch environment's steps and the torch policy's forward captured with torch.cuda.graph and replayed.  A replay gives
the bits an eager twin (the same arguments and seed) gives, step for step, across eager resets and a weight update; sampling
draws afresh on each replay; errors of replayed steps surface at check() as an eager step's do; each capture that would need the
host is refused before anything is enqueued, and the environment then steps on as its twin; and every byte comes back."""
import numpy as np
import pytest

from test_gpu_torch_env import _assert_same, _draw

pytestmark = pytest.mark.gpu

OUT_KEYS = ('model', 'graph_features', 'action_mask', 'reward', 'done')


def _res2():
    from ddls_b200 import synth
    return synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3)


def _workload(kind):
    """(shape, graphs, kwargs): one model, and two models in one batch; the device tables decide every placement of both"""
    from ddls_b200 import synth
    if kind == 'one':
        return (4, 4, 4), [_res2()], dict(n_episodes=64, jobs_per_episode=6, seed=2)
    if kind == 'two':
        return (4, 4, 4), [_res2(), synth.chain_graph(6, 'chain6')], dict(n_episodes=96, jobs_per_episode=5, seed=5,
                                                                           interarrival=('exponential', 800.0))
    raise KeyError(kind)


def _twins(kind, **extra):
    from ddls_b200.torch_env import TorchRampJobPartitioningEnvironment
    shape, graphs, kw = _workload(kind)
    kw = dict(kw, prewarm=True, **extra)
    return TorchRampJobPartitioningEnvironment(shape, graphs, **kw), TorchRampJobPartitioningEnvironment(shape, graphs, **kw)


def _outs(env, n):
    import torch
    B, A = env.B, env.n_actions
    spec = {'model': ((B,), torch.int64), 'graph_features': ((B, 17 + A), torch.float32), 'action_mask': ((B, A), torch.bool),
            'reward': ((B,), torch.float64), 'done': ((B,), torch.bool)}
    return [{k: torch.empty(s, dtype=d, device=env.device) for k, (s, d) in spec.items()} for _ in range(n)]


def _step_out(obs, reward, done):
    return dict(obs, reward=reward, done=done)


def _assert_bits(got, want, where):
    for k in OUT_KEYS:
        a, b = got[k].cpu().numpy(), want[k].cpu().numpy()
        if a.dtype.kind == 'f':
            a, b = a.view(np.uint32 if a.itemsize == 4 else np.uint64), b.view(np.uint32 if b.itemsize == 4 else np.uint64)
        np.testing.assert_array_equal(a, b, err_msg=f'{where}: {k}')


def _capture_steps(env, actions, outs):
    import torch
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for a, o in zip(actions, outs):
            env.step(a, out=o)
    return g


def _fixed_actions(env, H, seed):
    """H steps of actions for every episode, fixed ahead: any action of the set (apply_action_mask=False places masked ones as 0)"""
    import torch
    gen = torch.Generator(device=env.device).manual_seed(seed)
    return [torch.randint(0, env.n_actions, (env.B,), generator=gen, device=env.device) for _ in range(H)]


def _segment(g, env, twin, static, outs, actions, where):
    """replays g once with `actions` copied into the static inputs, and steps the twin eagerly on them: equal at every step"""
    for s, a in zip(static, actions):
        s.copy_(a)
    g.replay()
    for t, a in enumerate(actions):
        want = _step_out(*twin.step(a)[:3])
        _assert_bits(outs[t], want, f'{where} step {t}')


def _assert_twins_equal(env, twin, where):
    env.check(); twin.check()
    np.testing.assert_array_equal(env.decisions(), twin.decisions(), err_msg=where)
    _assert_same(env.episode_stats(), twin.episode_stats(), f'{where} episode_stats')
    _assert_same(env.recorded_steps(), twin.recorded_steps(), f'{where} recorded_steps')


@pytest.mark.parametrize('kind', ['one', 'two'])
def test_replayed_steps_equal_the_eager_twins_bit_for_bit_past_the_episodes_end(kind):
    import torch
    env, twin = _twins(kind, apply_action_mask=False)
    H = 8
    for e in (env, twin):
        e.record_steps(64)
        e.reset()
    a0 = _fixed_actions(env, 1, seed=99)[0]
    env.step(a0); twin.step(a0)                                     # the eager step that sizes the buffers a capture needs
    static = [torch.zeros(env.B, dtype=torch.int64, device=env.device) for _ in range(H)]
    outs = _outs(env, H)
    counter = env.env.step_counter
    g = _capture_steps(env, static, outs)
    assert env.env.step_counter == counter + H                     # the host counter counts the captured calls once
    done = False
    for seg in range(12):                                           # until every episode is done, then two segments more
        _segment(g, env, twin, static, outs, _fixed_actions(env, H, seed=seg), f'{kind} segment {seg}')
        if done:
            if seg >= done_at + 2:
                break
        elif bool(outs[-1]['done'].all()):
            done, done_at = True, seg
    assert done, 'the episodes never ended'
    assert env.env.step_counter == counter + H                     # replays do not advance it
    _assert_twins_equal(env, twin, kind)
    del g
    env.close(); twin.close()


def test_one_graph_replayed_across_three_eager_resets_equals_three_eager_segments():
    import torch
    env, twin = _twins('two', apply_action_mask=False)
    H = 6
    for e in (env, twin):
        e.record_steps(32)
    static = [torch.zeros(env.B, dtype=torch.int64, device=env.device) for _ in range(H)]
    outs = _outs(env, H)
    g = None
    for r in range(3):
        obs, t_obs = env.reset(), twin.reset()
        for k in ('model', 'graph_features', 'action_mask'):
            assert torch.equal(obs[k], t_obs[k]), (r, k)
        if g is None:
            a0 = _fixed_actions(env, 1, seed=7)[0]
            env.step(a0); twin.step(a0)
            g = _capture_steps(env, static, outs)
        _segment(g, env, twin, static, outs, _fixed_actions(env, H, seed=100 + r), f'reset {r}')
        _assert_twins_equal(env, twin, f'reset {r}')
    del g
    env.close(); twin.close()


# ---- the torch policy in the same graph ---------------------------------------------------------------------------------------

def _module(env, seed=3):
    from ddls_b200.torch_policy import TorchGNNPolicy
    return TorchGNNPolicy(env.static, env.n_actions, seed=seed)


def _greedy_graph(env, mod, H, obs0):
    """one graph: H decisions of argmax(logits) from the static obs0 on, each observation into its own static dict"""
    import torch
    outs = _outs(env, H)
    acts = []
    g = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(g):
        obs = obs0
        for t in range(H):
            logits, _ = mod(obs)
            a = logits.argmax(-1)
            acts.append(a)
            env.step(a, out=outs[t])
            obs = {k: outs[t][k] for k in ('model', 'graph_features', 'action_mask')}
    return g, outs, acts


def _eager_greedy(twin, mod, obs, H):
    import torch
    res = []
    with torch.no_grad():
        for t in range(H):
            logits, _ = mod(obs)
            a = logits.argmax(-1)
            o, r, d, _ = twin.step(a)
            res.append((a, _step_out(o, r, d)))
            obs = o
    return res


def test_greedy_policy_and_step_in_one_graph_equal_the_eager_loop_before_and_after_an_adam_step():
    import torch
    env, twin = _twins('one')
    mod = _module(env)
    H = 6
    obs0 = {k: v.clone() for k, v in env.reset().items()}
    t_obs = twin.reset()
    with torch.no_grad():                                           # the eager decision that uploads, embeds and sizes everything
        a = mod(obs0)[0].argmax(-1)
    obs0 = {k: v.clone() for k, v in env.step(a)[0].items()}
    t_obs = twin.step(a)[0]
    g, outs, acts = _greedy_graph(env, mod, H, obs0)
    static0 = {k: v for k, v in obs0.items()}
    for phase in range(2):
        if phase == 1:                                              # an Adam step on a loss over the last observations, then refresh()
            opt = torch.optim.Adam(mod.parameters(), lr=1e-2)
            logits, value = mod(t_obs)
            loss = torch.where(t_obs['action_mask'], logits, 0.0).logsumexp(-1).mean() + value.square().mean()
            opt.zero_grad()
            loss.backward()
            opt.step()
            mod.refresh()
        for seg in range(3):
            for k in static0:
                static0[k].copy_(t_obs[k])
            g.replay()
            want = _eager_greedy(twin, mod, t_obs, H)
            for t, (a, w) in enumerate(want):
                assert torch.equal(acts[t], a), (phase, seg, t)
                _assert_bits(outs[t], w, f'phase {phase} segment {seg} step {t}')
            t_obs = {k: want[-1][1][k] for k in ('model', 'graph_features', 'action_mask')}
    env.check(); twin.check()
    np.testing.assert_array_equal(env.decisions(), twin.decisions())
    _assert_same(env.episode_stats(), twin.episode_stats(), 'episode_stats')
    del g
    mod.close(); env.close(); twin.close()


def test_categorical_sampling_draws_afresh_on_each_replay_and_never_a_masked_action():
    import torch
    env, _twin = _twins('one')
    _twin.close()
    mod = _module(env, seed=5)
    obs = env.reset()
    gen = torch.Generator(device=env.device).manual_seed(2)
    with torch.no_grad():
        mod(obs)
    obs = {k: v.clone() for k, v in env.step(_draw(obs['action_mask'], gen))[0].items()}
    out = _outs(env, 1)[0]
    g = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(g):
        logits, _ = mod(obs)
        a = torch.distributions.Categorical(logits=logits, validate_args=False).sample()
        u = torch.rand(64, device=env.device)                       # the same generator's next draws, on their own
        mask_in = obs['action_mask'].clone()
        live_in = obs['model'] >= 0
        env.step(a, out=out)
    uniforms, n_live = [], []
    for r in range(10):
        g.replay()
        live = live_in.cpu().numpy()
        got = a.cpu().numpy()
        m = mask_in.cpu().numpy()
        assert m[live, got[live]].all(), f'replay {r}: a masked action was drawn'
        uniforms.append(u.cpu().numpy())
        n_live.append(int(live.sum()))
        for k in obs:
            obs[k].copy_(out[k])
    env.check()                                                     # apply_action_mask=True: a masked action would raise here
    assert all(not np.array_equal(x, y) for x, y in zip(uniforms, uniforms[1:])), 'a replay repeated the draws of the one before'
    n = env.decisions()
    assert n_live[0] == env.B and (n >= 2).all() and (n <= 11).all()
    del g
    mod.close(); env.close()


# ---- errors of replayed steps ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize('bad,apply_action_mask', [(17, True), (-1, False), (3, True)])
def test_a_bad_action_in_a_replay_is_reported_at_check_as_an_eager_step_reports_it(bad, apply_action_mask):
    import torch
    env, twin = _twins('one', apply_action_mask=apply_action_mask)
    obs, _ = env.reset(), twin.reset()
    assert not bool(obs['action_mask'][:, 3].any())                 # an odd degree above 1 is masked everywhere
    a = torch.zeros(env.B, dtype=torch.int64, device=env.device)
    env.step(a); twin.step(a)
    static = torch.zeros_like(a)
    out = _outs(env, 1)[0]
    g = _capture_steps(env, [static], [out])
    for r in range(3):                                              # good replays first: the call numbers move on
        g.replay(); twin.step(a)
    env.check(); twin.check()
    bad_a = a.clone()
    bad_a[4] = bad
    if bad != 3:                                                    # out of the set: the lowest episode of the call is the one kept
        bad_a[9] = bad
    static.copy_(bad_a)
    g.replay()
    twin.step(bad_a)
    with pytest.raises(Exception) as want:
        twin.check()
    with pytest.raises(Exception) as err:
        env.check()
    assert str(err.value) == str(want.value) and str(err.value).startswith('episode 4: '), (str(err.value), str(want.value))
    env.check()                                                     # raised once
    del g
    env.close(); twin.close()


# ---- refusals ----------------------------------------------------------------------------------------------------------------

def _refused(env, match):
    import torch
    a = torch.zeros(env.B, dtype=torch.int64, device=env.device)
    g = torch.cuda.CUDAGraph()
    with pytest.raises(Exception, match=match):
        with torch.cuda.graph(g):
            env.step(a)
    del g


def _steps_on_as_its_twin(env, twin, n=4, seed=6):
    """the environment's eager steps after a refused capture equal its twin's"""
    import torch
    gen = torch.Generator(device=env.device).manual_seed(seed)
    mask = env._export(None)['action_mask']
    for t in range(n):
        a = _draw(mask, gen)
        got = _step_out(*env.step(a)[:3])
        want = _step_out(*twin.step(a)[:3])
        _assert_bits(got, want, f'after the refusal, step {t}')
        mask = got['action_mask']
    env.check(); twin.check()
    np.testing.assert_array_equal(env.decisions(), twin.decisions())
    _assert_same(env.episode_stats(), twin.episode_stats(), 'episode_stats after the refusal')


def test_a_capture_before_any_eager_step_is_refused_and_the_environment_steps_on():
    env, twin = _twins('one')
    env.reset(); twin.reset()
    _refused(env, 'no eager step has run yet')
    _steps_on_as_its_twin(env, twin)
    env.close(); twin.close()


@pytest.mark.parametrize('place_on_device', [False, True])
def test_a_capture_the_device_tables_cannot_decide_is_refused(place_on_device):
    import torch
    from ddls_b200.torch_env import TorchRampJobPartitioningEnvironment
    shape, graphs, kw = _workload('one')
    env, twin = (TorchRampJobPartitioningEnvironment(shape, graphs, prewarm=False, place_on_device=place_on_device, **kw)
                 for _ in range(2))
    env.reset(); twin.reset()
    a = torch.zeros(env.B, dtype=torch.int64, device=env.device)
    env.step(a); twin.step(a)
    _refused(env, 'do not decide every placement')
    _steps_on_as_its_twin(env, twin)
    env.close(); twin.close()


def test_a_capture_with_a_template_on_the_cta_kernel_is_refused(monkeypatch):
    import torch
    monkeypatch.setenv('RAMP_LOOKAHEAD_MODE', 'cta')
    env, twin = _twins('one')
    env.reset(); twin.reset()
    a = torch.ones(env.B, dtype=torch.int64, device=env.device)
    env.step(a); twin.step(a)
    _refused(env, 'run on the CTA kernel')
    _steps_on_as_its_twin(env, twin)
    env.close(); twin.close()


def test_a_capture_after_a_template_was_registered_is_refused_until_an_eager_step():
    import torch
    from ddls_b200.template_builder import RampShape, build_template
    env, twin = _twins('one')
    env.reset(); twin.reset()
    a = torch.ones(env.B, dtype=torch.int64, device=env.device)
    env.step(a); twin.step(a)
    env.env.eng.register_template(build_template(_res2(), 8, RampShape(4, 4, 4)))
    _refused(env, 'registered since the last eager step')
    _steps_on_as_its_twin(env, twin)
    static, out = torch.zeros_like(a), _outs(env, 1)[0]
    g = _capture_steps(env, [static], [out])                         # the eager steps sized the scratch again
    g.replay()
    want = _step_out(*twin.step(static)[:3])
    _assert_bits(out, want, 'the capture after an eager step')
    del g
    env.close(); twin.close()


def test_policy_captures_that_would_need_the_host_are_refused_by_name():
    import torch
    env, twin = _twins('one')
    mod = _module(env)
    obs = env.reset()
    twin.reset()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(Exception, match='weights changed since they were last uploaded'):   # never uploaded
        with torch.no_grad(), torch.cuda.graph(g):
            mod(obs)
    with torch.no_grad():
        mod(obs)
    with torch.no_grad():
        mod.weight.add_(1e-3)                                        # an in-place change: a new version
    with pytest.raises(Exception, match='weights changed since they were last uploaded'):
        with torch.no_grad(), torch.cuda.graph(torch.cuda.CUDAGraph()):
            mod(obs)
    mod.refresh()
    big = {k: torch.cat([v, v]) for k, v in obs.items()}
    with pytest.raises(Exception, match='staging would have to grow'):
        with torch.no_grad(), torch.cuda.graph(torch.cuda.CUDAGraph()):
            mod(big)
    with pytest.raises(Exception, match='backward of TorchGNNPolicy is not capturable'):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            logits, value = mod(obs)
            (logits.sum() + value.sum()).backward()
    mod.weight.grad = None
    with pytest.raises(Exception, match='reset\\(\\) draws the arrival streams'):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            env.reset()
    # the module still gives the eager bits, and the environment steps on as its twin
    with torch.no_grad():
        logits, value = mod(obs)
        mod2 = _module(env)
        mod2.load_gnn_state_dict(mod.gnn_state_dict())
        l2, v2 = mod2(obs)
    assert torch.equal(logits, l2) and torch.equal(value, v2)
    _steps_on_as_its_twin(env, twin)
    mod.close(); mod2.close(); env.close(); twin.close()


# ---- memory ----------------------------------------------------------------------------------------------------------------

def test_every_byte_comes_back_after_the_graph_is_destroyed():
    import torch
    from ddls_b200 import engine
    before = engine.device_bytes()
    env, twin = _twins('one')
    twin.close()
    mod = _module(env)
    obs0 = {k: v.clone() for k, v in env.reset().items()}
    with torch.no_grad():
        a = mod(obs0)[0].argmax(-1)
    obs0 = {k: v.clone() for k, v in env.step(a)[0].items()}
    g, outs, acts = _greedy_graph(env, mod, 4, obs0)
    for _ in range(3):
        g.replay()
    env.check()
    assert engine.device_bytes()[0] > before[0]
    del g, outs, acts
    torch.cuda.synchronize()
    env.close(); mod.close()
    assert engine.device_bytes() == before
