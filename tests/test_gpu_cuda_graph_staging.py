"""-m gpu: what a captured graph holds stays where it is while the graph lives.  A forward captured at B rows keeps its staging
when a training forward and backward over a larger batch outgrow it, so replays after the Adam step and refresh() still equal the
eager twin.  Once a step was captured, registering a template (which could regrow the lookahead scratch) and re-making the tick
lists are refused by name, and the graph replays on as before."""
import pytest

from test_gpu_cuda_graph import _assert_bits, _capture_steps, _eager_greedy, _greedy_graph, _module, _outs, _res2, _step_out, _twins

pytestmark = pytest.mark.gpu

OBS = ('model', 'graph_features', 'action_mask')


def test_replays_after_a_larger_training_batch_an_adam_step_and_refresh_equal_the_eager_twin():
    import torch
    env, twin = _twins('one')
    mod = _module(env, seed=4)
    H = 4
    obs0 = {k: v.clone() for k, v in env.reset().items()}
    t_obs = twin.reset()
    with torch.no_grad():
        a = mod(obs0)[0].argmax(-1)
    obs0 = {k: v.clone() for k, v in env.step(a)[0].items()}
    t_obs = twin.step(a)[0]
    g, outs, acts = _greedy_graph(env, mod, H, obs0)                # the forward's staging holds B rows
    # a training forward and backward over a [4, B] batch: four times the rows the captured forward staged
    batch = {k: torch.stack([t_obs[k]] * 4) for k in OBS}
    opt = torch.optim.Adam(mod.parameters(), lr=1e-2)
    logits, value = mod(batch)
    loss = torch.where(batch['action_mask'], logits, 0.0).logsumexp(-1).mean() + value.square().mean()
    opt.zero_grad()
    loss.backward()
    opt.step()
    mod.refresh()
    junk = [torch.full((1 << 20,), 7.0, device=env.device) for _ in range(16)]   # memory freed staging could have gone back to
    for seg in range(3):
        for k in OBS:
            obs0[k].copy_(t_obs[k])
        g.replay()
        want = _eager_greedy(twin, mod, t_obs, H)
        for t, (a, w) in enumerate(want):
            assert torch.equal(acts[t], a), (seg, t)
            _assert_bits(outs[t], w, f'segment {seg} step {t}')
        t_obs = {k: want[-1][1][k] for k in OBS}
    assert all(bool((j == 7.0).all()) for j in junk)
    env.check(); twin.check()
    del g
    mod.close(); env.close(); twin.close()


def test_once_a_step_was_captured_template_registration_and_new_tick_lists_are_refused():
    import torch
    from ddls_b200.template_builder import RampShape, build_template
    env, twin = _twins('one')
    env.reset(); twin.reset()
    a = torch.ones(env.B, dtype=torch.int64, device=env.device)
    env.step(a); twin.step(a)
    static, out = torch.zeros_like(a), _outs(env, 1)[0]
    g = _capture_steps(env, [static], [out])
    with pytest.raises(Exception, match='no template can be registered once a step was captured'):
        env.env.eng.register_template(build_template(_res2(), 8, RampShape(4, 4, 4)))
    with pytest.raises(Exception, match='a step was captured into a CUDA graph'):
        env.env.eng.enable_tick_lists(64)
    for r in range(3):
        g.replay()
        _assert_bits(out, _step_out(*twin.step(static)[:3]), f'replay {r}')
    env.check(); twin.check()
    del g
    env.close(); twin.close()
