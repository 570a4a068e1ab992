"""-m gpu: the device GNN policy as a torch module (ddls_b200/torch_policy.py: ramp_policy_forward_device / _backward_device on the
caller's stream).  Its forward and its autograd gradient are the host-input path's bits (ramp_policy_forward / ramp_policy_backward)
on every configuration the kernel tests use, at 1 to 16,385 rows, int32 and int64 models, dead rows and strided graph features; it
reads the torch environment as DeviceGNNPolicy.act reads the device environment; PPO and PG losses written in torch give the fused
learners' statistics and gradients; calls are ordered on the caller's stream without a synchronisation; autograd's rules hold;
and it gives back every byte it took.

Losses: both sides compute the same forward bits, so they differ only by the fp32 rounding of the upstream gradient (torch's
autograd of the loss against the learner kernel's own derivative).  Statistics agree to 1e-6 and each weight tensor's gradient to
1e-5 relative (its norm)."""
import numpy as np
import pytest

from test_gpu_algo_model import _model as algo_model
from test_gpu_policy_kernels import CONFIGS, _cfg, graphs, raw_policy

pytestmark = pytest.mark.gpu

SEED = 3
STAT_TOL = 1e-6
PART_REL = 1e-5
ALL = dict({k: (_cfg(over), A, big) for k, (over, A, _, big) in CONFIGS.items()},
           **{'H17-separate': (algo_model(17, 0), 17, False), 'H17-shared': (algo_model(17, 1), 17, False)})


def _statics(gs):
    return [dict(node_features=g.nf, edge_features=g.ef, edges_src=g.src, edges_dst=g.dst, graph_static=g.gs) for g in gs]


class Case:
    pass


@pytest.fixture(scope='module', params=list(ALL))
def case(request):
    """the host-input policy and the torch module on the same raw graphs and weights"""
    from ddls_b200 import policy as P
    from ddls_b200.torch_policy import TorchGNNPolicy
    c, A, big = ALL[request.param]
    k = Case()
    k.id, k.c, k.A = request.param, c, A
    rng = np.random.default_rng(5)
    k.graphs = [g.features(c, rng) for g in graphs(big)]
    k.sd = P.random_state_dict(c, A, seed=SEED)
    k.pol = raw_policy(c, A, k.graphs, k.sd)
    k.mod = TorchGNNPolicy(_statics(k.graphs), A, c, k.sd)
    yield k
    k.mod.close()
    k.pol.close()


def _rows(k, n, seed):
    """n rows: random models with dead rows (-1) scattered, N(0, 1) graph features, masks at p = 0.7 with one valid action"""
    rng = np.random.default_rng(seed)
    model = rng.integers(0, k.pol.n_models, n).astype(np.int32)
    model[rng.random(n) < 0.1] = -1
    gf = rng.standard_normal((n, k.c['in_features_graph'])).astype(np.float32)
    mask = (rng.random((n, k.A)) < 0.7).astype(np.uint8)
    mask[np.arange(n), rng.integers(0, k.A, n)] = 1
    return model, gf, mask


def _obs(k, model, gf, mask, dtype, layout):
    """the rows as the module takes them: graph features as the environment's [n, G + A] rows, or a non-contiguous slice"""
    import torch
    dev = k.mod.device
    m = torch.from_numpy(model.astype(np.int64)).to(dev).to(getattr(torch, dtype))
    g = torch.from_numpy(gf).to(dev)
    msk = torch.from_numpy(mask.astype(bool)).to(dev)
    if layout == 'env':
        g = torch.cat([g, msk.to(torch.float32)], 1)
    elif layout == 'slice':
        big = torch.full((2 * len(gf), gf.shape[1] + 3), np.nan, device=dev)
        big[::2, 1:1 + gf.shape[1]] = g
        g = big[::2, 1:1 + gf.shape[1]]
        assert len(gf) == 1 or not g.is_contiguous()
    return {'model': m, 'graph_features': g, 'action_mask': msk}


def _bits_equal(got, want, what):
    got = got.detach().cpu().numpy() if hasattr(got, 'detach') else np.asarray(got)
    want = np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.flatnonzero(got.view(np.uint32).ravel() != want.astype(np.float32).view(np.uint32).ravel())
    assert not len(bad), f'{what}: {len(bad)} of {got.size} differ, first at {bad[0]}: {got.ravel()[bad[0]]!r} vs {want.ravel()[bad[0]]!r}'


# ---- forward and backward against the host-input path -----------------------------------------------------------------------

@pytest.mark.parametrize('n', [1, 33, 4096, 16385])
@pytest.mark.parametrize('dtype,layout', [('int32', 'env'), ('int64', 'env'), ('int64', 'slice'), ('int32', 'plain')])
def test_forward_equals_the_host_path_bit_for_bit(case, n, dtype, layout):
    import torch
    model, gf, mask = _rows(case, n, seed=n)
    obs = _obs(case, model, gf, mask, dtype, layout)
    if dtype == 'int64' and n > 2:
        obs['model'][1] = 2 ** 32 + int(model[1] if model[1] >= 0 else 0)      # would wrap into range as int32
        model = model.copy(); model[1] = -1
    with torch.no_grad():
        logits, value = case.mod(obs)
    wl, wv = case.pol.forward(model, gf, mask)
    _bits_equal(logits, wl, f'{case.id} n={n} logits')
    _bits_equal(value, wv, f'{case.id} n={n} value')
    dead = model < 0
    assert (wl[dead] == 0).all() and (wv[dead] == 0).all()


def test_a_rollout_buffer_goes_in_whole(case):
    import torch
    T, B = 3, 50
    model, gf, mask = _rows(case, T * B, seed=11)
    obs = _obs(case, model, gf, mask, 'int64', 'env')
    obs = {k: v.reshape((T, B) + tuple(v.shape[1:])) for k, v in obs.items()}
    with torch.no_grad():
        logits, value = case.mod(obs)
    assert logits.shape == (T, B, case.A) and value.shape == (T, B)
    wl, wv = case.pol.forward(model, gf, mask)
    _bits_equal(logits.reshape(T * B, case.A), wl, 'logits')
    _bits_equal(value.reshape(-1), wv, 'value')


@pytest.mark.parametrize('n', [1, 33, 4096, 16385])
def test_backward_equals_the_host_path_bit_for_bit(case, n):
    import torch
    model, gf, mask = _rows(case, n, seed=100 + n)
    rng = np.random.default_rng(n)
    gl = rng.standard_normal((n, case.A)).astype(np.float32)
    gv = rng.standard_normal(n).astype(np.float32)
    obs = _obs(case, model, gf, mask, 'int64', 'env')
    logits, value = case.mod(obs)
    loss = (torch.from_numpy(gl).to(logits.device) * logits).sum() + (torch.from_numpy(gv).to(value.device) * value).sum()
    (grad,) = torch.autograd.grad(loss, case.mod.weight)
    want = case.pol.backward(model, gf, mask, gl, gv)
    _bits_equal(grad, want, f'{case.id} n={n} weight gradient')


# ---- on the torch environment --------------------------------------------------------------------------------------------

def test_it_reads_the_torch_environment_as_the_device_policy_reads_its_twin():
    import torch
    from ddls_b200 import policy as P
    from ddls_b200 import synth
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    from ddls_b200.torch_policy import TorchGNNPolicy
    from ddls_b200.torch_env import TorchRampJobPartitioningEnvironment
    graphs = [synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3), synth.chain_graph(6, 'chain6')]
    kw = dict(n_episodes=256, jobs_per_episode=6, seed=9, prewarm=True)
    t_env = TorchRampJobPartitioningEnvironment((4, 4, 4), graphs, **kw)
    h_env = DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, **kw)
    A = t_env.n_actions
    sd = P.random_state_dict(dict(P.DEFAULT_CONFIG), A, seed=7)
    pol = P.DeviceGNNPolicy(graphs, A, state_dict=sd)
    mod = TorchGNNPolicy(t_env.static, A, state_dict=sd)
    obs = t_env.reset(); h_env.reset()
    done = torch.zeros(t_env.B, dtype=torch.bool, device=t_env.device)
    rows = 0
    for n in range(10):
        pol.act(h_env, sample=True, seed=n)
        got = pol.read(h_env)
        with torch.no_grad():
            logits, value = mod(obs)
        live = ((obs['model'] >= 0) & ~done).cpu().numpy()             # act also skips the finished episodes
        _bits_equal(logits[live], got['logits'][live], f'step {n} logits')
        _bits_equal(value[live], got['value'][live], f'step {n} value')
        rows += int(live.sum())
        obs, reward, done, _ = t_env.step(torch.from_numpy(got['actions']).to(t_env.device))
        h_env.step_device()
        if bool(done.all()):
            break
    t_env.check()
    assert rows > 256
    mod.close(); pol.close(); t_env.close(); h_env.close()


# ---- losses written in torch against the fused learners ------------------------------------------------------------------

def _learner_case(A=17, n=300, seed=4, config=None):
    """a DeviceGNNPolicy and the module at the same weights, and one minibatch whose rows are all live"""
    from ddls_b200 import policy as P
    from ddls_b200 import synth
    from ddls_b200.torch_policy import TorchGNNPolicy
    gs = [synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3), synth.chain_graph(6, 'chain6')]
    c = dict(config or P.DEFAULT_CONFIG)
    sd = P.random_state_dict(c, A, seed=seed)
    pol = P.DeviceGNNPolicy(gs, A, c, sd)
    mod = TorchGNNPolicy(gs, A, c, sd)
    k = Case()
    k.c, k.A, k.pol, k.mod = c, A, pol, mod
    model, gf, mask = _rows(k, n, seed=seed)
    model = np.abs(model) % len(gs)
    rng = np.random.default_rng(seed + 1)
    action = np.array([rng.choice(np.flatnonzero(m)) for m in mask], dtype=np.int32)
    return k, dict(model=model, graph_features=gf, action_mask=mask, action=action,
                   advantage=rng.standard_normal(n).astype(np.float32), value_target=rng.standard_normal(n).astype(np.float32))


def _check_parts(grad, want, c, A, what):
    from ddls_b200 import policy as P
    got = grad.detach().cpu().numpy()
    parts = P.unpack_weights(got, c, A)
    for key, ref in P.unpack_weights(want, c, A).items():
        d = np.linalg.norm(parts[key].astype(np.float64) - ref)
        assert d <= PART_REL * max(np.linalg.norm(ref.astype(np.float64)), 1e-30), f'{what} {key}: relative difference {d / np.linalg.norm(ref):.3e}'


def test_ppo_loss_in_torch_agrees_with_the_fused_learner():
    import torch
    from ddls_b200.learn import DevicePPOLearner, PPOConfig
    from ppo_reference import ppo_loss64
    k, b = _learner_case()
    cfg = PPOConfig()
    old, _ = k.pol.forward(b['model'], b['graph_features'], b['action_mask'])
    old = old + np.random.default_rng(3).normal(0, 0.05, old.shape).astype(np.float32)
    stats, want = DevicePPOLearner(k.pol, cfg).loss_and_grad(dict(b, old_logits=old))
    obs = _obs(k, b['model'], b['graph_features'], b['action_mask'], 'int32', 'env')
    logits, value = k.mod(obs)
    total, st = ppo_loss64(logits.cpu(), value.cpu(), b['action'], old, b['advantage'], b['value_target'], cfg)   # autograd follows .cpu()
    (grad,) = torch.autograd.grad(total, k.mod.weight)
    for key in ('total_loss', 'policy_loss', 'vf_loss', 'entropy', 'kl'):
        assert abs(st[key] - stats[key]) <= STAT_TOL * max(1.0, abs(stats[key])), (key, st[key], stats[key])
    _check_parts(grad, want, k.c, k.A, 'ppo')
    k.mod.close(); k.pol.close()


def test_pg_loss_in_torch_agrees_with_the_fused_learner():
    import torch
    from ddls_b200.learn import DevicePGLearner
    k, b = _learner_case(seed=6)
    stats, want = DevicePGLearner(k.pol).loss_and_grad(b)
    obs = _obs(k, b['model'], b['graph_features'], b['action_mask'], 'int64', 'env')
    logits, _ = k.mod(obs)
    dev = logits.device
    logp = torch.log_softmax(logits, -1).gather(1, torch.from_numpy(b['action'].astype(np.int64)).to(dev)[:, None])[:, 0]
    loss = -(logp * torch.from_numpy(b['advantage']).to(dev)).mean()
    ent = -(torch.softmax(logits, -1) * torch.log_softmax(logits, -1)).sum(-1).mean()
    (grad,) = torch.autograd.grad(loss, k.mod.weight)
    for key, x in (('policy_loss', loss), ('entropy', ent)):
        assert abs(float(x.detach()) - stats[key]) <= STAT_TOL * max(1.0, abs(stats[key])), (key, float(x.detach()), stats[key])
    _check_parts(grad, want, k.c, k.A, 'pg')
    k.mod.close(); k.pol.close()


# ---- stream order ------------------------------------------------------------------------------------------------------------

def _small_module():
    from ddls_b200 import policy as P
    from ddls_b200 import synth
    from ddls_b200.torch_policy import TorchGNNPolicy
    gs = [synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3), synth.chain_graph(6, 'chain6')]
    sd = P.random_state_dict(dict(P.DEFAULT_CONFIG), 17, seed=2)
    k = Case()
    k.c, k.A = dict(P.DEFAULT_CONFIG), 17
    k.pol, k.mod = P.DeviceGNNPolicy(gs, 17, state_dict=sd), TorchGNNPolicy(gs, 17, state_dict=sd)
    return k


def _fwd_bwd(k, obs, gl):
    import torch
    logits, value = k.mod(obs)
    (grad,) = torch.autograd.grad((gl * logits).sum() + value.sum(), k.mod.weight)
    return logits.detach(), value.detach(), grad


def test_calls_on_a_side_stream_behind_a_sleep_and_alternating_streams_give_the_same_bits():
    import torch
    k = _small_module()
    cur = torch.cuda.current_stream(k.mod.device)
    batches = []
    for s in range(4):
        model, gf, mask = _rows(k, 500 + 37 * s, seed=s)
        obs = _obs(k, model, gf, mask, 'int64', 'env')
        batches.append((obs, torch.randn(len(model), k.A, device=k.mod.device)))
    ref = [_fwd_bwd(k, obs, gl) for obs, gl in batches]
    sides = [torch.cuda.Stream(device=k.mod.device), torch.cuda.Stream(device=k.mod.device)]
    for s in sides:
        s.wait_stream(cur)
    outs = []
    for i, (obs, gl) in enumerate(batches):
        with torch.cuda.stream(sides[i % 2]):
            torch.cuda._sleep(20_000_000)
            outs.append(_fwd_bwd(k, obs, gl))
    for s in sides:
        cur.wait_stream(s)
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(outs, ref)):
        for x, y, what in zip(a, b, ('logits', 'value', 'grad')):
            assert torch.equal(x, y), (i, what)
    k.mod.close(); k.pol.close()


def test_after_warm_up_forward_and_backward_do_not_wait_for_the_stream():
    import torch
    k = _small_module()
    model, gf, mask = _rows(k, 777, seed=9)
    obs = _obs(k, model, gf, mask, 'int64', 'env')
    gl = torch.randn(777, k.A, device=k.mod.device)
    with torch.no_grad():
        k.mod(obs)
    _fwd_bwd(k, obs, gl)                                            # every buffer sized, the row count seen once
    cur = torch.cuda.current_stream(k.mod.device)
    cur.synchronize()
    torch.cuda._sleep(500_000_000)
    with torch.no_grad():
        logits, value = k.mod(obs)
    assert not cur.query()                                          # the no-grad forward returned while the stream slept
    cur.synchronize()
    torch.cuda._sleep(500_000_000)
    l2, v2, grad = _fwd_bwd(k, obs, gl)
    assert not cur.query()                                          # forward + backward returned while the stream slept
    cur.synchronize()
    wl, wv = k.pol.forward(model, gf, mask)
    _bits_equal(logits, wl, 'logits'); _bits_equal(l2, wl, 'logits'); _bits_equal(value, wv, 'value')
    _bits_equal(grad, k.pol.backward(model, gf, mask, gl.cpu().numpy(), np.ones(777, np.float32)), 'grad')
    k.mod.close(); k.pol.close()


def test_an_optimizer_step_refreshes_the_embeddings():
    import torch
    k = _small_module()
    model, gf, mask = _rows(k, 300, seed=12)
    obs = _obs(k, model, gf, mask, 'int32', 'env')
    opt = torch.optim.Adam(k.mod.parameters(), lr=1e-2)
    for it in range(3):
        logits, value = k.mod(obs)
        loss = logits.logsumexp(-1).mean() + value.square().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        k.pol.set_weights(k.mod.weight.detach().cpu().numpy())
        with torch.no_grad():
            logits, value = k.mod(obs)
        wl, wv = k.pol.forward(model, gf, mask)
        _bits_equal(logits, wl, f'iteration {it} logits'); _bits_equal(value, wv, f'iteration {it} value')
    k.mod.close(); k.pol.close()


# ---- autograd's rules --------------------------------------------------------------------------------------------------------

def test_autograd_rules():
    import torch
    k = _small_module()
    model, gf, mask = _rows(k, 400, seed=13)
    obs = _obs(k, model, gf, mask, 'int64', 'env')
    obs['graph_features'].requires_grad_(True)
    logits, value = k.mod(obs)
    (g,) = torch.autograd.grad(logits.sum() + value.sum(), k.mod.weight, create_graph=True)
    with pytest.raises(RuntimeError):                                # once_differentiable: no double backward
        torch.autograd.grad(g.sum(), k.mod.weight)
    logits, value = k.mod(obs)
    gw, gx = torch.autograd.grad(logits.sum(), [k.mod.weight, obs['graph_features']], allow_unused=True)
    assert gw is not None and (gx is None or not bool(gx.any()))     # the observation gets no gradient
    logits, value = k.mod(obs)
    with torch.no_grad():
        k.mod.weight.add_(1e-3)
    with pytest.raises(RuntimeError, match='modified by an inplace operation'):
        (logits.sum() + value.sum()).backward()
    # the summed losses of two halves are the whole batch's gradient
    obs = {kk: v.detach() for kk, v in obs.items()}
    def loss_of(o):                                                  # a masked logit is -FLT_MAX: leave it out of the square
        logits, value = k.mod(o)
        return torch.where(o['action_mask'], logits, 0.0).square().sum() + value.square().sum()
    whole = torch.autograd.grad(loss_of(obs), k.mod.weight)[0]
    halves = [{kk: v[s] for kk, v in obs.items()} for s in (slice(0, 200), slice(200, 400))]
    loss = sum(loss_of(h) for h in halves)
    split = torch.autograd.grad(loss, k.mod.weight)[0]
    assert float((split - whole).norm()) <= 1e-6 * float(whole.norm())
    k.mod.close(); k.pol.close()


def test_bad_inputs_raise_with_a_message():
    import torch
    k = _small_module()
    model, gf, mask = _rows(k, 8, seed=1)
    obs = _obs(k, model, gf, mask, 'int64', 'env')
    with pytest.raises(TypeError, match='model must be int32 or int64'):
        k.mod(dict(obs, model=obs['model'].float()))
    with pytest.raises(ValueError, match='is on cpu'):
        k.mod(dict(obs, action_mask=obs['action_mask'].cpu()))
    with pytest.raises(ValueError, match='graph_features have shape'):
        k.mod(dict(obs, graph_features=obs['graph_features'][:, :5]))
    with pytest.raises(TypeError, match='graph_features must be float32'):
        k.mod(dict(obs, graph_features=obs['graph_features'].double()))
    with pytest.raises(ValueError, match='action_mask has shape'):
        k.mod(dict(obs, action_mask=obs['action_mask'][:, :3]))
    k.mod.close(); k.pol.close()


# ---- memory ----------------------------------------------------------------------------------------------------------------

def test_every_byte_comes_back_a_failed_construction_included():
    import torch
    from ddls_b200 import engine, synth
    from ddls_b200.torch_policy import TorchGNNPolicy
    gs = [synth.chain_graph(6, 'chain6')]
    before = engine.device_bytes()
    mod = TorchGNNPolicy(gs, 17)
    model = torch.zeros(64, dtype=torch.int64, device=mod.device)
    obs = {'model': model, 'graph_features': torch.randn(64, 34, device=mod.device),
           'action_mask': torch.ones(64, 17, dtype=torch.bool, device=mod.device)}
    logits, value = mod(obs)
    (logits.sum() + value.sum()).backward()
    torch.cuda.synchronize()
    assert engine.device_bytes()[0] > before[0]
    mod.close()
    assert engine.device_bytes() == before
    with pytest.raises(Exception, match='fcnet_hidden'):
        TorchGNNPolicy(gs, 17, config={'fcnet_hiddens': (100,)})
    assert engine.device_bytes() == before
    # a failure after ramp_policy_create: the second job type names a node it does not have, which ramp_policy_set_model refuses
    # once the first one is registered, so the constructor's clean-up frees the policy
    from ddls_b200.observation import static_observation
    st = dict(static_observation(gs[0]))
    bad = dict(st, edges_src=np.array(st['edges_src']).copy())
    bad['edges_src'][0] = len(st['node_features']) + 5
    with pytest.raises(Exception, match='names node'):
        TorchGNNPolicy([st, bad], 17)
    assert engine.device_bytes() == before


# ---- held to float64, and a training step written in torch against the fused one ---------------------------------------

def _module_grad(mod, b, loss_fn):
    """the module's autograd gradient (blob order) of loss_fn(logits, value) over the rows of b; the loss is computed on the host
    in fp32 from the module's outputs, autograd following .cpu()"""
    import torch
    dev = mod.device
    obs = {'model': torch.from_numpy(np.asarray(b['model'], dtype=np.int64)).to(dev),
           'graph_features': torch.from_numpy(np.ascontiguousarray(b['graph_features'], dtype=np.float32)).to(dev),
           'action_mask': torch.from_numpy(np.asarray(b['action_mask']).astype(bool)).to(dev)}
    logits, value = mod(obs)
    (g,) = torch.autograd.grad(loss_fn(logits.cpu(), value.cpu()), mod.weight)
    return g.cpu().numpy()


@pytest.mark.parametrize('wseed', [2, 4])
@pytest.mark.parametrize('eid', ['cfg3', 'mix128', 'bench_types'])
def test_module_gradients_on_recorded_batches_are_held_to_float64(eid, wseed):
    """tests/test_gpu_learn_grad_recorded.py's rule for the module: PPO's and PG's gradients on the batches those learners form
    from a recorded segment, each tensor within max(1e-4, 10 e32) of float64 once tie_reference.explain() has accounted for the
    flips of named near-tied units"""
    from test_gpu_learn_grad_recorded import ENVS, _make_env
    kind, B, J = ENVS[eid]
    env, graphs = _make_env(kind, B, J)
    module_gradients_on_a_recorded_batch(env, graphs, J, wseed, f'module {eid} seed {wseed}')


def module_gradients_on_a_recorded_batch(env, graphs, J, wseed, tag):
    """TorchGNNPolicy's PPO and PG gradients on a J-step segment of env recorded at weight seed wseed, explained against float64.
    Closes env."""
    from ddls_b200 import policy as P
    from ddls_b200.learn import DevicePPOLearner, PGConfig, PPOConfig
    from ddls_b200.torch_policy import TorchGNNPolicy
    from pg_reference import train_rows
    from test_gpu_learn_grad_recorded import check_explained, pg_loss, ppo_loss
    from test_gpu_policy_learn import host_batch
    A = env.max_partitions_per_op + 1
    sd = P.random_state_dict(P.DEFAULT_CONFIG, A, seed=wseed)
    pol = P.DeviceGNNPolicy(graphs, A, None, sd)
    mod = TorchGNNPolicy(pol.static, A, state_dict=sd)
    try:
        traj = {k: np.array(v) for k, v in pol.collect(env, J, sample=True, seed=3).items()}
        probe = DevicePPOLearner(pol, PPOConfig(num_sgd_iter=0))
        probe.learn(env, J)
        b = host_batch(pol, traj, probe.train_batch(env))
        assert len(b['model']) > 100
        g = _module_grad(mod, b, ppo_loss(b, PPOConfig()))
        check_explained(pol, f'ppo {tag}', g, b['model'], b['graph_features'], b['action_mask'], ppo_loss(b, PPOConfig()))
        b = train_rows(pol, traj, PGConfig().gamma)
        g = _module_grad(mod, b, pg_loss(b))
        check_explained(pol, f'pg {tag}', g, b['model'], b['graph_features'], b['action_mask'], pg_loss(b))
    finally:
        mod.close(); pol.close(); env.close()


@pytest.mark.parametrize('cid', ['truncated', 'mid_segment'])
def test_a_torch_adam_step_on_the_pg_loss_gives_the_fused_learners_weights(cid):
    """one torch.optim.Adam step on the module's PG loss (pg_torch_loss: -mean(log p(a) return)) over DevicePGLearner's train
    batch gives DevicePGLearner.learn's weights, each tensor to tests/test_gpu_pg_learn.py's composition-replay bound (1e-5)"""
    import torch
    from ddls_b200 import policy as P
    from ddls_b200.learn import DevicePGLearner, PGConfig
    from ddls_b200.torch_policy import TorchGNNPolicy
    from pg_reference import train_rows
    from test_gpu_pg_learn import CASES, PARTS_REL, _policy, _rel
    from test_gpu_policy_learn import _env
    case = CASES[cid]
    env, graphs = _env(B=case['B'], J=case['J'], seed=7)
    pol = _policy(graphs)
    mod = TorchGNNPolicy(pol.static, pol.n_actions, state_dict=pol.state_dict())
    try:
        H, cfg = case['H'], PGConfig(**case['cfg'])
        traj = {k: np.array(v) for k, v in pol.collect(env, H, sample=True, seed=3).items()}
        b = train_rows(pol, traj, cfg.gamma)
        assert len(b['model']) > 100
        lrn = DevicePGLearner(pol, cfg)
        lrn.reset()
        lrn.learn(env, H)
        want = pol.get_weights()
        opt = torch.optim.Adam(mod.parameters(), lr=cfg.lr, betas=(cfg.adam_beta1, cfg.adam_beta2), eps=cfg.adam_eps)
        dev = mod.device
        obs = {'model': torch.from_numpy(np.asarray(b['model'], dtype=np.int64)).to(dev),
               'graph_features': torch.from_numpy(np.ascontiguousarray(b['graph_features'], dtype=np.float32)).to(dev),
               'action_mask': torch.from_numpy(np.asarray(b['action_mask']).astype(bool)).to(dev)}
        logits, _ = mod(obs)
        action = torch.from_numpy(np.asarray(b['action'], dtype=np.int64)).to(dev)
        ret = torch.from_numpy(np.asarray(b['advantage'], dtype=np.float32)).to(dev)
        loss = -(torch.log_softmax(logits, -1).gather(1, action[:, None])[:, 0] * ret).mean()
        opt.zero_grad()
        loss.backward()
        if cfg.grad_clip > 0:
            torch.nn.utils.clip_grad_norm_(mod.parameters(), cfg.grad_clip)
        opt.step()
        got = P.unpack_weights(mod.weight.detach().cpu().numpy(), pol.config, pol.n_actions)
        ref = P.unpack_weights(want, pol.config, pol.n_actions)
        errs = {k: _rel(got[k], ref[k].astype(np.float64)) for k in ref}
        bad = {k: e for k, e in errs.items() if not e <= PARTS_REL}
        assert not bad, f'{cid}: the torch step is off the fused learner: {bad}'
    finally:
        mod.close(); pol.close(); env.close()
