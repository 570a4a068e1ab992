"""-m gpu: the policy's gradient and the PPO learner step on the device (ddls_b200/csrc/ramp_policy_learn.cuh) against float64 torch
restatements (tests/ppo_reference.py): the backward at every configuration tests/test_gpu_policy_kernels.py uses, PPO's loss and
gradient, the first pass's recomputed log-probabilities, GAE, Adam + clipping, determinism, progress on a fixed batch, memory.

Gradient bound: for every weight tensor ||g - g64|| / ||g64|| <= max(1e-4, 10 e32), where e32 is the same error of torch's own
fp32 autograd through the same restatement, computed in the test.  Where fp32 reaches 1e-4 that is the bound; where it cannot --
'max': 8 leaky-relu rounds over the 20,000-node graph, where pre-activations within rounding of 0 take the other slope in any
fp32 computation -- the kernel is held to fp32's own error.  The largest error per case, and torch fp32's on the same tensor,
are printed (pytest -s)."""
import dataclasses

import numpy as np
import pytest

from ppo_reference import shuffle_order

pytestmark = pytest.mark.gpu

REL = 1e-4
FP32_FACTOR = 10


def _kernels():
    import test_gpu_policy_kernels as K
    return K


def tensor_errors(got_blob, ref, c, A):
    from ddls_b200 import policy as P
    got = P.unpack_weights(got_blob, c, A)
    out = {}
    for k, g64 in ref.items():
        err, nrm = np.linalg.norm(got[k].astype(np.float64) - g64), np.linalg.norm(g64)
        out[k] = err / nrm if nrm > 0 else err
    return out


def check_tensors(errs, what, fp32=None):
    """errs: per tensor relative errors; fp32: torch fp32 autograd's on the same tensors (None: the bound is REL)"""
    bound = {k: max(REL, FP32_FACTOR * fp32[k]) if fp32 else REL for k in errs}
    worst = max(errs, key=errs.get)
    print(f'{what}: largest relative error {errs[worst]:.3e} ({worst})' + (f', torch fp32 {fp32[worst]:.3e}' if fp32 else '') +
          (f'; torch fp32 worst {max(fp32.values()):.3e}' if fp32 else ''))
    bad = {k: (v, bound[k]) for k, v in errs.items() if not v <= bound[k]}
    assert not bad, f'{what}: {bad}'


def ref_grads(loss, p):
    import torch
    gs = torch.autograd.grad(loss, list(p.values()), allow_unused=True)
    return {k: (g.numpy() if g is not None else np.zeros(tuple(v.shape))) for (k, v), g in zip(p.items(), gs)}


def rows(n_models, A, c, n, seed, dead=True):
    rng = np.random.default_rng(seed)
    model = rng.integers(0, n_models, n).astype(np.int32)
    if dead:
        model[[1, n // 2]] = -1
    gf = rng.standard_normal((n, c['in_features_graph'])).astype(np.float32)
    mask = (rng.random((n, A)) < 0.6).astype(np.uint8)
    mask[np.arange(n), rng.integers(0, A, n)] = 1                     # at least one valid action (action 0 always is, in the env)
    return model, gf, mask


def backward_case(pol, c, A, gs, sd, seed, what):
    from ppo_reference import params64, policy64
    import torch
    n = 48
    model, gf, mask = rows(len(gs), A, c, n, seed)
    rng = np.random.default_rng(seed + 1)
    gl = rng.standard_normal((n, A)).astype(np.float32)
    gv = rng.standard_normal(n).astype(np.float32)
    got = pol.backward(model, gf, mask, gl, gv)
    live = model >= 0
    grads = {}
    for dt in (torch.float64, torch.float32):                               # the reference, and torch's own fp32 autograd
        p = params64(sd, dtype=dt)
        logits, value = policy64(p, c, gs, model[live], gf[live], mask[live])
        loss = (torch.as_tensor(gl[live], dtype=dt) * logits).sum() + (torch.as_tensor(gv[live], dtype=dt) * value).sum()
        grads[dt] = ref_grads(loss, p)
    g64 = grads[torch.float64]
    from ddls_b200 import policy as P
    e32 = tensor_errors(P.pack_weights(grads[torch.float32], c, A), g64, c, A)
    check_tensors(tensor_errors(got, g64, c, A), what, e32)
    np.testing.assert_array_equal(pol.backward(model, gf, mask, gl, gv), got)          # the same bits again


@pytest.mark.parametrize('cid', ['yaml', 'max', 'min', 'odd', 'wide-fc', 'unmasked'])
def test_backward_matches_float64_autograd(cid):
    """random upstream gradients, masked actions, rows with model -1; one-node graph, zero-in-degree nodes, and for yaml / max the
    4,096-leaf star and the 20,000-node graph"""
    from ddls_b200 import policy as P
    K = _kernels()
    over, A, _, big = K.CONFIGS[cid]
    c = K._cfg(over)
    rng = np.random.default_rng(5)
    gs = [g.features(c, rng) for g in K.graphs(big)]
    sd = P.random_state_dict(c, A, seed=K.SEED)
    pol = K.raw_policy(c, A, gs, sd)
    try:
        backward_case(pol, c, A, gs, sd, 11, f'backward {cid}')
    finally:
        pol.close()


class _Static:
    def __init__(self, st):
        self.nf, self.ef, self.src, self.dst = st['node_features'], st['edge_features'], st['edges_src'], st['edges_dst']


def test_backward_on_the_bench_job_types():
    from ddls_b200 import policy as P, workload
    graphs = [workload.make_graph(k) for k in ('resnet', 'bert', 'gpt2')]
    sd = P.random_state_dict(P.DEFAULT_CONFIG, 17, seed=2)
    pol = P.DeviceGNNPolicy(graphs, 17, None, sd)
    try:
        backward_case(pol, pol.config, 17, [_Static(st) for st in pol.static], sd, 12, 'backward bench job types')
    finally:
        pol.close()


def _loss_setup(noise, seed=21):
    from ddls_b200 import policy as P
    from ddls_b200.learn import DevicePPOLearner, PPOConfig
    K = _kernels()
    c = K._cfg({})
    A = 17
    rng = np.random.default_rng(5)
    gs = [g.features(c, rng) for g in K.graphs(False)]
    sd = P.random_state_dict(c, A, seed=K.SEED)
    pol = K.raw_policy(c, A, gs, sd)
    n = 96
    model, gf, mask = rows(len(gs), A, c, n, seed, dead=False)
    logits, value = pol.forward(model, gf, mask)
    rng = np.random.default_rng(seed + 1)
    old = logits.copy()
    old[mask.astype(bool)] += (noise * rng.standard_normal(int(mask.sum()))).astype(np.float32)
    action = np.array([rng.choice(np.flatnonzero(mk)) for mk in mask], dtype=np.int32)
    batch = dict(model=model, graph_features=gf, action_mask=mask, action=action, old_logits=old,
                 advantage=rng.standard_normal(n).astype(np.float32), value_target=(value + rng.standard_normal(n)).astype(np.float32))
    cfg = PPOConfig(vf_clip_param=0.5)
    return pol, c, A, gs, sd, batch, DevicePPOLearner(pol, cfg)


@pytest.mark.parametrize('noise', [0.0, 0.6])
def test_ppo_loss_and_gradient_match_float64(noise):
    """noise 0: the old logits are the current ones (ratio 1, nothing clipped); 0.6: clipping active; value clipping and masked
    actions in both"""
    import torch
    from ppo_reference import params64, policy64, ppo_loss64
    pol, c, A, gs, sd, b, lrn = _loss_setup(noise)
    try:
        stats, grad = lrn.loss_and_grad(b)
        p = params64(sd)
        logits, value = policy64(p, c, gs, b['model'], b['graph_features'], b['action_mask'])
        total, want = ppo_loss64(logits, value, b['action'], b['old_logits'], b['advantage'], b['value_target'], lrn.config)
        n = len(b['model'])
        for k in ('total_loss', 'policy_loss', 'vf_loss', 'entropy', 'kl'):
            assert abs(stats[k] - want[k]) <= 1e-5 * abs(want[k]) + 1e-7, (k, stats[k], want[k])
        assert abs(stats['clip_frac'] - want['clip_frac']) <= 1.5 / n
        assert (want['clip_frac'] > 0) == (noise > 0) and stats['rows'] == n
        assert 0 < want['vf_loss'] < lrn.config.vf_clip_param                  # some rows clipped, some not
        g64 = ref_grads(total, p)
        check_tensors(tensor_errors(grad, g64, c, A), f'ppo loss noise {noise}')
        norm64 = np.sqrt(sum(float((g ** 2).sum()) for g in g64.values()))
        assert abs(stats['grad_gnorm'] - norm64) <= REL * norm64
    finally:
        pol.close()


# ---- the learner on collected trajectories ----

def _env(B=256, J=8, seed=5):
    from ddls_b200 import workload
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    graphs = [workload.make_graph('resnet')]                                  # config 3: 64 workers, ResNet-50
    env = DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=B, jobs_per_episode=J, seed=seed)
    return env, graphs


def _policy(graphs, seed=4):
    from ddls_b200 import policy as P
    return P.DeviceGNNPolicy(graphs, 17, None, P.random_state_dict(P.DEFAULT_CONFIG, 17, seed=seed))


def host_batch(pol, traj, tb):
    """the train batch's rows (t-major) as host arrays, with the collection weights' logits"""
    live = traj['live'] & (traj['model'] < pol.n_models)
    model = traj['model'][live]
    stat = np.stack([st['graph_static'] for st in pol.static])[model]
    dyn = traj['graph_features_dynamic'][live]
    gf = np.concatenate([dyn[:, :9], stat, dyn[:, 9:]], axis=1).astype(np.float32)
    mask = traj['action_mask'][live].astype(np.uint8)
    old, _ = pol.forward(model, gf, mask)
    return dict(model=model, graph_features=gf, action_mask=mask, action=traj['action'][live], old_logits=old,
                advantage=tb['advantage'], value_target=tb['value_target'])


def test_first_pass_recomputes_the_collected_log_probabilities_bit_for_bit():
    J = 8
    env, graphs = _env(J=J)
    first_pass_recomputes_the_collected_log_probabilities(env, _policy(graphs), J)


def first_pass_recomputes_the_collected_log_probabilities(env, pol, J):
    """a J-step segment collected by pol, then one PPO pass over all of it: the pass's log-probabilities are the collected ones,
    bit for bit (EMB_FORWARD's embeddings are the embed kernel's).  Closes env and pol."""
    from ddls_b200.learn import DevicePPOLearner, PPOConfig
    try:
        traj = pol.collect(env, J, sample=True, seed=3)
        lrn = DevicePPOLearner(pol, PPOConfig(num_sgd_iter=1, sgd_minibatch_size=J * env.B))
        stats = lrn.learn(env, J)
        tb = lrn.train_batch(env)
        live = traj['live'] & (traj['model'] < pol.n_models)
        assert stats['rows'] == live.sum() == len(tb['logp'])
        np.testing.assert_array_equal(tb['logp'], traj['logp'][live])
        np.testing.assert_array_equal(tb['logp_old'].view(np.uint32), tb['logp'].view(np.uint32))
        # the head-gradient kernel's own forward gives those bits too: the ratio is exactly 1, so the KL is exactly 0 and the
        # policy loss is exactly -mean(advantage), summed in the minibatch's row order as the kernel sums it
        assert stats['clip_frac'] == 0.0 and stats['kl'] == 0.0
        n, s = len(tb['advantage']), 0.0
        for i in shuffle_order(lrn.config.seed, 0, n):
            s += -float(tb['advantage'][i])
        assert stats['policy_loss'] == s / n
    finally:
        pol.close(); env.close()


@pytest.mark.parametrize('kind', ['full', 'truncated', 'prefix', 'past_the_end', 'wide'])
def test_gae_matches_numpy_float64(kind):
    """full episodes; a segment that ends before its episodes do (bootstrapped with the value of the environment's current state);
    the first half of a recorded segment (bootstrapped with the value recorded at the next step); episodes that end early; full
    episodes of 1,300 episodes, which the one-CTA kernel compacts and standardises in chunks of 1,024"""
    from ppo_reference import gae64, standardize64
    from ddls_b200.learn import DevicePPOLearner, PPOConfig
    J = 8
    H = {'full': J, 'truncated': J // 2, 'prefix': J, 'past_the_end': J + 3, 'wide': J}[kind]
    env, graphs = _env(B=1300 if kind == 'wide' else 256, J=J, seed=9)
    pol = _policy(graphs)
    try:
        traj = pol.collect(env, H, sample=True, seed=7)
        if kind == 'prefix':
            L = J // 2
            boot = traj['value'][L]
            traj = {k: v[:L] for k, v in traj.items()}
        else:
            L = H
            obs, _, done_now = env.read()
            m = np.clip(obs['model'], 0, None)
            stat = np.stack([st['graph_static'] for st in pol.static])[m]
            dyn = obs['graph_features_dynamic']
            _, boot = pol.forward(m, np.concatenate([dyn[:, :9], stat, dyn[:, 9:]], axis=1), obs['action_mask'])
        if kind in ('truncated', 'prefix'):
            assert (~traj['done'][-1]).any()
        else:
            assert traj['done'][-1].all()
        cfg = PPOConfig(num_sgd_iter=0, standardize_advantages=False)
        lrn = DevicePPOLearner(pol, cfg)
        lrn.learn(env, L)
        tb = lrn.train_batch(env)
        adv, vt, live = gae64(traj['reward'], traj['value'], traj['done'], traj['model'], boot, cfg.gamma, cfg.lambda_, pol.n_models)
        np.testing.assert_array_equal(live, traj['live'] & (traj['model'] < pol.n_models))
        np.testing.assert_allclose(tb['advantage'], adv, rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(tb['value_target'], vt, rtol=1e-6, atol=1e-6)
        lrn.config.standardize_advantages = True
        lrn.learn(env, L)
        np.testing.assert_allclose(lrn.train_batch(env)['advantage'], standardize64(adv), rtol=1e-5, atol=1e-5)
        with pytest.raises(Exception, match='recorded'):
            lrn.learn(env, H + 1)                                       # more steps than were recorded
    finally:
        pol.close(); env.close()


def check_adam(w0, w1, m1, v1, want, wm, wv, what):
    """the update against torch's, to 1e-6 relative -- it is only seen through the fp32 weights, which round it to their own ulp
    (2.8e-4 updates on 0.1 weights: about 3e-5 of the update) -- and the moments to 1e-6 relative"""
    u, wu = w0.astype(np.float64) - w1, w0.astype(np.float64) - want
    ulp = np.spacing(np.maximum(np.abs(w0), np.abs(w1))).astype(np.float64)
    bad = np.abs(u - wu) > 1e-6 * np.abs(wu) + ulp
    assert not bad.any(), f'{what}: {int(bad.sum())} updates off, e.g. {u[bad][:3]} vs {wu[bad][:3]}'
    assert np.abs(wu).max() > 1e3 * ulp.max()                           # the updates are far above the weights' rounding
    for name, got, ref in (('exp_avg', m1, wm), ('exp_avg_sq', v1, wv)):
        scale = float(np.abs(ref).max())
        np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-7 * scale, err_msg=f'{what} {name}')


@pytest.mark.parametrize('grad_clip', [1e-3, 1e6])
def test_adam_steps_match_torch(grad_clip):
    """two learn calls of one pass of one minibatch each: the gradient is ramp_ppo_loss_grad's on the rows in the pass's shuffled
    order (the same bits), and each update torch.optim.Adam + clip_grad_norm_'s fp32 step from it -- the first from zero moments,
    the second from the first's"""
    from ppo_reference import adam_step
    from ddls_b200.learn import DevicePPOLearner, PPOConfig
    J = 6
    env, graphs = _env(B=64, J=J, seed=13)
    pol = _policy(graphs)
    try:
        traj = pol.collect(env, J, sample=True, seed=1)
        probe = DevicePPOLearner(pol, PPOConfig(num_sgd_iter=0))
        probe.learn(env, J)
        tb = probe.train_batch(env)
        n = len(tb['advantage'])
        cfg = PPOConfig(num_sgd_iter=1, sgd_minibatch_size=n, grad_clip=grad_clip, seed=77)
        lrn = DevicePPOLearner(pol, cfg)
        lrn.reset()
        w0, (m0, v0, t0) = pol.get_weights(), lrn.adam_state()
        assert t0 == 0 and not m0.any() and not v0.any()
        for call in range(2):
            b = host_batch(pol, traj, tb)                                   # old logits at the current weights, as learn takes them
            order = shuffle_order(cfg.seed + call, 0, n)
            _, g = DevicePPOLearner(pol, dataclasses.replace(cfg, kl_coeff=lrn.config.kl_coeff)).loss_and_grad(
                {k: v[order] for k, v in b.items()})
            want, wm, wv, norm = adam_step(w0, g, m0 if call else None, v0 if call else None, call, cfg)
            stats = lrn.learn(env, J)
            w1, (m1, v1, t1) = pol.get_weights(), lrn.adam_state()
            assert t1 == call + 1
            assert abs(stats['grad_gnorm'] - norm) <= 1e-5 * norm
            assert (norm > grad_clip) == (grad_clip < 1)
            check_adam(w0, w1, m1, v1, want, wm, wv, f'step {call + 1}')
            w0, m0, v0 = w1, m1, v1
    finally:
        pol.close(); env.close()


def test_learn_is_deterministic():
    from ddls_b200.learn import DevicePPOLearner, PPOConfig
    J = 6
    env, graphs = _env(B=128, J=J, seed=17)
    pol = _policy(graphs)
    try:
        pol.collect(env, J, sample=True, seed=2)
        w0 = pol.get_weights()
        cfg = PPOConfig(num_sgd_iter=3, sgd_minibatch_size=128, seed=5)
        out = []
        for _ in range(2):
            pol.set_weights(w0)
            lrn = DevicePPOLearner(pol, cfg)
            lrn.reset()
            stats = lrn.learn(env, J)
            out.append((pol.get_weights(), stats))
        np.testing.assert_array_equal(out[0][0].view(np.uint32), out[1][0].view(np.uint32))
        assert out[0][1] == out[1][1]
        assert np.abs(out[0][0] - w0).max() > 0
    finally:
        pol.close(); env.close()


def test_twenty_updates_lower_the_loss_on_a_fixed_batch():
    from ddls_b200.learn import DevicePPOLearner, PPOConfig
    J = 6
    env, graphs = _env(B=64, J=J, seed=19)
    pol = _policy(graphs)
    try:
        traj = pol.collect(env, J, sample=True, seed=4)
        probe = DevicePPOLearner(pol, PPOConfig(num_sgd_iter=0))
        probe.learn(env, J)
        tb = probe.train_batch(env)
        b = host_batch(pol, traj, tb)
        fixed = PPOConfig()
        before, _ = DevicePPOLearner(pol, fixed).loss_and_grad(b)
        lrn = DevicePPOLearner(pol, dataclasses.replace(fixed, num_sgd_iter=20, sgd_minibatch_size=len(tb['advantage'])))
        lrn.reset()
        lrn.learn(env, J)
        after, _ = DevicePPOLearner(pol, fixed).loss_and_grad(b)
        print(f"total loss on the batch: {before['total_loss']:.6f} -> {after['total_loss']:.6f}")
        assert after['total_loss'] < before['total_loss']
    finally:
        pol.close(); env.close()


def test_learner_memory_is_given_back_on_close():
    from ddls_b200 import engine
    from ddls_b200.learn import DevicePPOLearner, PPOConfig
    J = 4
    env, graphs = _env(B=64, J=J, seed=23)
    warm = _policy(graphs)                                                  # the environment's own buffers, made as it first runs
    warm.collect(env, J, sample=True, seed=0)
    warm.close()
    base = engine.device_bytes()
    pol = _policy(graphs)
    before_learn = engine.device_bytes()
    pol.collect(env, J, sample=True, seed=0)
    DevicePPOLearner(pol, PPOConfig(num_sgd_iter=1)).learn(env, J)
    assert engine.device_bytes()[0] > before_learn[0]
    pol.close()
    assert engine.device_bytes() == base
    env.close()
