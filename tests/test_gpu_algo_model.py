"""-m gpu: the read-out the algorithm configs train (scripts/ramp_job_partitioning_configs/algo/*.yaml): one hidden layer as wide as
the action space (fcnet_hiddens [action_space.n]), with the value layer on the policy's hidden layer (vf_share_layers, impala / pg /
es.yaml) or a separate value branch (ppo.yaml).

* forward: H = n_actions in {1, 17, 31}, shared or not, on raw graphs up to 20,000 nodes: embeddings, unmasked logits and values
  within 1e-5 + 1e-5 |ref| of float64 (tests/shared_vf_reference.py's head64), masked logits -FLT_MAX, greedy ties to the first index, sampled
  actions draw for draw; act / collect / agents.evaluate on a device environment at both yaml models
* gradients on recorded batches: PPO at (17, separate), IMPALA and PG at (17, shared), against float64 through
  tie_reference.explain(); under IMPALA with sharing the value loss reaches _hidden_layers.0
* whole learn calls: PPO (17, separate) and IMPALA (17, shared) against the composition replay (the device's loss_and_grad,
  torch's fp32 Adam), a short last minibatch / train batch included; two learners with one seed give the same weights
* ES at es.yaml's model: a weight set's episodes decide what one DeviceGNNPolicy with that set's weights decides, bit for bit;
  learn() equals update() on its own record"""
import dataclasses
import math

import numpy as np
import pytest

import shared_vf_reference as SV
from test_gpu_learn_grad_recorded import check_explained, impala_rows, pg_loss, ppo_loss
from test_gpu_policy_kernels import NEG_FLT_MAX_BITS, batch, check_close, expected_draws, graphs, log_softmax_at, raw_policy

pytestmark = pytest.mark.gpu

SEED = 3
PARTS_REL = 1e-5


def _model(A, shared):
    from ddls_b200 import policy as P
    return dict(P.DEFAULT_CONFIG, fcnet_hiddens=(A,), vf_share_layers=bool(shared))


class Case:
    pass


def check_readout(k, model, gf, mask, out, what):
    """logits / value against float64 on the float64 embeddings; masked logits -FLT_MAX bit for bit; the largest errors"""
    logits, value = out[0], out[1]
    wl, wv = SV.head64(k.sd, k.c, k.emb64[model], gf, mask)
    valid = mask.astype(bool)
    el = check_close(logits[valid], wl[valid], f'{what} logits')
    assert (logits[~valid].view(np.uint32) == NEG_FLT_MAX_BITS).all(), f'{what}: a masked logit is not -FLT_MAX'
    ev = check_close(value, wv, f'{what} value')
    return el, ev


@pytest.fixture(scope='module', params=[(A, s) for A in (1, 17, 31) for s in (0, 1)], ids=lambda p: f'H{p[0]}-{"shared" if p[1] else "separate"}')
def case(request):
    from ddls_b200 import policy as P
    from gnn_reference import embed64
    A, shared = request.param
    k = Case()
    k.id, k.A, k.c = f'H{A}-{shared}', A, _model(A, shared)
    rng = np.random.default_rng(5)
    k.graphs = [g.features(k.c, rng) for g in graphs(True)]
    k.sd = P.random_state_dict(k.c, A, seed=SEED)
    assert ('logit_module._value_branch_separate.0._model.0.weight' in k.sd) == (not shared)
    k.emb64 = np.stack([embed64(k.sd, k.c, g.nf, g.ef, g.src, g.dst) for g in k.graphs])
    k.pol = raw_policy(k.c, A, k.graphs, k.sd)
    yield k
    k.pol.close()


def test_embeddings_and_readout_match_fp64(case):
    emb = case.pol.embed()
    for m, g in enumerate(case.graphs):
        check_close(emb[m], case.emb64[m], f'{case.id} {g.name} embedding')
    for n in (1, 9, 2113, 50000):
        model, gf, mask = batch(case, n, seed=n)
        out = case.pol.decide(model, gf, mask)
        el, ev = check_readout(case, model, gf, mask, out, f'{case.id} n={n}')
        logits, _, logp, action = out
        np.testing.assert_array_equal(action, np.argmax(logits, 1))                        # the first maximal logit
        np.testing.assert_allclose(logp, log_softmax_at(logits, action), rtol=0, atol=1e-5)
        np.testing.assert_array_equal(case.pol.forward(model, gf, mask)[0], logits)
        if case.A > 1:
            assert (logits[mask == 0].view(np.uint32) == NEG_FLT_MAX_BITS).all()
    print(f'[algo-model] {case.id}: logits max |err| {el:.3e}, value max |err| {ev:.3e}')


def test_sampler_draw_for_draw(case):
    n, seed = 50000, 0x5DEECE66D2F1A3B7
    model, gf, mask = batch(case, n, seed=123)
    logits, value, logp, action = case.pol.decide(model, gf, mask, sample=True, seed=seed)
    greedy = case.pol.decide(model, gf, mask)
    np.testing.assert_array_equal(logits, greedy[0])
    np.testing.assert_array_equal(value, greedy[1])
    want, near = expected_draws(logits, seed)
    assert near.mean() < 0.005, near.mean()
    np.testing.assert_array_equal(action[~near], want[~near])
    if case.A > 1:
        assert len(np.unique(action)) > 1


@pytest.mark.parametrize('shared', [0, 1])
def test_greedy_ties_go_to_the_first_index(shared):
    """two logit rows made equal give bitwise-equal logits at H = 31 (one lane with no hidden unit); the action is the first"""
    from ddls_b200 import policy as P
    A = 31
    c = _model(A, shared)
    rng = np.random.default_rng(8)
    gs = [g.features(c, rng) for g in graphs(False)]
    sd = P.random_state_dict(c, A, seed=SEED)
    pol = raw_policy(c, A, gs, sd)
    n = 512
    model = rng.integers(0, len(gs), n).astype(np.int32)
    gf = rng.standard_normal((n, c['in_features_graph'])).astype(np.float32)
    W, b = 'logit_module._logits._model.0.weight', 'logit_module._logits._model.0.bias'
    try:
        for i, j in [(0, 30), (15, 16), (7, 23)]:
            s = {key: v.copy() for key, v in sd.items()}
            s[W][j] = s[W][i]
            s[b][i] += 20.0
            s[b][j] = s[b][i]
            pol.set_weights(s)
            mask = np.ones((n, A), dtype=np.uint8)
            mask[n // 2:, i] = 0
            logits, _, _, action = pol.decide(model, gf, mask)
            np.testing.assert_array_equal(logits[:n // 2, i].view(np.uint32), logits[:n // 2, j].view(np.uint32))
            assert (action[:n // 2] == i).all() and (action[n // 2:] == j).all(), (i, j)
    finally:
        pol.close()


def _env(B=64, J=6, seed=7):
    from ddls_b200 import workload
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    graphs_ = [workload.make_graph('resnet')]                                     # config 3: 64 workers, ResNet-50
    return DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs_, n_episodes=B, jobs_per_episode=J, seed=seed), graphs_


def _static(pol):
    return np.stack([st['graph_static'] for st in pol.static])


@pytest.mark.parametrize('algo', ['ppo', 'impala'])
def test_act_collect_and_evaluate_on_a_device_environment(algo):
    """the yaml models (ppo: separate value branch, 5,668 weights; impala / pg / es: shared, 5,243) drive a device environment:
    act() decides what decide() decides on the same rows, collect() records act's values, evaluate() runs whole episodes"""
    from ddls_b200 import agents
    from ddls_b200 import policy as P
    env, gs = _env(B=256, J=6)
    A = env.max_partitions_per_op + 1
    assert A == 17
    pol = P.DeviceGNNPolicy(gs, A, P.algo_model_config(algo, A), seed=2)
    try:
        assert len(pol.get_weights()) == (5668 if algo == 'ppo' else 5243)
        obs = env.reset()
        pol.act(env, sample=False)
        r = pol.read(env)
        model = np.where(obs['done'], -1, obs['model']).astype(np.int32)
        gf = np.concatenate([obs['graph_features_dynamic'][:, :9], _static(pol)[np.maximum(model, 0)], obs['graph_features_dynamic'][:, 9:]], 1)
        lg, v, _, a = pol.decide(model, gf.astype(np.float32), obs['action_mask'])
        live = model >= 0
        np.testing.assert_array_equal(r['logits'][live], lg[live])
        np.testing.assert_array_equal(r['value'][live], v[live])
        np.testing.assert_array_equal(r['actions'][live], a[live])
        traj = pol.collect(env, 6, sample=True, seed=3)
        assert traj['live'].any() and np.isfinite(traj['value'][traj['live']]).all()
        assert len(np.unique(traj['action'][traj['live']])) > 1
        res = agents.evaluate(env, pol)
        print(f'[algo-model] {algo} evaluate: {res if not isinstance(res, dict) else {k: res[k] for k in list(res)[:4]}}')
    finally:
        pol.close(); env.close()


# ---- gradients on recorded batches ----

@pytest.mark.parametrize('wseed', [2, 4])
def test_learner_gradients_on_recorded_batches(wseed):
    from ddls_b200 import policy as P
    from ddls_b200.learn import DeviceIMPALALearner, DevicePGLearner, DevicePPOLearner, IMPALAConfig, PGConfig, PPOConfig
    from impala_reference import fragments
    from pg_reference import train_rows
    J = 6
    env, gs = _env(B=64, J=J)
    A = env.max_partitions_per_op + 1
    pols = {s: P.DeviceGNNPolicy(gs, A, _model(A, s), P.random_state_dict(_model(A, s), A, seed=wseed)) for s in (0, 1)}
    try:
        # PPO at ppo.yaml's model (separate value branch)
        pol = pols[0]
        traj = {k: np.array(v) for k, v in pol.collect(env, J, sample=True, seed=3).items()}
        probe = DevicePPOLearner(pol, PPOConfig(num_sgd_iter=0))
        probe.learn(env, J)
        from test_gpu_policy_learn import host_batch
        b = host_batch(pol, traj, probe.train_batch(env))
        _, g = DevicePPOLearner(pol, PPOConfig()).loss_and_grad(b)
        check_explained(pol, f'ppo H17 separate seed {wseed}', g, b['model'], b['graph_features'], b['action_mask'], ppo_loss(b, PPOConfig()))
        # IMPALA and PG at impala / pg.yaml's model (shared value layer)
        pol = pols[1]
        traj = {k: np.array(v) for k, v in pol.collect(env, J, sample=True, seed=3).items()}
        icfg = IMPALAConfig()
        fr = fragments(traj, [st['graph_static'] for st in pol.static], pol.n_models, J)
        _, g, _ = DeviceIMPALALearner(pol, icfg).loss_and_grad(fr)
        model, gf, mask, loss = impala_rows(fr, icfg)
        SV.check_explained(pol, f'impala H17 shared seed {wseed}', g, model, gf, mask, loss)
        # the value loss reaches the shared hidden layer: without it that layer's gradient changes
        _, g0, _ = DeviceIMPALALearner(pol, dataclasses.replace(icfg, vf_loss_coeff=0.0)).loss_and_grad(fr)
        hk = 'logit_module._hidden_layers.0._model.0.weight'
        gh, gh0 = P.unpack_weights(g, pol.config, A)[hk], P.unpack_weights(g0, pol.config, A)[hk]
        dv = np.linalg.norm(gh.astype(np.float64) - gh0) / np.linalg.norm(gh)
        assert dv > 1e-3, dv
        print(f'[algo-model] impala shared seed {wseed}: the value loss moves _hidden_layers.0 by {dv:.3e} (relative)')
        pcfg = PGConfig()
        b = train_rows(pol, traj, pcfg.gamma)
        _, g = DevicePGLearner(pol, pcfg).loss_and_grad(b)
        SV.check_explained(pol, f'pg H17 shared seed {wseed}', g, b['model'], b['graph_features'], b['action_mask'], pg_loss(b))
    finally:
        for p in pols.values():
            p.close()
        env.close()


# ---- whole learn calls ----

def _rel(got, ref):
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    n = np.linalg.norm(ref)
    return float(np.linalg.norm(got - ref) / n) if n > 0 else float(np.linalg.norm(got))


def _check_same(pol, a, b, tag):
    from ddls_b200 import policy as P
    for name, x, y in zip('wmv', a, b):
        ga, gb = P.unpack_weights(x, pol.config, pol.n_actions), P.unpack_weights(y, pol.config, pol.n_actions)
        errs = {k: _rel(ga[k], gb[k]) for k in gb}
        bad = {k: e for k, e in errs.items() if not e <= PARTS_REL}
        assert not bad, f'{tag}: {name} off the composition replay: {bad}'


def test_ppo_learn_call_at_ppo_yaml_model():
    """two learn calls (a short last minibatch) against learn_by_parts; a second learner with the same seed gives the same bits"""
    from ddls_b200 import policy as P
    from ddls_b200.learn import DevicePPOLearner, PPOConfig
    from ppo_reference import learn_by_parts
    from test_gpu_policy_learn import host_batch
    H = 6
    env, gs = _env(B=64, J=H)
    env2, _ = _env(B=64, J=H)
    A = env.max_partitions_per_op + 1
    c = P.algo_model_config('ppo', A)
    pol = P.DeviceGNNPolicy(gs, A, c, seed=4)
    twin = P.DeviceGNNPolicy(gs, A, c, seed=4)
    try:
        traj = {k: np.array(v) for k, v in pol.collect(env, H, sample=True, seed=3).items()}
        probe = DevicePPOLearner(pol, PPOConfig(num_sgd_iter=0))
        probe.learn(env, H)
        n = len(probe.train_batch(env)['advantage'])
        cfg = PPOConfig(num_sgd_iter=3, sgd_minibatch_size=n // 3 + 5, seed=21)    # three minibatches, the last short
        assert n % cfg.sgd_minibatch_size != 0
        lrn = DevicePPOLearner(pol, cfg)
        for call in range(2):
            c_cfg = dataclasses.replace(cfg, seed=cfg.seed + call, kl_coeff=lrn.config.kl_coeff)
            probe = DevicePPOLearner(pol, dataclasses.replace(c_cfg, num_sgd_iter=0))
            probe.learn(env, H)
            b = host_batch(pol, traj, probe.train_batch(env))
            w0 = pol.get_weights()
            parts = learn_by_parts(lrn, b, c_cfg)
            pol.set_weights(w0)
            stats = lrn.learn(env, H)
            w1, (m1, v1, t1) = pol.get_weights(), lrn.adam_state()
            assert t1 == parts['step'] == (call + 1) * cfg.num_sgd_iter * math.ceil(n / cfg.sgd_minibatch_size)
            _check_same(pol, (w1, m1, v1), (parts['weights'], parts['m'], parts['v']), f'ppo call {call}')
            assert np.abs(w1 - w0).max() > 0 and np.isfinite(stats['total_loss'])
        # determinism: the twin policy on a twin environment (same seed), a learner with the same configuration
        twin.collect(env2, H, sample=True, seed=3)
        tl = DevicePPOLearner(twin, cfg)
        for call in range(2):
            tl.learn(env2, H)
        np.testing.assert_array_equal(twin.get_weights().view(np.uint32), pol.get_weights().view(np.uint32))
    finally:
        pol.close(); twin.close(); env.close(); env2.close()


def test_impala_learn_call_at_impala_yaml_model():
    """one learn call of three train batches, the last short, against impala_learn_by_parts; a twin learner gives the same bits"""
    from ddls_b200 import policy as P
    from ddls_b200.learn import DeviceIMPALALearner, IMPALAConfig
    from impala_reference import fragments, impala_learn_by_parts, train_batches
    H = L = 6
    env, gs = _env(B=64, J=H)
    env2, _ = _env(B=64, J=H)
    A = env.max_partitions_per_op + 1
    c = P.algo_model_config('impala', A)
    pol = P.DeviceGNNPolicy(gs, A, c, seed=4)
    twin = P.DeviceGNNPolicy(gs, A, c, seed=4)
    try:
        traj = {k: np.array(v) for k, v in pol.collect(env, H, sample=True, seed=3).items()}
        b = fragments(traj, [st['graph_static'] for st in pol.static], pol.n_models, L)
        cfg = IMPALAConfig(rollout_fragment_length=L, train_batch_size=150)
        steps = train_batches(len(b['model']), L, cfg.train_batch_size)
        assert len(steps) >= 2 and (steps[-1][1] - steps[-1][0]) < (steps[0][1] - steps[0][0])
        lrn = DeviceIMPALALearner(pol, cfg)
        w0 = pol.get_weights()
        parts = impala_learn_by_parts(lrn, b, cfg)
        pol.set_weights(w0)
        lrn.learn(env, H)
        w1, (m1, v1, t1) = pol.get_weights(), lrn.adam_state()
        assert t1 == parts['step'] == len(steps)
        _check_same(pol, (w1, m1, v1), (parts['weights'], parts['m'], parts['v']), 'impala')
        twin.collect(env2, H, sample=True, seed=3)
        DeviceIMPALALearner(twin, cfg).learn(env2, H)
        np.testing.assert_array_equal(twin.get_weights().view(np.uint32), w1.view(np.uint32))
    finally:
        pol.close(); twin.close(); env.close(); env2.close()


# ---- ES at es.yaml's model ----

def test_es_population_and_update_at_es_yaml_model():
    """every episode of the population decides what a DeviceGNNPolicy holding its set's weights decides on the same rows, bit for
    bit, each step; then a learn() of the same configuration equals update() on its own record"""
    from ddls_b200 import policy as P
    from ddls_b200.learn import DeviceESLearner, ESConfig
    from es_reference import act_seed, noise_indices, perturbed
    J, B = 5, 64
    env, gs = _env(B=B, J=J, seed=5)
    A = env.max_partitions_per_op + 1
    c = P.algo_model_config('es', A)
    pol = P.DeviceGNNPolicy(gs, A, c, seed=4)
    theta = pol.get_weights()
    assert len(theta) == 5243
    noise = np.random.default_rng(11).standard_normal(len(theta) + 3000).astype(np.float32)
    cfg = ESConfig(noise_stdev=0.05, n_eval=2, episodes_per_batch=1, train_batch_size=0, seed=9)
    lrn = DeviceESLearner(pol, cfg, noise=noise)
    N = (B - 2) // 2
    refs = {}
    try:
        env.reset()
        lrn.begin_round(env, 0)
        idx = noise_indices(9, 0, 0, N, len(noise), len(theta))
        sets = [0, 1, 2 * N - 1, 2 * N]
        refs = {s: P.DeviceGNNPolicy(gs, A, c, state_dict=(theta if s == 2 * N else perturbed(theta, noise, int(idx[s // 2]), 0.05,
                                                                                              +1 if s % 2 == 0 else -1))) for s in sets}
        stat = _static(pol)
        compared = 0
        for t in range(J):
            o = env.read()[0]
            lrn.act(env, t)
            lg, lp, ac = lrn.act_read(env)
            model = np.where(o['done'], -1, o['model']).astype(np.int32)
            gf = np.concatenate([o['graph_features_dynamic'][:, :9], stat[np.maximum(model, 0)], o['graph_features_dynamic'][:, 9:]], 1)
            for s, ref in refs.items():
                wl, _, wp, wa = ref.decide(model, gf.astype(np.float32), o['action_mask'], sample=True, seed=act_seed(9, 0, 0, t))
                eps = [2 * N, 2 * N + 1] if s == 2 * N else [s]
                for b in eps:
                    if model[b] < 0:
                        continue
                    np.testing.assert_array_equal(lg[b].view(np.uint32), wl[b].view(np.uint32), err_msg=f'set {s} t {t} b {b}')
                    assert lp[b].view(np.uint32) == wp[b].view(np.uint32) and ac[b] == wa[b], (s, t, b)
                    compared += 1
            env.step_device()
        lrn.end_round(env)
        assert compared > 0
    finally:
        for r in refs.values():
            r.close()
        lrn.close(); pol.close(); env.close()
    # learn() against update() on its record
    env, gs = _env(B=B, J=J, seed=5)
    pa, pb = P.DeviceGNNPolicy(gs, A, c, seed=4), P.DeviceGNNPolicy(gs, A, c, seed=4)
    la, lb = DeviceESLearner(pa, cfg, noise=noise), DeviceESLearner(pb, cfg, noise=noise)
    try:
        la.learn(env)
        rec = la.last_step()
        _, ranks, g = lb.update(rec['noise_index'], rec['returns'])
        np.testing.assert_array_equal(pa.get_weights().view(np.uint32), pb.get_weights().view(np.uint32))
        np.testing.assert_array_equal(ranks, rec['ranks'])
        np.testing.assert_array_equal(g, rec['g'])
        assert np.abs(pa.get_weights() - theta).max() > 0
    finally:
        la.close(); lb.close(); pa.close(); pb.close(); env.close()
