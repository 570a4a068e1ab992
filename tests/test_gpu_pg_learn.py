"""-m gpu: the PG learner step on the device (ramp_pg_loss_grad, ramp_policy_learn_pg) against the float64 restatement in
tests/pg_reference.py.

* ramp_pg_loss_grad on host rows: the gradient per weight tensor to ||g - g64|| / ||g64|| <= max(1e-4, 10 e32), e32 being torch's
  own fp32 error on that tensor (the rule of tests/test_gpu_policy_learn.py); statistics to 1e-5.
* after learn: the head-gradient kernel's log p(a) at the collection weights is the collected one bit for bit, the advantages are
  the float64 discounted returns, policy_loss is -mean(logp adv).
* whole learn calls against pg_learn_by_parts (the device's loss_and_grad, torch's fp32 Adam, set_weights): weights and Adam's
  moments per tensor to 1e-5, the step count exactly; the call's statistics against float64 to 1e-5, and its gradient on the
  recorded batch per tensor to max(1e-4, 10 e32) after the flips of named near-tied ReLU units (tests/tie_reference.py).
* determinism, the Adam step count shared with PPO, bad arguments, memory.  pytest -s prints the largest errors per case."""
import numpy as np
import pytest

from pg_reference import discounted_returns, pg_learn_by_parts, pg_loss64, train_rows
from test_gpu_policy_learn import _Static, _env, check_tensors, ref_grads, rows, tensor_errors

pytestmark = pytest.mark.gpu

PARTS_REL = 1e-5
REL = 1e-4
FP32_FACTOR = 10


def _policy(graphs, A=17, seed=4):
    from ddls_b200 import policy as P
    return P.DeviceGNNPolicy(graphs, A, None, P.random_state_dict(P.DEFAULT_CONFIG, A, seed=seed))


def _rel(got, ref):
    err, nrm = np.linalg.norm(np.asarray(got, np.float64) - ref), np.linalg.norm(ref)
    return err / nrm if nrm > 0 else err


def _loss_case(cid):
    """(policy, config, |A|, graphs with nf / ef / src / dst, state_dict) of one loss_and_grad case"""
    from ddls_b200 import policy as P, workload
    import test_gpu_policy_kernels as K
    if cid == 'bench':
        graphs = [workload.make_graph(k) for k in ('resnet', 'bert', 'gpt2')]
        sd = P.random_state_dict(P.DEFAULT_CONFIG, 17, seed=2)
        pol = P.DeviceGNNPolicy(graphs, 17, None, sd)
        return pol, pol.config, 17, [_Static(st) for st in pol.static], sd
    over, A, _, big = K.CONFIGS['yaml' if cid == 'two_types' else cid]
    c = K._cfg(over)
    rng = np.random.default_rng(5)
    gs = [g.features(c, rng) for g in K.graphs(big)]
    if cid == 'two_types':
        gs = gs[2:4]
    sd = P.random_state_dict(c, A, seed=K.SEED)
    return K.raw_policy(c, A, gs, sd), c, A, gs, sd


@pytest.mark.parametrize('cid', ['yaml', 'wide-fc', 'unmasked', 'two_types', 'bench'])
def test_loss_grad_matches_float64(cid):
    import torch
    from ddls_b200 import policy as P
    from ddls_b200.learn import DevicePGLearner, PGConfig
    from ppo_reference import params64, policy64
    pol, c, A, gs, sd = _loss_case(cid)
    try:
        n = 96
        model, gf, mask = rows(len(gs), A, c, n, 31, dead=False)
        rng = np.random.default_rng(32)
        action = np.array([rng.choice(np.flatnonzero(mk)) for mk in mask], dtype=np.int32)
        adv = (3.0 * rng.standard_normal(n)).astype(np.float32)
        b = dict(model=model, graph_features=gf, action_mask=mask, action=action, advantage=adv)
        lrn = DevicePGLearner(pol, PGConfig())
        stats, grad = lrn.loss_and_grad(b)
        grads, want = {}, None
        for dt in (torch.float64, torch.float32):
            p = params64(sd, dtype=dt)
            logits, _ = policy64(p, c, gs, model, gf, mask)
            loss, st = pg_loss64(logits, action, adv)
            grads[dt] = ref_grads(loss, p)
            if dt == torch.float64:
                want = st
        e32 = tensor_errors(P.pack_weights(grads[torch.float32], c, A), grads[torch.float64], c, A)
        check_tensors(tensor_errors(grad, grads[torch.float64], c, A), f'pg loss {cid}', e32)
        for k in ('policy_loss', 'entropy'):
            assert abs(stats[k] - want[k]) <= 1e-5 * abs(want[k]) + 1e-7, (k, stats[k], want[k])
        assert stats['rows'] == n
        norm64 = np.sqrt(sum(float((g ** 2).sum()) for g in grads[torch.float64].values()))
        assert abs(stats['grad_gnorm'] - norm64) <= REL * norm64
        vb = P.unpack_weights(grad, c, A)
        assert not any(vb[k].any() for k in vb if 'value_branch' in k)         # PG's loss has no value term
        np.testing.assert_array_equal(lrn.loss_and_grad(b)[1], grad)            # the same bits again
    finally:
        pol.close()


def test_learn_reads_back_the_collected_log_probabilities_and_the_returns():
    from ddls_b200.learn import DevicePGLearner, PGConfig
    J = 8
    env, graphs = _env(B=128, J=J, seed=5)
    pol = _policy(graphs)
    try:
        traj = {k: np.array(v) for k, v in pol.collect(env, J, sample=True, seed=3).items()}
        lrn = DevicePGLearner(pol, PGConfig(gamma=0.97))
        lrn.reset()
        stats = lrn.learn(env, J)
        tb = lrn.train_batch(env)
        adv32, adv64, live = discounted_returns(traj['reward'], traj['done'], traj['model'], 0.97, pol.n_models)
        assert stats['rows'] == live.sum() == len(tb['logp']) > 100
        np.testing.assert_array_equal(tb['model'], traj['model'][live])
        np.testing.assert_array_equal(tb['logp'], traj['logp'][live])
        np.testing.assert_array_equal(tb['logp_old'].view(np.uint32), tb['logp'].view(np.uint32))
        err = np.abs(tb['advantage'] - adv64).max() / np.abs(adv64).max()
        print(f'returns: largest error {err:.2e} relative to the largest return')
        assert err <= 1e-6
        np.testing.assert_array_equal(tb['advantage'], adv32)
        np.testing.assert_array_equal(tb['value_target'], tb['advantage'])
        want = -np.mean(tb['logp'].astype(np.float64) * tb['advantage'].astype(np.float64))
        assert abs(stats['policy_loss'] - want) <= 1e-12 * abs(want) + 1e-15, (stats['policy_loss'], want)
        assert lrn.adam_state()[2] == 1
    finally:
        pol.close(); env.close()


# env size B, jobs per episode J (an episode ends after J decisions), H (steps collected and learned), cfg overrides
CASES = {
    'truncated': dict(B=64, J=8, H=5, cfg={}),                  # every episode goes on past the segment: no bootstrap
    'mid_segment': dict(B=48, J=4, H=7, cfg=dict(gamma=0.9)),   # episodes end inside the segment, rows after are dead
    'clipped': dict(B=64, J=6, H=6, cfg=dict(grad_clip=1e-3, lr=1e-3)),
    'episodes_1300': dict(B=1300, J=4, H=4, cfg={}),            # the one-CTA compaction in chunks of 1,024
}


def check_call(pol, lrn, env, H, b, cfg, tag):
    """one lrn.learn(env, H) against pg_learn_by_parts from the same start, and its gradient against float64"""
    from ddls_b200 import policy as P
    c, A = pol.config, pol.n_actions
    w0, (m0, v0, t0) = pol.get_weights(), lrn.adam_state()
    parts = pg_learn_by_parts(lrn, b, cfg)
    pol.set_weights(w0)
    stats = lrn.learn(env, H)
    w1, (m1, v1, t1) = pol.get_weights(), lrn.adam_state()
    assert t1 == parts['step'] == t0 + (1 if len(b['model']) else 0), (t0, t1, parts['step'])
    assert stats['rows'] == len(b['model'])
    worst = {}
    for name, got, ref in (('w', w1, parts['weights']), ('m', m1, parts['m']), ('v', v1, parts['v'])):
        got, ref = P.unpack_weights(got, c, A), P.unpack_weights(ref, c, A)
        errs = {k: _rel(got[k], ref[k].astype(np.float64)) for k in ref}
        key = max(errs, key=errs.get)
        worst[name] = (errs[key], key)
        bad = {k: e for k, e in errs.items() if not e <= PARTS_REL}
        assert not bad, f'{tag}: {name} off the composition replay: {bad}'
    for k in ('policy_loss', 'entropy', 'grad_gnorm'):
        assert abs(stats[k] - parts['stats'][k]) <= PARTS_REL * abs(parts['stats'][k]) + 1e-7, (tag, k, stats[k], parts['stats'][k])
    # the call's gradient against float64 autograd on its train batch at the starting weights, through explain(): each tensor
    # within max(1e-4, 10 e32) once the flips of named near-tied ReLU units are added to float64's.  The net update is not
    # compared with a float64 replay: Adam's first step is about lr sign(g).
    import torch
    from ppo_reference import params64, policy64
    from test_gpu_learn_grad_recorded import check_explained
    params, graphs = P.unpack_weights(w0, c, A), [_Static(st) for st in pol.static]
    with torch.no_grad():
        logits, _ = policy64(params64(params, requires_grad=False), c, graphs, b['model'], b['graph_features'], b['action_mask'])
        _, want = pg_loss64(logits, b['action'], b['advantage'])
    print(f'{tag}: {len(b["model"])} rows; vs composition: w {worst["w"][0]:.1e} ({worst["w"][1]}), m {worst["m"][0]:.1e}, '
          f'v {worst["v"][0]:.1e}')
    _, _, g64 = check_explained(pol, f'{tag} gradient', parts['grad'], b['model'], b['graph_features'], b['action_mask'],
                                lambda lg, v: pg_loss64(lg, b['action'], b['advantage'])[0], params=params)
    for k in ('policy_loss', 'entropy'):
        assert abs(stats[k] - want[k]) <= 1e-5 * abs(want[k]) + 1e-7, (tag, k, stats[k], want[k])
    norm64 = np.sqrt(sum(float((g ** 2).sum()) for g in g64.values()))
    assert abs(stats['grad_gnorm'] - norm64) <= REL * norm64
    return stats


@pytest.mark.parametrize('cid', list(CASES))
def test_learn_call_matches_its_replays(cid):
    from ddls_b200.learn import DevicePGLearner, PGConfig
    case = CASES[cid]
    env, graphs = _env(B=case['B'], J=case['J'], seed=7)
    pol = _policy(graphs)
    try:
        H = case['H']
        traj = {k: np.array(v) for k, v in pol.collect(env, H, sample=True, seed=3).items()}
        cfg = PGConfig(**case['cfg'])
        b = train_rows(pol, traj, cfg.gamma)
        if cid == 'truncated':
            assert not traj['done'][-1].all()
        if cid == 'mid_segment':
            assert traj['done'][:-1].any()
        lrn = DevicePGLearner(pol, cfg)
        lrn.reset()
        check_call(pol, lrn, env, H, b, cfg, cid)
        check_call(pol, lrn, env, H, b, cfg, cid + ' second call')               # Adam from a running state
    finally:
        pol.close(); env.close()


def test_segment_without_a_decision_is_no_update():
    from ddls_b200.learn import DevicePGLearner, PGConfig
    J = 4
    env, graphs = _env(B=32, J=J, seed=9)
    pol = _policy(graphs)
    try:
        pol.collect(env, J, sample=True, seed=1)
        lrn = DevicePGLearner(pol, PGConfig(lr=1e-3))
        lrn.reset()
        lrn.learn(env, J)
        w0, (m0, v0, t0) = pol.get_weights(), lrn.adam_state()
        assert t0 == 1
        traj = pol.collect(env, 3, sample=True, seed=2, reset=False)           # every episode has finished: nothing queued
        assert not traj['live'].any()
        stats = lrn.learn(env, 3)
        assert stats['rows'] == 0 and stats['policy_loss'] == 0.0
        m1, v1, t1 = lrn.adam_state()
        assert t1 == t0
        np.testing.assert_array_equal(pol.get_weights(), w0)
        np.testing.assert_array_equal(m1, m0)
        np.testing.assert_array_equal(v1, v0)
        assert lrn.train_batch(env)['model'].size == 0
    finally:
        pol.close(); env.close()


def test_learn_is_deterministic():
    from ddls_b200.learn import DevicePGLearner, PGConfig
    J = 6
    env, graphs = _env(B=128, J=J, seed=17)
    pol = _policy(graphs)
    try:
        pol.collect(env, J, sample=True, seed=2)
        w0 = pol.get_weights()
        out = []
        for _ in range(2):
            pol.set_weights(w0)
            lrn = DevicePGLearner(pol, PGConfig(lr=1e-3))
            lrn.reset()
            stats = [lrn.learn(env, J) for _ in range(3)]                      # three calls on the one recorded trajectory
            out.append((pol.get_weights(), stats, lrn.adam_state()))
        np.testing.assert_array_equal(out[0][0].view(np.uint32), out[1][0].view(np.uint32))
        np.testing.assert_array_equal(out[0][2][0].view(np.uint32), out[1][2][0].view(np.uint32))
        np.testing.assert_array_equal(out[0][2][1].view(np.uint32), out[1][2][1].view(np.uint32))
        assert out[0][1] == out[1][1] and out[0][2][2] == 3
        assert np.abs(out[0][0] - w0).max() > 0
    finally:
        pol.close(); env.close()


def test_pg_after_ppo_continues_the_adam_state():
    from ddls_b200.learn import DevicePGLearner, DevicePPOLearner, PGConfig, PPOConfig
    J = 6
    env, graphs = _env(B=64, J=J, seed=21)
    pol = _policy(graphs)
    try:
        traj = {k: np.array(v) for k, v in pol.collect(env, J, sample=True, seed=4).items()}
        ppo = DevicePPOLearner(pol, PPOConfig(num_sgd_iter=1, sgd_minibatch_size=128))
        ppo.reset()
        ppo.learn(env, J)
        _, _, t_ppo = ppo.adam_state()
        assert t_ppo > 1
        cfg = PGConfig(lr=1e-3)
        lrn = DevicePGLearner(pol, cfg)
        check_call(pol, lrn, env, J, train_rows(pol, traj, cfg.gamma), cfg, 'after ppo')
        assert lrn.adam_state()[2] == ppo.adam_state()[2] == t_ppo + 1
    finally:
        pol.close(); env.close()


def test_bad_arguments():
    from ddls_b200.learn import DevicePGLearner, PGConfig
    J = 6
    env, graphs = _env(B=16, J=J, seed=19)
    other, _ = _env(B=8, J=J, seed=19)
    pol = _policy(graphs)
    try:
        with pytest.raises(Exception, match='recorded'):
            DevicePGLearner(pol).learn(env, J)                                 # no trajectory
        pol.collect(env, J, sample=True, seed=1)
        w0 = pol.get_weights()
        with pytest.raises(Exception, match='another environment'):
            DevicePGLearner(pol).learn(other, J)
        with pytest.raises(Exception, match='recorded'):
            DevicePGLearner(pol).learn(env, J + 1)
        with pytest.raises(Exception, match='adam_eps'):
            DevicePGLearner(pol, PGConfig(adam_eps=0.0)).learn(env, J)
        np.testing.assert_array_equal(pol.get_weights(), w0)                   # nothing was updated
    finally:
        pol.close(); env.close(); other.close()


def test_learner_memory_is_given_back_on_close():
    from ddls_b200 import engine
    from ddls_b200.learn import DevicePGLearner
    J = 4
    env, graphs = _env(B=64, J=J, seed=23)
    warm = _policy(graphs)
    warm.collect(env, J, sample=True, seed=0)
    warm.close()
    base = engine.device_bytes()
    pol = _policy(graphs)
    before_learn = engine.device_bytes()
    pol.collect(env, J, sample=True, seed=0)
    DevicePGLearner(pol).learn(env, J)
    assert engine.device_bytes()[0] > before_learn[0]
    pol.close()
    assert engine.device_bytes() == base
    env.close()
