"""-m gpu: the IMPALA learner step on the device (ramp_impala_loss_grad, ramp_policy_learn_impala) against the float64
restatement in tests/impala_reference.py.

* ramp_impala_loss_grad on collected fragments: the gradient per weight tensor to ||g - g64|| / ||g64|| <= max(1e-4, 10 e32), e32
  being torch's own fp32 error on that tensor (as tests/test_gpu_policy_learn.py measures it); statistics, vs and pg_adv to 1e-5.
* whole learn calls against impala_learn_by_parts (the device's loss_and_grad, torch's fp32 Adam, set_weights): weights and
  Adam's moments per tensor to 1e-5, the step count exactly, statistics to 1e-5; and each tensor's net update against the float64
  replay to max(1e-4, 10 e32).
* the first train batch's log rho is exactly 0, a second call, determinism, the learned weights in later calls, bad arguments,
  memory.  pytest -s prints the largest errors per case."""
import dataclasses

import numpy as np
import pytest

from impala_reference import STAT_KEYS, fragments, impala_learn_by_parts, impala_learn_replay, impala_loss64, read_out, train_batches
from test_gpu_policy_learn import _Static, _env, check_tensors, ref_grads, tensor_errors

pytestmark = pytest.mark.gpu

PARTS_REL = 1e-5
REL = 1e-4
FP32_FACTOR = 10
VT_TOL = 1e-5


def _make_env(kind, B, J):
    if kind == 'mix128':
        from test_gpu_eval_step_stats import _mix128
        env = _mix128(B=B, J=J, seed=4)
        return env, [m.graph for m in env.models]
    return _env(B=B, J=J, seed=7)


def _policy(graphs, A, seed=4):
    from ddls_b200 import policy as P
    return P.DeviceGNNPolicy(graphs, A, None, P.random_state_dict(P.DEFAULT_CONFIG, A, seed=seed))


def _frags(pol, traj, H, L):
    tr = {k: np.asarray(v)[:H] for k, v in traj.items()}
    return fragments(tr, [st['graph_static'] for st in pol.static], pol.n_models, L)


def _rel(got, ref):
    err, nrm = np.linalg.norm(np.asarray(got, np.float64) - ref), np.linalg.norm(ref)
    return err / nrm if nrm > 0 else err


def _close(got, want, tol=VT_TOL):
    return abs(got - want) <= tol * abs(want) + 1e-7


def test_first_batch_log_rho_is_exactly_zero():
    from ddls_b200.learn import DeviceIMPALALearner, IMPALAConfig
    J = 6
    env, graphs = _env(B=64, J=J, seed=7)
    pol = _policy(graphs, 17)
    try:
        traj = {k: np.array(v) for k, v in pol.collect(env, J, sample=True, seed=3).items()}
        cfg = IMPALAConfig(rollout_fragment_length=3, train_batch_size=60, lr=1e-3)
        lrn = DeviceIMPALALearner(pol, cfg)
        lrn.reset()
        stats = lrn.learn(env, J)
        vt = lrn.vtrace()
        fr = _frags(pol, traj, J, 3)
        s, e = train_batches(len(fr['model']), 3, cfg.train_batch_size)[0]
        dec = fr['model'][s:e] >= 0
        assert dec.sum() > 20
        np.testing.assert_array_equal(vt['log_rho'].reshape(-1, 3)[s:e], 0.0)
        np.testing.assert_array_equal(vt['target_logp'].reshape(-1, 3)[s:e][dec].view(np.uint32),
                                      fr['behaviour_logp'][s:e][dec].view(np.uint32))
        later = vt['log_rho'].reshape(-1, 3)[e:][fr['model'][e:] >= 0]
        assert np.abs(later).max() > 0                                  # after an update the steps are off-policy
        assert stats['sgd_steps'] == len(train_batches(len(fr['model']), 3, cfg.train_batch_size))
    finally:
        pol.close(); env.close()


@pytest.mark.parametrize('noise', [0.0, 0.5])
def test_loss_grad_matches_float64(noise):
    """collected fragments with the behaviour log-probabilities moved by `noise` (0.5: rho both sides of the thresholds)"""
    import torch
    from ddls_b200 import policy as P
    from ddls_b200.learn import DeviceIMPALALearner, IMPALAConfig
    from ppo_reference import params64
    J, L = 6, 3
    env, graphs = _env(B=32, J=J, seed=11)
    pol = _policy(graphs, 17)
    try:
        traj = {k: np.array(v) for k, v in pol.collect(env, J, sample=True, seed=5).items()}
        b = _frags(pol, traj, J, L)
        rng = np.random.default_rng(1)
        b['behaviour_logp'] = (b['behaviour_logp'] + noise * rng.standard_normal(b['behaviour_logp'].shape)).astype(np.float32)
        cfg = IMPALAConfig(vtrace_clip_rho_threshold=1.2, vtrace_clip_pg_rho_threshold=0.9)
        stats, grad, vt = DeviceIMPALALearner(pol, cfg).loss_and_grad(b)
        c, A = pol.config, pol.n_actions
        sd = P.unpack_weights(pol.get_weights(), c, A)
        gs = [_Static(st) for st in pol.static]
        grads, want = {}, None
        for dt in (torch.float64, torch.float32):
            p = params64(sd, dtype=dt)
            logits, value = read_out(p, c, gs, b)
            total, st, out = impala_loss64(logits, value, b, cfg)
            grads[dt] = ref_grads(total, p)
            if dt == torch.float64:
                want, want_vt = st, out
        e32 = tensor_errors(P.pack_weights(grads[torch.float32], c, A), grads[torch.float64], c, A)
        check_tensors(tensor_errors(grad, grads[torch.float64], c, A), f'impala loss noise {noise}', e32)
        for k in ('total_loss', 'policy_loss', 'vf_loss', 'entropy', 'mean_rho', 'rows'):
            assert _close(stats[k], want[k]), (k, stats[k], want[k])
        norm64 = np.sqrt(sum(float((g ** 2).sum()) for g in grads[torch.float64].values()))
        assert abs(stats['grad_gnorm'] - norm64) <= REL * norm64
        assert stats['sgd_steps'] == 0
        for k in ('vs', 'pg_advantages'):
            ref = want_vt[k]
            assert np.abs(vt[k] - ref).max() <= VT_TOL * np.abs(ref).max(), k
        np.testing.assert_allclose(vt['log_rho'], want_vt['log_rho'], rtol=0, atol=1e-6)
        if noise == 0:
            assert not vt['log_rho'].any()
        else:
            rho = np.exp(want_vt['log_rho'])[:, :-1][b['model'][:, :-1] >= 0]
            assert (rho > 1.2).any() and (rho < 0.9).any()
        again = DeviceIMPALALearner(pol, cfg).loss_and_grad(b)
        np.testing.assert_array_equal(again[1], grad)
    finally:
        pol.close(); env.close()


# env, B, J (jobs per episode: an episode ends after J decisions), H (steps learned), L (rollout_fragment_length, 0: H),
# tbs (train_batch_size), cfg overrides
CASES = {
    'whole': dict(env='cfg3', B=64, J=6, H=6, L=0, tbs=96, cfg={}, again=True),
    'divides': dict(env='cfg3', B=64, J=6, H=8, L=4, tbs=128, cfg={}),
    'short_last': dict(env='cfg3', B=64, J=6, H=6, L=3, tbs=200, cfg={}),
    'mid_fragment': dict(env='cfg3', B=32, J=5, H=8, L=4, tbs=40, cfg=dict(gamma=0.9)),
    'mixed_types': dict(env='mix128', B=64, J=6, H=6, L=3, tbs=60, cfg={}, again=True),
    'large_lr': dict(env='cfg3', B=64, J=6, H=6, L=6, tbs=60, cfg=dict(lr=3e-3, vtrace_clip_rho_threshold=1.0,
                                                                       vtrace_clip_pg_rho_threshold=1.0)),
    'one_fragment': dict(env='cfg3', B=16, J=4, H=4, L=4, tbs=7, cfg=dict(grad_clip=1e-3)),
}


def check_call(pol, lrn, env, H, b, cfg, tag):
    """one lrn.learn(env, H) against impala_learn_by_parts from the same start and impala_learn_replay in float64 / float32"""
    import torch
    from ddls_b200 import policy as P
    c, A = pol.config, pol.n_actions
    w0, (m0, v0, t0) = pol.get_weights(), lrn.adam_state()
    parts = impala_learn_by_parts(lrn, b, cfg)
    pol.set_weights(w0)
    stats = lrn.learn(env, H)
    w1, (m1, v1, t1) = pol.get_weights(), lrn.adam_state()
    n_steps = len(train_batches(len(b['model']), np.shape(b['model'])[1], cfg.train_batch_size))
    assert t1 - t0 == n_steps == parts['step'] - t0 == stats['sgd_steps'], (t0, t1, n_steps, stats['sgd_steps'])
    ref_w, ref_m, ref_v = (P.unpack_weights(x, c, A) for x in (parts['weights'], parts['m'], parts['v']))
    got_w, got_m, got_v = (P.unpack_weights(x, c, A) for x in (w1, m1, v1))
    worst = {}
    for name, got, ref in (('w', got_w, ref_w), ('m', got_m, ref_m), ('v', got_v, ref_v)):
        errs = {k: _rel(got[k], ref[k].astype(np.float64)) for k in ref}
        key = max(errs, key=errs.get)
        worst[name] = (errs[key], key)
        bad = {k: e for k, e in errs.items() if not e <= PARTS_REL}
        assert not bad, f'{tag}: {name} off the composition replay: {bad}'
    for k in STAT_KEYS:
        assert abs(stats[k] - parts['stats'][k]) <= PARTS_REL * abs(parts['stats'][k]) + 1e-7, (tag, k, stats[k], parts['stats'][k])
    params, graphs = P.unpack_weights(w0, c, A), [_Static(st) for st in pol.static]
    r64 = impala_learn_replay(params, c, graphs, b, cfg, (m0, v0, t0), torch.float64)
    r32 = impala_learn_replay(params, c, graphs, b, cfg, (m0, v0, t0), torch.float32)
    errs, e32 = {}, {}
    for k, w in params.items():
        d64 = r64['weights'][k] - w.astype(np.float64)
        errs[k] = _rel(got_w[k].astype(np.float64) - w, d64)
        e32[k] = _rel(r32['weights'][k].astype(np.float64) - w, d64)
    k64 = max(errs, key=errs.get)
    print(f'{tag}: {len(b["model"])} fragments, {n_steps} steps; vs composition: w {worst["w"][0]:.1e} ({worst["w"][1]}), '
          f'm {worst["m"][0]:.1e}, v {worst["v"][0]:.1e}; vs float64: {errs[k64]:.2e} ({k64}, e32 {e32[k64]:.2e}), '
          f'e32 worst {max(e32.values()):.2e}')
    bad = {k: (e, e32[k]) for k, e in errs.items() if not e <= max(REL, FP32_FACTOR * e32[k])}
    assert not bad, f'{tag}: net update off float64: {bad}'
    for k in STAT_KEYS:
        assert abs(stats[k] - r64['stats'][k]) <= 1e-4 * abs(r64['stats'][k]) + 1e-6, (tag, k, stats[k], r64['stats'][k])
    return stats, w0, w1, r64


@pytest.mark.parametrize('cid', list(CASES))
def test_learn_call_matches_its_replays(cid):
    from ddls_b200 import policy as P
    from ddls_b200.learn import DeviceIMPALALearner, IMPALAConfig
    case = CASES[cid]
    env, graphs = _make_env(case['env'], case['B'], case['J'])
    A = env.max_partitions_per_op + 1
    pol = _policy(graphs, A)
    H = case['H']
    L = case['L'] or H
    fresh = None
    try:
        traj = {k: np.array(v) for k, v in pol.collect(env, H, sample=True, seed=3).items()}
        b = _frags(pol, traj, H, L)
        cfg = IMPALAConfig(rollout_fragment_length=case['L'], train_batch_size=case['tbs'], **case['cfg'])
        n_frag = len(b['model'])
        F = cfg.train_batch_size // L
        if cid == 'short_last':
            assert n_frag % F != 0 and n_frag > F
        if cid == 'mid_fragment':                                       # episodes end inside a fragment, rows after are dead
            assert ((b['done'][:, :-1] == 1) & (b['model'][:, 1:] < 0)).any()
        if cid == 'one_fragment':
            assert F == 1
        lrn = DeviceIMPALALearner(pol, cfg)
        lrn.reset()
        stats, w0, w1, r64 = check_call(pol, lrn, env, H, b, cfg, cid)
        if cid == 'large_lr':                                           # later batches clip rho on some rows
            lr64 = r64['vtrace']['log_rho'][:, :-1][b['model'][:, :-1] >= 0]
            assert (np.exp(lr64) > cfg.vtrace_clip_rho_threshold * (1 + 1e-3)).sum() > 0
            vt = lrn.vtrace()
            got = vt['log_rho'].reshape(n_frag, L)[:, :-1][b['model'][:, :-1] >= 0]
            assert (np.exp(got) > cfg.vtrace_clip_rho_threshold).sum() > 0
        if case.get('again'):
            check_call(pol, lrn, env, H, b, cfg, cid + ' second call')
        fresh = P.DeviceGNNPolicy(graphs, A, None, pol.get_weights())
        dec = b['model'].reshape(-1) >= 0
        m, gf = b['model'].reshape(-1)[dec], b['graph_features'].reshape(-1, b['graph_features'].shape[-1])[dec]
        mk = b['action_mask'].reshape(-1, A)[dec]
        for x, y in zip(pol.forward(m, gf, mk), fresh.forward(m, gf, mk)):
            np.testing.assert_array_equal(x, y)
        for x, y in zip(pol.decide(m, gf, mk, sample=True, seed=11), fresh.decide(m, gf, mk, sample=True, seed=11)):
            np.testing.assert_array_equal(x, y)
        ea, _ = _make_env(case['env'], case['B'], case['J'])
        eb, _ = _make_env(case['env'], case['B'], case['J'])
        try:
            ta = {k: np.array(v) for k, v in pol.collect(ea, H, sample=False, seed=5).items()}
            tf = fresh.collect(eb, H, sample=False, seed=5)
            for k, v in ta.items():
                np.testing.assert_array_equal(v, tf[k], err_msg=k)
        finally:
            ea.close(); eb.close()
    finally:
        if fresh is not None:
            fresh.close()
        pol.close(); env.close()


def test_learn_is_deterministic():
    from ddls_b200.learn import DeviceIMPALALearner, IMPALAConfig
    J = 6
    env, graphs = _env(B=128, J=J, seed=17)
    pol = _policy(graphs, 17)
    try:
        pol.collect(env, J, sample=True, seed=2)
        w0 = pol.get_weights()
        cfg = IMPALAConfig(rollout_fragment_length=3, train_batch_size=90, lr=1e-3)
        out = []
        for _ in range(2):
            pol.set_weights(w0)
            lrn = DeviceIMPALALearner(pol, cfg)
            lrn.reset()
            stats = lrn.learn(env, J)
            out.append((pol.get_weights(), stats, lrn.adam_state()))
        np.testing.assert_array_equal(out[0][0].view(np.uint32), out[1][0].view(np.uint32))
        np.testing.assert_array_equal(out[0][2][0].view(np.uint32), out[1][2][0].view(np.uint32))
        assert out[0][1] == out[1][1]
        assert np.abs(out[0][0] - w0).max() > 0
    finally:
        pol.close(); env.close()


def test_bad_arguments():
    from ddls_b200.learn import DeviceIMPALALearner, IMPALAConfig
    J = 6
    env, graphs = _env(B=16, J=J, seed=19)
    other, _ = _env(B=8, J=J, seed=19)
    pol = _policy(graphs, 17)
    try:
        with pytest.raises(Exception, match='recorded'):
            DeviceIMPALALearner(pol, IMPALAConfig()).learn(env, J)             # no trajectory
        pol.collect(env, J, sample=True, seed=1)
        w0 = pol.get_weights()
        for cfg, match in ((IMPALAConfig(rollout_fragment_length=4), 'divide'), (IMPALAConfig(train_batch_size=5), 'below'),
                           (IMPALAConfig(rollout_fragment_length=2, train_batch_size=1), 'below')):
            with pytest.raises(Exception, match=match):
                DeviceIMPALALearner(pol, cfg).learn(env, J)
        with pytest.raises(Exception, match='another environment'):
            DeviceIMPALALearner(pol, IMPALAConfig()).learn(other, J)
        with pytest.raises(Exception, match='recorded'):
            DeviceIMPALALearner(pol, IMPALAConfig()).learn(env, J + 1)
        np.testing.assert_array_equal(pol.get_weights(), w0)                   # nothing was updated
        DeviceIMPALALearner(pol, IMPALAConfig(rollout_fragment_length=2, train_batch_size=2)).learn(env, J)
    finally:
        pol.close(); env.close(); other.close()


def test_learner_memory_is_given_back_on_close():
    from ddls_b200 import engine
    from ddls_b200.learn import DeviceIMPALALearner, IMPALAConfig
    J = 4
    env, graphs = _env(B=64, J=J, seed=23)
    warm = _policy(graphs, 17)
    warm.collect(env, J, sample=True, seed=0)
    warm.close()
    base = engine.device_bytes()
    pol = _policy(graphs, 17)
    before_learn = engine.device_bytes()
    pol.collect(env, J, sample=True, seed=0)
    DeviceIMPALALearner(pol, IMPALAConfig()).learn(env, J)
    assert engine.device_bytes()[0] > before_learn[0]
    pol.close()
    assert engine.device_bytes() == base
    env.close()
