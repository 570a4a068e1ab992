"""-m gpu: the ES learner on the device (ramp_es_*, ddls_b200/csrc/ramp_es.cuh) against tests/es_reference.py.

* the population: episodes of a weight set decide, return and last exactly as a single policy with that set's numpy-formed weights
  driving a twin environment through ramp_policy_decide with the recorded seeds
* the update on host inputs: ranks exactly, g to 1e-6 of float64, theta / m / v bit for bit against the float32 Adam given the
  device's g, statistics to 1e-6
* learn() equals update() on its record; the rounds rule; determinism; the policy's own Adam state; errors; memory"""
import gc

import numpy as np
import pytest

from es_reference import Adam, act_seed, compute_centered_ranks, es_gradient64, global_grad, noise_indices, perturbed

pytestmark = pytest.mark.gpu

J = 5


def _env(n_graphs, B, seed=5):
    from ddls_b200 import synth
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    gs = [synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3), synth.chain_graph(6, 'chain6')][:n_graphs]
    env = DeviceRampJobPartitioningEnvironment((4, 4, 2), gs, n_episodes=B, jobs_per_episode=J, max_partitions_per_op=16,
                                               min_op_run_time_quantum=2.0, interarrival=('exponential', 600.0), frac=(0.1, 1.0, 2),
                                               seed=seed, prewarm=True)
    return env, gs


def _policy(graphs, blob=None, seed=4):
    from ddls_b200 import policy as P
    sd = blob if blob is not None else P.random_state_dict(P.DEFAULT_CONFIG, 17, seed=seed)
    return P.DeviceGNNPolicy(graphs, 17, None, sd)


def _noise(n, extra=3000, seed=11):
    return np.random.default_rng(seed).standard_normal(n + extra).astype(np.float32)


def _cfg(**kw):
    from ddls_b200.learn import ESConfig
    base = dict(noise_stdev=0.05, n_eval=2, episodes_per_batch=1, train_batch_size=0, seed=9)
    base.update(kw)
    return ESConfig(**base)


@pytest.mark.parametrize('n_graphs', [1, 2])
def test_population_equals_single_policies(n_graphs):
    from ddls_b200.learn import DeviceESLearner
    B = 16                                                           # 7 pairs, eval episodes 14 and 15
    env, gs = _env(n_graphs, B)
    pol = _policy(gs)
    theta = pol.get_weights()
    noise = _noise(len(theta))
    lrn = DeviceESLearner(pol, _cfg(), noise=noise)
    sets = [0, 1, 12, 13, 14]                                        # first pair, last pair, eval
    twins = {s: _env(n_graphs, B) for s in sets}
    try:
        env.reset()
        lrn.begin_round(env, 0)
        idx = noise_indices(9, 0, 0, 7, len(noise), len(theta))
        blobs = {s: (theta if s == 14 else perturbed(theta, noise, int(idx[s // 2]), 0.05, +1 if s % 2 == 0 else -1)) for s in sets}
        pols = {s: _policy(gs, blobs[s]) for s in sets}
        obs = {s: twins[s][0].reset() for s in sets}
        stat = np.stack([st['graph_static'] for st in pols[0].static])
        es_logits = []
        for t in range(J):
            lrn.act(env, t)
            lg, lp, ac = lrn.act_read(env)
            es_logits.append((lg, lp, ac))
            env.step_device()
            for s in sets:
                o = obs[s]
                model = np.where(o['done'], -1, o['model']).astype(np.int32)
                gf = np.concatenate([o['graph_features_dynamic'][:, :9], stat[np.maximum(model, 0)], o['graph_features_dynamic'][:, 9:]],
                                    axis=1)
                wl, _, wp, wa = pols[s].decide(model, gf, o['action_mask'], sample=True, seed=act_seed(9, 0, 0, t))
                eps = [14, 15] if s == 14 else [s]
                live = [b for b in eps if model[b] >= 0]
                for b in live:
                    np.testing.assert_array_equal(lg[b].view(np.uint32), wl[b].view(np.uint32), err_msg=f'set {s} t {t} b {b}')
                    assert lp[b].view(np.uint32) == wp[b].view(np.uint32) and ac[b] == wa[b], (s, t, b)
                obs[s] = twins[s][0].step(wa)[0]
        more = lrn.end_round(env)
        assert not more
        rec = lrn.last_step()
        np.testing.assert_array_equal(rec['noise_index'], idx)
        np.testing.assert_array_equal(rec['seeds'], np.array([act_seed(9, 0, 0, t) for t in range(J)], np.uint64))
        for s in sets:
            tw = twins[s][0]
            ret = np.asarray(tw.episode_stats()['return']).astype(np.float32)
            n = tw.decisions()
            for b in ([14, 15] if s == 14 else [s]):
                got_r = rec['eval_returns'][b - 14] if b >= 14 else rec['returns'][b // 2, b % 2]
                got_n = rec['eval_lengths'][b - 14] if b >= 14 else rec['lengths'][b // 2, b % 2]
                assert got_r == ret[b] and got_n == n[b], (s, b, got_r, ret[b], got_n, n[b])
        assert any(len(np.unique([x[2][b] for x in es_logits])) > 1 for b in range(14))     # the draws are not all the same action
    finally:
        for s in sets:
            twins[s][0].close()
        for p in locals().get('pols', {}).values():
            p.close()
        lrn.close(); pol.close(); env.close()


def _check_update(lrn, pol, noise, idx, R, ref_adam, l2, theta):
    stats, ranks, g = lrn.update(idx, R)
    n = len(theta)
    want_ranks = compute_centered_ranks(np.asarray(R, np.float32))
    np.testing.assert_array_equal(ranks.view(np.uint32), want_ranks.view(np.uint32))
    g64 = es_gradient64(want_ranks, noise, idx, n)
    nrm = np.linalg.norm(g64)
    assert np.linalg.norm(g - g64) <= 1e-6 * nrm + 1e-12, (np.linalg.norm(g - g64), nrm)
    new, ratio = ref_adam.update(theta, global_grad(theta, g, l2))
    got = pol.get_weights()
    m, v, t = lrn.adam_state()
    np.testing.assert_array_equal(got.view(np.uint32), new.view(np.uint32))
    np.testing.assert_array_equal(m.view(np.uint32), ref_adam.m.view(np.uint32))
    np.testing.assert_array_equal(v.view(np.uint32), ref_adam.v.view(np.uint32))
    assert t == ref_adam.t
    want = dict(weights_norm=float(np.square(new.astype(np.float64)).sum()), grad_norm=float(np.square(g.astype(np.float64)).sum()),
                update_ratio=ratio, episodes_this_iter=2 * len(idx))
    for k, w in want.items():
        assert abs(stats[k] - w) <= 1e-6 * abs(w) + 1e-12, (k, stats[k], w)
    return new


@pytest.mark.parametrize('case', ['random', 'all_equal', 'one_pair', 'last_index', 'two_steps'])
def test_update_on_host_inputs(case):
    from ddls_b200.learn import DeviceESLearner
    env, gs = _env(1, 8)
    pol = _policy(gs)
    theta = pol.get_weights()
    n = len(theta)
    noise = _noise(n)
    lrn = DeviceESLearner(pol, _cfg(stepsize=0.02, l2_coeff=0.005), noise=noise)
    rng = np.random.default_rng(3)
    try:
        N = 1 if case == 'one_pair' else 300
        steps = 2 if case == 'two_steps' else 1
        ad = Adam(n, 0.02)
        for _ in range(steps):
            idx = rng.integers(0, len(noise) - n + 1, N)
            if case == 'last_index':
                idx[::7] = len(noise) - n
            R = np.full((N, 2), 2.0, np.float32) if case == 'all_equal' else rng.integers(-5, 6, (N, 2)).astype(np.float32)
            theta = _check_update(lrn, pol, noise, idx, R, ad, 0.005, theta)
    finally:
        lrn.close(); pol.close(); env.close()


@pytest.mark.parametrize('rule', ['episodes', 'timesteps'])
def test_learn_equals_update_and_runs_rounds(rule):
    from ddls_b200.learn import DeviceESLearner
    B = 16
    env, gs = _env(2, B)
    kw = dict(episodes_per_batch=30) if rule == 'episodes' else dict(episodes_per_batch=1, train_batch_size=14 * J + 1)
    pa, pb = _policy(gs), _policy(gs)
    noise = _noise(len(pa.get_weights()))
    la, lb = DeviceESLearner(pa, _cfg(**kw), noise=noise), DeviceESLearner(pb, _cfg(**kw), noise=noise)
    try:
        stats = la.learn(env)
        rec = la.last_step()
        rounds = int(stats['rounds'])
        steps = rec['lengths'].reshape(rounds, 14).sum(1).cumsum()
        done = [14 * (r + 1) >= kw['episodes_per_batch'] and steps[r] >= kw.get('train_batch_size', 0) for r in range(rounds)]
        assert done[-1] and not any(done[:-1])                          # rounds run until both counts are reached, no further
        assert rounds == 3 if rule == 'episodes' else rounds >= 2
        assert stats['episodes_this_iter'] == 14 * rounds
        assert len(rec['noise_index']) == 7 * rounds and len(rec['seeds']) == J * rounds and len(rec['eval_returns']) == 2 * rounds
        assert stats['timesteps_this_iter'] == rec['lengths'].sum()
        assert stats['eval_return_mean'] == pytest.approx(rec['eval_returns'].astype(np.float64).mean())
        assert stats['episode_reward_mean'] == pytest.approx(stats['eval_return_mean'])
        assert stats['episode_len_mean'] == pytest.approx(rec['eval_lengths'].mean())
        for r in range(rounds):
            np.testing.assert_array_equal(rec['noise_index'][7 * r:7 * (r + 1)], noise_indices(9, 0, r, 7, len(noise), len(pa.get_weights())))
        _, ranks, g = lb.update(rec['noise_index'], rec['returns'])
        np.testing.assert_array_equal(pa.get_weights().view(np.uint32), pb.get_weights().view(np.uint32))
        np.testing.assert_array_equal(ranks, rec['ranks'])
        np.testing.assert_array_equal(g, rec['g'])
    finally:
        la.close(); lb.close(); pa.close(); pb.close(); env.close()


def test_determinism_and_the_policys_own_adam_state():
    from ddls_b200.learn import DeviceESLearner, DevicePPOLearner
    (env, gs), (env_b, _) = _env(2, 16), _env(2, 16)                  # the same seed: the same episode streams at every reset
    pa, pb = _policy(gs), _policy(gs)
    noise = _noise(len(pa.get_weights()))
    la, lb = DeviceESLearner(pa, _cfg(), noise=noise), DeviceESLearner(pb, _cfg(), noise=noise)
    try:
        w0 = pa.get_weights()
        for _ in range(3):
            sa, sb = la.learn(env), lb.learn(env_b)
            assert sa == sb or all((np.isnan(sa[k]) and np.isnan(sb[k])) or sa[k] == sb[k] for k in sa)
        wa = pa.get_weights()
        np.testing.assert_array_equal(wa.view(np.uint32), pb.get_weights().view(np.uint32))
        assert (wa != w0).any()
        assert la.adam_state()[2] == 3
        m, v, step = DevicePPOLearner(pa).adam_state()
        assert step == 0 and not m.any() and not v.any()
        # the policy's forward after the steps uses the new theta
        fresh = _policy(gs, wa)
        rng = np.random.default_rng(0)
        model, gf, mask = rng.integers(0, 2, 50), rng.standard_normal((50, 17)), np.ones((50, 17), np.uint8)
        for x, y in zip(pa.forward(model, gf, mask), fresh.forward(model, gf, mask)):
            np.testing.assert_array_equal(x, y)
        fresh.close()
        la.reset()
        m, v, t = la.adam_state()
        assert t == 0 and not m.any() and not v.any()
    finally:
        la.close(); lb.close(); pa.close(); pb.close(); env.close(); env_b.close()


def test_bad_sizes_raise_and_memory_comes_back():
    from ddls_b200 import engine
    from ddls_b200 import policy as P
    from ddls_b200.learn import DeviceESLearner
    env, gs = _env(2, 16)
    pol = _policy(gs)
    n = len(pol.get_weights())
    try:
        with pytest.raises(Exception, match='smaller than'):
            DeviceESLearner(pol, _cfg(), noise=np.zeros(n - 1, np.float32))
        lrn = DeviceESLearner(pol, _cfg(n_eval=15), noise=_noise(n))
        with pytest.raises(ValueError, match='no antithetic pair'):
            lrn.learn(env)
        lrn.close()
        lrn = DeviceESLearner(pol, _cfg(n_eval=3), noise=_noise(n))             # 13 noisy episodes: odd
        env.reset()
        with pytest.raises(Exception, match='even'):
            lrn.begin_round(env, 0)
        lrn.close()
        other = P.DeviceGNNPolicy(gs, 9, None, P.random_state_dict(P.DEFAULT_CONFIG, 9, seed=1))
        lrn = DeviceESLearner(other, _cfg(), noise=_noise(len(other.get_weights())))
        env.reset()
        with pytest.raises(Exception, match='actions'):
            lrn.begin_round(env, 0)
        lrn.close(); other.close()
        # the environment's own buffers grow with the steps it takes, so the cycle measured here takes none: every ES
        # allocation (table, Adam state, population, embedding scratch, update buffers) is made without a step
        env.reset()
        gc.collect()
        base = engine.device_bytes()
        lrn = DeviceESLearner(pol, _cfg(), noise=_noise(n))
        lrn.begin_round(env, 0)
        lrn.act(env, 0)
        lrn.end_round(env)
        lrn.step()
        lrn.update(np.zeros(3, np.int32), np.ones((3, 2), np.float32))
        assert engine.device_bytes()[0] > base[0]
        lrn.close()
        assert engine.device_bytes() == base
    finally:
        pol.close(); env.close()
