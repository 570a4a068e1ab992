"""-m gpu: the ES learner on the device (ramp_es_*, ddls_b200/csrc/ramp_es.cuh) against tests/es_reference.py.

* the population: episodes of a weight set decide, return and last exactly as a single policy with that set's numpy-formed weights
  driving a twin environment through ramp_policy_decide with the recorded seeds
* the update on host inputs: ranks exactly, g to 1e-6 of float64, theta / m / v bit for bit against the float32 Adam given the
  device's g, statistics to 1e-6
* the population at training sizes (a read-back check, no twins): the episodes of ~30 sets chosen so that every loop of the embed
  and head kernels runs (es_reference.coverage_sets) equal one reference policy holding that set's weights, deciding on all B rows;
  gnn.yaml at 8,704 episodes, a 128-wide 8-round policy on raw graphs (also held to float64), 512 hidden units, no action mask
* the update on host inputs: ranks exactly, g to 1e-6 of float64, theta / m / v bit for bit against the float32 Adam given the
  device's g, statistics to 1e-6; over several pair chunks and several passes of the weight loop
* learn() equals update() on its record; the rounds rule; determinism; the policy's own Adam state; errors; memory
* the iteration count across steps, update() and reset(); one learner on environments of different sizes; no eval episodes

Every case asserts and prints (pytest -s) the loop trip counts it is there for, from the device's SM count."""
import gc

import numpy as np
import pytest

from es_reference import (ES_PAIR_CHUNK, Adam, act_seed, compute_centered_ranks, coverage_sets, episodes_of_set, es_gradient64, global_grad,
                          noise_indices, perturbed, population_loops, reward_mean, update_loops)

pytestmark = pytest.mark.gpu

J = 5


def _graphs(n_graphs):
    from ddls_b200 import synth
    return [synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3), synth.chain_graph(6, 'chain6'),
            synth.residual_small_graph(), synth.transformer_like_graph(n_layers=1, name='tfm1', seed=4)][:n_graphs]


def _env(n_graphs, B, seed=5, **kw):
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    gs = _graphs(n_graphs)
    args = dict(max_partitions_per_op=16)
    args.update(kw)
    env = DeviceRampJobPartitioningEnvironment((4, 4, 2), gs, n_episodes=B, jobs_per_episode=J, min_op_run_time_quantum=2.0,
                                               interarrival=('exponential', 600.0), frac=(0.1, 1.0, 2), seed=seed, prewarm=True, **args)
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


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _wide_raw(names=('single', 'pair', 'multi300', 'star4096')):
    """the policy suite's MAX widths (128-wide node / edge / msg / hidden, 8 rounds, leaky_relu, tanh read-out of 128 units) with the
    environment's 17 graph features, and raw job-type graphs: self-loops, duplicate edges, zero in-degree nodes, a 4,096-message
    mailbox"""
    from test_gpu_policy_kernels import MAX, graphs
    from test_gpu_policy_kernels import _cfg as policy_cfg
    c = policy_cfg(dict(MAX, in_features_graph=17))
    rng = np.random.default_rng(5)
    return c, [g.features(c, rng) for g in graphs(True) if g.name in names]


def _population_case(case):
    """(env, the learner's policy, a reference policy with the same weights, graph_static [models, 6], config, actions, raw graphs)"""
    from ddls_b200 import policy as P
    from test_gpu_policy_kernels import UNMASKED, WIDE_FC, raw_policy
    from test_gpu_policy_kernels import _cfg as policy_cfg
    raw = None
    if case == 'scale':                                              # gnn.yaml, 8,704 episodes, three job types
        env, gs = _env(3, 8704)
        c, A, over = policy_cfg({}), 17, None
    elif case == 'wide':                                             # 305,187 weights on raw graphs; 32 actions
        c, raw = _wide_raw()
        env, _ = _env(4, 1024, max_partitions_per_op=31)
        A = 32
    else:
        over, A, kw = (WIDE_FC, 17, {}) if case == 'wide-fc' else (UNMASKED, 9, dict(max_partitions_per_op=8, apply_action_mask=False))
        env, gs = _env(2, 1024, **kw)
        c = policy_cfg(over)
    sd = P.random_state_dict(c, A, seed=4)
    if raw is not None:
        pol, ref = raw_policy(c, A, raw, sd), raw_policy(c, A, raw, sd)
        stat = np.stack([g.gs for g in raw])
    else:
        pol, ref = P.DeviceGNNPolicy(gs, A, over, sd), P.DeviceGNNPolicy(gs, A, over, sd)
        stat = np.stack([st['graph_static'] for st in pol.static])
    return env, pol, ref, stat, c, A, raw


def _round_readback(lrn, env, rnd):
    """one round run by hand as learn() runs it: [(the observation each act saw, the act's logits / log p / actions)], more"""
    o = env.reset()
    lrn.begin_round(env, rnd)
    seen = []
    for t in range(J):
        lrn.act(env, t)
        seen.append((o, lrn.act_read(env)))
        env.step_device()
        o = env.read()[0]
    return seen, lrn.end_round(env)


def _graph_features(o, stat):
    model = np.where(o['done'], -1, o['model']).astype(np.int32)
    gf = np.concatenate([o['graph_features_dynamic'][:, :9], stat[np.maximum(model, 0)], o['graph_features_dynamic'][:, 9:]], axis=1)
    return model, gf


def _set_weights(theta, noise, idx, s, N, sigma=0.05):
    return theta if s == 2 * N else perturbed(theta, noise, int(idx[s // 2]), sigma, +1 if s % 2 == 0 else -1)


def _check_population(lrn, env, ref, stat, theta, noise, sets, it, rnd, seen, seed=9):
    """every live episode of each set in `sets` equals ref holding that set's weights, deciding on all B rows (row b = episode b,
    so the draw keys agree): logits, log p and action bit for bit; dead rows give zeros.  Returns the decisions compared and the
    distinct actions among them."""
    B = env.B
    N = (B - lrn.n_eval(B)) // 2
    idx = noise_indices(seed, it, rnd, N, len(noise), len(theta))
    for o, (lg, lp, ac) in seen:
        dead = o['done'] | (o['model'] < 0)
        assert not lg[dead].any() and not lp[dead].any() and not ac[dead].any()
    checked, actions = 0, set()
    for s in sets:
        ref.set_weights(_set_weights(theta, noise, idx, s, N))
        eps = np.array(episodes_of_set(s, B, N), dtype=np.int64)
        for t, (o, (lg, lp, ac)) in enumerate(seen):
            model, gf = _graph_features(o, stat)
            wl, _, wp, wa = ref.decide(model, gf, o['action_mask'], sample=True, seed=act_seed(seed, it, rnd, t))
            live = eps[model[eps] >= 0]
            np.testing.assert_array_equal(lg[live].view(np.uint32), wl[live].view(np.uint32), err_msg=f'set {s} t {t} episodes {live}')
            np.testing.assert_array_equal(lp[live].view(np.uint32), wp[live].view(np.uint32), err_msg=f'set {s} t {t} episodes {live}')
            np.testing.assert_array_equal(ac[live], wa[live], err_msg=f'set {s} t {t} episodes {live}')
            checked += len(live)
            actions.update(ac[live].tolist())
    return checked, actions


def _check_record(lrn, env, it, rnd, n_weights, noise_size, seed=9):
    """the round's part of last_step() is the environment's own per-episode returns and decisions(), its noise indices and seeds"""
    B = env.B
    E = lrn.n_eval(B)
    N = (B - E) // 2
    rec = lrn.last_step()
    ret, n = np.asarray(env.episode_stats()['return']).astype(np.float32), env.decisions()
    p0, e0 = len(rec['noise_index']) - N, len(rec['eval_returns']) - E
    np.testing.assert_array_equal(rec['returns'][p0:].view(np.uint32), ret[:2 * N].reshape(N, 2).view(np.uint32))
    np.testing.assert_array_equal(rec['lengths'][p0:], n[:2 * N].reshape(N, 2))
    np.testing.assert_array_equal(rec['eval_returns'][e0:].view(np.uint32), ret[2 * N:].view(np.uint32))
    np.testing.assert_array_equal(rec['eval_lengths'][e0:], n[2 * N:])
    np.testing.assert_array_equal(rec['noise_index'][p0:], noise_indices(seed, it, rnd, N, noise_size, n_weights))
    np.testing.assert_array_equal(rec['seeds'][-J:], np.array([act_seed(seed, it, rnd, t) for t in range(J)], np.uint64))
    return rec


def _check_fp64(lrn, env, c, A, raw, stat, blob, s, seen, it=0, seed=9):
    """set s's episodes against gnn_reference's float64 forward: unmasked logits within the policy suite's bound, masked logits
    -FLT_MAX, and the sampled action the draw expected_draws restates (rows near a boundary excepted)"""
    from ddls_b200 import policy as P
    from gnn_reference import embed64, head64
    from test_gpu_policy_kernels import NEG_FLT_MAX_BITS, check_close, expected_draws
    sd = P.unpack_weights(blob, c, A)
    emb = np.stack([embed64(sd, c, g.nf, g.ef, g.src, g.dst) for g in raw])
    N = (env.B - lrn.n_eval(env.B)) // 2
    eps = np.array(episodes_of_set(s, env.B, N))
    worst, rows = 0.0, 0
    for t, (o, (lg, lp, ac)) in enumerate(seen):
        model, gf = _graph_features(o, stat)
        live = eps[model[eps] >= 0]
        if not len(live):
            continue
        mask = o['action_mask'][live].astype(np.uint8)
        wl, _ = head64(sd, c, emb[model[live]], gf[live], mask)
        valid = mask.astype(bool)
        worst = max(worst, check_close(lg[live][valid], wl[valid], f'set {s} t {t} logits'))
        assert (lg[live][~valid].view(np.uint32) == NEG_FLT_MAX_BITS).all()
        want, near = expected_draws(lg, act_seed(seed, it, 0, t))
        ok = live[~near[live]]
        np.testing.assert_array_equal(ac[ok], want[ok], err_msg=f'set {s} t {t}')
        rows += len(live)
    assert rows > 0
    return worst, rows


@pytest.mark.parametrize('case', ['scale', 'wide', 'wide-fc', 'unmasked'])
def test_population_at_training_sizes_equals_single_policies(case):
    """scale: gnn.yaml, 8,704 episodes, three job types (~99 items per embed CTA, up to 3 episodes per head warp on 132 SMs);
    wide: 305,187 weights, 8 rounds, 128 wide, a 4,097-node star, 32 actions; wide-fc: 512 hidden units (16 per lane);
    unmasked: apply_action_mask off, 9 actions.  Sets: es_reference.coverage_sets."""
    from ddls_b200.learn import DeviceESLearner
    env, pol, ref, stat, c, A, raw = _population_case(case)
    theta = pol.get_weights()
    noise = _noise(len(theta))
    lrn = DeviceESLearner(pol, _cfg(), noise=noise)
    try:
        B, sm = env.B, _sm_count()
        k = population_loops(B, lrn.n_eval(B), pol.n_models, sm)
        cov = coverage_sets(B, lrn.n_eval(B), pol.n_models, sm)
        sets = sorted(set().union(*cov.values()))
        print(f'\n[es-loops] population {case}: {len(theta)} weights, {k["items"]} items on {k["embed_grid"]} embed CTAs '
              f'({k["items_per_cta"]} per CTA, {sm} SMs), {k["head_warps"]} head warps ({k["episodes_per_warp"]} episodes per warp)')
        for path, ss in cov.items():
            print(f'[es-loops]   {path}: sets {ss}')
        assert k['items'] >= 3 * k['embed_grid']
        if case == 'scale':
            assert k['episodes_per_warp'] >= 2 and len(theta) == 21_920
        if case == 'wide':
            assert len(theta) == 305_187 and A == 32
        seen, more = _round_readback(lrn, env, 0)
        assert not more
        checked, actions = _check_population(lrn, env, ref, stat, theta, noise, sets, 0, 0, seen)
        assert len(actions) > 1                                       # the draws are not all the same action
        _check_record(lrn, env, 0, 0, len(theta), len(noise))
        print(f'[es-loops]   {len(sets)} sets checked, {checked} live decisions bit for bit, actions drawn {sorted(actions)}')
        if raw is not None:
            N = k['n_pairs']
            idx = noise_indices(9, 0, 0, N, len(noise), len(theta))
            for s in (2 * N, 0):
                worst, rows = _check_fp64(lrn, env, c, A, raw, stat, _set_weights(theta, noise, idx, s, N), s, seen)
                print(f'[es-loops]   set {s} against float64: {rows} decisions, logits max |err| {worst:.3e}')
    finally:
        lrn.close(); pol.close(); ref.close(); env.close()


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


UPDATE_PAIRS = dict(random=300, all_equal=300, one_pair=1, last_index=300, two_steps=300, chunk_1024=1024, chunk_1025=1025,
                    three_chunks=2500, wide_two_steps=1100)


@pytest.mark.parametrize('case', list(UPDATE_PAIRS))
def test_update_on_host_inputs(case):
    """chunk_1024 / chunk_1025: the edge of the update kernel's 1,024-pair chunk; three_chunks: a partial third chunk; wide_two_steps:
    305,187 weights, 5 passes of the weight loop on CTAs 0-136 and 4 on the rest, norm partials carried across them, Adam's
    second step on that state"""
    from ddls_b200.learn import DeviceESLearner
    env = None
    if case.startswith('wide'):
        from ddls_b200 import policy as P
        from test_gpu_policy_kernels import raw_policy
        c, gs = _wide_raw(('single', 'pair'))
        pol = raw_policy(c, 32, gs, P.random_state_dict(c, 32, seed=3))
    else:
        env, gs = _env(1, 8)
        pol = _policy(gs)
    theta = pol.get_weights()
    n = len(theta)
    noise = _noise(n)
    lrn = DeviceESLearner(pol, _cfg(stepsize=0.02, l2_coeff=0.005), noise=noise)
    rng = np.random.default_rng(3)
    try:
        N = UPDATE_PAIRS[case]
        steps = 2 if case.endswith('two_steps') else 1
        k = update_loops(N, n)
        print(f'\n[es-loops] update {case}: {N} pairs in {k["pair_chunks"]} chunks of {ES_PAIR_CHUNK}, {n} weights in '
              f'{k["max_weight_passes"]} / {k["min_weight_passes"]} passes (first / last CTA), {steps} steps')
        if case == 'chunk_1025':
            assert k['pair_chunks'] == 2
        if case == 'three_chunks':
            assert N > 2 * ES_PAIR_CHUNK and k['pair_chunks'] == 3
        if case.startswith('wide'):
            assert n == 305_187 and k['max_weight_passes'] == 5 > k['min_weight_passes'] and k['pair_chunks'] == 2
        ad = Adam(n, 0.02)
        for _ in range(steps):
            idx = rng.integers(0, len(noise) - n + 1, N)
            if case == 'last_index':
                idx[::7] = len(noise) - n
            R = np.full((N, 2), 2.0, np.float32) if case == 'all_equal' else rng.integers(-5, 6, (N, 2)).astype(np.float32)
            theta = _check_update(lrn, pol, noise, idx, R, ad, 0.005, theta)
    finally:
        lrn.close(); pol.close()
        if env is not None:
            env.close()


@pytest.mark.parametrize('rule', ['episodes', 'timesteps', 'scale'])
def test_learn_equals_update_and_runs_rounds(rule):
    """scale: 1,024 episodes, episodes_per_batch 2,500: 3 rounds of 511 pairs, so the learn path's update crosses a pair chunk"""
    from ddls_b200.learn import DeviceESLearner
    B = 1024 if rule == 'scale' else 16
    N = (B - 2) // 2
    env, gs = _env(2, B)
    kw = dict(episodes=dict(episodes_per_batch=30), timesteps=dict(episodes_per_batch=1, train_batch_size=2 * N * J + 1),
              scale=dict(episodes_per_batch=2500))[rule]
    pa, pb = _policy(gs), _policy(gs)
    noise = _noise(len(pa.get_weights()))
    la, lb = DeviceESLearner(pa, _cfg(**kw), noise=noise), DeviceESLearner(pb, _cfg(**kw), noise=noise)
    try:
        stats = la.learn(env)
        rec = la.last_step()
        rounds = int(stats['rounds'])
        steps = rec['lengths'].reshape(rounds, 2 * N).sum(1).cumsum()
        done = [2 * N * (r + 1) >= kw['episodes_per_batch'] and steps[r] >= kw.get('train_batch_size', 0) for r in range(rounds)]
        assert done[-1] and not any(done[:-1])                          # rounds run until both counts are reached, no further
        assert rounds == 3 if rule != 'timesteps' else rounds >= 2
        if rule == 'scale':
            k = update_loops(N * rounds, len(pa.get_weights()))
            print(f'\n[es-loops] learn {rule}: {rounds} rounds, {N * rounds} pairs in {k["pair_chunks"]} chunks')
            assert N * rounds > ES_PAIR_CHUNK
        assert stats['episodes_this_iter'] == 2 * N * rounds
        assert len(rec['noise_index']) == N * rounds and len(rec['seeds']) == J * rounds and len(rec['eval_returns']) == 2 * rounds
        assert stats['timesteps_this_iter'] == rec['lengths'].sum()
        assert stats['eval_return_mean'] == pytest.approx(rec['eval_returns'].astype(np.float64).mean())
        assert stats['episode_reward_mean'] == pytest.approx(stats['eval_return_mean'])
        assert stats['episode_len_mean'] == pytest.approx(rec['eval_lengths'].mean())
        for r in range(rounds):
            np.testing.assert_array_equal(rec['noise_index'][N * r:N * (r + 1)], noise_indices(9, 0, r, N, len(noise), len(pa.get_weights())))
        _, ranks, g = lb.update(rec['noise_index'], rec['returns'])
        np.testing.assert_array_equal(pa.get_weights().view(np.uint32), pb.get_weights().view(np.uint32))
        np.testing.assert_array_equal(ranks, rec['ranks'])
        np.testing.assert_array_equal(g, rec['g'])
    finally:
        la.close(); lb.close(); pa.close(); pb.close(); env.close()


def test_the_iteration_counts_steps_not_updates_or_resets():
    """step i's record (2 rounds each) uses noise_indices(seed, i, r, ...) and act_seed(seed, i, r, t); update() between steps
    and reset() (Adam only) leave the count alone"""
    from ddls_b200.learn import DeviceESLearner
    env, gs = _env(2, 16)
    pol = _policy(gs)
    n = len(pol.get_weights())
    noise = _noise(n)
    lrn = DeviceESLearner(pol, _cfg(episodes_per_batch=20), noise=noise)

    def check(i):
        rec = lrn.last_step()
        assert len(rec['seeds']) == 2 * J
        for r in range(2):
            np.testing.assert_array_equal(rec['noise_index'][7 * r:7 * (r + 1)], noise_indices(9, i, r, 7, len(noise), n))
            np.testing.assert_array_equal(rec['seeds'][J * r:J * (r + 1)], np.array([act_seed(9, i, r, t) for t in range(J)], np.uint64))
    try:
        lrn.learn(env)
        check(0)
        lrn.update(np.array([0, 5, 9], np.int32), np.arange(6, dtype=np.float32).reshape(3, 2))
        assert lrn.adam_state()[2] == 2
        lrn.learn(env)
        check(1)
        lrn.reset()
        assert lrn.adam_state()[2] == 0
        lrn.learn(env)
        check(2)
        assert lrn.adam_state()[2] == 1
    finally:
        lrn.close(); pol.close(); env.close()


def test_one_learner_across_environment_sizes():
    """16 episodes, then 1,024 (the population grows), then 16 again (it runs below its capacity): one round per step, each
    checked as the population at training sizes is, under iterations 0, 1, 2"""
    from ddls_b200.learn import DeviceESLearner
    envs = {16: _env(2, 16), 1024: _env(2, 1024, seed=6)}
    gs = envs[16][1]
    pol, ref = _policy(gs), _policy(gs)
    stat = np.stack([st['graph_static'] for st in pol.static])
    noise = _noise(len(pol.get_weights()))
    lrn = DeviceESLearner(pol, _cfg(), noise=noise)
    try:
        for it, B in enumerate((16, 1024, 16)):
            env = envs[B][0]
            theta = pol.get_weights()
            sets = sorted(set().union(*coverage_sets(B, 2, 2, _sm_count()).values()))
            seen, more = _round_readback(lrn, env, 0)
            assert not more
            checked, actions = _check_population(lrn, env, ref, stat, theta, noise, sets, it, 0, seen)
            _check_record(lrn, env, it, 0, len(theta), len(noise))
            print(f'\n[es-loops] sizes: step {it} on {B} episodes, {len(sets)} sets, {checked} live decisions bit for bit')
            assert checked > 0 and len(actions) > 1
            lrn.step()
    finally:
        lrn.close(); pol.close(); ref.close()
        for env, _ in envs.values():
            env.close()


def test_no_eval_episodes():
    """n_eval 0 with B even: no eval episode, every episode runs its own set; eval_return_mean is NaN and episode_reward_mean the
    mean of the earlier steps' eval returns, NaN before there are any (steps with n_eval 0, 2, 0)"""
    from ddls_b200.learn import DeviceESLearner
    env, gs = _env(2, 16)
    pol, ref = _policy(gs), _policy(gs)
    stat = np.stack([st['graph_static'] for st in pol.static])
    noise = _noise(len(pol.get_weights()))
    lrn = DeviceESLearner(pol, _cfg(n_eval=0), noise=noise)
    evals = []
    try:
        for it, E in enumerate((0, 2, 0)):
            lrn.config.n_eval = E
            theta = pol.get_weights()
            seen, more = _round_readback(lrn, env, 0)
            assert not more
            if E == 0:
                checked, _ = _check_population(lrn, env, ref, stat, theta, noise, range(16), it, 0, seen)
                assert checked >= 16
            rec = _check_record(lrn, env, it, 0, len(theta), len(noise))
            assert len(rec['noise_index']) == (16 - E) // 2 and len(rec['eval_returns']) == E
            stats = lrn.step()
            if E:
                evals.append(rec['eval_returns'].astype(np.float64).mean())
                assert stats['eval_return_mean'] == pytest.approx(evals[-1])
            else:
                assert np.isnan(stats['eval_return_mean']) and np.isnan(stats['episode_len_mean'])
            want = reward_mean(evals, lrn.config.report_length)
            got = stats['episode_reward_mean']
            assert (np.isnan(want) and np.isnan(got)) or got == pytest.approx(want), (it, got, want)
            assert stats['episodes_this_iter'] == 16 - E
    finally:
        lrn.close(); pol.close(); ref.close(); env.close()


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
