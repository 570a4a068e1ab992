"""CPU: PopulationBasedTraining's decisions against a numpy restatement of Ray Tune's PBT rules (ranking with ties, quantile sizes,
donor choice, resample against perturb, list fields), its refusals, and the ctypes signatures of the training-state and copy
entry points.  No compute call is made: the population and learner are stand-ins that record the copies."""
import dataclasses
import math
import os
import re
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# ---- the numpy restatement ----
_G, _C1, _C2 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB)


def _sm64(x):
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over='ignore'):
        x = x + _G
        x = (x ^ (x >> np.uint64(30))) * _C1
        x = (x ^ (x >> np.uint64(27))) * _C2
    return x ^ (x >> np.uint64(31))


def _u(seed, step, k, slot, j):
    """splitmix64 chained over (seed, step, set, slot, draw), top 53 bits, for an array of sets k"""
    k = np.asarray(k, dtype=np.uint64)
    x = _sm64(np.full(k.shape, seed, dtype=np.uint64))
    for v in (np.uint64(step), k, np.uint64(slot), np.uint64(j)):
        x = _sm64(x ^ v)
    return (x >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def _q(K, frac=0.25):
    n = int(math.ceil(K * frac))
    return n if n <= K / 2 else int(math.floor(K / 2))     # Ray's _quantiles


def ref_decide(scores, values, mutations, step, seed, p=0.25, factors=(1.2, 0.8)):
    """values: {field: array [K]}.  Returns (bottom, donors, {field: new values of the bottom sets}, {field: resampled mask})"""
    s = np.asarray(scores, dtype=np.float64)
    K = len(s)
    order = np.lexsort((np.arange(K), np.where(np.isnan(s), -np.inf, s)))
    n = _q(K)
    bottom, top = order[:n], order[K - n:]
    donors = top[np.minimum((_u(seed, step, bottom, 0, 0) * n).astype(np.int64), max(n - 1, 0))] if n else bottom
    new, resampled = {}, {}
    for f_i, (f, spec) in enumerate(mutations.items()):
        u0, u1 = _u(seed, step, bottom, f_i + 1, 0), _u(seed, step, bottom, f_i + 1, 1)
        v = np.asarray(values[f], dtype=object)[donors]
        out = []
        if isinstance(spec, list):
            rs = (u0 < p) | np.array([x not in spec for x in v], dtype=bool)
            for x, r, w in zip(v, rs, u1):
                if r:
                    out.append(spec[min(int(w * len(spec)), len(spec) - 1)])
                else:
                    i = spec.index(x) + (-1 if w < 0.5 else 1)
                    out.append(spec[int(np.clip(i, 0, len(spec) - 1))])
        else:
            rs = u0 < p
            for x, r, w in zip(v, rs, u1):
                y = spec(w) if r else x * factors[min(int(w * len(factors)), len(factors) - 1)]
                out.append(int(y) if isinstance(x, int) else y)
        new[f], resampled[f] = out, rs
    return bottom, donors, new, resampled


# ---- stand-ins ----

def _population(K, shapes=None):
    from ddls_b200 import policy as P
    cfg = P.c_config(P.DEFAULT_CONFIG, 17, 1)
    ccfgs = [cfg] * K
    if shapes:
        ccfgs = [P.c_config(dict(P.DEFAULT_CONFIG, out_features_msg=s), 17, 1) for s in shapes]
    pop = types.SimpleNamespace(K=K, _ccfgs=ccfgs, copies=[])
    pop.copy_sets = lambda dst, src: pop.copies.append((list(dst), list(src)))
    return pop


def _learner(cls, K, configs, pop=None):
    lrn = cls.__new__(cls)
    lrn.population = pop or _population(K)
    lrn.configs = configs
    if cls.__name__ == 'DevicePopulationESLearner':
        lrn.es_copies = []
        lrn.copy_sets = lambda dst, src: lrn.es_copies.append((list(dst), list(src)))
    return lrn


def test_quantile_sizes():
    from ddls_b200.pbt import quantile_size
    for K, n in {1: 0, 2: 1, 3: 1, 4: 1, 8: 2, 128: 32}.items():
        assert quantile_size(K) == _q(K) == n, K


def test_ranking_breaks_ties_by_set_index():
    from ddls_b200.pbt import ranking
    assert ranking([1.0] * 5) == [0, 1, 2, 3, 4]
    assert ranking([2.0, 1.0, 2.0, 1.0]) == [1, 3, 0, 2]
    assert ranking([0.0, float('nan'), -5.0]) == [1, 2, 0]                # NaN ranks lowest
    s = [3.0, 1.0, 1.0, 3.0, 2.0, 1.0, 3.0, 2.0]
    assert ranking(s) == list(np.lexsort((np.arange(8), s)))


def test_draws_are_splitmix64_keyed():
    from ddls_b200.pbt import draw
    for seed, step, k, slot, j in [(0, 0, 0, 0, 0), (7, 3, 127, 2, 1), (2 ** 64 - 1, 10, 5, 0, 1)]:
        assert draw(seed, step, k, slot, j) == _u(seed, step, [k], slot, j)[0]
    assert len({draw(1, 0, k, 0, 0) for k in range(64)}) == 64


@pytest.mark.parametrize('K', [1, 2, 3, 4, 8, 128])
def test_decide_matches_the_restatement(K):
    from ddls_b200 import pbt
    from ddls_b200.learn import PPOConfig
    rng = np.random.default_rng(K)
    mutations = {'lr': pbt.log_uniform(1e-5, 1e-3), 'entropy_coeff': [0.0, 0.001, 0.003, 0.01, 0.03]}
    configs = [PPOConfig(lr=float(rng.uniform(1e-5, 1e-3)), entropy_coeff=[0.0, 0.001, 0.003, 0.01, 0.5][k % 5], seed=k) for k in range(K)]
    resampled = {f: 0 for f in mutations}
    for step in range(6):
        scores = np.round(rng.normal(size=K), 1)                              # ties
        recs = pbt.decide(scores, configs, mutations, step, seed=9)
        bottom, donors, new, rs = ref_decide(scores, {f: [getattr(c, f) for c in configs] for f in mutations}, mutations, step, 9)
        assert [r['set'] for r in recs] == list(bottom) and [r['donor'] for r in recs] == list(donors)
        for f in mutations:
            assert [r['new'][f] for r in recs] == new[f], (K, step, f)
            assert [r['old'][f] for r in recs] == [getattr(configs[k], f) for k in bottom]
            resampled[f] += int(np.sum(rs[f]))
    if K == 128:                                                               # both branches, in both kinds of field
        n = 6 * 32
        assert all(0 < resampled[f] < n for f in mutations), resampled


def test_int_field_stays_int_and_list_moves_one_index():
    from ddls_b200.pbt import explore, draw
    for k in range(40):
        v = explore(100, lambda u: 1 + 1000 * u, 3, 0, k, 1)
        assert isinstance(v, int)
        u0, u1 = draw(3, 0, k, 1, 0), draw(3, 0, k, 1, 1)
        assert v == (int(1 + 1000 * u1) if u0 < 0.25 else int(100 * (1.2 if u1 < 0.5 else 0.8)))
        w = explore(4, [1, 2, 4, 8], 3, 0, k, 1)
        if u0 >= 0.25:
            assert w == (2 if u1 < 0.5 else 8)
    assert explore(3, [1, 2, 4], 0, 0, 0, 1) in (1, 2, 4)                     # a value not in the list is resampled


@pytest.mark.parametrize('algo', ['ppo', 'impala', 'pg', 'es'])
def test_scheduler_makes_the_restated_decisions(algo):
    """recorded score sequences: every interval-th step() copies the restatement's pairs and sets its configs"""
    from ddls_b200 import learn, pbt
    K, interval = 8, 2
    cls, cfg = {'ppo': (learn.DevicePopulationPPOLearner, lambda k: learn.PPOConfig(lr=1e-4 * (k + 1), seed=100 + k, kl_coeff=0.01 * k)),
                'impala': (learn.DevicePopulationIMPALALearner, lambda k: learn.IMPALAConfig(lr=1e-4 * (k + 1))),
                'pg': (learn.DevicePopulationPGLearner, lambda k: learn.PGConfig(lr=1e-4 * (k + 1), gamma=[0.9, 0.99][k % 2])),
                'es': (learn.DevicePopulationESLearner, lambda k: learn.ESConfig(stepsize=0.01 * (k + 1), seed=100 + k))}[algo]
    field = {'ppo': 'lr', 'impala': 'lr', 'pg': 'lr', 'es': 'stepsize'}[algo]
    second = {'ppo': ('entropy_coeff', [0.0, 0.01]), 'impala': ('entropy_coeff', [0.0, 0.01]), 'pg': ('gamma', [0.9, 0.99, 0.999]),
              'es': ('noise_stdev', [0.01, 0.02, 0.05])}[algo]
    mutations = {field: pbt.log_uniform(1e-5, 1e-1), second[0]: second[1]}
    lrn = _learner(cls, K, [cfg(k) for k in range(K)])
    sched = pbt.PopulationBasedTraining(lrn, mutations, interval=interval, seed=5)
    mirror = [dataclasses.replace(c) for c in lrn.configs]
    rng = np.random.default_rng(1)
    for call in range(1, 9):
        scores = np.round(rng.normal(size=K), 1)
        recs = sched.step(scores)
        if call % interval:
            assert recs == []
            continue
        bottom, donors, new, _ = ref_decide(scores, {f: [getattr(c, f) for c in mirror] for f in mutations}, mutations, call // interval - 1, 5)
        assert lrn.population.copies[-1] == (list(bottom), list(donors))
        if algo == 'es':
            assert lrn.es_copies[-1] == (list(bottom), list(donors))
        for i, (k, j) in enumerate(zip(bottom, donors)):
            want = dataclasses.replace(mirror[j], **{f: new[f][i] for f in mutations})
            if hasattr(want, 'seed'):
                want = dataclasses.replace(want, seed=mirror[k].seed)          # the recipient keeps its own seed
            mirror[k] = want
        assert lrn.configs == mirror, call
    assert len(lrn.population.copies) == 4


def test_refusals():
    from ddls_b200 import learn, pbt
    K = 4
    ppo = _learner(learn.DevicePopulationPPOLearner, K, [learn.PPOConfig() for _ in range(K)])
    for field in ('sgd_minibatch_size', 'num_sgd_iter'):
        with pytest.raises(ValueError, match=f"mutation of '{field}': DevicePopulationPPOLearner needs it to be the same for every set"):
            pbt.PopulationBasedTraining(ppo, {field: [64, 128]})
    imp = _learner(learn.DevicePopulationIMPALALearner, K, [learn.IMPALAConfig() for _ in range(K)])
    for field in ('rollout_fragment_length', 'train_batch_size'):
        with pytest.raises(ValueError, match=f"mutation of '{field}': DevicePopulationIMPALALearner needs it"):
            pbt.PopulationBasedTraining(imp, {field: [4, 8]})
    es = _learner(learn.DevicePopulationESLearner, K, [learn.ESConfig() for _ in range(K)])
    with pytest.raises(ValueError, match="mutation of 'noise_size': DevicePopulationESLearner needs it"):
        pbt.PopulationBasedTraining(es, {'noise_size': [1000, 2000]})
    with pytest.raises(ValueError, match="mutation of 'seed'"):
        pbt.PopulationBasedTraining(ppo, {'seed': [1, 2]})
    with pytest.raises(ValueError, match="mutation of 'lambda': PPOConfig has no such field"):
        pbt.PopulationBasedTraining(ppo, {'lambda': [0.9]})
    with pytest.raises(ValueError, match="mutation of 'lr': an empty list"):
        pbt.PopulationBasedTraining(ppo, {'lr': []})
    mixed = _learner(learn.DevicePopulationPGLearner, K, [learn.PGConfig() for _ in range(K)], pop=_population(K, shapes=[32, 32, 16, 32]))
    with pytest.raises(ValueError, match='every set must have one shape: set 2 differs from set 0'):
        pbt.PopulationBasedTraining(mixed, {'lr': pbt.uniform(0, 1)})
    with pytest.raises(TypeError, match='PBT wraps a population learner'):
        pbt.PopulationBasedTraining(learn.DevicePGLearner.__new__(learn.DevicePGLearner), {'lr': [1e-4]})
    sched = pbt.PopulationBasedTraining(ppo, {'lr': pbt.uniform(0, 1)})
    with pytest.raises(ValueError, match='3 scores for a population of 4 sets'):
        sched.step([1.0, 2.0, 3.0])


def test_fitness_helpers():
    from ddls_b200.pbt import group_returns, es_scores
    reward = np.array([[1.0, 2.0, 3.0, 4.0], [5.0, 6.0, 7.0, 8.0]])
    live = np.array([[True, True, True, True], [True, False, True, True]])
    assert np.allclose(group_returns({'reward': reward, 'live': live}, 2), [(6.0 + 2.0) / 2, (10.0 + 12.0) / 2])
    assert np.array_equal(es_scores([{'episode_reward_mean': 1.5}, {'episode_reward_mean': -2.0}]), [1.5, -2.0])


_NEW = ('ramp_policy_set_learner_state', 'ramp_policy_get_act_count', 'ramp_policy_set_act_count', 'ramp_es_set_state',
        'ramp_es_get_progress', 'ramp_es_set_progress', 'ramp_population_set_learner_state', 'ramp_population_copy_sets',
        'ramp_population_get_act_count', 'ramp_population_set_act_count', 'ramp_population_set_es_state',
        'ramp_population_get_es_progress', 'ramp_population_set_es_progress', 'ramp_population_copy_es_sets')


def test_ctypes_argument_types_follow_the_header():
    import ctypes as C
    from ddls_b200 import build, engine, learn, policy
    build.build()
    lib = engine.load_library()
    learn._bind(lib)
    policy._bind(lib)
    policy._bind_population(lib)
    src = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'ramp_b200.h')).read(), flags=re.S)
    decl = {m.group(1): [a.strip() for a in m.group(2).split(',')] for m in re.finditer(r'\b(ramp_[a-z_0-9]+)\s*\(([^)]*)\)', src)}
    for name in _NEW:
        assert name in engine.EXPORTED_SYMBOLS and name in decl, name
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and len(fn.argtypes) == len(decl[name]), name
        for ct, p in zip(fn.argtypes, decl[name]):
            if '*' in p:
                assert ct is C.c_void_p or issubclass(ct, C._Pointer), (name, p)
            else:
                assert ct is {'int32_t': C.c_int32, 'int64_t': C.c_int64, 'uint64_t': C.c_uint64}[p.split()[0]], (name, p)
