"""CPU: DevicePopulationESLearner's configuration checks, the round rule's numpy model (es_population_reference.es_rounds) and
the ctypes signatures of ramp_population_es_*.  No compute call is made."""
import os
import re
import types

import numpy as np
import pytest

from es_population_reference import es_rounds

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def lib():
    from ddls_b200 import build, engine
    build.build()
    return engine.load_library()


def _population(lib, K=3, n_weights=100):
    """what the learner reads of a population before it creates anything: K, the library and each set's weight count"""
    return types.SimpleNamespace(K=K, _L=lib, _h=None, weight_count=lambda k: n_weights)


def _cfgs(K=3, **kw):
    from ddls_b200.learn import ESConfig
    return [ESConfig(noise_size=1000, n_eval=2, **kw) for _ in range(K)]


def test_config_count_names_the_population_size(lib):
    from ddls_b200.learn import DevicePopulationESLearner
    with pytest.raises(ValueError, match='2 configs for a population of 3 sets'):
        DevicePopulationESLearner(_population(lib), _cfgs(2), noise=np.zeros(1000, np.float32))


def test_noise_size_is_shared(lib):
    from ddls_b200.learn import DevicePopulationESLearner
    cfgs = _cfgs()
    cfgs[2].noise_size = 2000
    with pytest.raises(ValueError, match='noise_size must be the same for every set.*set 2 differs'):
        DevicePopulationESLearner(_population(lib), cfgs, noise=np.zeros(1000, np.float32))


def test_noise_table_covers_every_set(lib):
    from ddls_b200.learn import DevicePopulationESLearner
    pop = _population(lib)
    pop.weight_count = lambda k: 5000 if k == 1 else 100
    with pytest.raises(ValueError, match='set 1: a noise table of 1000 floats is smaller than its 5000 weights'):
        DevicePopulationESLearner(pop, _cfgs(), noise=np.zeros(1000, np.float32))


@pytest.mark.parametrize('field,value,rule', [('observation_filter', 'MeanStdFilter', "'NoFilter'"), ('noise_stdev', -1.0, '>= 0'),
                                              ('adam_beta1', 1.0, r'in \[0, 1\)'), ('report_length', 0, '>= 1'), ('n_eval', -2, 'None or >= 0')])
def test_each_config_is_checked_naming_the_set(lib, field, value, rule):
    from ddls_b200.learn import DevicePopulationESLearner
    cfgs = _cfgs()
    setattr(cfgs[1], field, value)
    with pytest.raises(ValueError, match=f'set 1: {field} = .*it must be {rule}'):
        DevicePopulationESLearner(_population(lib), cfgs, noise=np.zeros(1000, np.float32))


def test_too_few_noisy_episodes_in_a_group_names_the_set():
    from ddls_b200.learn import DevicePopulationESLearner
    lrn = DevicePopulationESLearner.__new__(DevicePopulationESLearner)
    lrn.configs = _cfgs()
    lrn.configs[2].n_eval = 5
    with pytest.raises(ValueError, match='set 2: 6 episodes per group less 5 eval episodes leave 1'):
        lrn._check_groups(6)
    lrn.configs[2].n_eval = 3
    with pytest.raises(ValueError, match='set 2: .* leave 3, which must be even'):
        lrn._check_groups(6)
    lrn.configs[2].n_eval = None                      # eval_prob's share: 1 of 6, made even with b: 2
    assert lrn.n_eval(6)[2] == 2
    lrn._check_groups(6)


def test_round_rule_model():
    """group 0 stops on its episodes, group 1 on its env-steps, group 2 after one round; the population runs 3 rounds"""
    K, b, R = 3, 6, 4
    n_pairs = [2, 2, 3]
    lengths = np.full((R, K, b), 5)
    lengths[:, 1, :] = 2                              # 4 noisy episodes of 2 env-steps a round: 8 a round
    records, r_k, rounds = es_rounds(lengths, n_pairs, episodes_per_batch=[12, 1, 6], train_batch_size=[0, 20, 30])
    assert list(r_k) == [3, 3, 1] and rounds == 3
    assert records[:3].tolist() == [[True, True, True], [True, True, False], [True, True, False]]
    lengths[1, 1, :2] = 10                            # a longer round 1: group 1's 20 env-steps come a round earlier
    _, r_k, rounds = es_rounds(lengths, n_pairs, episodes_per_batch=[12, 1, 6], train_batch_size=[0, 20, 30])
    assert list(r_k) == [3, 2, 1] and rounds == 3
    # the eval episodes' env-steps never count
    lengths[:] = 1
    lengths[:, :, 4:] = 100
    _, r_k, _ = es_rounds(lengths, [2, 2, 2], episodes_per_batch=[0, 0, 0], train_batch_size=[4, 8, 12])
    assert list(r_k) == [1, 2, 3]
    with pytest.raises(ValueError, match='group 2 needs more than 4 rounds'):
        es_rounds(lengths, [2, 2, 2], episodes_per_batch=[0, 0, 0], train_batch_size=[4, 8, 17])


def _declared():
    src = open(os.path.join(ROOT, 'include', 'ramp_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return {m.group(1): [a.strip() for a in m.group(2).split(',')]
            for m in re.finditer(r'\b(ramp_population_es_[a-z_]+)\s*\(([^)]*)\)', src)}


def test_ctypes_argument_types_follow_the_header(lib):
    import ctypes as C
    from ddls_b200 import learn
    learn._bind(lib)
    decl = _declared()
    assert len(decl) == 12
    for name, params in decl.items():
        fn = getattr(lib, name)
        assert len(fn.argtypes) == len(params), name
        for ct, p in zip(fn.argtypes, params):
            if '*' in p:
                assert ct is C.c_void_p or issubclass(ct, C._Pointer), (name, p)
            else:
                assert ct is {'int32_t': C.c_int32, 'int64_t': C.c_int64}[p.split()[0]], (name, p)
        assert fn.restype is (None if name.endswith('_destroy') else C.c_int), name
    assert lib.ramp_population_es_round_begin.argtypes[2]._type_ is learn._CESConfig
