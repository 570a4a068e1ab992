"""CPU: the population's C symbols are exported, its configuration errors are raised before anything runs on a device, and the
per-group act draw restated in Python is the single policy's draw on the group's twin environment."""
import types

import numpy as np
import pytest

POPULATION_SYMBOLS = ['ramp_population_create', 'ramp_population_destroy', 'ramp_population_set_weights', 'ramp_population_get_weights',
                      'ramp_population_act', 'ramp_population_learn', 'ramp_population_learner_state', 'ramp_population_embed_ctas']


def test_population_symbols_exported():
    from ddls_b200 import build, engine
    build.build()
    lib = engine.load_library()
    for name in POPULATION_SYMBOLS:
        assert hasattr(lib, name), name
        assert name in engine.EXPORTED_SYMBOLS, name


def test_environment_not_divisible_by_the_sets_is_refused():
    from ddls_b200.policy import DeviceGNNPolicyPopulation
    pop = types.SimpleNamespace(K=3)
    assert DeviceGNNPolicyPopulation.group_size(pop, types.SimpleNamespace(B=12)) == 4
    with pytest.raises(ValueError, match='do not split into 3 groups'):
        DeviceGNNPolicyPopulation.group_size(pop, types.SimpleNamespace(B=10))


@pytest.mark.parametrize('field', ['sgd_minibatch_size', 'num_sgd_iter'])
def test_configs_must_share_the_launch_loop(field):
    import dataclasses
    from ddls_b200.learn import DevicePopulationPPOLearner, PPOConfig
    pop = types.SimpleNamespace(K=2, _L=None)
    cfgs = [PPOConfig(), dataclasses.replace(PPOConfig(), **{field: getattr(PPOConfig(), field) + 1})]
    with pytest.raises(ValueError, match=field):
        DevicePopulationPPOLearner(pop, cfgs)
    with pytest.raises(ValueError, match='3 configs for a population of 2'):
        DevicePopulationPPOLearner(pop, [PPOConfig()] * 3)


def test_state_dict_of_the_wrong_shape_names_its_set():
    from ddls_b200 import policy as P
    sds = [P.random_state_dict(P.DEFAULT_CONFIG, 17, seed=s) for s in range(3)]
    sds[2]['graph_module.1.weight'] = np.zeros((3, 3), np.float32)
    with pytest.raises(ValueError, match=r'state_dicts\[2\]: graph_module.1.weight'):
        P.DeviceGNNPolicyPopulation([], 17, None, sds)
    with pytest.raises(ValueError, match=r'state_dicts\[1\]: a blob'):
        P.DeviceGNNPolicyPopulation([], 17, None, [sds[0], np.zeros(5, np.float32)])


def test_group_draw_is_the_twin_policys_draw():
    """episode b of the population's call c draws as episode b - k b0 of a single policy's call c with group k's seed"""
    from ddls_b200 import policy as P
    seeds, b0 = [11, 2 ** 63 + 5, 0, 97], 6
    for calls in (1, 2, 9):
        for b in range(len(seeds) * b0):
            k, i, key = P.population_draw(seeds, calls, b, b0)
            assert (k, i) == divmod(b, b0)
            assert key == P.act_draw_key(seeds[k], calls, i)
    # ramp_policy_head_kernel's formula, written out: splitmix64((seed ^ golden calls) ^ row_mix b)
    seed, calls, b = 12345, 3, 7
    x = (seed ^ (0x9E3779B97F4A7C15 * calls % 2 ** 64)) ^ (b * 0xD1342543DE82EF95 % 2 ** 64)
    assert P.act_draw_key(seed, calls, b) == P.splitmix64(x)
    assert P.splitmix64(0) == 0xE220A8397B1DCDAF                          # splitmix64's published first output for seed 0
