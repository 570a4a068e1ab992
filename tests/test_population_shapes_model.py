"""CPU: a population with one configuration per set -- its C symbol is exported and bound, and its configuration errors are raised,
naming the set, before anything runs on a device."""
import numpy as np
import pytest

A = 17
SMALL = dict(out_features_msg=8, out_features_hidden=16, out_features_node=8, out_features_graph=4, num_rounds=3, fcnet_hiddens=(32,),
             vf_share_layers=True)


def test_create_configs_exported_and_bound():
    from ddls_b200 import build, engine
    from ddls_b200 import policy as P
    build.build()
    lib = engine.load_library()
    assert hasattr(lib, 'ramp_population_create_configs')
    assert 'ramp_population_create_configs' in engine.EXPORTED_SYMBOLS
    P._bind_population(lib)
    assert lib.ramp_population_create_configs.argtypes[2]._type_ is P._Config


def _sds(configs):
    from ddls_b200 import policy as P
    return [P.random_state_dict(dict(P.DEFAULT_CONFIG, **c), A, seed=k) for k, c in enumerate(configs)]


@pytest.mark.parametrize('field', ['in_features_node', 'in_features_edge', 'in_features_graph'])
def test_a_field_the_environment_fixes_names_its_set(field):
    from ddls_b200 import policy as P
    cfgs = [{}, SMALL, dict(SMALL, **{field: P.DEFAULT_CONFIG[field] + 1})]
    with pytest.raises(ValueError, match=rf'configs\[2\]: {field} = '):
        P.DeviceGNNPolicyPopulation([], A, cfgs, _sds(cfgs))


def test_a_state_dict_of_another_sets_shape_names_its_set():
    from ddls_b200 import policy as P
    cfgs = [{}, SMALL, {}]
    sds = _sds(cfgs)
    with pytest.raises(ValueError, match=r'state_dicts\[1\]: '):
        P.DeviceGNNPolicyPopulation([], A, cfgs, [sds[0], sds[0], sds[2]])
    with pytest.raises(ValueError, match=r'state_dicts\[2\]: '):
        P.DeviceGNNPolicyPopulation([], A, cfgs, [sds[0], sds[1], sds[1]])
    blob = P.pack_weights(sds[0], P.DEFAULT_CONFIG, A)
    with pytest.raises(ValueError, match=r"state_dicts\[1\]: a blob of shape .*set 1's configuration has"):
        P.DeviceGNNPolicyPopulation([], A, cfgs, [blob, blob, blob])


def test_the_wrong_number_of_configs_is_refused():
    from ddls_b200 import policy as P
    cfgs = [{}, SMALL]
    with pytest.raises(ValueError, match='2 configs for 3 state_dicts'):
        P.DeviceGNNPolicyPopulation([], A, cfgs, _sds(cfgs + [{}]))


def test_a_read_out_the_device_lacks_names_its_set():
    from ddls_b200 import policy as P
    cfgs = [{}, dict(SMALL, fcnet_hiddens=(32, 32))]
    with pytest.raises(ValueError, match=r'configs\[1\]: the device read-out has one hidden layer'):
        P.DeviceGNNPolicyPopulation([], A, cfgs, _sds([{}, {}]))
    with pytest.raises(ValueError, match=r'configs\[1\]: module_depth must be 1'):
        P.DeviceGNNPolicyPopulation([], A, [{}, dict(SMALL, module_depth=2)], _sds([{}, SMALL]))


def test_weight_count_is_the_blob_length():
    from ddls_b200 import policy as P
    for c in ({}, SMALL, dict(SMALL, vf_share_layers=False, fcnet_hiddens=(A,))):
        cfg = dict(P.DEFAULT_CONFIG, **c)
        assert P.weight_count(cfg, A) == len(P.pack_weights(P.random_state_dict(cfg, A), cfg, A))
    # PHASE 3's 128 shapes at gnn.yaml's read-out: 13,972 to 66,728 weights, 3.74 M in all
    grid = [dict(P.DEFAULT_CONFIG, out_features_msg=m, out_features_hidden=h, out_features_node=n, num_rounds=r)
            for m in (8, 16, 32, 64) for h in (8, 16, 32, 64) for n in (8, 16, 32, 64) for r in (2, 4)]
    counts = np.array([P.weight_count(c, A) for c in grid])
    assert len(grid) == 128 and counts.min() == 13_972 and counts.max() == 66_728 and round(counts.sum() / 1e6, 2) == 3.74
