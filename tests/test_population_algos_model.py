"""CPU: the IMPALA and PG population learners' C symbols are exported and bound, and their configuration errors -- configs that
disagree on what sets IMPALA's launch loop, the wrong number of configs, one set's invalid config -- are raised, naming the field and
the set, before anything runs on a device."""
import dataclasses
import types

import pytest

SYMBOLS = ['ramp_population_learn_impala', 'ramp_population_learn_pg', 'ramp_population_vtrace_read']


class _Lib:
    """a stand-in library: every function is a namespace that takes the signature _bind gives it"""
    def __getattr__(self, name):
        f = types.SimpleNamespace()
        setattr(self, name, f)
        return f


def _pop(K):
    return types.SimpleNamespace(K=K, _L=_Lib())


def test_population_algo_symbols_exported_and_bound():
    from ddls_b200 import build, engine, learn
    build.build()
    lib = engine.load_library()
    learn._bind(lib)
    for name in SYMBOLS:
        assert hasattr(lib, name), name
        assert name in engine.EXPORTED_SYMBOLS, name
        assert getattr(lib, name).argtypes, name
    assert getattr(lib, 'ramp_population_learn_impala').argtypes[3]._type_ is learn._CIMPALAConfig
    assert getattr(lib, 'ramp_population_learn_pg').argtypes[3]._type_ is learn._CPGConfig


@pytest.mark.parametrize('field', ['rollout_fragment_length', 'train_batch_size'])
def test_impala_configs_must_share_the_launch_loop(field):
    from ddls_b200.learn import DevicePopulationIMPALALearner, IMPALAConfig
    cfgs = [IMPALAConfig(rollout_fragment_length=4), IMPALAConfig(rollout_fragment_length=4), IMPALAConfig(rollout_fragment_length=4)]
    cfgs[2] = dataclasses.replace(cfgs[2], **{field: getattr(cfgs[2], field) * 2})
    with pytest.raises(ValueError, match=rf'{field} must be the same for every set.*set 2 differs'):
        DevicePopulationIMPALALearner(_pop(3), cfgs)


def test_impala_per_set_hyperparameters_may_differ():
    """only the launch loop's fields are shared: configs that differ in everything else are accepted, and kept as copies"""
    from ddls_b200.learn import DevicePopulationIMPALALearner, DevicePopulationPGLearner, IMPALAConfig, PGConfig
    cfgs = [IMPALAConfig(), IMPALAConfig(gamma=0.9, vtrace_clip_rho_threshold=0.5, vtrace_clip_pg_rho_threshold=2.0, vf_loss_coeff=1.0,
                                         entropy_coeff=0.0, grad_clip=0.0, lr=1e-3, adam_beta1=0.8, adam_beta2=0.99, adam_eps=1e-6)]
    lrn = DevicePopulationIMPALALearner(_pop(2), cfgs)
    assert lrn.configs == cfgs and lrn.configs[1] is not cfgs[1]
    pg = [PGConfig(), PGConfig(gamma=0.5, lr=1e-3, grad_clip=2.0)]
    assert DevicePopulationPGLearner(_pop(2), pg).configs == pg


@pytest.mark.parametrize('cls', ['DevicePopulationIMPALALearner', 'DevicePopulationPGLearner'])
def test_wrong_number_of_configs(cls):
    from ddls_b200 import learn
    cfg = learn.IMPALAConfig() if 'IMPALA' in cls else learn.PGConfig()
    with pytest.raises(ValueError, match='3 configs for a population of 2'):
        getattr(learn, cls)(_pop(2), [cfg] * 3)
    with pytest.raises(ValueError, match='1 configs for a population of 2'):
        getattr(learn, cls)(_pop(2), [cfg])


@pytest.mark.parametrize('cls,field,value', [
    ('DevicePopulationIMPALALearner', 'vtrace_clip_rho_threshold', 0.0),
    ('DevicePopulationIMPALALearner', 'vtrace_clip_pg_rho_threshold', -1.0),
    ('DevicePopulationIMPALALearner', 'adam_eps', 0.0),
    ('DevicePopulationIMPALALearner', 'lr', -1e-4),
    ('DevicePopulationPGLearner', 'gamma', -0.5),
    ('DevicePopulationPGLearner', 'adam_eps', 0.0),
    ('DevicePopulationPGLearner', 'lr', -1e-4),
])
def test_invalid_config_names_its_set(cls, field, value):
    from ddls_b200 import learn
    base = learn.IMPALAConfig() if 'IMPALA' in cls else learn.PGConfig()
    cfgs = [base, base, dataclasses.replace(base, **{field: value}), base]
    with pytest.raises(ValueError, match=rf'set 2: {field} = '):
        getattr(learn, cls)(_pop(4), cfgs)


def test_population_learners_share_adam_state_and_checks():
    from ddls_b200 import learn
    for cls in (learn.DevicePopulationPPOLearner, learn.DevicePopulationIMPALALearner, learn.DevicePopulationPGLearner):
        assert issubclass(cls, learn._PopulationLearner)
        assert cls.adam_state is learn._PopulationLearner.adam_state
    assert learn.DevicePopulationPGLearner._shared == ()
