"""CPU: the torch module of the device GNN policy (ddls_b200/torch_policy.py, include/ramp_b200.h: ramp_policy_set_weights_device /
ramp_policy_forward_device / ramp_policy_backward_device) -- the new C ABI symbols and the argument types the binding gives them,
the model dtype codes against the header, and the mapping between the module's flat weight vector and the reference's GNNPolicy
state_dict.  No compute call is made."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, 'include', 'ramp_b200.h')).read()
NAMES = ('ramp_policy_set_weights_device', 'ramp_policy_forward_device', 'ramp_policy_backward_device')


@pytest.fixture(scope='module')
def lib():
    from ddls_b200 import build, engine
    build.build()
    return engine.load_library()


def _prototype(name):
    m = re.search(r'int\s+' + name + r'\s*\(([^)]*)\)\s*;', HEADER)
    assert m, name
    return [re.sub(r'\s+', ' ', a.strip()) for a in m.group(1).split(',')]


def _ctype(arg):
    """the ctypes type a prototype argument is bound with"""
    t = arg.rsplit(' ', 1)[0]
    if '*' in t:
        return C.c_void_p
    return {'int32_t': C.c_int32, 'int64_t': C.c_int64}[t]


def test_new_symbols_are_declared_exported_and_bound_as_their_prototypes_state(lib):
    from ddls_b200 import engine, torch_policy
    for n in NAMES:
        assert n in engine.EXPORTED_SYMBOLS and hasattr(lib, n)
    assert _prototype('ramp_policy_set_weights_device') == ['ramp_policy_t* p', 'const float* weights', 'int64_t n', 'void* stream']
    rows = ['int32_t n', 'const void* model', 'int32_t model_dtype', 'const float* graph_features', 'int64_t graph_features_stride',
            'const uint8_t* action_mask']
    assert _prototype('ramp_policy_forward_device') == ['ramp_policy_t* p', 'void* stream'] + rows + ['float* logits_out', 'float* value_out']
    assert _prototype('ramp_policy_backward_device') == ['ramp_policy_t* p', 'void* stream'] + rows + \
        ['const float* grad_logits', 'const float* grad_value', 'float* grad_weights_out']
    torch_policy._bind(lib)
    for n in NAMES:
        assert getattr(lib, n).argtypes == [_ctype(a) for a in _prototype(n)], n
        assert getattr(lib, n).restype == C.c_int


def test_model_dtype_codes_match_the_header():
    from ddls_b200 import torch_env, torch_policy
    assert int(re.search(r'#define RAMP_MODEL_INT32 (\d+)', HEADER).group(1)) == torch_policy.MODEL_INT32
    assert int(re.search(r'#define RAMP_MODEL_INT64 (\d+)', HEADER).group(1)) == torch_policy.MODEL_INT64
    assert (torch_policy.MODEL_INT32, torch_policy.MODEL_INT64) == (torch_env.ACTIONS_INT32, torch_env.ACTIONS_INT64)


def _configs():
    from ddls_b200 import policy as P
    return {'gnn': (dict(P.DEFAULT_CONFIG), 17), 'algo-separate': (P.algo_model_config('ppo', 17), 17),
            'algo-shared': (P.algo_model_config('pg', 17), 17), 'algo-shared-9': (P.algo_model_config('impala', 9), 9)}


@pytest.mark.parametrize('cid', ['gnn', 'algo-separate', 'algo-shared', 'algo-shared-9'])
@pytest.mark.parametrize('as_torch', [False, True], ids=['numpy', 'torch'])
def test_gnn_state_dict_round_trips_through_the_flat_weight(cid, as_torch):
    import torch
    from ddls_b200 import policy as P
    from ddls_b200.torch_policy import flat_weights_of, gnn_state_dict_of
    c, A = _configs()[cid]
    sd = P.random_state_dict(c, A, seed=7)
    given = {k: torch.from_numpy(v) for k, v in sd.items()} if as_torch else sd
    flat = flat_weights_of(given, c, A)
    assert flat.dtype == torch.float32 and flat.shape == (int(sum(v.size for v in sd.values())),)
    np.testing.assert_array_equal(flat.numpy(), P.pack_weights(sd, c, A))
    back = gnn_state_dict_of(flat, c, A)
    assert list(back) == list(P.weight_keys(c))
    for k, v in back.items():
        assert isinstance(v, torch.Tensor) and v.dtype == torch.float32 and tuple(v.shape) == sd[k].shape, k
        np.testing.assert_array_equal(v.numpy(), sd[k], err_msg=k)
    # the state_dict of the flat weight loads back into the same blob, and into DeviceGNNPolicy's packing
    np.testing.assert_array_equal(P.pack_weights(back, c, A), flat.numpy())


def test_a_state_dict_of_the_other_read_out_is_refused_by_name():
    from ddls_b200 import policy as P
    from ddls_b200.torch_policy import flat_weights_of
    sep, shared = P.algo_model_config('ppo', 17), P.algo_model_config('pg', 17)
    with pytest.raises(KeyError, match='_value_branch_separate'):
        flat_weights_of(P.random_state_dict(sep, 17), shared, 17)
    with pytest.raises(KeyError, match='_value_branch_separate'):
        flat_weights_of(P.random_state_dict(shared, 17), sep, 17)
