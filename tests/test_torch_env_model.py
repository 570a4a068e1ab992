"""CPU: the torch-facing i/o of the device environment (ddls_b200/torch_env.py, include/ramp_b200.h: ramp_env_ingest / ramp_env_export)
-- the new C ABI symbols and the argument types the binding gives them, the export struct's layout against the header, and the
static per-job-type tensors against ``observation.static_observation``.  No compute call is made."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, 'include', 'ramp_b200.h')).read()


@pytest.fixture(scope='module')
def lib():
    from ddls_b200 import build, engine
    build.build()
    return engine.load_library()


def _prototype(name):
    m = re.search(r'int\s+' + name + r'\s*\(([^)]*)\)\s*;', HEADER)
    assert m, name
    return [re.sub(r'\s+', ' ', a.strip()) for a in m.group(1).split(',')]


def test_new_symbols_are_declared_exported_and_bound(lib):
    from ddls_b200 import engine, torch_env
    names = ('ramp_env_set_graph_static', 'ramp_env_ingest', 'ramp_env_export')
    for n in names:
        assert n in engine.EXPORTED_SYMBOLS and hasattr(lib, n)
    assert _prototype('ramp_env_set_graph_static') == ['ramp_engine_t* eng', 'const float* graph_static']
    assert _prototype('ramp_env_ingest') == ['ramp_engine_t* eng', 'const void* actions', 'int32_t dtype', 'void* stream']
    assert _prototype('ramp_env_export') == ['ramp_engine_t* eng', 'void* stream', 'const ramp_env_export_t* out']
    torch_env._bind(lib)
    assert lib.ramp_env_set_graph_static.argtypes == [C.c_void_p, C.c_void_p]
    assert lib.ramp_env_ingest.argtypes == [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    assert lib.ramp_env_export.argtypes == [C.c_void_p, C.c_void_p, C.POINTER(torch_env._Export)]
    assert all(getattr(lib, n).restype == C.c_int for n in names)


def test_action_dtypes_and_export_struct_match_the_header():
    from ddls_b200 import torch_env
    assert int(re.search(r'#define RAMP_ACTIONS_INT32 (\d+)', HEADER).group(1)) == torch_env.ACTIONS_INT32
    assert int(re.search(r'#define RAMP_ACTIONS_INT64 (\d+)', HEADER).group(1)) == torch_env.ACTIONS_INT64
    body = re.search(r'typedef struct \{([^{}]*)\} ramp_env_export_t;', HEADER).group(1)
    body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
    fields = re.findall(r'(\w+)\*\s+(\w+);', body)
    assert [f for _, f in fields] == [f for f, _ in torch_env._Export._fields_] == list(torch_env.OUTPUTS)
    assert [t for t, _ in fields] == ['int64_t', 'float', 'uint8_t', 'double', 'uint8_t']
    assert C.sizeof(torch_env._Export) == 5 * 8


def test_static_tensors_are_the_static_observation():
    import torch
    from ddls_b200 import synth
    from ddls_b200.observation import static_observation
    from ddls_b200.torch_env import static_tensors
    graphs = [synth.resnet_like_graph(), synth.chain_graph(6, 'chain6'), synth.transformer_like_graph(n_layers=1, name='tfm1', seed=4)]
    for g, st in zip(graphs, static_tensors(graphs)):
        ref = static_observation(g)
        assert set(st) == {'node_features', 'edge_features', 'edges_src', 'edges_dst', 'graph_static'}
        for k, t in st.items():
            assert t.device.type == 'cpu'
            want = ref[k].astype(np.int64) if k.startswith('edges_') else ref[k]
            assert t.dtype == (torch.int64 if k.startswith('edges_') else torch.float32), k
            np.testing.assert_array_equal(t.numpy(), want, err_msg=k)
        assert st['node_features'].shape[1] == 5 and st['edge_features'].shape[1] == 2 and st['graph_static'].shape == (6,)
        assert int(st['edges_src'].max()) < len(st['node_features']) and int(st['edges_dst'].max()) < len(st['node_features'])
