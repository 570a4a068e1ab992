"""CPU: the CUDA-graph capture surface without a device.  The two new C entry points are declared, exported and refuse null
handles; the torch environment and the torch policy refuse, by name and before any library call, the captures they can decide on
the host: a step whose placements the device tables do not all decide, reset() and refresh() inside a capture, a forward whose
weights would be uploaded inside the graph, and a backward.  Capture is faked by patching torch.cuda.is_current_stream_capturing."""
import ctypes as C

import pytest
import torch

from ddls_b200 import engine
from ddls_b200.torch_env import TorchRampJobPartitioningEnvironment
from ddls_b200.torch_policy import TorchGNNPolicy


RAMP_ERR_BAD_ARG = -2                      # include/ramp_b200.h


class _Recorder:
    """a library stand-in: every ramp_* call is recorded and succeeds"""
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            self.calls.append(name)
            return engine.RAMP_OK
        return call


@pytest.fixture
def capturing(monkeypatch):
    monkeypatch.setattr(torch.cuda, 'is_current_stream_capturing', lambda: True)


@pytest.fixture(scope='module')
def lib():
    from ddls_b200 import build
    build.build()
    return engine.load_library()


def test_the_new_entry_points_are_exported_and_refuse_null_handles(lib):
    assert {'ramp_env_join', 'ramp_policy_refresh_device'} <= set(engine.EXPORTED_SYMBOLS)
    lib.ramp_env_join.restype = C.c_int
    lib.ramp_env_join.argtypes = [C.c_void_p, C.c_void_p]
    assert lib.ramp_env_join(None, None) == RAMP_ERR_BAD_ARG
    assert lib.ramp_last_error().decode() == 'no environment'
    lib.ramp_policy_refresh_device.restype = C.c_int
    lib.ramp_policy_refresh_device.argtypes = [C.c_void_p, C.c_void_p]
    assert lib.ramp_policy_refresh_device(None, None) == RAMP_ERR_BAD_ARG
    assert lib.ramp_last_error().decode() == 'null argument'


class _FakeDeviceEnv:
    def __init__(self, decides_everything):
        self._device_decides_everything = decides_everything
        self.stepped = 0

    def step_device(self):
        self.stepped += 1

    def reset(self):
        raise AssertionError('reset() reached the device environment')


def _env(decides_everything):
    env = TorchRampJobPartitioningEnvironment.__new__(TorchRampJobPartitioningEnvironment)
    env.env, env.device, env.B, env.n_actions = _FakeDeviceEnv(decides_everything), torch.device('cpu'), 4, 17
    env._L, env._h = _Recorder(), None
    return env


def test_a_step_the_device_tables_cannot_decide_is_refused_before_any_call(capturing):
    env = _env(decides_everything=False)
    with pytest.raises(RuntimeError, match='the device tables do not decide every placement'):
        env.step(torch.zeros(4, dtype=torch.int64))
    assert env._L.calls == [] and env.env.stepped == 0


def test_reset_inside_a_capture_is_refused_and_check_does_nothing(capturing):
    env = _env(decides_everything=True)
    with pytest.raises(RuntimeError, match=r'reset\(\) draws the arrival streams on the host'):
        env.reset()
    env.check()
    assert env._L.calls == []


def test_outside_a_capture_check_orders_the_engine_behind_the_callers_stream_first(monkeypatch):
    monkeypatch.setattr(torch.cuda, 'is_current_stream_capturing', lambda: False)
    monkeypatch.setattr(torch.cuda, 'current_stream', lambda device=None: type('S', (), {'cuda_stream': 0})())
    env = _env(decides_everything=True)
    env.check()
    assert env._L.calls == ['ramp_env_join', 'ramp_env_read']


def _module():
    mod = TorchGNNPolicy.__new__(TorchGNNPolicy)
    torch.nn.Module.__init__(mod)
    mod.device, mod.n_actions, mod._L, mod._h, mod._key = torch.device('cpu'), 17, _Recorder(), 1, None
    mod.weight = torch.nn.Parameter(torch.zeros(8))
    return mod


def test_a_forward_that_would_upload_weights_inside_the_graph_is_refused(capturing):
    mod = _module()
    with pytest.raises(RuntimeError, match='the weights changed since they were last uploaded'):
        mod._upload(mod.weight, 0)
    mod._key = (mod.weight.data_ptr(), mod.weight._version)
    mod._upload(mod.weight, 0)                                       # the weights the library holds: nothing to do
    with torch.no_grad():
        mod.weight.add_(1.0)
    with pytest.raises(RuntimeError, match='the weights changed since they were last uploaded'):
        mod._upload(mod.weight, 0)
    assert mod._L.calls == []


def test_backward_and_refresh_inside_a_capture_are_refused(capturing):
    mod = _module()
    with pytest.raises(RuntimeError, match='the backward of TorchGNNPolicy is not capturable'):
        mod._backward_rows(mod.weight, torch.zeros(2, dtype=torch.int64), torch.zeros(2, 34), torch.ones(2, 17, dtype=torch.bool),
                           None, None)
    with pytest.raises(RuntimeError, match=r'refresh\(\) runs eagerly'):
        mod.refresh()
    assert mod._L.calls == []
