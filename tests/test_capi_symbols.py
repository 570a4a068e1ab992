"""CPU: the C-ABI shared library builds (nvcc cross-compiles sm_90a without a GPU), loads, and exports every
function include/ramp_b200.h declares.  No compute call is made."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def lib():
    from ddls_b200 import build, engine
    build.build()
    return engine.load_library()


def declared_functions():
    src = open(os.path.join(ROOT, 'include', 'ramp_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(ramp_[a-z_0-9]+)\s*\(', src)))


def test_header_functions_exported(lib):
    names = declared_functions()
    assert len(names) >= 18
    for n in names:
        assert hasattr(lib, n), f'{n} declared in include/ramp_b200.h but not exported'


def test_binding_lists_every_symbol():
    from ddls_b200 import engine
    assert sorted(engine.EXPORTED_SYMBOLS) == declared_functions()


def test_struct_layouts_match_header(lib):
    """ctypes / numpy mirrors of the wire structs have the C sizes."""
    from ddls_b200 import engine
    assert engine.ACTION_DTYPE.itemsize == 48
    assert engine.ARRIVAL_DTYPE.itemsize == 24
    assert engine.JOB_RECORD_DTYPE.itemsize == 64
    assert engine.LOOKAHEAD_RESULT_DTYPE.itemsize == 32
    assert engine.STEP_STATS_LEN == 32 and engine.EP_LEN == 12


def test_sass_is_sm90a():
    import subprocess
    from ddls_b200 import build
    build.build()
    cuobjdump = os.path.join(os.path.dirname(build.nvcc_path()), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-lelf', build.LIB_PATH], capture_output=True, text=True).stdout
    assert 'sm_90a' in out and 'sm_100' not in out


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from ddls_b200 import engine
    monkeypatch.setattr(engine, '_lib', None)
    monkeypatch.setattr(engine, 'LIB_PATH', str(tmp_path / 'nope.so'))
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        engine.load_library()
