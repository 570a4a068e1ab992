"""Builds ddls_b200/libramp_b200.so (the C-ABI shared library) with nvcc for sm_90a, in-tree."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'libramp_b200.so')
SOURCES = [os.path.join(HERE, 'csrc', 'ramp_engine.cu'), os.path.join(HERE, 'csrc', 'ramp_expand.cpp'),
           os.path.join(HERE, 'csrc', 'ramp_quotient.cpp'), os.path.join(HERE, 'csrc', 'ramp_policy.cu')]
DEPS = SOURCES + [os.path.join(HERE, 'csrc', 'ramp_kernels.cuh'), os.path.join(HERE, 'csrc', 'ramp_lookahead_cta.cuh'),
                  os.path.join(HERE, 'csrc', 'ramp_lookahead_thread.cuh'), os.path.join(HERE, 'csrc', 'ramp_env.cuh'),
                  os.path.join(HERE, 'csrc', 'ramp_owned.cuh'), os.path.join(HERE, 'csrc', 'ramp_policy_learn.cuh'),
                  os.path.join(HERE, 'csrc', 'ramp_es.cuh'),
                  os.path.join(os.path.dirname(HERE), 'include', 'ramp_b200.h')]

NVCC_FLAGS = ['-O3', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo',
              '-fmad=false',            # no FMA contraction: f64 results must equal CPython's
              '-Xcompiler', '-fPIC', '-Xcompiler', '-ffp-contract=off', '-shared', '-cudart', 'static']


def nvcc_path():
    p = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    if not os.path.exists(p):
        raise RuntimeError('nvcc not found; cannot build ddls_b200/libramp_b200.so')
    return p


def is_stale(out=LIB_PATH):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False, extra_flags=(), out=LIB_PATH):
    """out: where the library goes; measurement variants (extra -D flags) are built elsewhere than LIB_PATH."""
    if not force and not is_stale(out):
        return out
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    cmd = [nvcc_path()] + NVCC_FLAGS + list(extra_flags) + ['-o', out] + SOURCES
    if verbose:
        print(' '.join(cmd))
    subprocess.check_call(cmd)
    return out


if __name__ == '__main__':
    import sys
    build(force=True, verbose=True, extra_flags=['-Xptxas', '-v'] if '-v' in sys.argv else [])
