"""CPU: every device buffer, pinned host buffer, stream and event of the engine and the policy is allocated and released through
the owner types of ddls_b200/csrc/ramp_owned.cuh, and both translation units share one error reporter and one guard on the
kernels' dynamic shared memory limit."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'ddls_b200', 'csrc')
OWNER_HEADER = 'ramp_owned.cuh'
RAW_CALLS = ('cudaMalloc(', 'cudaMallocHost(', 'cudaFree(', 'cudaFreeHost(', 'cudaStreamCreate', 'cudaStreamDestroy',
             'cudaEventCreate', 'cudaEventDestroy')
# memory the C ABI hands to the caller, who owns it
CALLER_OWNED = ('ramp_pinned_alloc', 'ramp_pinned_free')


def strip_comments(src):
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return re.sub(r'//[^\n]*', '', src)


def without_functions(src, names):
    """src without the definitions of the top-level functions `names` (their braces balanced)"""
    for name in names:
        m = re.search(r'^[^\n;{}]*\b' + name + r'\s*\([^)]*\)\s*\{', src, flags=re.M)
        assert m, f'{name} is not defined'
        depth, i = 0, m.end() - 1
        while True:
            depth += {'{': 1, '}': -1}.get(src[i], 0)
            i += 1
            if depth == 0:
                break
        src = src[:m.start()] + src[i:]
    return src


def sources():
    out = {}
    for path in sorted(glob.glob(os.path.join(CSRC, '*'))):
        if path.endswith(('.cu', '.cuh', '.cpp', '.h')):
            out[os.path.basename(path)] = strip_comments(open(path).read())
    assert 'ramp_engine.cu' in out and 'ramp_policy.cu' in out and OWNER_HEADER in out
    return out


def test_no_raw_allocations_outside_the_owner_header():
    for name, src in sources().items():
        if name == OWNER_HEADER:
            continue
        if name == 'ramp_policy.cu':
            src = without_functions(src, CALLER_OWNED)
        for call in RAW_CALLS:
            assert call not in src, f'{name} calls {call} outside the owner types'


def test_one_error_reporter():
    for name, src in sources().items():
        assert not re.search(r'\bperr\b|\bPCUDA\b', src), f'{name} still has its own error reporter'
        if name != OWNER_HEADER:
            assert not re.search(r'#define\s+CUDA_TRY\b', src), f'{name} defines CUDA_TRY again'
            assert not re.search(r'\bint\s+set_error\s*\(', src), f'{name} defines set_error again'


def test_dynamic_shared_memory_limit_is_set_only_by_reserve_dynamic_smem():
    """The limit belongs to the kernel in the process, so every engine and policy raises it through the one guard that never
    lowers it."""
    calls = []
    for name, src in sources().items():
        for m in re.finditer(r'cudaFuncSetAttribute\s*\(([^;]*)\)\s*;', src):
            if 'cudaFuncAttributeMaxDynamicSharedMemorySize' in m.group(1):
                calls.append((name, m.start()))
    assert len(calls) == 1, calls
    name, at = calls[0]
    src = sources()[name]
    guard = re.search(r'cudaError_t\s+(ramp::)?reserve_dynamic_smem\s*\([^)]*\)\s*\{', src)
    assert name == 'ramp_engine.cu' and guard and guard.end() < at
    assert src.rfind('\n}', guard.end(), at) == -1, 'the call is not inside reserve_dynamic_smem'
    assert 'reserve_dynamic_smem((const void*)ramp_policy_head_kernel' in sources()['ramp_policy.cu']
