"""Where a tick of the thread-per-lookahead kernel spends its cycles (run on the GPU box).

    python scripts/tick_cycles.py [--n 4096] [--run-times reference] [--out-lib build_variants/tick_clocks/libramp_b200.so]

Builds the library with -DRAMP_TICK_CLOCKS into --out-lib (never over ddls_b200/libramp_b200.so) and runs the bench's four
quotient templates (ResNet-50-like job at degrees 2 / 4 / 8 / 16, 4x4x4 RAMP, like scripts/microbench_thread.py): first all
four mixed, n lookaheads, then each degree alone, n / 4 lookaheads.  For each run it prints lane 0's cycles per tick by
phase and by frontier shape (ready op classes O, ready flow entries F, non-flow tick nf) with each shape's share of the
ticks.  Beside it: microseconds per tick of the instrumented build and of the normal build (the clock() reads cost a
little), and the static side from the normal build's SASS -- instructions of the kernel, of thread_lookahead<false>
(the hinted instantiation, which every lookahead after a template's first runs), of its tick loop and of its small-frontier
half.
"""
import argparse
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ['A/B', 'D/E+ring', 'H', 'G', 'compact+exit']
NPH = len(PHASES)
NSHAPES = 64
KERNEL = '_ZN4ramp28ramp_lookahead_thread_kernelENS_10ThreadArgsE'
CUH = os.path.join(ROOT, 'ddls_b200', 'csrc', 'ramp_lookahead_thread.cuh')


def shape_name(s):
    o, f, nf = s // 16, (s // 2) % 8, s % 2
    return f"O={'>2' if o == 3 else o} F={'>6' if f == 7 else f}{' nf' if nf else ''}"


def templates(eng, run_times):
    from ddls_b200 import synth
    from ddls_b200.template_builder import build_template, RampShape
    g = synth.resnet_like_graph()
    return [eng.register_template(build_template(g, d, RampShape(4, 4, 4), run_times=run_times)) for d in (2, 4, 8, 16)]


def us_per_tick(eng, ids):
    best = 1e9
    for _ in range(3):
        res, ms = eng.run_lookaheads(ids)
        best = min(best, ms)
    assert (res['status'] == 0).all()
    T = int(res['n_ticks'].max())
    return best, T, best * 1e3 / T


def measure(lib, n, run_times, ledger):
    """One process per library: prints one JSON line per run."""
    import numpy as np
    from ddls_b200 import engine
    engine.LIB_PATH = lib
    eng = engine.RampEngine(n_episodes=n, n_cluster_workers=64, max_jobs=1, trace_cap=4096)
    tids = templates(eng, run_times)
    eng.run_lookaheads(np.array(tids, dtype=np.int32))          # records every template's hints: later runs take the fast path
    L = engine.load_library()
    table = np.zeros(NSHAPES * (NPH + 1), dtype=np.uint64)
    if ledger:
        L.ramp_debug_tick_clocks.argtypes = [C.c_void_p, C.c_int]
        L.ramp_debug_tick_clocks(table.ctypes.data, 1)
    runs = [('mixed', [tids[k % 4] for k in range(n)])] + [(f'degree {d}', [t] * (n // 4)) for d, t in zip((2, 4, 8, 16), tids)]
    for name, ids in runs:
        ms, T, us = us_per_tick(eng, np.array(ids, dtype=np.int32))
        out = dict(run=name, n=len(ids), ms=round(ms, 4), T=T, us_per_tick=round(us, 4))
        if ledger:
            _check = L.ramp_debug_tick_clocks(table.ctypes.data, 1)      # three launches of the run, summed
            assert _check == 0, engine.load_library().ramp_last_error()
            out['table'] = table.reshape(NSHAPES, NPH + 1).tolist()
        print(json.dumps(out), flush=True)
    eng.close()


def sub(lib, args, ledger):
    cmd = [sys.executable, os.path.abspath(__file__), '--measure', lib, '--n', str(args.n), '--run-times', args.run_times]
    if ledger:
        cmd.append('--ledger')
    out = subprocess.run(cmd, check=True, capture_output=True, text=True, cwd=ROOT).stdout
    return [json.loads(l) for l in out.splitlines() if l.startswith('{')]


def report(run, normal):
    import numpy as np
    t = np.array(run['table'], dtype=np.float64)
    ticks = t[:, NPH]
    tot = ticks.sum()
    print(f"\n== {run['run']}: {run['n']} lookaheads, T = {run['T']} ticks (longest), {int(tot)} ticks on lane 0 of the CTAs ==")
    print(f"   us per tick: {run['us_per_tick']:.4f} instrumented, {normal['us_per_tick']:.4f} normal build "
          f"(kernel {run['ms']:.4f} / {normal['ms']:.4f} ms)")
    hdr = f"   {'shape':<14}{'share':>7}" + ''.join(f'{p:>14}' for p in PHASES) + f"{'cycles/tick':>13}"
    print(hdr)
    for s in np.argsort(-ticks):
        if ticks[s] == 0:
            break
        c = t[s, :NPH] / ticks[s]
        print(f"   {shape_name(s):<14}{ticks[s] / tot:>7.1%}" + ''.join(f'{v:>14.0f}' for v in c) + f'{c.sum():>13.0f}')
    c = t[:, :NPH].sum(0) / tot
    print(f"   {'all':<14}{1:>7.1%}" + ''.join(f'{v:>14.0f}' for v in c) + f'{c.sum():>13.0f}')
    print(f"   share of a tick:     " + ''.join(f'{v / c.sum():>14.1%}' for v in c))


def cuda_tool(name):
    nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    p = os.path.join(os.path.dirname(os.path.realpath(nvcc)), name)
    return p if os.path.exists(p) else (shutil.which(name) or name)


def static_side(lib, tmp):
    """Instruction counts from the normal build's SASS, attributed by the line info (-lineinfo) nvdisasm -gi prints."""
    src = open(CUH).read().splitlines()
    def line_of(pat):
        return next(i + 1 for i, l in enumerate(src) if pat in l)
    call = line_of('if (fast) thread_lookahead<false>(x);')
    loop0, loop1 = line_of('for (;;) {       // left through ONE'), line_of('feed.finish(R);')
    fast0, fast1 = line_of('if (nF <= RAMP_T_FASTF && nO <= 2) {'), line_of('// ---- A, B: winners per worker group')
    subprocess.run([cuda_tool('cuobjdump'), '-xelf', 'all', os.path.abspath(lib)], check=True, cwd=tmp, capture_output=True)
    cubin = next(os.path.join(tmp, f) for f in sorted(os.listdir(tmp)) if f.startswith('ramp_engine.') and f.endswith('.cubin'))
    dis = subprocess.run([cuda_tool('nvdisasm'), '-gi', cubin], check=True, capture_output=True, text=True).stdout
    body = re.split(r'\n\t\.section\s', dis.split(f'\n{KERNEL}:\n', 1)[1], maxsplit=1)[0]
    ann = re.compile(r'//## File "([^"]+)", line (\d+)(?: inlined at "([^"]+)", line (\d+))?')
    ins = re.compile(r'^\s+/\*[0-9a-f]{4,}\*/\s+\S')
    bra = re.compile(r'^\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?(BRA|BSSY)\b')
    n_all = n_inst = n_loop = n_fast = 0
    n_bra = {'BRA': 0, 'BSSY': 0}
    # nvdisasm prints an instruction's inline chain (innermost frame first, the kernel's own line last) when it changes
    cur, fresh = [], True
    for l in body.splitlines():
        m = ann.search(l)
        if m:
            if fresh:
                cur, fresh = [], False
            cur.append((int(m.group(2)), m.group(4) and int(m.group(4))))
            continue
        if not ins.match(l):
            continue
        n_all += 1
        fresh = True
        # the kernel's frame is the call line; the frame inlined at it is a line of thread_lookahead
        if len(cur) >= 2 and cur[-1][0] == call and cur[-2][1] == call:
            n_inst += 1
            inner = cur[-2][0]
            if loop0 <= inner < loop1:
                n_loop += 1
                b = bra.match(l)
                if b:
                    n_bra[b.group(1)] += 1
            if fast0 <= inner < fast1:
                n_fast += 1
    return dict(kernel=n_all, instantiation=n_inst, tick_loop=n_loop, small_frontier_path=n_fast,
                tick_loop_bra=n_bra['BRA'], tick_loop_bssy=n_bra['BSSY'])


def gpu_line():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as ex:  # noqa: BLE001
        return f'nvidia-smi unavailable ({ex})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=4096)
    ap.add_argument('--run-times', default='reference', choices=['reference', 'one_to_one'])
    ap.add_argument('--out-lib', default=os.path.join(ROOT, 'build_variants', 'tick_clocks', 'libramp_b200.so'))
    ap.add_argument('--static-only', action='store_true', help='print the SASS counts of the normal build and stop (no GPU)')
    ap.add_argument('--measure', default=None, help=argparse.SUPPRESS)
    ap.add_argument('--ledger', action='store_true', help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.measure:
        return measure(args.measure, args.n, args.run_times, args.ledger)
    from ddls_b200 import build
    normal_lib = build.LIB_PATH
    assert os.path.exists(normal_lib), 'build the library first (python -m ddls_b200.build)'
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        st = static_side(normal_lib, tmp)
    print(f'thread_lookahead<false> in the normal build: {st["instantiation"]} instructions ({st["instantiation"] * 16} B), '
          f'tick loop {st["tick_loop"]} ({st["tick_loop_bra"]} BRA, {st["tick_loop_bssy"]} BSSY), small-frontier half '
          f'{st["small_frontier_path"]}; whole kernel {st["kernel"]} ({st["kernel"] * 16} B)')
    if args.static_only:
        return
    variant = build.build(extra_flags=['-DRAMP_TICK_CLOCKS'], out=args.out_lib)
    print(f'GPU: {gpu_line()}')
    normal = sub(normal_lib, args, False)
    inst = sub(variant, args, True)
    for r, n in zip(inst, normal):
        report(r, n)
    print(f'\nGPU: {gpu_line()}')


if __name__ == '__main__':
    main()
