"""Where a bench step's time goes on the GPU: every kernel, the idle gaps between them and the bubble around each reset.

    python scripts/step_breakdown.py [--config cfg3-resnet50-64w] [--steps 64] [--warmup 16] [--out FILE.json]

Builds the workload exactly as `bench.py` does (`workload.generate` with the engine's JCTs, seed 0, reference run times, memo
mode 0, trace_cap 4096) and runs bench.py's device-resident step loop: a reset every L = 8 steps after reading the memo
counters, `step_device` with fused empty steps, and the episode-state export every L steps.

Two runs of that loop, after the warm-up:
  1. timed with CUDA events around the whole window, no profiler: ms per step as bench.py measures it;
  2. traced with torch.profiler (CUDA activities) in a run of its own: each GPU activity of the window, grouped into steps.

Per step it reports the mean duration of each activity (counter memset, plan, bucket, thread, step, and the reset's copies,
memsets and kernel), the idle gap before each of the step's launches, and the bubble between the last kernel of a step that is
followed by a reset and the first activity of the next step.  A negative gap is an overlap (programmatic dependent launch).
Tracing slows the host, so host-bound gaps in run 2 are upper bounds; run 1 is the number to compare against bench.py.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# kernel name fragment -> label, in step order
KERNELS = [('ramp_plan_kernel', 'plan'), ('ramp_bucket_kernel', 'bucket'), ('ramp_lookahead_thread_kernel', 'thread'),
           ('ramp_lookahead', 'lookahead_other'), ('ramp_step_kernel', 'step'), ('ramp_reset_kernel', 'reset_kernel'),
           ('ramp_export_episode_state_kernel', 'export')]


def card_info():
    import torch
    info = {'name': torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        lim, sm, mx = [x.strip() for x in out.split(',')]
        info.update(power_limit_w=float(lim), sm_clock_mhz=float(sm), sm_max_mhz=float(mx))
    except Exception:
        info.update(power_limit_w=None, sm_clock_mhz=None, sm_max_mhz=None)
    return info


def label_of(ev):
    cat, name = ev.get('cat', ''), ev.get('name', '')
    if cat == 'gpu_memset':
        return 'memset'
    if cat == 'gpu_memcpy':
        return 'memcpy_' + ('h2d' if 'HtoD' in name else 'd2h' if 'DtoH' in name else 'other')
    for frag, lab in KERNELS:
        if frag in name:
            return lab
    return 'other_kernel'


def setup(args):
    import torch
    from ddls_b200 import engine, workload
    cfg = workload.CONFIGS[args.config]
    B, L = cfg['n_episodes'], 8
    eng = engine.RampEngine(n_episodes=B, n_cluster_workers=int(np.prod(cfg['shape'])), max_jobs=L, device=0, memo_mode=0,
                            trace_cap=4096)
    tmap = {}

    def engine_jcts(templates):
        for i, t in enumerate(templates):
            tmap[i] = eng.register_template(t)
        res, _ = eng.run_lookaheads([tmap[i] for i in range(len(templates))])
        assert (res['status'] == 0).all()
        return res['jct']

    wl = workload.generate(args.config, engine_jcts, n_episodes=B, n_steps=L, seed=args.seed, run_times='reference')
    on_dev = []
    for p in range(L):
        a = wl.actions[p].copy()
        placed = a['template_id'] >= 0
        a['template_id'][placed] = np.array([tmap[int(t)] for t in a['template_id'][placed]], dtype=np.int32)
        on_dev.append(torch.from_numpy(a.view(np.uint8).reshape(B, -1).copy()).cuda())
    stats = torch.empty((B, engine.STEP_STATS_LEN), dtype=torch.float64, device='cuda')
    ncs = torch.empty(B, dtype=torch.int32, device='cuda')
    ep = torch.empty((B, engine.EP_LEN), dtype=torch.float64, device='cuda')

    def device_step(s):                   # bench.py's device_step with one gather buffer and world = 1
        p = s % L
        if p == 0:
            if s > 0:
                eng.memo_stats()
            eng.reset(wl.arrivals)
        eng.step_device(on_dev[p].data_ptr(), True, stats.data_ptr(), ncs.data_ptr())
        if (s + 1) % L == 0:
            eng.export_episode_state_to(ep.data_ptr())

    return eng, device_step, B


def breakdown(events, n_steps):
    """events: the GPU activities of the window in start order -> per-step means."""
    evs = [dict(lab=label_of(e), ts=float(e['ts']), end=float(e['ts']) + float(e['dur']), dur=float(e['dur'])) for e in events]
    plans = [i for i, e in enumerate(evs) if e['lab'] == 'plan']
    # a step = the counter memset right before its plan kernel through its step kernel; everything between two steps is the
    # gap (or, when it holds a reset, the reset bubble)
    steps = []
    for k, i in enumerate(plans):
        first = i - 1 if i > 0 and evs[i - 1]['lab'] == 'memset' else i
        j = i
        while j < len(evs) and evs[j]['lab'] != 'step':
            j += 1
        if j == len(evs):
            break
        steps.append((first, j))
    dur, gap_before = {}, {}
    resets, between = [], []
    for k, (first, last) in enumerate(steps):
        prev_end = None
        for i in range(first, last + 1):
            e = evs[i]
            dur.setdefault(e['lab'], []).append(e['dur'])
            if prev_end is not None:
                gap_before.setdefault(e['lab'], []).append(e['ts'] - prev_end)
            prev_end = max(prev_end, e['end']) if prev_end is not None else e['end']
        if k + 1 < len(steps):
            nxt = steps[k + 1][0]
            mid = evs[last + 1:nxt]
            span = evs[nxt]['ts'] - evs[last]['end']
            if any(e['lab'] == 'reset_kernel' for e in mid):
                busy = sum(e['dur'] for e in mid)
                resets.append(dict(bubble_us=span, busy_us=busy, activities=[(e['lab'], round(e['dur'], 2)) for e in mid]))
            else:
                between.append(span)
    n = len(steps)
    mean = lambda v: float(np.mean(v)) if v else 0.0
    window_us = evs[steps[-1][1]]['end'] - evs[steps[0][0]]['ts'] if steps else 0.0
    out = {'steps_traced': n,
           'us_per_step_traced': window_us / max(n - 1, 1) if n > 1 else window_us,
           'kernel_us_mean': {k: mean(v) for k, v in dur.items()},
           'kernel_us_per_step': {k: float(np.sum(v)) / n for k, v in dur.items()},
           'gap_before_us_mean': {k: mean(v) for k, v in gap_before.items()},
           'gap_between_steps_us_mean': mean(between),
           'reset_bubble_us_mean': mean([r['bubble_us'] for r in resets]),
           'reset_busy_us_mean': mean([r['busy_us'] for r in resets]),
           'n_resets': len(resets),
           'reset_example': resets[0]['activities'] if resets else []}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default='cfg3-resnet50-64w')
    ap.add_argument('--steps', type=int, default=64, help='steps per window (a multiple of 8 keeps the resets aligned)')
    ap.add_argument('--warmup', type=int, default=16)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None, help='also write the result as JSON here')
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise RuntimeError('step_breakdown.py needs a CUDA device')
    torch.cuda.set_device(0)
    eng, device_step, B = setup(args)
    ext = torch.cuda.ExternalStream(eng.stream, device=torch.device('cuda', 0))
    W, K = args.warmup, args.steps
    for s in range(W):
        device_step(s)
    eng.sync()
    eng.lookahead_kernel_time(reset=True)

    # run 1: timed, no profiler
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(ext)
    for s in range(W, W + K):
        device_step(s)
    e1.record(ext)
    eng.sync()
    torch.cuda.synchronize()
    ms_per_step = e0.elapsed_time(e1) / K
    card = card_info()
    # the kernel-time figure bench.py reports, over run 1
    kt = eng.lookahead_kernel_time(reset=True)

    # run 2: traced
    for s in range(W):
        device_step(s)
    eng.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(W, W + K):
            device_step(s)
        eng.sync()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'trace.json')
        prof.export_chrome_trace(path)
        trace = json.load(open(path))
    gpu = [e for e in trace.get('traceEvents', []) if e.get('ph') == 'X' and e.get('cat') in ('kernel', 'gpu_memset', 'gpu_memcpy')]
    gpu.sort(key=lambda e: float(e['ts']))
    bd = breakdown(gpu, K)
    res = dict(config=args.config, episodes=B, steps=K, warmup=W, card=card, ms_per_step_timed=ms_per_step,
               lookahead_kernel_ms_per_launch=kt['total_ms'] / max(kt['launches'], 1), traced=bd)
    print(f"{card['name']}, power limit {card['power_limit_w']} W, SM clock {card['sm_clock_mhz']} MHz (max {card['sm_max_mhz']})")
    print(f"{args.config}: {B} episodes, {K} steps after {W} warm-up")
    print(f"timed (CUDA events, no profiler): {ms_per_step * 1e3:.1f} us/step; lookahead window (bucket + thread) "
          f"{res['lookahead_kernel_ms_per_launch'] * 1e3:.1f} us per step")
    print(f"traced: {bd['us_per_step_traced']:.1f} us/step over {bd['steps_traced']} steps")
    print('  activity          mean us   us/step   gap before (mean us)')
    for k in sorted(bd['kernel_us_per_step'], key=lambda k: -bd['kernel_us_per_step'][k]):
        print(f"  {k:16s} {bd['kernel_us_mean'][k]:8.1f}  {bd['kernel_us_per_step'][k]:8.1f}   {bd['gap_before_us_mean'].get(k, 0.0):8.1f}")
    print(f"  gap between steps without a reset: {bd['gap_between_steps_us_mean']:.1f} us")
    print(f"  reset bubble (step kernel end -> next step's first activity): {bd['reset_bubble_us_mean']:.1f} us over "
          f"{bd['n_resets']} resets, of which GPU busy {bd['reset_busy_us_mean']:.1f} us; "
          f"= {bd['reset_bubble_us_mean'] / 8:.1f} us per step at one reset every 8 steps")
    print(f"  one reset's activities: {bd['reset_example']}")
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)
    eng.close()


if __name__ == '__main__':
    main()
