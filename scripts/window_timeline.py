"""When each lookahead window of an overlapped step runs, against the segment it belongs to.

    python scripts/window_timeline.py [--config cfg3-resnet50-64w] [--steps 64] [--warmup 16] [--out FILE.json]

Runs bench.py's device-resident step loop as scripts/step_breakdown.py does (same workload, a reset every L = 8 steps): an
untraced timed run first, then the same window traced with torch.profiler (CUDA activities) in a run of its own.

Overlapped steps (DESIGN.md §4) run each step's thread kernel on the stream of its lookahead window and the commit, the repair
bucket and thread kernel and the step kernel on the engine stream, so activities in start order do not describe a step.  Here a
step's activities are matched by launch order instead (the profiler's correlation id): the k-th window thread kernel launched
and the k-th step kernel belong to the same step.  Per step, all times in µs relative to the start of its segment's reset
kernel:
  window     its window's thread kernel: start, end, and the stream (window) it ran on;
  chain      commit, repair bucket, repair thread kernel and step kernel on the engine stream: start and end of each;
  waits      start of the window kernel minus the end of the step kernel that consumed the same window last
             (`after_consumed`: about 0 means the window queued behind that step), and minus the end of the previous
             step's window kernel (`after_prev_window`: >= 0 means this window ran after the previous one, not beside it).
Per segment: the reset bubble, from the end of the segment's last step kernel to the start of the next segment's first window
kernel, and the span from the reset to the segment's last step kernel end.
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from step_breakdown import card_info, setup  # noqa: E402

L = 8


def kernel_label(name):
    for frag, lab in (('ramp_spec_plan_kernel', 'spec_plan'), ('ramp_commit_kernel', 'commit'), ('ramp_bucket_kernel', 'bucket'),
                      ('ramp_lookahead_thread_kernel', 'thread'), ('ramp_step_kernel', 'step'), ('ramp_reset_kernel', 'reset')):
        if frag in name:
            return lab
    return None


def timeline(trace, n_steps):
    evs = []
    for e in trace.get('traceEvents', []):
        if e.get('ph') != 'X' or e.get('cat') != 'kernel':
            continue
        lab = kernel_label(e.get('name', ''))
        if lab is None:
            continue
        a = e.get('args', {})
        evs.append(dict(lab=lab, ts=float(e['ts']), end=float(e['ts']) + float(e['dur']), stream=int(a.get('stream', e.get('tid', -1))),
                        corr=int(a.get('correlation', 0))))
    evs.sort(key=lambda e: e['corr'])
    steps_k = [e for e in evs if e['lab'] == 'step']
    engine = steps_k[0]['stream']
    windows = [e for e in evs if e['lab'] == 'thread' and e['stream'] != engine]
    resets = [e for e in evs if e['lab'] == 'reset']
    n = min(len(steps_k), len(windows), n_steps)
    n_windows = len({w['stream'] for w in windows})
    # the engine-stream chain of step i: what was launched on the engine stream after step i - 1's step kernel
    eng = [e for e in evs if e['stream'] == engine]
    out, pos = [], 0
    for i in range(n):
        chain = {}
        while pos < len(eng) and eng[pos]['corr'] <= steps_k[i]['corr']:
            e = eng[pos]
            pos += 1
            if e['lab'] in ('commit', 'bucket', 'thread', 'step'):
                chain[{'bucket': 'repair_bucket', 'thread': 'repair_thread'}.get(e['lab'], e['lab'])] = e
        seg = i // L
        base = resets[seg]['ts'] if seg < len(resets) else steps_k[seg * L]['ts']
        w = windows[i]
        rec = dict(step=i, segment=seg, window_stream=w['stream'],
                   window=[round(w['ts'] - base, 1), round(w['end'] - base, 1)],
                   chain={k: [round(v['ts'] - base, 1), round(v['end'] - base, 1)] for k, v in chain.items()})
        if i >= n_windows:
            rec['after_consumed'] = round(w['ts'] - steps_k[i - n_windows]['end'], 1)
        if i >= 1:
            rec['after_prev_window'] = round(w['ts'] - windows[i - 1]['end'], 1)
        out.append(rec)
    segs = []
    for s in range(n // L):
        last = steps_k[s * L + L - 1]
        base = resets[s]['ts'] if s < len(resets) else steps_k[s * L]['ts']
        d = dict(segment=s, span_us=round(last['end'] - base, 1))
        if (s + 1) * L < n:
            d['reset_bubble_us'] = round(windows[(s + 1) * L]['ts'] - last['end'], 1)
        segs.append(d)
    return dict(n_windows=n_windows, steps=out, segments=segs)


def summary(tl):
    """Per position in the segment: mean window start / end / length, the mean waits, and the mean segment span."""
    pos = {}
    for r in tl['steps']:
        p = pos.setdefault(r['step'] % L, dict(start=[], end=[], len=[], after_consumed=[], after_prev_window=[], step_end=[]))
        p['start'].append(r['window'][0]); p['end'].append(r['window'][1]); p['len'].append(r['window'][1] - r['window'][0])
        if 'step' in r['chain']:
            p['step_end'].append(r['chain']['step'][1])
        for k in ('after_consumed', 'after_prev_window'):
            if k in r:
                p[k].append(r[k])
    mean = lambda v: round(float(np.mean(v)), 1) if v else None
    return dict(by_position={k: {f: mean(v) for f, v in p.items()} for k, p in sorted(pos.items())},
                span_us=mean([s['span_us'] for s in tl['segments']]),
                reset_bubble_us=mean([s['reset_bubble_us'] for s in tl['segments'] if 'reset_bubble_us' in s]))


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
        raise RuntimeError('window_timeline.py needs a CUDA device')
    torch.cuda.set_device(0)
    eng, device_step, B = setup(args)
    ext = torch.cuda.ExternalStream(eng.stream, device=torch.device('cuda', 0))
    W, K = args.warmup, args.steps
    for s in range(W):
        device_step(s)
    eng.sync()

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
    tl = timeline(trace, K)
    sm = summary(tl)
    res = dict(config=args.config, episodes=B, steps=K, warmup=W, card=card, ms_per_step_timed=ms_per_step, summary=sm, timeline=tl)
    print(f"{card['name']}, power limit {card['power_limit_w']} W, SM clock {card['sm_clock_mhz']} MHz (max {card['sm_max_mhz']})")
    print(f"{args.config}: {B} episodes, {K} steps after {W} warm-up, {tl['n_windows']} lookahead windows")
    print(f"timed (CUDA events, no profiler): {ms_per_step * 1e3:.1f} us/step")
    print(f"traced: reset -> last step kernel end {sm['span_us']} us per segment; reset bubble {sm['reset_bubble_us']} us")
    print('  pos  window start    end    len   after consumed  after prev window   step kernel end   (us from the reset, means)')
    for p, v in sm['by_position'].items():
        print(f"  {p:3d}  {v['start']!s:>10} {v['end']!s:>8} {v['len']!s:>6} {v['after_consumed']!s:>16} {v['after_prev_window']!s:>18} "
              f"{v['step_end']!s:>17}")
    print('  first two segments, step by step (window [start, end] on stream; engine chain):')
    for r in tl['steps'][:2 * L]:
        print(f"    step {r['step']:2d} window {r['window']} s{r['window_stream']} after_consumed={r.get('after_consumed')} "
              f"after_prev={r.get('after_prev_window')} chain={r['chain']}")
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)
    eng.close()


if __name__ == '__main__':
    main()
