"""Env-steps/s of masked-random rollouts of DeviceRampJobPartitioningEnvironment with place_on_device off and on, alternated in one
process, on workloads whose jobs split their ops unevenly; the place kernel's own time (torch.profiler, a separate pass) and the
host placer calls per step.  One JSON line per run and per workload summary to stdout and to --out.

    python scripts/device_placer_rollouts.py --runs 3 --out profiles/h100_device_placer_rollouts.jsonl
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def workload(kind):
    from ddls_b200 import synth
    if kind == 'host_placer':
        graphs = [synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3), synth.chain_graph(6, 'chain6'),
                  synth.transformer_like_graph(n_layers=1, name='tfm1', seed=4)]
        return (4, 4, 4), graphs, dict(n_episodes=768, jobs_per_episode=7, seed=11, interarrival=('exponential', 600.0))
    if kind == 'bert16':
        return (8, 8, 4), [synth.transformer_like_graph(n_layers=12, name='bert_base_like', seed=2)], \
            dict(n_episodes=4096, jobs_per_episode=6, seed=4, interarrival=('exponential', 800.0), max_partitions_per_op=16)
    raise KeyError(kind)


def rollout(env, seed):
    rng = np.random.default_rng(seed)
    obs = env.reset()
    steps = 0
    while not obs['done'].all():
        m = obs['action_mask'].astype(bool)
        obs, _, _, _ = env.step((rng.random(m.shape) * m).argmax(axis=1))
        steps += 1
    return steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--rollouts', type=int, default=4, help='reset-and-rollouts per timed run')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    lines = []

    def emit(rec):
        rec['gpu'] = gpu
        print(json.dumps(rec), flush=True)
        lines.append(json.dumps(rec))
    for kind in ('host_placer', 'bert16'):
        shape, graphs, kw = workload(kind)
        envs = {False: DeviceRampJobPartitioningEnvironment(shape, graphs, **kw),
                True: DeviceRampJobPartitioningEnvironment(shape, graphs, place_on_device=True, **kw)}
        for on, env in envs.items():                      # warm-up: every template these rollouts reach is registered
            for r in range(args.rollouts):
                rollout(env, 100 + r)
        rates = {False: [], True: []}
        for run in range(args.runs):
            for on in (False, True):
                env = envs[on]
                calls0 = env.stats['placer_calls']
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                steps = sum(rollout(env, 100 + r) for r in range(args.rollouts))
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                rate = steps * env.B / dt
                rates[on].append(rate)
                emit({'workload': kind, 'place_on_device': on, 'run': run, 'env_steps_per_s': rate, 'steps': steps, 'seconds': dt,
                      'host_placer_calls_per_step': (env.stats['placer_calls'] - calls0) / steps})
        # the place kernel's own time, in a pass of its own
        env = envs[True]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            steps = rollout(env, 100)
            torch.cuda.synchronize()
        k = [e for e in prof.key_averages() if 'ramp_env_place_kernel' in e.key]
        d = [e for e in prof.key_averages() if 'ramp_env_decide_kernel' in e.key]
        emit({'workload': kind, 'summary': True, 'episodes': envs[True].B,
              'env_steps_per_s_off': rates[False], 'env_steps_per_s_on': rates[True],
              'median_ratio_on_over_off': float(np.median(rates[True]) / np.median(rates[False])),
              'place_kernel_us_per_step': (k[0].device_time_total / steps) if k else None,
              'decide_kernel_us_per_step': (d[0].device_time_total / steps) if d else None,
              'geometry_entries': len(env._geom_mask_set)})
        for env in envs.values():
            env.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
