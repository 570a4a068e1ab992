"""Times ``ddls_b200.agents.evaluate`` -- EvalLoop over every episode of a device environment at once -- with each of the
reference's heuristic agents, on bench.py's config 3 (4,096 episodes of a 64-worker RAMP, the ResNet-50-like job, every block
geometry prewarmed so that the loop never waits for the host).  Prints one line per agent: env-steps per second (live
episodes' decisions over the wall time of evaluate(), which ends in a synchronise), and the episodes' mean acceptance rate,
with the card's name and power limit.  --step-stats times evaluate(step_stats=True): the device also records every env-step's
EvalLoop row, action and reward, and the timed window includes reading the record back.

    python scripts/eval_rollouts.py [--episodes 4096] [--jobs 8] [--repeats 3] [--step-stats]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(',')]
        return name, power
    except Exception as ex:                                      # the figures are still printed, without the card
        return f'unknown ({ex!r})', 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--episodes', type=int, default=4096)
    ap.add_argument('--jobs', type=int, default=8)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--step-stats', action='store_true', help="evaluate(step_stats=True): EvalLoop's per-env-step record as well")
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('eval_rollouts.py measures the GPU: no CUDA device')
    from ddls_b200 import workload
    from ddls_b200.agents import AGENTS, DeviceHeuristicAgents, evaluate
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    cfg = workload.CONFIGS['cfg3-resnet50-64w']
    graphs = [workload.make_graph(kind, **kw) for kind, kw in cfg['graphs']]
    env = DeviceRampJobPartitioningEnvironment(tuple(cfg['shape']), graphs, n_episodes=args.episodes, jobs_per_episode=args.jobs,
                                               seed=args.seed, prewarm=True)
    name, power = card()
    for kind in AGENTS:
        agents = DeviceHeuristicAgents(env, kind)            # SiPML without a maximum: the largest valid degree
        evaluate(env, agents, seed=args.seed, step_stats=args.step_stats)     # warm-up: memo, lookahead hints, module loads
        rates = []
        for r in range(args.repeats):
            t0 = time.perf_counter()
            es = evaluate(env, agents, seed=args.seed + r, step_stats=args.step_stats)
            dt = time.perf_counter() - t0
            if args.step_stats:
                es = es['episode_stats']
            rates.append(float(env.decisions().sum()) / dt)
        print(json.dumps({'agent': kind, 'step_stats': args.step_stats, 'episodes': args.episodes, 'jobs_per_episode': args.jobs,
                          'env_steps_per_s': [round(x, 1) for x in rates], 'acceptance_rate': round(float(np.mean(es['acceptance_rate'])), 4),
                          'mean_return': round(float(np.mean(es['return'])), 4), 'card': name, 'power_limit': power}), flush=True)
    env.close()


if __name__ == '__main__':
    main()
