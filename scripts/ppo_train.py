"""PPO on the device: a config-3-like environment (64-worker RAMP cluster, ResNet-50 jobs), N iterations of collect + learn with the
reference's PPO settings (ddls_b200.learn.PPOConfig).  Per iteration it prints the mean return, the fraction of decisions that placed their
job (reward > 0 at the decision step; not EvalLoop's acceptance_rate, which counts jobs completed over jobs arrived), the loss
statistics, and the wall time of collect and of learn, and writes them as JSON lines to --out if given.

    python scripts/ppo_train.py --iters 5 --episodes 1024 --jobs 16"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--episodes', type=int, default=1024)
    ap.add_argument('--jobs', type=int, default=16, help='jobs per episode = the segment horizon (whole episodes)')
    ap.add_argument('--num-sgd-iter', type=int, default=None, help="override ppo.yaml's 50 passes")
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None)
    ap.add_argument('--model', choices=('gnn', 'algo'), default='gnn',
                    help="gnn: gnn.yaml's read-out ([256], separate value branch); algo: algo/ppo.yaml's (policy.algo_model_config)")
    args = ap.parse_args()
    from ddls_b200 import workload
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    from ddls_b200.learn import DevicePPOLearner, PPOConfig
    from ddls_b200.policy import DeviceGNNPolicy, algo_model_config

    graphs = [workload.make_graph('resnet')]
    env = DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=args.episodes, jobs_per_episode=args.jobs, seed=args.seed)
    n_actions = env.max_partitions_per_op + 1
    model = algo_model_config('ppo', n_actions) if args.model == 'algo' else None
    pol = DeviceGNNPolicy(graphs, n_actions, config=model, seed=args.seed)
    cfg = PPOConfig(seed=args.seed)
    if args.num_sgd_iter is not None:
        cfg.num_sgd_iter = args.num_sgd_iter
    lrn = DevicePPOLearner(pol, cfg)
    out = open(args.out, 'w') if args.out else None
    for it in range(args.iters):
        t0 = time.perf_counter()
        traj = pol.collect(env, args.jobs, sample=True, seed=args.seed + 1000 * it)
        t1 = time.perf_counter()
        stats = lrn.learn(env, args.jobs)
        t2 = time.perf_counter()
        live = traj['live'] & (traj['model'] >= 0)
        ret = traj['reward'].sum(0)                       # every episode ends inside the segment (horizon = jobs per episode)
        placed = live & (traj['reward'] > 0)
        row = dict(iter=it, mean_return=float(ret.mean()), placed_per_decision=float(placed.sum() / max(1, live.sum())),
                   collect_s=t1 - t0, learn_s=t2 - t1,
                   **{k: stats[k] for k in ('total_loss', 'policy_loss', 'vf_loss', 'entropy', 'kl', 'clip_frac', 'grad_gnorm',
                                             'kl_coeff', 'rows')})
        print(json.dumps(row), flush=True)
        if out:
            out.write(json.dumps(row) + '\n')
            out.flush()
    pol.close()
    env.close()


if __name__ == '__main__':
    main()
