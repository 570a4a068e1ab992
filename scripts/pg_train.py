"""PG on the device: a config-3-like environment (64-worker RAMP cluster, ResNet-50 jobs), N iterations of collect + learn with the
reference's PG settings (ddls_b200.learn.PGConfig: rllib_config.yaml's gamma and lr, torch.optim.Adam's defaults, no clipping).
Each iteration's segment is every episode's whole run (horizon = jobs per episode), one train batch of complete episodes, one
Adam step.  Per iteration it prints the mean return, the fraction of decisions that placed their job (reward > 0 at the decision
step), PG's statistics, and the wall time of collect and of learn, and writes them as JSON lines to --out if given.

    python scripts/pg_train.py --iters 5 --episodes 1024 --jobs 16"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--episodes', type=int, default=1024)
    ap.add_argument('--jobs', type=int, default=16, help='jobs per episode = the segment horizon (whole episodes)')
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from ddls_b200 import workload
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    from ddls_b200.learn import DevicePGLearner, PGConfig
    from ddls_b200.policy import DeviceGNNPolicy

    graphs = [workload.make_graph('resnet')]
    env = DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=args.episodes, jobs_per_episode=args.jobs, seed=args.seed)
    pol = DeviceGNNPolicy(graphs, env.max_partitions_per_op + 1, seed=args.seed)
    lrn = DevicePGLearner(pol, PGConfig())
    out = open(args.out, 'w') if args.out else None
    for it in range(args.iters):
        stats, traj = lrn.collect_and_learn(env, args.jobs, seed=args.seed + 1000 * it)
        live = traj['live'] & (traj['model'] >= 0)
        ret = traj['reward'].sum(0)                       # every episode ends inside the segment (horizon = jobs per episode)
        placed = live & (traj['reward'] > 0)
        row = dict(iter=it, mean_return=float(ret.mean()), placed_per_decision=float(placed.sum() / max(1, live.sum())),
                   **{k: stats[k] for k in ('policy_loss', 'entropy', 'grad_gnorm', 'rows', 'collect_s', 'learn_s')})
        print(json.dumps(row), flush=True)
        if out:
            out.write(json.dumps(row) + '\n')
            out.flush()
    pol.close()
    env.close()


if __name__ == '__main__':
    main()
