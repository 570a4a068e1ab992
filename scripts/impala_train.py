"""IMPALA on the device: a config-3-like environment (64-worker RAMP cluster, ResNet-50 jobs), N iterations of collect + learn with the
reference's IMPALA settings (ddls_b200.learn.IMPALAConfig: algo/impala.yaml over rllib_config.yaml's base).  Per iteration it prints
the mean return, the fraction of decisions that placed their job (reward > 0 at the decision step), IMPALA's loss statistics (means
over the call's SGD steps), the number of SGD steps, and the wall time of collect, of learn and of one SGD step, and writes them as
JSON lines to --out if given.

    python scripts/impala_train.py --iters 5 --episodes 1024 --jobs 16"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--episodes', type=int, default=1024)
    ap.add_argument('--jobs', type=int, default=16, help='jobs per episode = the segment horizon (whole episodes)')
    ap.add_argument('--rollout-fragment-length', type=int, default=0, help='0: the horizon (one fragment per episode)')
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from ddls_b200 import workload
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    from ddls_b200.learn import DeviceIMPALALearner, IMPALAConfig
    from ddls_b200.policy import DeviceGNNPolicy

    graphs = [workload.make_graph('resnet')]
    env = DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=args.episodes, jobs_per_episode=args.jobs, seed=args.seed)
    pol = DeviceGNNPolicy(graphs, env.max_partitions_per_op + 1, seed=args.seed)
    lrn = DeviceIMPALALearner(pol, IMPALAConfig(rollout_fragment_length=args.rollout_fragment_length))
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
                   collect_s=t1 - t0, learn_s=t2 - t1, ms_per_sgd_step=1e3 * (t2 - t1) / max(1, stats['sgd_steps']),
                   **{k: stats[k] for k in ('total_loss', 'policy_loss', 'vf_loss', 'entropy', 'grad_gnorm', 'mean_rho', 'rows',
                                             'sgd_steps')})
        print(json.dumps(row), flush=True)
        if out:
            out.write(json.dumps(row) + '\n')
            out.flush()
    pol.close()
    env.close()


if __name__ == '__main__':
    main()
