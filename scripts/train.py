"""PPO, IMPALA or PG on the device: a config-3-like environment (64-worker RAMP cluster, ResNet-50 jobs), N iterations of collect +
learn with the reference's settings for the algorithm (ddls_b200.learn: PPOConfig; IMPALAConfig, algo/impala.yaml over
rllib_config.yaml's base; PGConfig, rllib_config.yaml's gamma and lr, torch.optim.Adam's defaults, no clipping).  Each iteration's
segment is every episode's whole run (horizon = jobs per episode); PG makes it one train batch of complete episodes, one Adam step.
Per iteration it prints the mean return, the fraction of decisions that placed their job (reward > 0 at the decision step; not
EvalLoop's acceptance_rate, which counts jobs completed over jobs arrived), the wall time of collect and of learn (IMPALA: also of
one SGD step) and the learner's statistics (IMPALA: means over the call's SGD steps, and their number), and writes them as JSON
lines to --out if given.

    python scripts/train.py --algo ppo --iters 5 --episodes 1024 --jobs 16"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--algo', choices=('ppo', 'impala', 'pg'), required=True)
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--episodes', type=int, default=1024)
    ap.add_argument('--jobs', type=int, default=16, help='jobs per episode = the segment horizon (whole episodes)')
    ap.add_argument('--num-sgd-iter', type=int, default=None, help="ppo: override ppo.yaml's 50 passes")
    ap.add_argument('--rollout-fragment-length', type=int, default=None, help='impala: 0 (default): the horizon, one fragment per episode')
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None)
    ap.add_argument('--model', choices=('gnn', 'algo'), default='gnn',
                    help="gnn: gnn.yaml's read-out ([256], separate value branch); algo: algo/<algo>.yaml's (policy.algo_model_config)")
    args = ap.parse_args()
    if args.num_sgd_iter is not None and args.algo != 'ppo':
        ap.error('--num-sgd-iter applies to --algo ppo only')
    if args.rollout_fragment_length is not None and args.algo != 'impala':
        ap.error('--rollout-fragment-length applies to --algo impala only')
    from ddls_b200 import learn, workload
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    from ddls_b200.policy import DeviceGNNPolicy, algo_model_config

    graphs = [workload.make_graph('resnet')]
    env = DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=args.episodes, jobs_per_episode=args.jobs, seed=args.seed)
    n_actions = env.max_partitions_per_op + 1
    model = algo_model_config(args.algo, n_actions) if args.model == 'algo' else None
    pol = DeviceGNNPolicy(graphs, n_actions, config=model, seed=args.seed)
    if args.algo == 'ppo':
        cfg = learn.PPOConfig(seed=args.seed)
        if args.num_sgd_iter is not None:
            cfg.num_sgd_iter = args.num_sgd_iter
        lrn, keys = learn.DevicePPOLearner(pol, cfg), learn.STATS
    elif args.algo == 'impala':
        cfg = learn.IMPALAConfig(rollout_fragment_length=args.rollout_fragment_length or 0)
        lrn, keys = learn.DeviceIMPALALearner(pol, cfg), learn.IMPALA_STATS
    else:
        lrn, keys = learn.DevicePGLearner(pol, learn.PGConfig()), learn.PG_STATS
    out = open(args.out, 'w') if args.out else None
    for it in range(args.iters):
        stats, traj = lrn.collect_and_learn(env, args.jobs, seed=args.seed + 1000 * it)
        live = traj['live'] & (traj['model'] >= 0)
        ret = traj['reward'].sum(0)                       # every episode ends inside the segment (horizon = jobs per episode)
        placed = live & (traj['reward'] > 0)
        row = dict(iter=it, mean_return=float(ret.mean()), placed_per_decision=float(placed.sum() / max(1, live.sum())),
                   collect_s=stats['collect_s'], learn_s=stats['learn_s'])
        if args.algo == 'impala':
            row['ms_per_sgd_step'] = 1e3 * stats['learn_s'] / max(1, stats['sgd_steps'])
        row.update({k: stats[k] for k in keys})
        print(json.dumps(row), flush=True)
        if out:
            out.write(json.dumps(row) + '\n')
            out.flush()
    pol.close()
    env.close()


if __name__ == '__main__':
    main()
