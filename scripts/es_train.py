"""Evolution strategies on the device: a config-3-like environment (64-worker RAMP cluster, ResNet-50 jobs), N training steps with
the reference's ES settings (ddls_b200.learn.ESConfig: algo/es.yaml).  The environment's episodes are one population per round:
(B - E) / 2 antithetic pairs and E eval episodes.  Per step it prints ES's statistics and the wall time of the embeddings (every
(weight set, job type)), of the rollouts and of the update, and writes them as JSON lines to --out if given.

    python scripts/es_train.py --iters 5 --episodes 1024 --jobs 16

--noise-size below the default 250,000,000 draws a shorter table (RLlib's table is its first noise_size values either way)."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--episodes', type=int, default=1024, help='environment episodes per round (the population and eval episodes)')
    ap.add_argument('--jobs', type=int, default=16, help='jobs per episode')
    ap.add_argument('--noise-size', type=int, default=250_000_000)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None)
    ap.add_argument('--model', choices=('gnn', 'algo'), default='gnn',
                    help="gnn: gnn.yaml's read-out ([256], separate value branch); algo: algo/es.yaml's (policy.algo_model_config)")
    args = ap.parse_args()
    from ddls_b200 import workload
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    from ddls_b200.learn import DeviceESLearner, ESConfig, shared_noise_table
    from ddls_b200.policy import DeviceGNNPolicy, algo_model_config

    graphs = [workload.make_graph('resnet')]
    env = DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=args.episodes, jobs_per_episode=args.jobs, seed=args.seed,
                                               prewarm=True)
    n_actions = env.max_partitions_per_op + 1
    model = algo_model_config('es', n_actions) if args.model == 'algo' else None
    pol = DeviceGNNPolicy(graphs, n_actions, config=model, seed=args.seed)
    t0 = time.perf_counter()
    noise = shared_noise_table(args.noise_size)
    noise_s = time.perf_counter() - t0
    lrn = DeviceESLearner(pol, ESConfig(noise_size=args.noise_size, seed=args.seed), noise=noise)
    del noise
    out = open(args.out, 'w') if args.out else None
    for it in range(args.iters):
        t0 = time.perf_counter()
        stats = lrn.learn(env, timing=True)
        row = dict(iter=it, step_s=time.perf_counter() - t0, episodes=env.B, n_eval=lrn.n_eval(env.B), **stats)
        if it == 0:
            row['noise_table_s'] = noise_s
        print(json.dumps(row), flush=True)
        if out:
            out.write(json.dumps(row) + '\n')
            out.flush()
    lrn.close()
    pol.close()
    env.close()


if __name__ == '__main__':
    main()
