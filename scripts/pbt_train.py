"""Population-based training on a config-3-like environment (64 workers, ResNet-50): the 8-set grid of population_train.py (lr x
entropy_coeff; PG: lr x gamma; ES: stepsize x noise_stdev) trained twice for --iters iterations on the same seeds, once without
PBT and once with PopulationBasedTraining every --interval iterations, and the time of a PBT step on its own.

    python scripts/pbt_train.py --algo ppo --out profiles/h100_population_pbt_ppo.jsonl

Rows:
  'card'      the card's name, power limit and max SM clock, read in the same process, and the run's settings
  'returns'   per run ('none' / 'pbt') and iteration: each set's fitness (PPO / IMPALA / PG: pbt.group_returns of the iteration's
              collect; ES: episode_reward_mean) and its mutated hyperparameters before the iteration's PBT step
  'pbt'       the PBT step's decisions: recipient, donor, old and new values
  'timing'    for each K in --ks: a PBT step (the copy launch, the ES copy for ES, and the host bookkeeping) between a device
              synchronise before and after, with scores that make every call a PBT step, against the population's learn call
              (ES: its step) timed the same way; --repeats each, alternating, after a warm-up of both.
The scores of the PBT timing are fixed, so every step moves the same pairs; the copy's work is ceil(K / 4) weight sets."""
import argparse
import dataclasses
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from population_train import card, env_of, timed  # noqa: E402

A = 17


def _setup(algo, a, graphs, K, grid, seed_env):
    import numpy as np
    from ddls_b200 import learn, pbt, policy as P
    cfg0 = P.algo_model_config(algo, A)
    pop = P.DeviceGNNPolicyPopulation(graphs, A, cfg0, [P.random_state_dict(cfg0, A, seed=0)] * K)
    if algo == 'es':
        noise = np.random.default_rng(0).standard_normal(pop.weight_count(0) + 1_000_000).astype(np.float32)
        cfgs = [learn.ESConfig(seed=k, stepsize=s, noise_stdev=n, noise_size=len(noise)) for k, (s, n) in enumerate(grid)]
        lrn = learn.DevicePopulationESLearner(pop, cfgs, noise=noise)
        mutations = {'stepsize': pbt.log_uniform(1e-3, 1e-1), 'noise_stdev': [0.005, 0.01, 0.02, 0.05]}
    else:
        second = 'gamma' if algo == 'pg' else 'entropy_coeff'
        Pop, base = {'ppo': (learn.DevicePopulationPPOLearner, learn.PPOConfig(num_sgd_iter=a.num_sgd_iter)),
                     'impala': (learn.DevicePopulationIMPALALearner, learn.IMPALAConfig()),
                     'pg': (learn.DevicePopulationPGLearner, learn.PGConfig())}[algo]
        cfgs = [dataclasses.replace(base, lr=lr, **{second: x}) for lr, x in grid]
        if algo == 'ppo':
            cfgs = [dataclasses.replace(c, seed=k) for k, c in enumerate(cfgs)]
        lrn = Pop(pop, cfgs)
        mutations = {'lr': pbt.log_uniform(1e-5, 1e-2), second: [0.9, 0.95, 0.99, 0.997] if algo == 'pg' else [0.0, 0.003, 0.01, 0.03]}
    return pop, lrn, mutations, env_of(graphs, K * a.b, a.jobs, seed=seed_env)


def _iteration(algo, pop, lrn, env, a, it):
    """one training iteration; the K fitness values"""
    from ddls_b200 import pbt
    if algo == 'es':
        return pbt.es_scores(lrn.learn(env))
    traj = pop.collect(env, a.jobs, seed=[100 * it + k for k in range(pop.K)])
    scores = pbt.group_returns(traj, pop.K)
    lrn.learn(env, a.jobs)
    return scores


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--algo', choices=('ppo', 'impala', 'pg', 'es'), default='ppo')
    ap.add_argument('--b', type=int, default=128, help='episodes per group')
    ap.add_argument('--jobs', type=int, default=4, help='jobs per episode; the collect horizon')
    ap.add_argument('--num-sgd-iter', type=int, default=1, help='ppo: ppo.yaml has 50')
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--interval', type=int, default=2)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--ks', default='8,32,128')
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--out', default=None, help='default: profiles/h100_population_pbt_<algo>.jsonl')
    a = ap.parse_args()
    import torch
    from ddls_b200 import pbt, workload
    if not torch.cuda.is_available():
        raise SystemExit('pbt_train.py measures on the GPU; no CUDA device is visible')
    sync = torch.cuda.synchronize
    graphs = [workload.make_graph('resnet')]
    out_path = a.out or f'profiles/h100_population_pbt_{a.algo}.jsonl'
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    out = open(out_path, 'w')

    def emit(row):                                               # written as measured: a cut-short run keeps what it measured
        print(json.dumps(row), flush=True)
        out.write(json.dumps(row) + '\n')
        out.flush()

    emit(dict(kind='card', **card(), algo=a.algo, b=a.b, jobs=a.jobs, iters=a.iters, interval=a.interval,
              **(dict(num_sgd_iter=a.num_sgd_iter) if a.algo == 'ppo' else {})))
    if a.algo == 'es':
        grid = [(s, n) for s in (0.003, 0.01, 0.03, 0.1) for n in (0.01, 0.05)]
    else:
        grid = [(lr, x) for lr in (1e-4, 3e-4, 1e-3, 3e-3) for x in ((0.99, 0.9) if a.algo == 'pg' else (0.0, 0.01))]
    K = len(grid)
    for run in ('none', 'pbt'):
        pop, lrn, mutations, env = _setup(a.algo, a, graphs, K, grid, seed_env=2)
        sched = pbt.PopulationBasedTraining(lrn, mutations, interval=a.interval, seed=a.seed)
        for it in range(a.iters):
            hp = [{f: getattr(c, f) for f in mutations} for c in lrn.configs]
            scores = _iteration(a.algo, pop, lrn, env, a, it)
            emit(dict(kind='returns', run=run, iteration=it, sets=[dict(h, score=float(s)) for h, s in zip(hp, scores)]))
            if run == 'pbt':
                recs = sched.step(scores)
                if recs:
                    emit(dict(kind='pbt', iteration=it, decisions=recs))
        pop.close()
        del env
    for K in [int(k) for k in a.ks.split(',')]:
        grid_k = [grid[k % len(grid)] for k in range(K)]
        pop, lrn, mutations, env = _setup(a.algo, a, graphs, K, grid_k, seed_env=3)
        sched = pbt.PopulationBasedTraining(lrn, mutations, interval=1, seed=a.seed)
        scores = list(range(K))
        _iteration(a.algo, pop, lrn, env, a, 0)                  # warm-up: the learner's buffers
        sched.step(scores)                                       # warm-up: the copy's staging and launch
        if a.algo != 'es':
            pop.collect(env, a.jobs, seed=list(range(K)))
        for r in range(a.repeats):
            tp, recs = timed(lambda: sched.step(scores), sync)
            tl, _ = timed(lambda: lrn.learn(env) if a.algo == 'es' else lrn.learn(env, a.jobs), sync)
            emit(dict(kind='timing', K=K, repeat=r, pairs=len(recs), pbt_step_s=tp, learn_s=tl))
        pop.close()
        del env
    out.close()


if __name__ == '__main__':
    main()
