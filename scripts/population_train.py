"""K PPO, IMPALA or PG trainings in one batch on a config-3-like environment (64 workers, ResNet-50): learn-call and
minibatch-step time of DevicePopulation{PPO,IMPALA,PG}Learner against K sequential single-learner calls, and every set's mean
return per iteration.

    python scripts/population_train.py --out profiles/h100_population_ppo_train.jsonl
    python scripts/population_train.py --algo impala --out profiles/h100_population_impala_train.jsonl
    python scripts/population_train.py --algo pg --out profiles/h100_population_pg_train.jsonl

Timing rows ('kind': 'timing'): for each K, one collect on a K b-episode environment (b episodes per group) with the algorithm's
settings (ppo.yaml's except num_sgd_iter; IMPALAConfig's, PGConfig's), then learn calls timed with a device synchronise around
each, alternating with the single learner's call on a b-episode environment; the single call is timed once per repeat and
multiplied by K (the K sequential calls would do the same work K times).  minibatch_step_ms is the call's time over its minibatch
steps (PPO: num_sgd_iter x minibatches; IMPALA: its SGD steps; PG: its one step).  Each measurement repeats `--repeats` times.
Return rows ('kind': 'returns'): a grid over lr x entropy_coeff (PG, which has no entropy term: lr x gamma), --iters iterations
of collect + learn, each set's mean episode return (the group's summed rewards over its episodes).  The first row names the card,
its power limit and max SM clock, read in the same process.

    python scripts/population_train.py --shapes sweep --algo {ppo,impala,pg}

writes profiles/h100_population_shapes_<algo>_train.jsonl instead: scripts/wandb_sweep_config.yaml's PHASE 3 grid (out_features_msg,
_hidden, _node over {8, 16, 32, 64}, num_rounds over {2, 4}: 128 shapes at gnn.yaml's other settings), one shape per set.  Rows
'mixed' time the 128-shape population's learn call, rows 'same' homogeneous K = 128 populations at gnn.yaml's shape and at the
grid's largest, --repeats each, alternating; the row 'sequential' sums 128 single learners' calls, one per shape, each on its own
b-episode environment and timed once after a warm-up call.

    python scripts/population_train.py --algo es [--shapes sweep]

writes profiles/h100_population_es_train.jsonl: for each K, one learn() step of DevicePopulationESLearner on a K b-episode
environment (ESConfig's es.yaml defaults: about 8 rounds of --jobs env-steps at b = 128) with timing=True's embed / rollout /
update split, alternating with K sequential DeviceESLearner steps on a b-episode environment, one per set, with the same split
summed over the K steps (--shapes sweep: set k has PHASE 3 shape k mod 128; otherwise gnn.yaml's shape).  Each measurement
repeats `--repeats` times after a warm-up step."""
import argparse
import dataclasses
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True).stdout.strip().splitlines()[0].split(', ')
        return {'gpu': q[0], 'power_limit': q[1], 'max_sm_clock': q[2]}
    except Exception as e:                                       # noqa: BLE001 -- recorded, not hidden
        return {'gpu': f'unknown ({e})'}


def env_of(graphs, B, J, seed):
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    return DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=B, jobs_per_episode=J, seed=seed)


def timed(fn, sync):
    sync()
    t0 = time.perf_counter()
    out = fn()
    sync()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--algo', choices=('ppo', 'impala', 'pg', 'es'), default='ppo')
    ap.add_argument('--ks', default='1,8,32,128')
    ap.add_argument('--b', type=int, default=128, help='episodes per group')
    ap.add_argument('--horizon', type=int, default=4)
    ap.add_argument('--jobs', type=int, default=4)
    ap.add_argument('--num-sgd-iter', type=int, default=1, help='ppo: ppo.yaml has 50; the timed calls run this many passes')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--grid-k', type=int, default=8)
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--shapes', choices=('same', 'sweep'), default='same', help='sweep: one PHASE 3 shape per set')
    ap.add_argument('--out', default=None, help='default: profiles/h100_population_<algo>_train.jsonl (--shapes sweep: '
                    'profiles/h100_population_shapes_<algo>_train.jsonl)')
    a = ap.parse_args()
    import torch
    from ddls_b200 import learn, policy as P, workload
    if not torch.cuda.is_available():
        raise SystemExit('population_train.py measures on the GPU; no CUDA device is visible')
    sync = torch.cuda.synchronize
    graphs = [workload.make_graph('resnet')]
    A = 17
    if a.algo == 'es':
        es_timing(a, graphs, A, sync)
        return
    cfg0 = P.algo_model_config(a.algo, A)
    Pop, Single, base = {'ppo': (learn.DevicePopulationPPOLearner, learn.DevicePPOLearner, learn.PPOConfig(num_sgd_iter=a.num_sgd_iter)),
                         'impala': (learn.DevicePopulationIMPALALearner, learn.DeviceIMPALALearner, learn.IMPALAConfig()),
                         'pg': (learn.DevicePopulationPGLearner, learn.DevicePGLearner, learn.PGConfig())}[a.algo]
    seeded = (lambda c, k: dataclasses.replace(c, seed=k)) if a.algo == 'ppo' else (lambda c, k: c)
    out_path = a.out or f'profiles/h100_population_{"shapes_" if a.shapes == "sweep" else ""}{a.algo}_train.jsonl'
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    out = open(out_path, 'w')

    def emit(row):                                               # written as measured: a cut-short run keeps what it measured
        print(json.dumps(row), flush=True)
        out.write(json.dumps(row) + '\n')
        out.flush()

    def steps(rows):
        """the minibatch / SGD steps of one call on a group of `rows` rows"""
        if a.algo == 'ppo':
            return -(-rows // base.sgd_minibatch_size) * a.num_sgd_iter
        if a.algo == 'impala':
            L = base.rollout_fragment_length or a.horizon
            n_frag = rows // L
            return -(-n_frag // min(base.train_batch_size // L, n_frag))
        return 1

    head = dict(kind='card', **card(), **({} if a.algo == 'ppo' else dict(algo=a.algo)), b=a.b, horizon=a.horizon, jobs=a.jobs)
    if a.algo == 'ppo':
        head.update(num_sgd_iter=a.num_sgd_iter, sgd_minibatch_size=base.sgd_minibatch_size)
    elif a.algo == 'impala':
        head.update(rollout_fragment_length=base.rollout_fragment_length, train_batch_size=base.train_batch_size)
    emit(head)
    if a.shapes == 'sweep':
        sweep(a, graphs, A, Pop, Single, base, seeded, steps, emit, sync)
        out.close()
        return
    # the single learner on a b-episode environment
    senv = env_of(graphs, a.b, a.jobs, seed=1)
    spol = P.DeviceGNNPolicy(graphs, A, cfg0, P.random_state_dict(cfg0, A, seed=0))
    slrn = Single(spol, base)
    spol.collect(senv, a.horizon, seed=0)
    slrn.learn(senv, a.horizon)                                  # warm-up
    for K in [int(k) for k in a.ks.split(',')]:
        env = env_of(graphs, K * a.b, a.jobs, seed=1)
        pop = P.DeviceGNNPolicyPopulation(graphs, A, cfg0, [P.random_state_dict(cfg0, A, seed=k) for k in range(K)])
        lrn = Pop(pop, [seeded(base, k) for k in range(K)])
        pop.collect(env, a.horizon, seed=list(range(K)))
        lrn.learn(env, a.horizon)                                # warm-up: every buffer and launch shape
        for r in range(a.repeats):
            tp, stats = timed(lambda: lrn.learn(env, a.horizon), sync)
            ts, _ = timed(lambda: slrn.learn(senv, a.horizon), sync)
            n_mb = steps(a.horizon * a.b)
            emit(dict(kind='timing', K=K, repeat=r, population_learn_s=tp, population_minibatch_step_ms=1e3 * tp / n_mb,
                      single_learn_s=ts, single_x_K_learn_s=ts * K, single_minibatch_step_ms=1e3 * ts / n_mb,
                      embed_ctas=pop.embed_ctas(), train_rows=[int(s['rows']) for s in stats][:4]))
        pop.close()
        del env
    # returns: a grid over lr x entropy_coeff (PG: lr x gamma)
    lrs, second = [1e-4, 3e-4, 1e-3, 3e-3], ('gamma', [0.99, 0.9]) if a.algo == 'pg' else ('entropy_coeff', [0.0, 0.01])
    grid = [(lr, e) for lr in lrs for e in second[1]][:a.grid_k]
    K = len(grid)
    env = env_of(graphs, K * a.b, a.jobs, seed=2)
    pop = P.DeviceGNNPolicyPopulation(graphs, A, cfg0, [P.random_state_dict(cfg0, A, seed=0)] * K)
    lrn = Pop(pop, [seeded(dataclasses.replace(base, lr=lr, **{second[0]: e}), k) for k, (lr, e) in enumerate(grid)])
    for it in range(a.iters):
        traj = pop.collect(env, a.jobs, seed=[100 * it + k for k in range(K)])
        ret = (traj['reward'] * traj['live']).sum(axis=0).reshape(K, a.b).mean(axis=1)
        lrn.learn(env, a.jobs)
        emit(dict(kind='returns', iteration=it, sets=[{'lr': lr, second[0]: e, 'mean_return': float(x)} for (lr, e), x in zip(grid, ret)]))
    pop.close()
    out.close()


def es_timing(a, graphs, A, sync):
    """the population's ES step against K sequential single ES steps, alternating; see the module docstring"""
    import numpy as np
    from ddls_b200 import learn, policy as P
    out_path = a.out or 'profiles/h100_population_es_train.jsonl'
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    out = open(out_path, 'w')

    def emit(row):
        print(json.dumps(row), flush=True)
        out.write(json.dumps(row) + '\n')
        out.flush()

    ks = [int(k) for k in a.ks.split(',')]
    shapes = [dict(P.DEFAULT_CONFIG, **s) for s in phase3_grid()] if a.shapes == 'sweep' else [dict(P.DEFAULT_CONFIG)]
    base = learn.ESConfig(noise_size=1 << 25)
    noise = np.random.default_rng(0).standard_normal(base.noise_size, dtype=np.float32)   # its values do not change the work
    emit(dict(kind='card', **card(), algo='es', shapes=a.shapes, b=a.b, jobs=a.jobs, episodes_per_batch=base.episodes_per_batch,
              train_batch_size=base.train_batch_size, eval_prob=base.eval_prob))
    senv = env_of(graphs, a.b, a.jobs, seed=1)
    singles = []                                                 # a policy and an ES learner per shape, each warmed up once
    for k, c in enumerate(shapes[:max(ks)]):
        spol = P.DeviceGNNPolicy(graphs, A, c, P.random_state_dict(c, A, seed=k))
        slrn = learn.DeviceESLearner(spol, dataclasses.replace(base, seed=k), noise=noise)
        slrn.learn(senv)
        singles.append((spol, slrn))
    for K in ks:
        env = env_of(graphs, K * a.b, a.jobs, seed=1)
        cfgs = [shapes[k % len(shapes)] for k in range(K)]
        pop = P.DeviceGNNPolicyPopulation(graphs, A, cfgs, [P.random_state_dict(c, A, seed=k) for k, c in enumerate(cfgs)])
        lrn = learn.DevicePopulationESLearner(pop, [dataclasses.replace(base, seed=k) for k in range(K)], noise=noise)
        lrn.learn(env)                                           # warm-up: every buffer and launch shape
        for r in range(a.repeats):
            tp, stats = timed(lambda: lrn.learn(env, timing=True), sync)
            ts, split = [], dict(embed_s=0.0, rollout_s=0.0, update_s=0.0)
            for k in range(K):
                t, st = timed(lambda: singles[k % len(singles)][1].learn(senv, timing=True), sync)
                ts.append(t)
                for key in split:
                    split[key] += st[key]
            ctas, items = lrn.embed_ctas()
            emit(dict(kind='timing', K=K, repeat=r, population_step_s=tp, embed_s=stats[0]['embed_s'], rollout_s=stats[0]['rollout_s'],
                      update_s=stats[0]['update_s'], rounds=max(int(s['rounds']) for s in stats), single_steps_s=sum(ts),
                      single_step_s_min=min(ts), single_step_s_max=max(ts), single_embed_s=split['embed_s'],
                      single_rollout_s=split['rollout_s'], single_update_s=split['update_s'], last_embed_ctas=ctas, last_embed_items=items))
        lrn.close()
        pop.close()
        del env
    for spol, slrn in singles:
        slrn.close()
        spol.close()
    out.close()


def phase3_grid():
    """scripts/wandb_sweep_config.yaml's PHASE 3: out_features_msg, _hidden, _node over {8, 16, 32, 64}, num_rounds over {2, 4}"""
    return [dict(out_features_msg=m, out_features_hidden=h, out_features_node=n, num_rounds=r)
            for m in (8, 16, 32, 64) for h in (8, 16, 32, 64) for n in (8, 16, 32, 64) for r in (2, 4)]


def sweep(a, graphs, A, Pop, Single, base, seeded, steps, emit, sync):
    """the 128-shape population's learn call against homogeneous K = 128 populations and 128 sequential single learners"""
    from ddls_b200 import policy as P
    shapes = [dict(P.DEFAULT_CONFIG, **s) for s in phase3_grid()]
    K = len(shapes)
    n_mb = steps(a.horizon * a.b)
    largest = dict(P.DEFAULT_CONFIG, **max(phase3_grid(), key=lambda s: P.weight_count(dict(P.DEFAULT_CONFIG, **s), A)))
    runs = {'mixed': shapes, 'gnn_yaml': [dict(P.DEFAULT_CONFIG)] * K, 'largest': [largest] * K}
    emit(dict(kind='shapes', K=K, weights=[P.weight_count(c, A) for c in shapes], largest=largest))
    live = {}
    for name, cfgs in runs.items():
        env = env_of(graphs, K * a.b, a.jobs, seed=1)
        pop = P.DeviceGNNPolicyPopulation(graphs, A, cfgs, [P.random_state_dict(c, A, seed=k) for k, c in enumerate(cfgs)])
        lrn = Pop(pop, [seeded(base, k) for k in range(K)])
        pop.collect(env, a.horizon, seed=list(range(K)))
        lrn.learn(env, a.horizon)                                # warm-up: every buffer and launch shape
        live[name] = (env, pop, lrn)
    for r in range(a.repeats):
        for name, (env, pop, lrn) in live.items():
            t, _ = timed(lambda: lrn.learn(env, a.horizon), sync)
            emit(dict(kind='mixed' if name == 'mixed' else 'same', shape=name, K=K, repeat=r, population_learn_s=t,
                      population_minibatch_step_ms=1e3 * t / n_mb, embed_ctas=pop.embed_ctas()))
    for env, pop, lrn in live.values():
        pop.close()
    live.clear()
    # 128 single learners, one per shape, each timed once
    times = []
    senv = env_of(graphs, a.b, a.jobs, seed=1)
    for k, c in enumerate(shapes):
        spol = P.DeviceGNNPolicy(graphs, A, c, P.random_state_dict(c, A, seed=k))
        slrn = Single(spol, seeded(base, k))
        spol.collect(senv, a.horizon, seed=k)
        slrn.learn(senv, a.horizon)                              # warm-up
        t, _ = timed(lambda: slrn.learn(senv, a.horizon), sync)
        times.append(t)
        spol.close()
    emit(dict(kind='sequential', K=K, single_learn_s_sum=sum(times), single_learn_s_min=min(times), single_learn_s_max=max(times),
              single_learn_s=times))


if __name__ == '__main__':
    main()
