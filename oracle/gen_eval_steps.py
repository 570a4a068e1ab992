"""TEST INFRASTRUCTURE -- records, env-step by env-step, what the unmodified reference's ``EvalLoop.run`` (loops/eval_loop.py:26-134)
reports in ``results['step_stats']`` for the 16 golden episodes, as tests/golden/observations/eval_steps.npz: the fixture both batched
environments' per-env-step rows are pinned against (tests/test_eval_step_stats_model.py, tests/test_gpu_eval_step_stats.py).  Build
container only (needs the reference):

    PYTHONHASHSEED=0 python oracle/gen_eval_steps.py

Every case of gen_golden.CASES is re-run with its seed and environment; the case's own agent decides, and each decision is checked
against the actions oracle/gen_env_obs.py recorded.  The episode runs inside ``EvalLoop.run`` itself.  Its reduction of a per-tick utilisation list over
an env-step of several cluster steps is ``np.mean`` of a list of lists; when their lengths differ numpy >= 1.24 raises ValueError,
which EvalLoop does not catch.  The episode is then finished step by step, and the rows come from EvalLoop's rules applied to the
recorded ``steps_log`` slices (``reduce_slices`` below).  Where EvalLoop completes, its own rows are the fixture's and the rules are
asserted to give them bit for bit.  Per case ``<name>_``:

  * ``keys``          the cluster's ``steps_log`` keys in insertion order
  * ``evalloop``      1 if ``EvalLoop.run`` completed (rows are its own), 0 if its rules were applied to the slices
  * ``cs``            cluster steps of every env-step
  * ``log``           [cluster steps, len(keys)] every cluster step's ``steps_log`` entry (the two per-tick lists: NaN)
  * ``ticks``         [cluster steps] length of the per-tick lists; ``util``: [sum(ticks), 2] their entries, in order
  * ``rows``          [env-steps, len(keys)] the per-env-step reduction of every key, env-step slices taken at the cluster-step
                      boundaries (the two per-tick lists: the mean over every entry of the env-step)
  * ``prev_idx``      [env-steps] where EvalLoop starts each env-step's slice: ``len()`` of the LAST key after the previous env-step
                      (eval_loop.py:99); ``start`` [env-steps] where the env-step's first cluster step is
  * ``actions``, ``rewards``  EvalLoop's ``action`` / ``reward`` entries
"""
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import gen_golden as G  # noqa: E402  (installs the import shim, imports the reference)
from ddls.loops.eval_loop import EvalLoop  # noqa: E402

UTIL_KEYS = ('mean_mounted_worker_utilisation_frac', 'mean_cluster_worker_utilisation_frac')


def reduce_slices(key, vals):
    """EvalLoop's rule for one key over the values one env-step's cluster steps appended (eval_loop.py:50-97); the per-tick lists
    are reduced by the mean over every entry."""
    if key == 'step_start_time':
        return vals[0]
    if key in ('step_end_time', 'step_counter'):
        return vals[-1]
    if key in UTIL_KEYS:
        return np.mean(np.concatenate([np.asarray(v, dtype=np.float64).reshape(-1) for v in vals]))
    if 'mean' in key:
        return np.mean(vals)
    return np.sum(vals)


class Replay:
    """The case's own agent, checked decision by decision against the recorded actions: Random draws from numpy's global
    generator, which the environment's job sampling shares, so the agent must still draw for the episode to be the recorded one."""

    def __init__(self, agent, actions):
        self.agent, self.actions, self.k = agent, [int(a) for a in actions], 0

    def compute_action(self, obs, job_to_place=None):
        a = int(self.agent.compute_action(obs, job_to_place=job_to_place))
        assert a == self.actions[self.k], (self.k, a, self.actions[self.k])
        self.k += 1
        return a


def run_case(name, spec, obs, out):
    actions = obs[name + '_actions']
    np.random.seed(spec['seed']); random.seed(spec['seed'])
    d = G.tempfile.mkdtemp(prefix='eval_steps_')
    for g in spec['graphs']:
        g.write(d)
    env = G.make_env(d, spec['shape'], spec['n_jobs'], spec['max_partitions'], spec['interarrival'],
                     G.Uniform(spec['frac'][0], spec['frac'][1], decimals=2), max_sim_time=spec.get('max_sim_time', 1e6))
    np.random.seed(spec['seed']); random.seed(spec['seed'])
    ends, prev_idx, state = [], [0], {'done': False}
    orig_step = env.step

    def step(a):
        o = orig_step(a)
        log = env.cluster.steps_log
        ends.append(len(log['step_end_time']))
        prev_idx.append(len(list(log.values())[-1]))
        state['done'] = bool(o[2])
        return o
    env.step = step
    agent = {'random': G.Random(), 'sipml': G.SiPML(spec['max_partitions']), 'acceptable_jct': G.AcceptableJCT()}[spec['actor']]
    actor = Replay(agent, actions)
    results, evalloop = None, 1
    try:
        results = EvalLoop(actor=actor, env=env).run()
    except ValueError as ex:                      # np.mean of ragged per-tick lists (numpy >= 1.24)
        evalloop = 0
        print(f'{name}: EvalLoop.run raised at env-step {len(ends)}: {ex}', flush=True)
        while not state['done']:
            env.step(actor.compute_action(env.obs, job_to_place=list(env.cluster.job_queue.jobs.values())[0]))
    assert actor.k == len(actions), (name, actor.k, len(actions))
    log = env.cluster.steps_log
    keys = list(log.keys())
    n_cs = len(log['step_end_time'])
    assert all(len(v) == n_cs for v in log.values()), name          # every cluster step sets every key (finding 2)
    start = [0] + ends[:-1]
    rows = np.zeros((len(ends), len(keys)))
    for e in range(len(ends)):
        for j, k in enumerate(keys):
            rows[e, j] = reduce_slices(k, log[k][start[e]:ends[e]])
    if results is not None:
        for j, k in enumerate(keys):
            got = np.array(results['step_stats'][k], dtype=np.float64)
            assert np.array_equal(got, rows[:, j]), (name, k, got, rows[:, j])
    ticks = np.array([len(v) for v in log[UTIL_KEYS[0]]], dtype=np.int32)
    util = np.stack([np.concatenate([np.asarray(v, dtype=np.float64).reshape(-1) for v in log[k]]) for k in UTIL_KEYS], axis=1)
    flat = np.array([[np.nan if k in UTIL_KEYS else float(log[k][c]) for k in keys] for c in range(n_cs)], dtype=np.float64)
    p = name + '_'
    out[p + 'keys'] = np.array(keys)
    out[p + 'evalloop'] = np.array(evalloop)
    out[p + 'cs'] = np.diff([0] + ends).astype(np.int32)
    out[p + 'log'] = flat
    out[p + 'ticks'] = ticks
    out[p + 'util'] = util
    out[p + 'rows'] = rows
    out[p + 'prev_idx'] = np.array(prev_idx[:-1], dtype=np.int32)
    out[p + 'start'] = np.array(start, dtype=np.int32)
    out[p + 'actions'] = np.array(actions, dtype=np.int32)
    rw = results['step_stats']['reward'] if results is not None else []
    out[p + 'rewards'] = np.array(rw, dtype=np.float64)
    n_shift = int(np.sum(out[p + 'prev_idx'] != out[p + 'start']))
    print(f'{name}: {len(ends)} env-steps, {n_cs} cluster steps, max {int(out[p + "cs"].max())} per env-step, EvalLoop '
          f'{"completed" if evalloop else "raised"}, {n_shift} env-steps whose EvalLoop slice starts elsewhere', flush=True)


def main():
    if os.environ.get('PYTHONHASHSEED') != '0':
        print('note: run with PYTHONHASHSEED=0 for byte-identical regeneration', file=sys.stderr)
    obs = np.load(os.path.join(ROOT, 'tests', 'golden', 'observations', 'env_obs.npz'))
    out = {}
    for name, spec in G.CASES.items():
        run_case(name, spec, obs, out)
    out['cases'] = np.array(list(G.CASES))
    path = os.path.join(ROOT, 'tests', 'golden', 'observations', 'eval_steps.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path) // 1024, 'KiB')


if __name__ == '__main__':
    main()
