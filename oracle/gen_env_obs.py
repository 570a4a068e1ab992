"""TEST INFRASTRUCTURE -- records, step by step, the observations the unmodified reference's RampJobPartitioningEnvironment hands
its agent in the 16 golden episodes, as tests/golden/observations/env_obs.npz: the fixture both batched environments' observations are pinned
against (tests/test_gpu_env_observation.py, tests/test_env_observation_model.py).  Build container only (needs the reference):

    PYTHONHASHSEED=0 python oracle/gen_env_obs.py

Every case of gen_golden.CASES is re-run with its seed, environment and actor.  Of the observations ``_encode_obs`` produces only
those ``RJPE._get_observation`` returns are kept -- the one from ``reset`` and the one after every ``step`` that is not the last --
so the k-th kept observation is the one the agent decided env-step k on (the extra encode inside ``observation_function.reset``
is dropped).  Per case ``<name>_``:

  * ``step``            env-steps taken before the observation (0 = the one from reset)
  * ``job_idx``, ``frac``  the queued job's index and max_acceptable_job_completion_time_frac
  * ``graph_features``  float32 [K, 17 + |A|], ``action_mask`` int16 [K, |A|]
  * ``n_mounted``, ``n_running``  len(cluster.mounted_workers), len(cluster.jobs_running)
  * ``max_partitions_per_op``, ``machine_epsilon``
  * ``jobs_params``     [8, 2]: (min, max) of jobs_generator.jobs_params for each of observation.PARAM_KEYS
  * ``arrivals``        (gap, orig_op_mem, orig_dep_size) per arrival, as gen_golden records them
  * ``actions``         the action of every env-step
"""
import os
import random
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import gen_golden as G  # noqa: E402  (installs the import shim, imports the reference)
from ddls.environments.ramp_job_partitioning.observations import ramp_job_partitioning_observation as O  # noqa: E402
from ddls_b200.observation import PARAM_KEYS  # noqa: E402

RJPE = G.RampJobPartitioningEnvironment


def run_case(name, spec, out):
    kept, arrivals = [], []
    state = {'step': 0, 'keep': False}
    orig_encode, orig_get_obs, orig_next = O.RampJobPartitioningObservation._encode_obs, RJPE._get_observation, G.RampClusterEnvironment._get_next_job

    def _encode_obs(self, job, env, flatten=True):
        obs = orig_encode(self, job, env, flatten=flatten)
        if state['keep']:
            cl = env.cluster
            kept.append(dict(step=state['step'], job_idx=job.details['job_idx'], frac=job.max_acceptable_job_completion_time_frac,
                             graph_features=np.array(obs['graph_features'], dtype=np.float32),
                             action_mask=np.array(obs['action_mask'], dtype=np.int16), n_mounted=len(cl.mounted_workers),
                             n_running=len(cl.jobs_running), eps=self.machine_epsilon))
        return obs

    def _get_observation(env):
        state['keep'] = True
        try:
            return orig_get_obs(env)
        finally:
            state['keep'] = False

    def _get_next_job(cluster):
        before = cluster.time_next_job_to_arrive
        job = orig_next(cluster)
        arrivals.append((float(cluster.time_next_job_to_arrive - before), float(job.original_job.details['job_total_op_memory_cost']),
                         float(job.original_job.details['job_total_dep_size'])))
        return job

    O.RampJobPartitioningObservation._encode_obs = _encode_obs
    RJPE._get_observation = _get_observation
    G.RampClusterEnvironment._get_next_job = _get_next_job
    try:
        np.random.seed(spec['seed']); random.seed(spec['seed'])
        d = tempfile.mkdtemp(prefix='env_obs_')
        for g in spec['graphs']:
            g.write(d)
        env = G.make_env(d, spec['shape'], spec['n_jobs'], spec['max_partitions'], spec['interarrival'],
                         G.Uniform(spec['frac'][0], spec['frac'][1], decimals=2), max_sim_time=spec.get('max_sim_time', 1e6))
        kept.clear(); arrivals.clear()                     # the constructor's own reset() is not part of the episode
        np.random.seed(spec['seed']); random.seed(spec['seed'])
        state['step'] = 0
        obs = env.reset()
        actor = {'random': G.Random(), 'sipml': G.SiPML(spec['max_partitions']), 'acceptable_jct': G.AcceptableJCT()}[spec['actor']]
        actions, done = [], False
        while not done:
            job = list(env.cluster.job_queue.jobs.values())[0]
            a = int(actor.compute_action(obs, job_to_place=job))
            actions.append(a)
            state['step'] = len(actions)
            obs, _, done, _ = env.step(a)
        jp = env.cluster.jobs_generator.jobs_params
    finally:
        O.RampJobPartitioningObservation._encode_obs = orig_encode
        RJPE._get_observation = orig_get_obs
        G.RampClusterEnvironment._get_next_job = orig_next
    p = name + '_'
    for k, dt in (('step', np.int32), ('job_idx', np.int32), ('frac', np.float64), ('n_mounted', np.int32), ('n_running', np.int32)):
        out[p + k] = np.array([o[k] for o in kept], dtype=dt)
    out[p + 'graph_features'] = np.stack([o['graph_features'] for o in kept])
    out[p + 'action_mask'] = np.stack([o['action_mask'] for o in kept])
    out[p + 'max_partitions_per_op'] = np.array(int(env.max_partitions_per_op))
    out[p + 'machine_epsilon'] = np.array(float(kept[0]['eps']))
    out[p + 'jobs_params'] = np.array([[float(jp['min_' + k]), float(jp['max_' + k])] for k in PARAM_KEYS], dtype=np.float64)
    out[p + 'arrivals'] = np.array(arrivals, dtype=np.float64).reshape(-1, 3)
    out[p + 'actions'] = np.array(actions, dtype=np.int32)
    print(f'{name}: {len(actions)} env-steps, {len(kept)} observations', flush=True)


def main():
    if os.environ.get('PYTHONHASHSEED') != '0':
        print('note: run with PYTHONHASHSEED=0 for byte-identical regeneration', file=sys.stderr)
    out = {}
    for name, spec in G.CASES.items():
        run_case(name, spec, out)
    out['cases'] = np.array(list(G.CASES))
    path = os.path.join(ROOT, 'tests', 'golden', 'observations', 'env_obs.npz')      # not beside the goldens: every *.npz there is a golden episode
    os.makedirs(os.path.dirname(path), exist_ok=True)
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path) // 1024, 'KiB')


if __name__ == '__main__':
    main()
