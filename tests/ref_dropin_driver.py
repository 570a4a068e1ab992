"""TEST INFRASTRUCTURE: drives the UNMODIFIED reference's RampJobPartitioningEnvironment + heuristic agents with
``ddls_b200.host.RampClusterEnvironment`` swapped in for the reference's cluster environment (the INTEGRATION.md stub:
RJPE:199-206), on one of the seeded golden episodes, and prints what the reference itself recorded for that episode
(tests/golden/<case>.npz) next to what this run produced.

    PYTHONHASHSEED=0 python tests/ref_dropin_driver.py <case> [--fake-engine] [--reference-cluster [--record]]

--fake-engine answers the engine calls with the CPU oracle (tests/fake_engine.py) so the host logic can be checked
without a GPU; without it the CUDA engine is used (needs cuda:0).  --reference-cluster runs the reference's own cluster
environment instead of the drop-in; with --record its result is stored as tests/golden/<case>_reference_cluster.json, the
run the drop-in is compared with in tests/test_reference_dropin.py."""
import json
import os
import random
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)


# The reference lists its job files with an UNSORTED glob (jobs_generator.py:96), so which file is "job type 0" depends on the
# file system's directory order.  These are the orders of the container the golden fixtures were generated in; the driver pins
# them so that the seeded episodes are the same episodes on every machine.
FILE_ORDER = {'mixed16': ['res2.txt', 'chain5.txt', 'tfm1.txt'], 'mixed64_busy': ['tfm1b.txt', 'chain4.txt', 'res1.txt'],
              'mix128_exp': ['resnet50_like.txt', 'gpt2_small_like.txt']}

EXTRA_CASES = {
    # a generator that never runs dry (the reference's default 'remove_and_repeat' sampling, heuristic_config.yaml:126): the
    # episode ends on max_simulation_run_time, arrivals keep coming until then
    'chain8_repeat': dict(base='chain8', sampling_mode='remove_and_repeat', max_sim_time=9500.0, n_jobs=3),
    'res16_repeat': dict(base='res16_flood', sampling_mode='remove_and_repeat', max_sim_time=700.0, n_jobs=2),
}


def main():
    case = sys.argv[1]
    fake = '--fake-engine' in sys.argv
    use_reference_cluster = '--reference-cluster' in sys.argv      # run the reference's own cluster environment instead
    from oracle import ref_shim
    ref_shim.install()
    from oracle import gen_golden                     # CASES / make_env / the reference imports (no recording here)
    import ddls.environments.ramp_job_partitioning.ramp_job_partitioning_environment as rjpe_mod
    from ddls.distributions.uniform import Uniform
    from ddls.environments.ramp_job_partitioning.agents.sip_ml import SiPML
    from ddls.environments.ramp_job_partitioning.agents.random import Random
    from ddls.environments.ramp_job_partitioning.agents.acceptable_jct import AcceptableJCT
    import ddls_b200.host.cluster as host_cluster
    from ddls_b200 import host
    if fake:
        from fake_engine import FakeEngine
        host_cluster._engine.RampEngine = FakeEngine
    if not use_reference_cluster:
        rjpe_mod.RampClusterEnvironment = host.RampClusterEnvironment        # the drop-in (RJPE:199-206)

    sampling_mode = 'remove'
    if case in EXTRA_CASES:
        extra = dict(EXTRA_CASES[case])
        spec = dict(gen_golden.CASES[extra.pop('base')])
        sampling_mode = extra.pop('sampling_mode')
        spec.update(extra)
    else:
        spec = gen_golden.CASES[case]
    seed = spec['seed']
    np.random.seed(seed)
    random.seed(seed)
    d = tempfile.mkdtemp(prefix='dropin_graphs_')
    for g in spec['graphs']:
        g.write(d)
    if case in FILE_ORDER:
        import ddls.demands.jobs.jobs_generator as jg_mod
        import glob as _glob
        real_glob = _glob.glob

        class _PinnedGlob:
            @staticmethod
            def glob(pattern, *a, **kw):
                found = real_glob(pattern, *a, **kw)
                rank = {n: i for i, n in enumerate(FILE_ORDER[case])}
                return sorted(found, key=lambda pth: rank.get(os.path.basename(pth), len(rank)))
        jg_mod.glob = _PinnedGlob
    env = gen_golden.make_env(d, spec['shape'], spec['n_jobs'], spec['max_partitions'], spec['interarrival'],
                              Uniform(spec['frac'][0], spec['frac'][1], decimals=2), max_sim_time=spec.get('max_sim_time', 1e6),
                              sampling_mode=sampling_mode)
    assert isinstance(env.cluster, host.RampClusterEnvironment) != use_reference_cluster
    np.random.seed(seed)
    random.seed(seed)
    obs = env.reset()
    actor = {'random': Random(), 'sipml': SiPML(spec['max_partitions']), 'acceptable_jct': AcceptableJCT()}[spec['actor']]
    done, n_env_steps, actions = False, 0, []
    while not done:
        job_to_place = list(env.cluster.job_queue.jobs.values())[0]
        a = actor.compute_action(obs, job_to_place=job_to_place)
        actions.append(int(a))
        obs, _, done, _ = env.step(int(a))
        n_env_steps += 1
    cluster = env.cluster
    es = cluster.episode_stats
    out = {'n_env_steps': n_env_steps, 'actions': actions, 'using_reference_classes': bool(host.USING_REFERENCE_CLASSES),
           'n_cluster_steps': len(cluster.steps_log['step_end_time']),
           'completed_job_idxs': [int(k) for k in cluster.jobs_completed.keys()],
           'blocked_job_idxs': [int(k) for k in cluster.jobs_blocked.keys()],
           'steps_log': {k: [float(x) for x in cluster.steps_log[k]] for k in
                         ('step_start_time', 'step_end_time', 'num_jobs_completed', 'num_jobs_arrived', 'num_jobs_blocked',
                          'mean_num_jobs_running', 'mean_compute_overhead_frac', 'mean_communication_overhead_frac',
                          'compute_info_processed', 'mean_cluster_throughput')},
           # the two step statistics the reference leaves as per-tick lists (RCE:989-994)
           'tick_lists': {k: [[float(x) for x in step] for step in cluster.steps_log[k]] for k in
                          ('mean_mounted_worker_utilisation_frac', 'mean_cluster_worker_utilisation_frac')}}
    for k in ('num_jobs_arrived', 'num_jobs_completed', 'num_jobs_blocked'):
        out[k] = int(es[k])
    for k in ('episode_end_time', 'mean_load_rate', 'blocking_rate', 'acceptance_rate', 'compute_info_processed', 'dep_info_processed',
              'flow_info_processed', 'cluster_info_processed', 'mean_compute_throughput', 'mean_cluster_throughput',
              'mean_compute_overhead_frac', 'mean_communication_overhead_frac', 'mean_num_jobs_running', 'mean_num_mounted_workers'):
        out[k] = float(es[k])
    for k in ('job_completion_time', 'job_completion_time_speedup', 'job_communication_overhead_time', 'job_computation_overhead_time',
              'jobs_completed_mean_mounted_worker_utilisation_frac', 'jobs_completed_num_mounted_workers',
              'jobs_completed_num_mounted_channels', 'jobs_completed_max_acceptable_job_completion_time',
              'jobs_blocked_max_acceptable_job_completion_time'):
        out[k] = [float(x) for x in es[k]]
    memo = cluster.job_model_to_max_num_partitions_to_init_details
    out['is_dropin'] = not use_reference_cluster
    out['last_step_stats'] = {k: float(cluster.step_stats[k]) for k in ('num_jobs_blocked', 'num_jobs_completed', 'num_jobs_arrived', 'step_end_time')}
    out['init_details_memo_keys'] = sorted([str(m), int(p)] for m in memo for p in memo[m])
    print('RESULT ' + json.dumps(out), flush=True)
    if '--record' in sys.argv:
        assert use_reference_cluster, '--record stores the reference cluster environment\'s run'
        with open(os.path.join(HERE, 'golden', f'{case}_reference_cluster.json'), 'w') as f:
            json.dump(out, f)


if __name__ == '__main__':
    main()
