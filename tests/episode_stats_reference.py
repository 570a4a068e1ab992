"""Host restatement of the episode-end finalisation (RampClusterEnvironment.episode_stats, RCE:1086-1106 appends, RCE:1123-1167
finalises) that ramp_episode_stats_kernel applies to its EF_ACC_* accumulators.  It reads one episode's cluster-step rows in order
(every RampClusterEnvironment.step since the reset, fused Action() steps included) and sums them one plain float addition at a
time, in cluster-step order, as the kernel does.  The two utilisation means are the mean over every per-tick entry of the episode
(the drop-in class's definition; the reference's np.mean over ragged per-step lists is not defined).
tests/test_oracle_bench_driver.py pins it to the reference's recorded es_* statistics; the GPU tests pin the kernel to it."""
from oracle.oracle import SS

ES_FIELDS = ['episode_start_time', 'episode_end_time', 'episode_time', 'num_jobs_arrived', 'num_jobs_completed', 'num_jobs_blocked',
             'mean_load_rate', 'blocking_rate', 'acceptance_rate',
             'compute_info_processed', 'dep_info_processed', 'flow_info_processed', 'cluster_info_processed',
             'demand_compute_info_processed', 'demand_dep_info_processed', 'demand_total_info_processed',
             'mean_compute_throughput', 'mean_dep_throughput', 'mean_flow_throughput', 'mean_cluster_throughput',
             'mean_demand_compute_throughput', 'mean_demand_dep_throughput', 'mean_demand_total_throughput',
             'mean_compute_overhead_frac', 'mean_communication_overhead_frac', 'mean_num_jobs_running', 'mean_num_mounted_workers',
             'mean_mounted_worker_utilisation_frac', 'mean_cluster_worker_utilisation_frac', 'num_cluster_steps', 'num_ticks', 'done']
INFO = ['compute_info_processed', 'dep_info_processed', 'flow_info_processed', 'cluster_info_processed',
        'demand_compute_info_processed', 'demand_dep_info_processed', 'demand_total_info_processed']
THROUGHPUT = ['mean_compute_throughput', 'mean_dep_throughput', 'mean_flow_throughput', 'mean_cluster_throughput',
              'mean_demand_compute_throughput', 'mean_demand_dep_throughput', 'mean_demand_total_throughput']
STEP_MEANS = ['mean_compute_overhead_frac', 'mean_communication_overhead_frac', 'mean_num_jobs_running', 'mean_num_mounted_workers']


def load_rate(rows, arrivals):
    """(sum, count) of the per-arrival load rates (RCE:362-364): the reset's arrival at time 0, then one at the end time of every
    cluster step that counts an arrival, each divided by the gap to the next arrival it schedules."""
    times = [0.0] + [float(r[SS['step_end_time']]) for r in rows for _ in range(int(r[SS['num_jobs_arrived']]))]
    total, next_arrival = 0.0, 0.0
    for k, now in enumerate(times):
        next_arrival = next_arrival + float(arrivals['interarrival'][k])
        total = total + (float(arrivals['orig_op_mem'][k]) + float(arrivals['orig_dep_size'][k])) / (next_arrival - now)
    return total, len(times)


def episode_stats(rows, arrivals):
    """rows: the episode's cluster-step rows [n, STEP_STATS_LEN] in order; arrivals: its ARRIVAL_DTYPE stream.
    Returns {ES field: float}, the values ramp_get_episode_stats writes for that episode."""
    out = {}
    t = float(rows[-1][SS['step_end_time']]) if len(rows) else 0.0                               # RCE:1125-1127
    out['episode_start_time'], out['episode_end_time'], out['episode_time'] = 0.0, t, t
    n_arr, n_comp, n_blk = 1, 0, 0                                                                 # the reset queues job 0
    for r in rows:
        n_arr += int(r[SS['num_jobs_arrived']])
        n_comp += int(r[SS['num_jobs_completed']])
        n_blk += int(r[SS['num_jobs_blocked']])
    out['num_jobs_arrived'], out['num_jobs_completed'], out['num_jobs_blocked'] = float(n_arr), float(n_comp), float(n_blk)
    lr_sum, lr_n = load_rate(rows, arrivals)
    out['mean_load_rate'] = lr_sum / lr_n                                                          # RCE:1129
    out['blocking_rate'] = n_blk / n_arr                                                           # RCE:1131-1134
    out['acceptance_rate'] = n_comp / n_arr                                                        # RCE:1135-1138
    for info_key, tp_key in zip(INFO, THROUGHPUT):                                                 # RCE:1140-1154
        info = 0.0
        for r in rows:
            info = info + float(r[SS[info_key]])
        out[info_key] = info
        out[tp_key] = info / t if (info != 0.0 and t != 0.0) else 0.0
    sums = {k: 0.0 for k in STEP_MEANS + ['util_mounted_sum', 'util_cluster_sum', 'num_ticks']}
    n_steps = 0.0
    for r in rows:
        for k in sums:
            sums[k] = sums[k] + float(r[SS[k]])
        n_steps = n_steps + 1.0
    n_ticks = sums['num_ticks']

    def mean(total, n):                                                                            # RCE:1156-1167
        return total / n if (t != 0.0 and n > 0.0) else 0.0
    for k in STEP_MEANS:
        out[k] = mean(sums[k], n_steps)
    out['mean_mounted_worker_utilisation_frac'] = mean(sums['util_mounted_sum'], n_ticks)
    out['mean_cluster_worker_utilisation_frac'] = mean(sums['util_cluster_sum'], n_ticks)
    out['num_cluster_steps'], out['num_ticks'] = n_steps, n_ticks
    out['done'] = float(rows[-1][SS['done']]) if len(rows) else 0.0
    return {k: out[k] for k in ES_FIELDS}


def as_row(es):
    """{ES field: value} -> the list in ramp_get_episode_stats' column order."""
    return [es[k] for k in ES_FIELDS]
