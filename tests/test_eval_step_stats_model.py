"""EvalLoop's per-env-step ``step_stats`` (loops/eval_loop.py:44-100) without a GPU: the key set the product reports
(``engine.ENV_STEP_STATS``, include/ramp_b200.h RAMP_ESS_*) against the ``steps_log`` keys the reference recorded, and a test-side
restatement of EvalLoop's rules applied to the golden episodes' cluster-step rows -- and to the CPU oracle's -- against the rows the
reference's EvalLoop produced (tests/golden/observations/eval_steps.npz, oracle/gen_eval_steps.py).

Exactness: np.sum / np.mean over fewer than 8 terms add left to right, so a sum in cluster-step order is numpy's for an env-step of
fewer than 8 cluster steps; longer ones are compared to 1e-12 relative.  The per-tick utilisation lists are reduced by the mean over
every entry of the env-step; the golden rows and the product carry each cluster step's sum of its entries, so that mean is exact
when the env-step is one cluster step of fewer than 8 ticks, and compared to 1e-12 relative otherwise."""
import os

import numpy as np
import pytest

from golden_io import Golden

FIXTURE = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'observations', 'eval_steps.npz'))
CASES = [str(c) for c in FIXTURE['cases']]
UTIL = {'mean_mounted_worker_utilisation_frac': 'util_mounted_sum', 'mean_cluster_worker_utilisation_frac': 'util_cluster_sum'}


def reduce_rows(rows, cs):
    """EvalLoop's rules (eval_loop.py:50-97) over cluster-step rows in the STEP_STATS layout (oracle.oracle / the goldens), env-step
    by env-step with `cs` cluster steps each: [env-steps, ENV_STEP_STATS_LEN]."""
    from ddls_b200.engine import ENV_STEP_STATS
    from oracle.oracle import SS
    out = np.zeros((len(cs), len(ENV_STEP_STATS)))
    ends = np.cumsum(cs)
    for e, (a, b) in enumerate(zip(ends - cs, ends)):
        r = rows[a:b]
        for j, k in enumerate(ENV_STEP_STATS):
            if k == 'step_start_time':
                out[e, j] = r[0, SS[k]]
            elif k in ('step_end_time', 'step_counter'):
                out[e, j] = r[-1, SS[k]]
            elif k in UTIL:
                s = 0.0
                for x in r[:, SS[UTIL[k]]]:
                    s += x
                out[e, j] = s / r[:, SS['num_ticks']].sum()
            else:
                s = 0.0
                for x in r[:, SS[k]]:
                    s += x
                out[e, j] = s / len(r) if 'mean' in k else s
    return out


def exact_mask(name):
    """[env-steps, ENV_STEP_STATS_LEN]: where the restatement must equal the fixture bit for bit (module docstring)."""
    from ddls_b200.engine import ENV_STEP_STATS
    cs, ticks = FIXTURE[name + '_cs'], FIXTURE[name + '_ticks']
    ends = np.cumsum(cs)
    one_short = np.array([c == 1 and ticks[e - 1] < 8 for c, e in zip(cs, ends)])
    return np.stack([one_short if k in UTIL else cs < 8 for k in ENV_STEP_STATS], axis=1)


def fixture_rows(name):
    """The fixture's rows with their columns in ENV_STEP_STATS order (the recorded steps_log order may differ)."""
    from ddls_b200.engine import ENV_STEP_STATS
    keys = [str(k) for k in FIXTURE[name + '_keys']]
    return FIXTURE[name + '_rows'][:, [keys.index(k) for k in ENV_STEP_STATS]]


def fixture_log(name, key):
    keys = [str(k) for k in FIXTURE[name + '_keys']]
    return FIXTURE[name + '_log'][:, keys.index(key)]


def check(name, got, blocked_at_end=None, exact=True):
    from ddls_b200.engine import ENV_STEP_STATS
    want = fixture_rows(name)
    ex = exact_mask(name) & exact
    got = got.copy()
    if blocked_at_end is not None:
        j = ENV_STEP_STATS.index('num_jobs_blocked')
        extra = got[-1, j] - want[-1, j]
        assert extra == blocked_at_end, (name, extra, blocked_at_end)
        got[-1, j] = want[-1, j]
    for j, k in enumerate(ENV_STEP_STATS):
        e = ex[:, j]
        np.testing.assert_array_equal(got[e, j], want[e, j], err_msg=f'{name} {k}')
        np.testing.assert_allclose(got[~e, j], want[~e, j], rtol=1e-12, atol=0, err_msg=f'{name} {k}')


def blocked_after_last_log(name):
    """Jobs still running when the episode ends: the cluster registers them blocked after RCE:1084 logged its last step, so the
    step's stats (which the goldens and the oracle record) count them and steps_log does not."""
    g = Golden(name)
    logged = fixture_log(name, 'num_jobs_blocked').sum()
    return float(g.d['es_num_jobs_blocked']) - logged


# steps_log's order when no job runs in the episode's first cluster step (its job was blocked): the throughput loop inserts the
# *_info_processed keys, each before the throughput that reads it (RCE:1064-1077)
NO_JOB_FIRST = ['step_counter', 'step_start_time', 'mean_num_mounted_workers', 'mean_num_mounted_channels', 'mean_compute_throughput',
                'mean_dep_throughput', 'mean_cluster_throughput', 'mean_demand_compute_throughput', 'mean_demand_dep_throughput',
                'mean_demand_total_throughput', 'mean_compute_overhead_frac', 'mean_communication_overhead_frac',
                'mean_mounted_worker_utilisation_frac', 'mean_cluster_worker_utilisation_frac', 'num_jobs_completed',
                'mean_num_jobs_running', 'num_jobs_arrived', 'num_jobs_blocked', 'step_end_time', 'step_time', 'compute_info_processed',
                'dep_info_processed', 'flow_info_processed', 'mean_flow_throughput', 'cluster_info_processed',
                'demand_compute_info_processed', 'demand_dep_info_processed', 'demand_total_info_processed', 'job_queue_length']


@pytest.mark.parametrize('name', CASES)
def test_key_set_and_order_are_the_references_steps_log(name):
    """The reference's steps_log keys, in insertion order.  When a job runs in the episode's first cluster step its outer loop adds
    the seven *_info_processed keys before step_end_time and the throughput loop adds mean_flow_throughput after step_time
    (RCE:306-338, 962-982, 1046-1084): ENV_STEP_STATS, the order the product reports.  When the first job is blocked the same 29
    keys come in NO_JOB_FIRST's order (3 of the 16 episodes)."""
    from ddls_b200.engine import ENV_STEP_STATS
    from oracle.oracle import SS
    keys = [str(k) for k in FIXTURE[name + '_keys']]
    job_first = Golden(name).d['step_stats'][0, SS['mean_num_jobs_running']] > 0
    assert keys == (ENV_STEP_STATS if job_first else NO_JOB_FIRST)
    assert sorted(NO_JOB_FIRST) == sorted(ENV_STEP_STATS)


@pytest.mark.parametrize('name', CASES)
def test_the_fixture_is_evalloops_own_and_its_slices_are_clean(name):
    """EvalLoop.run completed on every case under numpy 2 (no env-step's per-tick lists were ragged), and its prev_idx slice starts
    at the env-step's first cluster step at every env-step: every cluster step sets every steps_log key."""
    assert int(FIXTURE[name + '_evalloop']) == 1
    np.testing.assert_array_equal(FIXTURE[name + '_prev_idx'], FIXTURE[name + '_start'])
    assert FIXTURE[name + '_cs'].sum() == len(FIXTURE[name + '_log']) == len(FIXTURE[name + '_ticks'])
    assert len(FIXTURE[name + '_rewards']) == len(FIXTURE[name + '_actions']) == len(FIXTURE[name + '_cs'])


@pytest.mark.parametrize('name', CASES)
def test_evalloops_rules_on_the_golden_cluster_steps_give_the_fixture(name):
    g = Golden(name)
    cs = FIXTURE[name + '_cs']
    rows = g.d['step_stats']
    assert len(rows) == cs.sum(), name
    check(name, reduce_rows(rows, cs), blocked_after_last_log(name))


@pytest.mark.parametrize('name', CASES)
def test_evalloops_rules_on_the_oracles_cluster_steps_give_the_fixture(name, oracle_lib):
    """orc_run_scripted_rjpe_full_batch replaying the golden episode: the template of each env-step's action step, its mount row."""
    g = Golden(name)
    cs = FIXTURE[name + '_cs']
    first = np.cumsum(cs) - cs
    tid = g.d['step_tid'][first][None, :].astype(np.int32)
    mount = np.zeros(tid.shape, dtype=oracle_lib.MOUNT_DTYPE)
    m = g.d['step_mount'][first]
    for i, f in enumerate(oracle_lib.MOUNT_DTYPE.names):
        mount[f][0] = m[:, i]
    out = oracle_lib.run_scripted_episodes(g.templates, tid, mount, g.arrivals()[None], g.n_cluster_workers, max(g.n_models, 1),
                                           max_sim_time=g.max_sim_time, cs_cap=int(cs.sum()) + 4)
    np.testing.assert_array_equal(out['n_cluster_steps'][0], cs)
    rows = out['cluster_stats'][0, :int(out['n_cluster_stats'][0])]
    # the oracle restates the simulator in C; its rows may differ from the reference's in the last bits
    check(name, reduce_rows(rows, cs), blocked_after_last_log(name), exact=False)


def test_exactness_classes():
    """How many env-steps of the 16 episodes fall in each class (module docstring): all have fewer than 8 cluster steps; the
    per-tick means of the multi-cluster-step env-steps and of the long single ones are compared to 1e-12."""
    n = sum(len(FIXTURE[c + '_cs']) for c in CASES)
    short = sum(int((FIXTURE[c + '_cs'] < 8).sum()) for c in CASES)
    util_exact = sum(int(exact_mask(c)[:, 12].sum()) for c in CASES)
    assert (n, short, util_exact) == (153, 153, 106)
