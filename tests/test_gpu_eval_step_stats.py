"""-m gpu: EvalLoop's per-env-step ``step_stats`` (loops/eval_loop.py:44-100) from the step kernel.

* Both environments replay the 16 golden episodes with the reference's recorded actions; after every env-step ``env_step_stats()``
  is the row the reference's EvalLoop reported (tests/golden/observations/eval_steps.npz) -- bit for bit, or to 1e-12 relative for
  the keys _check_row names -- and the device environment's record of the whole
  episode (``record_steps`` / ``recorded_steps``) holds the same rows, actions and rewards.
* ``evaluate(step_stats=True)`` with each of the six heuristic agents and with DeviceGNNPolicy, on bench config 3 (prewarmed) and
  on the mix128_exp golden's cluster and models: its episode_stats are the default ``evaluate``'s on the same episodes, its record
  equals the host environment replaying the same actions, row for row, and sums to the episode statistics where the definitions
  coincide.
* The record's device memory returns to where it was."""
import gc

import numpy as np
import pytest

from test_eval_step_stats_model import CASES, FIXTURE, exact_mask, fixture_rows
from test_gpu_env_observation import replay_env
from test_gpu_episode_stats import set_job_counts

pytestmark = pytest.mark.gpu

EXACT = ('step_counter', 'step_start_time', 'step_end_time', 'step_time', 'num_jobs_completed', 'num_jobs_arrived', 'num_jobs_blocked',
         'job_queue_length')


def _check_row(name, e, got, where):
    from ddls_b200.engine import ENV_STEP_STATS
    want = fixture_rows(name)[e]
    ex = exact_mask(name)[e]
    for j, k in enumerate(ENV_STEP_STATS):
        g = float(got[k])
        # the counts and times are exact; every other key reduces per-cluster-step values that are themselves sums or np.means over
        # per-job / per-tick terms (numpy's pairwise order from 8 terms) or that scale the mounted job's partitioned sizes, which the
        # native expansion sums in its own order: those may differ from the reference's in the last bits
        if ex[j] and k in EXACT:
            assert g == want[j], (name, where, e, k, g, want[j])
        else:
            assert abs(g - want[j]) <= 1e-12 * abs(want[j]), (name, where, e, k, g, want[j])


@pytest.mark.parametrize('where', ['host', 'device'])
@pytest.mark.parametrize('name', CASES)
def test_every_env_step_row_is_evalloops(name, where):
    env, g, graphs, model = replay_env(name, where)
    env.reset()
    set_job_counts(env, [g])
    if where == 'device':
        env.record_steps(len(FIXTURE[name + '_cs']) + 2)
    actions = FIXTURE[name + '_actions']
    for e in range(len(actions)):
        assert not env.done[0], (name, e)
        _, r, _, _ = env.step(np.array([actions[e]], dtype=np.int64))
        assert r[0] == FIXTURE[name + '_rewards'][e], (name, e)
        _check_row(name, e, {k: v[0] for k, v in env.env_step_stats().items()}, where)
    assert env.done.all(), name
    if where == 'device':
        rec = env.recorded_steps()
        np.testing.assert_array_equal(rec['action'][0], actions)
        np.testing.assert_array_equal(rec['reward'][0], FIXTURE[name + '_rewards'])
        for e in range(len(actions)):
            _check_row(name, e, {k: v[0][e] for k, v in rec.items() if k not in ('action', 'reward')}, 'record')
    env.close()


def _config3(B=4096, J=8, seed=3, where='device'):
    from ddls_b200 import workload
    from ddls_b200.batched import BatchedRampJobPartitioningEnvironment, DeviceRampJobPartitioningEnvironment
    cfg = workload.CONFIGS['cfg3-resnet50-64w']
    graphs = [workload.make_graph(kind, **kw) for kind, kw in cfg['graphs']]
    kw = dict(n_episodes=B, jobs_per_episode=J, seed=seed)
    if where == 'host':
        return BatchedRampJobPartitioningEnvironment(tuple(cfg['shape']), graphs, **kw)
    return DeviceRampJobPartitioningEnvironment(tuple(cfg['shape']), graphs, prewarm=True, **kw)


def _mix128(B=512, J=6, seed=4, where='device'):
    from ddls_b200.batched import BatchedRampJobPartitioningEnvironment, DeviceRampJobPartitioningEnvironment
    from test_gpu_batched_env import SHAPES, _graphs
    graphs = _graphs()['mix128_exp']
    kw = dict(n_episodes=B, jobs_per_episode=J, seed=seed, interarrival=('exponential', 500.0), max_partitions_per_op=4)
    if where == 'host':
        return BatchedRampJobPartitioningEnvironment(SHAPES[128], graphs, **kw)
    return DeviceRampJobPartitioningEnvironment(SHAPES[128], graphs, prewarm=True, **kw)


def _assert_same_episode_stats(a, b):
    assert list(a) == list(b)
    for k, v in a.items():
        if isinstance(v, np.ndarray):
            np.testing.assert_array_equal(v, b[k], err_msg=k)
        else:
            assert len(v) == len(b[k]), k
            for x, y in zip(v, b[k]):
                np.testing.assert_array_equal(x, y, err_msg=k)


def _check_against_host(res, host):
    """The host environment replays the recorded actions; its env_step_stats() after every env-step is the record's row."""
    from ddls_b200.engine import ENV_STEP_STATS
    steps, es = res['step_stats'], res['episode_stats']
    assert list(steps) == ['action', 'reward'] + ENV_STEP_STATS
    B = host.B
    n = np.array([len(a) for a in steps['action']])
    assert (n >= 1).all() and (n <= host.J).all()
    host.reset()
    total = np.zeros(B)
    for t in range(int(n.max())):
        live = ~host.done
        np.testing.assert_array_equal(live, n > t)
        a = np.array([steps['action'][b][t] if n[b] > t else 0 for b in range(B)])
        _, r, _, _ = host.step(a)
        total += r
        rows = host.env_step_stats()
        idx = np.nonzero(live)[0]
        np.testing.assert_array_equal(r[idx], [steps['reward'][b][t] for b in idx])
        for k in ENV_STEP_STATS:
            np.testing.assert_array_equal(rows[k][idx], [steps[k][b][t] for b in idx], err_msg=f'{k} env-step {t}')
    assert host.done.all()
    np.testing.assert_array_equal(es['return'], total)
    # where steps_log and episode_stats count the same events: completions, and arrivals after the one reset() queues
    for b in range(B):
        assert steps['num_jobs_completed'][b].sum() == es['num_jobs_completed'][b]
        assert steps['num_jobs_arrived'][b].sum() == es['num_jobs_arrived'][b] - 1
        assert steps['num_jobs_blocked'][b].sum() <= es['num_jobs_blocked'][b]
        assert steps['step_end_time'][b][-1] == es['episode_end_time'][b]
        np.testing.assert_array_equal(steps['step_start_time'][b][1:], steps['step_end_time'][b][:-1])
    return int(n.sum())


@pytest.mark.parametrize('workload', ['cfg3', 'mix128_exp'])
def test_evaluate_step_stats_of_every_agent_equal_the_host_replay(workload):
    """Three environments with the same seed draw the same episodes at every reset: ``evaluate(step_stats=True)`` on one, the
    default ``evaluate`` on its twin -- whose result must be the first one's episode_stats, unchanged by the record -- and the
    host environment replaying the recorded actions."""
    from ddls_b200.agents import AGENTS, DeviceHeuristicAgents, evaluate
    from ddls_b200.policy import DeviceGNNPolicy
    make = _config3 if workload == 'cfg3' else _mix128
    dev, twin, host = make(), make(), make(where='host')
    A = dev.max_partitions_per_op + 1
    gnn = DeviceGNNPolicy([m.graph for m in dev.models], A, seed=2)
    actors = [(DeviceHeuristicAgents(dev, kind), DeviceHeuristicAgents(twin, kind)) for kind in AGENTS] + [(gnn, gnn)]
    for actor, actor_twin in actors:
        res = evaluate(dev, actor, seed=5, step_stats=True)
        assert set(res) == {'step_stats', 'episode_stats'}
        plain = evaluate(twin, actor_twin, seed=5)
        _assert_same_episode_stats(res['episode_stats'], plain)
        _check_against_host(res, host)
    gnn.close()
    for x in (dev, twin, host):
        x.close()


def test_the_record_returns_its_device_memory():
    from ddls_b200 import engine
    from ddls_b200.agents import DeviceHeuristicAgents, evaluate
    dev = _mix128(B=256, J=4)
    agents = DeviceHeuristicAgents(dev, 'sipml')
    evaluate(dev, agents)                               # the engine's own buffers grow on first use
    gc.collect()
    before = engine.device_bytes()
    dev.record_steps(64)
    assert engine.device_bytes()[0] > before[0]
    dev.record_steps(0)
    assert engine.device_bytes() == before
    evaluate(dev, agents, step_stats=True)             # evaluate frees its record at the end
    assert engine.device_bytes() == before
    dev.record_steps(16)
    dev.close()                                         # and close() frees one left behind
    gc.collect()
    assert engine.device_bytes()[0] < before[0]
