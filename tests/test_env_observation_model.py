"""CPU: what the batched environments observe of a job, against the unmodified reference's own episodes.  The 16 golden episodes'
arrival rows (tests/golden/<case>.npz) and the observations the reference's RampJobPartitioningEnvironment handed its agent at
every env-step of them (tests/golden/observations/env_obs.npz, oracle/gen_env_obs.py) pin the job totals on the arrival rows, the jobs_params
normalisers and the host environment's first observation; tests/test_gpu_env_observation.py replays every step on the GPU."""
import os

import numpy as np
import pytest

from golden_io import GOLDEN_DIR, Golden
from test_gpu_batched_env import SHAPES, _decisions, _graphs

OBS = np.load(os.path.join(GOLDEN_DIR, 'observations', 'env_obs.npz'))
CASES = [str(c) for c in OBS['cases']]
DETERMINISTIC = ('job_total_num_ops', 'job_total_num_deps', 'job_sequential_completion_times', 'job_total_op_memory_costs',
                 'job_total_dep_sizes', 'job_num_training_steps')
DYNAMIC = list(range(9)) + [15, 16]            # graph_features indices of graph_features_dynamic


def recorded_jobs_params(name):
    """The reference's jobs_generator.jobs_params of the case, as the mapping the environments take (min_<key> / max_<key>)."""
    from ddls_b200.observation import PARAM_KEYS
    t = OBS[name + '_jobs_params']
    out = {}
    for i, k in enumerate(PARAM_KEYS):
        out['min_' + k], out['max_' + k] = float(t[i, 0]), float(t[i, 1])
    return out


def model_of_arrivals(name, graphs):
    """Index into `graphs` of the model of every recorded arrival: the one whose job totals are the row's, bit for bit."""
    from ddls_b200.template_builder import original_job_totals
    totals = [original_job_totals(g) for g in graphs]
    out = []
    for row in Golden(name).d['arrivals']:
        m = [k for k, t in enumerate(totals) if t == (row[1], row[2])]
        assert len(m) == 1, (name, row, totals)
        out.append(m[0])
    return np.array(out, dtype=np.int64)


def test_fixture_covers_every_golden_episode():
    assert sorted(CASES) == sorted(f[:-4] for f in os.listdir(GOLDEN_DIR) if f.endswith('.npz'))
    # occupancy bit sets of 2 and 4 words with jobs running (bert256_shard's degree-8 blocks take one server per communication
    # group: servers 0, 32, ..., 224)
    for n in ('mix128_exp', 'bert256_shard'):
        assert Golden(n).n_cluster_workers > 64 and OBS[n + '_n_mounted'].max() > 0 and OBS[n + '_n_running'].max() > 1


@pytest.mark.parametrize('name', CASES)
def test_fixture_is_the_golden_episode(name):
    """The re-run is the golden's episode: the same arrival rows, the same degree at every env-step that placed a job (the
    golden records what was placed, so an action whose placement failed shows as 0 there), one observation per decision and the
    queued job of env-step e is job e."""
    g = Golden(name)
    np.testing.assert_array_equal(OBS[name + '_arrivals'], g.d['arrivals'])
    actions, placed = OBS[name + '_actions'], np.array([a for (_, a) in _decisions(g)])
    assert len(actions) == len(placed)
    np.testing.assert_array_equal(actions[placed > 0], placed[placed > 0])
    K = len(actions)
    np.testing.assert_array_equal(OBS[name + '_step'], np.arange(K))
    np.testing.assert_array_equal(OBS[name + '_job_idx'], np.arange(K))
    A = int(OBS[name + '_max_partitions_per_op']) + 1
    assert OBS[name + '_graph_features'].shape == (K, 17 + A) and OBS[name + '_action_mask'].shape == (K, A)
    np.testing.assert_array_equal(OBS[name + '_graph_features'][:, 17:], OBS[name + '_action_mask'])


@pytest.mark.parametrize('name', CASES)
def test_original_job_totals_are_the_recorded_arrival_rows(name):
    """Every model's (job_total_op_memory_cost, job_total_dep_size) is what the reference put on its arrival rows, bit for bit --
    the dep total sums each edge's source activation (not activation + parameters) in the job graph's edge order -- and every
    model of the case arrived at least once."""
    graphs = _graphs()[name]
    assert sorted(set(model_of_arrivals(name, graphs).tolist())) == list(range(len(graphs)))


@pytest.mark.parametrize('name', CASES)
def test_default_jobs_params_are_the_references_deterministic_keys(name):
    """jobs_params(models, ...) gives the reference's min / max of every key that does not depend on the sampled job pool:
    3 * max deps, max dep size times the edges of a fully connected largest job, the plain min / max of the rest."""
    from ddls_b200.batched import _Model, jobs_params
    from ddls_b200.observation import PARAM_KEYS
    got = jobs_params([_Model(g, 0.01, 50) for g in _graphs()[name]], (0.1, 1.0), 50)
    want = OBS[name + '_jobs_params']
    for i, k in enumerate(PARAM_KEYS):
        if k in DETERMINISTIC:
            assert got[i] == (want[i, 0], want[i, 1]), (name, k, got[i], want[i])


def _host_env(name, monkeypatch, **kw):
    """The host environment on one episode of the case, its engine answered by the CPU oracle (tests/fake_engine.py)."""
    from fake_engine import FakeEngine
    from ddls_b200 import batched
    monkeypatch.setattr(batched._engine, 'RampEngine', FakeEngine)
    g = Golden(name)
    graphs = _graphs()[name]
    model = model_of_arrivals(name, graphs)
    J = len(model)
    frac = np.ones(J)
    frac[OBS[name + '_job_idx']] = OBS[name + '_frac']
    script = {'model': model[None], 'gap': g.d['arrivals'][None, :, 0], 'frac': frac[None]}
    return batched.BatchedRampJobPartitioningEnvironment(
        SHAPES[g.n_cluster_workers], graphs, n_episodes=1, jobs_per_episode=J, max_partitions_per_op=int(OBS[name + '_max_partitions_per_op']),
        max_simulation_run_time=g.max_sim_time, script=script, machine_epsilon=float(OBS[name + '_machine_epsilon']), **kw)


@pytest.mark.parametrize('name', CASES)
def test_jobs_params_override_and_the_first_observation(name, monkeypatch):
    """``jobs_params=`` takes the reference's table as is: all 8 keys are then the reference's, and the observation after reset is
    the reference's, bit for bit (graph_features_dynamic, action mask, queued model)."""
    from ddls_b200.observation import PARAM_KEYS
    env = _host_env(name, monkeypatch, jobs_params=recorded_jobs_params(name))
    want = OBS[name + '_jobs_params']
    assert env.jobs_params() == [(want[i, 0], want[i, 1]) for i in range(len(PARAM_KEYS))]
    obs = env.reset()
    gf = OBS[name + '_graph_features'][0]
    assert obs['graph_features_dynamic'].dtype == np.float32
    np.testing.assert_array_equal(obs['graph_features_dynamic'][0], gf[DYNAMIC])
    np.testing.assert_array_equal(obs['action_mask'][0], OBS[name + '_action_mask'][0])
    assert obs['model'][0] == model_of_arrivals(name, _graphs()[name])[0]


def test_a_negative_normalised_feature_gets_machine_epsilon(monkeypatch):
    """A frac below the pool's minimum makes features 3 and 4 negative: the reference's encoder adds machine_epsilon to them
    (observation.py:441-444) in double before the float32 observation."""
    name = 'chain8_busy'
    jp = recorded_jobs_params(name)
    lo = jp['min_max_acceptable_job_completion_time_fracs']
    env = _host_env(name, monkeypatch, jobs_params=jp)
    env.script['frac'] = np.full_like(env.script['frac'], lo - 0.05)
    obs = env.reset()
    fr = lo - 0.05
    hi = jp['max_max_acceptable_job_completion_time_fracs']
    x4 = (fr - lo) / (hi - lo)
    assert x4 < 0
    assert obs['graph_features_dynamic'][0, 4] == np.float32(x4 + 1e-7) != np.float32(x4)
    seq = env.models[0].seq_time
    lo3, hi3 = jp['min_max_acceptable_job_completion_times'], jp['max_max_acceptable_job_completion_times']
    assert obs['graph_features_dynamic'][0, 3] == np.float32((fr * seq - lo3) / (hi3 - lo3) + 1e-7)
    assert obs['graph_features_dynamic'][0, 5] == np.float32(fr)
