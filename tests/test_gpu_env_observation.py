"""-m gpu: both batched environments' observations against the ones the unmodified reference's RampJobPartitioningEnvironment handed
its agent, step by step (tests/golden/observations/env_obs.npz, oracle/gen_env_obs.py).  Each of the 16 golden episodes is replayed with its
recorded fracs and actions and the reference's jobs_params table; the max acceptable JCT is the environment's own frac * seq_time.
One environment holds one jobs_params table and every case has its own (the reference takes it over the case's job pool), so each
case runs as an environment of its own."""
import numpy as np
import pytest

from golden_io import Golden
from test_env_observation_model import CASES, DYNAMIC, OBS, model_of_arrivals, recorded_jobs_params
from test_gpu_batched_env import SHAPES, _graphs
from test_gpu_episode_stats import set_job_counts

pytestmark = pytest.mark.gpu


def replay_env(name, where, jobs_params=True, B=1):
    """The environment replaying case `name` in B identical episodes: recorded models, gaps and fracs, the reference's jobs_params
    (unless jobs_params=False) and no max-acceptable-JCT override."""
    from ddls_b200 import batched
    cls = batched.BatchedRampJobPartitioningEnvironment if where == 'host' else batched.DeviceRampJobPartitioningEnvironment
    g = Golden(name)
    graphs = _graphs()[name]
    model = model_of_arrivals(name, graphs)
    J = len(model)
    frac = np.ones(J)
    frac[OBS[name + '_job_idx']] = OBS[name + '_frac']
    script = {'model': np.tile(model, (B, 1)), 'gap': np.tile(g.d['arrivals'][:, 0], (B, 1)), 'frac': np.tile(frac, (B, 1))}
    env = cls(SHAPES[g.n_cluster_workers], graphs, n_episodes=B, jobs_per_episode=J, max_partitions_per_op=int(OBS[name + '_max_partitions_per_op']),
              max_simulation_run_time=g.max_sim_time, script=script, machine_epsilon=float(OBS[name + '_machine_epsilon']),
              jobs_params=recorded_jobs_params(name) if jobs_params else None)
    return env, g, graphs, model


def replay(name, where, jobs_params=True):
    """Yields (env, env-step e, observation) for every recorded observation of the replay, then takes the recorded action."""
    env, g, graphs, model = replay_env(name, where, jobs_params)
    obs = env.reset()
    set_job_counts(env, [g])
    actions = OBS[name + '_actions']
    for e in range(len(actions)):
        assert not env.done[0], (name, e)
        yield env, e, obs
        obs = env.step(np.array([actions[e]], dtype=np.int64))[0]
    assert env.done.all(), name


@pytest.mark.parametrize('where', ['host', 'device'])
@pytest.mark.parametrize('name', CASES)
def test_every_observation_is_the_references(name, where):
    """At every env-step: graph_features_dynamic is the reference's graph_features[0..8, 15, 16] bit for bit, the action mask and
    queued job are the reference's, and the policy's per-model statistics are graph_features[9:15]; at the end the max acceptable
    JCT of every completed and blocked job -- frac * seq_time of the job as the environment mounted it -- is the reference's to
    1e-13 relative."""
    from ddls_b200.observation import static_observation
    graphs = _graphs()[name]
    model = model_of_arrivals(name, graphs)
    static = [static_observation(gr)['graph_static'] for gr in graphs]
    gf, mask = OBS[name + '_graph_features'], OBS[name + '_action_mask']
    env = None
    for env, e, obs in replay(name, where):
        q = int(OBS[name + '_job_idx'][e])
        dyn = obs['graph_features_dynamic'][0]
        assert dyn.dtype == np.float32
        bad = np.flatnonzero(dyn != gf[e, DYNAMIC])
        assert not len(bad), (name, e, [DYNAMIC[i] for i in bad], dyn[bad], gf[e, DYNAMIC][bad])
        np.testing.assert_array_equal(obs['action_mask'][0], mask[e], err_msg=f'{name} step {e}')
        assert obs['model'][0] == model[q], (name, e)
        np.testing.assert_array_equal(static[model[q]], gf[e, 9:15], err_msg=f'{name} step {e}')
    # a mounted job's sequential time is its lowered job's: the native expansion sums the sub-ops in its own order, not the
    # reference's node order, so frac * seq_time may differ in the last bits (observed: at most 1.1e-15 relative)
    es = env.episode_stats()
    g = Golden(name)
    np.testing.assert_array_equal(es['completed_job_idxs'][0], g.d['es_completed_job_idxs'])
    np.testing.assert_allclose(es['jobs_completed_max_acceptable_job_completion_time'][0], g.d['es_jobs_completed_max_acceptable_job_completion_time'],
                               rtol=1e-13, atol=0)
    order = np.argsort(g.d['es_blocked_job_idxs'], kind='stable')
    ours = np.argsort(es['blocked_job_idxs'][0], kind='stable')
    np.testing.assert_array_equal(es['blocked_job_idxs'][0][ours], g.d['es_blocked_job_idxs'][order])
    np.testing.assert_allclose(es['jobs_blocked_max_acceptable_job_completion_time'][0][ours],
                               g.d['es_jobs_blocked_max_acceptable_job_completion_time'][order], rtol=1e-13, atol=0)
    env.close()


@pytest.mark.parametrize('where', ['host', 'device'])
@pytest.mark.parametrize('name', CASES)
def test_without_the_references_table_the_pool_independent_features_still_match(name, where):
    """With the environment's own jobs_params only the two max-acceptable-JCT features (3, 4), which the reference normalises over
    its sampled job pool, may differ: features 0-2 and 5-10 are the reference's bit for bit."""
    keep = [0, 1, 2, 5, 6, 7, 8, 9, 10]
    gf = OBS[name + '_graph_features']
    env = None
    for env, e, obs in replay(name, where, jobs_params=False):
        dyn = obs['graph_features_dynamic'][0]
        np.testing.assert_array_equal(dyn[keep], gf[e, DYNAMIC][keep], err_msg=f'{name} step {e}')
    env.close()


@pytest.mark.parametrize('where', ['host', 'device'])
def test_a_frac_below_the_pools_minimum_gets_machine_epsilon(where):
    """Features 3 and 4 of a job whose frac lies below the pool's minimum are negative: both environments add machine_epsilon to
    them in double before the float32 observation, as the reference's encoder does (observation.py:441-444)."""
    name = 'chain8_busy'
    env, g, graphs, model = replay_env(name, where, B=2)
    jp = recorded_jobs_params(name)
    lo, hi = jp['min_max_acceptable_job_completion_time_fracs'], jp['max_max_acceptable_job_completion_time_fracs']
    lo3, hi3 = jp['min_max_acceptable_job_completion_times'], jp['max_max_acceptable_job_completion_times']
    fr = lo - 0.05
    env.script['frac'][1, :] = fr                         # episode 1: every job below the pool's minimum; episode 0 as recorded
    obs = env.reset()
    dyn = obs['graph_features_dynamic']
    seq = env.models[0].seq_time
    x3, x4 = (fr * seq - lo3) / (hi3 - lo3), (fr - lo) / (hi - lo)
    assert x3 < 0 and x4 < 0
    assert dyn[1, 3] == np.float32(x3 + 1e-7) and dyn[1, 4] == np.float32(x4 + 1e-7) and np.float32(x4 + 1e-7) != np.float32(x4)
    assert dyn[1, 5] == np.float32(fr)
    np.testing.assert_array_equal(dyn[0], OBS[name + '_graph_features'][0, DYNAMIC])
    env.close()


@pytest.mark.parametrize('name', ['chain8_busy', 'mixed16', 'tfm32_acceptable', 'residual32_deg16'])
def test_device_policy_on_the_replay_equals_the_reference_policy_on_the_recorded_observation(name):
    """DeviceGNNPolicy.act reads the device environment's own observation; its logits and values are within 2e-5 of the float32
    torch restatement of GNNPolicy (tests/gnn_reference.py) evaluated on the observation the reference recorded at that step
    (|A| = 9 for max_partitions_per_op 8, 17 for 16)."""
    import torch
    from ddls_b200 import policy as P
    from test_gpu_policy import ATOL, RTOL, _torch_policy
    graphs = _graphs()[name]
    A = int(OBS[name + '_max_partitions_per_op']) + 1
    cfg = dict(P.DEFAULT_CONFIG)
    sd = P.random_state_dict(cfg, A, seed=7)
    pol = P.DeviceGNNPolicy(graphs, A, cfg, sd)
    ref = _torch_policy(cfg, A, sd)
    model = model_of_arrivals(name, graphs)
    with torch.no_grad():
        emb = np.stack([ref.embed(torch.from_numpy(st['node_features']), torch.from_numpy(st['edge_features']),
                                  torch.from_numpy(st['edges_src'].astype(np.int64)), torch.from_numpy(st['edges_dst'].astype(np.int64))).numpy()
                        for st in pol.static])
    gf, mask = OBS[name + '_graph_features'], OBS[name + '_action_mask']
    n = 0
    for env, e, obs in replay(name, 'device'):
        pol.act(env)
        got = pol.read(env)
        m = model[int(OBS[name + '_job_idx'][e])]
        with torch.no_grad():
            wl, wv = ref(torch.from_numpy(emb[m:m + 1]), torch.from_numpy(gf[e:e + 1].astype(np.float32)),
                         torch.from_numpy(mask[e:e + 1].astype(np.float32)))
        valid = mask[e].astype(bool)
        np.testing.assert_allclose(got['logits'][0][valid], wl.numpy()[0][valid], atol=ATOL, rtol=RTOL, err_msg=f'{name} step {e}')
        np.testing.assert_allclose(got['value'], wv.numpy(), atol=ATOL, rtol=RTOL, err_msg=f'{name} step {e}')
        n += 1
    assert n == len(OBS[name + '_actions'])
    pol.close()
