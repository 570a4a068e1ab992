"""-m gpu: the reference's heuristic agents as a kernel (ramp_env_agent_kernel, ddls_b200.agents): they must take the reference's
own decisions on its recorded SiPML and AcceptableJCT episodes and reproduce its episode statistics, equal the host restatement
(tests/heuristic_reference.py) decision for decision on random masks, and drive ``evaluate()`` to the end of every episode."""
import numpy as np
import pytest

import heuristic_reference as H
from test_gpu_episode_stats import check_against_golden, golden_env, set_job_counts

pytestmark = pytest.mark.gpu

# golden -> (agent, SiPML's max_partitions_per_op = the environment's, as oracle/gen_golden.py recorded them)
GOLDEN_AGENTS = {'chain8_maxtime': ('sipml', 4), 'residual8_deg4': ('sipml', 4), 'res16_flood': ('sipml', 4),
                 'residual32_deg16': ('sipml', 16), 'bert256_shard': ('sipml', 8), 'resnet64_deg16_full': ('sipml', 16),
                 'resnet64_deg8_full': ('sipml', 8), 'resnet64_deg4_full': ('sipml', 4), 'resnet64_deg2_full': ('sipml', 2),
                 'tfm32_acceptable': ('acceptable_jct', 16)}


def _device_array(ptr, n, typestr):
    """A torch view of n elements of a raw device buffer of the environment (the engine stream must be idle)."""
    import torch

    class _Buf:
        __cuda_array_interface__ = {'shape': (n,), 'typestr': typestr, 'data': (ptr, False), 'version': 3}
    return torch.as_tensor(_Buf(), device='cuda')


@pytest.mark.parametrize('name', sorted(GOLDEN_AGENTS))
def test_device_agents_take_the_reference_decisions_on_its_golden_episodes(name):
    from ddls_b200.agents import DeviceHeuristicAgents
    kind, mpo = GOLDEN_AGENTS[name]
    env, (g,), (dec,) = golden_env([name], 'device', max_partitions_per_op=mpo)
    agents = DeviceHeuristicAgents(env, kind, mpo)
    env.reset()
    set_job_counts(env, [g])
    tid_buf = _device_array(env.device_buffers()['template_id'], 1, '<i4')
    for e, (s, want) in enumerate(dec):
        assert not env.done[0], (name, e)
        agents.act(seed=0)
        env.step(None)
        tid = int(tid_buf.cpu()[0])
        degree_of = {t: key[1] for key, t in env._template_cache.items()}
        got = degree_of[tid] if tid >= 0 else 0
        ref_tid = int(g.d['step_tid'][s])
        assert got == (g.templates[ref_tid].degree if ref_tid >= 0 else 0), (name, e, got)
    assert env.done.all()
    check_against_golden(env.episode_stats(), 0, g, name)
    env.close()


def _read_actions(env):
    """The actions the device holds (ramp_env_read_state)."""
    import ctypes as C
    from ddls_b200 import engine as _engine
    L = env.eng._L
    L.ramp_env_read_state.restype = C.c_int
    L.ramp_env_read_state.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    got = np.zeros(env.B, dtype=np.int32)
    _engine._check(L.ramp_env_read_state(env.eng._h, None, got.ctypes.data, None))
    return got


def _agent_env(B=4096, J=6, seed=0, apply_action_mask=False):
    from ddls_b200 import synth
    from ddls_b200.batched import DeviceRampJobPartitioningEnvironment
    graphs = [synth.resnet_like_graph(n_blocks=2, stem=2, name='res2', seed=7, body_per_block=3), synth.chain_graph(6, 'chain6')]
    return DeviceRampJobPartitioningEnvironment((4, 4, 4), graphs, n_episodes=B, jobs_per_episode=J, seed=seed,
                                                interarrival=('exponential', 400.0), apply_action_mask=apply_action_mask, prewarm=True)


def test_all_six_agents_equal_the_host_restatement_on_random_masks():
    """4,096 episodes, the six agents side by side (SiPML at None and at several maxima), masks and done flags drawn at random
    and written into the environment's device buffers before every decision; a quarter of the max acceptable JCTs divide the
    sequential time exactly."""
    from ddls_b200.agents import AGENTS, DeviceHeuristicAgents
    import torch
    from ddls_b200.engine import EP
    env = _agent_env()
    B, A = env.B, env.max_partitions_per_op + 1
    kinds = [AGENTS[b % 6] for b in range(B)]
    params = np.array([[0, 1, 2, 4, 8, 16, 100][(b // 6) % 7] for b in range(B)])
    agents = DeviceHeuristicAgents(env, kinds, params)
    env.reset()
    rng = np.random.default_rng(3)
    bufs = env.device_buffers()
    mask_buf, done_buf = _device_array(bufs['action_mask'], B * A, '|u1'), _device_array(bufs['done'], B, '|u1')
    seq = np.array([m.seq_time for m in env.models])
    n_exact = n_quirk = 0
    for t in range(env.J):
        true_done = env.read()[2]
        mask = rng.random((B, A)) < rng.uniform(0.1, 0.9, size=(B, 1))
        mask[:, 0] = rng.random(B) < 0.9
        done = true_done | (rng.random(B) < 0.1)
        mask_buf.copy_(torch.from_numpy(mask.astype(np.uint8).reshape(-1)))
        done_buf.copy_(torch.from_numpy(done.astype(np.uint8)))
        torch.cuda.synchronize()
        q = env.eng.episode_state()[:, EP['queued_job']].astype(np.int64)
        qq = np.clip(q, 0, env.J - 1)
        m = env.model_of[np.arange(B), qq]
        macc = env.frac[np.arange(B), qq] * seq[m]
        n_decided = env.decisions()
        seed = 1000 + t
        agents.act(seed)
        got = _read_actions(env)
        want = H.act_batch(kinds, params, mask, done, seq[m], macc, seed, n_decided)
        np.testing.assert_array_equal(got, want)
        assert (got[done] == 0).all()
        ratio = seq[m] / macc
        n_exact += int(np.sum((ratio == np.ceil(ratio)) & ~done))
        n_quirk += int(sum(1 for b in range(B) if kinds[b] == 'min_parallelism' and not done[b] and mask[b].sum() > 2 and not mask[b, 2]))
        done_buf.copy_(torch.from_numpy(true_done.astype(np.uint8)))
        torch.cuda.synchronize()
        env.step_device()
    assert n_quirk > 0 and n_exact > 0
    env.close()


def test_random_reaches_every_valid_nonzero_action_and_never_0():
    from ddls_b200.agents import DeviceHeuristicAgents
    import torch
    env = _agent_env(B=2048)
    B, A = env.B, env.max_partitions_per_op + 1
    agents = DeviceHeuristicAgents(env, 'random')
    env.reset()
    bufs = env.device_buffers()
    rng = np.random.default_rng(0)
    patterns = [rng.random(A) < 0.5 for _ in range(4)] + [np.ones(A, dtype=bool)]
    for p in patterns:
        p[0] = True
        if p.sum() < 2:
            p[1] = True
        _device_array(bufs['action_mask'], B * A, '|u1').copy_(torch.from_numpy(np.tile(p.astype(np.uint8), B)))
        _device_array(bufs['done'], B, '|u1').zero_()
        torch.cuda.synchronize()
        seen = set()
        for seed in range(4):
            agents.act(seed)
            got = _read_actions(env)
            want = H.act_batch(['random'] * B, np.zeros(B), np.tile(p, (B, 1)), np.zeros(B, dtype=bool), np.ones(B), np.ones(B), seed,
                               np.zeros(B, dtype=np.int64))
            np.testing.assert_array_equal(got, want)
            seen |= set(got.tolist())
        assert seen == set(np.nonzero(p)[0][1:].tolist()), (p, seen)
    env.close()


@pytest.mark.parametrize('actor', ['agents', 'gnn'])
def test_evaluate_finishes_every_episode_and_its_return_sums_the_rewards(actor):
    from ddls_b200.agents import AGENTS, DeviceHeuristicAgents, evaluate
    from ddls_b200.policy import DeviceGNNPolicy
    envs = [_agent_env(B=1024, J=5, seed=9, apply_action_mask=True) for _ in range(2)]
    B, A = envs[0].B, envs[0].max_partitions_per_op + 1
    if actor == 'agents':
        kinds = [AGENTS[b % 6] for b in range(B)]
        actors = [DeviceHeuristicAgents(e, kinds, 4) for e in envs]
    else:
        actors = [DeviceGNNPolicy([m.graph for m in envs[0].models], A, seed=2) for _ in envs]
    es = evaluate(envs[0], actors[0], seed=7)
    assert es['done'].all() and (es['num_jobs_arrived'] == 5).all()
    assert (es['num_jobs_completed'] + es['num_jobs_blocked'] == 5).all()
    # the twin: the same decisions one env-step at a time, the rewards summed on the host
    twin, total = envs[1], np.zeros(B)
    twin.reset()
    for t in range(twin.J):
        if actor == 'agents':
            actors[1].act(7)
        else:
            actors[1].act(twin, seed=7 + t)
        _, r, d, _ = twin.step(None)
        total += r
    assert d.all()
    np.testing.assert_array_equal(es['return'], total)
    es2 = twin.episode_stats()
    for k in ('num_jobs_completed', 'episode_time', 'mean_cluster_throughput'):
        np.testing.assert_array_equal(es[k], es2[k])
    for x in envs:
        x.close()
