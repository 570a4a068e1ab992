"""CPU: the host restatement of the device heuristic agents (tests/heuristic_reference.py, what ramp_env_agent_kernel is tested
against) equals the reference's own agent classes (ddls/environments/ramp_job_partitioning/agents/*.py) on random observations:
decision for decision for the deterministic agents, and the same set of reachable actions for Random.  Skips where the
reference is neither checked out nor staged under oracle/_ref."""
import importlib.util
import os
from types import SimpleNamespace

import numpy as np
import pytest

import heuristic_reference as H


def _reference_agents():
    from oracle import ref_shim
    if not ref_shim.reference_available():
        pytest.skip('the reference is not available')
    d = os.path.join(ref_shim.REFERENCE_ROOT, 'ddls', 'environments', 'ramp_job_partitioning', 'agents')
    mods = {}
    for name in ('random', 'sip_ml', 'acceptable_jct', 'max_parallelism', 'min_parallelism', 'no_parallelism'):
        spec = importlib.util.spec_from_file_location(f'_ref_agent_{name}', os.path.join(d, name + '.py'))
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        mods[name] = m
    return mods


def _observations(n, seed):
    """Random masks over action sets of 2..17 actions (0 masked in some), with the queued job's sequential time and max
    acceptable JCT; one in four ratios is an exact integer."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        A = int(rng.integers(2, 18))
        mask = rng.random(A) < rng.uniform(0.1, 0.9)
        mask[0] = rng.random() < 0.9
        seq = float(rng.uniform(10.0, 5000.0))
        macc = seq / int(rng.integers(1, 20)) if k % 4 == 0 else seq * float(rng.uniform(0.02, 1.5))
        out.append((np.arange(A, dtype=np.int16), mask, seq, macc))
    return out


def _job(seq, macc):
    return SimpleNamespace(details={'job_sequential_completion_time': {'A100': seq}, 'max_acceptable_job_completion_time': {'A100': macc}})


@pytest.mark.parametrize('kind', ['sipml', 'acceptable_jct', 'max_parallelism', 'min_parallelism', 'no_parallelism'])
def test_deterministic_agents_match_the_reference(kind):
    R = _reference_agents()
    n_checked = 0
    for action_set, mask, seq, macc in _observations(4000, 1):
        if not mask.any():
            continue
        obs = {'action_set': action_set, 'action_mask': mask.astype(np.int8)}
        if kind == 'sipml':
            for param in (None, 1, 2, 3, 4, 8, 16, 100):
                want = R['sip_ml'].SiPML(max_partitions_per_op=param).compute_action(obs)
                assert H.act(kind, mask, param=0 if param is None else param) == want, (mask, param)
        elif kind == 'acceptable_jct':
            want = R['acceptable_jct'].AcceptableJCT().compute_action(obs, job_to_place=_job(seq, macc))
            assert H.act(kind, mask, seq=seq, macc=macc) == want, (mask, seq, macc)
        else:
            cls = {'max_parallelism': R['max_parallelism'].MaxParallelism, 'min_parallelism': R['min_parallelism'].MinParallelism,
                   'no_parallelism': R['no_parallelism'].NoParallelism}[kind]
            assert H.act(kind, mask) == cls().compute_action(obs), mask
        n_checked += 1
    assert n_checked > 3500


def test_min_parallelism_returns_2_even_when_2_is_masked():
    R = _reference_agents()
    mask = np.array([1, 1, 0, 0, 1], dtype=bool)
    obs = {'action_set': np.arange(5, dtype=np.int16), 'action_mask': mask.astype(np.int8)}
    assert R['min_parallelism'].MinParallelism().compute_action(obs) == 2 == H.act('min_parallelism', mask)


def test_random_reaches_the_same_actions_as_the_reference():
    R = _reference_agents()
    np.random.seed(0)
    agent = R['random'].Random()
    for action_set, mask, _, _ in _observations(300, 2):
        if not mask.any():
            continue
        obs = {'action_set': action_set, 'action_mask': mask.astype(np.int8)}
        ref = {int(agent.compute_action(obs)) for _ in range(400)}
        ours = {H.act('random', mask, seed=s, b=b, n_decided=d) for s in range(4) for b in range(10) for d in range(10)}
        assert ours == ref, (mask, ours, ref)
