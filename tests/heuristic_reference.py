"""Host restatement of ramp_env_agent_kernel (ddls_b200/csrc/ramp_env.cuh): the reference's heuristic agents
(ddls/environments/ramp_job_partitioning/agents/*.py) on an action mask, and the kernel's counter-based draw for Random.
tests/test_heuristic_agents_model.py pins it to the reference's own classes; the GPU tests pin the kernel to it."""
import math

import numpy as np

AGENTS = ('random', 'sipml', 'acceptable_jct', 'max_parallelism', 'min_parallelism', 'no_parallelism')
M64 = (1 << 64) - 1


def splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def random_index(seed, b, n_decided, n):
    """Index into valid_actions[1:] (n entries) the kernel draws for episode b after n_decided decisions."""
    key = (seed & M64) ^ ((0x9E3779B97F4A7C15 * n_decided) & M64)
    r = splitmix64(key ^ ((b * 0xD1342543DE82EF95) & M64))
    return ((r >> 32) * n) >> 32


def act(kind, mask, param=0, seq=None, macc=None, seed=0, b=0, n_decided=0):
    """One decision of agent `kind` on a boolean action mask (action_set = 0..len(mask)-1)."""
    valid = [a for a in range(len(mask)) if mask[a]]
    if kind == 'min_parallelism':                                  # min_parallelism.py:8-17
        return 2 if len(valid) > 2 else 1 if len(valid) == 2 else 0
    if kind == 'no_parallelism':                                   # no_parallelism.py:5-13
        return 1 if len(valid) > 1 else 0
    if len(valid) <= 1:
        return valid[0] if valid else 0
    if kind == 'random':                                           # random.py:8-16
        return valid[1 + random_index(seed, b, n_decided, len(valid) - 1)]
    if kind == 'sipml':                                            # sip_ml.py:13-25
        return min(param, valid[-1]) if param > 0 else valid[-1]
    if kind == 'acceptable_jct':                                   # acceptable_jct.py:21-44
        target = int(math.ceil(seq / macc))
        for action in valid:
            if action >= target:
                return action
        return valid[-1]
    if kind == 'max_parallelism':                                  # max_parallelism.py:5-13
        return valid[1:][-1]
    raise ValueError(kind)


def act_batch(kinds, params, mask, done, seq, macc, seed, n_decided):
    """act() for every episode: kinds [B] names, params [B], mask [B, A], done [B], seq / macc [B] of the queued job,
    n_decided [B] decisions taken before this one.  Finished episodes get 0."""
    out = np.zeros(len(kinds), dtype=np.int64)
    for b in range(len(kinds)):
        if not done[b]:
            out[b] = act(kinds[b], mask[b], int(params[b]), float(seq[b]), float(macc[b]), seed, b, int(n_decided[b]))
    return out
