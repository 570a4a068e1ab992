"""The reference's heuristic partitioning agents on the device, and a batched EvalLoop.

``DeviceHeuristicAgents`` binds ``ramp_env_set_agents`` / ``ramp_env_agent_act`` (include/ramp_b200.h; the rules are in
ddls_b200/csrc/ramp_env.cuh): ``Random``, ``SiPML``, ``AcceptableJCT``, ``MaxParallelism``, ``MinParallelism`` and
``NoParallelism`` (ddls/environments/ramp_job_partitioning/agents/*.py), one per episode of a
``DeviceRampJobPartitioningEnvironment``, deciding from the action mask and queued job the environment left on the device.

``evaluate`` is EvalLoop (ddls/loops/eval_loop.py:26-134, "use for validating heuristics") for all the episodes at once: reset,
then actor -> ``step_device()`` until every episode is done, then the episodes' ``episode_stats`` and, on request, EvalLoop's
per-env-step ``step_stats``.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence, Union

import numpy as np

from . import engine as _engine

AGENTS = ('random', 'sipml', 'acceptable_jct', 'max_parallelism', 'min_parallelism', 'no_parallelism')   # RAMP_AGENT_* order
AGENT = {k: i for i, k in enumerate(AGENTS)}


class DeviceHeuristicAgents:
    def __init__(self, env, kinds: Union[str, Sequence[str]], params: Union[None, int, Sequence[int]] = None):
        """env: a DeviceRampJobPartitioningEnvironment.  kinds: one agent name (``AGENTS``) for every episode, or one per episode.
        params: SiPML's max_partitions_per_op (None or <= 0: no maximum), one for all or one per episode; the other agents
        ignore it."""
        B = env.B
        names = [kinds] * B if isinstance(kinds, str) else list(kinds)
        if len(names) != B:
            raise ValueError(f'{len(names)} agent kinds for {B} episodes')
        unknown = sorted({n for n in names if n not in AGENT})
        if unknown:
            raise ValueError(f'unknown agents {unknown}; known: {list(AGENTS)}')
        self.kinds = np.ascontiguousarray([AGENT[n] for n in names], dtype=np.int32)
        if params is None or np.ndim(params) == 0:
            p = [0 if params is None else int(params)] * B
        else:
            p = [0 if x is None else int(x) for x in params]
        if len(p) != B:
            raise ValueError(f'{len(p)} agent parameters for {B} episodes')
        self.params = np.ascontiguousarray(p, dtype=np.int32)
        self.env = env
        L = env.eng._L
        L.ramp_env_set_agents.restype = C.c_int
        L.ramp_env_set_agents.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.ramp_env_agent_act.restype = C.c_int
        L.ramp_env_agent_act.argtypes = [C.c_void_p, C.c_uint64]
        _engine._check(L.ramp_env_set_agents(env.eng._h, self.kinds.ctypes.data, self.params.ctypes.data))

    def act(self, seed: int = 0):
        """One decision per episode into the environment's device action buffer; nothing crosses PCIe.  Follow with
        ``env.step_device()`` (or ``env.step(None)``)."""
        _engine._check(self.env.eng._L.ramp_env_agent_act(self.env.eng._h, C.c_uint64(int(seed) & (2 ** 64 - 1))))


def evaluate(env, actor, seed: int = 0, sample: bool = False, step_stats: bool = False):
    """EvalLoop.run (loops/eval_loop.py:26-134) for every episode of a DeviceRampJobPartitioningEnvironment at once: reset, then
    ``jobs_per_episode`` rounds of actor -> ``env.step_device()`` (an env-step consumes the one queued job, so no episode takes
    more), then ``env.episode_stats()``.  actor: a DeviceHeuristicAgents, or a DeviceGNNPolicy (greedy unless ``sample``).  The
    loop does not synchronise when ``prewarm()`` lets the device decide every placement.  Raises if an episode is not done.

    step_stats=False returns ``env.episode_stats()``.  step_stats=True returns EvalLoop.run's ``{'step_stats': ...,
    'episode_stats': ...}``: the device records every env-step's action, reward and reduced steps_log row while the loop runs
    (``env.record_steps``), still without synchronising, and ``step_stats`` is ``env.recorded_steps()`` -- per key a list of B
    arrays, one entry per env-step of the episode."""
    from .policy import DeviceGNNPolicy
    env.reset()
    if step_stats:
        env.record_steps(env.J)
    for t in range(env.J):
        if isinstance(actor, DeviceGNNPolicy):
            actor.act(env, sample=sample, seed=seed + t)
        else:
            actor.act(seed)                                # Random's draws are keyed by the episode's decision count
        env.step_device()
    _, _, done = env.read()                                # raises what a step would have raised
    if not done.all():
        raise Exception(f'{int((~done).sum())} of {env.B} episodes are not done after {env.J} env-steps')
    if not step_stats:
        return env.episode_stats()
    steps = env.recorded_steps()
    env.record_steps(0)
    return {'step_stats': steps, 'episode_stats': env.episode_stats()}
