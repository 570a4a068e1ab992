"""Population-based training (Jaderberg et al. 2017) of a device population learner: every ``interval`` calls the worst sets take
the training state of the best ("exploit") and perturb their hyperparameters ("explore").

``PopulationBasedTraining(learner, mutations)`` wraps a DevicePopulation{PPO,IMPALA,PG,ES}Learner.  Its K sets already sit in one
device batch with their optimiser state beside them, so exploit is one device-to-device copy between slices of the population's
buffers (DeviceGNNPolicyPopulation.copy_sets, and DevicePopulationESLearner.copy_sets for ES's own Adam state): no checkpoint
round trip and no host copy of the weights.

The rules restate Ray Tune's documented PBT scheduler (tune/schedulers/pbt.py: _quantiles, _explore), with its defaults
quantile_fraction 0.25, resample_probability 0.25 and perturbation_factors (1.2, 0.8).  Ray is not installed, so they are restated,
not pinned against it.  Where Ray draws from Python's global random state, every draw here is splitmix64 keyed by (seed, PBT step,
set, field, draw), so the decisions are a pure function of the scores and the configs (tests/test_pbt_model.py restates them)."""
from __future__ import annotations

import dataclasses
import math
from typing import Callable, Dict, List, Sequence

import numpy as np

from . import learn as _learn
from .policy import splitmix64

_M64 = 2 ** 64 - 1
QUANTILE_FRACTION = 0.25
RESAMPLE_PROBABILITY = 0.25
PERTURBATION_FACTORS = (1.2, 0.8)
DONOR = 0                             # draw slot of the donor choice; mutation field f (in the order given) draws in slot f + 1


def uniform(lo: float, hi: float) -> Callable[[float], float]:
    """a sampler for a continuous field: u in [0, 1) -> lo + u (hi - lo)"""
    return lambda u: lo + u * (hi - lo)


def log_uniform(lo: float, hi: float) -> Callable[[float], float]:
    """a sampler for a continuous field: u in [0, 1) -> lo (hi / lo)^u (tune.loguniform)"""
    return lambda u: lo * (hi / lo) ** u


def draw(seed: int, step: int, k: int, slot: int, j: int) -> float:
    """the uniform in [0, 1) of draw j in slot `slot` for set k at PBT step `step`: splitmix64 chained over the key, top 53 bits"""
    x = splitmix64(int(seed) & _M64)
    for v in (step, k, slot, j):
        x = splitmix64(x ^ (int(v) & _M64))
    return (x >> 11) * 2.0 ** -53


def _pick(u: float, n: int) -> int:
    return min(int(u * n), n - 1)


def quantile_size(K: int, quantile_fraction: float = QUANTILE_FRACTION) -> int:
    """sets in each of the bottom and top quantiles: ceil(fraction K), at most floor(K / 2) so that they never overlap (Ray's
    _quantiles)"""
    n = int(math.ceil(K * quantile_fraction))
    return min(n, K // 2)


def ranking(scores: Sequence[float]) -> List[int]:
    """the sets from worst to best: by score, ties by set index (the lower index ranks lower); NaN ranks lowest"""
    key = [(-math.inf if math.isnan(float(s)) else float(s), k) for k, s in enumerate(scores)]
    return [k for _, k in sorted(key)]


def explore(value, spec, seed: int, step: int, k: int, slot: int, resample_probability: float = RESAMPLE_PROBABILITY,
            perturbation_factors: Sequence[float] = PERTURBATION_FACTORS):
    """Ray's _explore for one field of set k's (donor's) config value.  spec a list: resampled (draw 0 < resample_probability,
    or the value is not in it) as spec[draw 1], else moved one index down (draw 1 < 0.5) or up, clamped to the ends.  spec a
    sampler: resampled as spec(draw 1), else multiplied by perturbation_factors[draw 1]; an int field stays an int."""
    u0, u1 = draw(seed, step, k, slot, 0), draw(seed, step, k, slot, 1)
    if isinstance(spec, (list, tuple)):
        if u0 < resample_probability or value not in spec:
            return spec[_pick(u1, len(spec))]
        i = list(spec).index(value) + (-1 if u1 < 0.5 else 1)
        return spec[min(max(i, 0), len(spec) - 1)]
    new = spec(u1) if u0 < resample_probability else value * perturbation_factors[_pick(u1, len(perturbation_factors))]
    return int(new) if isinstance(value, int) and not isinstance(value, bool) else new


def decide(scores: Sequence[float], configs: Sequence, mutations: Dict, step: int, seed: int = 0,
           quantile_fraction: float = QUANTILE_FRACTION, resample_probability: float = RESAMPLE_PROBABILITY,
           perturbation_factors: Sequence[float] = PERTURBATION_FACTORS) -> List[Dict]:
    """One PBT step's decisions, a pure function: for each set of the bottom quantile, worst first, its donor (top[draw]) and
    the new values of the mutated fields, explored from the donor's config.  Each record: set, donor, old (the set's values
    before), new."""
    order = ranking(scores)
    n = quantile_size(len(scores), quantile_fraction)
    bottom, top = order[:n], order[len(order) - n:]
    out = []
    for k in bottom:
        donor = top[_pick(draw(seed, step, k, DONOR, 0), len(top))]
        new = {f: explore(getattr(configs[donor], f), spec, seed, step, k, DONOR + 1 + i, resample_probability, perturbation_factors)
               for i, (f, spec) in enumerate(mutations.items())}
        out.append(dict(set=k, donor=donor, old={f: getattr(configs[k], f) for f in mutations}, new=new))
    return out


def group_returns(traj, K: int) -> np.ndarray:
    """PPO / IMPALA / PG fitness from a population's collect(): per group, its episodes' mean return over the segment's live rows
    (reward summed over each episode's live rows, averaged over the group's b episodes)"""
    reward = np.where(traj['live'], traj['reward'], 0.0).sum(axis=0)
    return reward.reshape(K, -1).mean(axis=1)


def es_scores(stats) -> np.ndarray:
    """ES fitness from DevicePopulationESLearner.learn(): stats[k]['episode_reward_mean']"""
    return np.array([s['episode_reward_mean'] for s in stats], dtype=np.float64)


_LEARNERS = (_learn.DevicePopulationPPOLearner, _learn.DevicePopulationIMPALALearner, _learn.DevicePopulationPGLearner,
             _learn.DevicePopulationESLearner)


class PopulationBasedTraining:
    """PBT over a population learner's K sets.  mutations: {config field: a list of values or a sampler (uniform, log_uniform, or
    any u in [0, 1) -> value)}.  step(scores) every learn call; every `interval`-th call ranks the sets and, for each of the bottom
    quantile_size(K) sets, copies a top-quantile donor's training state onto it in one launch (plus the ES learner's for ES), makes
    its config a copy of the donor's with its own seed (so the groups' draws stay distinct), and explores each mutated field."""

    def __init__(self, learner, mutations: Dict, interval: int = 1, quantile_fraction: float = QUANTILE_FRACTION,
                 resample_probability: float = RESAMPLE_PROBABILITY, perturbation_factors: Sequence[float] = PERTURBATION_FACTORS,
                 seed: int = 0):
        if not isinstance(learner, _LEARNERS):
            raise TypeError(f'{type(learner).__name__}: PBT wraps a population learner ({", ".join(c.__name__ for c in _LEARNERS)})')
        if interval < 1:
            raise ValueError(f'interval {interval} must be >= 1')
        if not 0 < quantile_fraction <= 0.5:
            raise ValueError(f'quantile_fraction {quantile_fraction} must be in (0, 0.5]')
        pop = learner.population
        shapes = [bytes(c) for c in pop._ccfgs]
        if len(set(shapes)) > 1:
            k = next(k for k, s in enumerate(shapes) if s != shapes[0])
            raise ValueError(f'PBT copies training state between sets, so every set must have one shape: set {k} differs from set 0')
        fields = {f.name for f in dataclasses.fields(learner.configs[0])}
        fixed = tuple(learner._shared) + (('noise_size',) if isinstance(learner, _learn.DevicePopulationESLearner) else ())
        for f, spec in mutations.items():
            if f not in fields:
                raise ValueError(f'mutation of {f!r}: {type(learner.configs[0]).__name__} has no such field')
            if f in fixed:
                raise ValueError(f'mutation of {f!r}: {type(learner).__name__} needs it to be the same for every set')
            if f == 'seed':
                raise ValueError("mutation of 'seed': each set keeps its own seed")
            if isinstance(spec, (list, tuple)) and not spec:
                raise ValueError(f'mutation of {f!r}: an empty list of values')
            if not isinstance(spec, (list, tuple)) and not callable(spec):
                raise ValueError(f'mutation of {f!r}: a list of values or a sampler u -> value')
        self.learner, self.mutations, self.interval = learner, dict(mutations), int(interval)
        self.quantile_fraction, self.resample_probability = quantile_fraction, resample_probability
        self.perturbation_factors, self.seed = tuple(perturbation_factors), int(seed)
        self.calls = 0                # step() calls
        self.steps = 0                # PBT steps taken: the draws' step key

    def step(self, scores: Sequence[float]) -> List[Dict]:
        """after a learn call, with its K fitness values (group_returns, es_scores): every interval-th call, exploit and explore;
        returns decide()'s records of what was done (empty on the other calls, and when K < 2)"""
        lrn = self.learner
        K = lrn.population.K
        if len(scores) != K:
            raise ValueError(f'{len(scores)} scores for a population of {K} sets')
        self.calls += 1
        if self.calls % self.interval:
            return []
        recs = decide(scores, lrn.configs, self.mutations, self.steps, self.seed, self.quantile_fraction, self.resample_probability,
                      self.perturbation_factors)
        self.steps += 1
        if not recs:
            return recs
        dst, src = [r['set'] for r in recs], [r['donor'] for r in recs]
        lrn.population.copy_sets(dst, src)
        if isinstance(lrn, _learn.DevicePopulationESLearner):
            lrn.copy_sets(dst, src)
        for r in recs:
            k = r['set']
            keep = {'seed': lrn.configs[k].seed} if hasattr(lrn.configs[k], 'seed') else {}
            lrn.configs[k] = dataclasses.replace(lrn.configs[r['donor']], **keep, **r['new'])
        return recs
