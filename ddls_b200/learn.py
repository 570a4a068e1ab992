"""RLlib's PPO learner step for the device GNN policy (include/ramp_b200.h: ramp_ppo_loss_grad, ramp_policy_learn).

``DevicePPOLearner(policy, config).learn(env, horizon)`` learns from the rollout segment the policy's last ``collect(env, ...)``
recorded (``collect_and_learn`` does both) without moving the batch to the host: GAE and advantage standardisation, ``num_sgd_iter`` shuffled passes of minibatch PPO loss
gradients, global-norm clipping and Adam, all on the device.  ``PPOConfig``'s defaults are the reference's tuned PPO settings
(scripts/ramp_job_partitioning_configs/algo/ppo.yaml; lambda is RLlib's default 1.0).

The loss, GAE and the KL-coefficient update restate RLlib's PPO (ppo_torch_policy.py, postprocessing.compute_advantages,
PPO.update_kl) as published for the ray the reference pins; RLlib itself is not installed, so they are pinned against a float64
restatement (tests/test_ppo_model.py, tests/test_gpu_policy_learn.py), not against RLlib.

``DeviceIMPALALearner(policy, config)`` is RLlib's IMPALA learner step on the same trajectory (include/ramp_b200.h:
ramp_impala_loss_grad, ramp_policy_learn_impala): V-trace (vtrace_torch.py) over fragments of rollout_fragment_length rows and
VTraceLoss (impala_torch_policy.py), one Adam step per train batch, through the same gradient kernels.  ``IMPALAConfig``'s defaults
are algo/impala.yaml's; its restatement is tests/impala_reference.py.

``DevicePGLearner(policy, config)`` is RLlib's PG learner step (include/ramp_b200.h: ramp_pg_loss_grad, ramp_policy_learn_pg):
discounted returns with no bootstrap (postprocessing.compute_advantages, use_critic False) and -mean(logp(a) return)
(pg_torch_policy.py), one Adam step per segment, through the same gradient kernels.  ``PGConfig``'s defaults are algo/pg.yaml's
over rllib_config.yaml's base; its restatement is tests/pg_reference.py.

``DeviceESLearner(policy, config)`` is RLlib's evolution strategies (include/ramp_b200.h: ramp_es_*): the environment's episodes
are a population of antithetic weight perturbations, one weight set per episode in one batch, then centered ranks, the
noise-weighted sum and optimizers.Adam on the device.  ``ESConfig``'s defaults are algo/es.yaml's; its restatement is
tests/es_reference.py.

There is no CPU fallback: the CUDA library is required."""
from __future__ import annotations

import ctypes as C
import dataclasses
import time
from typing import Dict

import numpy as np

from . import engine as _engine

STATS = ('total_loss', 'policy_loss', 'vf_loss', 'entropy', 'kl', 'clip_frac', 'grad_gnorm', 'kl_coeff', 'rows')


@dataclasses.dataclass
class PPOConfig:
    gamma: float = 0.997
    lambda_: float = 1.0
    clip_param: float = 0.18
    vf_clip_param: float = 128.8
    vf_loss_coeff: float = 0.5
    entropy_coeff: float = 0.003
    kl_coeff: float = 0.01
    kl_target: float = 0.001
    grad_clip: float = 1.5            # <= 0: no clipping
    lr: float = 2.785e-4
    sgd_minibatch_size: int = 128
    num_sgd_iter: int = 50
    adam_beta1: float = 0.9
    adam_beta2: float = 0.999
    adam_eps: float = 1e-8
    standardize_advantages: bool = True
    seed: int = 0


class _CConfig(C.Structure):
    _fields_ = [('seed', C.c_uint64)] + [(n, C.c_double) for n in (
        'gamma', 'lambda_', 'clip_param', 'vf_clip_param', 'vf_loss_coeff', 'entropy_coeff', 'kl_coeff', 'kl_target', 'grad_clip', 'lr',
        'adam_beta1', 'adam_beta2', 'adam_eps')] + [('sgd_minibatch_size', C.c_int32), ('num_sgd_iter', C.c_int32),
                                                    ('standardize_advantages', C.c_int32)]


def _c_struct(struct, cfg, **override):
    """the config dataclass cfg as the C structure `struct`, field by field of its _fields_ (a keyword overrides cfg's attribute):
    a uint64 masked to 64 bits, an int32 as int, a double as float"""
    c = struct()
    for name, ct in struct._fields_:
        v = override[name] if name in override else getattr(cfg, name)
        setattr(c, name, int(v) & (2 ** 64 - 1) if ct is C.c_uint64 else int(v) if ct is C.c_int32 else float(v))
    return c


IMPALA_STATS = ('total_loss', 'policy_loss', 'vf_loss', 'entropy', 'grad_gnorm', 'mean_rho', 'rows', 'sgd_steps')


@dataclasses.dataclass
class IMPALAConfig:
    """algo/impala.yaml's values; gamma, lr and train_batch_size from rllib_config.yaml's base, which impala.yaml does not
    override; torch.optim.Adam's defaults, since RLlib passes it only the lr.  rollout_fragment_length 0: the learn call's
    horizon (one fragment per episode)."""
    gamma: float = 0.99
    vtrace_clip_rho_threshold: float = 1.0
    vtrace_clip_pg_rho_threshold: float = 1.0
    vf_loss_coeff: float = 0.5
    entropy_coeff: float = 0.01
    grad_clip: float = 40.0           # <= 0: no clipping
    lr: float = 1e-4
    adam_beta1: float = 0.9
    adam_beta2: float = 0.999
    adam_eps: float = 1e-8
    rollout_fragment_length: int = 0
    train_batch_size: int = 200


class _CIMPALAConfig(C.Structure):
    _fields_ = [(n, C.c_double) for n in (
        'gamma', 'vtrace_clip_rho_threshold', 'vtrace_clip_pg_rho_threshold', 'vf_loss_coeff', 'entropy_coeff', 'grad_clip', 'lr',
        'adam_beta1', 'adam_beta2', 'adam_eps')] + [('rollout_fragment_length', C.c_int32), ('train_batch_size', C.c_int32)]


def _bind(L):
    """every learner call's signature, once per library"""
    if getattr(L, '_learn_bound', False):
        return
    for name, args in (('ramp_ppo_loss_grad', [C.c_void_p, C.POINTER(_CConfig), C.c_int32] + [C.c_void_p] * 9),
                       ('ramp_policy_learn', [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(_CConfig), C.c_void_p]),
                       ('ramp_policy_train_batch_read', [C.c_void_p, C.c_void_p] + [C.c_void_p] * 7),
                       ('ramp_policy_learner_state', [C.c_void_p] * 4),
                       ('ramp_policy_learner_reset', [C.c_void_p]),
                       ('ramp_impala_loss_grad', [C.c_void_p, C.POINTER(_CIMPALAConfig), C.c_int32, C.c_int32] + [C.c_void_p] * 12),
                       ('ramp_policy_learn_impala', [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(_CIMPALAConfig), C.c_void_p]),
                       ('ramp_impala_vtrace_read', [C.c_void_p] * 6),
                       ('ramp_pg_loss_grad', [C.c_void_p, C.POINTER(_CPGConfig), C.c_int32] + [C.c_void_p] * 7),
                       ('ramp_policy_learn_pg', [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(_CPGConfig), C.c_void_p]),
                       ('ramp_es_create', [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
                       ('ramp_es_round_begin', [C.c_void_p, C.c_void_p, C.POINTER(_CESConfig), C.c_int32]),
                       ('ramp_es_act', [C.c_void_p, C.c_void_p, C.c_int32]),
                       ('ramp_es_round_end', [C.c_void_p, C.c_void_p, C.c_void_p]),
                       ('ramp_es_step', [C.c_void_p, C.POINTER(_CESConfig), C.c_void_p]),
                       ('ramp_es_update', [C.c_void_p, C.POINTER(_CESConfig), C.c_int32] + [C.c_void_p] * 5),
                       ('ramp_es_read', [C.c_void_p] * 12),
                       ('ramp_es_act_read', [C.c_void_p] * 5),
                       ('ramp_es_state', [C.c_void_p] * 4),
                       ('ramp_es_reset', [C.c_void_p]),
                       ('ramp_population_learn', [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(_CConfig), C.c_void_p]),
                       ('ramp_population_learner_state', [C.c_void_p, C.c_int32] + [C.c_void_p] * 3),
                       ('ramp_population_learn_impala', [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(_CIMPALAConfig), C.c_void_p]),
                       ('ramp_population_learn_pg', [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(_CPGConfig), C.c_void_p]),
                       ('ramp_population_vtrace_read', [C.c_void_p, C.c_int32] + [C.c_void_p] * 5),
                       ('ramp_population_es_create', [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
                       ('ramp_population_es_round_begin', [C.c_void_p, C.c_void_p, C.POINTER(_CESConfig), C.c_int32]),
                       ('ramp_population_es_act', [C.c_void_p, C.c_void_p, C.c_int32]),
                       ('ramp_population_es_round_end', [C.c_void_p, C.c_void_p, C.c_void_p]),
                       ('ramp_population_es_step', [C.c_void_p, C.POINTER(_CESConfig), C.c_void_p]),
                       ('ramp_population_es_update', [C.c_void_p, C.POINTER(_CESConfig)] + [C.c_void_p] * 4),
                       ('ramp_population_es_read', [C.c_void_p, C.c_int32] + [C.c_void_p] * 11),
                       ('ramp_population_es_act_read', [C.c_void_p] * 5),
                       ('ramp_population_es_state', [C.c_void_p, C.c_int32] + [C.c_void_p] * 3),
                       ('ramp_population_es_reset', [C.c_void_p]),
                       ('ramp_population_es_embed_ctas', [C.c_void_p] * 3),
                       ('ramp_policy_set_learner_state', [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32]),
                       ('ramp_population_set_learner_state', [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32]),
                       ('ramp_es_set_state', [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32]),
                       ('ramp_es_get_progress', [C.c_void_p] * 4),
                       ('ramp_es_set_progress', [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]),
                       ('ramp_population_set_es_state', [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32]),
                       ('ramp_population_get_es_progress', [C.c_void_p, C.c_int32] + [C.c_void_p] * 3),
                       ('ramp_population_set_es_progress', [C.c_void_p, C.c_int32, C.c_int64, C.c_int32, C.c_void_p]),
                       ('ramp_population_copy_es_sets', [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p])):
        getattr(L, name).restype = C.c_int
        getattr(L, name).argtypes = args
    for name in ('ramp_es_destroy', 'ramp_population_es_destroy'):
        getattr(L, name).restype = None
        getattr(L, name).argtypes = [C.c_void_p]
    L._learn_bound = True


def _stats(keys, out) -> Dict[str, float]:
    return {k: float(v) for k, v in zip(keys, out)}


def _state_array(state, key: str, n: int) -> np.ndarray:
    """state[key] as the n float32 values the library reads through a raw pointer, refusing any other count"""
    a = np.ascontiguousarray(state[key], dtype=np.float32).ravel()
    if a.shape != (n,):
        raise ValueError(f'training state: {key} has {a.size} values, the set has {n} weights')
    return a


def _es_progress(fn, *args):
    """(iteration, eval means [n]) from ramp_es_get_progress / ramp_population_get_es_progress"""
    it, n = C.c_int64(), C.c_int32()
    _engine._check(fn(*args, C.byref(it), C.byref(n), None))
    means = np.zeros(n.value, np.float64)
    _engine._check(fn(*args, None, None, means.ctypes.data))
    return it.value, means


class _GradientLearner:
    """What the PPO, IMPALA and PG learners share: the policy whose weights they update in place, and Adam's moments and step
    count, which are the policy's -- one set, whichever of the three learners made the step."""
    _Config = None                    # the learner's config dataclass

    def __init__(self, policy, config=None):
        """policy: a DeviceGNNPolicy, whose weights the learner updates in place (Adam's state lives with the policy)."""
        self.policy = policy
        self.config = dataclasses.replace(config) if config is not None else self._Config()
        self._L = policy._L
        _bind(self._L)

    def collect_and_learn(self, env, horizon: int, seed: int = 0):
        """policy.collect(env, horizon) then learn(); also returns the wall time of each (seconds) and the segment's trajectory."""
        t0 = time.perf_counter()
        traj = self.policy.collect(env, horizon, sample=True, seed=seed)
        t1 = time.perf_counter()
        stats = self.learn(env, horizon)
        stats['collect_s'], stats['learn_s'] = t1 - t0, time.perf_counter() - t1
        return stats, traj

    def adam_state(self):
        """torch.optim.Adam's state of the flat weight vector: exp_avg, exp_avg_sq (blob order) and the step count"""
        n = self._L.ramp_policy_weight_count(C.byref(self.policy._cfg))
        m, v, step = np.zeros(n, np.float32), np.zeros(n, np.float32), C.c_int32()
        _engine._check(self._L.ramp_policy_learner_state(self.policy._h, m.ctypes.data, v.ctypes.data, C.byref(step)))
        return m, v, step.value

    def reset(self):
        """zero Adam's moments and step count"""
        _engine._check(self._L.ramp_policy_learner_reset(self.policy._h))

    def training_state(self) -> Dict:
        """everything the next collect -> learn call depends on besides the config: the weights, Adam's moments and step count,
        and the policy's act count (its draws mix it in).  np.savez of the dict is a checkpoint."""
        m, v, step = self.adam_state()
        return dict(weights=self.policy.get_weights(), exp_avg=m, exp_avg_sq=v, step=step, act_count=self.policy.act_count())

    def load_training_state(self, state):
        """resume from a training_state() (or np.load of its np.savez): this learner, made with the config the saving one had,
        then computes what the saving one would have, bit for bit"""
        n = self._L.ramp_policy_weight_count(C.byref(self.policy._cfg))
        w, m, v = (_state_array(state, key, n) for key in ('weights', 'exp_avg', 'exp_avg_sq'))
        self.policy.set_weights(w)
        _engine._check(self._L.ramp_policy_set_learner_state(self.policy._h, m.ctypes.data, v.ctypes.data, n, int(state['step'])))
        self.policy.set_act_count(int(state['act_count']))


def _train_batch(self, env) -> Dict[str, np.ndarray]:
    """the last learn()'s train batch: per live row, t-major, the job type, action, collected log-probability, the one the gradient
    kernel recomputed from the collection weights (logp_old), the advantage and the value target (PPO: standardised when configured,
    and GAE's target; PG: both the discounted return)"""
    cap = self.policy._traj_key[0] * env.B            # the segment's rows: (horizon, B, |A|) of the last collect()
    n = C.c_int32()
    arrs = {'model': np.zeros(cap, np.int32), 'action': np.zeros(cap, np.int32), 'logp': np.zeros(cap, np.float32),
            'logp_old': np.zeros(cap, np.float32), 'advantage': np.zeros(cap, np.float32), 'value_target': np.zeros(cap, np.float32)}
    _engine._check(self._L.ramp_policy_train_batch_read(self.policy._h, env.eng._h, C.byref(n), *[a.ctypes.data for a in arrs.values()]))
    return {k: v[:n.value].copy() for k, v in arrs.items()}


class DevicePPOLearner(_GradientLearner):
    _Config = PPOConfig
    _calls = 0
    train_batch = _train_batch

    def learn(self, env, horizon: int) -> Dict[str, float]:
        """One PPO learner step on the first ``horizon`` steps of the segment the policy's last collect(env, ...) recorded (a shorter
        horizon bootstraps its advantages with the value recorded at the next step): the statistics averaged over the
        last pass's minibatches (STATS); kl_coeff is the adapted coefficient, which this learner uses from the next call on.
        Call k of this learner shuffles with the seed config.seed + k."""
        cfg = dataclasses.replace(self.config, seed=self.config.seed + self._calls)
        out = np.zeros(len(STATS), dtype=np.float64)
        _engine._check(self._L.ramp_policy_learn(self.policy._h, env.eng._h, int(horizon), C.byref(_c_struct(_CConfig, cfg)),
                                                 out.ctypes.data))
        self._calls += 1
        stats = _stats(STATS, out)
        self.config.kl_coeff = stats['kl_coeff']
        return stats

    def training_state(self) -> Dict:
        """_GradientLearner.training_state, plus the adapted kl_coeff and the call count (the next call shuffles with
        config.seed + calls)"""
        return dict(super().training_state(), kl_coeff=self.config.kl_coeff, calls=self._calls)

    def load_training_state(self, state):
        super().load_training_state(state)
        self.config.kl_coeff = float(state['kl_coeff'])
        self._calls = int(state['calls'])

    def loss_and_grad(self, batch: Dict[str, np.ndarray]):
        """PPO's loss statistics (STATS) and gradient (blob order) on one minibatch of host arrays, with no update: model [n],
        graph_features [n, in_features_graph], action_mask [n, |A|], action [n], old_logits [n, |A|], advantage [n],
        value_target [n]."""
        pol = self.policy
        model, gf, mask = pol._host_inputs(batch['model'], batch['graph_features'], batch['action_mask'])
        n, A = len(model), pol.n_actions
        act = np.ascontiguousarray(batch['action'], dtype=np.int32).reshape(n)
        old = np.ascontiguousarray(batch['old_logits'], dtype=np.float32).reshape(n, A)
        adv = np.ascontiguousarray(batch['advantage'], dtype=np.float32).reshape(n)
        vt = np.ascontiguousarray(batch['value_target'], dtype=np.float32).reshape(n)
        grad = np.zeros(pol._L.ramp_policy_weight_count(C.byref(pol._cfg)), dtype=np.float32)
        out = np.zeros(len(STATS), dtype=np.float64)
        _engine._check(self._L.ramp_ppo_loss_grad(pol._h, C.byref(_c_struct(_CConfig, self.config)), n, model.ctypes.data,
                                                  gf.ctypes.data, mask.ctypes.data, act.ctypes.data, old.ctypes.data, adv.ctypes.data,
                                                  vt.ctypes.data, grad.ctypes.data, out.ctypes.data))
        return _stats(STATS, out), grad


class _PopulationLearner:
    """What the population's PPO, IMPALA and PG learners share: one config per set, the fields every set must agree on (they set
    the launch loop), each config's own checks before anything runs, and Adam's moments and step counts, which are the
    population's -- one per set, whichever of the three learners made the step."""
    _shared = ()                      # config fields every set must share
    _checks = ()                      # (field, predicate, rule): each config's own rules, as the C learner checks them

    def __init__(self, population, configs):
        configs = [dataclasses.replace(c) for c in configs]
        if len(configs) != population.K:
            raise ValueError(f'{len(configs)} configs for a population of {population.K} sets')
        for name in self._shared:
            values = [getattr(c, name) for c in configs]
            if len(set(values)) > 1:
                k = next(k for k, v in enumerate(values) if v != values[0])
                raise ValueError(f'{name} must be the same for every set (it sets the launch loop): {values}; set {k} differs from set 0')
        for k, c in enumerate(configs):
            for name, ok, rule in self._checks:
                if not ok(getattr(c, name)):
                    raise ValueError(f'set {k}: {name} = {getattr(c, name)} (it must be {rule})')
        self.population, self.configs = population, configs
        self._L = population._L
        _bind(self._L)

    def adam_state(self, k: int):
        """set k's torch.optim.Adam state: exp_avg, exp_avg_sq (blob order) and the step count"""
        n = self.population.weight_count(k)
        m, v, step = np.zeros(n, np.float32), np.zeros(n, np.float32), C.c_int32()
        _engine._check(self._L.ramp_population_learner_state(self.population._h, int(k), m.ctypes.data, v.ctypes.data, C.byref(step)))
        return m, v, step.value

    def training_state(self, k: int) -> Dict:
        """set k's training state, as the single learner's training_state(): its weights, Adam state, and the population's act
        count, which every group's draws mix in"""
        k = self.population._set(k)
        m, v, step = self.adam_state(k)
        return dict(weights=self.population.get_weights(k), exp_avg=m, exp_avg_sq=v, step=step, act_count=self.population.act_count())

    def load_training_state(self, k: int, state):
        """set k resumes from a training_state (a population's set or a single learner's of the same shape).  The act count is one
        for every set: loading it through any set sets it for all."""
        k = self.population._set(k)
        n = self.population.weight_count(k)
        w, m, v = (_state_array(state, key, n) for key in ('weights', 'exp_avg', 'exp_avg_sq'))
        self.population.set_weights(k, w)
        _engine._check(self._L.ramp_population_set_learner_state(self.population._h, k, m.ctypes.data, v.ctypes.data, n, int(state['step'])))
        self.population.set_act_count(int(state['act_count']))


class DevicePopulationPPOLearner(_PopulationLearner):
    """DevicePPOLearner for every set of a DeviceGNNPolicyPopulation at once: group k of the environment learns only from its own
    episodes with configs[k], and ends each call with the weights, Adam state, statistics and kl_coeff a DevicePPOLearner with
    configs[k] would reach on a group-sized environment with the same episode streams, bit for bit.  Every minibatch step runs
    all K sets in the same launches.  sgd_minibatch_size and num_sgd_iter set that launch loop, so the K configs must agree on them."""
    _shared = ('sgd_minibatch_size', 'num_sgd_iter')

    def __init__(self, population, configs):
        super().__init__(population, configs)
        self._calls = 0

    def learn(self, env, horizon: int):
        """One PPO learner step per set on the first ``horizon`` steps of the population's last collect(env, ...): a list of K stats
        dicts (STATS).  Set k's call c shuffles with configs[k].seed + c, and its kl_coeff is adapted as DevicePPOLearner's."""
        pop = self.population
        pop.group_size(env)
        cfgs = (_CConfig * pop.K)(*[_c_struct(_CConfig, c, seed=c.seed + self._calls) for c in self.configs])
        out = np.zeros((pop.K, len(STATS)), dtype=np.float64)
        _engine._check(self._L.ramp_population_learn(pop._h, env.eng._h, int(horizon), cfgs, out.ctypes.data))
        self._calls += 1
        stats = [_stats(STATS, row) for row in out]
        for c, s in zip(self.configs, stats):
            c.kl_coeff = s['kl_coeff']
        return stats

    def training_state(self, k: int) -> Dict:
        """_PopulationLearner.training_state, plus configs[k]'s adapted kl_coeff and the call count (one for every set)"""
        return dict(super().training_state(k), kl_coeff=self.configs[k].kl_coeff, calls=self._calls)

    def load_training_state(self, k: int, state):
        super().load_training_state(k, state)
        self.configs[k].kl_coeff = float(state['kl_coeff'])
        self._calls = int(state['calls'])


class DeviceIMPALALearner(_GradientLearner):
    """RLlib's IMPALA learner step (V-trace, VTraceLoss, clip_grad_norm_, Adam) on the segment the policy's last collect()
    recorded, on the device.  Adam's moments and step count are the policy's, shared with DevicePPOLearner."""
    _Config = IMPALAConfig

    def learn(self, env, horizon: int) -> Dict[str, float]:
        """One IMPALA learner step on the first ``horizon`` steps of the segment the policy's last collect(env, ...) recorded: the
        fragments of rollout_fragment_length rows (0: horizon), one Adam step per train batch of train_batch_size // L fragments,
        in order.  Returns the means over the call's SGD steps (IMPALA_STATS), and their number as sgd_steps."""
        out = np.zeros(len(IMPALA_STATS), dtype=np.float64)
        _engine._check(self._L.ramp_policy_learn_impala(self.policy._h, env.eng._h, int(horizon),
                                                        C.byref(_c_struct(_CIMPALAConfig, self.config)), out.ctypes.data))
        return _stats(IMPALA_STATS, out)

    def vtrace(self) -> Dict[str, np.ndarray]:
        """per fragment row (r = f L + t) of the last learn() or loss_and_grad(), as the step that used it computed it: the target
        log-probability of the action (0 on a row without decision), log rho, vs and pg_advantages"""
        n = C.c_int32()
        _engine._check(self._L.ramp_impala_vtrace_read(self.policy._h, C.byref(n), None, None, None, None))
        arrs = {k: np.zeros(n.value, np.float32) for k in ('target_logp', 'log_rho', 'vs', 'pg_advantages')}
        _engine._check(self._L.ramp_impala_vtrace_read(self.policy._h, C.byref(n), *[a.ctypes.data for a in arrs.values()]))
        return arrs

    def loss_and_grad(self, batch: Dict[str, np.ndarray]):
        """VTraceLoss's statistics (IMPALA_STATS, sgd_steps 0) and gradient (blob order) on host fragments, with no update, and
        the V-trace values (vs, pg_advantages, log_rho; [n, L]).  batch: arrays with leading shape [n fragments, L rows]: model,
        graph_features [.., in_features_graph], action_mask [.., |A|], action, behaviour_logp, reward, done."""
        pol = self.policy
        n, L = np.shape(batch['model'])[:2]
        model, gf, mask = pol._host_inputs(np.reshape(batch['model'], -1), np.reshape(batch['graph_features'], (n * L, -1)),
                                           np.reshape(batch['action_mask'], (n * L, -1)))
        act = np.ascontiguousarray(batch['action'], dtype=np.int32).reshape(n * L)
        blogp = np.ascontiguousarray(batch['behaviour_logp'], dtype=np.float32).reshape(n * L)
        reward = np.ascontiguousarray(batch['reward'], dtype=np.float64).reshape(n * L)
        done = np.ascontiguousarray(batch['done'], dtype=np.uint8).reshape(n * L)
        grad = np.zeros(pol._L.ramp_policy_weight_count(C.byref(pol._cfg)), dtype=np.float32)
        out = np.zeros(len(IMPALA_STATS), dtype=np.float64)
        vt = {k: np.zeros(n * L, np.float32) for k in ('vs', 'pg_advantages', 'log_rho')}
        _engine._check(self._L.ramp_impala_loss_grad(pol._h, C.byref(_c_struct(_CIMPALAConfig, self.config)), int(n), int(L),
                                                     model.ctypes.data, gf.ctypes.data, mask.ctypes.data, act.ctypes.data,
                                                     blogp.ctypes.data, reward.ctypes.data, done.ctypes.data, grad.ctypes.data,
                                                     out.ctypes.data, *[a.ctypes.data for a in vt.values()]))
        return _stats(IMPALA_STATS, out), grad, {k: v.reshape(n, L) for k, v in vt.items()}


PG_STATS = ('policy_loss', 'entropy', 'grad_gnorm', 'rows')


@dataclasses.dataclass
class PGConfig:
    """rllib_config.yaml's gamma and lr (algo/pg.yaml sets neither); torch.optim.Adam's defaults, since RLlib passes it only the lr;
    PG sets no grad_clip (<= 0: no clipping)."""
    gamma: float = 0.99
    lr: float = 1e-4
    grad_clip: float = 0.0
    adam_beta1: float = 0.9
    adam_beta2: float = 0.999
    adam_eps: float = 1e-8


class _CPGConfig(C.Structure):
    _fields_ = [(n, C.c_double) for n in ('gamma', 'grad_clip', 'lr', 'adam_beta1', 'adam_beta2', 'adam_eps')]


class DevicePGLearner(_GradientLearner):
    """RLlib's PG learner step (discounted returns, pg_torch_loss, Adam) on the segment the policy's last collect() recorded, on
    the device.  Adam's moments and step count are the policy's, shared with DevicePPOLearner and DeviceIMPALALearner."""
    _Config = PGConfig
    train_batch = _train_batch

    def learn(self, env, horizon: int) -> Dict[str, float]:
        """One PG learner step on the first ``horizon`` steps of the segment the policy's last collect(env, ...) recorded: one train
        batch of every decision of the segment, one Adam step.  Each episode's advantage is its discounted return; a segment that
        ends before its episode does is not bootstrapped (PG's last_r is 0).  There is no train_batch_size: under RLlib's
        batch_mode complete_episodes a train batch is whole episodes, so the caller sizes env.B and the horizon so that the
        segment holds the env-steps it wants per update (pg's train_batch_size is 200) and its episodes end inside it.  Returns
        PG_STATS; a segment with no decision makes no update and leaves Adam's step count as it was."""
        out = np.zeros(len(PG_STATS), dtype=np.float64)
        _engine._check(self._L.ramp_policy_learn_pg(self.policy._h, env.eng._h, int(horizon), C.byref(_c_struct(_CPGConfig, self.config)),
                                                    out.ctypes.data))
        return _stats(PG_STATS, out)

    def loss_and_grad(self, batch: Dict[str, np.ndarray]):
        """pg_torch_loss's statistics (PG_STATS) and gradient (blob order) on host rows, with no update: model [n],
        graph_features [n, in_features_graph], action_mask [n, |A|], action [n], advantage [n]."""
        pol = self.policy
        model, gf, mask = pol._host_inputs(batch['model'], batch['graph_features'], batch['action_mask'])
        n = len(model)
        act = np.ascontiguousarray(batch['action'], dtype=np.int32).reshape(n)
        adv = np.ascontiguousarray(batch['advantage'], dtype=np.float32).reshape(n)
        grad = np.zeros(pol._L.ramp_policy_weight_count(C.byref(pol._cfg)), dtype=np.float32)
        out = np.zeros(len(PG_STATS), dtype=np.float64)
        _engine._check(self._L.ramp_pg_loss_grad(pol._h, C.byref(_c_struct(_CPGConfig, self.config)), n, model.ctypes.data,
                                                 gf.ctypes.data, mask.ctypes.data, act.ctypes.data, adv.ctypes.data, grad.ctypes.data,
                                                 out.ctypes.data))
        return _stats(PG_STATS, out), grad


class DevicePopulationIMPALALearner(_PopulationLearner):
    """DeviceIMPALALearner for every set of a DeviceGNNPolicyPopulation at once: group k learns only from its own episodes with
    configs[k], and ends each call with the weights, Adam state, statistics and V-trace values a DeviceIMPALALearner with configs[k]
    would reach on a group-sized environment with the same episode streams, bit for bit.  SGD step j of every set runs in the same
    launches.  rollout_fragment_length and train_batch_size fix the fragments and the SGD steps, so the K configs must agree on
    them; gamma, the clip thresholds, the loss coefficients, grad_clip and Adam's settings are each set's own."""
    _shared = ('rollout_fragment_length', 'train_batch_size')
    _checks = (('vtrace_clip_rho_threshold', lambda v: v > 0, '> 0'), ('vtrace_clip_pg_rho_threshold', lambda v: v > 0, '> 0'),
               ('lr', lambda v: v >= 0, '>= 0'), ('adam_eps', lambda v: v > 0, '> 0'),
               ('rollout_fragment_length', lambda v: v >= 0, '>= 0'), ('train_batch_size', lambda v: v >= 1, '>= 1'))

    def learn(self, env, horizon: int):
        """One IMPALA learner step per set on the first ``horizon`` steps of the population's last collect(env, ...): a list of K
        stats dicts (IMPALA_STATS), each the means over its set's SGD steps."""
        pop = self.population
        pop.group_size(env)
        cfgs = (_CIMPALAConfig * pop.K)(*[_c_struct(_CIMPALAConfig, c) for c in self.configs])
        out = np.zeros((pop.K, len(IMPALA_STATS)), dtype=np.float64)
        _engine._check(self._L.ramp_population_learn_impala(pop._h, env.eng._h, int(horizon), cfgs, out.ctypes.data))
        return [_stats(IMPALA_STATS, row) for row in out]

    def vtrace(self, k: int) -> Dict[str, np.ndarray]:
        """set k's per fragment row values of the last learn(), as DeviceIMPALALearner.vtrace() gives them for its group"""
        n = C.c_int32()
        _engine._check(self._L.ramp_population_vtrace_read(self.population._h, int(k), C.byref(n), None, None, None, None))
        arrs = {key: np.zeros(n.value, np.float32) for key in ('target_logp', 'log_rho', 'vs', 'pg_advantages')}
        _engine._check(self._L.ramp_population_vtrace_read(self.population._h, int(k), C.byref(n), *[a.ctypes.data for a in arrs.values()]))
        return arrs


class DevicePopulationPGLearner(_PopulationLearner):
    """DevicePGLearner for every set of a DeviceGNNPolicyPopulation at once: group k learns only from its own episodes with
    configs[k], and ends each call with the weights, Adam state and statistics a DevicePGLearner with configs[k] would reach on a
    group-sized environment with the same episode streams, bit for bit.  Nothing has to agree across the configs."""
    _checks = (('gamma', lambda v: v >= 0, '>= 0'), ('lr', lambda v: v >= 0, '>= 0'), ('adam_eps', lambda v: v > 0, '> 0'))

    def learn(self, env, horizon: int):
        """One PG learner step per set on the first ``horizon`` steps of the population's last collect(env, ...): a list of K stats
        dicts (PG_STATS).  A group whose segment has no decision makes no update and keeps its step count."""
        pop = self.population
        pop.group_size(env)
        cfgs = (_CPGConfig * pop.K)(*[_c_struct(_CPGConfig, c) for c in self.configs])
        out = np.zeros((pop.K, len(PG_STATS)), dtype=np.float64)
        _engine._check(self._L.ramp_population_learn_pg(pop._h, env.eng._h, int(horizon), cfgs, out.ctypes.data))
        return [_stats(PG_STATS, row) for row in out]


ES_STATS = ('episode_reward_mean', 'episode_len_mean', 'timesteps_this_iter', 'episodes_this_iter', 'weights_norm', 'grad_norm',
            'update_ratio', 'eval_return_mean', 'rounds')


@dataclasses.dataclass
class ESConfig:
    """algo/es.yaml's algo_config over the epoch loop's base (train_batch_size 200: es.yaml comments its own out); optimizers.Adam's
    betas and epsilon.  action_noise_std is accepted and has no effect on a Discrete action space, as in RLlib.
    observation_filter: 'NoFilter' only -- RLlib's MeanStdFilter (es.yaml) standardises the flattened observation, padded edge
    indices and action mask included, which the GNN reads back as they are."""
    noise_stdev: float = 0.02
    stepsize: float = 0.01
    l2_coeff: float = 0.005
    eval_prob: float = 0.03
    episodes_per_batch: int = 1000
    train_batch_size: int = 200
    report_length: int = 10
    noise_size: int = 250_000_000
    adam_beta1: float = 0.99
    adam_beta2: float = 0.999
    adam_eps: float = 1e-8
    action_noise_std: float = 0.01
    observation_filter: str = 'NoFilter'
    n_eval: int = None                # eval episodes per round; None: max(1, round(B eval_prob / (2 - eval_prob))), made even with B
    seed: int = 0


class _CESConfig(C.Structure):
    _fields_ = [('seed', C.c_uint64)] + [(n, C.c_double) for n in (
        'noise_stdev', 'stepsize', 'l2_coeff', 'adam_beta1', 'adam_beta2', 'adam_eps')] + [
        (n, C.c_int32) for n in ('episodes_per_batch', 'train_batch_size', 'n_eval', 'report_length')]


def es_n_eval(config: ESConfig, B: int) -> int:
    """eval episodes per round of a B-episode environment (a population's: of one group): config.n_eval, else RLlib's expected
    share of eval episodes B eval_prob / (2 - eval_prob), at least 1, plus one when B - E would be odd"""
    if config.n_eval is not None:
        return int(config.n_eval)
    p = config.eval_prob
    E = max(1, int(round(B * p / (2.0 - p))))
    return E + ((B - E) & 1)


def _es_learn(self, env, timing: bool = False):
    """One ES training step: rounds until end_round() says no more are needed, then step().  Each round resets env and runs
    env.J env-steps, so every episode ends in it; the round synchronises once, at its end.  timing=True also synchronises after
    the embeddings and adds the wall time (seconds) of the embeddings (embed_s), of the rollouts (rollout_s) and of the update
    (update_s)."""
    B = env.B
    times = dict(embed_s=0.0, rollout_s=0.0)
    rnd, more = 0, True
    while more:
        env.reset()
        t0 = time.perf_counter()
        self.begin_round(env, rnd)
        if timing:
            env.eng.sync()
        t1 = time.perf_counter()
        for t in range(env.J):
            self.act(env, t)
            env.step_device()
        more = self.end_round(env)
        _, _, done = env.read()                        # raises what a step would have raised
        if not done.all():
            raise Exception(f'{int((~done).sum())} of {B} episodes are not done after {env.J} env-steps')
        t2 = time.perf_counter()
        times['embed_s'] += t1 - t0
        times['rollout_s'] += t2 - t1
        rnd += 1
    t3 = time.perf_counter()
    stats = self.step()
    if timing:
        for s in (stats if isinstance(stats, list) else [stats]):
            s.update(times, update_s=time.perf_counter() - t3)
    return stats


def shared_noise_table(size: int) -> np.ndarray:
    """RLlib's shared noise table (es.py create_shared_noise), bit for bit.  At the default size it takes seconds and 1 GB as
    float32 (2 GB more while numpy draws it in float64)."""
    return np.random.RandomState(123).randn(int(size)).astype(np.float32)


class DeviceESLearner:
    """RLlib's ES training step (es.py training_step) with a DeviceRampJobPartitioningEnvironment's B episodes as the population:
    per round, N = (B - E) / 2 antithetic pairs (episode 2i at theta + sigma eps_i, 2i + 1 at theta - sigma eps_i) and E eval
    episodes at theta, one weight set per episode in one batch; rounds repeat until episodes_per_batch noisy episodes and
    train_batch_size noisy env-steps were collected; then centered ranks, the noise-weighted sum and optimizers.Adam on the
    device.  The Adam state is this learner's own: the policy's (DevicePPOLearner / DeviceIMPALALearner) is left alone."""

    def __init__(self, policy, config: ESConfig = None, noise: np.ndarray = None):
        """policy: a DeviceGNNPolicy, whose weights the learner updates in place.  noise: the shared noise table (float32); None
        draws shared_noise_table(config.noise_size)."""
        self.policy = policy
        self.config = dataclasses.replace(config) if config is not None else ESConfig()
        if self.config.observation_filter != 'NoFilter':
            raise ValueError(f"observation_filter {self.config.observation_filter!r}: only 'NoFilter' is supported (MeanStdFilter would "
                             'standardise the padded edge indices and the action mask the GNN reads back from the observation)')
        self._L = policy._L
        _bind(self._L)
        noise = shared_noise_table(self.config.noise_size) if noise is None else np.ascontiguousarray(noise, dtype=np.float32).ravel()
        self.noise_size = len(noise)
        self._h = C.c_void_p()
        _engine._check(self._L.ramp_es_create(policy._h, noise.ctypes.data, self.noise_size, C.byref(self._h)))
        self._B = 0

    def close(self):
        if getattr(self, '_h', None):
            self._L.ramp_es_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def n_eval(self, B: int) -> int:
        """eval episodes per round of a B-episode environment (es_n_eval)"""
        return es_n_eval(self.config, B)

    def _c(self, B: int) -> _CESConfig:
        return _c_struct(_CESConfig, self.config, n_eval=self.n_eval(B))

    def begin_round(self, env, rnd: int):
        """after env.reset(): round rnd's noise indices, weight sets and embeddings (round 0 starts a new step)"""
        B = self._B = env.B
        if B - self.n_eval(B) < 2:
            raise ValueError(f'{B} episodes less {self.n_eval(B)} eval episodes leave no antithetic pair')
        _engine._check(self._L.ramp_es_round_begin(self._h, env.eng._h, C.byref(self._c(B)), int(rnd)))

    def act(self, env, t: int):
        """env-step t of the round: every episode's sampled action from its own weight set into the environment's action buffer"""
        _engine._check(self._L.ramp_es_act(self._h, env.eng._h, int(t)))

    def end_round(self, env) -> bool:
        """the round's returns and env-steps into the step record; True while another round is needed"""
        more = C.c_int32()
        _engine._check(self._L.ramp_es_round_end(self._h, env.eng._h, C.byref(more)))
        return bool(more.value)

    def step(self) -> Dict[str, float]:
        """the update on the step record of the rounds since the last begin_round(env, 0) (ranks, g, Adam); ES_STATS"""
        out = np.zeros(len(ES_STATS), dtype=np.float64)
        _engine._check(self._L.ramp_es_step(self._h, C.byref(self._c(self._B)), out.ctypes.data))
        return _stats(ES_STATS, out)

    def learn(self, env, timing: bool = False) -> Dict[str, float]:
        """One ES training step (ES_STATS); see _es_learn."""
        return _es_learn(self, env, timing)

    def update(self, noise_index, returns):
        """the update on host inputs: noise_index [n], returns [n, 2] (R+, R-) -> (ES_STATS, ranks [n, 2], g [n_weights]); theta
        and the Adam state change as in learn()"""
        idx = np.ascontiguousarray(noise_index, dtype=np.int32).ravel()
        ret = np.ascontiguousarray(returns, dtype=np.float32).reshape(len(idx), 2)
        ranks = np.zeros((len(idx), 2), np.float32)
        g = np.zeros(self._L.ramp_policy_weight_count(C.byref(self.policy._cfg)), np.float32)
        out = np.zeros(len(ES_STATS), dtype=np.float64)
        _engine._check(self._L.ramp_es_update(self._h, C.byref(self._c(2 * len(idx) + 1)), len(idx), idx.ctypes.data, ret.ctypes.data,
                                              ranks.ctypes.data, g.ctypes.data, out.ctypes.data))
        return _stats(ES_STATS, out), ranks, g

    def last_step(self) -> Dict[str, np.ndarray]:
        """the last step's record: noise_index [n], returns and lengths [n, 2], the act seeds in order (round-major, env-step t of
        a round at r J + t), ranks [n, 2], g, eval_returns and eval_lengths"""
        n, ne, ns = C.c_int32(), C.c_int32(), C.c_int32()
        _engine._check(self._L.ramp_es_read(self._h, C.byref(n), C.byref(ne), C.byref(ns), *([None] * 9)))
        n, ne, ns = n.value, ne.value, ns.value
        out = dict(noise_index=np.zeros(n, np.int32), returns=np.zeros((n, 2), np.float32), lengths=np.zeros((n, 2), np.int32),
                   seeds=np.zeros(ns, np.uint64), ranks=np.zeros((n, 2), np.float32),
                   g=np.zeros(self._L.ramp_policy_weight_count(C.byref(self.policy._cfg)), np.float32),
                   eval_returns=np.zeros(ne, np.float32), eval_lengths=np.zeros(ne, np.int32))
        _engine._check(self._L.ramp_es_read(self._h, None, None, None, *[a.ctypes.data for a in out.values()]))
        return out

    def act_read(self, env):
        """the last act's logits [B, |A|], log-probabilities [B] and actions [B]"""
        B, A = env.B, self.policy.n_actions
        logits, logp, actions = np.zeros((B, A), np.float32), np.zeros(B, np.float32), np.zeros(B, np.int32)
        _engine._check(self._L.ramp_es_act_read(self._h, env.eng._h, logits.ctypes.data, logp.ctypes.data, actions.ctypes.data))
        return logits, logp, actions

    def adam_state(self):
        """optimizers.Adam's m, v (blob order) and t"""
        n = self._L.ramp_policy_weight_count(C.byref(self.policy._cfg))
        m, v, t = np.zeros(n, np.float32), np.zeros(n, np.float32), C.c_int32()
        _engine._check(self._L.ramp_es_state(self._h, m.ctypes.data, v.ctypes.data, C.byref(t)))
        return m, v, t.value

    def reset(self):
        """zero the ES Adam state"""
        _engine._check(self._L.ramp_es_reset(self._h))

    def training_state(self) -> Dict:
        """everything the next step depends on besides the config and the noise table: theta, the ES Adam state (m, v, t), the
        iteration count (it keys the noise indices and act seeds) and the steps' mean eval returns (episode_reward_mean's
        window).  np.savez of the dict is a checkpoint."""
        m, v, t = self.adam_state()
        it, means = _es_progress(self._L.ramp_es_get_progress, self._h)
        return dict(weights=self.policy.get_weights(), m=m, v=v, t=t, iteration=it, eval_means=means)

    def load_training_state(self, state):
        """resume from a training_state(): this learner, made with the saving one's config and noise table, then steps as it would"""
        n = self._L.ramp_policy_weight_count(C.byref(self.policy._cfg))
        w, m, v = (_state_array(state, key, n) for key in ('weights', 'm', 'v'))
        means = np.ascontiguousarray(state['eval_means'], dtype=np.float64).ravel()
        self.policy.set_weights(w)
        _engine._check(self._L.ramp_es_set_state(self._h, m.ctypes.data, v.ctypes.data, n, int(state['t'])))
        _engine._check(self._L.ramp_es_set_progress(self._h, int(state['iteration']), len(means), means.ctypes.data))


class DevicePopulationESLearner(_PopulationLearner):
    """DeviceESLearner for every set of a DeviceGNNPolicyPopulation at once (include/ramp_b200.h: ramp_population_es_*): group k
    of the environment's B = K b episodes is set k's ES population, N_k = (b - E_k) / 2 antithetic pairs and E_k eval episodes
    with configs[k], and ends each step where a DeviceESLearner(population.policy(k), configs[k]) ends on a b-episode environment
    with the same episode streams, bit for bit: the step record, the statistics, the weights and the ES Adam state.  A group stops
    collecting after the round its twin would stop after (rounds_k of them); the population runs rounds until every group has
    stopped, and in the later rounds a stopped group's episodes all run its unperturbed weights and count for nothing.  The
    population's torch-Adam state (DevicePopulationPPOLearner's) is not touched; the ES Adam state is this learner's own.  One
    shared noise table serves every set, so noise_size must be the same in every config."""
    _checks = (('noise_stdev', lambda v: v >= 0, '>= 0'), ('stepsize', lambda v: v >= 0, '>= 0'), ('adam_eps', lambda v: v > 0, '> 0'),
               ('adam_beta1', lambda v: 0 <= v < 1, 'in [0, 1)'), ('adam_beta2', lambda v: 0 <= v < 1, 'in [0, 1)'),
               ('episodes_per_batch', lambda v: v >= 0, '>= 0'), ('train_batch_size', lambda v: v >= 0, '>= 0'),
               ('report_length', lambda v: v >= 1, '>= 1'), ('observation_filter', lambda v: v == 'NoFilter',
                                                              "'NoFilter' (MeanStdFilter would standardise the padded edge indices and "
                                                              'the action mask the GNN reads back from the observation)'),
               ('n_eval', lambda v: v is None or v >= 0, 'None or >= 0'))

    def __init__(self, population, configs, noise: np.ndarray = None):
        """population: a DeviceGNNPolicyPopulation, whose sets the learner updates in place; configs: one ESConfig per set.  noise:
        the shared noise table (float32); None draws shared_noise_table(noise_size)."""
        super().__init__(population, configs)
        sizes = [c.noise_size for c in self.configs]
        if len(set(sizes)) > 1:
            k = next(k for k, v in enumerate(sizes) if v != sizes[0])
            raise ValueError(f'noise_size must be the same for every set (one noise table serves them all): {sizes}; set {k} differs '
                             'from set 0')
        noise = shared_noise_table(sizes[0]) if noise is None else np.ascontiguousarray(noise, dtype=np.float32).ravel()
        self.noise_size = len(noise)
        for k in range(population.K):
            if population.weight_count(k) > self.noise_size:
                raise ValueError(f'set {k}: a noise table of {self.noise_size} floats is smaller than its {population.weight_count(k)} weights')
        self._h = C.c_void_p()
        _engine._check(self._L.ramp_population_es_create(population._h, noise.ctypes.data, self.noise_size, C.byref(self._h)))
        self._B = 0

    def close(self):
        if getattr(self, '_h', None):
            self._L.ramp_population_es_destroy(self._h)
            self._h = None

    def _handle(self):
        """the learner's handle; every call but close() reads the population's sets, so both must still be open"""
        if not getattr(self, '_h', None):
            raise RuntimeError('the ES learner is closed')
        if not self.population._h:
            raise RuntimeError('the population was closed before its ES learner')
        return self._h

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def n_eval(self, b: int):
        """each group's eval episodes per round when a group has b episodes (es_n_eval)"""
        return [es_n_eval(c, b) for c in self.configs]

    def _c(self, B: int):
        b = B // self.population.K
        cfgs = [_c_struct(_CESConfig, c, n_eval=E) for c, E in zip(self.configs, self.n_eval(b))]
        return (_CESConfig * self.population.K)(*cfgs)

    def _check_groups(self, b: int):
        for k, E in enumerate(self.n_eval(b)):
            if b - E < 2 or (b - E) & 1:
                raise ValueError(f'set {k}: {b} episodes per group less {E} eval episodes leave {b - E}, which must be even and >= 2')

    def begin_round(self, env, rnd: int):
        """after env.reset(): round rnd's noise indices, weight sets and embeddings of every group still collecting (round 0 starts
        a new step)"""
        self._check_groups(self.population.group_size(env))
        self._B = env.B
        _engine._check(self._L.ramp_population_es_round_begin(self._handle(), env.eng._h, self._c(env.B), int(rnd)))

    def act(self, env, t: int):
        """env-step t of the round: every episode's sampled action from its own weight set"""
        _engine._check(self._L.ramp_population_es_act(self._handle(), env.eng._h, int(t)))

    def end_round(self, env) -> bool:
        """the round's returns and env-steps into the records of the groups that ran pairs; True while any group needs more"""
        more = C.c_int32()
        _engine._check(self._L.ramp_population_es_round_end(self._handle(), env.eng._h, C.byref(more)))
        return bool(more.value)

    def step(self):
        """every set's update on its step record: a list of K ES_STATS dicts; stats[k]['rounds'] is group k's rounds"""
        out = np.zeros((self.population.K, len(ES_STATS)), dtype=np.float64)
        _engine._check(self._L.ramp_population_es_step(self._handle(), self._c(self._B), out.ctypes.data))
        return [_stats(ES_STATS, row) for row in out]

    learn = _es_learn

    def update(self, noise_index, returns):
        """the update on host inputs, per set: noise_index[k] [n_k], returns[k] [n_k, 2] -> a list of K (ES_STATS, ranks [n_k, 2],
        g), as DeviceESLearner.update gives them for set k"""
        K = self.population.K
        if len(noise_index) != K or len(returns) != K:
            raise ValueError(f'{len(noise_index)} noise index lists and {len(returns)} return lists for {K} sets')
        idx = [np.ascontiguousarray(i, dtype=np.int32).ravel() for i in noise_index]
        ret = [np.ascontiguousarray(r, dtype=np.float32).reshape(len(i), 2) for i, r in zip(idx, returns)]
        n = np.array([len(i) for i in idx], np.int32)
        for k in range(K):
            if n[k] < 1:
                raise ValueError(f'set {k}: an update needs at least one pair')
        flat_i, flat_r = np.concatenate(idx), np.ascontiguousarray(np.concatenate(ret))
        out = np.zeros((K, len(ES_STATS)), dtype=np.float64)
        _engine._check(self._L.ramp_population_es_update(self._handle(), self._c(K * (2 * int(n.max()) + 1)), n.ctypes.data, flat_i.ctypes.data,
                                                         flat_r.ctypes.data, out.ctypes.data))
        res = []
        for k in range(K):
            rec = self.last_step(k)
            res.append((_stats(ES_STATS, out[k]), rec['ranks'], rec['g']))
        return res

    def last_step(self, k: int) -> Dict[str, np.ndarray]:
        """set k's last step record, as DeviceESLearner.last_step gives its own"""
        k = self.population._set(k)
        n, ne, ns = C.c_int32(), C.c_int32(), C.c_int32()
        _engine._check(self._L.ramp_population_es_read(self._handle(), k, C.byref(n), C.byref(ne), C.byref(ns), *([None] * 9)))
        n, ne, ns = n.value, ne.value, ns.value
        out = dict(noise_index=np.zeros(n, np.int32), returns=np.zeros((n, 2), np.float32), lengths=np.zeros((n, 2), np.int32),
                   seeds=np.zeros(ns, np.uint64), ranks=np.zeros((n, 2), np.float32), g=np.zeros(self.population.weight_count(k), np.float32),
                   eval_returns=np.zeros(ne, np.float32), eval_lengths=np.zeros(ne, np.int32))
        _engine._check(self._L.ramp_population_es_read(self._handle(), k, None, None, None, *[a.ctypes.data for a in out.values()]))
        return out

    def act_read(self, env):
        """the last act's logits [B, |A|], log-probabilities [B] and actions [B]"""
        B, A = env.B, self.population.n_actions
        logits, logp, actions = np.zeros((B, A), np.float32), np.zeros(B, np.float32), np.zeros(B, np.int32)
        _engine._check(self._L.ramp_population_es_act_read(self._handle(), env.eng._h, logits.ctypes.data, logp.ctypes.data, actions.ctypes.data))
        return logits, logp, actions

    def adam_state(self, k: int):
        """set k's optimizers.Adam m, v (blob order) and t"""
        k = self.population._set(k)
        n = self.population.weight_count(k)
        m, v, t = np.zeros(n, np.float32), np.zeros(n, np.float32), C.c_int32()
        _engine._check(self._L.ramp_population_es_state(self._handle(), k, m.ctypes.data, v.ctypes.data, C.byref(t)))
        return m, v, t.value

    def reset(self):
        """zero every set's ES Adam state"""
        _engine._check(self._L.ramp_population_es_reset(self._handle()))

    def training_state(self, k: int) -> Dict:
        """set k's training state, as DeviceESLearner.training_state(); the iteration count is the learner's, one for every set"""
        k = self.population._set(k)
        m, v, t = self.adam_state(k)
        it, means = _es_progress(self._L.ramp_population_get_es_progress, self._handle(), k)
        return dict(weights=self.population.get_weights(k), m=m, v=v, t=t, iteration=it, eval_means=means)

    def load_training_state(self, k: int, state):
        """set k resumes from a training_state (a population's set or a DeviceESLearner's of the same shape).  The iteration
        count is one for every set: loading it through any set sets it for all."""
        k = self.population._set(k)
        n = self.population.weight_count(k)
        w, m, v = (_state_array(state, key, n) for key in ('weights', 'm', 'v'))
        means = np.ascontiguousarray(state['eval_means'], dtype=np.float64).ravel()
        self.population.set_weights(k, w)
        _engine._check(self._L.ramp_population_set_es_state(self._handle(), k, m.ctypes.data, v.ctypes.data, n, int(state['t'])))
        _engine._check(self._L.ramp_population_set_es_progress(self._handle(), k, int(state['iteration']), len(means), means.ctypes.data))

    def copy_sets(self, dst, src):
        """population.copy_sets' exploit for this learner's own state: set src[i]'s ES Adam state and mean eval returns onto set
        dst[i], with the same checks.  The weights are the population's: population.copy_sets copies them."""
        d = np.ascontiguousarray(dst, dtype=np.int32).ravel()
        s = np.ascontiguousarray(src, dtype=np.int32).ravel()
        if len(d) != len(s):
            raise ValueError(f'{len(d)} destinations for {len(s)} sources')
        _engine._check(self._L.ramp_population_copy_es_sets(self._handle(), len(d), d.ctypes.data, s.ctypes.data))

    def embed_ctas(self):
        """the last round's embedding launch: (CTAs, (ES weight set, job type) items); each CTA runs items c, c + ctas, ..."""
        ctas, items = C.c_int32(), C.c_int32()
        _engine._check(self._L.ramp_population_es_embed_ctas(self._handle(), C.byref(ctas), C.byref(items)))
        return ctas.value, items.value
