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


def c_config(cfg: PPOConfig) -> _CConfig:
    c = _CConfig()
    for f in _CConfig._fields_:
        v = getattr(cfg, f[0])
        setattr(c, f[0], int(v) & (2 ** 64 - 1) if f[0] == 'seed' else (int(v) if f[1] is C.c_int32 else float(v)))
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


def c_impala_config(cfg: IMPALAConfig) -> _CIMPALAConfig:
    c = _CIMPALAConfig()
    for name, ct in _CIMPALAConfig._fields_:
        setattr(c, name, int(getattr(cfg, name)) if ct is C.c_int32 else float(getattr(cfg, name)))
    return c


def _bind(L):
    if getattr(L, '_learn_bound', False):
        return
    L.ramp_ppo_loss_grad.restype = C.c_int
    L.ramp_ppo_loss_grad.argtypes = [C.c_void_p, C.POINTER(_CConfig), C.c_int32] + [C.c_void_p] * 9
    L.ramp_policy_learn.restype = C.c_int
    L.ramp_policy_learn.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(_CConfig), C.c_void_p]
    L.ramp_policy_train_batch_read.restype = C.c_int
    L.ramp_policy_train_batch_read.argtypes = [C.c_void_p, C.c_void_p] + [C.c_void_p] * 7
    L.ramp_policy_learner_state.restype = C.c_int
    L.ramp_policy_learner_state.argtypes = [C.c_void_p] * 4
    L.ramp_policy_learner_reset.restype = C.c_int
    L.ramp_policy_learner_reset.argtypes = [C.c_void_p]
    L.ramp_impala_loss_grad.restype = C.c_int
    L.ramp_impala_loss_grad.argtypes = [C.c_void_p, C.POINTER(_CIMPALAConfig), C.c_int32, C.c_int32] + [C.c_void_p] * 12
    L.ramp_policy_learn_impala.restype = C.c_int
    L.ramp_policy_learn_impala.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(_CIMPALAConfig), C.c_void_p]
    L.ramp_impala_vtrace_read.restype = C.c_int
    L.ramp_impala_vtrace_read.argtypes = [C.c_void_p] * 6
    L._learn_bound = True


def _stats(raw) -> Dict[str, float]:
    return {k: float(v) for k, v in zip(STATS, raw)}


class DevicePPOLearner:
    def __init__(self, policy, config: PPOConfig = None):
        """policy: a DeviceGNNPolicy, whose weights the learner updates in place (Adam's state lives with the policy)."""
        self.policy = policy
        self.config = dataclasses.replace(config) if config is not None else PPOConfig()
        self._L = policy._L
        _bind(self._L)
        self._calls = 0

    def collect_and_learn(self, env, horizon: int, seed: int = 0) -> Dict[str, float]:
        """policy.collect(env, horizon) then learn(); also returns the wall time of each (seconds) and the segment's trajectory."""
        t0 = time.perf_counter()
        traj = self.policy.collect(env, horizon, sample=True, seed=seed)
        t1 = time.perf_counter()
        stats = self.learn(env, horizon)
        stats['collect_s'], stats['learn_s'] = t1 - t0, time.perf_counter() - t1
        return stats, traj

    def learn(self, env, horizon: int) -> Dict[str, float]:
        """One PPO learner step on the first ``horizon`` steps of the segment the policy's last collect(env, ...) recorded (a shorter
        horizon bootstraps its advantages with the value recorded at the next step): the statistics averaged over the
        last pass's minibatches (STATS); kl_coeff is the adapted coefficient, which this learner uses from the next call on.
        Call k of this learner shuffles with the seed config.seed + k."""
        cfg = dataclasses.replace(self.config, seed=self.config.seed + self._calls)
        out = np.zeros(len(STATS), dtype=np.float64)
        _engine._check(self._L.ramp_policy_learn(self.policy._h, env.eng._h, int(horizon), C.byref(c_config(cfg)), out.ctypes.data))
        self._calls += 1
        stats = _stats(out)
        self.config.kl_coeff = stats['kl_coeff']
        return stats

    def train_batch(self, env) -> Dict[str, np.ndarray]:
        """the last learn()'s train batch: per live row, t-major, the job type, action, collected log-probability, the one
        recomputed from the collection weights, the advantage (standardised when configured) and the value target"""
        cap = self.policy._traj_key[0] * env.B            # the segment's rows: (horizon, B, |A|) of the last collect()
        n = C.c_int32()
        arrs = {'model': np.zeros(cap, np.int32), 'action': np.zeros(cap, np.int32), 'logp': np.zeros(cap, np.float32),
                'logp_old': np.zeros(cap, np.float32), 'advantage': np.zeros(cap, np.float32), 'value_target': np.zeros(cap, np.float32)}
        _engine._check(self._L.ramp_policy_train_batch_read(self.policy._h, env.eng._h, C.byref(n), *[a.ctypes.data for a in arrs.values()]))
        return {k: v[:n.value].copy() for k, v in arrs.items()}

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
        _engine._check(self._L.ramp_ppo_loss_grad(pol._h, C.byref(c_config(self.config)), n, model.ctypes.data, gf.ctypes.data,
                                                  mask.ctypes.data, act.ctypes.data, old.ctypes.data, adv.ctypes.data, vt.ctypes.data,
                                                  grad.ctypes.data, out.ctypes.data))
        return _stats(out), grad

    def adam_state(self):
        """torch.optim.Adam's state of the flat weight vector: exp_avg, exp_avg_sq (blob order) and the step count"""
        n = self._L.ramp_policy_weight_count(C.byref(self.policy._cfg))
        m, v, step = np.zeros(n, np.float32), np.zeros(n, np.float32), C.c_int32()
        _engine._check(self._L.ramp_policy_learner_state(self.policy._h, m.ctypes.data, v.ctypes.data, C.byref(step)))
        return m, v, step.value

    def reset(self):
        """zero Adam's moments and step count"""
        _engine._check(self._L.ramp_policy_learner_reset(self.policy._h))


class DeviceIMPALALearner:
    """RLlib's IMPALA learner step (V-trace, VTraceLoss, clip_grad_norm_, Adam) on the segment the policy's last collect()
    recorded, on the device.  Adam's moments and step count are the policy's, shared with DevicePPOLearner."""

    def __init__(self, policy, config: IMPALAConfig = None):
        """policy: a DeviceGNNPolicy, whose weights the learner updates in place"""
        self.policy = policy
        self.config = dataclasses.replace(config) if config is not None else IMPALAConfig()
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

    def learn(self, env, horizon: int) -> Dict[str, float]:
        """One IMPALA learner step on the first ``horizon`` steps of the segment the policy's last collect(env, ...) recorded: the
        fragments of rollout_fragment_length rows (0: horizon), one Adam step per train batch of train_batch_size // L fragments,
        in order.  Returns the means over the call's SGD steps (IMPALA_STATS), and their number as sgd_steps."""
        out = np.zeros(len(IMPALA_STATS), dtype=np.float64)
        _engine._check(self._L.ramp_policy_learn_impala(self.policy._h, env.eng._h, int(horizon), C.byref(c_impala_config(self.config)),
                                                        out.ctypes.data))
        return {k: float(v) for k, v in zip(IMPALA_STATS, out)}

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
        _engine._check(self._L.ramp_impala_loss_grad(pol._h, C.byref(c_impala_config(self.config)), int(n), int(L), model.ctypes.data,
                                                     gf.ctypes.data, mask.ctypes.data, act.ctypes.data, blogp.ctypes.data,
                                                     reward.ctypes.data, done.ctypes.data, grad.ctypes.data, out.ctypes.data,
                                                     *[a.ctypes.data for a in vt.values()]))
        return {k: float(v) for k, v in zip(IMPALA_STATS, out)}, grad, {k: v.reshape(n, L) for k, v in vt.items()}

    def adam_state(self):
        """torch.optim.Adam's state of the flat weight vector (the policy's, shared with DevicePPOLearner)"""
        return DevicePPOLearner.adam_state(self)

    def reset(self):
        """zero Adam's moments and step count"""
        _engine._check(self._L.ramp_policy_learner_reset(self.policy._h))


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


def c_pg_config(cfg: PGConfig) -> _CPGConfig:
    return _CPGConfig(*(float(getattr(cfg, n)) for n, _ in _CPGConfig._fields_))


def _bind_pg(L):
    if getattr(L, '_pg_bound', False):
        return
    _bind(L)
    L.ramp_pg_loss_grad.restype = C.c_int
    L.ramp_pg_loss_grad.argtypes = [C.c_void_p, C.POINTER(_CPGConfig), C.c_int32] + [C.c_void_p] * 7
    L.ramp_policy_learn_pg.restype = C.c_int
    L.ramp_policy_learn_pg.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(_CPGConfig), C.c_void_p]
    L._pg_bound = True


class DevicePGLearner:
    """RLlib's PG learner step (discounted returns, pg_torch_loss, Adam) on the segment the policy's last collect() recorded, on
    the device.  Adam's moments and step count are the policy's, shared with DevicePPOLearner and DeviceIMPALALearner."""

    def __init__(self, policy, config: PGConfig = None):
        """policy: a DeviceGNNPolicy, whose weights the learner updates in place"""
        self.policy = policy
        self.config = dataclasses.replace(config) if config is not None else PGConfig()
        self._L = policy._L
        _bind_pg(self._L)

    def collect_and_learn(self, env, horizon: int, seed: int = 0):
        """policy.collect(env, horizon) then learn(); also returns the wall time of each (seconds) and the segment's trajectory."""
        t0 = time.perf_counter()
        traj = self.policy.collect(env, horizon, sample=True, seed=seed)
        t1 = time.perf_counter()
        stats = self.learn(env, horizon)
        stats['collect_s'], stats['learn_s'] = t1 - t0, time.perf_counter() - t1
        return stats, traj

    def learn(self, env, horizon: int) -> Dict[str, float]:
        """One PG learner step on the first ``horizon`` steps of the segment the policy's last collect(env, ...) recorded: one train
        batch of every decision of the segment, one Adam step.  Each episode's advantage is its discounted return; a segment that
        ends before its episode does is not bootstrapped (PG's last_r is 0).  There is no train_batch_size: under RLlib's
        batch_mode complete_episodes a train batch is whole episodes, so the caller sizes env.B and the horizon so that the
        segment holds the env-steps it wants per update (pg's train_batch_size is 200) and its episodes end inside it.  Returns
        PG_STATS; a segment with no decision makes no update and leaves Adam's step count as it was."""
        out = np.zeros(len(PG_STATS), dtype=np.float64)
        _engine._check(self._L.ramp_policy_learn_pg(self.policy._h, env.eng._h, int(horizon), C.byref(c_pg_config(self.config)),
                                                    out.ctypes.data))
        return {k: float(v) for k, v in zip(PG_STATS, out)}

    def train_batch(self, env) -> Dict[str, np.ndarray]:
        """the last learn()'s train batch: per live row, t-major, the job type, action, collected log-probability, the one the
        gradient kernel recomputed at the collection weights (logp_old) and the discounted return (advantage, value_target)"""
        return DevicePPOLearner.train_batch(self, env)

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
        _engine._check(self._L.ramp_pg_loss_grad(pol._h, C.byref(c_pg_config(self.config)), n, model.ctypes.data, gf.ctypes.data,
                                                 mask.ctypes.data, act.ctypes.data, adv.ctypes.data, grad.ctypes.data, out.ctypes.data))
        return {k: float(v) for k, v in zip(PG_STATS, out)}, grad

    def adam_state(self):
        """torch.optim.Adam's state of the flat weight vector (the policy's, shared with DevicePPOLearner)"""
        return DevicePPOLearner.adam_state(self)

    def reset(self):
        """zero Adam's moments and step count"""
        _engine._check(self._L.ramp_policy_learner_reset(self.policy._h))


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


def shared_noise_table(size: int) -> np.ndarray:
    """RLlib's shared noise table (es.py create_shared_noise), bit for bit.  At the default size it takes seconds and 1 GB as
    float32 (2 GB more while numpy draws it in float64)."""
    return np.random.RandomState(123).randn(int(size)).astype(np.float32)


def _bind_es(L):
    if getattr(L, '_es_bound', False):
        return
    for name, args in (('ramp_es_create', [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
                       ('ramp_es_round_begin', [C.c_void_p, C.c_void_p, C.POINTER(_CESConfig), C.c_int32]),
                       ('ramp_es_act', [C.c_void_p, C.c_void_p, C.c_int32]),
                       ('ramp_es_round_end', [C.c_void_p, C.c_void_p, C.c_void_p]),
                       ('ramp_es_step', [C.c_void_p, C.POINTER(_CESConfig), C.c_void_p]),
                       ('ramp_es_update', [C.c_void_p, C.POINTER(_CESConfig), C.c_int32] + [C.c_void_p] * 5),
                       ('ramp_es_read', [C.c_void_p] * 12),
                       ('ramp_es_act_read', [C.c_void_p] * 5),
                       ('ramp_es_state', [C.c_void_p] * 4),
                       ('ramp_es_reset', [C.c_void_p])):
        getattr(L, name).restype = C.c_int
        getattr(L, name).argtypes = args
    L.ramp_es_destroy.restype = None
    L.ramp_es_destroy.argtypes = [C.c_void_p]
    L._es_bound = True


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
        _bind_es(self._L)
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
        """eval episodes per round of a B-episode environment: config.n_eval, else RLlib's expected share of eval episodes
        B eval_prob / (2 - eval_prob), at least 1, plus one when B - E would be odd"""
        if self.config.n_eval is not None:
            return int(self.config.n_eval)
        p = self.config.eval_prob
        E = max(1, int(round(B * p / (2.0 - p))))
        return E + ((B - E) & 1)

    def _c(self, B: int) -> _CESConfig:
        c = self.config
        return _CESConfig(int(c.seed) & (2 ** 64 - 1), float(c.noise_stdev), float(c.stepsize), float(c.l2_coeff), float(c.adam_beta1),
                          float(c.adam_beta2), float(c.adam_eps), int(c.episodes_per_batch), int(c.train_batch_size), self.n_eval(B),
                          int(c.report_length))

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
        return {k: float(v) for k, v in zip(ES_STATS, out)}

    def learn(self, env, timing: bool = False) -> Dict[str, float]:
        """One ES training step (ES_STATS).  Each round resets env and runs env.J env-steps, so every episode ends in it; the
        round synchronises once, at its end.  timing=True also synchronises after the embeddings and adds the wall time (seconds)
        of the embeddings (embed_s), of the rollouts (rollout_s) and of the update (update_s)."""
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
            stats.update(times, update_s=time.perf_counter() - t3)
        return stats

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
        return {k: float(v) for k, v in zip(ES_STATS, out)}, ranks, g

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
