"""ctypes binding of the C ABI in include/ramp_b200.h (ddls_b200/libramp_b200.so).

This is the only way the Python host side reaches the simulator: there is no CPU fallback.  If the
shared library is missing or CUDA is unavailable, importing/constructing raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .lowered import LoweredJob

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libramp_b200.so')

RAMP_OK = 0
MEMO_REFERENCE, MEMO_EXACT, MEMO_OFF, MEMO_SHARED = 0, 1, 2, 3
ACT_SKIP = 1

STEP_STATS = [
    'step_counter', 'step_start_time', 'step_end_time', 'step_time', 'num_jobs_completed', 'num_jobs_arrived',
    'num_jobs_blocked', 'job_queue_length', 'mean_num_jobs_running', 'mean_num_mounted_workers',
    'mean_num_mounted_channels', 'mean_compute_overhead_frac', 'mean_communication_overhead_frac',
    'compute_info_processed', 'dep_info_processed', 'flow_info_processed', 'cluster_info_processed',
    'demand_compute_info_processed', 'demand_dep_info_processed', 'demand_total_info_processed',
    'mean_compute_throughput', 'mean_dep_throughput', 'mean_flow_throughput', 'mean_cluster_throughput',
    'mean_demand_compute_throughput', 'mean_demand_dep_throughput', 'mean_demand_total_throughput',
    'util_mounted_sum', 'util_cluster_sum', 'num_ticks', 'done', 'lookahead_ran']
SS = {k: i for i, k in enumerate(STEP_STATS)}
STEP_STATS_LEN = len(STEP_STATS)

EP_FIELDS = ['time', 'next_arrival', 'num_arrived', 'num_completed', 'num_blocked', 'queued_job', 'num_running',
             'step_counter', 'load_rate_sum', 'load_rate_n', 'done', 'status']
EP = {k: i for i, k in enumerate(EP_FIELDS)}
EP_LEN = len(EP_FIELDS)

# RampClusterEnvironment.episode_stats' scalars (RCE:1123-1167), include/ramp_b200.h RAMP_ES_*: the reference's names, plus the
# number of cluster steps and ticks the means run over and the done flag
ES_FIELDS = ['episode_start_time', 'episode_end_time', 'episode_time', 'num_jobs_arrived', 'num_jobs_completed', 'num_jobs_blocked',
             'mean_load_rate', 'blocking_rate', 'acceptance_rate',
             'compute_info_processed', 'dep_info_processed', 'flow_info_processed', 'cluster_info_processed',
             'demand_compute_info_processed', 'demand_dep_info_processed', 'demand_total_info_processed',
             'mean_compute_throughput', 'mean_dep_throughput', 'mean_flow_throughput', 'mean_cluster_throughput',
             'mean_demand_compute_throughput', 'mean_demand_dep_throughput', 'mean_demand_total_throughput',
             'mean_compute_overhead_frac', 'mean_communication_overhead_frac', 'mean_num_jobs_running', 'mean_num_mounted_workers',
             'mean_mounted_worker_utilisation_frac', 'mean_cluster_worker_utilisation_frac', 'num_cluster_steps', 'num_ticks', 'done']
ES = {k: i for i, k in enumerate(ES_FIELDS)}
ES_LEN = len(ES_FIELDS)
ES_COUNTS = ('num_jobs_arrived', 'num_jobs_completed', 'num_jobs_blocked', 'num_cluster_steps', 'num_ticks')

# EvalLoop's results['step_stats'] row of one env-step (loops/eval_loop.py:50-100), include/ramp_b200.h RAMP_ESS_*: the keys of the
# cluster's steps_log in the order it first sees them; ENV_STEP_COUNTS are integers in the reference
ENV_STEP_STATS = ['step_counter', 'step_start_time', 'mean_num_mounted_workers', 'mean_num_mounted_channels', 'mean_compute_throughput',
                  'mean_dep_throughput', 'mean_cluster_throughput', 'mean_demand_compute_throughput', 'mean_demand_dep_throughput',
                  'mean_demand_total_throughput', 'mean_compute_overhead_frac', 'mean_communication_overhead_frac',
                  'mean_mounted_worker_utilisation_frac', 'mean_cluster_worker_utilisation_frac', 'num_jobs_completed',
                  'mean_num_jobs_running', 'num_jobs_arrived', 'num_jobs_blocked', 'compute_info_processed', 'dep_info_processed',
                  'flow_info_processed', 'cluster_info_processed', 'demand_compute_info_processed', 'demand_dep_info_processed',
                  'demand_total_info_processed', 'step_end_time', 'step_time', 'mean_flow_throughput', 'job_queue_length']
ENV_STEP_STATS_LEN = len(ENV_STEP_STATS)
ENV_STEP_COUNTS = ('step_counter', 'num_jobs_completed', 'num_jobs_arrived', 'num_jobs_blocked', 'job_queue_length')


def env_step_columns(rows):
    """{name: rows[..., i]} for the RAMP_ESS_* columns of `rows` (last axis ENV_STEP_STATS_LEN), the counts as int64."""
    return {k: rows[..., i].astype(np.int64) if k in ENV_STEP_COUNTS else rows[..., i].copy() for i, k in enumerate(ENV_STEP_STATS)}

JS_NOT_ARRIVED, JS_QUEUED, JS_RUNNING, JS_COMPLETED, JS_BLOCKED = range(5)

ACTION_DTYPE = np.dtype([('max_acceptable_jct', np.float64), ('part_op_mem', np.float64), ('part_dep_size', np.float64),
                         ('flow_size', np.float64), ('n_mounted_workers', np.int32), ('n_mounted_channels', np.int32),
                         ('template_id', np.int32), ('flags', np.int32)])
ARRIVAL_DTYPE = np.dtype([('interarrival', np.float64), ('orig_op_mem', np.float64), ('orig_dep_size', np.float64)])
JOB_RECORD_DTYPE = np.dtype([('status', np.int32), ('event_seq', np.int32), ('time_arrived', np.float64),
                             ('time_started', np.float64), ('time_completed', np.float64), ('jct', np.float64),
                             ('comm', np.float64), ('comp', np.float64), ('util', np.float64)])
LOOKAHEAD_RESULT_DTYPE = np.dtype([('jct', np.float64), ('comm', np.float64), ('comp', np.float64),
                                   ('n_ticks', np.int32), ('status', np.int32)])


class _Config(C.Structure):
    _fields_ = [('device', C.c_int32), ('n_episodes', C.c_int32), ('n_cluster_workers', C.c_int32),
                ('max_jobs', C.c_int32), ('max_running', C.c_int32), ('max_templates', C.c_int32),
                ('memo_mode', C.c_int32), ('memo_capacity_log2', C.c_int32), ('trace_cap', C.c_int32),
                ('job_queue_capacity', C.c_int32), ('machine_epsilon', C.c_double),
                ('max_simulation_run_time', C.c_double)]


class _LoweredJob(C.Structure):
    _fields_ = [('n_ops', C.c_int32), ('n_deps', C.c_int32), ('n_workers', C.c_int32), ('n_channels', C.c_int32),
                ('num_training_steps', C.c_int32), ('model_id', C.c_int32), ('degree', C.c_int32), ('_pad', C.c_int32),
                ('op_cost', C.c_void_p), ('op_prio', C.c_void_p), ('op_worker', C.c_void_p),
                ('op_n_parents', C.c_void_p), ('row_ptr', C.c_void_p), ('dep_dst', C.c_void_p),
                ('dep_run_time', C.c_void_p), ('dep_prio', C.c_void_p), ('dep_channel', C.c_void_p),
                ('dep_is_flow', C.c_void_p)]


_lib = None


def load_library():
    """Loads libramp_b200.so; raises if it has not been built (``python -m ddls_b200.build``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f'{LIB_PATH} is missing: the CUDA extension has not been built. Run '
                           f'`python -c "import __graft_entry__ as g; g.build()"` (there is no CPU fallback).')
    L = C.CDLL(LIB_PATH)
    L.ramp_last_error.restype = C.c_char_p
    L.ramp_engine_create.argtypes = [C.POINTER(_Config), C.POINTER(C.c_void_p)]
    L.ramp_engine_destroy.argtypes = [C.c_void_p]
    L.ramp_engine_stream.restype = C.c_void_p
    L.ramp_engine_stream.argtypes = [C.c_void_p]
    L.ramp_register_template.argtypes = [C.c_void_p, C.POINTER(_LoweredJob), C.POINTER(C.c_int32)]
    L.ramp_template_count.argtypes = [C.c_void_p]
    L.ramp_reset.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
    L.ramp_set_arrivals.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32]
    L.ramp_set_job_count.restype = C.c_int
    L.ramp_set_job_count.argtypes = [C.c_void_p, C.c_int32, C.c_int32]
    L.ramp_set_limits.restype = C.c_int
    L.ramp_set_limits.argtypes = [C.c_void_p, C.c_double, C.c_int32]
    L.ramp_step_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    L.ramp_step_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
    L.ramp_sync.argtypes = [C.c_void_p]
    L.ramp_check_status.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.ramp_get_job_records.argtypes = [C.c_void_p, C.c_void_p]
    L.ramp_get_episode_state.argtypes = [C.c_void_p, C.c_void_p]
    L.ramp_episode_state_device.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
    L.ramp_export_episode_state_to.argtypes = [C.c_void_p, C.c_void_p]
    L.ramp_get_episode_stats.argtypes = [C.c_void_p, C.c_void_p]
    L.ramp_get_memo_stats.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.ramp_get_memo_stats_ex.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    L.ramp_get_memo_speculative_unused.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
    L.ramp_get_lookahead_kernel_union.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
    L.ramp_get_last_lookahead.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32]
    L.ramp_run_lookaheads.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int32, C.POINTER(C.c_float)]
    L.ramp_debug_template_info.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_double)]
    L.ramp_launch_count.restype = C.c_int64
    L.ramp_launch_count.argtypes = [C.c_void_p]
    L.ramp_debug_device_bytes.argtypes = [C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    L.ramp_get_lookahead_kernel_time.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int64),
                                                 C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_int32]
    for name in ('ramp_engine_create', 'ramp_engine_destroy', 'ramp_register_template', 'ramp_template_count',
                 'ramp_reset', 'ramp_set_arrivals', 'ramp_step_host', 'ramp_step_device', 'ramp_sync', 'ramp_check_status',
                 'ramp_get_job_records', 'ramp_get_episode_state', 'ramp_episode_state_device', 'ramp_export_episode_state_to',
                 'ramp_get_episode_stats', 'ramp_get_memo_stats', 'ramp_get_memo_stats_ex', 'ramp_get_last_lookahead', 'ramp_run_lookaheads',
                 'ramp_debug_template_info', 'ramp_debug_device_bytes', 'ramp_get_lookahead_kernel_time',
                 'ramp_get_memo_speculative_unused', 'ramp_get_lookahead_kernel_union'):
        getattr(L, name).restype = C.c_int
    _lib = L
    return L


EXPORTED_SYMBOLS = ['ramp_last_error', 'ramp_engine_create', 'ramp_engine_destroy', 'ramp_engine_stream',
                    'ramp_register_template', 'ramp_template_count', 'ramp_reset', 'ramp_set_arrivals', 'ramp_step_host',
                    'ramp_step_device', 'ramp_sync', 'ramp_check_status', 'ramp_get_job_records',
                    'ramp_get_episode_state', 'ramp_episode_state_device', 'ramp_export_episode_state_to', 'ramp_get_episode_stats',
                    'ramp_get_memo_stats', 'ramp_get_memo_stats_ex', 'ramp_get_memo_speculative_unused', 'ramp_get_lookahead_kernel_union',
                    'ramp_get_last_lookahead', 'ramp_run_lookaheads', 'ramp_debug_template_info', 'ramp_launch_count', 'ramp_debug_device_bytes',
                    'ramp_get_lookahead_kernel_time', 'ramp_expand_template', 'ramp_free_expanded_job', 'ramp_free_expanded_aux', 'ramp_first_fit_place',
                    'ramp_quotient_template', 'ramp_free_quotient', 'ramp_get_quotient_bytes', 'ramp_set_job_count',
                    'ramp_set_limits', 'ramp_first_fit_place_many', 'ramp_env_create', 'ramp_env_set_template',
                    'ramp_env_reset', 'ramp_env_buffers', 'ramp_env_host_mirror', 'ramp_env_decide', 'ramp_env_patch', 'ramp_env_set_placer_tables', 'ramp_env_set_geometry_template', 'ramp_env_advance', 'ramp_env_read', 'ramp_get_last_step_stats', 'ramp_env_read_state',
                    'ramp_enable_env_step_stats', 'ramp_get_env_step_stats', 'ramp_env_steplog_begin', 'ramp_env_steplog_read',
                    'ramp_enable_tick_lists', 'ramp_get_tick_lists', 'ramp_policy_weight_count', 'ramp_policy_create', 'ramp_policy_destroy', 'ramp_policy_set_weights', 'ramp_policy_set_model',
                    'ramp_policy_embed', 'ramp_policy_forward', 'ramp_policy_decide', 'ramp_policy_act', 'ramp_policy_read',
                    'ramp_pinned_alloc', 'ramp_pinned_free', 'ramp_policy_trajectory_begin', 'ramp_policy_trajectory_record', 'ramp_policy_trajectory_read',
                    'ramp_env_read_episode', 'ramp_env_set_agents', 'ramp_env_agent_act', 'ramp_policy_get_weights',
                    'ramp_policy_backward', 'ramp_ppo_loss_grad', 'ramp_policy_learn', 'ramp_policy_train_batch_read',
                    'ramp_policy_learner_state', 'ramp_policy_learner_reset', 'ramp_impala_loss_grad', 'ramp_policy_learn_impala',
                    'ramp_impala_vtrace_read', 'ramp_es_create', 'ramp_es_destroy', 'ramp_es_round_begin', 'ramp_es_act',
                    'ramp_es_round_end', 'ramp_es_step', 'ramp_es_update', 'ramp_es_read', 'ramp_es_act_read', 'ramp_es_state',
                    'ramp_es_reset', 'ramp_pg_loss_grad', 'ramp_policy_learn_pg',
                    'ramp_env_set_graph_static', 'ramp_env_ingest', 'ramp_env_export',
                    'ramp_policy_set_weights_device', 'ramp_policy_forward_device', 'ramp_policy_backward_device',
                    'ramp_population_create', 'ramp_population_destroy', 'ramp_population_set_weights', 'ramp_population_get_weights',
                    'ramp_population_act', 'ramp_population_learn', 'ramp_population_learner_state', 'ramp_population_embed_ctas',
                    'ramp_population_learn_impala', 'ramp_population_learn_pg', 'ramp_population_vtrace_read',
                    'ramp_population_create_configs', 'ramp_population_es_create', 'ramp_population_es_destroy',
                    'ramp_population_es_round_begin', 'ramp_population_es_act', 'ramp_population_es_round_end',
                    'ramp_population_es_step', 'ramp_population_es_update', 'ramp_population_es_read', 'ramp_population_es_act_read',
                    'ramp_population_es_state', 'ramp_population_es_reset', 'ramp_population_es_embed_ctas',
                    'ramp_policy_set_learner_state', 'ramp_policy_get_act_count', 'ramp_policy_set_act_count', 'ramp_es_set_state',
                    'ramp_es_get_progress', 'ramp_es_set_progress', 'ramp_population_set_learner_state', 'ramp_population_copy_sets',
                    'ramp_population_get_act_count', 'ramp_population_set_act_count', 'ramp_population_set_es_state',
                    'ramp_population_get_es_progress', 'ramp_population_set_es_progress', 'ramp_population_copy_es_sets',
                    'ramp_env_join', 'ramp_policy_refresh_device']


def device_bytes():
    """(device bytes, page-locked host bytes) that the library's engines and policies hold right now, over the whole process.
    Unlike cudaMemGetInfo it does not move with other processes on the same GPU."""
    dev, pinned = C.c_int64(), C.c_int64()
    _check(load_library().ramp_debug_device_bytes(C.byref(dev), C.byref(pinned)))
    return dev.value, pinned.value


def _check(rc):
    if rc != RAMP_OK:
        msg = load_library().ramp_last_error().decode('utf-8', 'replace')
        # the reference raises bare `Exception` (e.g. RCE:462, RCE:1328); so do we
        raise Exception(msg)


def _ptr(a):
    return None if a is None else a.ctypes.data


class RampEngine:
    """Batched, device-resident RampClusterEnvironment state for ``n_episodes`` independent episodes."""

    def __init__(self, n_episodes, n_cluster_workers, max_jobs, max_running=0, device=0, memo_mode=MEMO_REFERENCE,
                 trace_cap=0, max_templates=0, memo_capacity_log2=0, job_queue_capacity=10, machine_epsilon=1e-7,
                 max_simulation_run_time=float('inf'), env_step_stats=False):
        """env_step_stats: keep EvalLoop's per-env-step rows (``env_step_stats()``, ramp_enable_env_step_stats); the step kernel
        skips them otherwise."""
        L = load_library()
        self._L = L
        cfg = _Config(device, n_episodes, n_cluster_workers, max_jobs, max_running, max_templates, memo_mode,
                      memo_capacity_log2, trace_cap, job_queue_capacity, machine_epsilon, max_simulation_run_time)
        h = C.c_void_p()
        _check(L.ramp_engine_create(C.byref(cfg), C.byref(h)))
        self._h = h
        self.n_episodes = n_episodes
        self.max_jobs = max_jobs
        self.trace_cap = trace_cap if trace_cap > 0 else 16384
        self.device = device
        self._templates = []
        if env_step_stats:
            L.ramp_enable_env_step_stats.restype = C.c_int
            L.ramp_enable_env_step_stats.argtypes = [C.c_void_p]
            _check(L.ramp_enable_env_step_stats(self._h))

    def close(self):
        if getattr(self, '_h', None):
            self._L.ramp_engine_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- templates -------------------------------------------------------------------------------
    def register_template(self, job: LoweredJob) -> int:
        job.canonicalise()
        cj = _LoweredJob(job.n_ops, job.n_deps, job.n_workers, job.n_channels, job.num_training_steps,
                         job.model_id, job.degree, 0,
                         job.op_cost.ctypes.data, job.op_prio.ctypes.data, job.op_worker.ctypes.data,
                         job.op_n_parents.ctypes.data, job.row_ptr.ctypes.data, job.dep_dst.ctypes.data,
                         job.dep_run_time.ctypes.data, job.dep_prio.ctypes.data, job.dep_channel.ctypes.data,
                         job.dep_is_flow.ctypes.data)
        tid = C.c_int32(-1)
        _check(self._L.ramp_register_template(self._h, C.byref(cj), C.byref(tid)))
        self._templates.append(job)
        return tid.value

    @property
    def stream(self):
        return self._L.ramp_engine_stream(self._h)

    # ---- batched reset / step ---------------------------------------------------------------------
    def reset(self, arrivals: np.ndarray):
        """arrivals: structured array [n_episodes, n_jobs] of ARRIVAL_DTYPE (RCE:202-295 for every episode)."""
        arr = np.ascontiguousarray(arrivals, dtype=ARRIVAL_DTYPE)
        assert arr.ndim == 2 and arr.shape[0] == self.n_episodes
        _check(self._L.ramp_reset(self._h, arr.ctypes.data, arr.shape[1]))
        self.n_jobs = arr.shape[1]

    def set_arrivals(self, episode, first_job, rows):
        rows = np.ascontiguousarray(rows, dtype=ARRIVAL_DTYPE).reshape(-1)
        _check(self._L.ramp_set_arrivals(self._h, episode, first_job, rows.ctypes.data, len(rows)))

    def set_job_count(self, episode, n_jobs):
        """len(jobs_generator) > 0 of one episode, as a count of jobs its arrival stream holds so far (RCE:1019-1040)."""
        _check(self._L.ramp_set_job_count(self._h, episode, n_jobs))

    def set_limits(self, max_simulation_run_time=float('inf'), job_queue_capacity=10):
        _check(self._L.ramp_set_limits(self._h, float(max_simulation_run_time), int(job_queue_capacity)))

    def make_actions(self):
        a = np.zeros(self.n_episodes, dtype=ACTION_DTYPE)
        a['template_id'] = -1
        return a

    def step(self, actions: np.ndarray, fuse_empty_steps=False, want_stats=True, want_cluster_steps=False):
        """One RampClusterEnvironment.step (RCE:894-1179) per episode through HOST buffers."""
        assert actions.dtype == ACTION_DTYPE and actions.shape == (self.n_episodes,) and actions.flags.c_contiguous
        stats = np.empty((self.n_episodes, STEP_STATS_LEN), dtype=np.float64) if want_stats else None
        ncs = np.empty(self.n_episodes, dtype=np.int32) if want_cluster_steps else None
        _check(self._L.ramp_step_host(self._h, actions.ctypes.data, 1 if fuse_empty_steps else 0, _ptr(stats), _ptr(ncs)))
        if want_cluster_steps:
            return stats, ncs
        return stats

    def step_device(self, d_actions_ptr, fuse_empty_steps=False, d_stats_ptr=None, d_ncs_ptr=None):
        """Same with raw device pointers (ints), asynchronous on the engine stream."""
        _check(self._L.ramp_step_device(self._h, d_actions_ptr, 1 if fuse_empty_steps else 0, d_stats_ptr, d_ncs_ptr))

    def sync(self):
        _check(self._L.ramp_sync(self._h))

    def enable_tick_lists(self, cap=256):
        self._L.ramp_enable_tick_lists.restype = C.c_int
        self._L.ramp_enable_tick_lists.argtypes = [C.c_void_p, C.c_int32]
        _check(self._L.ramp_enable_tick_lists(self._h, int(cap)))
        self._tick_cap = int(cap)

    def tick_lists(self, episode=0):
        """The last cluster step's per-tick lists (RCE:989-994) of one episode: (mounted utilisation, cluster utilisation)."""
        self._L.ramp_get_tick_lists.restype = C.c_int
        self._L.ramp_get_tick_lists.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]
        cap = self._tick_cap
        a, b, n = np.zeros(cap), np.zeros(cap), C.c_int32(0)
        _check(self._L.ramp_get_tick_lists(self._h, int(episode), a.ctypes.data, b.ctypes.data, cap, C.byref(n)))
        return a[:n.value], b[:n.value]

    def check_status(self):
        ep, st = C.c_int32(), C.c_int32()
        _check(self._L.ramp_check_status(self._h, C.byref(ep), C.byref(st)))

    # ---- read-back -----------------------------------------------------------------------------------
    def job_records(self):
        out = np.empty((self.n_episodes, self.max_jobs), dtype=JOB_RECORD_DTYPE)
        _check(self._L.ramp_get_job_records(self._h, out.ctypes.data))
        return out

    def episode_state(self):
        out = np.empty((self.n_episodes, EP_LEN), dtype=np.float64)
        _check(self._L.ramp_get_episode_state(self._h, out.ctypes.data))
        return out

    def episode_stats(self):
        """[n_episodes, ES_LEN] f64: RampClusterEnvironment.episode_stats' scalars (RCE:1123-1167) from every cluster step since the
        reset; rows of episodes that are not done hold the same formulas over the episode so far (include/ramp_b200.h)."""
        out = np.empty((self.n_episodes, ES_LEN), dtype=np.float64)
        _check(self._L.ramp_get_episode_stats(self._h, out.ctypes.data))
        return out

    def env_step_stats(self):
        """[n_episodes, ENV_STEP_STATS_LEN] f64: every episode's last env-step row as the step kernel closed it (EvalLoop's
        reduction over the cluster steps of the env-step, loops/eval_loop.py:50-100; include/ramp_b200.h RAMP_ESS_*)."""
        out = np.empty((self.n_episodes, ENV_STEP_STATS_LEN), dtype=np.float64)
        self._L.ramp_get_env_step_stats.restype = C.c_int
        self._L.ramp_get_env_step_stats.argtypes = [C.c_void_p, C.c_void_p]
        _check(self._L.ramp_get_env_step_stats(self._h, out.ctypes.data))
        return out

    def episode_state_device_ptr(self):
        p = C.c_void_p()
        _check(self._L.ramp_episode_state_device(self._h, C.byref(p)))
        return p.value

    def export_episode_state_to(self, d_dst_ptr):
        """Writes [n_episodes, EP_LEN] f64 into a caller-owned device buffer (async on the engine stream)."""
        _check(self._L.ramp_export_episode_state_to(self._h, d_dst_ptr))

    def memo_stats(self):
        a, b, c = C.c_int64(), C.c_int64(), C.c_int64()
        _check(self._L.ramp_get_memo_stats(self._h, C.byref(a), C.byref(b), C.byref(c)))
        return dict(lookups=a.value, hits=b.value, lookaheads=c.value)

    def memo_stats_ex(self):
        out = (C.c_int64 * 4)()
        _check(self._L.ramp_get_memo_stats_ex(self._h, out))
        return dict(lookups=out[0], hits=out[1], shared_hits=out[2], lookaheads=out[3])

    def speculative_unused(self):
        """Lookaheads executed since the last reset that no plan used: overlapped steps run the lookaheads of episodes that turn
        out not to be live when their step runs."""
        unused = C.c_int64()
        _check(self._L.ramp_get_memo_speculative_unused(self._h, C.byref(unused)))
        return unused.value

    def last_lookahead(self, episode):
        res = np.zeros(1, dtype=LOOKAHEAD_RESULT_DTYPE)
        tn = np.zeros(self.trace_cap, dtype=np.int32)
        tt = np.zeros(self.trace_cap, dtype=np.float64)
        _check(self._L.ramp_get_last_lookahead(self._h, episode, res.ctypes.data, tn.ctypes.data, tt.ctypes.data, self.trace_cap))
        T = min(int(res['n_ticks'][0]), self.trace_cap)
        return dict(jct=float(res['jct'][0]), comm=float(res['comm'][0]), comp=float(res['comp'][0]),
                    n_ticks=int(res['n_ticks'][0]), status=int(res['status'][0]),
                    trace_n_active=tn[:T].copy(), trace_tick=tt[:T].copy())

    # ---- the lookahead kernel on its own --------------------------------------------------------------
    def run_lookaheads(self, template_ids, want_trace=False, trace_cap=None):
        """RCE:379-467 for each template id.  Returns (results[LOOKAHEAD_RESULT_DTYPE], kernel_ms[, trace_n, trace_tick])."""
        tids = np.ascontiguousarray(template_ids, dtype=np.int32)
        n = len(tids)
        res = np.zeros(n, dtype=LOOKAHEAD_RESULT_DTYPE)
        ms = C.c_float(0.0)
        tn = tt = None
        cap = 0
        if want_trace:
            cap = min(trace_cap or self.trace_cap, self.trace_cap)
            tn = np.zeros((n, cap), dtype=np.int32)
            tt = np.zeros((n, cap), dtype=np.float64)
        _check(self._L.ramp_run_lookaheads(self._h, tids.ctypes.data, n, res.ctypes.data, _ptr(tn), _ptr(tt), cap, C.byref(ms)))
        if want_trace:
            return res, ms.value, tn, tt
        return res, ms.value

    def template_info(self, template_id):
        """How a registered template runs: size_class (2 = resident, on the thread-per-lookahead kernel), the resident
        quotient's n_ops / n_deps, and the TemplateHints its first completed lookahead recorded (n_ticks, max_o, max_f,
        max_nf; 0 before) with hint_jct."""
        out = (C.c_int32 * 7)()
        hj = C.c_double(0.0)
        _check(self._L.ramp_debug_template_info(self._h, int(template_id), out, C.byref(hj)))
        return dict(size_class=out[0], res_n_ops=out[1], res_n_deps=out[2], n_ticks=out[3], max_o=out[4], max_f=out[5],
                    max_nf=out[6], hint_jct=hj.value)

    @property
    def launch_count(self):
        return int(self._L.ramp_launch_count(self._h))

    def lookahead_kernel_time(self, reset=False):
        ms, nl, ni, nb, qb = C.c_double(), C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()
        self._L.ramp_get_quotient_bytes.restype = C.c_int
        self._L.ramp_get_quotient_bytes.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
        _check(self._L.ramp_get_quotient_bytes(self._h, C.byref(qb)))
        union = C.c_double()
        _check(self._L.ramp_get_lookahead_kernel_union(self._h, C.byref(union)))
        _check(self._L.ramp_get_lookahead_kernel_time(self._h, C.byref(ms), C.byref(nl), C.byref(ni), C.byref(nb),
                                                      1 if reset else 0))
        # total_ms adds up every step's lookahead interval; union_ms counts the overlapping windows of overlapped steps once
        return dict(total_ms=ms.value, union_ms=union.value, launches=nl.value, work_items=ni.value, algorithmic_bytes=nb.value,
                    quotient_bytes=qb.value)


def action_row(actions, b, template_id, mount):
    """Fills row ``b`` of an ACTION_DTYPE array from a template id and MountScalars."""
    actions[b] = (mount.max_acceptable_jct, mount.part_op_mem, mount.part_dep_size, mount.flow_size,
                  mount.n_mounted_workers, mount.n_mounted_channels, template_id, 0)
