/*
 * ramp_b200 -- C ABI of the GPU-native (H100, sm_90a) RAMP cluster simulator hot path.
 *
 * The reference (cwfparsonson/ddls @ 9e0b5ba) is pure Python and has no FFI; the interface this
 * library sits behind is the Python class surface of
 *   ddls/environments/ramp_cluster/ramp_cluster_environment.py  ("RCE")
 *     RampClusterEnvironment.__init__  RCE:75-83    -> ramp_engine_create
 *     RampClusterEnvironment.reset     RCE:202-295  -> ramp_reset
 *     RampClusterEnvironment.step      RCE:894-1179 -> ramp_step_host / ramp_step_device
 *       _place_ops/_schedule_ops/_place_deps/_schedule_deps RCE:1305-1415 -> ramp_register_template (+ per-step mount rows)
 *       _perform_lookahead_job_completion_time + memo dicts RCE:469-518, RCE:269-275 -> memo hash table inside the step
 *       _run_lookahead                  RCE:379-467  -> ramp_lookahead_thread_kernel, or
 *                                                       ramp_lookahead_cta_kernel for jobs too large for it
 *                                                       (also callable alone: ramp_run_lookaheads)
 *       _register_completed_lookahead   RCE:793-888  -> ramp_step_kernel
 *       outer event loop + stats        RCE:942-1167 -> ramp_step_kernel
 *     RampClusterEnvironment.is_done   RCE:1542-1557 -> stats[RAMP_SS_DONE]
 * batched over `n_episodes` independent cluster instances (one per RL rollout) that advance in lock step.
 * ddls_b200/engine.py is the ctypes binding; INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions: every function returns RAMP_OK (0) or a negative error code; ramp_last_error() returns a
 * message for the calling thread (the Python wrapper re-raises it as `Exception`, the type the reference
 * raises, e.g. RCE:462, RCE:1328).  All pointers are plain host or device pointers as documented; the
 * library owns only what ramp_engine_create / ramp_register_template allocate.  One host thread per engine.
 */
#ifndef RAMP_B200_H
#define RAMP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RAMP_OK 0
#define RAMP_ERR_CUDA (-1)
#define RAMP_ERR_BAD_ARG (-2)
#define RAMP_ERR_CAPACITY (-3)       /* a table / pool configured at create time is full             */
#define RAMP_ERR_SIM (-4)            /* the simulation itself raised (see per-episode status codes)   */

#define RAMP_NO_CHANNEL 0xFFFFu

/* per-lookahead / per-episode status codes written by the kernels */
#define RAMP_ST_OK 0
#define RAMP_ST_INFINITE_TICK 1      /* RCE:462 "Last tick was infinite" (deadlocked job graph)       */
#define RAMP_ST_TRACE_OVERFLOW 2     /* more ticks than ramp_config_t.trace_cap                       */
#define RAMP_ST_TABLE_FULL 3         /* running-job table full (ramp_config_t.max_running)            */
#define RAMP_ST_NO_QUEUED_JOB 4      /* an action was given for an episode with an empty job queue    */
#define RAMP_ST_JOBS_EXHAUSTED 5     /* more arrivals than ramp_config_t.max_jobs                     */
#define RAMP_ST_BAD_TEMPLATE 6       /* an action names a template id that was never registered       */

/* memo modes (RCE:269-277, RCE:488-506) */
#define RAMP_MEMO_REFERENCE 0        /* key = (episode, model, max partition degree): first seen wins, per episode */
#define RAMP_MEMO_EXACT 1            /* key = 64-bit fingerprint of the lowered job: shared across episodes        */
#define RAMP_MEMO_OFF 2              /* every mount runs its lookahead                                              */
#define RAMP_MEMO_SHARED 3           /* reference semantics (per-episode first-seen-wins on (model, degree)) on top of a batch-wide
                                        result cache keyed by the byte-identical lowered job: the lookahead an episode would run is
                                        executed once per batch and survives ramp_reset -- same results, far fewer lookaheads */

typedef struct ramp_engine ramp_engine_t;

typedef struct {
    int32_t device;              /* CUDA device ordinal                                                   */
    int32_t n_episodes;          /* B: independent cluster instances                                      */
    int32_t n_cluster_workers;   /* topology.graph.graph['num_workers'] RCE:991                           */
    int32_t max_jobs;            /* arrivals per episode the arrival stream can hold                      */
    int32_t max_running;         /* rows of the per-episode running-job table (<= n_cluster_workers suffices) */
    int32_t max_templates;       /* lowered jobs that can be registered                                    */
    int32_t memo_mode;           /* RAMP_MEMO_*                                                            */
    int32_t memo_capacity_log2;  /* hash table slots = 1 << this (0 -> sized from n_episodes)              */
    int32_t trace_cap;           /* max ticks recorded per lookahead (0 -> 16384)                          */
    int32_t job_queue_capacity;  /* RCE:205 (default 10; the queue never holds more than one job)          */
    double  machine_epsilon;     /* RCE:83 (1e-7)                                                          */
    double  max_simulation_run_time; /* RCE:204                                                            */
} ramp_config_t;

/* One lowered (partitioned + placed + scheduled) job == the complete input of _run_lookahead.
 * Op index = rank of the op id in sorted() order; dep index = rank of (u, v, k) in sorted() order
 * (== CSR-by-source position).  HOST pointers; copied to the device by ramp_register_template. */
typedef struct {
    int32_t n_ops, n_deps, n_workers, n_channels;
    int32_t num_training_steps;   /* JOB:82, RCE:450-452                                   */
    int32_t model_id;             /* dense id of job.details['model'] RCE:489              */
    int32_t degree;               /* max partition degree RCE:488                          */
    int32_t _pad;
    const double*   op_cost;      /* [N] compute_cost[device_type] RCE:1334                */
    const int64_t*  op_prio;      /* [N] worker.mounted_job_op_to_priority RCE:1397        */
    const uint16_t* op_worker;    /* [N] job-local worker id RCE:1336                      */
    const uint16_t* op_n_parents; /* [N] predecessors that are not also successors JOB:508-523 */
    const int32_t*  row_ptr;      /* [N+1] CSR out-edges                                   */
    const int32_t*  dep_dst;      /* [E]                                                   */
    const double*   dep_run_time; /* [E] init_run_time after RCE:542-560                   */
    const int64_t*  dep_prio;     /* [E] channel.mounted_job_dep_to_priority RCE:1412      */
    const uint16_t* dep_channel;  /* [E] job-local channel id or RAMP_NO_CHANNEL           */
    const uint8_t*  dep_is_flow;  /* [E] RCE:531-536                                       */
} ramp_lowered_job_t;

/* Result of one lookahead (RCE:467). */
typedef struct {
    double  jct, comm, comp;      /* x num_training_steps RCE:450-452 */
    int32_t n_ticks;
    int32_t status;               /* RAMP_ST_*                        */
} ramp_lookahead_result_t;

/* Per-arrival job description (JobsGenerator stays host-side Python; RCE:351-377 reads only these). */
typedef struct {
    double interarrival;          /* gap added to time_next_job_to_arrive when THIS job arrives RCE:363 (inf after the last) */
    double orig_op_mem;           /* original_job.details['job_total_op_memory_cost'] RCE:364, RCE:971 */
    double orig_dep_size;         /* original_job.details['job_total_dep_size']                        */
} ramp_arrival_t;

/* Per-episode, per-step action row.  template_id < 0 is Action() (RJPE:395): no job handled, a queued
 * job is blocked (RCE:914-919). */
typedef struct {
    double  max_acceptable_jct;   /* details['max_acceptable_job_completion_time'][device] RCE:815 */
    double  part_op_mem;          /* partitioned job details['job_total_op_memory_cost'] RCE:966    */
    double  part_dep_size;        /* partitioned job details['job_total_dep_size'] RCE:967          */
    double  flow_size;            /* details['job_total_flow_size'] RCE:882-888                     */
    int32_t n_mounted_workers;    /* len(details['mounted_workers'])  RCE:832                       */
    int32_t n_mounted_channels;   /* len(details['mounted_channels']) RCE:979                       */
    int32_t template_id;          /* from ramp_register_template, or -1                             */
    int32_t flags;                /* RAMP_ACT_*                                                     */
} ramp_action_t;

#define RAMP_ACT_SKIP 1           /* leave this episode untouched this call (e.g. it is done)          */

/* step statistics: double[RAMP_STEP_STATS_LEN] per episode; same names as step_stats RCE:306-338, 1046-1084 */
enum {
    RAMP_SS_STEP_COUNTER = 0, RAMP_SS_STEP_START_TIME, RAMP_SS_STEP_END_TIME, RAMP_SS_STEP_TIME,
    RAMP_SS_NUM_JOBS_COMPLETED, RAMP_SS_NUM_JOBS_ARRIVED, RAMP_SS_NUM_JOBS_BLOCKED, RAMP_SS_JOB_QUEUE_LENGTH,
    RAMP_SS_MEAN_NUM_JOBS_RUNNING, RAMP_SS_MEAN_NUM_MOUNTED_WORKERS, RAMP_SS_MEAN_NUM_MOUNTED_CHANNELS,
    RAMP_SS_MEAN_COMPUTE_OVERHEAD_FRAC, RAMP_SS_MEAN_COMMUNICATION_OVERHEAD_FRAC,
    RAMP_SS_COMPUTE_INFO_PROCESSED, RAMP_SS_DEP_INFO_PROCESSED, RAMP_SS_FLOW_INFO_PROCESSED,
    RAMP_SS_CLUSTER_INFO_PROCESSED, RAMP_SS_DEMAND_COMPUTE_INFO_PROCESSED, RAMP_SS_DEMAND_DEP_INFO_PROCESSED,
    RAMP_SS_DEMAND_TOTAL_INFO_PROCESSED,
    RAMP_SS_MEAN_COMPUTE_THROUGHPUT, RAMP_SS_MEAN_DEP_THROUGHPUT, RAMP_SS_MEAN_FLOW_THROUGHPUT,
    RAMP_SS_MEAN_CLUSTER_THROUGHPUT, RAMP_SS_MEAN_DEMAND_COMPUTE_THROUGHPUT, RAMP_SS_MEAN_DEMAND_DEP_THROUGHPUT,
    RAMP_SS_MEAN_DEMAND_TOTAL_THROUGHPUT,
    RAMP_SS_UTIL_MOUNTED_SUM,     /* sum of the step's 'mean_mounted_worker_utilisation_frac' list RCE:990 */
    RAMP_SS_UTIL_CLUSTER_SUM,     /* sum of the step's 'mean_cluster_worker_utilisation_frac' list RCE:991 */
    RAMP_SS_NUM_TICKS,            /* outer-loop iterations (= length of the two lists above)               */
    RAMP_SS_DONE,                 /* is_done() after the step RCE:1176                                     */
    RAMP_SS_LOOKAHEAD_RAN,        /* 1 if this step executed _run_lookahead (memo miss)                    */
    RAMP_STEP_STATS_LEN
};

/* env-step statistics: EvalLoop's results['step_stats'] row of one env-step (loops/eval_loop.py:50-100), double[RAMP_ENV_STEP_STATS_LEN]
 * per episode, in the order the cluster's steps_log first sees the keys (RCE:306-338, the outer loop RCE:962-982 when a job runs in
 * the episode's first cluster step, RCE:1046-1084).  Every key is reduced over the cluster steps of the env-step, the fused empty
 * steps after the action step included (RJPE:394-395): step_start_time takes the first value, step_end_time and step_counter the
 * last, keys containing 'mean' the mean, the others the sum.  The two per-tick utilisation lists are reduced by the mean over every
 * entry of the env-step. */
enum {
    RAMP_ESS_STEP_COUNTER = 0, RAMP_ESS_STEP_START_TIME, RAMP_ESS_MEAN_NUM_MOUNTED_WORKERS, RAMP_ESS_MEAN_NUM_MOUNTED_CHANNELS,
    RAMP_ESS_MEAN_COMPUTE_THROUGHPUT, RAMP_ESS_MEAN_DEP_THROUGHPUT, RAMP_ESS_MEAN_CLUSTER_THROUGHPUT,
    RAMP_ESS_MEAN_DEMAND_COMPUTE_THROUGHPUT, RAMP_ESS_MEAN_DEMAND_DEP_THROUGHPUT, RAMP_ESS_MEAN_DEMAND_TOTAL_THROUGHPUT,
    RAMP_ESS_MEAN_COMPUTE_OVERHEAD_FRAC, RAMP_ESS_MEAN_COMMUNICATION_OVERHEAD_FRAC,
    RAMP_ESS_MEAN_MOUNTED_WORKER_UTILISATION_FRAC, RAMP_ESS_MEAN_CLUSTER_WORKER_UTILISATION_FRAC,
    RAMP_ESS_NUM_JOBS_COMPLETED, RAMP_ESS_MEAN_NUM_JOBS_RUNNING, RAMP_ESS_NUM_JOBS_ARRIVED, RAMP_ESS_NUM_JOBS_BLOCKED,
    RAMP_ESS_COMPUTE_INFO_PROCESSED, RAMP_ESS_DEP_INFO_PROCESSED, RAMP_ESS_FLOW_INFO_PROCESSED, RAMP_ESS_CLUSTER_INFO_PROCESSED,
    RAMP_ESS_DEMAND_COMPUTE_INFO_PROCESSED, RAMP_ESS_DEMAND_DEP_INFO_PROCESSED, RAMP_ESS_DEMAND_TOTAL_INFO_PROCESSED,
    RAMP_ESS_STEP_END_TIME, RAMP_ESS_STEP_TIME, RAMP_ESS_MEAN_FLOW_THROUGHPUT, RAMP_ESS_JOB_QUEUE_LENGTH,
    RAMP_ENV_STEP_STATS_LEN
};

/* job record table: one row per (episode, job idx) */
enum { RAMP_JS_NOT_ARRIVED = 0, RAMP_JS_QUEUED = 1, RAMP_JS_RUNNING = 2, RAMP_JS_COMPLETED = 3, RAMP_JS_BLOCKED = 4 };
typedef struct {
    int32_t status;               /* RAMP_JS_*                                        */
    int32_t event_seq;            /* order of the completion / blocking event          */
    double  time_arrived, time_started, time_completed;
    double  jct, comm, comp, util; /* lookahead results + mean_mounted_worker_utilisation_frac RCE:830-832 */
} ramp_job_record_t;

/* ---- lifecycle ---------------------------------------------------------------------------------- */
const char* ramp_last_error(void);
int ramp_engine_create(const ramp_config_t* cfg, ramp_engine_t** out);
int ramp_engine_destroy(ramp_engine_t* eng);
/* the CUDA stream all engine work is issued on (cudaStream_t as void*) */
void* ramp_engine_stream(ramp_engine_t* eng);

/* Copies a lowered job to HBM, derives the priority-rank keys and the initial ready set, and returns its id. */
int ramp_register_template(ramp_engine_t* eng, const ramp_lowered_job_t* job, int32_t* template_id_out);
int ramp_template_count(ramp_engine_t* eng);

/* ---- batched RampClusterEnvironment.reset / step ------------------------------------------------ */
/* RCE:202-295 for every episode.  arrivals: HOST [n_episodes][n_jobs], copied before the call returns (the caller may reuse
 * the array at once); clears the memo (RCE:269-275).  Asynchronous on the engine stream: it does not wait for the device. */
int ramp_reset(ramp_engine_t* eng, const ramp_arrival_t* arrivals, int32_t n_jobs);

/* Overwrites arrival rows [first_job, first_job + n) of one episode (HOST rows).  Lets a host-driven caller (the
 * drop-in RampClusterEnvironment, whose JobsGenerator samples the next job only when needed, RCE:351-377) stream
 * the arrival process instead of fixing it at reset. */
int ramp_set_arrivals(ramp_engine_t* eng, int32_t episode, int32_t first_job, const ramp_arrival_t* rows, int32_t n);
/* How many jobs one episode's arrival stream holds so far (<= max_jobs).  The engine treats `n_jobs - arrived > 0` as the
 * reference's `len(self.jobs_generator) > 0` (RCE:1019-1040, RCE:1542-1557): a host that draws jobs lazily from a generator
 * that never runs dry ('remove_and_repeat' sampling) keeps it one ahead of the arrivals instead of fixing it at reset. */
int ramp_set_job_count(ramp_engine_t* eng, int32_t episode, int32_t n_jobs);
/* max_simulation_run_time / job_queue_capacity of the NEXT ramp_reset (RCE:202-205), so that one engine serves every
 * reset() of a drop-in environment */
int ramp_set_limits(ramp_engine_t* eng, double max_simulation_run_time, int32_t job_queue_capacity);

/* One RampClusterEnvironment.step for every episode.  HOST buffers; the host<->device copies are issued
 * on the engine stream inside the call:  actions [n_episodes] in,  stats [n_episodes][RAMP_STEP_STATS_LEN]
 * out (may be NULL).  fuse_empty_steps != 0 additionally runs, per episode, the RJPE:394-395 loop
 * `while len(job_queue) == 0 and not done: step(Action())` on the device; stats then describe the action
 * step, n_cluster_steps_out[b] (may be NULL) how many cluster steps episode b took in total. */
int ramp_step_host(ramp_engine_t* eng, const ramp_action_t* actions, int32_t fuse_empty_steps,
                   double* stats_out, int32_t* n_cluster_steps_out);
/* Same with DEVICE pointers (inputs already resident in HBM, outputs left there); asynchronous on the
 * engine stream -- call ramp_sync() before reading.
 * Action readiness: the actions may be written in stream order on the engine stream after the previous call returns.  With
 * RAMP_MEMO_REFERENCE and every template resident, the lookaheads of a call are planned from the actions as soon as the call
 * is made, while earlier steps still run, and the plan is checked against the actions in stream order: an episode whose
 * action changed since is planned again and its lookaheads run before the step (DESIGN.md section 4).  Actions written
 * ahead of the call are never planned again; engine-owned action buffers always take the in-order path. */
int ramp_step_device(ramp_engine_t* eng, const ramp_action_t* d_actions, int32_t fuse_empty_steps,
                     double* d_stats_out, int32_t* d_n_cluster_steps_out);
int ramp_sync(ramp_engine_t* eng);
/* Raises (returns RAMP_ERR_SIM) if any episode recorded a RAMP_ST_* error since the last check. */
int ramp_check_status(ramp_engine_t* eng, int32_t* first_bad_episode_out, int32_t* status_out);

/* ---- state read-back (HOST destinations) -------------------------------------------------------- */
int ramp_get_job_records(ramp_engine_t* eng, ramp_job_record_t* out /* [n_episodes][max_jobs] */);
/* per-episode scalars: double[n_episodes][RAMP_EP_LEN] */
enum { RAMP_EP_TIME = 0, RAMP_EP_NEXT_ARRIVAL, RAMP_EP_NUM_ARRIVED, RAMP_EP_NUM_COMPLETED, RAMP_EP_NUM_BLOCKED,
       RAMP_EP_QUEUED_JOB, RAMP_EP_NUM_RUNNING, RAMP_EP_STEP_COUNTER, RAMP_EP_LOAD_RATE_SUM, RAMP_EP_LOAD_RATE_N,
       RAMP_EP_DONE, RAMP_EP_STATUS, RAMP_EP_LEN };
int ramp_get_episode_state(ramp_engine_t* eng, double* out);
/* device pointer of the same table (for NCCL all-gather of episode metrics without a host bounce) */
int ramp_episode_state_device(ramp_engine_t* eng, double** d_out);
/* writes the table into a caller-owned DEVICE buffer [n_episodes][RAMP_EP_LEN] (asynchronous on the engine stream),
 * e.g. a torch tensor that is then all-gathered over NCCL */
int ramp_export_episode_state_to(ramp_engine_t* eng, double* d_dst);
/* RampClusterEnvironment.episode_stats' scalars (RCE:1086-1106 appends, RCE:1123-1167 finalises): double[n_episodes][RAMP_ES_LEN].
 * The step kernel adds every cluster step's values to per-episode accumulators (including the empty steps RJPE:394-395 fuses),
 * in cluster-step order; this applies the finalisation to them:
 *   blocking / acceptance rate      0 when no job arrived
 *   *_throughput                    *_info_processed / episode_time unless either is 0 (then 0)
 *   the four step means             sum of the per-cluster-step means / number of cluster steps; 0 when episode_time == 0
 *   the two utilisation means       the mean over every per-tick entry of the episode (sum of the per-step list sums / the
 *                                   number of ticks), 0 when episode_time == 0.  The reference's np.mean over its list of
 *                                   per-step lists is not defined when the lists are ragged; this is the definition of the
 *                                   drop-in class (ddls_b200/host/cluster.py), which flattens them.
 * Rows of episodes that are not done (RAMP_ES_DONE = 0) hold the same formulas over the episode so far.  Waits for the engine
 * stream. */
enum { RAMP_ES_EPISODE_START_TIME = 0, RAMP_ES_EPISODE_END_TIME, RAMP_ES_EPISODE_TIME,
       RAMP_ES_NUM_JOBS_ARRIVED, RAMP_ES_NUM_JOBS_COMPLETED, RAMP_ES_NUM_JOBS_BLOCKED,
       RAMP_ES_MEAN_LOAD_RATE, RAMP_ES_BLOCKING_RATE, RAMP_ES_ACCEPTANCE_RATE,
       RAMP_ES_COMPUTE_INFO_PROCESSED, RAMP_ES_DEP_INFO_PROCESSED, RAMP_ES_FLOW_INFO_PROCESSED, RAMP_ES_CLUSTER_INFO_PROCESSED,
       RAMP_ES_DEMAND_COMPUTE_INFO_PROCESSED, RAMP_ES_DEMAND_DEP_INFO_PROCESSED, RAMP_ES_DEMAND_TOTAL_INFO_PROCESSED,
       RAMP_ES_MEAN_COMPUTE_THROUGHPUT, RAMP_ES_MEAN_DEP_THROUGHPUT, RAMP_ES_MEAN_FLOW_THROUGHPUT, RAMP_ES_MEAN_CLUSTER_THROUGHPUT,
       RAMP_ES_MEAN_DEMAND_COMPUTE_THROUGHPUT, RAMP_ES_MEAN_DEMAND_DEP_THROUGHPUT, RAMP_ES_MEAN_DEMAND_TOTAL_THROUGHPUT,
       RAMP_ES_MEAN_COMPUTE_OVERHEAD_FRAC, RAMP_ES_MEAN_COMMUNICATION_OVERHEAD_FRAC, RAMP_ES_MEAN_NUM_JOBS_RUNNING,
       RAMP_ES_MEAN_NUM_MOUNTED_WORKERS, RAMP_ES_MEAN_MOUNTED_WORKER_UTILISATION_FRAC, RAMP_ES_MEAN_CLUSTER_WORKER_UTILISATION_FRAC,
       RAMP_ES_NUM_CLUSTER_STEPS, RAMP_ES_NUM_TICKS, RAMP_ES_DONE, RAMP_ES_LEN };
int ramp_get_episode_stats(ramp_engine_t* eng, double* out /* HOST [n_episodes][RAMP_ES_LEN] */);
/* memo statistics since the last reset: lookups, hits, lookaheads executed */
int ramp_get_memo_stats(ramp_engine_t* eng, int64_t* lookups, int64_t* hits, int64_t* lookaheads);
/* {lookups, per-episode hits, batch-wide (shared) hits, lookaheads executed} since the last reset */
int ramp_get_memo_stats_ex(ramp_engine_t* eng, int64_t out[4]);
/* lookaheads executed since the last reset whose plan did not use them: overlapped steps plan every episode with a valid,
 * non-skip action, and the ones that are not live when their step runs leave their lookahead unused */
int ramp_get_memo_speculative_unused(ramp_engine_t* eng, int64_t* unused);
/* the lookahead (memoised or fresh) used by episode `episode`'s most recent mount: result + trace
 * (tick_counter_to_active_workers_tick_size RCE:467); trace buffers are HOST, capacity trace_cap. */
int ramp_get_last_lookahead(ramp_engine_t* eng, int32_t episode, ramp_lookahead_result_t* res,
                            int32_t* trace_n_active, double* trace_tick, int32_t trace_cap);

/* ---- the lookahead kernels on their own --------------------------------------------------------- */
/* Runs _run_lookahead (RCE:379-467) for n work items; item k uses template template_ids[k] (HOST array).
 * The items go to the lookahead kernels by the rule a step uses for its memo misses.
 * results: HOST [n].  trace_n_active / trace_tick: HOST [n][trace_cap] or NULL.  kernel_ms_out (may be
 * NULL) receives the CUDA-event duration of the lookahead kernels, without the uploads and the grouping of
 * the resident items by template. */
int ramp_run_lookaheads(ramp_engine_t* eng, const int32_t* template_ids, int32_t n,
                        ramp_lookahead_result_t* results, int32_t* trace_n_active, double* trace_tick,
                        int32_t trace_cap, float* kernel_ms_out);
/* How a registered template runs, for tests and diagnostics: out[0] size class (2 = resident: the thread-per-lookahead
 * kernel on its quotient, 0 = the CTA kernel), out[1..2] the resident quotient's classes and dep entries
 * (0 when not resident), out[3..6] what the first completed lookahead of the template recorded for the later ones
 * (ticks, largest ready-op / ready-flow / ready-non-flow frontiers; all 0 before), *hint_jct (may be NULL) its job
 * completion time.  Waits for the engine stream. */
int ramp_debug_template_info(ramp_engine_t* eng, int32_t template_id, int32_t out[7], double* hint_jct);

/* kernel launch counter (gpu_launches in bench.py) and device time spent in the lookahead kernel inside
 * ramp_step_* since the last call (CUDA events on the engine stream) */
int64_t ramp_launch_count(ramp_engine_t* eng);
/* Bytes of device memory and of page-locked host memory the library's engines and policies hold right now, over the whole
 * process (either pointer may be NULL).  Memory ramp_pinned_alloc hands to the caller is not counted. */
int ramp_debug_device_bytes(int64_t* device_bytes, int64_t* pinned_bytes);
int ramp_get_lookahead_kernel_time(ramp_engine_t* eng, double* total_ms, int64_t* launches, int64_t* work_items,
                                   int64_t* algorithmic_bytes, int32_t reset);
/* the same 20 N + 19 E + 12 T + 24 accounting on the sizes of the symmetry quotients the thread-per-lookahead kernel really
 * simulated (since the last reset of the counters above; read it BEFORE resetting them) */
int ramp_get_quotient_bytes(ramp_engine_t* eng, int64_t* quotient_bytes);
/* total_ms above adds every step's lookahead interval; the lookaheads of overlapped steps run at the same time, so this is
 * the union of the same intervals (ms, reset with them) */
int ramp_get_lookahead_kernel_union(ramp_engine_t* eng, double* union_ms);

/* ---- native template expansion (SURVEY.md 8f-1): what OpPartition / update_dep_run_times / the SRPT schedulers /
 * FirstFitDepPlacer compute for ONE job placed on a block of servers (sub-op k of every split op on server k), without
 * the reference's Python objects.  Replaces RJPE:320-360 + agents/partitioners/utils.py:42-110 + actions/utils.py:13-393 +
 * srpt_*_scheduler.py for that case; the Python twin is ddls_b200/template_builder.py.  Host-only: needs no GPU. ---- */
typedef struct {
    int32_t n_fwd;                /* forward ops 1..n of the un-mirrored job graph (ddls/utils.py:278-340)          */
    int32_t n_edges;
    const double*  fwd_cost;      /* [n] forward_compute_time                                                       */
    const double*  bwd_cost;      /* [n] backward_compute_time                                                      */
    const double*  act_size;      /* [n] activation_size                                                            */
    const double*  par_size;      /* [n] parameter_size                                                             */
    const int32_t* edge_src;      /* [n_edges] 1-based forward op ids                                               */
    const int32_t* edge_dst;
} ramp_forward_graph_t;

typedef struct {
    int32_t n_servers;            /* servers of the block, in sorted server-id order                                */
    int32_t num_communication_groups;  /* of the whole topology (x in actions/utils.py:40)                          */
    const int32_t* coords;        /* [n_servers][3] (communication group, rack, server)                             */
    double channel_bandwidth, latency, io_latency;   /* topologies/ramp.py:27, heuristic_config.yaml:73-82          */
} ramp_block_t;

enum { RAMP_RUN_TIMES_ONE_TO_ONE = 0, RAMP_RUN_TIMES_REFERENCE = 1 };

/* What the mount scalars (ramp_action_t) are summed from: edge sizes, op memory costs, and the op indices in the job
 * graph's node order (the order the reference's Python sums run in, JOB:224-248). */
typedef struct {
    double*  dep_size;            /* [n_deps] */
    double*  op_mem;              /* [n_ops]  */
    int32_t* node_order;          /* [n_ops]  */
} ramp_expanded_aux_t;

/* Fills `out` (and `aux` if not NULL) with malloc'ed arrays; release with ramp_free_expanded_job / ramp_free_expanded_aux. */
int ramp_expand_template(const ramp_forward_graph_t* graph, int32_t degree, double min_op_run_time_quantum,
                         const ramp_block_t* block, int32_t run_time_mode, int32_t num_training_steps,
                         ramp_lowered_job_t* out, ramp_expanded_aux_t* aux);
void ramp_free_expanded_aux(ramp_expanded_aux_t* aux);

/* RampFirstFitOpPlacer.get (agents/placers/ramp_first_fit_op_placer.py:27-113, agents/placers/utils.py:68-582) for one job:
 * which server every (sub-)op goes to on a possibly busy cluster.  Server index = (cg * racks + rack) * servers + server. */
typedef struct {
    int32_t shape[3];             /* communication groups, racks per group, servers per rack (ramp.py:36-41)        */
    int32_t _pad;
    const double*  free_mem;      /* [servers] memory_capacity - memory_occupied of the server's worker (utils.py:235) */
    const uint8_t* busy;          /* [servers] a job is mounted there (one job per worker, ramp_rules.py:6-39)       */
} ramp_cluster_state_t;

/* splits[n_fwd]: sub-ops per forward op (1 = unsplit).  server_out: servers of op 1's sub-ops 0.., then op 2's ... (the
 * backward op shares them); offset_out[n_fwd + 1]: where each op's servers start.  Returns RAMP_OK, 1 if the job cannot be
 * placed (the reference then leaves it out of the Action and RCE:914-919 blocks it), or a negative RAMP_ERR_*. */
int ramp_first_fit_place(const ramp_forward_graph_t* graph, const int32_t* splits, const ramp_cluster_state_t* state,
                         int32_t* server_out, int32_t* offset_out);
void ramp_free_expanded_job(ramp_lowered_job_t* job);
/* ramp_first_fit_place for many cluster states in one call: busy_words[k] / server_mask_out[k] are bit sets over the servers
 * (n_words x 64 bits each); ok_out[k] = 0 when the job cannot be placed on state k.  Free servers have memory_capacity bytes free
 * (one job per worker, ramp_rules.py:6-39). */
int ramp_first_fit_place_many(const ramp_forward_graph_t* graph, const int32_t* splits, const int32_t shape[3], double memory_capacity,
                              int32_t n_states, int32_t n_words, const uint64_t* busy_words, uint64_t* server_mask_out, uint8_t* ok_out);

/* ---- symmetry quotient of a lowered job (host-only; ddls_b200/csrc/ramp_quotient.cpp).  ramp_register_template applies it
 * by itself; it is exported so that tests can check it without a GPU.  The quotient job is what _run_lookahead
 * (RCE:379-467) is simulated on: one op per class of ops that provably tick in lock step (e.g. the n sub-ops of a
 * partitioned op, agents/partitioners/utils.py:42-110), one dep entry per (class of deps, group of identical channels).
 *   op_weight     class size: what a winning class adds to the trace's active-worker count (RCE:709-715)
 *   op_threshold  n_parents x class size: the class is readied when its counter passes through it (JOB:525-536)
 *   dep_inc       members of the entry: what its completion adds to the child class's counter
 *   op_class[N], dep_entry[E]: where every original op / dep went.  Keys are unique ranks (larger wins). ---- */
typedef struct {
    int32_t n_ops, n_deps, n_workers, n_channels;     /* classes, entries, worker groups, channel groups */
    double*   op_cost;
    uint32_t* op_key;
    uint32_t* op_worker;
    uint32_t* op_weight;
    uint32_t* op_threshold;
    int32_t*  row_ptr;
    int32_t*  dep_dst;
    double*   dep_run_time;
    uint32_t* dep_key;
    uint32_t* dep_channel;       /* split entries: the channel group; 0xFFFFFFFF = none, or merged (see dep_group_mask) */
    uint64_t* dep_group_mask;    /* bit g set: members of the entry lie on channels of group g (valid when masks_valid)   */
    uint8_t*  dep_is_flow;
    uint32_t* dep_inc;
    int32_t*  op_class;
    int32_t*  dep_entry;
    int32_t   merged;            /* 1: one entry per dep class with a group set; 0: one entry per (dep class, group)        */
    int32_t   masks_valid;       /* 0 when there are more than 64 channel groups                                            */
} ramp_quotient_t;
int ramp_quotient_template(const ramp_lowered_job_t* job, ramp_quotient_t* out);
void ramp_free_quotient(ramp_quotient_t* q);


/* ---- device-resident rollouts (SURVEY.md 8f-2 / 8f-4 on the device, 8g): one RampJobPartitioningEnvironment.step for every
 * episode without the host in the loop.  Per episode the action is the maximum partition degree of the queued job
 * (RJPE:300-343).  ramp_env_decide places the job with the reference's first-fit rule (agents/placers/utils.py:394-443, 532-582:
 * the first free block in the (block shape, origin) order the host enumerated into `cand_*`), looks the lowered job up by
 * (model, degree, block geometry) and writes the engine's action rows; ramp_env_advance runs the batched cluster step with the
 * RJPE:394-395 loop fused and then, per episode, the reward (rewards/job_acceptance.py), the occupancy of the cluster, and the
 * dynamic observation features + action mask of the next queued job (observations/...observation.py:80-131, 358-498).
 * Episodes the tables cannot decide (ops of one job split different numbers of times, a block geometry whose template is not
 * registered yet) are listed for the host, which patches their rows before ramp_env_advance. ---- */
typedef struct {
    int32_t shape[3];             /* communication groups, racks per group, servers per rack                       */
    int32_t n_models, max_degree, n_geoms, jobs_per_episode, n_words;   /* n_words = ceil(servers / 64)             */
    int32_t apply_action_mask;    /* 1: an invalid action is an error (RJPE:317-319); 0: it becomes action 0       */
    int32_t num_training_steps;
    double  fail_reward, success_reward;
    double  machine_epsilon;      /* added to a normalised observation feature that is negative (observation.py:441-444, 493-496) */
    const int32_t*  cand_ptr;    /* [max_degree + 2] candidates of degree d are [cand_ptr[d], cand_ptr[d + 1])    */
    const uint64_t* cand_mask;    /* [n_cand][n_words] servers of the block (bit set)                              */
    const int32_t*  cand_geom;    /* [n_cand] geometry index of the block (what the lowered job depends on)        */
    const uint8_t*  uniform;      /* [n_models][max_degree + 1] 1: every op of the model takes `degree` sub-ops and the job fits
                                     the block's memory, so placing it is one first-fit search                    */
    const uint8_t*  shape_ok;     /* [max_degree + 1] a RAMP-symmetric block shape exists (action mask)            */
    const double*   model_params; /* [n_models][5] sequential completion time, #ops, #deps, op memory, dep size    */
    const double*   jobs_params;  /* [8][2] (min, max) of JobsGenerator.jobs_params in observation.PARAM_KEYS order */
} ramp_env_config_t;

/* device buffers of the environment (valid until the engine is destroyed): what a device-resident policy reads and writes */
typedef struct {
    int32_t*  actions;            /* [B] in: max partition degree chosen for the queued job (0 = do not place)      */
    double*   reward;             /* [B] out                                                                        */
    uint8_t*  done;               /* [B] out                                                                        */
    int32_t*  queued_model;       /* [B] out: model of the queued job (-1 none)                                     */
    float*    obs_dynamic;        /* [B][11] out: graph features that change per job / cluster state                */
    uint8_t*  action_mask;        /* [B][max_degree + 1] out                                                        */
    uint64_t* busy;               /* [B][n_words] occupancy of the cluster                                          */
    int32_t*  template_id;        /* [B] template the decision mounted (-1 none)                                    */
    int32_t   n_episodes, n_actions, n_models;   /* B, max_degree + 1, job types                                    */
} ramp_env_buffers_t;

/* page-locked HOST arrays of the same shapes (valid until the engine is destroyed): give them to ramp_env_decide / ramp_env_read
 * so that the per-step copies are true asynchronous DMA transfers (busy / template_id are not mirrored: NULL) */
int ramp_env_host_mirror(ramp_engine_t* eng, ramp_env_buffers_t* out);

int ramp_env_create(ramp_engine_t* eng, const ramp_env_config_t* cfg);
int ramp_env_set_template(ramp_engine_t* eng, int32_t model, int32_t degree, int32_t geom, int32_t template_id, const double mount[6]);
/* model_of / frac / max_acceptable_jct (NaN = frac x sequential time): HOST [n_episodes][jobs_per_episode]; arrivals as ramp_reset */
int ramp_env_reset(ramp_engine_t* eng, const int32_t* model_of, const double* frac, const double* max_acceptable_jct,
                   const ramp_arrival_t* arrivals);
int ramp_env_buffers(ramp_engine_t* eng, ramp_env_buffers_t* out);
/* actions: HOST [n_episodes] (copied) or NULL (already in ramp_env_buffers_t.actions).  need_host_out: HOST [n_episodes] list of
 * episodes the tables could not decide, n_need_host_out their number (pass NULL for both when `uniform` covers every model). */
int ramp_env_decide(ramp_engine_t* eng, const int32_t* actions, int32_t* n_need_host_out, int32_t* need_host_out);
int ramp_env_patch(ramp_engine_t* eng, int32_t episode, int32_t template_id, const uint64_t* server_mask, const double mount[6]);
int ramp_env_advance(ramp_engine_t* eng);

/* Device placement of jobs whose ops split unevenly.  Once ramp_env_set_placer_tables ran, ramp_env_decide places every episode
 * the tables above list for the host on the device instead (ramp_env_place_kernel, one warp per episode): the reference's
 * first-fit op placer, op by op in topological order (parent collective placement first, then the first free candidate block
 * with the memory), then the lowered job by (model, degree, canonical mask of the servers used) from a table filled by
 * ramp_env_set_geometry_template.  need_host_out then lists only the episodes whose canonical mask is not in that table yet, and
 * uniform jobs whose block geometry has no template.  The canonical mask relabels each coordinate axis of the used servers to
 * 0, 1, ... in order and sets bit (c * R + r) * S + s of each relabelled server.  Per warp the kernel keeps the free memory of
 * every server and one candidate index per op in shared memory: 8 * (servers + 8) + 4 * (ops of the largest model) bytes, which
 * must not exceed RAMP_ENV_PLACE_SMEM_PER_WARP. */
#define RAMP_ENV_PLACE_SMEM_PER_WARP 12288
typedef struct {
    int32_t n_ops_total;          /* ops of every model together                                                   */
    double  memory_capacity;      /* free bytes of every server when the job is placed                             */
    const int32_t* op_ptr;        /* [n_models + 1] the ops of model m are op_ptr[m] .. op_ptr[m + 1] - 1          */
    const int32_t* topo;          /* [n_ops_total] per model: op indices (within the model, from 0) in topo_sort order */
    const int32_t* par_ptr;       /* [n_ops_total + 1] parents of op g are parents[par_ptr[g] .. par_ptr[g + 1])   */
    const int32_t* parents;       /* op indices within the model, in the graph's edge order                        */
    const double*  need;          /* [n_ops_total] activation + parameter bytes of each op                         */
    const int32_t* splits;        /* [max_degree + 1][n_ops_total] sub-ops of each op at each degree (>= 1)        */
    const int32_t* cand_offset;   /* [n_cand + 1] servers of candidate c are cand_servers[cand_offset[c] ..)       */
    const int32_t* cand_servers;  /* the servers of each candidate block in the placer's block order               */
} ramp_env_placer_tables_t;
int ramp_env_set_placer_tables(ramp_engine_t* eng, const ramp_env_placer_tables_t* tables);
/* (model, degree, canonical_mask [n_words]) -> template_id; mount as ramp_env_set_template.  Replaces an existing entry. */
int ramp_env_set_geometry_template(ramp_engine_t* eng, int32_t model, int32_t degree, const uint64_t* canonical_mask,
                                   int32_t template_id, const double mount[6]);
/* HOST copies of the outputs (any may be NULL) */
/* The reference leaves step_stats['mean_mounted_worker_utilisation_frac'] / ['mean_cluster_worker_utilisation_frac'] as LISTS with
 * one entry per outer-loop iteration of the step (RCE:989-994); RAMP_SS_UTIL_*_SUM / RAMP_SS_NUM_TICKS carry their sum and length.
 * ramp_enable_tick_lists makes the step kernel also keep the entries of the last cluster step (up to `cap` per episode);
 * ramp_get_tick_lists copies one episode's to HOST arrays [cap] and returns the length in n_out (RAMP_ERR_CAPACITY when the
 * step had more iterations than `cap` given to ramp_enable_tick_lists). */
int ramp_enable_tick_lists(ramp_engine_t* eng, int32_t cap);
int ramp_get_tick_lists(ramp_engine_t* eng, int32_t episode, double* mounted_out, double* cluster_out, int32_t cap, int32_t* n_out);
/* step statistics / cluster-step counts of the last ramp_env_advance (the engine's own buffers): HOST [n_episodes][RAMP_STEP_STATS_LEN], [n_episodes] */
int ramp_get_last_step_stats(ramp_engine_t* eng, double* stats_out, int32_t* n_cluster_steps_out);
/* ramp_enable_env_step_stats makes the step kernel keep EvalLoop's per-env-step rows (both batched environments enable it; the
 * engine alone does not pay for them).  The env-step row (RAMP_ESS_*) of every episode's last env-step -- the last step call with fuse_empty_steps, ramp_env_advance or
 * ramp_step_host -- as the step kernel closed it: HOST [n_episodes][RAMP_ENV_STEP_STATS_LEN] (EvalLoop's reduction of one env-step,
 * loops/eval_loop.py:50-100).  A finished episode keeps its last row. */
int ramp_enable_env_step_stats(ramp_engine_t* eng);
int ramp_get_env_step_stats(ramp_engine_t* eng, double* out);
/* EvalLoop's results['step_stats'] for every episode, kept on the device (loops/eval_loop.py:44-100).  ramp_env_steplog_begin
 * allocates room for `horizon` env-steps per episode ([horizon][RAMP_ENV_STEP_STATS_LEN][n_episodes] f64, actions and rewards
 * [horizon][n_episodes]) and clears it; horizon 0 frees it.  From then on every ramp_env_advance writes, for every episode that was
 * not done, env-step n_decided - 1's row, its action (as the agent chose it, before apply_action_mask=False turns an invalid one
 * into 0, eval_loop.py:44-47) and its reward, on the engine stream without synchronising.  ramp_env_steplog_read copies the
 * record back once: HOST stats [horizon][RAMP_ENV_STEP_STATS_LEN][n_episodes], actions / rewards [horizon][n_episodes], and
 * n_steps [n_episodes], the env-steps each episode took (rows beyond `horizon` are not kept; any pointer may be NULL). */
int ramp_env_steplog_begin(ramp_engine_t* eng, int32_t horizon);
int ramp_env_steplog_read(ramp_engine_t* eng, int32_t horizon, double* stats_out, int32_t* actions_out, double* rewards_out,
                          int32_t* n_steps_out);
/* HOST copies of the occupancy [n_episodes][n_words], of the actions the device holds, and of the number of decisions every episode
 * has taken since ramp_env_reset (= its env-steps; a finished episode takes none) -- any may be NULL */
int ramp_env_read_state(ramp_engine_t* eng, uint64_t* busy_out, int32_t* actions_out, int32_t* n_decided_out);
/* What the per-job lists of episode_stats need beyond the job records, as HOST copies (either may be NULL): the template every
 * accepted job was mounted with ([n_episodes][jobs_per_episode], -1 for the others) and every episode's return, the sum of its
 * rewards since ramp_env_reset (EvalLoop's episode_stats['return'], loops/eval_loop.py:26-134). */
int ramp_env_read_episode(ramp_engine_t* eng, int32_t* job_template_out, double* return_out);

/* The reference's heuristic agents (ddls/environments/ramp_job_partitioning/agents/*.py) on the device.  ramp_env_set_agents
 * uploads one agent per episode (kind: HOST [n_episodes] RAMP_AGENT_*; param: HOST [n_episodes], SiPML's max_partitions_per_op,
 * <= 0 = None, ignored by the others, may be NULL), so that one batch can run different agents side by side.
 * ramp_env_agent_act writes ramp_env_buffers_t.actions from the current action mask, queued model, max acceptable JCT and
 * model_params, one thread per episode on the engine stream, with no host transfer; finished episodes get 0.  Random draws
 * from splitmix64 keyed by (seed, episode, decisions the episode has taken), not numpy's stream.  See ramp_env.cuh for each
 * agent's rule. */
enum { RAMP_AGENT_RANDOM = 0, RAMP_AGENT_SIPML, RAMP_AGENT_ACCEPTABLE_JCT, RAMP_AGENT_MAX_PARALLELISM, RAMP_AGENT_MIN_PARALLELISM,
       RAMP_AGENT_NO_PARALLELISM, RAMP_AGENT_COUNT };
int ramp_env_set_agents(ramp_engine_t* eng, const int32_t* kind, const int32_t* param);
int ramp_env_agent_act(ramp_engine_t* eng, uint64_t seed);
/* also raises what ramp_check_status would (RAMP_ERR_SIM) -- one synchronisation per step for a host-side policy.  After a
 * ramp_env_ingest it also raises the first action outside the action set (see below). */
int ramp_env_read(ramp_engine_t* eng, double* reward, uint8_t* done, int32_t* queued_model, float* obs_dynamic, uint8_t* action_mask);

/* ---- the environment's i/o in caller-owned DEVICE memory (e.g. PyTorch CUDA tensors), ordered on the caller's stream.
 * ramp_env_ingest runs one thread per episode on `stream`: it reads actions [n_episodes] (dtype RAMP_ACTIONS_INT32 / _INT64) and
 * writes ramp_env_buffers_t.actions, for ramp_env_decide(eng, NULL, ...) to use.  An action of a live episode outside the action set
 * [0, max_degree] is written as 0 and the first one is kept in a sticky word: the next ramp_env_read, or ramp_env_decide with
 * need_host_out, raises it as RJPE:314-316 does ("Action a not in action set [...]"), whatever apply_action_mask says.
 * ramp_env_export writes, on `stream`, RampJobPartitioningObservation's row for every episode (ramp_job_partitioning_observation.py:
 * 275) and the step's reward and done; any pointer of `out` may be NULL.  Values of finished episodes are what ramp_env_read gives.
 * Both calls fence the engine stream with events: the caller's stream first waits for the engine's queued work (the last
 * ramp_env_advance), and the engine stream then waits for the kernel, so neither stream reads a buffer the other still writes and
 * the caller's allocator may reuse its memory in its own stream order.  ramp_env_set_graph_static uploads the six per-graph
 * statistics of every model (HOST [n_models][6] float32, observation.py:425-469), which graph_features needs. */
#define RAMP_ACTIONS_INT32 0
#define RAMP_ACTIONS_INT64 1
typedef struct {
    int64_t* model;               /* [B] model of the queued job (-1 none)                                           */
    float*   graph_features;      /* [B][17 + n_actions]: obs_dynamic[0:9], graph_static[model][0:6], obs_dynamic[9:11],
                                     then the action mask as 0.0 / 1.0                                                */
    uint8_t* action_mask;         /* [B][n_actions] 0 / 1                                                            */
    double*  reward;              /* [B]                                                                             */
    uint8_t* done;                /* [B] 0 / 1                                                                       */
} ramp_env_export_t;
int ramp_env_set_graph_static(ramp_engine_t* eng, const float* graph_static);
int ramp_env_ingest(ramp_engine_t* eng, const void* actions, int32_t dtype, void* stream);
int ramp_env_export(ramp_engine_t* eng, void* stream, const ramp_env_export_t* out);

/* ---- CUDA-graph capture of a step (DESIGN.md §7 g).  ramp_env_ingest, ramp_env_decide(eng, NULL, NULL, NULL), ramp_env_advance
 * and ramp_env_export may be captured into a CUDA graph on `stream` (e.g. inside torch.cuda.graph): each call asks
 * cudaStreamIsCapturing of the stream it runs on, and there is no flag to set.  Under capture a step records no timing event, never
 * synchronises, allocates nothing and reads nothing back; the ingest's fence forks the engine stream into the capture and the
 * export's joins it back, and the export leaves no fork open.  ramp_env_ingest refuses to start a captured step (RAMP_ERR_BAD_ARG,
 * nothing enqueued) when a replay would need the host: a template on the CTA kernel (its launch shape needs a work count on the
 * host), no eager step yet (the i/o buffers and lookahead scratch are sized by eager steps), or a template registered since the
 * last eager step (the scratch may have to grow).  ramp_env_decide refuses host actions and need_host_out under capture.  The
 * caller refuses a capture when the device tables do not decide every placement.  Replays advance the ingest call number on
 * the device, so their errors are those of eager steps: the next ramp_env_read raises them.  Once a step was captured, the
 * env-step record (ramp_env_steplog_begin) keeps its buffers: it can be cleared at its horizon, not replaced; and
 * ramp_register_template and ramp_enable_tick_lists are refused, as the graph keeps the template count, the lookahead scratch
 * and the lists' addresses.  Host-set values a
 * captured launch carries (ramp_set_limits, the record's horizon) are those of the capture.
 * ramp_env_join makes the engine stream wait for the work queued on `stream` so far, without a synchronisation: after a replay
 * on `stream`, call it before engine-stream calls (ramp_env_read, ramp_env_reset, the statistics) so they see the replay.
 * Refused while `stream` captures. */
int ramp_env_join(ramp_engine_t* eng, void* stream);


/* ---- the GNN policy forward on the device (SURVEY.md 8f-3): GNNPolicy.forward (ml_models/policies/gnn_policy.py:137-296) =
 * num_rounds MeanPool message-passing rounds over the queued job's graph (ml_models/models/mean_pool.py:107-150, gnn.py:84-92),
 * the mean of the node embeddings, a graph module over [graph features | action mask] (gnn_policy.py:96-109), and an RLlib
 * FullyConnectedNetwork read-out (fcnet_hiddens; a separate value branch, or the value layer on the policy's hidden layer under
 * vf_share_layers) with the log-mask added to the logits
 * (gnn_policy.py:283-290).  What the policy sees of a job's ops and deps is fixed per job TYPE (node / edge features:
 * observation.py:503-567), so the message passing is run once per model and weight set (ramp_policy_embed: one CTA per model);
 * per decision only the graph module + read-out run (one warp per episode, weights staged in shared memory), reading the
 * environment's device buffers and writing its `actions` -- a rollout step never leaves the device.  fp32 throughout.
 * DGL semantics restated: a node without incoming edges keeps a zero embedding after a round (dgl update_all fills
 * zero-in-degree nodes with zeros); every other node averages reduce_module over [its own (node | zeros) state, messages]. ---- */
typedef struct {
    int32_t in_features_node, in_features_edge, in_features_graph;   /* 5, 2, 17 (gnn.yaml)                          */
    int32_t n_actions;                                               /* action_space.n = max_partitions_per_op + 1    */
    int32_t out_features_msg, out_features_hidden, out_features_node, out_features_graph;   /* 32, 64, 16, 8          */
    int32_t num_rounds;                                              /* >= 2 (gnn.py:40-41)                           */
    int32_t fcnet_hidden;                                            /* one hidden layer of the read-out (256): a     */
                                                                     /* multiple of 32 in [32, 512], or n_actions     */
    int32_t aggregator_activation;                                   /* 0 relu, 1 leaky_relu(0.01)                    */
    int32_t fcnet_activation;                                        /* 0 relu, 2 tanh                                */
    int32_t apply_action_mask;
    int32_t n_models;
    int32_t vf_share_layers;                                         /* 0: separate value branch; 1: RLlib's          */
                                                                     /* vf_share_layers, the value layer [1][H] reads */
                                                                     /* the policy's hidden layer                     */
} ramp_policy_config_t;
typedef struct ramp_policy ramp_policy_t;
/* number of fp32 words of the weight blob for `cfg`, in torch state_dict order of GNNPolicy: per round [node LN w,b | node
 * Linear W,b | edge LN w,b | edge Linear W,b | reduce LN w,b | reduce Linear W,b]; graph LN w,b | graph Linear W,b; read-out hidden
 * W,b | logits W,b | value hidden W,b (not under vf_share_layers) | value W,b.  Every W is [out][in] row-major as torch.nn.Linear
 * keeps it. */
int64_t ramp_policy_weight_count(const ramp_policy_config_t* cfg);
int ramp_policy_create(int device, const ramp_policy_config_t* cfg, ramp_policy_t** out);
void ramp_policy_destroy(ramp_policy_t* p);
/* weights: HOST [ramp_policy_weight_count]; the per-model embeddings become stale until the next ramp_policy_embed */
int ramp_policy_set_weights(ramp_policy_t* p, const float* weights, int64_t n);
/* one job type: HOST node features [n_nodes][in_node], edge features [n_edges][in_edge], edge endpoints (node indices), and the
 * per-graph statistics that sit between the dynamic graph features ([6]: observation.py:425-469) */
int ramp_policy_set_model(ramp_policy_t* p, int32_t model, int32_t n_nodes, int32_t n_edges, const float* node_features,
                          const float* edge_features, const int32_t* edges_src, const int32_t* edges_dst, const float* graph_static);
/* message passing + node mean of every registered model; embeddings_out: HOST [n_models][out_features_node] or NULL */
int ramp_policy_embed(ramp_policy_t* p, float* embeddings_out);
/* read-out on HOST inputs (tests, host-side policies): model [n], graph_features [n][in_features_graph], action_mask
 * [n][n_actions] -> logits [n][n_actions], value [n] (either may be NULL).  Uses buffers of its own: what the last
 * ramp_policy_act left for ramp_policy_read / ramp_policy_trajectory_record is not touched. */
int ramp_policy_forward(ramp_policy_t* p, int32_t n, const int32_t* model, const float* graph_features, const uint8_t* action_mask,
                        float* logits_out, float* value_out);
/* ramp_policy_forward plus the action selection of ramp_policy_act on HOST inputs: log-probability of the chosen action [n] and the
 * action [n] (any output may be NULL).  Row b draws with the key (seed, b); `seed` is used as given (act mixes in its call count).
 * Rows whose model is outside [0, n_models) get zero logits, value and log-probability and action 0. */
int ramp_policy_decide(ramp_policy_t* p, int32_t n, const int32_t* model, const float* graph_features, const uint8_t* action_mask,
                       int32_t sample, uint64_t seed, float* logits_out, float* value_out, float* logp_out, int32_t* actions_out);
/* one decision for every episode of `eng`'s environment on the engine's stream: reads queued_model / obs_dynamic / action_mask,
 * writes ramp_env_buffers_t.actions (greedy: the first maximal logit; sample: categorical over softmax(logits) from a counter-based
 * generator keyed by (seed, episode)); finished episodes get action 0.  No host transfer. */
int ramp_policy_act(ramp_policy_t* p, ramp_engine_t* eng, int32_t sample, uint64_t seed);
/* HOST copies of the last ramp_policy_act: logits [B][n_actions], value [B], log-probability of the chosen action [B], actions [B] (any may be NULL);
 * RAMP_ERR_BAD_ARG unless that act ran for an environment of `eng`'s size */
int ramp_policy_read(ramp_policy_t* p, ramp_engine_t* eng, float* logits_out, float* value_out, float* logp_out, int32_t* actions_out);

/* A rollout segment recorded on the device, for a trainer: ramp_policy_trajectory_begin sizes [horizon][n_episodes] slots;
 * ramp_policy_trajectory_record(t, 0) after ramp_policy_act stores what the policy saw and decided in slot t (dynamic graph features,
 * model of the queued job, action mask, action, its log-probability, the value estimate), (t, 1) after ramp_env_advance stores the
 * reward and done flag that came back -- device-to-device copies on the engine's stream, no synchronisation;
 * ramp_policy_trajectory_read copies the first n_steps slots to HOST arrays (any may be NULL): ONE transfer per segment instead of
 * one per step.  (The static part of the observation is a function of `model`: ramp_policy_set_model.) */
/* page-locked host memory for the read-back targets (any HOST pointer works; page-locked ones make the copies asynchronous DMA) */
void* ramp_pinned_alloc(size_t bytes);
void ramp_pinned_free(void* ptr);
int ramp_policy_trajectory_begin(ramp_policy_t* p, ramp_engine_t* eng, int32_t horizon);
int ramp_policy_trajectory_record(ramp_policy_t* p, ramp_engine_t* eng, int32_t t, int32_t phase);
int ramp_policy_trajectory_read(ramp_policy_t* p, ramp_engine_t* eng, int32_t n_steps, float* obs_dynamic_out, int32_t* model_out,
                                uint8_t* action_mask_out, int32_t* action_out, float* logp_out, float* value_out, double* reward_out,
                                uint8_t* done_out);

/* ---- the policy's gradient and RLlib's PPO learner step on the device.  fp32 kernels; every weight gradient is summed over the
 * rows (and a job type's nodes, edges and messages) in a fixed order with f64 accumulators and no atomics, so one call on one
 * batch gives the same bits every time.  Derivatives as torch defines them: relu (y > 0), leaky_relu (y > 0 ? 1 : 0.01), tanh
 * (1 - y^2), LayerNorm with a biased variance and eps 1e-5; a zero-in-degree node passes no gradient (its output is the constant 0). */
/* HOST copy of the current weight blob [ramp_policy_weight_count] (after a learn call: the updated weights) */
int ramp_policy_get_weights(ramp_policy_t* p, float* out);
/* gradient of sum(grad_logits . logits) + sum(grad_value . value) with respect to every weight, in blob order, for the read-out on
 * HOST inputs (as ramp_policy_forward): grad_logits [n][n_actions], grad_value [n] -> grad_weights_out [ramp_policy_weight_count].
 * The mask is added to the logits with derivative 1 (torch: logits + max(log(mask), finfo.min)); rows whose model is outside
 * [0, n_models) contribute nothing. */
int ramp_policy_backward(ramp_policy_t* p, int32_t n, const int32_t* model, const float* graph_features, const uint8_t* action_mask,
                         const float* grad_logits, const float* grad_value, float* grad_weights_out);

/* ---- the policy's forward and backward on caller-owned DEVICE memory (e.g. PyTorch CUDA tensors), ordered on the caller's stream,
 * for a training loop written outside the library.  None of the three synchronises the host once every buffer has grown to its
 * size and each row count has been seen once: growing a buffer synchronises once, and the first backward of a new row count n
 * allocates and uploads that count's head-gradient segment table (a small table per distinct n, kept until the per-row scratch
 * grows past its largest n) and synchronises the stream once.  A loop whose batch sizes vary pays this once per size.  The policy's staging,
 * per-row records, gradient and embeddings are reused by every call: each call's stream first waits for an event recorded at the
 * end of the policy's previous call, on whatever stream that ran, host-input calls included, and records it again when done, so
 * calls alternating between streams are ordered without a device synchronisation.
 * ramp_policy_set_weights_device: a device-to-device copy of weights [ramp_policy_weight_count] into the policy's blob, enqueued on
 * `stream`; the embeddings become stale.
 * ramp_policy_forward_device: ramp_policy_forward's read-out of n rows (the job types embedded first on `stream` when stale):
 * model [n] (model_dtype RAMP_MODEL_INT32 / _INT64; any value outside [0, n_models) -- a finished episode's -1, an int64 that
 * int32 would wrap -- makes its row dead: logits and value 0), graph_features rows graph_features_stride floats apart of which the
 * first in_features_graph are read (the environment's [n][17 + n_actions] rows in place), action_mask [n][n_actions] bytes (0 / non-0)
 * -> logits_out [n][n_actions], value_out [n], the bits ramp_policy_forward gives for the same inputs.
 * ramp_policy_backward_device: ramp_policy_backward's gradient for the same inputs and grad_logits [n][n_actions], grad_value [n]
 * -> grad_weights_out [ramp_policy_weight_count]: ramp_policy_backward's bits.  A dead row passes no gradient.  Once a backward has
 * run, a forward that finds the embeddings stale remakes them with the gradient kernel's forward instance (the same bits) and
 * keeps its MeanPool states, and the next backward at the same weights reuses them instead of running the rounds again. */
#define RAMP_MODEL_INT32 0
#define RAMP_MODEL_INT64 1
int ramp_policy_set_weights_device(ramp_policy_t* p, const float* weights, int64_t n, void* stream);
int ramp_policy_forward_device(ramp_policy_t* p, void* stream, int32_t n, const void* model, int32_t model_dtype,
                               const float* graph_features, int64_t graph_features_stride, const uint8_t* action_mask,
                               float* logits_out, float* value_out);
int ramp_policy_backward_device(ramp_policy_t* p, void* stream, int32_t n, const void* model, int32_t model_dtype,
                                const float* graph_features, int64_t graph_features_stride, const uint8_t* action_mask,
                                const float* grad_logits, const float* grad_value, float* grad_weights_out);
/* CUDA-graph capture: ramp_policy_forward_device may be captured on `stream` (detected with cudaStreamIsCapturing).  Under capture
 * it launches the row gather and the read-out only, reading the embeddings from the buffer the policy holds for its whole life,
 * and does not use the fencing event: replays are ordered by the stream they run on.  It refuses (RAMP_ERR_BAD_ARG, nothing
 * enqueued) when the embeddings are stale, which would put a re-embed inside the graph, and when n is more rows than an eager call
 * has staged.  ramp_policy_backward_device refuses any capture.  A replay cannot see new weights:
 * ramp_policy_refresh_device re-embeds, eagerly on `stream` and into the same buffer, when the embeddings are stale (after
 * ramp_policy_set_weights_device), and does nothing otherwise; call it before the next replay.  Once a forward was captured,
 * staging that a later, larger call outgrows is kept until ramp_policy_destroy instead of being freed, so the graph's addresses
 * stay valid. */
int ramp_policy_refresh_device(ramp_policy_t* p, void* stream);

/* PPO's settings (RLlib PPOConfig names; scripts/ramp_job_partitioning_configs/algo/ppo.yaml holds the reference's values) */
typedef struct {
    uint64_t seed;                        /* minibatch shuffles: pass p draws its permutation from splitmix64 keyed by (seed, p)   */
    double gamma, lambda;                 /* GAE                                                                                   */
    double clip_param, vf_clip_param, vf_loss_coeff, entropy_coeff;
    double kl_coeff, kl_target;           /* the KL term's coefficient, and the target update_kl adapts it to                      */
    double grad_clip;                     /* global-norm clip (clip_grad_norm_); <= 0: none                                        */
    double lr, adam_beta1, adam_beta2, adam_eps;   /* torch.optim.Adam                                                             */
    int32_t sgd_minibatch_size, num_sgd_iter;
    int32_t standardize_advantages;       /* 1: (a - mean) / max(1e-4, std) over the train batch (RLlib standardize_fields)       */
} ramp_ppo_config_t;

/* a minibatch's statistics (stats_out of ramp_ppo_loss_grad; ramp_policy_learn: the mean over the last pass's minibatches) */
enum { RAMP_PPO_TOTAL_LOSS = 0, RAMP_PPO_POLICY_LOSS, RAMP_PPO_VF_LOSS, RAMP_PPO_ENTROPY, RAMP_PPO_KL,
       RAMP_PPO_CLIP_FRAC,                /* rows whose clipped surrogate was the smaller term, so the ratio passed no gradient   */
       RAMP_PPO_GRAD_NORM,                /* global norm of the gradient before clipping                                          */
       RAMP_PPO_KL_COEFF,                 /* loss_grad: the coefficient used; learn: the coefficient after update_kl              */
       RAMP_PPO_ROWS,                     /* loss_grad: rows of the minibatch; learn: rows of the train batch                     */
       RAMP_PPO_STATS_LEN };

/* PPOTorchPolicy.loss (ray/rllib/algorithms/ppo/ppo_torch_policy.py of the ray 3.0.0.dev0 the reference pins) on one minibatch of
 * HOST inputs, and its gradient, with no update:
 *   ratio = exp(logp(a) - logp_old(a)),  logp_old from old_logits (the collection weights' logits, masked entries included)
 *   loss  = mean(-min(adv ratio, adv clamp(ratio, 1 - clip, 1 + clip)) + vf_loss_coeff clamp((V - value_target)^2, 0, vf_clip)
 *                - entropy_coeff H(pi)) + kl_coeff mean(KL(pi_old || pi))
 * with torch.distributions.Categorical's entropy and KL: a masked action has probability 0 and adds exactly 0.  grad_out:
 * [ramp_policy_weight_count] or NULL; stats_out: [RAMP_PPO_STATS_LEN] or NULL. */
int ramp_ppo_loss_grad(ramp_policy_t* p, const ramp_ppo_config_t* cfg, int32_t n, const int32_t* model, const float* graph_features,
                       const uint8_t* action_mask, const int32_t* action, const float* old_logits, const float* advantage,
                       const float* value_target, float* grad_out, double* stats_out);
/* One PPO learner step on the first n_steps slots of the trajectory of the last ramp_policy_trajectory_begin (RAMP_ERR_BAD_ARG
 * unless that many slots were recorded since, both phases, in order), on the engine's stream, nothing read back but stats_out:
 *   1. GAE per episode (RLlib compute_advantages): delta = r + gamma V' (1 - done) - V, adv = delta + gamma lambda (1 - done) adv';
 *      value_target = adv + V.  A segment that ends before its episode does (truncate_episodes) bootstraps with V of the
 *      state after its last step: the value recorded in slot n_steps when more slots were recorded, else the value of the
 *      environment's current state.  The rows of episodes not finished when the decision was taken, t-major, form the train
 *      batch; its advantages are standardised when cfg asks.
 *   2. the collection weights' logits of every row, recomputed once (the same kernel and inputs as ramp_policy_act: its bits)
 *   3. num_sgd_iter passes, each over the train batch shuffled, of minibatch updates: the loss above, its gradient, clip_grad_norm_
 *      to grad_clip, torch.optim.Adam (moments and step count kept by the policy across calls)
 *   4. stats_out [RAMP_PPO_STATS_LEN]: the means over the last pass's minibatches, and kl_coeff after RLlib's update_kl (x 1.5 above
 *      2 kl_target, x 0.5 below kl_target / 2) -- the caller passes it as cfg->kl_coeff next time.
 * The embeddings become stale (the next forward re-embeds).  num_sgd_iter 0 builds the train batch only. */
int ramp_policy_learn(ramp_policy_t* p, ramp_engine_t* eng, int32_t n_steps, const ramp_ppo_config_t* cfg, double* stats_out);
/* HOST copies of the last ramp_policy_learn's train batch (any array may be NULL): n_out rows; per row the job type, the action,
 * the collected log-probability, the one recomputed from the collection weights' logits (written by the first pass), the
 * advantage (standardised when asked) and the value target.  After a ramp_policy_learn_pg, PG's batch: advantage and value
 * target are the discounted return. */
int ramp_policy_train_batch_read(ramp_policy_t* p, ramp_engine_t* eng, int32_t* n_out, int32_t* model_out, int32_t* action_out,
                                 float* logp_out, float* logp_old_out, float* advantage_out, float* value_target_out);
/* HOST copies of Adam's state (any may be NULL): exp_avg and exp_avg_sq [ramp_policy_weight_count], and the step count --
 * torch.optim.Adam's state for the one flat parameter; zeros before the first update */
int ramp_policy_learner_state(ramp_policy_t* p, float* exp_avg_out, float* exp_avg_sq_out, int32_t* step_out);
/* zeroes Adam's moments and step count */
int ramp_policy_learner_reset(ramp_policy_t* p);
/* loads Adam's state from HOST arrays exp_avg, exp_avg_sq [n] and the step count (checkpoint and resume): n must be
 * ramp_policy_weight_count, step >= 0.  Allocates the learner's buffers when no learn call has yet. */
int ramp_policy_set_learner_state(ramp_policy_t* p, const float* exp_avg, const float* exp_avg_sq, int64_t n, int32_t step);
/* ramp_policy_act's call count, which its draws mix in (seed ^ 0x9E3779B97F4A7C15 * count); setting it makes a resumed policy
 * draw what the uninterrupted one would */
int ramp_policy_get_act_count(ramp_policy_t* p, uint64_t* out);
int ramp_policy_set_act_count(ramp_policy_t* p, uint64_t n);

/* ---- RLlib's IMPALA learner step on the device (ray 3.0.0.dev0, as the reference pins it): ray/rllib/algorithms/impala/
 * impala_torch_policy.py (VTraceLoss, ImpalaTorchPolicy.loss with _make_time_major and vtrace_drop_last_ts) and
 * vtrace_torch.py (multi_from_logits, from_importance_weights).  It reuses PPO's gradient kernels and Adam, and Adam's moments
 * and step count are the same policy-owned state (ramp_policy_learner_state / _reset serve both learners).  Only the reference's
 * IMPALA is supported: opt_type adam, num_sgd_iter 1, minibatch_buffer_size 1, vtrace_drop_last_ts True. */
typedef struct {
    double gamma;                         /* rllib_config.yaml's base (impala.yaml does not set it): 0.99                          */
    double vtrace_clip_rho_threshold;     /* rho-bar = min(rho, this) in the TD errors (algo/impala.yaml: 1.0)                     */
    double vtrace_clip_pg_rho_threshold;  /* min(rho, this) weights pg_adv (algo/impala.yaml: 1.0)                                 */
    double vf_loss_coeff, entropy_coeff;  /* VTraceLoss's coefficients (algo/impala.yaml: 0.5, 0.01)                               */
    double grad_clip;                     /* global-norm clip (clip_grad_norm_; algo/impala.yaml: 40); <= 0: none                  */
    double lr, adam_beta1, adam_beta2, adam_eps;   /* torch.optim.Adam; RLlib passes only lr (rllib_config.yaml's base: 1e-4)      */
    int32_t rollout_fragment_length;      /* L: rows per fragment (0: the call's n_steps)                                          */
    int32_t train_batch_size;             /* rows per SGD step: floor(train_batch_size / L) whole fragments (rllib_config.yaml: 200) */
} ramp_impala_config_t;

/* statistics (stats_out of ramp_policy_learn_impala: the means over the call's SGD steps; of ramp_impala_loss_grad: its one batch) */
enum { RAMP_IMPALA_TOTAL_LOSS = 0,        /* pi_loss + vf_loss_coeff vf_loss - entropy_coeff sum(H): VTraceLoss.total_loss        */
       RAMP_IMPALA_POLICY_LOSS,           /* -sum(valid logp(a) pg_adv)                                                           */
       RAMP_IMPALA_VF_LOSS,               /* 0.5 sum(valid (V - vs)^2)                                                            */
       RAMP_IMPALA_ENTROPY,               /* mean H(pi) over the valid rows (VTraceLoss.mean_entropy; 0 with no valid row)        */
       RAMP_IMPALA_GRAD_NORM,             /* global norm of the gradient before clipping                                          */
       RAMP_IMPALA_MEAN_RHO,              /* mean rho = exp(log rho) over the valid rows (0 with no valid row)                    */
       RAMP_IMPALA_ROWS,                  /* valid rows: decisions in rows 0 .. L-2 of their fragment                             */
       RAMP_IMPALA_SGD_STEPS,             /* learn: the call's Adam steps; loss_grad: 0                                           */
       RAMP_IMPALA_STATS_LEN };

/* VTraceLoss on n_fragments fragments of fragment_length (L >= 1) HOST rows each, row r = f L + t, and its gradient, with no
 * update.  Per row: model (outside [0, n_models): no decision), graph_features, action_mask, action, behaviour_logp (the collected
 * log-probability), reward, done.  With V and log p(a) from the read-out at the current weights, per fragment:
 *   log rho = log p(a) - behaviour_logp (0 on a row without decision), rho-bar = min(rho, clip_rho), c = min(rho, 1),
 *   discount = gamma (1 - done); rows 0 .. L-2 are the loss's, V_{L-1} is the bootstrap and vs_{L-1} = V_{L-1};
 *   delta_t = rho-bar_t (r_t + discount_t V_{t+1} - V_t), vs_t - V_t = delta_t + discount_t c_t (vs_{t+1} - V_{t+1}),
 *   pg_adv_t = min(rho_t, clip_pg_rho) (r_t + discount_t vs_{t+1} - V_t)          (f64, stored as fp32)
 *   total = -sum valid logp(a) pg_adv + vf_loss_coeff 0.5 sum valid (V - vs)^2 - entropy_coeff sum valid H(pi)
 * valid: a decision in rows 0 .. L-2; vs and pg_adv are constants.  grad_out [ramp_policy_weight_count], stats_out
 * [RAMP_IMPALA_STATS_LEN], vs_out / pg_adv_out / log_rho_out [n_fragments L]: each may be NULL.  cfg's rollout_fragment_length
 * and train_batch_size are not used. */
int ramp_impala_loss_grad(ramp_policy_t* p, const ramp_impala_config_t* cfg, int32_t n_fragments, int32_t fragment_length,
                          const int32_t* model, const float* graph_features, const uint8_t* action_mask, const int32_t* action,
                          const float* behaviour_logp, const double* reward, const uint8_t* done, float* grad_out,
                          double* stats_out, float* vs_out, float* pg_adv_out, float* log_rho_out);
/* One IMPALA learner step on the first n_steps slots of the trajectory of the last ramp_policy_trajectory_begin (the same checks
 * as ramp_policy_learn), on the engine's stream, nothing read back but stats_out.  L = rollout_fragment_length (0: n_steps);
 * RAMP_ERR_BAD_ARG unless L divides n_steps and train_batch_size >= L.  Fragments are each episode's column over L consecutive
 * slots, ordered time block by time block, then by episode; SGD step k takes fragments [k F, (k + 1) F), F =
 * floor(train_batch_size / L) (the last step may take fewer), in order, not shuffled.  Per step: the embeddings and the read-out
 * at the current weights (at the collection weights the target log p(a) is the collected one bit for bit), V-trace and the loss
 * of ramp_impala_loss_grad over the step's fragments, its gradient, clip_grad_norm_ to grad_clip, torch.optim.Adam.  A row
 * whose episode had already finished, or had nothing queued, is a row without decision.  stats_out [RAMP_IMPALA_STATS_LEN]:
 * the means over the call's steps, and their number.  The embeddings become stale (the next forward re-embeds). */
int ramp_policy_learn_impala(ramp_policy_t* p, ramp_engine_t* eng, int32_t n_steps, const ramp_impala_config_t* cfg, double* stats_out);
/* HOST copies of the per-row V-trace values of the last ramp_policy_learn_impala or ramp_impala_loss_grad, fragment-major (row
 * r = f L + t; each as the step that used it computed it): n_out rows, target log p(a) (0 on a row without decision), log rho, vs,
 * pg_adv.  Any array may be NULL. */
int ramp_impala_vtrace_read(ramp_policy_t* p, int32_t* n_out, float* target_logp_out, float* log_rho_out, float* vs_out,
                            float* pg_adv_out);

/* ---- RLlib's PG (REINFORCE) learner step on the device (ray 3.0.0.dev0, as the reference pins it): ray/rllib/algorithms/pg/
 * pg_torch_policy.py (pg_torch_loss; postprocess_trajectory -> utils.post_process_advantages) and
 * ray/rllib/evaluation/postprocessing.py (compute_advantages with use_gae False, use_critic False, last_r 0; discount_cumsum).
 * It reuses PPO's gradient kernels and Adam, and Adam's moments and step count are the same policy-owned state
 * (ramp_policy_learner_state / _reset serve every gradient learner). */
typedef struct {
    double gamma;                         /* discount_cumsum's gamma (rllib_config.yaml: 0.99)                                     */
    double grad_clip;                     /* global-norm clip (clip_grad_norm_); <= 0: none (PG sets none, the default)            */
    double lr, adam_beta1, adam_beta2, adam_eps;   /* torch.optim.Adam; RLlib passes only lr (rllib_config.yaml: 1e-4)             */
} ramp_pg_config_t;

/* statistics (stats_out of ramp_policy_learn_pg and ramp_pg_loss_grad) */
enum { RAMP_PG_POLICY_LOSS = 0,           /* -sum(logp(a) advantage) / rows: pg_torch_loss's policy_loss                           */
       RAMP_PG_ENTROPY,                   /* mean H(pi) over the rows with a decision (reporting only: not in the loss)            */
       RAMP_PG_GRAD_NORM,                 /* global norm of the gradient before clipping                                          */
       RAMP_PG_ROWS,                      /* rows the loss is averaged over                                                       */
       RAMP_PG_STATS_LEN };

/* pg_torch_loss on n HOST rows, and its gradient, with no update: loss = -mean(logp(a) advantage) over the n rows, log p(a) the
 * log-softmax of the masked logits at the current weights; no value, entropy or KL term.  A row whose model is outside
 * [0, n_models) adds nothing but counts in the mean.  grad_out [ramp_policy_weight_count] and stats_out [RAMP_PG_STATS_LEN] may
 * be NULL; cfg's gamma is not used. */
int ramp_pg_loss_grad(ramp_policy_t* p, const ramp_pg_config_t* cfg, int32_t n, const int32_t* model, const float* graph_features,
                      const uint8_t* action_mask, const int32_t* action, const float* advantage, float* grad_out, double* stats_out);
/* One PG learner step on the first n_steps slots of the trajectory of the last ramp_policy_trajectory_begin (the same checks as
 * ramp_policy_learn), on the engine's stream, nothing read back but stats_out:
 *   1. per episode, the discounted return adv_t = r_t + gamma (1 - done_t) adv_{t+1} (f64, stored as fp32), with adv = 0 after
 *      the segment's last slot even when the episode goes on: PG does not bootstrap.  The rows of episodes not finished when the
 *      decision was taken and with a queued job, t-major, form the train batch (ramp_ppo_gae_kernel's batch); no standardisation.
 *   2. one Adam step over the whole batch: the loss of ramp_pg_loss_grad at the current (collection) weights, its gradient,
 *      clip_grad_norm_ to grad_clip when > 0, torch.optim.Adam.  A batch with no row is no update: the step count stays.
 *   3. stats_out [RAMP_PG_STATS_LEN].
 * The embeddings become stale (the next forward re-embeds).  ramp_policy_train_batch_read then returns this batch: logp_old is the
 * log p(a) the gradient kernel recomputed at the collection weights, advantage and value_target are both the discounted return. */
int ramp_policy_learn_pg(ramp_policy_t* p, ramp_engine_t* eng, int32_t n_steps, const ramp_pg_config_t* cfg, double* stats_out);

/* ---- RLlib's evolution strategies (ES) training step on the device (ray/rllib/algorithms/es: es.py training_step,
 * utils.py compute_centered_ranks / batched_weighted_sum, optimizers.py Adam).  The B episodes of a device environment are one
 * population: episode 2i runs theta + sigma eps_i, episode 2i + 1 runs theta - sigma eps_i (i < N = (B - n_eval) / 2), the last
 * n_eval episodes run theta; eps_i = noise[k_i : k_i + n] of a HOST table given at creation.  The ES Adam state belongs to the
 * ES object: the policy's torch-Adam state (ramp_policy_learner_state) is never touched.  No float atomics: one seed gives the
 * same weights bit for bit. */
typedef struct ramp_es ramp_es_t;

typedef struct {
    uint64_t seed;                        /* noise indices and the sampled actions' draws are keyed by (seed, iteration, round, .)  */
    double noise_stdev;                   /* sigma (algo/es.yaml: 0.02)                                                            */
    double stepsize, l2_coeff;            /* Adam's step size, the L2 term of -g + l2_coeff theta (es.yaml: 0.01, 0.005)          */
    double adam_beta1, adam_beta2, adam_eps;       /* optimizers.Adam: 0.99, 0.999, 1e-8                                           */
    int32_t episodes_per_batch;           /* rounds run until at least this many noisy episodes ... (es.yaml: 1000)                 */
    int32_t train_batch_size;             /* ... and at least this many noisy env-steps were collected (200)                        */
    int32_t n_eval;                       /* unperturbed evaluation episodes per round: the last n_eval of the environment's       */
    int32_t report_length;                /* episode_reward_mean: the mean over the last report_length steps' eval means (10)      */
} ramp_es_config_t;

/* statistics of a training step (es.py's result and info) */
enum { RAMP_ES_EPISODE_REWARD_MEAN = 0,   /* mean of the last report_length steps' mean eval return (NaN before any eval episode) */
       RAMP_ES_EPISODE_LEN_MEAN,          /* mean env-steps of this step's eval episodes (NaN without one)                        */
       RAMP_ES_TIMESTEPS_THIS_ITER,       /* env-steps of the noisy episodes (ramp_es_update: 0)                                  */
       RAMP_ES_EPISODES_THIS_ITER,        /* noisy episodes: 2 x pairs                                                            */
       RAMP_ES_WEIGHTS_NORM,              /* sum theta^2 after the update                                                         */
       RAMP_ES_GRAD_NORM,                 /* sum g^2                                                                              */
       RAMP_ES_UPDATE_RATIO,              /* ||step|| / ||theta before the update||                                               */
       RAMP_ES_EVAL_RETURN_MEAN,          /* mean return of this step's eval episodes (NaN without one)                           */
       RAMP_ES_ROUNDS,                    /* rounds of the environment this step ran (ramp_es_update: 0)                          */
       RAMP_ES_STATS_LEN };

/* An ES learner for the policy: uploads noise[noise_size] (a HOST float32 table, RLlib's shared noise table); RAMP_ERR_BAD_ARG
 * when noise_size < ramp_policy_weight_count. */
int ramp_es_create(ramp_policy_t* p, const float* noise, int64_t noise_size, ramp_es_t** out);
void ramp_es_destroy(ramp_es_t* es);
/* One round of a training step starts: the caller has just reset the environment (its episode streams are drawn on the host).
 * Round r of iteration it draws pair i's noise index uniformly on [0, noise_size - n] from splitmix64 keyed by (seed, it, r,
 * 2i), forms every set's weights fl(theta +- fl(sigma eps)) and embeds every (set, job type) in one launch, on the engine's
 * stream.  Round 0 starts a new step record.  RAMP_ERR_BAD_ARG unless B - n_eval is even and >= 2, or when the policy does
 * not fit the environment (as ramp_policy_act). */
int ramp_es_round_begin(ramp_es_t* es, ramp_engine_t* eng, const ramp_es_config_t* cfg, int32_t round);
/* Env-step t of the round: every episode's sampled action from its own set's weights into the environment's action buffer, one
 * warp per episode -- ramp_policy_decide's arithmetic and draw (row b, sample 1) with the seed splitmix64 keyed by (seed,
 * iteration, round, 2t + 1), which is recorded.  No synchronisation. */
int ramp_es_act(ramp_es_t* es, ramp_engine_t* eng, int32_t t);
/* The round's end: every episode's return (float of the environment's f64 sum) and env-step count into the step record, one
 * synchronisation.  *more_out = 1 while the record holds fewer than episodes_per_batch noisy episodes or train_batch_size noisy
 * env-steps. */
int ramp_es_round_end(ramp_es_t* es, ramp_engine_t* eng, int32_t* more_out);
/* The update on the step record: ramp_es_update on its pairs, plus the eval statistics; the policy's weights change in place
 * and its embeddings become stale.  stats_out [RAMP_ES_STATS_LEN] or NULL. */
int ramp_es_step(ramp_es_t* es, const ramp_es_config_t* cfg, double* stats_out);
/* The update on HOST inputs: returns [n_pairs][2] (R+, R-) of pairs with noise indices noise_index [n_pairs] ->
 *   ranks = compute_centered_ranks over the 2 n_pairs returns in pair order, ties in index order (a stable argsort)
 *   g = sum_i (rank+_i - rank-_i) eps_i / (2 n_pairs)          (f64 sums in pair order, stored as float32)
 *   optimizers.Adam on -g + l2_coeff theta, every operation float32, theta written in place.
 * ranks_out [n_pairs][2], grad_out [ramp_policy_weight_count], stats_out [RAMP_ES_STATS_LEN]: each may be NULL. */
int ramp_es_update(ramp_es_t* es, const ramp_es_config_t* cfg, int32_t n_pairs, const int32_t* noise_index, const float* returns,
                   float* ranks_out, float* grad_out, double* stats_out);
/* HOST copies of the last step's record (any array may be NULL; the counts first): its pairs' noise indices [n_pairs], returns
 * and env-steps [n_pairs][2], the act seeds in order [n_seeds], the ranks [n_pairs][2], g [ramp_policy_weight_count], the eval
 * episodes' returns and env-steps [n_eval] */
int ramp_es_read(ramp_es_t* es, int32_t* n_pairs_out, int32_t* n_eval_out, int32_t* n_seeds_out, int32_t* noise_index_out,
                 float* returns_out, int32_t* lengths_out, uint64_t* seeds_out, float* ranks_out, float* grad_out,
                 float* eval_returns_out, int32_t* eval_lengths_out);
/* HOST copies of the last ramp_es_act's logits [B][n_actions], log-probabilities [B] and actions [B] (any may be NULL) */
int ramp_es_act_read(ramp_es_t* es, ramp_engine_t* eng, float* logits_out, float* logp_out, int32_t* actions_out);
/* HOST copies of the ES Adam state (any may be NULL): m, v [ramp_policy_weight_count] and t; ramp_es_reset zeroes them */
int ramp_es_state(ramp_es_t* es, float* m_out, float* v_out, int32_t* t_out);
int ramp_es_reset(ramp_es_t* es);
/* loads the ES Adam state from HOST arrays m, v [n] and t: n must be ramp_policy_weight_count, t >= 0 (checkpoint and resume) */
int ramp_es_set_state(ramp_es_t* es, const float* m, const float* v, int64_t n, int32_t t);
/* What the next steps read besides theta and the Adam state: the iteration count (ramp_es_step calls so far, unless set: it keys
 * the noise indices and the act seeds) and every step's mean eval return so far (episode_reward_mean's report_length window).
 * get: any pointer may be NULL (rewards_out NULL to learn *n_rewards_out first); set: iteration >= 0, rewards [n_rewards] HOST. */
int ramp_es_get_progress(ramp_es_t* es, int64_t* iteration_out, int32_t* n_rewards_out, double* rewards_out);
int ramp_es_set_progress(ramp_es_t* es, int64_t iteration, int32_t n_rewards, const double* rewards);

/* ---- A population of K independent PPO, IMPALA or PG trainings in one environment batch.  The environment's B = K b episodes
 * are K contiguous groups of b; group k acts with weight set k and learns only from its own episodes with its own config.  Group
 * k computes, bit for bit, what one policy holding set k's weights (ramp_policy_act, ramp_policy_learn* with config k) computes
 * on a b-episode environment with the same episode streams.  The kernels run every group in the same launches: the MeanPool rounds
 * and their backward on one CTA per (set, job type) item, grid-strided past the resident CTAs; no float atomics. */
typedef struct ramp_population ramp_population_t;
/* K = n_sets weight sets with p's configuration and job types, each a copy of p's current weights, and K Adam states at zero.  p
 * stays the population's template: its job types must not change, and it must outlive the population.  The population's act
 * writes p's act outputs, so ramp_policy_read and ramp_policy_trajectory_* on p record the population's decisions. */
int ramp_population_create(ramp_policy_t* p, int32_t n_sets, ramp_population_t** out);
/* K = n_sets weight sets whose shapes may differ: set k has configuration cfgs[k] (HOST, [n_sets]), K Adam states at zero and no
 * weights yet -- act and learn refuse to run, naming the set, until ramp_population_set_weights gave every set its blob.  Each
 * cfgs[k] must be a valid configuration with the template's in_features_node / _edge / _graph, n_actions and n_models (the
 * environment and its job types fix them); widths, rounds, fcnet_hidden, the activations and vf_share_layers are the set's own.
 * Errors name the set.  p is the template as for ramp_population_create; its weights are not used.  Every set runs in the same
 * launches as a population of one shape; the read-out launches reserve the largest set's shared memory.
 * ramp_population_create(p, K) is this call with K copies of p's configuration, followed by a copy of p's weights into every set. */
int ramp_population_create_configs(ramp_policy_t* p, int32_t n_sets, const ramp_policy_config_t* cfgs, ramp_population_t** out);
void ramp_population_destroy(ramp_population_t* q);
/* set k's weights from / to a HOST blob of ramp_policy_weight_count(cfgs[k]) floats: set_weights refuses any other n */
int ramp_population_set_weights(ramp_population_t* q, int32_t set, const float* weights, int64_t n);
int ramp_population_get_weights(ramp_population_t* q, int32_t set, float* out);
/* ramp_policy_act for every group: episode k b + i draws as episode i of a policy whose ramp_policy_act got seeds[k] (HOST,
 * [n_sets]; may be NULL when sample is 0) with the population's call count.  RAMP_ERR_BAD_ARG unless n_sets divides B. */
int ramp_population_act(ramp_population_t* q, ramp_engine_t* eng, int32_t sample, const uint64_t* seeds);
/* ramp_policy_learn for every group on its columns of the template's trajectory, with cfgs[k] (HOST, [n_sets]); every config must
 * have the same sgd_minibatch_size and num_sgd_iter.  stats_out: [n_sets][RAMP_PPO_STATS_LEN] or NULL. */
int ramp_population_learn(ramp_population_t* q, ramp_engine_t* eng, int32_t n_steps, const ramp_ppo_config_t* cfgs, double* stats_out);
/* ramp_policy_learn_impala for every group on its columns of the template's trajectory, with cfgs[k] (HOST, [n_sets]).  Group k's
 * fragments are ordered as a b-episode environment's: time block by time block, then episode.  rollout_fragment_length and
 * train_batch_size fix the SGD steps, so every config must have the same values; gamma, the clip thresholds, the loss
 * coefficients, grad_clip and Adam's settings are the set's own.  SGD step k of every set runs in the same launches.  Adam's
 * moments and step counts are the population's, the same state ramp_population_learn updates.  stats_out:
 * [n_sets][RAMP_IMPALA_STATS_LEN] or NULL.  A configuration error names the set. */
int ramp_population_learn_impala(ramp_population_t* q, ramp_engine_t* eng, int32_t n_steps, const ramp_impala_config_t* cfgs, double* stats_out);
/* ramp_policy_learn_pg for every group on its columns of the template's trajectory, with cfgs[k] (HOST, [n_sets]); nothing has to
 * agree across sets.  A group whose batch has no row makes no update and keeps its step count.  stats_out:
 * [n_sets][RAMP_PG_STATS_LEN] or NULL.  A configuration error names the set. */
int ramp_population_learn_pg(ramp_population_t* q, ramp_engine_t* eng, int32_t n_steps, const ramp_pg_config_t* cfgs, double* stats_out);
/* ramp_impala_vtrace_read for set k after the last ramp_population_learn_impala: its group's n_out fragment rows */
int ramp_population_vtrace_read(ramp_population_t* q, int32_t set, int32_t* n_out, float* target_logp_out, float* log_rho_out,
                                float* vs_out, float* pg_adv_out);
/* HOST copies of set k's Adam state, as ramp_policy_learner_state: ramp_policy_weight_count(cfgs[k]) floats each */
int ramp_population_learner_state(ramp_population_t* q, int32_t set, float* exp_avg_out, float* exp_avg_sq_out, int32_t* step_out);
/* loads set k's Adam state, as ramp_policy_set_learner_state: n must be ramp_policy_weight_count(cfgs[k]) */
int ramp_population_set_learner_state(ramp_population_t* q, int32_t set, const float* exp_avg, const float* exp_avg_sq, int64_t n, int32_t step);
/* Population-based training's exploit: for every i < n_pairs, set src[i]'s weights, Adam exp_avg / exp_avg_sq and step count onto
 * set dst[i] (HOST [n_pairs] each), in one kernel launch (one CTA row per pair, grid-strided over the slice) on the default
 * stream, ordered after the population's last call and before its next by the template's completion event; no host
 * synchronisation.  Every population cache of a destination is stale afterwards: its MeanPool embeddings are recomputed by the
 * next act or learn call.  Refused, naming the pair: a set outside [0, n_sets), two sets of different ramp_policy_config_t, a set
 * that is the destination of two pairs, a set that is both a source and a destination (so the result does not depend on the
 * order the pairs run in), a source without weights. */
int ramp_population_copy_sets(ramp_population_t* q, int32_t n_pairs, const int32_t* dst, const int32_t* src);
/* the population's act call count, which every group's draws mix in (ramp_policy_get_act_count) */
int ramp_population_get_act_count(ramp_population_t* q, uint64_t* out);
int ramp_population_set_act_count(ramp_population_t* q, uint64_t n);
/* the CTAs of the population's MeanPool launches: n_sets n_models items, at most the resident CTAs, each CTA runs items
 * c, c + ctas, ... */
int ramp_population_embed_ctas(ramp_population_t* q, int32_t* ctas_out);

/* ---- ES for every set of a population: group k of the environment's B = K b episodes is the ES population of weight set k
 * with cfgs[k] (HOST, [K]): 2 N_k = b - n_eval_k noisy episodes, then n_eval_k eval episodes at theta_k.  Group k ends each step
 * where ramp_es_* on a policy holding set k's weights (and that set's configuration) ends on a b-episode environment with the same
 * episode streams, bit for bit: its step record, statistics, theta_k and ES Adam state.  Noise indices and act seeds are keyed by
 * (cfgs[k].seed, iteration, round, .) with the group's own pair and episode indices; the iteration count is the learner's.
 * theta_k is the population's set k, updated in place; the ES Adam state (m, v, t per set) belongs to the learner, and the
 * population's torch-Adam state (ramp_population_learner_state) is not touched.  Every configuration error names the set. */
typedef struct ramp_population_es ramp_population_es_t;
/* uploads noise[noise_size] (RLlib's shared noise table, HOST float32), which must cover the largest set's weights */
int ramp_population_es_create(ramp_population_t* q, const float* noise, int64_t noise_size, ramp_population_es_t** out);
void ramp_population_es_destroy(ramp_population_es_t* es);
/* ramp_es_round_begin for every group (the same checks per set; n_sets must divide B).  A group's twin stops after the round at
 * whose end its record holds episodes_per_batch noisy episodes and train_batch_size noisy env-steps; in every later round of the
 * step the group has no pairs: all its episodes run theta_k and nothing of theirs is recorded.  A round after every group
 * stopped is refused. */
int ramp_population_es_round_begin(ramp_population_es_t* es, ramp_engine_t* eng, const ramp_es_config_t* cfgs, int32_t round);
/* ramp_es_act for every group: episode k b + i is episode i of group k's twin, with group k's act seed */
int ramp_population_es_act(ramp_population_es_t* es, ramp_engine_t* eng, int32_t t);
/* ramp_es_round_end for every group that ran pairs in the round; *more_out = 1 while any group's twin would run another round */
int ramp_population_es_round_end(ramp_population_es_t* es, ramp_engine_t* eng, int32_t* more_out);
/* ramp_es_step for every set, each on its own record with cfgs[k]: ranks over its own pairs, g, Adam and the norms in the single
 * update's partition and order.  stats_out [n_sets][RAMP_ES_STATS_LEN] or NULL. */
int ramp_population_es_step(ramp_population_es_t* es, const ramp_es_config_t* cfgs, double* stats_out);
/* ramp_es_update for every set on HOST inputs: set k's n_pairs[k] pairs follow set k - 1's in noise_index [sum n_pairs] and
 * returns [sum n_pairs][2].  Its ranks and g are read back by ramp_population_es_read.  stats_out [n_sets][RAMP_ES_STATS_LEN] or NULL. */
int ramp_population_es_update(ramp_population_es_t* es, const ramp_es_config_t* cfgs, const int32_t* n_pairs, const int32_t* noise_index,
                              const float* returns, double* stats_out);
/* ramp_es_read of set k's last step record; grad_out has set k's weight count */
int ramp_population_es_read(ramp_population_es_t* es, int32_t set, int32_t* n_pairs_out, int32_t* n_eval_out, int32_t* n_seeds_out,
                            int32_t* noise_index_out, float* returns_out, int32_t* lengths_out, uint64_t* seeds_out, float* ranks_out,
                            float* grad_out, float* eval_returns_out, int32_t* eval_lengths_out);
/* HOST copies of the last ramp_population_es_act's logits [B][n_actions], log-probabilities [B] and actions [B] (any may be NULL) */
int ramp_population_es_act_read(ramp_population_es_t* es, ramp_engine_t* eng, float* logits_out, float* logp_out, int32_t* actions_out);
/* set k's ES Adam state, as ramp_es_state; ramp_population_es_reset zeroes every set's */
int ramp_population_es_state(ramp_population_es_t* es, int32_t set, float* m_out, float* v_out, int32_t* t_out);
int ramp_population_es_reset(ramp_population_es_t* es);
/* loads set k's ES Adam state, as ramp_es_set_state: n must be ramp_policy_weight_count(cfgs[k]) */
int ramp_population_set_es_state(ramp_population_es_t* es, int32_t set, const float* m, const float* v, int64_t n, int32_t t);
/* ramp_es_get_progress / _set_progress for set k: the iteration count is the learner's, one for every set (setting it through
 * any set sets it for all); the eval means are set k's own */
int ramp_population_get_es_progress(ramp_population_es_t* es, int32_t set, int64_t* iteration_out, int32_t* n_rewards_out, double* rewards_out);
int ramp_population_set_es_progress(ramp_population_es_t* es, int32_t set, int64_t iteration, int32_t n_rewards, const double* rewards);
/* ramp_population_copy_sets' exploit for the ES learner's state: set src[i]'s ES Adam m and v onto set dst[i]'s in one launch of
 * the same kernel, its t and its eval means (episode_reward_mean's window) on the host; the same checks, naming the pair.  The
 * weights are the population's: copy them with ramp_population_copy_sets. */
int ramp_population_copy_es_sets(ramp_population_es_t* es, int32_t n_pairs, const int32_t* dst, const int32_t* src);
/* the last round's embedding launch: its CTAs and its (ES weight set, job type) items; each CTA runs items c, c + ctas, ... */
int ramp_population_es_embed_ctas(ramp_population_es_t* es, int32_t* ctas_out, int32_t* items_out);

#ifdef __cplusplus
}
#endif
#endif
