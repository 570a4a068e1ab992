/*
 * TEST INFRASTRUCTURE -- CPU oracle for the RampClusterEnvironment.step() hot path.
 *
 * A plain-C restatement of the reference's algorithm (cwfparsonson/ddls @ 9e0b5ba,
 * ddls/environments/ramp_cluster/ramp_cluster_environment.py = "RCE",
 * ddls/demands/jobs/job.py = "JOB").  It is the checker the CUDA path is diffed
 * against; it is pinned against outputs of the reference itself run in the build
 * container (oracle/gen_golden.py -> tests/golden/).  Only tests/, bench.py's
 * cpu_baseline / --impl reference legs and __graft_entry__.smoke() may load it.
 * The product (ddls_b200/) never does.
 *
 * All floating point is IEEE f64 with no FMA contraction (-ffp-contract=off), the
 * same arithmetic as CPython floats.
 */
#ifndef RAMP_ORACLE_H
#define RAMP_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ORC_NO_CHANNEL 0xFFFFu

/* status codes */
#define ORC_OK 0
#define ORC_ERR_INFINITE_TICK 1   /* RCE:462 "Last tick was infinite" (deadlock)      */
#define ORC_ERR_TRACE_OVERFLOW 2  /* caller's trace buffer too small                   */
#define ORC_ERR_RULE_WORKER 3     /* RCE:1326-1328 one_job_per_worker                  */
#define ORC_ERR_RULE_CHANNEL 4    /* RCE:1367-1369 one_job_per_channel                 */
#define ORC_ERR_TABLE_FULL 5      /* running-job table capacity exceeded               */
#define ORC_ERR_BAD_ARG 6

/* One lowered (partitioned + placed + scheduled) job: the complete input of
 * RampClusterEnvironment._run_lookahead (RCE:379-467).  Op index = rank of the op id
 * in sorted() order, dep index = rank of the (u, v, k) tuple in sorted() order, so
 * that "first in sorted order wins ties" (RCE:56-66, RCE:672-685) is "lowest index
 * wins".  Out-edges are CSR by source op; because dep ids sort by (u, v, k) the CSR
 * position of a dep IS its dep index. */
typedef struct {
    int32_t n_ops;              /* N */
    int32_t n_deps;             /* E */
    int32_t n_workers;          /* workers this job is mounted on (job-local ids 0..W-1)  */
    int32_t n_channels;         /* channels this job is mounted on (job-local ids 0..C-1) */
    int32_t num_training_steps; /* JOB:82; jct, comm, comp are multiplied by it RCE:450-452 */
    int32_t model_id;           /* memo key part 1: job.details['model'] RCE:489          */
    int32_t degree;             /* memo key part 2: max partition degree RCE:488          */
    int32_t _pad;
    const double*   op_cost;      /* [N] compute_cost[device_type] -> initial remaining_run_time RCE:1334 */
    const int64_t*  op_prio;      /* [N] worker.mounted_job_op_to_priority RCE:1397          */
    const uint16_t* op_worker;    /* [N] job-local worker id RCE:1336                        */
    const uint16_t* op_n_parents; /* [N] |{p in pred(op): p not in succ(op)}| JOB:508-523    */
    const int32_t*  row_ptr;      /* [N+1] CSR out-edges; dep index range of op's out-edges  */
    const int32_t*  dep_dst;      /* [E] child op index                                      */
    const double*   dep_run_time; /* [E] init_run_time after RCE:542-560 (0 for non-flows)   */
    const int64_t*  dep_prio;     /* [E] channel.mounted_job_dep_to_priority RCE:1412        */
    const uint16_t* dep_channel;  /* [E] job-local channel id or ORC_NO_CHANNEL              */
    const uint8_t*  dep_is_flow;  /* [E] 0 if size == 0 or src server == dst server RCE:531-536 */
} orc_lowered_job_t;

/* Result of one lookahead (RCE:467). */
typedef struct {
    double jct;        /* lookahead_job_completion_time (x num_training_steps) */
    double comm;       /* communication_overhead_time   (x num_training_steps) */
    double comp;       /* computation_overhead_time     (x num_training_steps) */
    int32_t n_ticks;   /* T: len(tick_counter_to_active_workers_tick_size)     */
    int32_t status;
} orc_lookahead_result_t;

/* Runs RCE:379-467 on one lowered job.  trace_n_active/trace_tick (capacity
 * trace_cap, may be NULL with cap 0 to skip recording) receive
 * tick_counter_to_active_workers_tick_size[t] = [n_active, tick] for t = 1..T. */
int orc_run_lookahead(const orc_lowered_job_t* job,
                      int32_t* trace_n_active, double* trace_tick, int32_t trace_cap,
                      orc_lookahead_result_t* out);

/* mean_mounted_worker_utilisation_frac (RCE:830-832), serial sum in tick order. */
double orc_utilisation(const int32_t* trace_n_active, const double* trace_tick, int32_t n_ticks,
                       int32_t n_mounted_workers, double jct);

/* ------------------------------------------------------------------------- */
/* Episode-level oracle: RampClusterEnvironment.reset()/step() (RCE:202-295,
 * RCE:894-1179) driven by lowered jobs.                                      */

/* per-step statistics vector: indices into double[ORC_STEP_STATS_LEN]        */
enum {
    SS_STEP_COUNTER = 0,
    SS_STEP_START_TIME,
    SS_STEP_END_TIME,
    SS_STEP_TIME,
    SS_NUM_JOBS_COMPLETED,
    SS_NUM_JOBS_ARRIVED,
    SS_NUM_JOBS_BLOCKED,
    SS_JOB_QUEUE_LENGTH,
    SS_MEAN_NUM_JOBS_RUNNING,
    SS_MEAN_NUM_MOUNTED_WORKERS,
    SS_MEAN_NUM_MOUNTED_CHANNELS,
    SS_MEAN_COMPUTE_OVERHEAD_FRAC,
    SS_MEAN_COMMUNICATION_OVERHEAD_FRAC,
    SS_COMPUTE_INFO_PROCESSED,
    SS_DEP_INFO_PROCESSED,
    SS_FLOW_INFO_PROCESSED,
    SS_CLUSTER_INFO_PROCESSED,
    SS_DEMAND_COMPUTE_INFO_PROCESSED,
    SS_DEMAND_DEP_INFO_PROCESSED,
    SS_DEMAND_TOTAL_INFO_PROCESSED,
    SS_MEAN_COMPUTE_THROUGHPUT,
    SS_MEAN_DEP_THROUGHPUT,
    SS_MEAN_FLOW_THROUGHPUT,
    SS_MEAN_CLUSTER_THROUGHPUT,
    SS_MEAN_DEMAND_COMPUTE_THROUGHPUT,
    SS_MEAN_DEMAND_DEP_THROUGHPUT,
    SS_MEAN_DEMAND_TOTAL_THROUGHPUT,
    SS_UTIL_MOUNTED_SUM,   /* sum over outer-loop iterations of step_stats['mean_mounted_worker_utilisation_frac'] entries (a list in the reference, RCE:990) */
    SS_UTIL_CLUSTER_SUM,   /* same for 'mean_cluster_worker_utilisation_frac' RCE:991 */
    SS_NUM_TICKS,          /* number of outer-loop iterations this step (= len of the two lists above) */
    SS_DONE,               /* is_done() after the step RCE:1176 */
    SS_LOOKAHEAD_RAN,      /* 1 if this step executed _run_lookahead (memo miss), 0 otherwise */
    ORC_STEP_STATS_LEN
};

/* job status in the per-episode job record table */
enum { JS_NOT_ARRIVED = 0, JS_QUEUED = 1, JS_RUNNING = 2, JS_COMPLETED = 3, JS_BLOCKED = 4 };

/* Per-arrival description of a job as sampled by JobsGenerator (host ingest stays
 * Python; these are the only fields the hot path reads). */
typedef struct {
    double interarrival;      /* sample_interarrival_time() drawn when THIS job arrives RCE:363 (inf after the last job) */
    double orig_op_mem;       /* job.original_job.details['job_total_op_memory_cost'] */
    double orig_dep_size;     /* job.original_job.details['job_total_dep_size']       */
} orc_arrival_t;

/* Per-mount scalars of the partitioned job (read off Job.details by the lowering). */
typedef struct {
    double max_acceptable_jct;  /* details['max_acceptable_job_completion_time'][device] RCE:815 */
    double part_op_mem;         /* details['job_total_op_memory_cost'] of the partitioned job RCE:966 */
    double part_dep_size;       /* details['job_total_dep_size'] of the partitioned job RCE:967     */
    double flow_size;           /* sum of size over deps with run_time != 0 RCE:882-888            */
    int32_t n_mounted_workers;  /* len(job.details['mounted_workers'])  */
    int32_t n_mounted_channels; /* len(job.details['mounted_channels']) */
} orc_mount_t;

typedef struct {
    int32_t status;           /* JS_*                                 */
    int32_t event_seq;        /* order of completion / blocking event */
    double time_arrived;
    double time_started;
    double time_completed;
    double jct;               /* details['lookahead_job_completion_time'] */
    double comm;
    double comp;
    double util;              /* details['mean_mounted_worker_utilisation_frac'] */
} orc_job_record_t;

typedef struct orc_env orc_env_t;

orc_env_t* orc_env_create(int32_t n_cluster_workers, int32_t max_running_jobs, int32_t max_jobs,
                          int32_t memo_models, int32_t memo_degrees, int32_t trace_cap, double machine_epsilon);
void orc_env_destroy(orc_env_t* env);

/* RCE:202-295.  arrivals[0..n_jobs) is the arrival stream; arrivals[k].interarrival
 * is the gap added to time_next_job_to_arrive when job k arrives. */
int orc_env_reset(orc_env_t* env, double max_simulation_run_time, int32_t job_queue_capacity,
                  const orc_arrival_t* arrivals, int32_t n_jobs);

/* RCE:894-1179.  job == NULL is Action() (no job handled).  Otherwise the queued job
 * is partitioned/placed/scheduled as described by `job` + `mount`.
 * stats: double[ORC_STEP_STATS_LEN].  Returns ORC_OK or an error status. */
int orc_env_step(orc_env_t* env, const orc_lowered_job_t* job, const orc_mount_t* mount, double* stats);

/* lazily drawn arrival streams (see ramp_oracle.c) */
int orc_env_set_arrival(orc_env_t* env, int32_t k, const orc_arrival_t* row);
int orc_env_set_job_count(orc_env_t* env, int32_t n_jobs);

/* accessors */
int32_t orc_env_queued_job(const orc_env_t* env);   /* job idx at head of queue or -1 */
int32_t orc_env_num_jobs_arrived(const orc_env_t* env);
double  orc_env_time(const orc_env_t* env);
/* the last step's per-tick utilisation lists (RCE:989-994): returns their length, copies at most cap entries of each */
int32_t orc_env_tick_lists(const orc_env_t* env, double* mounted_out, double* cluster_out, int32_t cap);
double  orc_env_mean_load_rate(const orc_env_t* env);
const orc_job_record_t* orc_env_job_records(const orc_env_t* env);
/* last lookahead trace run or looked up by the env (for parity checks) */
int32_t orc_env_last_trace(const orc_env_t* env, const int32_t** n_active, const double** tick);

/* the episode scalars in the layout of the product's episode-state row (include/ramp_b200.h RAMP_EP_*) */
enum { ORC_EP_TIME = 0, ORC_EP_NEXT_ARRIVAL, ORC_EP_NUM_ARRIVED, ORC_EP_NUM_COMPLETED, ORC_EP_NUM_BLOCKED, ORC_EP_QUEUED_JOB,
       ORC_EP_NUM_RUNNING, ORC_EP_STEP_COUNTER, ORC_EP_LOAD_RATE_SUM, ORC_EP_LOAD_RATE_N, ORC_EP_DONE, ORC_EP_STATUS, ORC_EP_LEN };
void orc_env_episode_state(const orc_env_t* env, double* out /* [ORC_EP_LEN] */);

/* ------------------------------------------------------------------------- */
/* batched drivers (ramp_oracle_batch.c): one orc_env_t per episode, episodes spread over n_threads host threads.
 * script_tid / script_mount: [n_episodes][n_steps], tid -1 = Action(); arrivals: [n_episodes][n_jobs]. */
int orc_run_lookahead_batch(const orc_lowered_job_t* const* jobs, int32_t n, orc_lookahead_result_t* results, int32_t n_threads);
/* n_steps cluster steps per episode; stats_out [n_episodes][n_steps][ORC_STEP_STATS_LEN] may be NULL */
int orc_run_scripted_batch(const orc_lowered_job_t* templates, int32_t n_templates, int32_t n_episodes, int32_t n_steps,
                           const int32_t* script_tid, const orc_mount_t* script_mount, const orc_arrival_t* arrivals, int32_t n_jobs,
                           double max_sim_time, int32_t n_cluster_workers, int32_t memo_models, int32_t memo_degrees,
                           double* stats_out, orc_job_record_t* records_out, int32_t n_threads);
/* n_steps RampJobPartitioningEnvironment.step calls per episode (the action step, then Action() until a job is queued or the
 * episode is done); stats_out rows are the action steps' with SS_DONE taken after the whole env-step */
int orc_run_scripted_rjpe_batch(const orc_lowered_job_t* templates, int32_t n_templates, int32_t n_episodes, int32_t n_steps,
                                const int32_t* script_tid, const orc_mount_t* script_mount, const orc_arrival_t* arrivals, int32_t n_jobs,
                                double max_sim_time, int32_t n_cluster_workers, int32_t memo_models, int32_t memo_degrees,
                                double* stats_out, orc_job_record_t* records_out, int32_t n_threads);
/* The same env-steps with everything the product's step path hands back.  An episode that is done is not stepped again: its
 * later env-steps run no cluster step, and their stats_out rows are zero but for SS_STEP_COUNTER, SS_JOB_QUEUE_LENGTH and
 * SS_DONE, as the product writes them for a finished episode.  Outputs (each may be NULL):
 *   stats_out       [n_episodes][n_steps][ORC_STEP_STATS_LEN]   as orc_run_scripted_rjpe_batch
 *   ncs_out         [n_episodes][n_steps]                        cluster steps of each env-step
 *   cs_stats_out    [n_episodes][cs_cap][ORC_STEP_STATS_LEN]     every cluster step's row in order, fused Action() steps included
 *   cs_total_out    [n_episodes]                                 rows written to cs_stats_out
 *   records_out     [n_episodes][n_jobs]
 *   ep_out          [n_episodes][ORC_EP_LEN]                     orc_env_episode_state after the last env-step
 * Returns ORC_ERR_TRACE_OVERFLOW if an episode runs more than cs_cap cluster steps (cs_stats_out != NULL). */
int orc_run_scripted_rjpe_full_batch(const orc_lowered_job_t* templates, int32_t n_templates, int32_t n_episodes, int32_t n_steps,
                                     const int32_t* script_tid, const orc_mount_t* script_mount, const orc_arrival_t* arrivals,
                                     int32_t n_jobs, double max_sim_time, int32_t n_cluster_workers, int32_t memo_models,
                                     int32_t memo_degrees, double* stats_out, int32_t* ncs_out, double* cs_stats_out, int32_t cs_cap,
                                     int32_t* cs_total_out, orc_job_record_t* records_out, double* ep_out, int32_t n_threads);

#ifdef __cplusplus
}
#endif
#endif
