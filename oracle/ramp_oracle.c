/*
 * TEST INFRASTRUCTURE -- CPU oracle (see ramp_oracle.h).  NOT part of the product.
 *
 * Restates, function by function, the reference hot path:
 *   orc_run_lookahead        <- RampClusterEnvironment._run_lookahead            RCE:379-467
 *     worker winners         <- get_highest_priority_job_op_synchronous           RCE:44-67, RCE:562-590
 *     t_op                   <- _get_shortest_remaining_run_time_of_priority_job_ops RCE:592-606
 *     non-flow test          <- gather_job_ready_non_flow_deps                    RCE:520-540
 *     channel winners        <- _get_channel_to_priority_job_dep / _get_highest_priority_job_dep RCE:608-629, 665-689
 *                               (_resolve_contending_channels RCE:631-651 is a structural no-op: every
 *                               channel in priority_job_dep_to_channels[dep] already has dep as its winner)
 *     t_comm                 <- _get_shortest_remaining_communication_time_of_priority_job_deps RCE:653-663
 *     tick ops / deps        <- _tick_mounted_ops RCE:691-716, _tick_non_flow_deps RCE:718-731,
 *                               _tick_flow_deps RCE:733-775, Job.tick_op/tick_dep JOB:553-563,
 *                               Job.register_completed_op/dep JOB:492-536
 *     overheads              <- _record_communication_computation_overhead         RCE:777-791
 *   orc_env_step             <- RampClusterEnvironment.step                       RCE:894-1179
 *     memo                   <- _perform_lookahead_job_completion_time             RCE:469-518
 *     registration           <- _register_completed_lookahead                      RCE:793-888
 *     outer loop             <- RCE:942-1044, completion RCE:1466-1502, blocking RCE:1504-1540
 *
 * Compile with -O2 -ffp-contract=off (no FMA) so f64 results equal CPython's.
 */
#include "ramp_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------- */
/* lookahead                                                                  */

/* Python: x -= min(tick, x)   (JOB:555, JOB:561).  min(a, b) returns a unless b < a. */
static inline double tick_down(double rem, double tick) {
    double m = (rem < tick) ? rem : tick;
    return rem - m;
}

int orc_run_lookahead(const orc_lowered_job_t* job,
                      int32_t* trace_n_active, double* trace_tick, int32_t trace_cap,
                      orc_lookahead_result_t* out) {
    const int32_t N = job->n_ops, E = job->n_deps, W = job->n_workers, C = job->n_channels;
    memset(out, 0, sizeof(*out));
    if (N < 0 || E < 0 || W < 0 || C < 0) { out->status = ORC_ERR_BAD_ARG; return ORC_ERR_BAD_ARG; }

    double*  op_rem   = (double*)malloc(sizeof(double) * (size_t)(N > 0 ? N : 1));
    double*  dep_rem  = (double*)malloc(sizeof(double) * (size_t)(E > 0 ? E : 1));
    int32_t* par_done = (int32_t*)calloc((size_t)(N > 0 ? N : 1), sizeof(int32_t));
    int32_t* in_deg   = (int32_t*)calloc((size_t)(N > 0 ? N : 1), sizeof(int32_t));
    int32_t* ops_rdy  = (int32_t*)malloc(sizeof(int32_t) * (size_t)(N > 0 ? N : 1));
    int32_t* ops_nxt  = (int32_t*)malloc(sizeof(int32_t) * (size_t)(N > 0 ? N : 1));
    int32_t* deps_rdy = (int32_t*)malloc(sizeof(int32_t) * (size_t)(E > 0 ? E : 1));
    int32_t* deps_nxt = (int32_t*)malloc(sizeof(int32_t) * (size_t)(E > 0 ? E : 1));
    int32_t* w_best   = (int32_t*)malloc(sizeof(int32_t) * (size_t)(W > 0 ? W : 1));
    int32_t* c_best   = (int32_t*)malloc(sizeof(int32_t) * (size_t)(C > 0 ? C : 1));
    uint8_t* op_win   = (uint8_t*)calloc((size_t)(N > 0 ? N : 1), 1);

    for (int32_t i = 0; i < N; ++i) op_rem[i] = job->op_cost[i];        /* RCE:1334 */
    for (int32_t e = 0; e < E; ++e) { dep_rem[e] = job->dep_run_time[e]; in_deg[job->dep_dst[e]]++; } /* RCE:542-560 */

    /* JOB:474-484: source nodes (in_degree == 0) start ready */
    int32_t n_ops_rdy = 0, n_deps_rdy = 0;
    for (int32_t i = 0; i < N; ++i) if (in_deg[i] == 0) ops_rdy[n_ops_rdy++] = i;

    int32_t ops_completed = 0, deps_completed = 0;
    double t = 0.0, comm = 0.0, comp = 0.0;          /* Stopwatch UT:485-496; JOB:170-171 */
    int32_t tick_no = 0;                              /* lookahead_tick_counter - 1 */
    int status = ORC_OK;

    for (;;) {
        /* A. highest priority ready op per worker: iterate in sorted() order with strict '>'
         *    == max priority, lowest index on ties (RCE:56-66). */
        for (int32_t w = 0; w < W; ++w) w_best[w] = -1;
        for (int32_t k = 0; k < n_ops_rdy; ++k) {
            int32_t i = ops_rdy[k], w = job->op_worker[i], b = w_best[w];
            if (b < 0 || job->op_prio[i] > job->op_prio[b] || (job->op_prio[i] == job->op_prio[b] && i < b))
                w_best[w] = i;
        }
        /* B. RCE:592-606 */
        double t_op = INFINITY;
        for (int32_t w = 0; w < W; ++w)
            if (w_best[w] >= 0 && op_rem[w_best[w]] < t_op) t_op = op_rem[w_best[w]];

        /* C. RCE:520-540 */
        int any_non_flow = 0;
        for (int32_t k = 0; k < n_deps_rdy; ++k) if (!job->dep_is_flow[deps_rdy[k]]) { any_non_flow = 1; break; }

        /* D. RCE:412-422 */
        double t_comm;
        if (!any_non_flow) {
            for (int32_t c = 0; c < C; ++c) c_best[c] = -1;
            for (int32_t k = 0; k < n_deps_rdy; ++k) {
                int32_t e = deps_rdy[k];
                uint32_t c = job->dep_channel[e];
                if (c == ORC_NO_CHANNEL) continue;
                int32_t b = c_best[c];
                if (b < 0 || job->dep_prio[e] > job->dep_prio[b] || (job->dep_prio[e] == job->dep_prio[b] && e < b))
                    c_best[c] = e;
            }
            t_comm = INFINITY;
            for (int32_t c = 0; c < C; ++c)
                if (c_best[c] >= 0 && dep_rem[c_best[c]] < t_comm) t_comm = dep_rem[c_best[c]];
        } else {
            t_comm = 0.0;
        }

        /* E. RCE:426 */
        const double tick = (t_comm < t_op) ? t_comm : t_op;

        /* F. deps_ready snapshot RCE:429 == deps_rdy[0..n_deps_rdy); deps made ready by op
         *    completions below go to deps_nxt and are first ticked next iteration. */
        int32_t n_ops_nxt = 0, n_deps_nxt = 0;

        /* G. RCE:691-716 */
        int32_t n_active = 0;
        for (int32_t w = 0; w < W; ++w) if (w_best[w] >= 0) op_win[w_best[w]] = 1;
        for (int32_t k = 0; k < n_ops_rdy; ++k) {
            int32_t i = ops_rdy[k];
            if (op_win[i]) {
                op_win[i] = 0;
                n_active++;
                op_rem[i] = tick_down(op_rem[i], tick);               /* JOB:555 */
                if (op_rem[i] == 0) {                                  /* JOB:556, JOB:492-501 */
                    ops_completed++;
                    for (int32_t e = job->row_ptr[i]; e < job->row_ptr[i + 1]; ++e) deps_nxt[n_deps_nxt++] = e;
                    continue;
                }
            }
            ops_nxt[n_ops_nxt++] = i;
        }
        if (tick_no < trace_cap) { trace_n_active[tick_no] = n_active; trace_tick[tick_no] = tick; }
        else if (trace_cap > 0) status = ORC_ERR_TRACE_OVERFLOW;

        /* H. RCE:434-439 */
        int ticked_flows = 0;
        int32_t n_deps_keep = 0;
        for (int32_t k = 0; k < n_deps_rdy; ++k) {
            int32_t e = deps_rdy[k];
            if (any_non_flow && job->dep_is_flow[e]) { deps_rdy[n_deps_keep++] = e; continue; } /* RCE:720: only non-flows */
            if (!any_non_flow) ticked_flows = 1;                        /* RCE:767 */
            dep_rem[e] = tick_down(dep_rem[e], tick);                   /* JOB:561 */
            if (dep_rem[e] == 0) {                                      /* JOB:562, JOB:525-536 */
                deps_completed++;
                int32_t child = job->dep_dst[e];
                par_done[child]++;
                if (par_done[child] == (int32_t)job->op_n_parents[child]) ops_nxt[n_ops_nxt++] = child;
            } else {
                deps_rdy[n_deps_keep++] = e;
            }
        }
        /* merge surviving + newly ready deps */
        for (int32_t k = 0; k < n_deps_nxt; ++k) deps_rdy[n_deps_keep++] = deps_nxt[k];
        n_deps_rdy = n_deps_keep;
        { int32_t* tmp = ops_rdy; ops_rdy = ops_nxt; ops_nxt = tmp; n_ops_rdy = n_ops_nxt; }

        /* I. RCE:777-791 */
        const int ticked_ops = n_active > 0;
        if (ticked_ops && ticked_flows) { comm += tick; comp += tick; }
        else if (ticked_flows) comm += tick;
        else if (ticked_ops) comp += tick;

        /* J. RCE:445 */
        t += tick;
        tick_no++;

        /* K. RCE:447-453, JOB:549-551 */
        if (ops_completed == N && deps_completed == E) {
            out->jct = t * (double)job->num_training_steps;
            out->comm = comm * (double)job->num_training_steps;
            out->comp = comp * (double)job->num_training_steps;
            break;
        }
        /* L. RCE:462 */
        if (isinf(tick)) { status = ORC_ERR_INFINITE_TICK; break; }
    }
    out->n_ticks = tick_no;
    out->status = status;

    free(op_rem); free(dep_rem); free(par_done); free(in_deg); free(ops_rdy); free(ops_nxt);
    free(deps_rdy); free(deps_nxt); free(w_best); free(c_best); free(op_win);
    return status;
}

double orc_utilisation(const int32_t* trace_n_active, const double* trace_tick, int32_t n_ticks,
                       int32_t n_mounted_workers, double jct) {
    /* RCE:830-832 */
    double u = 0.0;
    for (int32_t k = 0; k < n_ticks; ++k)
        u += ((double)trace_n_active[k] / (double)n_mounted_workers) * (trace_tick[k] / jct);
    return u;
}

/* ------------------------------------------------------------------------- */
/* episode-level oracle                                                       */

typedef struct {
    int32_t job_idx;
    double jct, time_started, comm, comp, util;
    double part_op_mem, part_dep_size, flow_size, orig_op_mem, orig_dep_size;
    int32_t n_workers, n_channels;
} orc_running_t;

typedef struct {
    int valid;
    orc_lookahead_result_t res;
    int32_t* trace_n;
    double* trace_tick;
} orc_memo_t;

struct orc_env {
    int32_t n_cluster_workers, max_running, max_jobs, memo_models, memo_degrees, trace_cap;
    double eps;
    /* episode state */
    double now, next_arrival, last_arrival, max_sim_time;
    int32_t queue_capacity, queued_job, n_jobs, num_arrived, num_completed, num_blocked, step_counter, event_seq;
    const orc_arrival_t* arrivals; orc_arrival_t* arrivals_own;
    double load_rate_sum; int32_t load_rate_n;
    orc_running_t* running; int32_t n_running;
    orc_job_record_t* records;
    orc_memo_t* memo;
    const orc_memo_t* last_memo;
    double* stats; /* current step stats */
    /* the two per-tick lists of the last step (RCE:989-994): step_stats['mean_mounted_worker_utilisation_frac'] and
       ['mean_cluster_worker_utilisation_frac'] hold one entry per outer-loop iteration */
    double* tick_util_mounted; double* tick_util_cluster; int32_t n_tick_util, tick_util_cap;
};

orc_env_t* orc_env_create(int32_t n_cluster_workers, int32_t max_running_jobs, int32_t max_jobs,
                          int32_t memo_models, int32_t memo_degrees, int32_t trace_cap, double machine_epsilon) {
    orc_env_t* env = (orc_env_t*)calloc(1, sizeof(orc_env_t));
    env->n_cluster_workers = n_cluster_workers;
    env->max_running = max_running_jobs;
    env->max_jobs = max_jobs;
    env->memo_models = memo_models;
    env->memo_degrees = memo_degrees;
    env->trace_cap = trace_cap;
    env->eps = machine_epsilon;
    env->running = (orc_running_t*)calloc((size_t)max_running_jobs, sizeof(orc_running_t));
    env->records = (orc_job_record_t*)calloc((size_t)max_jobs, sizeof(orc_job_record_t));
    env->memo = (orc_memo_t*)calloc((size_t)memo_models * (size_t)memo_degrees, sizeof(orc_memo_t));
    env->arrivals_own = (orc_arrival_t*)calloc((size_t)max_jobs, sizeof(orc_arrival_t));
    return env;
}

static void memo_clear(orc_env_t* env) {
    for (int32_t k = 0; k < env->memo_models * env->memo_degrees; ++k) {
        free(env->memo[k].trace_n); free(env->memo[k].trace_tick);
        memset(&env->memo[k], 0, sizeof(orc_memo_t));
    }
    env->last_memo = NULL;
}

void orc_env_destroy(orc_env_t* env) {
    if (!env) return;
    memo_clear(env);
    free(env->running); free(env->records); free(env->memo); free(env->arrivals_own);
    free(env->tick_util_mounted); free(env->tick_util_cluster);
    free(env);
}

/* RCE:351-377 */
static void get_next_job(orc_env_t* env) {
    int32_t k = env->num_arrived;
    orc_job_record_t* r = &env->records[k];
    memset(r, 0, sizeof(*r));
    r->status = JS_QUEUED;
    r->time_arrived = env->now;
    env->last_arrival = env->now;                                   /* RCE:362 */
    env->next_arrival += env->arrivals[k].interarrival;             /* RCE:363 */
    env->load_rate_sum += (env->arrivals[k].orig_op_mem + env->arrivals[k].orig_dep_size)
                          / (env->next_arrival - env->last_arrival); /* RCE:364 */
    env->load_rate_n++;
    env->num_arrived++;
}

int orc_env_reset(orc_env_t* env, double max_simulation_run_time, int32_t job_queue_capacity,
                  const orc_arrival_t* arrivals, int32_t n_jobs) {
    if (n_jobs > env->max_jobs || n_jobs < 1) return ORC_ERR_BAD_ARG;
    memcpy(env->arrivals_own, arrivals, sizeof(orc_arrival_t) * (size_t)n_jobs);
    env->arrivals = env->arrivals_own;
    env->n_jobs = n_jobs;
    env->now = 0.0;                                  /* RCE:221 */
    env->max_sim_time = max_simulation_run_time;     /* RCE:227 */
    env->queue_capacity = job_queue_capacity;
    env->num_arrived = env->num_completed = env->num_blocked = 0;
    env->step_counter = 0; env->event_seq = 0;
    env->load_rate_sum = 0.0; env->load_rate_n = 0;
    env->n_running = 0;
    memset(env->records, 0, sizeof(orc_job_record_t) * (size_t)env->max_jobs);
    memo_clear(env);                                 /* RCE:269-275 */
    env->next_arrival = 0.0;                         /* RCE:280 */
    get_next_job(env);                               /* RCE:281 */
    env->queued_job = 0;
    return ORC_OK;
}

/* A host that draws jobs lazily from the reference's JobsGenerator (RCE:351-377) streams the arrival rows one ahead and
 * tells the env whether the generator still holds a job: `n_jobs - num_arrived > 0` stands for `len(jobs_generator) > 0`
 * (RCE:1019-1040).  Mirrors ramp_set_arrivals / ramp_set_job_count of the product's C ABI. */
int orc_env_set_arrival(orc_env_t* env, int32_t k, const orc_arrival_t* row) {
    if (k < 0 || k >= env->max_jobs) return ORC_ERR_BAD_ARG;
    env->arrivals_own[k] = *row;
    return ORC_OK;
}
int orc_env_set_job_count(orc_env_t* env, int32_t n_jobs) {
    if (n_jobs < 0 || n_jobs > env->max_jobs) return ORC_ERR_BAD_ARG;
    env->n_jobs = n_jobs;
    return ORC_OK;
}

/* RCE:1504-1540 (the counters; per-job lists are rebuilt from the records) */
static void register_blocked(orc_env_t* env, int32_t job_idx) {
    orc_job_record_t* r = &env->records[job_idx];
    if (env->queued_job == job_idx) env->queued_job = -1;
    if (r->status == JS_BLOCKED) return;
    r->status = JS_BLOCKED;
    r->event_seq = env->event_seq++;
    env->num_blocked++;
    env->stats[SS_NUM_JOBS_BLOCKED] += 1;
}

static void remove_running(orc_env_t* env, int32_t pos) {
    for (int32_t k = pos; k + 1 < env->n_running; ++k) env->running[k] = env->running[k + 1];
    env->n_running--;
    memset(&env->running[env->n_running], 0, sizeof(orc_running_t));
}

/* RCE:1542-1557 */
static int is_done(const orc_env_t* env) {
    if (env->now >= env->max_sim_time) return 1;
    if ((env->n_jobs - env->num_arrived) == 0 && env->n_running == 0 && env->queued_job < 0) return 1;
    return 0;
}

int orc_env_step(orc_env_t* env, const orc_lowered_job_t* job, const orc_mount_t* mount, double* stats) {
    memset(stats, 0, sizeof(double) * ORC_STEP_STATS_LEN);
    env->stats = stats;
    stats[SS_STEP_COUNTER] = (double)env->step_counter;       /* RCE:309 */
    stats[SS_STEP_START_TIME] = env->now;                     /* RCE:310 */

    const int32_t handled = (job != NULL) ? env->queued_job : -1;
    /* RCE:914-919: queued jobs not handled by the action are blocked */
    if (env->queued_job >= 0 && job == NULL) register_blocked(env, env->queued_job);
    if (job != NULL && handled < 0) return ORC_ERR_BAD_ARG;   /* action for a job that is not queued */

    if (job != NULL) {
        /* RCE:1305-1347, 1417-1423: place ops, register running */
        if (env->n_running >= env->max_running) return ORC_ERR_TABLE_FULL;
        orc_job_record_t* r = &env->records[handled];
        r->status = JS_RUNNING;
        r->time_started = env->now;                            /* RCE:1418 */
        env->queued_job = -1;                                  /* RCE:1420 */
        orc_running_t* run = &env->running[env->n_running++];
        memset(run, 0, sizeof(*run));
        run->job_idx = handled;
        run->time_started = env->now;
        run->part_op_mem = mount->part_op_mem; run->part_dep_size = mount->part_dep_size;
        run->flow_size = mount->flow_size;
        run->orig_op_mem = env->arrivals[handled].orig_op_mem;
        run->orig_dep_size = env->arrivals[handled].orig_dep_size;
        run->n_workers = mount->n_mounted_workers; run->n_channels = mount->n_mounted_channels;

        /* RCE:469-518: lookahead with the (model, max_num_partitions) memo */
        if (job->model_id < 0 || job->model_id >= env->memo_models || job->degree < 0 || job->degree >= env->memo_degrees)
            return ORC_ERR_BAD_ARG;
        orc_memo_t* m = &env->memo[(size_t)job->model_id * (size_t)env->memo_degrees + (size_t)job->degree];
        if (!m->valid) {
            int32_t cap = env->trace_cap > 0 ? env->trace_cap : (job->n_ops + job->n_deps + 1);
            m->trace_n = (int32_t*)malloc(sizeof(int32_t) * (size_t)cap);
            m->trace_tick = (double*)malloc(sizeof(double) * (size_t)cap);
            int st = orc_run_lookahead(job, m->trace_n, m->trace_tick, cap, &m->res);
            stats[SS_LOOKAHEAD_RAN] = 1;
            if (st != ORC_OK) { free(m->trace_n); free(m->trace_tick); m->trace_n = NULL; m->trace_tick = NULL; return st; }
            m->valid = 1;                                      /* RCE:503-506 */
        }
        env->last_memo = m;
        /* RCE:793-888 */
        if (m->res.jct > mount->max_acceptable_jct) {          /* RCE:815 strict '>' */
            register_blocked(env, handled);                    /* RCE:821 */
            remove_running(env, env->n_running - 1);           /* RCE:824 */
        } else {
            run->jct = m->res.jct; run->comm = m->res.comm; run->comp = m->res.comp;
            run->util = orc_utilisation(m->trace_n, m->trace_tick, m->res.n_ticks, mount->n_mounted_workers, m->res.jct);
            r->jct = run->jct; r->comm = run->comm; r->comp = run->comp; r->util = run->util;
        }
    }

    /* RCE:942-1044 */
    double util_mounted_sum = 0.0, util_cluster_sum = 0.0;
    double sum_jobs_running = 0.0, sum_workers = 0.0, sum_channels = 0.0, sum_comp_frac = 0.0, sum_comm_frac = 0.0;
    int32_t n_frac = 0, n_iter = 0;
    int step_done = 0;
    while (!step_done) {
        double tick = env->next_arrival - env->now;                           /* RCE:950 */
        { double b = env->max_sim_time - env->now; if (b < tick) tick = b; }
        for (int32_t k = 0; k < env->n_running; ++k) {                        /* RCE:951-954 */
            double elapsed = env->now - env->running[k].time_started;
            double remaining = env->running[k].jct - elapsed;
            if (remaining < tick) tick = remaining;
        }
        int32_t mounted_workers = 0, mounted_channels = 0;
        double util_sum = 0.0;
        for (int32_t k = 0; k < env->n_running; ++k) {                        /* RCE:962-982 */
            const orc_running_t* j = &env->running[k];
            double frac = tick / j->jct;
            stats[SS_COMPUTE_INFO_PROCESSED] += j->part_op_mem * frac;
            stats[SS_DEP_INFO_PROCESSED] += j->part_dep_size * frac;
            stats[SS_FLOW_INFO_PROCESSED] += j->flow_size * frac;
            stats[SS_CLUSTER_INFO_PROCESSED] += (j->part_op_mem + j->part_dep_size) * frac;
            stats[SS_DEMAND_COMPUTE_INFO_PROCESSED] += j->orig_op_mem * frac;
            stats[SS_DEMAND_DEP_INFO_PROCESSED] += j->orig_dep_size * frac;
            stats[SS_DEMAND_TOTAL_INFO_PROCESSED] += (j->orig_op_mem + j->orig_dep_size) * frac;
            sum_comp_frac += j->comp / j->jct; sum_comm_frac += j->comm / j->jct; n_frac++;
            mounted_workers += j->n_workers;      /* workers/channels of distinct jobs are disjoint (ramp_rules.py) */
            mounted_channels += j->n_channels;
            util_sum += j->util;
        }
        sum_jobs_running += (double)env->n_running;                           /* RCE:984 */
        sum_workers += (double)mounted_workers; sum_channels += (double)mounted_channels; /* RCE:986-987 */
        double tick_mounted = 0.0, tick_cluster = 0.0;
        if (env->n_running > 0) {                                             /* RCE:989-994 */
            double mean_util = util_sum / (double)env->n_running;
            tick_mounted = mean_util;
            tick_cluster = ((double)mounted_workers / (double)env->n_cluster_workers) * mean_util;
            util_mounted_sum += tick_mounted;
            util_cluster_sum += tick_cluster;
        }
        if (n_iter >= env->tick_util_cap) {
            env->tick_util_cap = env->tick_util_cap ? 2 * env->tick_util_cap : 64;
            env->tick_util_mounted = (double*)realloc(env->tick_util_mounted, sizeof(double) * (size_t)env->tick_util_cap);
            env->tick_util_cluster = (double*)realloc(env->tick_util_cluster, sizeof(double) * (size_t)env->tick_util_cap);
        }
        env->tick_util_mounted[n_iter] = tick_mounted; env->tick_util_cluster[n_iter] = tick_cluster;
        n_iter++;
        env->n_tick_util = n_iter;

        env->now += tick;                                                     /* RCE:998 */

        /* RCE:1004-1017: collect, then register in running-table (dict) order RCE:1466-1502 */
        {
            int32_t k = 0;
            while (k < env->n_running) {
                double elapsed = env->now - env->running[k].time_started;
                double remaining = (env->running[k].jct - elapsed) - env->eps;
                if (remaining <= 0) {
                    orc_job_record_t* r = &env->records[env->running[k].job_idx];
                    r->status = JS_COMPLETED; r->time_completed = env->now;
                    r->event_seq = env->event_seq++;
                    env->num_completed++; stats[SS_NUM_JOBS_COMPLETED] += 1;
                    remove_running(env, k);      /* keeps the order of the remaining rows */
                    step_done = 1;
                } else {
                    ++k;
                }
            }
        }

        /* RCE:1019-1040 */
        if ((env->n_jobs - env->num_arrived) > 0) {
            if (env->now + env->eps >= env->next_arrival) {
                int32_t idx = env->num_arrived;
                get_next_job(env);
                stats[SS_NUM_JOBS_ARRIVED] += 1;
                if (env->queued_job < 0 && env->queue_capacity >= 1) env->queued_job = idx;  /* RCE:1030-1031 */
                else register_blocked(env, idx);                                             /* RCE:1034 */
                step_done = 1;
            }
        } else {
            env->next_arrival = INFINITY;                                      /* RCE:1040 */
        }
        if (is_done(env)) step_done = 1;                                       /* RCE:1043 */
    }

    /* RCE:1046-1084 */
    stats[SS_STEP_END_TIME] = env->now;
    stats[SS_STEP_TIME] = stats[SS_STEP_END_TIME] - stats[SS_STEP_START_TIME];
    stats[SS_MEAN_NUM_JOBS_RUNNING] = sum_jobs_running / (double)n_iter;
    stats[SS_MEAN_NUM_MOUNTED_WORKERS] = sum_workers / (double)n_iter;
    stats[SS_MEAN_NUM_MOUNTED_CHANNELS] = sum_channels / (double)n_iter;
    stats[SS_MEAN_COMPUTE_OVERHEAD_FRAC] = n_frac > 0 ? sum_comp_frac / (double)n_frac : 0.0;
    stats[SS_MEAN_COMMUNICATION_OVERHEAD_FRAC] = n_frac > 0 ? sum_comm_frac / (double)n_frac : 0.0;
    {
        static const int pairs[7][2] = {
            {SS_MEAN_COMPUTE_THROUGHPUT, SS_COMPUTE_INFO_PROCESSED}, {SS_MEAN_DEP_THROUGHPUT, SS_DEP_INFO_PROCESSED},
            {SS_MEAN_FLOW_THROUGHPUT, SS_FLOW_INFO_PROCESSED}, {SS_MEAN_CLUSTER_THROUGHPUT, SS_CLUSTER_INFO_PROCESSED},
            {SS_MEAN_DEMAND_COMPUTE_THROUGHPUT, SS_DEMAND_COMPUTE_INFO_PROCESSED},
            {SS_MEAN_DEMAND_DEP_THROUGHPUT, SS_DEMAND_DEP_INFO_PROCESSED},
            {SS_MEAN_DEMAND_TOTAL_THROUGHPUT, SS_DEMAND_TOTAL_INFO_PROCESSED}};
        for (int p = 0; p < 7; ++p) {                                          /* RCE:1064-1077 */
            double info = stats[pairs[p][1]];
            stats[pairs[p][0]] = (info != 0 && stats[SS_STEP_TIME] != 0) ? info / stats[SS_STEP_TIME] : 0.0;
        }
    }
    stats[SS_UTIL_MOUNTED_SUM] = util_mounted_sum;
    stats[SS_UTIL_CLUSTER_SUM] = util_cluster_sum;
    stats[SS_NUM_TICKS] = (double)n_iter;
    stats[SS_JOB_QUEUE_LENGTH] = env->queued_job >= 0 ? 1.0 : 0.0;            /* RCE:1082 */

    env->step_counter++;                                                        /* RCE:1109 */

    if (is_done(env)) {                                                         /* RCE:1111-1121 */
        while (env->n_running > 0) {
            /* blocked in running-table order; stats of this step are not re-logged (already appended RCE:1084)
             * but the reference does bump step_stats['num_jobs_blocked'] after logging, so do we. */
            register_blocked(env, env->running[0].job_idx);
            remove_running(env, 0);
        }
    }
    stats[SS_DONE] = is_done(env) ? 1.0 : 0.0;
    env->stats = NULL;
    return ORC_OK;
}

int32_t orc_env_queued_job(const orc_env_t* env) { return env->queued_job; }
int32_t orc_env_num_jobs_arrived(const orc_env_t* env) { return env->num_arrived; }
double orc_env_time(const orc_env_t* env) { return env->now; }
/* the last step's per-tick utilisation lists (RCE:989-994); returns their length, copies at most cap entries of each */
int32_t orc_env_tick_lists(const orc_env_t* env, double* mounted_out, double* cluster_out, int32_t cap) {
    for (int32_t k = 0; k < env->n_tick_util && k < cap; ++k) { mounted_out[k] = env->tick_util_mounted[k]; cluster_out[k] = env->tick_util_cluster[k]; }
    return env->n_tick_util;
}
double orc_env_mean_load_rate(const orc_env_t* env) { return env->load_rate_n > 0 ? env->load_rate_sum / (double)env->load_rate_n : 0.0; }
const orc_job_record_t* orc_env_job_records(const orc_env_t* env) { return env->records; }
void orc_env_episode_state(const orc_env_t* env, double* out) {
    out[ORC_EP_TIME] = env->now; out[ORC_EP_NEXT_ARRIVAL] = env->next_arrival;
    out[ORC_EP_NUM_ARRIVED] = env->num_arrived; out[ORC_EP_NUM_COMPLETED] = env->num_completed;
    out[ORC_EP_NUM_BLOCKED] = env->num_blocked; out[ORC_EP_QUEUED_JOB] = env->queued_job;
    out[ORC_EP_NUM_RUNNING] = env->n_running; out[ORC_EP_STEP_COUNTER] = env->step_counter;
    out[ORC_EP_LOAD_RATE_SUM] = env->load_rate_sum; out[ORC_EP_LOAD_RATE_N] = env->load_rate_n;
    out[ORC_EP_DONE] = is_done(env) ? 1.0 : 0.0; out[ORC_EP_STATUS] = ORC_OK;
}
int32_t orc_env_last_trace(const orc_env_t* env, const int32_t** n_active, const double** tick) {
    if (!env->last_memo) return 0;
    *n_active = env->last_memo->trace_n; *tick = env->last_memo->trace_tick;
    return env->last_memo->res.n_ticks;
}
