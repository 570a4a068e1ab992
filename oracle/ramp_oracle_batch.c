/*
 * TEST INFRASTRUCTURE -- multi-threaded driver around the CPU oracle, used as the
 * reported CPU baseline (bench.py cpu_baseline / --impl reference).  Episodes are
 * independent, so they are spread over host threads with OpenMP.
 */
#include "ramp_oracle.h"
#include <stdlib.h>
#include <string.h>
#include <pthread.h>
#include <stdatomic.h>

/* minimal dynamic-scheduling parallel-for over pthreads (this image's gcc has no libgomp) */
typedef void (*orc_body_fn)(int32_t k, void* ctx);
typedef struct { atomic_int next; int32_t n; orc_body_fn body; void* ctx; } orc_pf_t;
static void* orc_pf_worker(void* arg) {
    orc_pf_t* pf = (orc_pf_t*)arg;
    for (;;) {
        int32_t k = atomic_fetch_add(&pf->next, 1);
        if (k >= pf->n) break;
        pf->body(k, pf->ctx);
    }
    return NULL;
}
static void orc_parallel_for(int32_t n, int32_t n_threads, orc_body_fn body, void* ctx) {
    orc_pf_t pf; atomic_init(&pf.next, 0); pf.n = n; pf.body = body; pf.ctx = ctx;
    if (n_threads < 1) n_threads = 1;
    if (n_threads > n) n_threads = n > 0 ? n : 1;
    if (n_threads > 256) n_threads = 256;
    pthread_t th[256];
    for (int32_t t = 1; t < n_threads; ++t) pthread_create(&th[t], NULL, orc_pf_worker, &pf);
    orc_pf_worker(&pf);
    for (int32_t t = 1; t < n_threads; ++t) pthread_join(th[t], NULL);
}

/* Runs n independent lookaheads (RCE:379-467).  jobs[k] may repeat the same template. */
typedef struct { const orc_lowered_job_t* const* jobs; orc_lookahead_result_t* results; atomic_int bad; } orc_lb_t;
static void orc_lb_body(int32_t k, void* c) {
    orc_lb_t* x = (orc_lb_t*)c;
    if (orc_run_lookahead(x->jobs[k], NULL, NULL, 0, &x->results[k]) != ORC_OK) atomic_store(&x->bad, 1);
}
int orc_run_lookahead_batch(const orc_lowered_job_t* const* jobs, int32_t n,
                            orc_lookahead_result_t* results, int32_t n_threads) {
    orc_lb_t x; x.jobs = jobs; x.results = results; atomic_init(&x.bad, 0);
    orc_parallel_for(n, n_threads, orc_lb_body, &x);
    return atomic_load(&x.bad) ? ORC_ERR_BAD_ARG : ORC_OK;
}

/* Scripted batched episodes: episode b performs n_steps RampClusterEnvironment.step calls;
 * step s of episode b uses template script_tid[b*n_steps+s] (or -1 = Action()) with mount
 * scalars script_mount[b*n_steps+s].  stats_out: [n_episodes][n_steps][ORC_STEP_STATS_LEN]
 * (may be NULL).  Each episode has its own env (own memo), like independent reference envs. */
typedef struct {
    const orc_lowered_job_t* templates; int32_t n_templates, n_steps, n_jobs, n_cluster_workers, memo_models, memo_degrees;
    const int32_t* script_tid; const orc_mount_t* script_mount; const orc_arrival_t* arrivals;
    double max_sim_time; double* stats_out; orc_job_record_t* records_out; atomic_int bad; int rjpe;
    /* orc_run_scripted_rjpe_full_batch only (NULL / 0 otherwise): see ramp_oracle.h */
    int skip_done; int32_t* ncs_out; double* cs_stats_out; int32_t cs_cap; int32_t* cs_total_out; double* ep_out;
    atomic_int overflow;
} orc_sb_t;
/* one cluster step: orc_env_step, its row appended to the episode's cs_stats_out rows */
static int orc_sb_cluster_step(orc_sb_t* x, int32_t b, orc_env_t* env, int32_t tid, size_t idx, double* st, int32_t* n_cs) {
    int rc = tid >= 0 ? orc_env_step(env, &x->templates[tid], &x->script_mount[idx], st) : orc_env_step(env, NULL, NULL, st);
    if (rc != ORC_OK) return rc;
    if (x->cs_stats_out) {
        if (*n_cs >= x->cs_cap) { atomic_store(&x->overflow, 1); return ORC_ERR_TRACE_OVERFLOW; }
        memcpy(x->cs_stats_out + ((size_t)b * (size_t)x->cs_cap + (size_t)*n_cs) * ORC_STEP_STATS_LEN, st,
               sizeof(double) * ORC_STEP_STATS_LEN);
    }
    ++*n_cs;
    return ORC_OK;
}
static void orc_sb_body(int32_t b, void* c) {
    orc_sb_t* x = (orc_sb_t*)c;
    orc_env_t* env = orc_env_create(x->n_cluster_workers, x->n_cluster_workers > 0 ? x->n_cluster_workers : 1, x->n_jobs,
                                    x->memo_models, x->memo_degrees, 0, 1e-7);
    double local[ORC_STEP_STATS_LEN];
    int bad = 0, done = 0;
    int32_t n_cs = 0;
    if (orc_env_reset(env, x->max_sim_time, 10, x->arrivals + (size_t)b * (size_t)x->n_jobs, x->n_jobs) != ORC_OK) bad = 1;
    double scratch[ORC_STEP_STATS_LEN];
    for (int32_t s = 0; s < x->n_steps && !bad; ++s) {
        size_t idx = (size_t)b * (size_t)x->n_steps + (size_t)s;
        int32_t tid = x->script_tid[idx];
        double* st = x->stats_out ? x->stats_out + idx * ORC_STEP_STATS_LEN : local;
        const int32_t n_cs0 = n_cs;
        if (x->skip_done && done) {   /* a finished episode is left as it is (RAMP_ACT_SKIP / a done episode on the device) */
            memset(st, 0, sizeof(double) * ORC_STEP_STATS_LEN);
            double ep[ORC_EP_LEN];
            orc_env_episode_state(env, ep);
            st[SS_STEP_COUNTER] = ep[ORC_EP_STEP_COUNTER];
            st[SS_JOB_QUEUE_LENGTH] = orc_env_queued_job(env) >= 0 ? 1.0 : 0.0;
            st[SS_DONE] = 1.0;
            if (x->ncs_out) x->ncs_out[idx] = 0;
            continue;
        }
        if (!(tid >= 0 && tid < x->n_templates && orc_env_queued_job(env) >= 0)) tid = -1;
        if (orc_sb_cluster_step(x, b, env, tid, idx, st, &n_cs) != ORC_OK) bad = 1;
        if (x->rjpe) {   /* RJPE:394-395: while len(job_queue) == 0 and not done: step(Action()) */
            const double* last = st;
            while (!bad && orc_env_queued_job(env) < 0 && last[SS_DONE] == 0.0) {
                if (orc_sb_cluster_step(x, b, env, -1, idx, scratch, &n_cs) != ORC_OK) bad = 1;
                last = scratch;
            }
            st[SS_DONE] = last[SS_DONE];
        }
        done = st[SS_DONE] != 0.0;
        if (x->ncs_out) x->ncs_out[idx] = n_cs - n_cs0;
    }
    if (x->records_out)
        memcpy(x->records_out + (size_t)b * (size_t)x->n_jobs, orc_env_job_records(env), sizeof(orc_job_record_t) * (size_t)x->n_jobs);
    if (x->cs_total_out) x->cs_total_out[b] = n_cs;
    if (x->ep_out) orc_env_episode_state(env, x->ep_out + (size_t)b * ORC_EP_LEN);
    orc_env_destroy(env);
    if (bad) atomic_store(&x->bad, 1);
}
static void orc_sb_init(orc_sb_t* x) {
    memset(x, 0, sizeof(*x));
    atomic_init(&x->bad, 0); atomic_init(&x->overflow, 0);
}
int orc_run_scripted_batch(const orc_lowered_job_t* templates, int32_t n_templates,
                           int32_t n_episodes, int32_t n_steps,
                           const int32_t* script_tid, const orc_mount_t* script_mount,
                           const orc_arrival_t* arrivals /* [n_episodes][n_jobs] */, int32_t n_jobs,
                           double max_sim_time, int32_t n_cluster_workers, int32_t memo_models, int32_t memo_degrees,
                           double* stats_out, orc_job_record_t* records_out /* [n_episodes][n_jobs] or NULL */,
                           int32_t n_threads) {
    orc_sb_t x;
    orc_sb_init(&x);
    x.templates = templates; x.n_templates = n_templates; x.n_steps = n_steps; x.n_jobs = n_jobs;
    x.n_cluster_workers = n_cluster_workers; x.memo_models = memo_models; x.memo_degrees = memo_degrees;
    x.script_tid = script_tid; x.script_mount = script_mount; x.arrivals = arrivals; x.max_sim_time = max_sim_time;
    x.stats_out = stats_out; x.records_out = records_out; x.rjpe = 0;
    orc_parallel_for(n_episodes, n_threads, orc_sb_body, &x);
    return atomic_load(&x.bad) ? ORC_ERR_BAD_ARG : ORC_OK;
}

/* Same, but each scripted decision is one RampJobPartitioningEnvironment.step (RJPE:300-420): the action step
 * followed by Action() steps until a job is queued or the episode is done.  stats_out rows describe the action
 * step (with SS_DONE = done after the whole env-step). */
int orc_run_scripted_rjpe_batch(const orc_lowered_job_t* templates, int32_t n_templates,
                                int32_t n_episodes, int32_t n_steps,
                                const int32_t* script_tid, const orc_mount_t* script_mount,
                                const orc_arrival_t* arrivals, int32_t n_jobs,
                                double max_sim_time, int32_t n_cluster_workers, int32_t memo_models, int32_t memo_degrees,
                                double* stats_out, orc_job_record_t* records_out, int32_t n_threads) {
    orc_sb_t x;
    orc_sb_init(&x);
    x.templates = templates; x.n_templates = n_templates; x.n_steps = n_steps; x.n_jobs = n_jobs;
    x.n_cluster_workers = n_cluster_workers; x.memo_models = memo_models; x.memo_degrees = memo_degrees;
    x.script_tid = script_tid; x.script_mount = script_mount; x.arrivals = arrivals; x.max_sim_time = max_sim_time;
    x.stats_out = stats_out; x.records_out = records_out; x.rjpe = 1;
    orc_parallel_for(n_episodes, n_threads, orc_sb_body, &x);
    return atomic_load(&x.bad) ? ORC_ERR_BAD_ARG : ORC_OK;
}

/* The same env-steps, with every output the product's step path has (ramp_oracle.h); done episodes are not stepped again. */
int orc_run_scripted_rjpe_full_batch(const orc_lowered_job_t* templates, int32_t n_templates, int32_t n_episodes, int32_t n_steps,
                                     const int32_t* script_tid, const orc_mount_t* script_mount, const orc_arrival_t* arrivals,
                                     int32_t n_jobs, double max_sim_time, int32_t n_cluster_workers, int32_t memo_models,
                                     int32_t memo_degrees, double* stats_out, int32_t* ncs_out, double* cs_stats_out, int32_t cs_cap,
                                     int32_t* cs_total_out, orc_job_record_t* records_out, double* ep_out, int32_t n_threads) {
    orc_sb_t x;
    orc_sb_init(&x);
    x.templates = templates; x.n_templates = n_templates; x.n_steps = n_steps; x.n_jobs = n_jobs;
    x.n_cluster_workers = n_cluster_workers; x.memo_models = memo_models; x.memo_degrees = memo_degrees;
    x.script_tid = script_tid; x.script_mount = script_mount; x.arrivals = arrivals; x.max_sim_time = max_sim_time;
    x.stats_out = stats_out; x.records_out = records_out; x.rjpe = 1;
    x.skip_done = 1; x.ncs_out = ncs_out; x.cs_stats_out = cs_stats_out; x.cs_cap = cs_cap; x.cs_total_out = cs_total_out;
    x.ep_out = ep_out;
    orc_parallel_for(n_episodes, n_threads, orc_sb_body, &x);
    if (atomic_load(&x.overflow)) return ORC_ERR_TRACE_OVERFLOW;
    return atomic_load(&x.bad) ? ORC_ERR_BAD_ARG : ORC_OK;
}
