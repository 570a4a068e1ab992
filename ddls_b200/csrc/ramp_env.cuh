// ramp_env.cuh -- device-resident rollouts: the decision and bookkeeping either side of the batched cluster step
// (include/ramp_b200.h: ramp_env_*).  One thread per episode; everything an episode needs is a few words.
//
//   ramp_env_decide_kernel  RJPE:300-343 + RampFirstFitOpPlacer (agents/placers/utils.py:394-443, 532-582) for jobs whose ops all
//                           take `degree` sub-ops: the first candidate block (host-enumerated in the reference's shape / origin
//                           order) with no busy server; template by (model, degree, geometry); action row for the engine
//   ramp_env_update_kernel  after the cluster step: reward (rewards/job_acceptance.py), servers of the accepted job, occupancy =
//                           OR over the running jobs, and the next queued job's dynamic graph features + action mask
//                           (observations/ramp_job_partitioning_observation.py:80-131, 358-498); the template id of the
//                           accepted job and the episode's return (EvalLoop's episode_stats['return'], loops/eval_loop.py:26-134)
//   ramp_env_agent_kernel   the reference's six heuristic agents (ddls/environments/ramp_job_partitioning/agents/*.py), one per
//                           episode, writing `actions`
#pragma once

namespace ramp {

struct EnvDev {
    int32_t B, J, n_words, n_models, max_degree, n_geoms, n_workers, apply_mask;
    double fail_reward, success_reward, num_training_steps, machine_epsilon;
    // tables
    const int32_t* cand_ptr; const unsigned long long* cand_mask; const int32_t* cand_geom;
    const uint8_t* uniform; const uint8_t* shape_ok;
    const double* model_params;     // [M][5]
    const double* jobs_params;      // [8][2]
    int32_t* tmpl_of;               // [M][D + 1][G]
    double* tmpl_mount;             // [max_templates][6]: seq_time, part_op_mem, part_dep, flow, n_workers, n_channels
    // per-episode streams
    const int32_t* model_of; const double* frac; const double* macc;   // [B][J]
    // state
    unsigned long long* busy;       // [B][n_words]
    unsigned long long* job_mask;   // [B][J][n_words]
    unsigned long long* placed;     // [B][n_words] block chosen this step
    int32_t* tid;                   // [B]
    int32_t* decided_job;           // [B] job idx the decision was for
    int32_t* n_decided;             // [B] decisions taken since the reset (env-steps of the episode)
    int32_t* job_tmpl;              // [B][J] template the job was mounted with when it was accepted (-1 otherwise)
    double* ret;                    // [B] sum of the rewards since the reset
    int32_t* agent_kind;            // [B] RAMP_AGENT_* (ramp_env_set_agents)
    int32_t* agent_param;           // [B] SiPML's max_partitions_per_op (<= 0: None)
    // i/o
    int32_t* actions; double* reward; uint8_t* done; int32_t* queued_model; float* obs_dyn; uint8_t* action_mask;
    int32_t* need_host; int32_t* n_need_host;
    int32_t* err;                   // first episode with an invalid action (+1)
    // EvalLoop's results['step_stats'] (ramp_env_steplog_begin; null / 0 when not recording)
    double* log_stats;              // [log_horizon][RAMP_ENV_STEP_STATS_LEN][B]
    int32_t* log_actions;           // [log_horizon][B]
    double* log_rewards;            // [log_horizon][B]
    int32_t log_horizon;
};

__device__ __forceinline__ int env_free_workers(const EnvDev& v, int b) {
    int busy = 0;
    for (int w = 0; w < v.n_words; ++w) busy += __popcll(v.busy[(size_t)b * v.n_words + w]);
    return v.n_workers - busy;
}

__device__ __forceinline__ bool env_action_valid(const EnvDev& v, int b, int a, int free_workers) {
    if (a == 0) return true;                                                     // observation.py:80-131
    if (a < 0 || a > v.max_degree) return false;
    if (!(a == 1 || (a % 2 == 0))) return false;
    return a <= free_workers && v.shape_ok[a] != 0;
}

__global__ void ramp_env_decide_kernel(const EnvDev v, const EpisodeState ep, ramp_action_t* rows) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    const int B = v.B;
    if (b >= B) return;
    ramp_action_t row;
    row.max_acceptable_jct = 0.0; row.part_op_mem = 0.0; row.part_dep_size = 0.0; row.flow_size = 0.0;
    row.n_mounted_workers = 0; row.n_mounted_channels = 0; row.template_id = -1; row.flags = 0;
    v.tid[b] = -1;
    for (int w = 0; w < v.n_words; ++w) v.placed[(size_t)b * v.n_words + w] = 0ull;
    const int q = ep.ei[EI_QUEUED * B + b];
    v.decided_job[b] = q;
    if (ep.ei[EI_DONE * B + b]) { row.flags = RAMP_ACT_SKIP; rows[b] = row; return; }
    int a = v.actions[b];
    v.n_decided[b] += 1;
    if (q < 0) { rows[b] = row; return; }                                        // cannot happen after ramp_env_advance (RJPE:394-395)
    const int free_workers = env_free_workers(v, b);
    if (!env_action_valid(v, b, a, free_workers)) {
        if (v.apply_mask) { atomicCAS(v.err, 0, b + 1); rows[b] = row; return; } // RJPE:314-319 raises
        a = 0;                                                                    // RJPE:320-322
    }
    if (a == 0) { rows[b] = row; return; }
    const int m = v.model_of[(size_t)b * v.J + q];
    if (!v.uniform[m * (v.max_degree + 1) + a]) {                                 // mixed split counts: the host's full placer decides
        v.need_host[atomicAdd(v.n_need_host, 1)] = b;
        rows[b] = row;
        return;
    }
    // first-fit over the candidate blocks of this degree (utils.py:394-443): first block without a busy server
    int geom = -1;
    const unsigned long long* busy = v.busy + (size_t)b * v.n_words;
    for (int c = v.cand_ptr[a]; c < v.cand_ptr[a + 1]; ++c) {
        const unsigned long long* cm = v.cand_mask + (size_t)c * v.n_words;
        bool ok = true;
        for (int w = 0; w < v.n_words; ++w) ok = ok && ((busy[w] & cm[w]) == 0ull);
        if (ok) {
            geom = v.cand_geom[c];
            for (int w = 0; w < v.n_words; ++w) v.placed[(size_t)b * v.n_words + w] = cm[w];
            break;
        }
    }
    if (geom < 0) { rows[b] = row; return; }                                      // no block: the job is left out of the Action and blocked (RCE:914-919)
    const int t = v.tmpl_of[((size_t)m * (v.max_degree + 1) + a) * v.n_geoms + geom];
    if (t < 0) {                                                                  // lowered job of this geometry not registered yet
        v.need_host[atomicAdd(v.n_need_host, 1)] = b;
        for (int w = 0; w < v.n_words; ++w) v.placed[(size_t)b * v.n_words + w] = 0ull;
        rows[b] = row;
        return;
    }
    const double* mt = v.tmpl_mount + (size_t)t * 6;
    const double ov = v.macc[(size_t)b * v.J + q];
    row.max_acceptable_jct = isnan(ov) ? __dmul_rn(v.frac[(size_t)b * v.J + q], mt[0]) : ov;
    row.part_op_mem = mt[1]; row.part_dep_size = mt[2]; row.flow_size = mt[3];
    row.n_mounted_workers = (int32_t)mt[4]; row.n_mounted_channels = (int32_t)mt[5];
    row.template_id = t;
    v.tid[b] = t;
    rows[b] = row;
}

// a graph feature as the reference stores it: a negative value gets machine_epsilon added (observation.py:441-444, 493-496), in
// double, before the float32 observation
__device__ __forceinline__ float env_feature(double x, double eps) {
    return (float)(x < 0.0 ? x + eps : x);
}

__device__ __forceinline__ float env_norm(double x, const double* jp, int k, double eps) {
    const double lo = jp[2 * k], hi = jp[2 * k + 1];
    return env_feature((hi - lo != 0.0) ? (x - lo) / (hi - lo) : 1.0, eps);     // observation.py _norm
}

__global__ void ramp_env_update_kernel(const EnvDev v, const EpisodeState ep, const int32_t* n_cluster_steps, int first) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    const int B = v.B, J = v.J, nw = v.n_words;
    if (b >= B) return;
    const ramp_job_record_t* rec = ep.rec + (size_t)b * ep.max_jobs;
    if (!first) {
        // ---- reward: the job counts as placed unless it was blocked by the end of the FIRST cluster step (RJPE:379-391); a
        //      lookahead-blocked job has no lookahead results in its record ----
        const int q = v.decided_job[b];
        const bool was_live = !v.done[b];
        bool accepted = false;
        if (was_live && q >= 0 && v.tid[b] >= 0) {
            accepted = rec[q].jct != 0.0;
            const bool blocked_in_action_step = accepted && rec[q].status == RAMP_JS_BLOCKED && n_cluster_steps[b] == 1;
            v.reward[b] = (accepted && !blocked_in_action_step) ? v.success_reward : v.fail_reward;
        } else {
            v.reward[b] = was_live ? v.fail_reward : 0.0;
        }
        v.ret[b] = __dadd_rn(v.ret[b], v.reward[b]);
        // eval_loop.py:44-100: env-step n_decided - 1 of a live episode -- its action, reward and the row the step kernel closed
        const int row = v.n_decided[b] - 1;
        if (was_live && row >= 0 && row < v.log_horizon) {
            const size_t r = (size_t)row * B + b;
            v.log_actions[r] = v.actions[b];
            v.log_rewards[r] = v.reward[b];
            for (int k = 0; k < RAMP_ENV_STEP_STATS_LEN; ++k)
                v.log_stats[((size_t)row * RAMP_ENV_STEP_STATS_LEN + k) * B + b] = ep.es[(size_t)b * ES_STRIDE + k];
        }
        if (accepted) {
            for (int w = 0; w < nw; ++w) v.job_mask[((size_t)b * J + q) * nw + w] = v.placed[(size_t)b * nw + w];
            v.job_tmpl[(size_t)b * J + q] = v.tid[b];
        }
    }
    // ---- occupancy: servers of the jobs that are running now (one job per worker, ramp_rules.py:6-39) ----
    int n_running = 0;
    for (int w = 0; w < nw; ++w) v.busy[(size_t)b * nw + w] = 0ull;
    const int n_arr = ep.ei[EI_NUM_ARRIVED * B + b];
    for (int j = 0; j < n_arr && j < J; ++j) {
        if (rec[j].status == RAMP_JS_RUNNING) {
            ++n_running;
            for (int w = 0; w < nw; ++w) v.busy[(size_t)b * nw + w] |= v.job_mask[((size_t)b * J + j) * nw + w];
        }
    }
    // ---- the next decision's observation: dynamic graph features + action mask ----
    const int dn = ep.ei[EI_DONE * B + b];
    v.done[b] = (uint8_t)(dn != 0);
    const int q2 = ep.ei[EI_QUEUED * B + b];
    const int free_workers = env_free_workers(v, b);
    uint8_t* am = v.action_mask + (size_t)b * (v.max_degree + 1);
    for (int a = 0; a <= v.max_degree; ++a) am[a] = env_action_valid(v, b, a, free_workers) ? 1 : 0;
    float* o = v.obs_dyn + (size_t)b * 11;
    if (q2 >= 0 && q2 < J) {
        const int m = v.model_of[(size_t)b * J + q2];
        v.queued_model[b] = m;
        const double* mp = v.model_params + (size_t)m * 5;
        const double fr = v.frac[(size_t)b * J + q2];
        const double* jp = v.jobs_params;
        const double eps = v.machine_epsilon;
        o[0] = env_norm(mp[1], jp, 0, eps); o[1] = env_norm(mp[2], jp, 1, eps); o[2] = env_norm(mp[0], jp, 2, eps);
        o[3] = env_norm(__dmul_rn(fr, mp[0]), jp, 3, eps); o[4] = env_norm(fr, jp, 4, eps); o[5] = env_feature(fr, eps);
        o[6] = env_norm(mp[3], jp, 5, eps); o[7] = env_norm(mp[4], jp, 6, eps); o[8] = env_norm(v.num_training_steps, jp, 7, eps);
    } else {
        v.queued_model[b] = -1;
        for (int k = 0; k < 9; ++k) o[k] = 0.f;
    }
    o[9] = env_feature((double)(v.n_workers - free_workers) / (double)v.n_workers, v.machine_epsilon);
    o[10] = env_feature((double)n_running / (double)v.n_workers, v.machine_epsilon);
}

// The reference's heuristic agents (ddls/environments/ramp_job_partitioning/agents/*.py), restated line for line on the action
// mask ramp_env_update_kernel left: valid_actions = action_set[action_mask] in ascending order.  With one valid action
// MinParallelism and NoParallelism return 0, the others valid_actions[0].  Otherwise:
//   Random          np.random.choice(valid_actions[1:]) (random.py:8-16): uniform over the valid actions after the first,
//                   drawn from splitmix64 keyed by (seed, episode, decisions taken so far) -- the policy's construction
//                   (ramp_policy.cu); it does not reproduce numpy's stream
//   SiPML           min(param, valid_actions[-1]), param <= 0 = None: valid_actions[-1] (sip_ml.py:13-25); not re-checked
//                   against the mask
//   AcceptableJCT   target = ceil(seq / max_acceptable_jct) in f64; the first valid action >= target, 0 included, else
//                   valid_actions[-1] (acceptable_jct.py:21-44)
//   MaxParallelism  valid_actions[1:][-1] (max_parallelism.py:5-13)
//   MinParallelism  2 when more than two actions are valid, even if 2 is masked; 1 when two are (min_parallelism.py:5-17)
//   NoParallelism   1 (no_parallelism.py:5-13)
// Finished episodes get 0.
__global__ void ramp_env_agent_kernel(const EnvDev v, const EpisodeState ep, unsigned long long seed) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= v.B) return;
    if (v.done[b]) { v.actions[b] = 0; return; }
    const uint8_t* am = v.action_mask + (size_t)b * (v.max_degree + 1);
    int n_valid = 0, first = 0, last = 0;
    for (int a = 0; a <= v.max_degree; ++a) {
        if (am[a]) { if (n_valid == 0) first = a; last = a; ++n_valid; }
    }
    const int kind = v.agent_kind[b];
    int action = first;
    if (kind == RAMP_AGENT_MIN_PARALLELISM) {
        action = n_valid > 2 ? 2 : n_valid == 2 ? 1 : 0;
    } else if (kind == RAMP_AGENT_NO_PARALLELISM) {
        action = n_valid > 1 ? 1 : 0;
    } else if (n_valid > 1) {
        switch (kind) {
            case RAMP_AGENT_RANDOM: {
                const unsigned long long key = seed ^ (0x9E3779B97F4A7C15ull * (unsigned long long)v.n_decided[b]);
                const unsigned long long r = splitmix64(key ^ ((unsigned long long)b * 0xD1342543DE82EF95ull));
                const int k = (int)(((r >> 32) * (unsigned long long)(n_valid - 1)) >> 32);   // valid_actions[1 + k]
                int seen = -1;
                for (int a = 0; a <= v.max_degree; ++a) {
                    if (am[a] && seen++ == k) { action = a; break; }
                }
                break;
            }
            case RAMP_AGENT_SIPML: {
                const int p = v.agent_param[b];
                action = (p > 0 && p < last) ? p : last;
                break;
            }
            case RAMP_AGENT_ACCEPTABLE_JCT: {
                const int q = ep.ei[EI_QUEUED * v.B + b];
                const int m = v.queued_model[b];
                const double seq = v.model_params[(size_t)m * 5];
                const double ov = v.macc[(size_t)b * v.J + q];
                const double macc = isnan(ov) ? __dmul_rn(v.frac[(size_t)b * v.J + q], seq) : ov;
                const double target = ceil(__ddiv_rn(seq, macc));
                action = last;
                for (int a = 0; a <= v.max_degree; ++a) {
                    if (am[a] && (double)a >= target) { action = a; break; }
                }
                break;
            }
            case RAMP_AGENT_MAX_PARALLELISM: action = last; break;
            default: action = 0; break;
        }
    }
    v.actions[b] = action;
}

}  // namespace ramp
