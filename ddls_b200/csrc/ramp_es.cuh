// ramp_es.cuh -- RLlib's evolution strategies training step on the device (include/ramp_b200.h: ramp_es_*; ray/rllib/algorithms/es:
// es.py training_step, utils.py, optimizers.py).  Included at the end of ramp_policy.cu: the population runs the policy's forward
// bodies (gnn_embed_body, head_row) with a weight set per episode.
//
//   ramp_es_perturb_kernel   the population's weight sets: set 2i = fl(theta + fl(sigma eps_i)), set 2i+1 = fl(theta - fl(sigma
//                            eps_i)), set 2N = theta
//   ramp_es_embed_kernel     gnn_embed_body for every (set, job type): persistent CTAs, each with its own scratch, so the scratch
//                            scales with the grid, not with the population
//   ramp_es_head_kernel      head_row with sample = 1, one warp per episode, reading its set's read-out weights from global memory
//                            (no value: ES does not use it)
//   ramp_es_collect_kernel   each episode's return (float of the f64 sum) and env-step count
//   ramp_es_rank_kernel      compute_centered_ranks, one thread per value; ties go to index order (a stable argsort)
//   ramp_es_update_kernel    g = sum_i (rank+_i - rank-_i) eps_i / 2N per weight (f64 in pair order), optimizers.Adam on
//                            -g + l2 theta in float32 (_rn intrinsics), per-CTA norm partials
//   ramp_es_stats_kernel     the partials, summed in CTA order
#pragma once

int ramp_internal_env_returns(ramp_engine_t* e, const double** ret, const int32_t** n_decided);

namespace ramp {

constexpr int ES_GRID = 264;             // CTAs of the update kernel: its norm partials are summed in this fixed order
constexpr int ES_PAIR_CHUNK = 1024;      // pairs staged in shared memory at a time by the update kernel

__global__ void ramp_es_perturb_kernel(const float* theta, const float* noise, const int32_t* noise_index, int32_t n_pairs,
                                       int64_t n, float sigma, float* sets) {
    const int s = blockIdx.y;             // set: 2 n_pairs + 1 of them
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        float w = theta[k];
        if (s < 2 * n_pairs) {
            const float d = __fmul_rn(sigma, noise[(int64_t)noise_index[s >> 1] + k]);
            w = (s & 1) ? __fsub_rn(w, d) : __fadd_rn(w, d);
        }
        sets[(size_t)s * n + k] = w;
    }
}

struct EsEmbedArgs {
    int32_t n_sets, n_models;
    int64_t n_weights;
    const float* sets;                    // [n_sets][n_weights]
    float* scratch;                       // [gridDim.x][slot_floats]: z0, z1 [max_nodes][POL_MAX_DIM], hn [max_nodes][half], he [max_edges][half]
    int64_t slot_floats;
    int32_t max_nodes, max_edges;
    float* emb;                           // [n_sets][n_models][out_node]
};

__global__ void __launch_bounds__(256) ramp_es_embed_kernel(const PolicyDev P, const ModelDev* models, const EsEmbedArgs a) {
    const int half = P.c.out_features_msg / 2;
    float* z0 = a.scratch + (size_t)blockIdx.x * a.slot_floats;
    float* z1 = z0 + (size_t)a.max_nodes * POL_MAX_DIM;
    float* hn = z1 + (size_t)a.max_nodes * POL_MAX_DIM;
    float* he = hn + (size_t)a.max_nodes * half;
    for (int item = blockIdx.x; item < a.n_sets * a.n_models; item += gridDim.x) {
        const int s = item / a.n_models, m = item - s * a.n_models;
        ModelDev M = models[m];
        M.z0 = z0; M.z1 = z1; M.hn = hn; M.he = he;
        gnn_embed_body(P, a.sets + (size_t)s * a.n_weights, M, a.emb + (size_t)item * P.c.out_features_node);
        __syncthreads();                  // the next item reuses the scratch
    }
}

struct EsHeadArgs {
    int32_t n_pairs;                      // episode b < 2 n_pairs runs set b, the others set 2 n_pairs
    int64_t n_weights;
    const float* sets;                    // [sets][n_weights]; HeadArgs::emb is [sets][n_models][out_node]
};

// head_row on each episode with its set's weights read from global memory; the act has no value
__global__ void __launch_bounds__(256) ramp_es_head_kernel(const PolicyDev P, const HeadArgs a, const EsHeadArgs e) {
    __shared__ float s_warp[8][2 * POL_MAX_DIM];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpc = blockDim.x >> 5;
    for (int b = blockIdx.x * wpc + warp; b < a.n; b += gridDim.x * wpc) {
        const int s = b < 2 * e.n_pairs ? b : 2 * e.n_pairs;
        head_row(P.c, ReadoutBlob(P, e.sets + (size_t)s * e.n_weights), a, a.emb + (size_t)s * P.c.n_models * P.c.out_features_node, b,
                 s_warp[warp], lane);
    }
}

__global__ void ramp_es_collect_kernel(int32_t B, const double* ret, const int32_t* n_decided, float* returns, int32_t* lengths) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    returns[b] = (float)ret[b];          // RLlib's float32 sum of float32 rewards, for the environment's +-1 rewards
    lengths[b] = n_decided[b];
}

// rank of x_i = #{j : x_j < x_i or (x_j == x_i and j < i)}; rank / (n - 1) - 0.5 in float32
__global__ void ramp_es_rank_kernel(const float* x, int32_t n, float* ranks) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float xi = x[i];
    int r = 0;
    for (int j = 0; j < n; ++j) { const float xj = x[j]; r += (xj < xi || (xj == xi && j < i)) ? 1 : 0; }
    ranks[i] = __fsub_rn(__fdiv_rn((float)r, (float)(n - 1)), 0.5f);
}

struct EsUpdateArgs {
    int64_t n;                            // weights
    int32_t n_pairs;
    const int32_t* noise_index; const float* ranks; const float* noise;
    float* theta; float* m; float* v; float* g;
    float l2, beta1, one_m_beta1, beta2, one_m_beta2, eps, neg_a;
    double* part;                         // [ES_GRID][4]: sum step^2, theta_old^2, theta_new^2, g^2
};

__global__ void __launch_bounds__(256) ramp_es_update_kernel(const EsUpdateArgs a) {
    __shared__ float s_w[ES_PAIR_CHUNK];
    __shared__ int32_t s_idx[ES_PAIR_CHUNK];
    __shared__ double s_red[4][256];
    const double count = 2.0 * (double)a.n_pairs;
    double q[4] = {0.0, 0.0, 0.0, 0.0};
    // every thread of the grid runs the same number of chunk iterations, so the barriers below are uniform
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < a.n; base += stride) {
        const int64_t k = base + threadIdx.x;
        double acc = 0.0;
        for (int p0 = 0; p0 < a.n_pairs; p0 += ES_PAIR_CHUNK) {
            const int np = min(ES_PAIR_CHUNK, a.n_pairs - p0);
            __syncthreads();
            for (int i = threadIdx.x; i < np; i += blockDim.x) {
                s_w[i] = __fsub_rn(a.ranks[2 * (p0 + i)], a.ranks[2 * (p0 + i) + 1]);
                s_idx[i] = a.noise_index[p0 + i];
            }
            __syncthreads();
            if (k < a.n)
                for (int i = 0; i < np; ++i) acc += (double)s_w[i] * (double)a.noise[(int64_t)s_idx[i] + k];
        }
        if (k < a.n) {
            const float g = (float)(acc / count);
            const float th = a.theta[k];
            const float gg = __fadd_rn(-g, __fmul_rn(a.l2, th));                 // -g + l2_coeff * theta
            const float m = __fadd_rn(__fmul_rn(a.beta1, a.m[k]), __fmul_rn(a.one_m_beta1, gg));
            const float v = __fadd_rn(__fmul_rn(a.beta2, a.v[k]), __fmul_rn(a.one_m_beta2, __fmul_rn(gg, gg)));
            const float step = __fdiv_rn(__fmul_rn(a.neg_a, m), __fadd_rn(__fsqrt_rn(v), a.eps));
            const float nt = __fadd_rn(th, step);
            a.g[k] = g; a.m[k] = m; a.v[k] = v; a.theta[k] = nt;
            q[0] += (double)step * step; q[1] += (double)th * th; q[2] += (double)nt * nt; q[3] += (double)g * g;
        }
    }
    for (int j = 0; j < 4; ++j) s_red[j][threadIdx.x] = q[j];
    __syncthreads();
    for (int o = blockDim.x / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o)
            for (int j = 0; j < 4; ++j) s_red[j][threadIdx.x] += s_red[j][threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x < 4) a.part[(size_t)blockIdx.x * 4 + threadIdx.x] = s_red[threadIdx.x][0];
}

// out: weights_norm, grad_norm, update_ratio
__global__ void ramp_es_stats_kernel(const double* part, int32_t n_part, double* out) {
    double q[4] = {0.0, 0.0, 0.0, 0.0};
    for (int c = 0; c < n_part; ++c)
        for (int j = 0; j < 4; ++j) q[j] += part[(size_t)c * 4 + j];
    out[0] = q[2];
    out[1] = q[3];
    out[2] = q[1] > 0.0 ? sqrt(q[0]) / sqrt(q[1]) : 0.0;
}

}  // namespace ramp

struct ramp_es {
    ramp_policy* p = nullptr;
    int64_t n = 0, noise_size = 0;
    DeviceArray<float> noise, m, v, g, ranks, returns;
    DeviceArray<int32_t> idx;
    DeviceArray<double> part, dstats;
    int32_t t = 0;                        // Adam's step count
    int64_t iteration = 0;                // ramp_es_step calls: keys the noise indices and the draws
    std::vector<double> reward_list;      // each step's mean eval return
    // the population of the current round: sets, embeddings, per-CTA embedding scratch, the round's returns / env-steps and the
    // last act's outputs, for `cap` episodes
    int32_t cap = 0, B = 0, n_pairs = 0, n_eval = 0, round = -1, embed_grid = 0;
    DeviceArray<float> sets, emb, scratch, r_ret, logits, logp;
    DeviceArray<int32_t> r_len, r_idx;
    ramp_es_config_t cfg{};
    // the step record: pairs over all rounds, eval episodes, act seeds; its update's ranks and g
    std::vector<int32_t> h_idx, h_len, h_eval_len;
    std::vector<float> h_ret, h_eval_ret, h_ranks;
    std::vector<uint64_t> h_seeds;
    int32_t rounds = 0;
    int64_t timesteps = 0;
};

namespace {

uint64_t es_key(uint64_t seed, int64_t iteration, int32_t round, uint64_t x) {
    uint64_t k = mix64(seed);
    k = mix64(k ^ (uint64_t)iteration);
    k = mix64(k ^ (uint64_t)round);
    return mix64(k ^ x);
}

int check_es_config(const ramp_es_config_t* cfg) {
    if (!cfg) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (!(cfg->noise_stdev >= 0) || !(cfg->stepsize >= 0) || !(cfg->adam_eps > 0) || !(cfg->adam_beta1 >= 0 && cfg->adam_beta1 < 1) ||
        !(cfg->adam_beta2 >= 0 && cfg->adam_beta2 < 1))
        return set_error(RAMP_ERR_BAD_ARG, "es: noise_stdev and stepsize must be >= 0, adam_eps > 0, the betas in [0, 1)");
    if (cfg->episodes_per_batch < 0 || cfg->train_batch_size < 0 || cfg->n_eval < 0 || cfg->report_length < 1)
        return set_error(RAMP_ERR_BAD_ARG, "es: episodes_per_batch, train_batch_size and n_eval must be >= 0, report_length >= 1");
    return RAMP_OK;
}

// ranks, g and Adam on the pairs in es->idx / es->returns (device), on stream 0; writes es->dstats
int es_update(ramp_es* es, const ramp_es_config_t& cfg, int32_t n_pairs) {
    ramp_policy* p = es->p;
    const int32_t nv = 2 * n_pairs;
    ramp_es_rank_kernel<<<(nv + 255) / 256, 256>>>(es->returns.get(), nv, es->ranks.get());
    es->t += 1;
    const double a = cfg.stepsize * (std::sqrt(1.0 - std::pow(cfg.adam_beta2, es->t)) / (1.0 - std::pow(cfg.adam_beta1, es->t)));
    EsUpdateArgs u{};
    u.n = es->n; u.n_pairs = n_pairs; u.noise_index = es->idx.get(); u.ranks = es->ranks.get(); u.noise = es->noise.get();
    u.theta = p->d_w.get(); u.m = es->m.get(); u.v = es->v.get(); u.g = es->g.get();
    u.l2 = (float)cfg.l2_coeff; u.beta1 = (float)cfg.adam_beta1; u.one_m_beta1 = (float)(1.0 - cfg.adam_beta1);
    u.beta2 = (float)cfg.adam_beta2; u.one_m_beta2 = (float)(1.0 - cfg.adam_beta2); u.eps = (float)cfg.adam_eps; u.neg_a = (float)(-a);
    u.part = es->part.get();
    ramp_es_update_kernel<<<ES_GRID, 256>>>(u);
    ramp_es_stats_kernel<<<1, 1>>>(es->part.get(), ES_GRID, es->dstats.get());
    CUDA_TRY(cudaGetLastError());
    p->emb_valid = false;
    return RAMP_OK;
}

// the update's inputs for n_pairs pairs on the device
int es_upload(ramp_es* es, int32_t n_pairs, const int32_t* idx, const float* returns) {
    if ((size_t)n_pairs > es->idx.size()) CUDA_TRY(es->idx.alloc(n_pairs));
    if ((size_t)(2 * n_pairs) > es->returns.size()) CUDA_TRY(alloc_each(2 * (size_t)n_pairs, es->returns, es->ranks));
    CUDA_TRY(cudaMemcpy(es->idx.get(), idx, sizeof(int32_t) * n_pairs, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(es->returns.get(), returns, sizeof(float) * 2 * n_pairs, cudaMemcpyHostToDevice));
    return RAMP_OK;
}

// the statistics es_update leaves on the device, the ranks and the eval means into `out`
int es_finish(ramp_es* es, const ramp_es_config_t& cfg, int32_t n_pairs, double* out) {
    double d[3];
    CUDA_TRY(cudaStreamSynchronize(0));
    CUDA_TRY(cudaMemcpy(d, es->dstats.get(), sizeof(d), cudaMemcpyDeviceToHost));
    es->h_ranks.resize(2 * (size_t)n_pairs);
    CUDA_TRY(cudaMemcpy(es->h_ranks.data(), es->ranks.get(), sizeof(float) * 2 * n_pairs, cudaMemcpyDeviceToHost));
    const double nan = std::nan("");
    double ev = nan, el = nan;
    if (!es->h_eval_ret.empty()) {
        double s = 0.0, l = 0.0;
        for (size_t i = 0; i < es->h_eval_ret.size(); ++i) { s += es->h_eval_ret[i]; l += es->h_eval_len[i]; }
        ev = s / (double)es->h_eval_ret.size();
        el = l / (double)es->h_eval_len.size();
        es->reward_list.push_back(ev);
    }
    double rm = nan;
    if (!es->reward_list.empty()) {
        const size_t k = std::min(es->reward_list.size(), (size_t)cfg.report_length);
        rm = 0.0;
        for (size_t i = es->reward_list.size() - k; i < es->reward_list.size(); ++i) rm += es->reward_list[i];
        rm /= (double)k;
    }
    if (out) {
        out[RAMP_ES_EPISODE_REWARD_MEAN] = rm; out[RAMP_ES_EPISODE_LEN_MEAN] = el; out[RAMP_ES_TIMESTEPS_THIS_ITER] = (double)es->timesteps;
        out[RAMP_ES_EPISODES_THIS_ITER] = 2.0 * n_pairs; out[RAMP_ES_WEIGHTS_NORM] = d[0]; out[RAMP_ES_GRAD_NORM] = d[1];
        out[RAMP_ES_UPDATE_RATIO] = d[2]; out[RAMP_ES_EVAL_RETURN_MEAN] = ev; out[RAMP_ES_ROUNDS] = es->rounds;
    }
    return RAMP_OK;
}

// the population buffers for B episodes (2 n_pairs + 1 sets)
int es_population(ramp_es* es, int32_t B) {
    if (B <= es->cap) return RAMP_OK;
    ramp_policy* p = es->p;
    const ramp_policy_config_t& c = p->P.c;
    es->cap = 0;
    const size_t S = (size_t)B + 1;
    CUDA_TRY(es->sets.alloc(S * (size_t)es->n));
    CUDA_TRY(es->emb.alloc(S * c.n_models * c.out_features_node));
    CUDA_TRY(alloc_each(B, es->r_ret, es->logp));
    CUDA_TRY(alloc_each(B, es->r_len, es->r_idx));
    CUDA_TRY(es->logits.alloc((size_t)B * c.n_actions));
    es->cap = B;
    return RAMP_OK;
}

// the embedding kernel's per-CTA scratch, sized by the largest job type
int es_scratch(ramp_es* es, int32_t* max_nodes, int32_t* max_edges, int64_t* slot) {
    ramp_policy* p = es->p;
    const int half = p->P.c.out_features_msg / 2;
    int32_t mn = 1, me = 1;
    for (const HostModel& hm : p->models) {
        if (!hm.set) return set_error(RAMP_ERR_BAD_ARG, "policy: a model was never registered (ramp_policy_set_model)");
        mn = std::max(mn, hm.d.n_nodes); me = std::max(me, hm.d.n_edges);
    }
    *max_nodes = mn; *max_edges = me;
    *slot = (int64_t)mn * (2 * POL_MAX_DIM + half) + (int64_t)me * half;
    if (!es->embed_grid) {
        int per_sm = 0;
        CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ramp_es_embed_kernel, 256, 0));
        es->embed_grid = p->sm_count * std::max(1, std::min(per_sm, 2));
    }
    if (es->scratch.size() < (size_t)es->embed_grid * (size_t)*slot) CUDA_TRY(es->scratch.alloc((size_t)es->embed_grid * (size_t)*slot));
    return RAMP_OK;
}

}  // namespace

extern "C" {

int ramp_es_create(ramp_policy_t* p, const float* noise, int64_t noise_size, ramp_es_t** out) {
    if (!p || !noise || !out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (noise_size < p->n_weights)
        return set_error(RAMP_ERR_BAD_ARG, "es: a noise table of %lld floats is smaller than the policy's %lld weights", (long long)noise_size,
                         (long long)p->n_weights);
    if (noise_size - p->n_weights + 1 > INT32_MAX) return set_error(RAMP_ERR_BAD_ARG, "es: noise indices must fit in int32");
    CUDA_TRY(cudaSetDevice(p->device));
    std::unique_ptr<ramp_es> es(new ramp_es());
    es->p = p;
    es->n = p->n_weights;
    es->noise_size = noise_size;
    CUDA_TRY(es->noise.alloc((size_t)noise_size));
    CUDA_TRY(cudaMemcpy(es->noise.get(), noise, sizeof(float) * (size_t)noise_size, cudaMemcpyHostToDevice));
    CUDA_TRY(alloc_each((size_t)es->n, es->m, es->v, es->g));
    CUDA_TRY(es->part.alloc((size_t)ES_GRID * 4));
    CUDA_TRY(es->dstats.alloc(3));
    CUDA_TRY(cudaMemset(es->m.get(), 0, sizeof(float) * (size_t)es->n));
    CUDA_TRY(cudaMemset(es->v.get(), 0, sizeof(float) * (size_t)es->n));
    CUDA_TRY(cudaMemset(es->g.get(), 0, sizeof(float) * (size_t)es->n));
    *out = es.release();
    return RAMP_OK;
}

void ramp_es_destroy(ramp_es_t* es) {
    if (!es) return;
    cudaSetDevice(es->p->device);
    cudaDeviceSynchronize();                                              // a round may still read the sets
    delete es;
}

int ramp_es_round_begin(ramp_es_t* es, ramp_engine_t* eng, const ramp_es_config_t* cfg, int32_t round) {
    if (!es || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_es_config(cfg);
    if (rc != RAMP_OK) return rc;
    ramp_policy* p = es->p;
    ramp_env_buffers_t eb{};
    if ((rc = ramp_env_buffers(eng, &eb)) != RAMP_OK) return rc;
    const ramp_policy_config_t& c = p->P.c;
    if (ramp_internal_device(eng) != p->device) return set_error(RAMP_ERR_BAD_ARG, "policy and engine live on different devices");
    if (eb.n_actions != c.n_actions) return set_error(RAMP_ERR_BAD_ARG, "policy has %d actions, the environment %d", c.n_actions, eb.n_actions);
    if (c.in_features_graph != 17) return set_error(RAMP_ERR_BAD_ARG, "the environment emits 17 graph features, the policy expects %d", c.in_features_graph);
    if (eb.n_models > c.n_models) return set_error(RAMP_ERR_BAD_ARG, "the environment has %d job types, the policy %d", eb.n_models, c.n_models);
    if (!p->weights_set) return set_error(RAMP_ERR_BAD_ARG, "policy: no weights (ramp_policy_set_weights)");
    const int32_t noisy = eb.n_episodes - cfg->n_eval;
    if (noisy < 2 || (noisy & 1))
        return set_error(RAMP_ERR_BAD_ARG, "es: %d episodes less %d eval episodes leave %d, which must be even and >= 2", eb.n_episodes,
                         cfg->n_eval, noisy);
    if (round < 0 || (round > 0 && round != es->round + 1)) return set_error(RAMP_ERR_BAD_ARG, "es: round %d does not follow round %d", round, es->round);
    if (round > 0 && (eb.n_episodes != es->B || cfg->n_eval != es->n_eval)) return set_error(RAMP_ERR_BAD_ARG, "es: the rounds of a step must share the environment");
    CUDA_TRY(cudaSetDevice(p->device));
    cudaStream_t st = ramp_internal_stream(eng);
    int32_t max_nodes, max_edges;
    int64_t slot;
    if ((rc = es_population(es, eb.n_episodes)) != RAMP_OK || (rc = es_scratch(es, &max_nodes, &max_edges, &slot)) != RAMP_OK) return rc;
    if (round == 0) {
        es->h_idx.clear(); es->h_ret.clear(); es->h_len.clear(); es->h_eval_ret.clear(); es->h_eval_len.clear(); es->h_seeds.clear();
        es->h_ranks.clear();
        es->rounds = 0; es->timesteps = 0;
    }
    es->cfg = *cfg; es->B = eb.n_episodes; es->n_eval = cfg->n_eval; es->n_pairs = noisy / 2; es->round = round;
    // the round's noise indices, uniform on [0, noise_size - n]
    const uint64_t range = (uint64_t)(es->noise_size - es->n + 1);
    std::vector<int32_t> idx(es->n_pairs);
    for (int32_t i = 0; i < es->n_pairs; ++i)
        idx[i] = (int32_t)(((unsigned __int128)es_key(cfg->seed, es->iteration, round, 2 * (uint64_t)i) * range) >> 64);
    CUDA_TRY(cudaMemcpyAsync(es->r_idx.get(), idx.data(), sizeof(int32_t) * es->n_pairs, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));                                   // `idx` is pageable
    es->h_idx.insert(es->h_idx.end(), idx.begin(), idx.end());
    const int S = 2 * es->n_pairs + 1;
    dim3 pg((unsigned)std::min<int64_t>((es->n + 255) / 256, 64), (unsigned)S);
    ramp_es_perturb_kernel<<<pg, 256, 0, st>>>(p->d_w.get(), es->noise.get(), es->r_idx.get(), es->n_pairs, es->n, (float)cfg->noise_stdev,
                                               es->sets.get());
    std::vector<ModelDev> h(p->models.size());
    for (size_t m = 0; m < h.size(); ++m) h[m] = p->models[m].d;
    CUDA_TRY(cudaMemcpyAsync(p->d_models.get(), h.data(), sizeof(ModelDev) * h.size(), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));                                   // `h` is pageable
    EsEmbedArgs ea{};
    ea.n_sets = S; ea.n_models = c.n_models; ea.n_weights = es->n; ea.sets = es->sets.get(); ea.scratch = es->scratch.get();
    ea.slot_floats = slot; ea.max_nodes = max_nodes; ea.max_edges = max_edges; ea.emb = es->emb.get();
    ramp_es_embed_kernel<<<(unsigned)std::min(es->embed_grid, S * c.n_models), 256, 0, st>>>(p->P, p->d_models.get(), ea);
    CUDA_TRY(cudaGetLastError());
    ramp_internal_count_launches(eng, 2);
    return RAMP_OK;
}

int ramp_es_act(ramp_es_t* es, ramp_engine_t* eng, int32_t t) {
    if (!es || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (es->round < 0) return set_error(RAMP_ERR_BAD_ARG, "es: no round (ramp_es_round_begin)");
    ramp_env_buffers_t eb{};
    int rc = ramp_env_buffers(eng, &eb);
    if (rc != RAMP_OK) return rc;
    if (eb.n_episodes != es->B) return set_error(RAMP_ERR_BAD_ARG, "es: the round was begun on another environment");
    ramp_policy* p = es->p;
    CUDA_TRY(cudaSetDevice(p->device));
    HeadArgs a{};
    a.n = es->B; a.obs_dyn = eb.obs_dynamic; a.graph_static = p->d_gstatic.get(); a.model = eb.queued_model; a.done = eb.done;
    a.mask = eb.action_mask; a.emb = es->emb.get(); a.logits = es->logits.get(); a.logp = es->logp.get(); a.actions = eb.actions;
    a.sample = 1; a.seed = es_key(es->cfg.seed, es->iteration, es->round, 2 * (uint64_t)(uint32_t)t + 1);
    es->h_seeds.push_back(a.seed);
    EsHeadArgs e{};
    e.n_pairs = es->n_pairs; e.n_weights = es->n; e.sets = es->sets.get();
    const int wpc = 8;
    int grid = std::min((a.n + wpc - 1) / wpc, p->sm_count * 4);
    ramp_es_head_kernel<<<std::max(grid, 1), wpc * 32, 0, ramp_internal_stream(eng)>>>(p->P, a, e);
    CUDA_TRY(cudaGetLastError());
    ramp_internal_count_launches(eng, 1);
    return RAMP_OK;
}

int ramp_es_round_end(ramp_es_t* es, ramp_engine_t* eng, int32_t* more_out) {
    if (!es || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (es->round < 0) return set_error(RAMP_ERR_BAD_ARG, "es: no round (ramp_es_round_begin)");
    const double* ret; const int32_t* n_decided;
    int rc = ramp_internal_env_returns(eng, &ret, &n_decided);
    if (rc != RAMP_OK) return rc;
    ramp_env_buffers_t eb{};
    if ((rc = ramp_env_buffers(eng, &eb)) != RAMP_OK) return rc;
    if (eb.n_episodes != es->B) return set_error(RAMP_ERR_BAD_ARG, "es: the round was begun on another environment");
    CUDA_TRY(cudaSetDevice(es->p->device));
    cudaStream_t st = ramp_internal_stream(eng);
    const int32_t B = es->B, nv = 2 * es->n_pairs;
    ramp_es_collect_kernel<<<(B + 255) / 256, 256, 0, st>>>(B, ret, n_decided, es->r_ret.get(), es->r_len.get());
    CUDA_TRY(cudaGetLastError());
    std::vector<float> r(B);
    std::vector<int32_t> l(B);
    CUDA_TRY(cudaMemcpyAsync(r.data(), es->r_ret.get(), sizeof(float) * B, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(l.data(), es->r_len.get(), sizeof(int32_t) * B, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    ramp_internal_count_launches(eng, 1);
    es->h_ret.insert(es->h_ret.end(), r.begin(), r.begin() + nv);
    es->h_len.insert(es->h_len.end(), l.begin(), l.begin() + nv);
    es->h_eval_ret.insert(es->h_eval_ret.end(), r.begin() + nv, r.end());
    es->h_eval_len.insert(es->h_eval_len.end(), l.begin() + nv, l.end());
    for (int32_t b = 0; b < nv; ++b) es->timesteps += l[b];
    es->rounds += 1;
    if (more_out)
        *more_out = ((int64_t)es->h_ret.size() < es->cfg.episodes_per_batch || es->timesteps < es->cfg.train_batch_size) ? 1 : 0;
    return RAMP_OK;
}

int ramp_es_step(ramp_es_t* es, const ramp_es_config_t* cfg, double* stats_out) {
    if (!es) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_es_config(cfg);
    if (rc != RAMP_OK) return rc;
    if (es->rounds < 1 || es->h_ret.size() != es->h_idx.size() * 2)
        return set_error(RAMP_ERR_BAD_ARG, "es: no complete round to learn from (ramp_es_round_begin / _end)");
    CUDA_TRY(cudaSetDevice(es->p->device));
    const int32_t n_pairs = (int32_t)es->h_idx.size();
    if ((rc = es_upload(es, n_pairs, es->h_idx.data(), es->h_ret.data())) != RAMP_OK || (rc = es_update(es, *cfg, n_pairs)) != RAMP_OK ||
        (rc = es_finish(es, *cfg, n_pairs, stats_out)) != RAMP_OK)
        return rc;
    es->iteration += 1;
    es->round = -1;
    return RAMP_OK;
}

int ramp_es_update(ramp_es_t* es, const ramp_es_config_t* cfg, int32_t n_pairs, const int32_t* noise_index, const float* returns,
                   float* ranks_out, float* grad_out, double* stats_out) {
    if (!es || !noise_index || !returns) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_es_config(cfg);
    if (rc != RAMP_OK) return rc;
    if (n_pairs < 1) return set_error(RAMP_ERR_BAD_ARG, "es: an update needs at least one pair, got %d", n_pairs);
    if (!es->p->weights_set) return set_error(RAMP_ERR_BAD_ARG, "policy: no weights (ramp_policy_set_weights)");
    for (int32_t i = 0; i < n_pairs; ++i)
        if (noise_index[i] < 0 || (int64_t)noise_index[i] > es->noise_size - es->n)
            return set_error(RAMP_ERR_BAD_ARG, "es: noise index %d of pair %d outside [0, %lld]", noise_index[i], i,
                             (long long)(es->noise_size - es->n));
    CUDA_TRY(cudaSetDevice(es->p->device));
    CUDA_TRY(cudaDeviceSynchronize());                                    // a round may still read theta
    // the update's record: these pairs, no eval episode, no env-steps
    es->h_idx.assign(noise_index, noise_index + n_pairs);
    es->h_ret.assign(returns, returns + 2 * (size_t)n_pairs);
    es->h_len.assign(2 * (size_t)n_pairs, 0);
    es->h_eval_ret.clear(); es->h_eval_len.clear(); es->h_seeds.clear();
    es->rounds = 0; es->timesteps = 0; es->round = -1;
    if ((rc = es_upload(es, n_pairs, noise_index, returns)) != RAMP_OK || (rc = es_update(es, *cfg, n_pairs)) != RAMP_OK ||
        (rc = es_finish(es, *cfg, n_pairs, stats_out)) != RAMP_OK)
        return rc;
    if (ranks_out) memcpy(ranks_out, es->h_ranks.data(), sizeof(float) * 2 * (size_t)n_pairs);
    if (grad_out) CUDA_TRY(cudaMemcpy(grad_out, es->g.get(), sizeof(float) * (size_t)es->n, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

int ramp_es_read(ramp_es_t* es, int32_t* n_pairs_out, int32_t* n_eval_out, int32_t* n_seeds_out, int32_t* noise_index_out,
                 float* returns_out, int32_t* lengths_out, uint64_t* seeds_out, float* ranks_out, float* grad_out,
                 float* eval_returns_out, int32_t* eval_lengths_out) {
    if (!es) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    const size_t np = es->h_idx.size();
    if (n_pairs_out) *n_pairs_out = (int32_t)np;
    if (n_eval_out) *n_eval_out = (int32_t)es->h_eval_ret.size();
    if (n_seeds_out) *n_seeds_out = (int32_t)es->h_seeds.size();
    if (noise_index_out) memcpy(noise_index_out, es->h_idx.data(), sizeof(int32_t) * np);
    if (returns_out) memcpy(returns_out, es->h_ret.data(), sizeof(float) * es->h_ret.size());
    if (lengths_out) memcpy(lengths_out, es->h_len.data(), sizeof(int32_t) * es->h_len.size());
    if (seeds_out) memcpy(seeds_out, es->h_seeds.data(), sizeof(uint64_t) * es->h_seeds.size());
    if (ranks_out) memcpy(ranks_out, es->h_ranks.data(), sizeof(float) * es->h_ranks.size());
    if (eval_returns_out) memcpy(eval_returns_out, es->h_eval_ret.data(), sizeof(float) * es->h_eval_ret.size());
    if (eval_lengths_out) memcpy(eval_lengths_out, es->h_eval_len.data(), sizeof(int32_t) * es->h_eval_len.size());
    if (grad_out) {
        CUDA_TRY(cudaSetDevice(es->p->device));
        CUDA_TRY(cudaDeviceSynchronize());
        CUDA_TRY(cudaMemcpy(grad_out, es->g.get(), sizeof(float) * (size_t)es->n, cudaMemcpyDeviceToHost));
    }
    return RAMP_OK;
}

int ramp_es_act_read(ramp_es_t* es, ramp_engine_t* eng, float* logits_out, float* logp_out, int32_t* actions_out) {
    if (!es || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    ramp_env_buffers_t eb{};
    int rc = ramp_env_buffers(eng, &eb);
    if (rc != RAMP_OK) return rc;
    if (es->cap < 1 || eb.n_episodes != es->B) return set_error(RAMP_ERR_BAD_ARG, "es: nothing to read (ramp_es_act was not called for this environment)");
    cudaStream_t st = ramp_internal_stream(eng);
    const size_t B = (size_t)es->B;
    if (logits_out) CUDA_TRY(cudaMemcpyAsync(logits_out, es->logits.get(), sizeof(float) * B * es->p->P.c.n_actions, cudaMemcpyDeviceToHost, st));
    if (logp_out) CUDA_TRY(cudaMemcpyAsync(logp_out, es->logp.get(), sizeof(float) * B, cudaMemcpyDeviceToHost, st));
    if (actions_out) CUDA_TRY(cudaMemcpyAsync(actions_out, eb.actions, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return RAMP_OK;
}

int ramp_es_state(ramp_es_t* es, float* m_out, float* v_out, int32_t* t_out) {
    if (!es) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    CUDA_TRY(cudaSetDevice(es->p->device));
    CUDA_TRY(cudaDeviceSynchronize());
    if (m_out) CUDA_TRY(cudaMemcpy(m_out, es->m.get(), sizeof(float) * (size_t)es->n, cudaMemcpyDeviceToHost));
    if (v_out) CUDA_TRY(cudaMemcpy(v_out, es->v.get(), sizeof(float) * (size_t)es->n, cudaMemcpyDeviceToHost));
    if (t_out) *t_out = es->t;
    return RAMP_OK;
}

int ramp_es_reset(ramp_es_t* es) {
    if (!es) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    CUDA_TRY(cudaSetDevice(es->p->device));
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemset(es->m.get(), 0, sizeof(float) * (size_t)es->n));
    CUDA_TRY(cudaMemset(es->v.get(), 0, sizeof(float) * (size_t)es->n));
    es->t = 0;
    return RAMP_OK;
}

}  // extern "C"
