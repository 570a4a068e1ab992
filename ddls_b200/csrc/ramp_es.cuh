// ramp_es.cuh -- RLlib's evolution strategies training step on the device (include/ramp_b200.h: ramp_es_*; ray/rllib/algorithms/es:
// es.py training_step, utils.py, optimizers.py), for one policy and for every set of a population (ramp_population_es_*, at the
// end of this file).  Included at the end of ramp_policy.cu, after ramp_population.cuh: the ES population runs the policy's
// forward bodies (gnn_embed_body, head_row) with a weight set per episode.  Each kernel below is a wrapper around its
// __device__ body, which the population's kernels run on one weight set's slice:
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
constexpr int ES_MAX_SETS = 65535;       // weight sets of a round: the perturb launch's gridDim.y

// set s of one weight set's population: 2i = fl(theta + fl(sigma eps_i)), 2i + 1 = fl(theta - fl(sigma eps_i)), 2 n_pairs = theta
__device__ __forceinline__ void es_perturb_body(const float* theta, const float* noise, const int32_t* noise_index, int32_t n_pairs, int64_t n,
                                                float sigma, float* sets, int s) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        float w = theta[k];
        if (s < 2 * n_pairs) {
            const float d = __fmul_rn(sigma, noise[(int64_t)noise_index[s >> 1] + k]);
            w = (s & 1) ? __fsub_rn(w, d) : __fadd_rn(w, d);
        }
        sets[(size_t)s * n + k] = w;
    }
}

__global__ void ramp_es_perturb_kernel(const float* theta, const float* noise, const int32_t* noise_index, int32_t n_pairs,
                                       int64_t n, float sigma, float* sets) {
    es_perturb_body(theta, noise, noise_index, n_pairs, n, sigma, sets, blockIdx.y);   // blockIdx.y = set: 2 n_pairs + 1 of them
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

// one (weight set, job type) item of the ES embedding on this CTA's scratch (the caller syncs before the scratch is reused)
__device__ __forceinline__ void es_embed_item_body(const PolicyDev& P, const ModelDev* models, int m, const float* w, float* z0, float* z1,
                                                   float* hn, float* he, float* emb) {
    ModelDev M = models[m];
    M.z0 = z0; M.z1 = z1; M.hn = hn; M.he = he;
    gnn_embed_body(P, w, M, emb);
}

__global__ void __launch_bounds__(256) ramp_es_embed_kernel(const PolicyDev P, const ModelDev* models, const EsEmbedArgs a) {
    const int half = P.c.out_features_msg / 2;
    float* z0 = a.scratch + (size_t)blockIdx.x * a.slot_floats;
    float* z1 = z0 + (size_t)a.max_nodes * POL_MAX_DIM;
    float* hn = z1 + (size_t)a.max_nodes * POL_MAX_DIM;
    float* he = hn + (size_t)a.max_nodes * half;
    for (int item = blockIdx.x; item < a.n_sets * a.n_models; item += gridDim.x) {
        const int s = item / a.n_models, m = item - s * a.n_models;
        es_embed_item_body(P, models, m, a.sets + (size_t)s * a.n_weights, z0, z1, hn, he, a.emb + (size_t)item * P.c.out_features_node);
        __syncthreads();                  // the next item reuses the scratch
    }
}

struct EsHeadArgs {
    int32_t n_pairs;                      // episode b < 2 n_pairs runs set b, the others set 2 n_pairs
    int64_t n_weights;
    const float* sets;                    // [sets][n_weights]; HeadArgs::emb is [sets][n_models][out_node]
};

// head_row on the episodes cta, cta + n_ctas, ... (a warp each) of one weight set's population, with each episode's set read
// from global memory
__device__ __forceinline__ void es_head_body(const PolicyDev& P, const HeadArgs& a, const EsHeadArgs& e, int cta, int n_ctas) {
    __shared__ float s_warp[8][2 * POL_MAX_DIM];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpc = blockDim.x >> 5;
    for (int b = cta * wpc + warp; b < a.n; b += n_ctas * wpc) {
        const int s = b < 2 * e.n_pairs ? b : 2 * e.n_pairs;
        head_row(P.c, ReadoutBlob(P, e.sets + (size_t)s * e.n_weights), a, a.emb + (size_t)s * P.c.n_models * P.c.out_features_node, b,
                 s_warp[warp], lane);
    }
}

// head_row on each episode with its set's weights read from global memory; the act has no value
__global__ void __launch_bounds__(256) ramp_es_head_kernel(const PolicyDev P, const HeadArgs a, const EsHeadArgs e) {
    es_head_body(P, a, e, blockIdx.x, gridDim.x);
}

__global__ void ramp_es_collect_kernel(int32_t B, const double* ret, const int32_t* n_decided, float* returns, int32_t* lengths) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    returns[b] = (float)ret[b];          // RLlib's float32 sum of float32 rewards, for the environment's +-1 rewards
    lengths[b] = n_decided[b];
}

// rank of x_i = #{j : x_j < x_i or (x_j == x_i and j < i)}; rank / (n - 1) - 0.5 in float32
__device__ __forceinline__ void es_rank_body(const float* x, int32_t n, float* ranks, int i) {
    if (i >= n) return;
    const float xi = x[i];
    int r = 0;
    for (int j = 0; j < n; ++j) { const float xj = x[j]; r += (xj < xi || (xj == xi && j < i)) ? 1 : 0; }
    ranks[i] = __fsub_rn(__fdiv_rn((float)r, (float)(n - 1)), 0.5f);
}

__global__ void ramp_es_rank_kernel(const float* x, int32_t n, float* ranks) {
    es_rank_body(x, n, ranks, blockIdx.x * blockDim.x + threadIdx.x);
}

struct EsUpdateArgs {
    int64_t n;                            // weights
    int32_t n_pairs;
    const int32_t* noise_index; const float* ranks; const float* noise;
    float* theta; float* m; float* v; float* g;
    float l2, beta1, one_m_beta1, beta2, one_m_beta2, eps, neg_a;
    double* part;                         // [ES_GRID][4]: sum step^2, theta_old^2, theta_new^2, g^2
};

// the update of one weight set by a grid of gridDim.x = ES_GRID CTAs: the weights and the norm partials are split by CTA, so
// the partials are summed in the same order whatever else runs in the launch
__device__ __forceinline__ void es_update_body(const EsUpdateArgs& a) {
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

__global__ void __launch_bounds__(256) ramp_es_update_kernel(const EsUpdateArgs a) {
    es_update_body(a);
}

// out: weights_norm, grad_norm, update_ratio
__device__ __forceinline__ void es_stats_body(const double* part, int32_t n_part, double* out) {
    double q[4] = {0.0, 0.0, 0.0, 0.0};
    for (int c = 0; c < n_part; ++c)
        for (int j = 0; j < 4; ++j) q[j] += part[(size_t)c * 4 + j];
    out[0] = q[2];
    out[1] = q[3];
    out[2] = q[1] > 0.0 ? sqrt(q[0]) / sqrt(q[1]) : 0.0;
}

__global__ void ramp_es_stats_kernel(const double* part, int32_t n_part, double* out) {
    es_stats_body(part, n_part, out);
}

}  // namespace ramp

// a training step's record: pairs over all rounds, eval episodes, act seeds; its update's ranks; and every step's mean eval return
struct EsRecord {
    std::vector<int32_t> idx, len, eval_len;
    std::vector<float> ret, eval_ret, ranks;
    std::vector<uint64_t> seeds;
    int32_t rounds = 0;
    int64_t timesteps = 0;
    std::vector<double> reward_list;      // kept across steps: episode_reward_mean's window
    void begin() {
        idx.clear(); ret.clear(); len.clear(); eval_ret.clear(); eval_len.clear(); seeds.clear(); ranks.clear();
        rounds = 0; timesteps = 0;
    }
};

struct ramp_es {
    ramp_policy* p = nullptr;
    int device = 0;                       // p's: ramp_es_destroy does not read p, which may be gone by then
    int64_t n = 0, noise_size = 0;
    DeviceArray<float> noise, m, v, g, ranks, returns;
    DeviceArray<int32_t> idx;
    DeviceArray<double> part, dstats;
    int32_t t = 0;                        // Adam's step count
    int64_t iteration = 0;                // ramp_es_step calls: keys the noise indices and the draws
    // the population of the current round: sets, embeddings, per-CTA embedding scratch, the round's returns / env-steps and the
    // last act's outputs, for `cap` episodes
    int32_t cap = 0, B = 0, n_pairs = 0, n_eval = 0, round = -1, embed_grid = 0;
    DeviceArray<float> sets, emb, scratch, r_ret, logits, logp;
    DeviceArray<int32_t> r_len, r_idx;
    ramp_es_config_t cfg{};
    EsRecord rec;                         // the step record; its g is `g`
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

// the record's eval means and the statistics row from the update's norms d
void es_stats_row(EsRecord& r, const ramp_es_config_t& cfg, int32_t n_pairs, const double* d, double* out) {
    const double nan = std::nan("");
    double ev = nan, el = nan;
    if (!r.eval_ret.empty()) {
        double s = 0.0, l = 0.0;
        for (size_t i = 0; i < r.eval_ret.size(); ++i) { s += r.eval_ret[i]; l += r.eval_len[i]; }
        ev = s / (double)r.eval_ret.size();
        el = l / (double)r.eval_len.size();
        r.reward_list.push_back(ev);
    }
    double rm = nan;
    if (!r.reward_list.empty()) {
        const size_t k = std::min(r.reward_list.size(), (size_t)cfg.report_length);
        rm = 0.0;
        for (size_t i = r.reward_list.size() - k; i < r.reward_list.size(); ++i) rm += r.reward_list[i];
        rm /= (double)k;
    }
    if (out) {
        out[RAMP_ES_EPISODE_REWARD_MEAN] = rm; out[RAMP_ES_EPISODE_LEN_MEAN] = el; out[RAMP_ES_TIMESTEPS_THIS_ITER] = (double)r.timesteps;
        out[RAMP_ES_EPISODES_THIS_ITER] = 2.0 * n_pairs; out[RAMP_ES_WEIGHTS_NORM] = d[0]; out[RAMP_ES_GRAD_NORM] = d[1];
        out[RAMP_ES_UPDATE_RATIO] = d[2]; out[RAMP_ES_EVAL_RETURN_MEAN] = ev; out[RAMP_ES_ROUNDS] = r.rounds;
    }
}

// the statistics es_update leaves on the device, the ranks and the eval means into `out`
int es_finish(ramp_es* es, const ramp_es_config_t& cfg, int32_t n_pairs, double* out) {
    double d[3];
    CUDA_TRY(cudaStreamSynchronize(0));
    CUDA_TRY(cudaMemcpy(d, es->dstats.get(), sizeof(d), cudaMemcpyDeviceToHost));
    es->rec.ranks.resize(2 * (size_t)n_pairs);
    CUDA_TRY(cudaMemcpy(es->rec.ranks.data(), es->ranks.get(), sizeof(float) * 2 * n_pairs, cudaMemcpyDeviceToHost));
    es_stats_row(es->rec, cfg, n_pairs, d, out);
    return RAMP_OK;
}

// a round's returns / env-steps of one weight set's b episodes (nv noisy, then the eval ones) into its record
void es_record_round(EsRecord& r, const float* ret, const int32_t* len, int32_t nv, int32_t b) {
    r.ret.insert(r.ret.end(), ret, ret + nv);
    r.len.insert(r.len.end(), len, len + nv);
    r.eval_ret.insert(r.eval_ret.end(), ret + nv, ret + b);
    r.eval_len.insert(r.eval_len.end(), len + nv, len + b);
    for (int32_t i = 0; i < nv; ++i) r.timesteps += len[i];
    r.rounds += 1;
}

// another round is needed: fewer than episodes_per_batch noisy episodes or train_batch_size noisy env-steps recorded
bool es_more(const EsRecord& r, const ramp_es_config_t& cfg) {
    return (int64_t)r.ret.size() < cfg.episodes_per_batch || r.timesteps < cfg.train_batch_size;
}

// an update's record on host inputs: these pairs, no eval episode, no env-steps
void es_host_record(EsRecord& r, int32_t n_pairs, const int32_t* noise_index, const float* returns) {
    r.begin();
    r.idx.assign(noise_index, noise_index + n_pairs);
    r.ret.assign(returns, returns + 2 * (size_t)n_pairs);
    r.len.assign(2 * (size_t)n_pairs, 0);
}

void es_read_record(const EsRecord& r, int32_t* n_pairs_out, int32_t* n_eval_out, int32_t* n_seeds_out, int32_t* noise_index_out,
                    float* returns_out, int32_t* lengths_out, uint64_t* seeds_out, float* ranks_out, float* eval_returns_out,
                    int32_t* eval_lengths_out) {
    const size_t np = r.idx.size();
    if (n_pairs_out) *n_pairs_out = (int32_t)np;
    if (n_eval_out) *n_eval_out = (int32_t)r.eval_ret.size();
    if (n_seeds_out) *n_seeds_out = (int32_t)r.seeds.size();
    if (noise_index_out) memcpy(noise_index_out, r.idx.data(), sizeof(int32_t) * np);
    if (returns_out) memcpy(returns_out, r.ret.data(), sizeof(float) * r.ret.size());
    if (lengths_out) memcpy(lengths_out, r.len.data(), sizeof(int32_t) * r.len.size());
    if (seeds_out) memcpy(seeds_out, r.seeds.data(), sizeof(uint64_t) * r.seeds.size());
    if (ranks_out) memcpy(ranks_out, r.ranks.data(), sizeof(float) * r.ranks.size());
    if (eval_returns_out) memcpy(eval_returns_out, r.eval_ret.data(), sizeof(float) * r.eval_ret.size());
    if (eval_lengths_out) memcpy(eval_lengths_out, r.eval_len.data(), sizeof(int32_t) * r.eval_len.size());
}

// what the next steps read besides the Adam state: the iteration count (it keys the noise indices and the act seeds) and the
// record's eval means so far (episode_reward_mean's window); rewards_out may be NULL to learn n_rewards first
void es_get_progress(int64_t iteration, const EsRecord& r, int64_t* iteration_out, int32_t* n_rewards_out, double* rewards_out) {
    if (iteration_out) *iteration_out = iteration;
    if (n_rewards_out) *n_rewards_out = (int32_t)r.reward_list.size();
    if (rewards_out) memcpy(rewards_out, r.reward_list.data(), sizeof(double) * r.reward_list.size());
}

int es_set_progress(int64_t* iteration, EsRecord& r, int64_t it, int32_t n_rewards, const double* rewards) {
    if (it < 0 || n_rewards < 0 || (n_rewards > 0 && !rewards))
        return set_error(RAMP_ERR_BAD_ARG, "es: iteration %lld and %d eval means (both must be >= 0)", (long long)it, n_rewards);
    *iteration = it;
    r.reward_list.assign(rewards, rewards + n_rewards);
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
    es->device = p->device;
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
    cudaSetDevice(es->device);
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
    if (noisy + 1 > ES_MAX_SETS)
        return set_error(RAMP_ERR_BAD_ARG, "es: %d noisy episodes and theta make %d weight sets a round, more than %d", noisy, noisy + 1, ES_MAX_SETS);
    if (round < 0 || (round > 0 && round != es->round + 1)) return set_error(RAMP_ERR_BAD_ARG, "es: round %d does not follow round %d", round, es->round);
    if (round > 0 && (eb.n_episodes != es->B || cfg->n_eval != es->n_eval)) return set_error(RAMP_ERR_BAD_ARG, "es: the rounds of a step must share the environment");
    CUDA_TRY(cudaSetDevice(p->device));
    cudaStream_t st = ramp_internal_stream(eng);
    int32_t max_nodes, max_edges;
    int64_t slot;
    if ((rc = es_population(es, eb.n_episodes)) != RAMP_OK || (rc = es_scratch(es, &max_nodes, &max_edges, &slot)) != RAMP_OK) return rc;
    if (round == 0) es->rec.begin();
    es->cfg = *cfg; es->B = eb.n_episodes; es->n_eval = cfg->n_eval; es->n_pairs = noisy / 2; es->round = round;
    // the round's noise indices, uniform on [0, noise_size - n]
    const uint64_t range = (uint64_t)(es->noise_size - es->n + 1);
    std::vector<int32_t> idx(es->n_pairs);
    for (int32_t i = 0; i < es->n_pairs; ++i)
        idx[i] = (int32_t)(((unsigned __int128)es_key(cfg->seed, es->iteration, round, 2 * (uint64_t)i) * range) >> 64);
    CUDA_TRY(cudaMemcpyAsync(es->r_idx.get(), idx.data(), sizeof(int32_t) * es->n_pairs, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));                                   // `idx` is pageable
    es->rec.idx.insert(es->rec.idx.end(), idx.begin(), idx.end());
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
    es->rec.seeds.push_back(a.seed);
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
    es_record_round(es->rec, r.data(), l.data(), nv, B);
    if (more_out) *more_out = es_more(es->rec, es->cfg) ? 1 : 0;
    return RAMP_OK;
}

int ramp_es_step(ramp_es_t* es, const ramp_es_config_t* cfg, double* stats_out) {
    if (!es) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_es_config(cfg);
    if (rc != RAMP_OK) return rc;
    if (es->rec.rounds < 1 || es->rec.ret.size() != es->rec.idx.size() * 2)
        return set_error(RAMP_ERR_BAD_ARG, "es: no complete round to learn from (ramp_es_round_begin / _end)");
    CUDA_TRY(cudaSetDevice(es->p->device));
    const int32_t n_pairs = (int32_t)es->rec.idx.size();
    if ((rc = es_upload(es, n_pairs, es->rec.idx.data(), es->rec.ret.data())) != RAMP_OK || (rc = es_update(es, *cfg, n_pairs)) != RAMP_OK ||
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
    es_host_record(es->rec, n_pairs, noise_index, returns);
    es->round = -1;
    if ((rc = es_upload(es, n_pairs, noise_index, returns)) != RAMP_OK || (rc = es_update(es, *cfg, n_pairs)) != RAMP_OK ||
        (rc = es_finish(es, *cfg, n_pairs, stats_out)) != RAMP_OK)
        return rc;
    if (ranks_out) memcpy(ranks_out, es->rec.ranks.data(), sizeof(float) * 2 * (size_t)n_pairs);
    if (grad_out) CUDA_TRY(cudaMemcpy(grad_out, es->g.get(), sizeof(float) * (size_t)es->n, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

int ramp_es_read(ramp_es_t* es, int32_t* n_pairs_out, int32_t* n_eval_out, int32_t* n_seeds_out, int32_t* noise_index_out,
                 float* returns_out, int32_t* lengths_out, uint64_t* seeds_out, float* ranks_out, float* grad_out,
                 float* eval_returns_out, int32_t* eval_lengths_out) {
    if (!es) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    es_read_record(es->rec, n_pairs_out, n_eval_out, n_seeds_out, noise_index_out, returns_out, lengths_out, seeds_out, ranks_out,
                   eval_returns_out, eval_lengths_out);
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

int ramp_es_set_state(ramp_es_t* es, const float* m, const float* v, int64_t n, int32_t t) {
    if (!es || !m || !v) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (n != es->n) return set_error(RAMP_ERR_BAD_ARG, "es: an Adam state of %lld weights given, the policy has %lld", (long long)n, (long long)es->n);
    if (t < 0) return set_error(RAMP_ERR_BAD_ARG, "es: Adam step count %d < 0", t);
    CUDA_TRY(cudaSetDevice(es->p->device));
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(es->m.get(), m, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(es->v.get(), v, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice));
    es->t = t;
    return RAMP_OK;
}

int ramp_es_get_progress(ramp_es_t* es, int64_t* iteration_out, int32_t* n_rewards_out, double* rewards_out) {
    if (!es) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    es_get_progress(es->iteration, es->rec, iteration_out, n_rewards_out, rewards_out);
    return RAMP_OK;
}

int ramp_es_set_progress(ramp_es_t* es, int64_t iteration, int32_t n_rewards, const double* rewards) {
    if (!es) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    return es_set_progress(&es->iteration, es->rec, iteration, n_rewards, rewards);
}

}  // extern "C"

// ---- a population's ES (include/ramp_b200.h: ramp_population_es_*): group k of the environment's K b episodes is the ES
// population of weight set k, with its own config.  The round's ES weight sets of every group lie one group after another in one
// buffer, each group's as the single learner lays out its own; the kernels below run the single kernels' bodies on one group's
// slice, the group taken from the launch or from the round's group table:
//
//   ramp_pop_es_perturb_kernel   blockIdx.y = one ES set of some group: es_perturb_body with the group's theta, sigma and pairs
//   ramp_pop_es_embed_kernel     persistent CTAs over (ES set, job type) items, the set's PopSet staged, scratch sized by the
//                                largest set
//   ramp_pop_es_head_kernel      blockIdx.y = group, one warp per episode: es_head_body on the group's episodes and sets
//   ramp_pop_es_rank_kernel      blockIdx.y = group: es_rank_body over the group's 2 N values
//   ramp_pop_es_update_kernel    (ES_GRID, K) CTAs: es_update_body on group k's EsUpdateArgs, so its g, Adam and norm partials
//                                are split and summed as the single kernel's
//   ramp_pop_es_stats_kernel     one thread per group: es_stats_body on its partials
//
// A group whose twin would have stopped (its record holds episodes_per_batch noisy episodes and train_batch_size noisy env-steps)
// gets no pairs in the later rounds: all its episodes run theta (the "episode >= 2 N runs theta" rule) and nothing of theirs is
// recorded.

namespace ramp {

struct EsPopGroup {
    int64_t n;                            // set k's weights
    int64_t theta_off;                    // set k's offset in the population's weights, and in the ES Adam state and g
    int64_t sets_off, emb_off;            // its first ES set in the round's set and embedding buffers
    int32_t set0;                         // its first ES set among the round's
    int32_t n_pairs;                      // the round's pairs: 2 n_pairs + 1 ES sets (0: the group only runs theta)
    int32_t pair0;                        // its first noise index among the round's
    float sigma;
    unsigned long long round_key;         // es_key(seed, iteration, round, .) before its last mix: act t draws with mix(key ^ (2t + 1))
};

struct EsPopArgs {
    int32_t n_models, b;                  // job types; episodes per group
    const EsPopGroup* groups;             // [K]
    const int32_t* set_group;             // [the round's ES sets] each one's group
    const PopSet* pop;                    // the population's set table
    const float* theta; const float* noise; const int32_t* noise_index;
    float* sets; float* emb;
    float* scratch;                       // [gridDim.x][slot_floats], laid out as EsEmbedArgs::scratch for the largest set
    int64_t slot_floats;
    int32_t max_nodes;
};

__global__ void ramp_pop_es_perturb_kernel(const EsPopArgs a) {
    const int e = blockIdx.y;
    const EsPopGroup G = a.groups[a.set_group[e]];
    es_perturb_body(a.theta + G.theta_off, a.noise, a.noise_index + G.pair0, G.n_pairs, G.n, G.sigma, a.sets + G.sets_off, e - G.set0);
}

__global__ void __launch_bounds__(256) ramp_pop_es_embed_kernel(const ModelDev* models, const EsPopArgs a, int32_t n_items) {
    __shared__ PopSet S;
    float* z0 = a.scratch + (size_t)blockIdx.x * a.slot_floats;
    float* z1 = z0 + (size_t)a.max_nodes * POL_MAX_DIM;
    float* hn = z1 + (size_t)a.max_nodes * POL_MAX_DIM;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int e = item / a.n_models, m = item - e * a.n_models, k = a.set_group[e];
        const EsPopGroup G = a.groups[k];
        pop_stage_set(a.pop, k, &S);
        const size_t s = e - G.set0;
        es_embed_item_body(S.P, models, m, a.sets + G.sets_off + s * G.n, z0, z1, hn, hn + (size_t)a.max_nodes * (S.P.c.out_features_msg / 2),
                           a.emb + G.emb_off + (s * a.n_models + m) * S.P.c.out_features_node);
        __syncthreads();                  // the next item reuses the scratch and the staging
    }
}

// base: the environment's buffers for all K b episodes (HeadArgs::emb unused)
__global__ void __launch_bounds__(256) ramp_pop_es_head_kernel(const EsPopArgs p, const HeadArgs base, int32_t t) {
    __shared__ PopSet S;
    const int k = blockIdx.y;
    pop_stage_set(p.pop, k, &S);
    const EsPopGroup G = p.groups[k];
    const size_t o = (size_t)k * p.b, A = S.P.c.n_actions;
    HeadArgs a = base;
    a.n = p.b;
    a.obs_dyn += o * 11; a.model += o; a.done += o; a.mask += o * A; a.logits += o * A; a.logp += o; a.actions += o;
    a.emb = p.emb + G.emb_off;
    a.seed = splitmix64(G.round_key ^ (2ull * (unsigned)t + 1));
    EsHeadArgs e{};
    e.n_pairs = G.n_pairs; e.n_weights = G.n; e.sets = p.sets + G.sets_off;
    es_head_body(S.P, a, e, blockIdx.x, gridDim.x);
}

// pair0: [K + 1] group k's pairs are [pair0[k], pair0[k + 1]) of x / ranks' pairs
__global__ void ramp_pop_es_rank_kernel(const float* x, const int32_t* pair0, float* ranks) {
    const int k = blockIdx.y, p0 = pair0[k];
    es_rank_body(x + 2 * p0, 2 * (pair0[k + 1] - p0), ranks + 2 * p0, blockIdx.x * blockDim.x + threadIdx.x);
}

__global__ void __launch_bounds__(256) ramp_pop_es_update_kernel(const EsUpdateArgs* args) {
    const EsUpdateArgs a = args[blockIdx.y];
    es_update_body(a);
}

__global__ void ramp_pop_es_stats_kernel(const double* part, int32_t K, double* out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < K) es_stats_body(part + (size_t)k * ES_GRID * 4, ES_GRID, out + 3 * (size_t)k);
}

}  // namespace ramp

struct ramp_population_es {
    ramp_population* q = nullptr;
    int device = 0;                       // q's: ramp_population_es_destroy does not read q, which may be gone by then
    int32_t K = 0;
    int64_t noise_size = 0;
    DeviceArray<float> noise, m, v, g;    // m, v, g: [sum n_w] in the population's layout (PopSet::w_off)
    DeviceArray<float> returns, ranks;    // the update's [sum pairs][2]
    DeviceArray<int32_t> idx, pair0;      // the update's [sum pairs] noise indices, [K + 1] each group's first pair
    DeviceArray<EsUpdateArgs> d_update;
    DeviceArray<double> part, dstats;     // [K][ES_GRID][4], [K][3]
    std::vector<int32_t> t;               // each set's Adam step count
    int64_t iteration = 0;                // ramp_population_es_step calls: keys the noise indices and the draws
    // the current round: every group's ES sets, embeddings, the round's returns / env-steps and the last act's outputs
    int32_t B = 0, b = 0, round = -1, embed_grid = 0, n_sets = 0;
    size_t sets_cap = 0, emb_cap = 0, b_cap = 0, groups_cap = 0;
    DeviceArray<float> sets, emb, scratch, r_ret, logits, logp;
    DeviceArray<int32_t> r_len, r_idx, set_group;
    DeviceArray<EsPopGroup> d_groups;
    std::vector<EsPopGroup> groups;
    std::vector<int32_t> n_eval;          // each group's eval episodes this step
    std::vector<uint8_t> more;            // group k's twin would run another round
    std::vector<ramp_es_config_t> cfgs;   // the configs of the current step
    std::vector<EsRecord> rec;            // each set's step record
};

namespace {

int pes_check_configs(const ramp_population_es* es, const ramp_es_config_t* cfgs) {
    if (!es || !cfgs) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    for (int k = 0; k < es->K; ++k)
        if (check_es_config(&cfgs[k]) != RAMP_OK) return set_error(RAMP_ERR_BAD_ARG, "population: set %d: %s", k, g_last_error.c_str());
    return RAMP_OK;
}

// the update of every group on the pairs in es->idx / es->returns (group k's from pair0[k]), on stream 0; writes es->dstats
int pes_update(ramp_population_es* es, const ramp_es_config_t* cfgs, const std::vector<int32_t>& pair0) {
    ramp_population* q = es->q;
    const int32_t K = es->K;
    int32_t max_nv = 0;
    std::vector<EsUpdateArgs> u(K);
    for (int k = 0; k < K; ++k) {
        const ramp_es_config_t& cfg = cfgs[k];
        const int32_t n_pairs = pair0[k + 1] - pair0[k];
        max_nv = std::max(max_nv, 2 * n_pairs);
        es->t[k] += 1;
        const double a = cfg.stepsize * (std::sqrt(1.0 - std::pow(cfg.adam_beta2, es->t[k])) / (1.0 - std::pow(cfg.adam_beta1, es->t[k])));
        const size_t o = q->sets[k].w_off;
        EsUpdateArgs& x = u[k];
        x.n = q->sets[k].n_w; x.n_pairs = n_pairs; x.noise_index = es->idx.get() + pair0[k]; x.ranks = es->ranks.get() + 2 * (size_t)pair0[k];
        x.noise = es->noise.get(); x.theta = q->d_w.get() + o; x.m = es->m.get() + o; x.v = es->v.get() + o; x.g = es->g.get() + o;
        x.l2 = (float)cfg.l2_coeff; x.beta1 = (float)cfg.adam_beta1; x.one_m_beta1 = (float)(1.0 - cfg.adam_beta1);
        x.beta2 = (float)cfg.adam_beta2; x.one_m_beta2 = (float)(1.0 - cfg.adam_beta2); x.eps = (float)cfg.adam_eps; x.neg_a = (float)(-a);
        x.part = es->part.get() + (size_t)k * ES_GRID * 4;
    }
    CUDA_TRY(cudaMemcpy(es->pair0.get(), pair0.data(), sizeof(int32_t) * (K + 1), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(es->d_update.get(), u.data(), sizeof(EsUpdateArgs) * K, cudaMemcpyHostToDevice));
    ramp_pop_es_rank_kernel<<<dim3((max_nv + 255) / 256, K), 256>>>(es->returns.get(), es->pair0.get(), es->ranks.get());
    ramp_pop_es_update_kernel<<<dim3(ES_GRID, K), 256>>>(es->d_update.get());
    ramp_pop_es_stats_kernel<<<(K + 127) / 128, 128>>>(es->part.get(), K, es->dstats.get());
    CUDA_TRY(cudaGetLastError());
    q->emb_valid = false;
    return RAMP_OK;
}

// the update's inputs on the device: n pairs in all
int pes_upload(ramp_population_es* es, int32_t n, const int32_t* idx, const float* returns) {
    if ((size_t)n > es->idx.size()) CUDA_TRY(es->idx.alloc(n));
    if ((size_t)(2 * n) > es->returns.size()) CUDA_TRY(alloc_each(2 * (size_t)n, es->returns, es->ranks));
    CUDA_TRY(cudaMemcpy(es->idx.get(), idx, sizeof(int32_t) * n, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(es->returns.get(), returns, sizeof(float) * 2 * n, cudaMemcpyHostToDevice));
    return RAMP_OK;
}

// every group's statistics row and ranks after pes_update
int pes_finish(ramp_population_es* es, const ramp_es_config_t* cfgs, const std::vector<int32_t>& pair0, double* out) {
    const int32_t K = es->K;
    std::vector<double> d(3 * (size_t)K);
    std::vector<float> ranks(2 * (size_t)pair0[K]);
    CUDA_TRY(cudaStreamSynchronize(0));
    CUDA_TRY(cudaMemcpy(d.data(), es->dstats.get(), sizeof(double) * d.size(), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(ranks.data(), es->ranks.get(), sizeof(float) * ranks.size(), cudaMemcpyDeviceToHost));
    for (int k = 0; k < K; ++k) {
        const int32_t n_pairs = pair0[k + 1] - pair0[k];
        es->rec[k].ranks.assign(ranks.begin() + 2 * (size_t)pair0[k], ranks.begin() + 2 * (size_t)pair0[k + 1]);
        es_stats_row(es->rec[k], cfgs[k], n_pairs, d.data() + 3 * (size_t)k, out ? out + (size_t)k * RAMP_ES_STATS_LEN : nullptr);
    }
    return RAMP_OK;
}

// the records' pairs, concatenated in set order, into the update's inputs
int pes_update_records(ramp_population_es* es, const ramp_es_config_t* cfgs, double* stats_out) {
    const int32_t K = es->K;
    std::vector<int32_t> pair0(K + 1, 0), idx;
    std::vector<float> ret;
    for (int k = 0; k < K; ++k) {
        pair0[k + 1] = pair0[k] + (int32_t)es->rec[k].idx.size();
        idx.insert(idx.end(), es->rec[k].idx.begin(), es->rec[k].idx.end());
        ret.insert(ret.end(), es->rec[k].ret.begin(), es->rec[k].ret.end());
    }
    int rc;
    if ((rc = pes_upload(es, pair0[K], idx.data(), ret.data())) != RAMP_OK || (rc = pes_update(es, cfgs, pair0)) != RAMP_OK ||
        (rc = pes_finish(es, cfgs, pair0, stats_out)) != RAMP_OK)
        return rc;
    es->round = -1;
    return RAMP_OK;
}

// the embedding kernel's per-CTA scratch, sized by the largest job type and the largest set's message width
int pes_scratch(ramp_population_es* es, int32_t* max_nodes, int64_t* slot) {
    ramp_policy* p = es->q->p;
    int half = 1;
    for (const ramp_policy_config_t& c : es->q->cfgs) half = std::max(half, c.out_features_msg / 2);
    int32_t mn = 1, me = 1;
    for (const HostModel& hm : p->models) {
        if (!hm.set) return set_error(RAMP_ERR_BAD_ARG, "policy: a model was never registered (ramp_policy_set_model)");
        mn = std::max(mn, hm.d.n_nodes); me = std::max(me, hm.d.n_edges);
    }
    *max_nodes = mn;
    *slot = (int64_t)mn * (2 * POL_MAX_DIM + half) + (int64_t)me * half;
    if (es->scratch.size() < (size_t)es->embed_grid * (size_t)*slot) CUDA_TRY(es->scratch.alloc((size_t)es->embed_grid * (size_t)*slot));
    return RAMP_OK;
}

}  // namespace

extern "C" {

int ramp_population_es_create(ramp_population_t* q, const float* noise, int64_t noise_size, ramp_population_es_t** out) {
    if (!q || !noise || !out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int64_t n_max = 0, n_min = INT64_MAX;
    for (int k = 0; k < q->K; ++k) { n_max = std::max(n_max, q->sets[k].n_w); n_min = std::min(n_min, q->sets[k].n_w); }
    if (noise_size < n_max) {
        int k = 0;
        while (q->sets[k].n_w <= noise_size) ++k;
        return set_error(RAMP_ERR_BAD_ARG, "es: a noise table of %lld floats is smaller than set %d's %lld weights", (long long)noise_size, k,
                         (long long)q->sets[k].n_w);
    }
    if (noise_size - n_min + 1 > INT32_MAX) return set_error(RAMP_ERR_BAD_ARG, "es: noise indices must fit in int32");
    CUDA_TRY(cudaSetDevice(q->p->device));
    std::unique_ptr<ramp_population_es> es(new ramp_population_es());
    es->q = q;
    es->device = q->p->device;
    es->K = q->K;
    es->noise_size = noise_size;
    const size_t K = q->K;
    CUDA_TRY(es->noise.alloc((size_t)noise_size));
    CUDA_TRY(cudaMemcpy(es->noise.get(), noise, sizeof(float) * (size_t)noise_size, cudaMemcpyHostToDevice));
    CUDA_TRY(alloc_each((size_t)q->nw, es->m, es->v, es->g));
    CUDA_TRY(es->part.alloc(K * ES_GRID * 4));
    CUDA_TRY(es->dstats.alloc(3 * K));
    CUDA_TRY(es->pair0.alloc(K + 1));
    CUDA_TRY(es->d_update.alloc(K));
    CUDA_TRY(es->d_groups.alloc(K));
    CUDA_TRY(cudaMemset(es->m.get(), 0, sizeof(float) * (size_t)q->nw));
    CUDA_TRY(cudaMemset(es->v.get(), 0, sizeof(float) * (size_t)q->nw));
    CUDA_TRY(cudaMemset(es->g.get(), 0, sizeof(float) * (size_t)q->nw));
    int per_sm = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ramp_pop_es_embed_kernel, 256, 0));
    es->embed_grid = q->p->sm_count * std::max(1, std::min(per_sm, 2));
    es->t.assign(K, 0);
    es->rec.resize(K);
    *out = es.release();
    return RAMP_OK;
}

void ramp_population_es_destroy(ramp_population_es_t* es) {
    if (!es) return;
    cudaSetDevice(es->device);
    cudaDeviceSynchronize();                                              // a round may still read the sets
    delete es;
}

int ramp_population_es_round_begin(ramp_population_es_t* es, ramp_engine_t* eng, const ramp_es_config_t* cfgs, int32_t round) {
    if (!es || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = pes_check_configs(es, cfgs);
    if (rc != RAMP_OK) return rc;
    ramp_population* q = es->q;
    ramp_policy* p = q->p;
    const int32_t K = es->K;
    ramp_env_buffers_t eb{};
    if ((rc = ramp_env_buffers(eng, &eb)) != RAMP_OK) return rc;
    const ramp_policy_config_t& c = p->P.c;
    if (ramp_internal_device(eng) != p->device) return set_error(RAMP_ERR_BAD_ARG, "policy and engine live on different devices");
    if (eb.n_actions != c.n_actions) return set_error(RAMP_ERR_BAD_ARG, "policy has %d actions, the environment %d", c.n_actions, eb.n_actions);
    if (c.in_features_graph != 17) return set_error(RAMP_ERR_BAD_ARG, "the environment emits 17 graph features, the policy expects %d", c.in_features_graph);
    if (eb.n_models > c.n_models) return set_error(RAMP_ERR_BAD_ARG, "the environment has %d job types, the policy %d", eb.n_models, c.n_models);
    if ((rc = pop_check_weights(q)) != RAMP_OK) return rc;
    if (eb.n_episodes % K)
        return set_error(RAMP_ERR_BAD_ARG, "population: %d episodes do not split into %d groups of equal size", eb.n_episodes, K);
    const int32_t b = eb.n_episodes / K;
    for (int k = 0; k < K; ++k) {
        const int32_t noisy = b - cfgs[k].n_eval;
        if (noisy < 2 || (noisy & 1))
            return set_error(RAMP_ERR_BAD_ARG, "population: set %d: es: %d episodes of its group less %d eval episodes leave %d, which must be even and >= 2",
                             k, b, cfgs[k].n_eval, noisy);
    }
    if (round < 0 || (round > 0 && round != es->round + 1)) return set_error(RAMP_ERR_BAD_ARG, "es: round %d does not follow round %d", round, es->round);
    if (round > 0) {
        if (eb.n_episodes != es->B) return set_error(RAMP_ERR_BAD_ARG, "es: the rounds of a step must share the environment");
        for (int k = 0; k < K; ++k)
            if (cfgs[k].n_eval != es->n_eval[k]) return set_error(RAMP_ERR_BAD_ARG, "population: set %d: es: the rounds of a step must share n_eval", k);
        if (std::find(es->more.begin(), es->more.end(), 1) == es->more.end())
            return set_error(RAMP_ERR_BAD_ARG, "es: every set has collected its step's episodes and env-steps: no round %d", round);
    }
    int64_t n_sets = 0;                                                   // 2 N_k + 1 for a group still collecting, else theta alone
    for (int k = 0; k < K; ++k) n_sets += (round == 0 || es->more[k]) ? b - cfgs[k].n_eval + 1 : 1;
    if (n_sets > ES_MAX_SETS)
        return set_error(RAMP_ERR_BAD_ARG, "population: es: the groups' noisy episodes and theta sets make %lld weight sets a round, more than %d",
                         (long long)n_sets, ES_MAX_SETS);
    CUDA_TRY(cudaSetDevice(p->device));
    cudaStream_t st = ramp_internal_stream(eng);
    if ((rc = fence_in(p, st)) != RAMP_OK) return rc;                    // a ramp_population_copy_sets may still write the weights
    if (round == 0) {
        for (EsRecord& r : es->rec) r.begin();
        es->n_eval.resize(K);
        es->more.assign(K, 1);
        for (int k = 0; k < K; ++k) es->n_eval[k] = cfgs[k].n_eval;
    }
    es->cfgs.assign(cfgs, cfgs + K);
    es->B = eb.n_episodes; es->b = b; es->round = round;
    // the groups' layout in the round's buffers, and the round's noise indices, uniform on [0, noise_size - n_k]
    es->groups.resize(K);
    std::vector<int32_t> idx, set_group;
    size_t n_sets_w = 0, n_emb = 0;
    for (int k = 0; k < K; ++k) {
        EsPopGroup& G = es->groups[k];
        const PopSet& S = q->sets[k];
        G.n = S.n_w; G.theta_off = S.w_off; G.sets_off = n_sets_w; G.emb_off = n_emb; G.set0 = (int32_t)set_group.size();
        G.n_pairs = es->more[k] ? (b - cfgs[k].n_eval) / 2 : 0;
        G.pair0 = (int32_t)idx.size(); G.sigma = (float)cfgs[k].noise_stdev;
        G.round_key = mix64(mix64(mix64(cfgs[k].seed) ^ (uint64_t)es->iteration) ^ (uint64_t)round);
        const uint64_t range = (uint64_t)(es->noise_size - G.n + 1);
        for (int32_t i = 0; i < G.n_pairs; ++i)
            idx.push_back((int32_t)(((unsigned __int128)es_key(cfgs[k].seed, es->iteration, round, 2 * (uint64_t)i) * range) >> 64));
        es->rec[k].idx.insert(es->rec[k].idx.end(), idx.begin() + G.pair0, idx.end());
        const int S_k = 2 * G.n_pairs + 1;
        set_group.insert(set_group.end(), S_k, k);
        n_sets_w += (size_t)S_k * G.n;
        n_emb += (size_t)S_k * c.n_models * q->cfgs[k].out_features_node;
    }
    es->n_sets = (int32_t)set_group.size();
    if (n_sets_w > es->sets_cap) { es->sets_cap = 0; CUDA_TRY(es->sets.alloc(n_sets_w)); es->sets_cap = n_sets_w; }
    if (n_emb > es->emb_cap) { es->emb_cap = 0; CUDA_TRY(es->emb.alloc(n_emb)); es->emb_cap = n_emb; }
    if (set_group.size() > es->groups_cap) { es->groups_cap = 0; CUDA_TRY(es->set_group.alloc(set_group.size())); es->groups_cap = set_group.size(); }
    if ((size_t)eb.n_episodes > es->b_cap) {
        es->b_cap = 0;
        CUDA_TRY(alloc_each(eb.n_episodes, es->r_ret, es->logp));
        CUDA_TRY(alloc_each(eb.n_episodes, es->r_len, es->r_idx));
        CUDA_TRY(es->logits.alloc((size_t)eb.n_episodes * c.n_actions));
        es->b_cap = eb.n_episodes;
    }
    int32_t max_nodes;
    int64_t slot;
    if ((rc = pes_scratch(es, &max_nodes, &slot)) != RAMP_OK) return rc;
    std::vector<ModelDev> h(p->models.size());
    for (size_t m = 0; m < h.size(); ++m) h[m] = p->models[m].d;
    if (!idx.empty()) CUDA_TRY(cudaMemcpyAsync(es->r_idx.get(), idx.data(), sizeof(int32_t) * idx.size(), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(es->set_group.get(), set_group.data(), sizeof(int32_t) * set_group.size(), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(es->d_groups.get(), es->groups.data(), sizeof(EsPopGroup) * K, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(p->d_models.get(), h.data(), sizeof(ModelDev) * h.size(), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));                                   // the vectors are pageable
    EsPopArgs a{};
    a.n_models = c.n_models; a.b = b; a.groups = es->d_groups.get(); a.set_group = es->set_group.get(); a.pop = q->d_sets.get();
    a.theta = q->d_w.get(); a.noise = es->noise.get(); a.noise_index = es->r_idx.get(); a.sets = es->sets.get(); a.emb = es->emb.get();
    a.scratch = es->scratch.get(); a.slot_floats = slot; a.max_nodes = max_nodes;
    int64_t n_max = 0;
    for (const EsPopGroup& G : es->groups) n_max = std::max(n_max, G.n);
    ramp_pop_es_perturb_kernel<<<dim3((unsigned)std::min<int64_t>((n_max + 255) / 256, 64), (unsigned)es->n_sets), 256, 0, st>>>(a);
    const int32_t items = es->n_sets * c.n_models;
    ramp_pop_es_embed_kernel<<<(unsigned)std::min(es->embed_grid, items), 256, 0, st>>>(p->d_models.get(), a, items);
    CUDA_TRY(cudaGetLastError());
    ramp_internal_count_launches(eng, 2);
    return RAMP_OK;
}

int ramp_population_es_act(ramp_population_es_t* es, ramp_engine_t* eng, int32_t t) {
    if (!es || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (es->round < 0) return set_error(RAMP_ERR_BAD_ARG, "es: no round (ramp_population_es_round_begin)");
    ramp_env_buffers_t eb{};
    int rc = ramp_env_buffers(eng, &eb);
    if (rc != RAMP_OK) return rc;
    if (eb.n_episodes != es->B) return set_error(RAMP_ERR_BAD_ARG, "es: the round was begun on another environment");
    ramp_population* q = es->q;
    ramp_policy* p = q->p;
    CUDA_TRY(cudaSetDevice(p->device));
    for (int k = 0; k < es->K; ++k)
        if (es->groups[k].n_pairs) es->rec[k].seeds.push_back(mix64(es->groups[k].round_key ^ (2 * (uint64_t)(uint32_t)t + 1)));
    HeadArgs a{};
    a.obs_dyn = eb.obs_dynamic; a.graph_static = p->d_gstatic.get(); a.model = eb.queued_model; a.done = eb.done;
    a.mask = eb.action_mask; a.logits = es->logits.get(); a.logp = es->logp.get(); a.actions = eb.actions; a.sample = 1;
    EsPopArgs pa{};
    pa.b = es->b; pa.groups = es->d_groups.get(); pa.pop = q->d_sets.get(); pa.sets = es->sets.get(); pa.emb = es->emb.get();
    const int wpc = 8;
    const int cap = std::max(1, (4 * p->sm_count + es->K - 1) / es->K);     // about the single launch's 4 CTAs per SM in all
    const int gx = std::max(1, std::min((es->b + wpc - 1) / wpc, cap));
    ramp_pop_es_head_kernel<<<dim3(gx, es->K), wpc * 32, 0, ramp_internal_stream(eng)>>>(pa, a, t);
    CUDA_TRY(cudaGetLastError());
    ramp_internal_count_launches(eng, 1);
    return RAMP_OK;
}

int ramp_population_es_round_end(ramp_population_es_t* es, ramp_engine_t* eng, int32_t* more_out) {
    if (!es || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (es->round < 0) return set_error(RAMP_ERR_BAD_ARG, "es: no round (ramp_population_es_round_begin)");
    const double* ret; const int32_t* n_decided;
    int rc = ramp_internal_env_returns(eng, &ret, &n_decided);
    if (rc != RAMP_OK) return rc;
    ramp_env_buffers_t eb{};
    if ((rc = ramp_env_buffers(eng, &eb)) != RAMP_OK) return rc;
    if (eb.n_episodes != es->B) return set_error(RAMP_ERR_BAD_ARG, "es: the round was begun on another environment");
    CUDA_TRY(cudaSetDevice(es->q->p->device));
    cudaStream_t st = ramp_internal_stream(eng);
    const int32_t B = es->B, b = es->b;
    ramp_es_collect_kernel<<<(B + 255) / 256, 256, 0, st>>>(B, ret, n_decided, es->r_ret.get(), es->r_len.get());
    CUDA_TRY(cudaGetLastError());
    std::vector<float> r(B);
    std::vector<int32_t> l(B);
    CUDA_TRY(cudaMemcpyAsync(r.data(), es->r_ret.get(), sizeof(float) * B, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(l.data(), es->r_len.get(), sizeof(int32_t) * B, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    ramp_internal_count_launches(eng, 1);
    int32_t any = 0;
    for (int k = 0; k < es->K; ++k) {
        if (!es->groups[k].n_pairs) continue;                             // its twin's step ended before this round
        es_record_round(es->rec[k], r.data() + (size_t)k * b, l.data() + (size_t)k * b, 2 * es->groups[k].n_pairs, b);
        es->more[k] = es_more(es->rec[k], es->cfgs[k]) ? 1 : 0;
        any |= es->more[k];
    }
    if (more_out) *more_out = any;
    return RAMP_OK;
}

int ramp_population_es_step(ramp_population_es_t* es, const ramp_es_config_t* cfgs, double* stats_out) {
    int rc = pes_check_configs(es, cfgs);
    if (rc != RAMP_OK) return rc;
    for (int k = 0; k < es->K; ++k)
        if (es->rec[k].rounds < 1 || es->rec[k].ret.size() != es->rec[k].idx.size() * 2)
            return set_error(RAMP_ERR_BAD_ARG, "population: set %d: es: no complete round to learn from (ramp_population_es_round_begin / _end)", k);
    CUDA_TRY(cudaSetDevice(es->q->p->device));
    if ((rc = pes_update_records(es, cfgs, stats_out)) != RAMP_OK) return rc;
    es->iteration += 1;
    return RAMP_OK;
}

int ramp_population_es_update(ramp_population_es_t* es, const ramp_es_config_t* cfgs, const int32_t* n_pairs, const int32_t* noise_index,
                              const float* returns, double* stats_out) {
    int rc = pes_check_configs(es, cfgs);
    if (rc != RAMP_OK) return rc;
    if (!n_pairs || !noise_index || !returns) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if ((rc = pop_check_weights(es->q)) != RAMP_OK) return rc;
    int64_t o = 0;
    for (int k = 0; k < es->K; ++k) {
        if (n_pairs[k] < 1) return set_error(RAMP_ERR_BAD_ARG, "population: set %d: es: an update needs at least one pair, got %d", k, n_pairs[k]);
        const int64_t hi = es->noise_size - es->q->sets[k].n_w;
        for (int32_t i = 0; i < n_pairs[k]; ++i)
            if (noise_index[o + i] < 0 || (int64_t)noise_index[o + i] > hi)
                return set_error(RAMP_ERR_BAD_ARG, "population: set %d: es: noise index %d of pair %d outside [0, %lld]", k, noise_index[o + i], i,
                                 (long long)hi);
        o += n_pairs[k];
    }
    CUDA_TRY(cudaSetDevice(es->q->p->device));
    CUDA_TRY(cudaDeviceSynchronize());                                    // a round may still read theta
    o = 0;
    for (int k = 0; k < es->K; ++k) {
        es_host_record(es->rec[k], n_pairs[k], noise_index + o, returns + 2 * o);
        o += n_pairs[k];
    }
    return pes_update_records(es, cfgs, stats_out);
}

int ramp_population_es_read(ramp_population_es_t* es, int32_t set, int32_t* n_pairs_out, int32_t* n_eval_out, int32_t* n_seeds_out,
                            int32_t* noise_index_out, float* returns_out, int32_t* lengths_out, uint64_t* seeds_out, float* ranks_out,
                            float* grad_out, float* eval_returns_out, int32_t* eval_lengths_out) {
    if (!es) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = pop_check_set(es->q, set);
    if (rc != RAMP_OK) return rc;
    es_read_record(es->rec[set], n_pairs_out, n_eval_out, n_seeds_out, noise_index_out, returns_out, lengths_out, seeds_out, ranks_out,
                   eval_returns_out, eval_lengths_out);
    if (grad_out) {
        const PopSet& S = es->q->sets[set];
        CUDA_TRY(cudaSetDevice(es->q->p->device));
        CUDA_TRY(cudaDeviceSynchronize());
        CUDA_TRY(cudaMemcpy(grad_out, es->g.get() + S.w_off, sizeof(float) * (size_t)S.n_w, cudaMemcpyDeviceToHost));
    }
    return RAMP_OK;
}

int ramp_population_es_act_read(ramp_population_es_t* es, ramp_engine_t* eng, float* logits_out, float* logp_out, int32_t* actions_out) {
    if (!es || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    ramp_env_buffers_t eb{};
    int rc = ramp_env_buffers(eng, &eb);
    if (rc != RAMP_OK) return rc;
    if (es->b_cap < 1 || eb.n_episodes != es->B)
        return set_error(RAMP_ERR_BAD_ARG, "es: nothing to read (ramp_population_es_act was not called for this environment)");
    cudaStream_t st = ramp_internal_stream(eng);
    const size_t B = (size_t)es->B;
    if (logits_out) CUDA_TRY(cudaMemcpyAsync(logits_out, es->logits.get(), sizeof(float) * B * es->q->p->P.c.n_actions, cudaMemcpyDeviceToHost, st));
    if (logp_out) CUDA_TRY(cudaMemcpyAsync(logp_out, es->logp.get(), sizeof(float) * B, cudaMemcpyDeviceToHost, st));
    if (actions_out) CUDA_TRY(cudaMemcpyAsync(actions_out, eb.actions, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return RAMP_OK;
}

int ramp_population_es_state(ramp_population_es_t* es, int32_t set, float* m_out, float* v_out, int32_t* t_out) {
    if (!es) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = pop_check_set(es->q, set);
    if (rc != RAMP_OK) return rc;
    const PopSet& S = es->q->sets[set];
    CUDA_TRY(cudaSetDevice(es->q->p->device));
    CUDA_TRY(cudaDeviceSynchronize());
    if (m_out) CUDA_TRY(cudaMemcpy(m_out, es->m.get() + S.w_off, sizeof(float) * (size_t)S.n_w, cudaMemcpyDeviceToHost));
    if (v_out) CUDA_TRY(cudaMemcpy(v_out, es->v.get() + S.w_off, sizeof(float) * (size_t)S.n_w, cudaMemcpyDeviceToHost));
    if (t_out) *t_out = es->t[set];
    return RAMP_OK;
}

int ramp_population_es_reset(ramp_population_es_t* es) {
    if (!es) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    CUDA_TRY(cudaSetDevice(es->q->p->device));
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemset(es->m.get(), 0, sizeof(float) * (size_t)es->q->nw));
    CUDA_TRY(cudaMemset(es->v.get(), 0, sizeof(float) * (size_t)es->q->nw));
    es->t.assign(es->K, 0);
    return RAMP_OK;
}

int ramp_population_set_es_state(ramp_population_es_t* es, int32_t set, const float* m, const float* v, int64_t n, int32_t t) {
    if (!es || !m || !v) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = pop_check_set(es->q, set);
    if (rc != RAMP_OK) return rc;
    const PopSet& S = es->q->sets[set];
    if (n != S.n_w)
        return set_error(RAMP_ERR_BAD_ARG, "population: es: an Adam state of %lld weights given for set %d, its configuration has %lld", (long long)n, set,
                         (long long)S.n_w);
    if (t < 0) return set_error(RAMP_ERR_BAD_ARG, "population: set %d: es: Adam step count %d < 0", set, t);
    CUDA_TRY(cudaSetDevice(es->q->p->device));
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpy(es->m.get() + S.w_off, m, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(es->v.get() + S.w_off, v, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice));
    es->t[set] = t;
    return RAMP_OK;
}

int ramp_population_get_es_progress(ramp_population_es_t* es, int32_t set, int64_t* iteration_out, int32_t* n_rewards_out, double* rewards_out) {
    if (!es) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = pop_check_set(es->q, set);
    if (rc != RAMP_OK) return rc;
    es_get_progress(es->iteration, es->rec[set], iteration_out, n_rewards_out, rewards_out);
    return RAMP_OK;
}

int ramp_population_set_es_progress(ramp_population_es_t* es, int32_t set, int64_t iteration, int32_t n_rewards, const double* rewards) {
    if (!es) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = pop_check_set(es->q, set);
    if (rc != RAMP_OK) return rc;
    return es_set_progress(&es->iteration, es->rec[set], iteration, n_rewards, rewards);
}

int ramp_population_copy_es_sets(ramp_population_es_t* es, int32_t n_pairs, const int32_t* dst, const int32_t* src) {
    if (!es) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = pop_check_pairs(es->q, n_pairs, dst, src);
    if (rc != RAMP_OK || (rc = pop_copy_sets(es->q, n_pairs, dst, src, es->m.get(), es->v.get(), nullptr, nullptr)) != RAMP_OK) return rc;
    for (int i = 0; i < n_pairs; ++i) {
        es->t[dst[i]] = es->t[src[i]];
        es->rec[dst[i]].reward_list = es->rec[src[i]].reward_list;
    }
    return RAMP_OK;
}

int ramp_population_es_embed_ctas(ramp_population_es_t* es, int32_t* ctas_out, int32_t* items_out) {
    if (!es || !ctas_out || !items_out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (es->round < 0 && es->n_sets == 0) return set_error(RAMP_ERR_BAD_ARG, "es: no round yet (ramp_population_es_round_begin)");
    *items_out = es->n_sets * es->q->p->P.c.n_models;
    *ctas_out = std::min(es->embed_grid, *items_out);
    return RAMP_OK;
}

}  // extern "C"
